"""Host-side text helpers around the hot path (outside the timed region).

Restates /root/reference/src/inference.rs:276-313 (`parse_asr_output`, `capitalize_first`) and wraps the
HF `tokenizers` runtime like /root/reference/src/tokenizer.rs:4-50.  SURVEY.md section 8f-3.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence, Tuple


def capitalize_first(s: str) -> str:                       # inference.rs:307-313
    return s[:1].upper() + s[1:] if s else ""


def parse_asr_output(raw: str, language_forced: bool) -> Tuple[str, str]:
    """(language, text) from the decoded string.  inference.rs:276-305."""
    if language_forced:
        return "forced", raw.strip()
    raw = raw.strip()
    if raw.startswith("language "):
        rest = raw[len("language "):]
        pos = rest.find("<asr_text>")
        if pos >= 0:
            return rest[:pos].strip(), rest[pos + len("<asr_text>"):].strip()
        lang_end = 0
        for i, c in enumerate(rest):
            if c.isspace() or not c.isalpha():
                lang_end = i
                break
            lang_end = i + 1
        if lang_end > 0:
            return rest[:lang_end], rest[lang_end:].strip()
    return "unknown", raw


NO_SPACE_LANGUAGES = ("chinese", "japanese", "cantonese")   # written without spaces between words


def join_segment_texts(texts: List[str], language: Optional[str]) -> str:
    """The text of a segmented recording: the non-empty segment texts in order, joined with a space, or with nothing
    when `language` is Chinese, Japanese or Cantonese (case-insensitive)."""
    sep = "" if (language or "").strip().lower() in NO_SPACE_LANGUAGES else " "
    return sep.join(t for t in texts if t)


def majority_language(languages: List[str]) -> str:
    """The most frequent of `languages`, the first to appear on ties ("unknown" when empty)."""
    counts: dict = {}
    for lang in languages:
        counts[lang] = counts.get(lang, 0) + 1
    return max(counts, key=lambda k: counts[k]) if counts else "unknown"


class AsrTokenizer:
    """tokenizer.json wrapper (tokenizer.rs:4-50): encode without special tokens, decode skipping them."""

    def __init__(self, tok):
        self._tok = tok

    @classmethod
    def from_dir(cls, model_dir: str) -> "AsrTokenizer":
        path = os.path.join(model_dir, "tokenizer.json")
        if not os.path.exists(path):
            raise FileNotFoundError(
                f"tokenizer.json not found in {model_dir}; generate it with transformers.AutoTokenizer(...)"
                ".backend_tokenizer.save(...) as the reference's tokenizer.rs:22-31 instructs")
        from tokenizers import Tokenizer
        return cls(Tokenizer.from_file(path))

    def encode(self, text: str) -> List[int]:
        return list(self._tok.encode(text, add_special_tokens=False).ids)

    def decode(self, ids: List[int]) -> str:
        return self._tok.decode(list(ids), skip_special_tokens=True)

    def token_to_id(self, token: str) -> Optional[int]:
        return self._tok.token_to_id(token)


def language_prompt_ids(tokenizer: Optional[AsrTokenizer], language: Optional[str]) -> Optional[List[int]]:
    """ids of "language Xxx" appended to the prompt when the language is forced (inference.rs:246-250)."""
    if language is None:
        return None
    if tokenizer is None:
        raise ValueError("forcing a language needs tokenizer.json (to encode the prompt suffix)")
    return tokenizer.encode(f"language {capitalize_first(language)}")


def context_prompt_ids(tokenizer: Optional[AsrTokenizer], context: Optional[str]) -> Optional[List[int]]:
    """ids of the context text placed in the prompt's system turn (None or "": no context)."""
    if not context:
        return None
    if tokenizer is None:
        raise ValueError("a context needs tokenizer.json (to encode the text)")
    return tokenizer.encode(context)


# the languages of the Qwen3-ASR model card, as the model writes them after "language "; no name is a prefix of another
LANGUAGES = ("Chinese", "English", "Cantonese", "Arabic", "German", "French", "Spanish", "Portuguese", "Indonesian",
             "Italian", "Korean", "Russian", "Thai", "Vietnamese", "Japanese", "Turkish", "Hindi", "Malay", "Dutch",
             "Swedish", "Danish", "Finnish", "Polish", "Czech", "Filipino", "Persian", "Greek", "Hungarian",
             "Macedonian", "Romanian")


def language_probabilities(names: List[str], sum_logprobs: List[float]) -> List[Tuple[str, float]]:
    """(name, probability) sorted by probability (then by the order given): a softmax over the candidates' summed
    log-probabilities, in float64."""
    if len(names) != len(sum_logprobs) or not names:
        raise ValueError("need one summed log-probability per language")
    m = max(sum_logprobs)
    w = [math.exp(x - m) for x in sum_logprobs]
    z = sum(w)
    order = sorted(range(len(names)), key=lambda i: -w[i])
    return [(names[i], w[i] / z) for i in order]


# ---- words of a transcript (word timestamps, DESIGN.md 4.10) ----------------------------------------------------------
PREPEND_PUNCTUATION = "\"'“¿([{-"          # merged into the next word (Whisper's defaults)
APPEND_PUNCTUATION = "\"'.。,，!！?？:：”)]}、"   # merged into the previous word


@dataclass
class Word:
    start_s: float
    end_s: float
    text: str            # as decoded, with its leading space
    probability: float   # mean of its tokens' exp(log p)


def split_units(decode: Callable[[List[int]], str], ids: Sequence[int]) -> List[Tuple[str, List[int]]]:
    """ids grouped into the shortest runs that decode to complete characters (a byte-level token can hold part of
    one): (text, indices into ids) per run."""
    out, cur = [], []
    for k in range(len(ids)):
        cur.append(k)
        text = decode([ids[x] for x in cur])
        if "\ufffd" not in text:
            out.append((text, cur))
            cur = []
    if cur:
        out.append((decode([ids[x] for x in cur]), cur))
    return out


def merge_punctuation(words: List[Tuple[str, List[int]]]) -> List[Tuple[str, List[int]]]:
    """Whisper's merge_punctuations: a word that is a space and a prepend mark joins the next word; an append mark
    that follows a word not ending in a space joins it.  Emptied words are dropped."""
    w = [[t, list(ix)] for t, ix in words]
    i, j = len(w) - 2, len(w) - 1
    while i >= 0:
        if w[i][0].startswith(" ") and w[i][0].strip() in PREPEND_PUNCTUATION and w[i][0].strip():
            w[j][0] = w[i][0] + w[j][0]
            w[j][1] = w[i][1] + w[j][1]
            w[i][0], w[i][1] = "", []
        else:
            j = i
        i -= 1
    i, j = 0, 1
    while j < len(w):
        if not w[i][0].endswith(" ") and w[j][0] and w[j][0] in APPEND_PUNCTUATION:
            w[i][0] = w[i][0] + w[j][0]
            w[i][1] = w[i][1] + w[j][1]
            w[j][0], w[j][1] = "", []
        else:
            i = j
        j += 1
    return [(t, ix) for t, ix in w if ix]


def split_words(decode: Callable[[List[int]], str], ids: Sequence[int], language: Optional[str]) -> List[Tuple[str, List[int]]]:
    """The words of a transcript's ids as (text, indices into ids), in order.  For Chinese, Japanese and Cantonese
    (NO_SPACE_LANGUAGES) each run of complete characters is a word; otherwise a word starts at a run whose text begins
    with a space.  Then the punctuation is merged (merge_punctuation)."""
    units = split_units(decode, ids)
    if (language or "").strip().lower() in NO_SPACE_LANGUAGES:
        words = [(t, list(ix)) for t, ix in units]
    else:
        words = []
        for t, ix in units:
            if not words or t.startswith(" "):
                words.append((t, list(ix)))
            else:
                words[-1] = (words[-1][0] + t, words[-1][1] + list(ix))
    return merge_punctuation(words)


def build_words(decode: Callable[[List[int]], str], ids: Sequence[int], start_s: Sequence[float], eos_start_s: float,
                logprobs: Optional[Sequence[float]], language: Optional[str], offset_s: float = 0.0) -> List[Word]:
    """Words of the transcript ids (the aligned ids without the EOS): start_s[i] is id i's start; a word starts at its
    first id's start and ends at the next word's start, the last word at the EOS row's start (eos_start_s).  Its
    probability is the mean of its ids' exp(logprob) (NaN without logprobs).  Times are shifted by offset_s."""
    words = split_words(decode, ids, language)
    out = []
    for k, (text, ix) in enumerate(words):
        start = start_s[ix[0]]
        end = start_s[words[k + 1][1][0]] if k + 1 < len(words) else eos_start_s
        prob = (sum(math.exp(logprobs[i]) for i in ix) / len(ix)) if logprobs is not None else float("nan")
        out.append(Word(offset_s + start, offset_s + end, text, prob))
    return out
