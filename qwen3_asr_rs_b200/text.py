"""Host-side text helpers around the hot path (outside the timed region).

Restates /root/reference/src/inference.rs:276-313 (`parse_asr_output`, `capitalize_first`) and wraps the
HF `tokenizers` runtime like /root/reference/src/tokenizer.rs:4-50.  SURVEY.md section 8f-3.
"""
from __future__ import annotations

import math
import os
from typing import List, Optional, Tuple


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
