"""Host-side mirror of the reference's public API for the hot path.

Reference: ``AsrInference::{load, transcribe}`` (/root/reference/src/inference.rs:19-213).
``transcribe()`` steps 2-8 (inference.rs:94-200: samples -> mel -> encoder -> prompt ->
prefill -> greedy ids) run inside libasr_b200.so; step 1 (file decode / resample,
src/audio.rs) and step 9 (detokenise, src/tokenizer.rs) are outside the hot path, so the
entry points here take f32 16 kHz samples and return token ids.  All arithmetic happens
in the CUDA library through the C ABI (include/asr_b200.h); numpy is only the container
for host buffers.  No fallback exists: a missing library or GPU raises.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from contextlib import contextmanager
from dataclasses import dataclass, replace
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from .config import AsrConfig
from .text import Word, build_words

EOS_TOKEN_IDS = (151643, 151645)      # inference.rs:154
MAX_NEW_TOKENS = 4096                 # inference.rs:153
SCORE_SLOTS = 32                      # candidates (KV slots) per scoring call; more run in waves of whole utterances
EOS_ID = 151645                       # <|im_end|>
MEL_SAMPLE_RATE = 16000               # inference.rs:16

_DT = {"float32": 0, "bfloat16": 1, "float16": 2}


def _dims_struct(cfg: AsrConfig) -> _lib.AsrbDims:
    a, t = cfg.audio, cfg.text
    d = _lib.AsrbDims()
    for k in ("d_model", "encoder_layers", "encoder_attention_heads", "encoder_ffn_dim", "num_mel_bins",
              "max_source_positions", "n_window", "n_window_infer", "downsample_hidden_size", "output_dim"):
        setattr(d, k, int(getattr(a, k)))
    for k in ("vocab_size", "hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads",
              "num_key_value_heads", "head_dim"):
        setattr(d, k, int(getattr(t, k)))
    d.tie_word_embeddings = int(bool(t.tie_word_embeddings))
    d.rms_norm_eps = float(t.rms_norm_eps)
    d.rope_theta = float(t.rope_theta)
    return d


def avg_logprob(token_logprobs: Sequence[float], eos_logprob: Optional[float]) -> Optional[float]:
    """Mean log-probability of an utterance: over the generated tokens, plus the EOS token when generation ended on it
    (Whisper's `avg_logprob`); None when there is nothing to average."""
    vals = list(token_logprobs) + ([eos_logprob] if eos_logprob is not None else [])
    return sum(vals) / len(vals) if vals else None


def check_top_logprobs(top_logprobs) -> int:
    """The `top_logprobs` argument as an int in 0..8 (0: off), else ValueError."""
    if not isinstance(top_logprobs, (int, np.integer)) or isinstance(top_logprobs, bool) or not 0 <= top_logprobs <= 8:
        raise ValueError(f"top_logprobs must be an int in 0..8, got {top_logprobs!r}")
    return int(top_logprobs)


def check_temperature(temperature) -> Tuple[float, ...]:
    """The `temperature` argument as a schedule: a float, or a non-empty sequence of floats (a fallback schedule), each
    0 (greedy) or finite in [1e-6, 100], else ValueError."""
    ts = tuple(temperature) if isinstance(temperature, (list, tuple)) else (temperature,)
    if not ts:
        raise ValueError("temperature schedule must not be empty")
    for t in ts:
        if isinstance(t, bool) or not isinstance(t, (int, float, np.integer, np.floating)) or not math.isfinite(float(t)) \
                or not (float(t) == 0.0 or 1e-6 <= float(t) <= 100.0):
            raise ValueError(f"temperature must be 0 or a finite value in [1e-6, 100], got {t!r}")
    return tuple(float(t) for t in ts)


def check_seed(seed) -> int:
    """The `seed` argument as an int in [0, 2^64), else ValueError."""
    if not isinstance(seed, (int, np.integer)) or isinstance(seed, bool) or not 0 <= int(seed) < 1 << 64:
        raise ValueError(f"seed must be an int in [0, 2^64), got {seed!r}")
    return int(seed)


BEAM_MAX = 6


def check_beam(beam_size, length_penalty) -> Tuple[int, Optional[float]]:
    """The `beam_size` (an int in 1..6; 1: greedy) and `length_penalty` (None, or a finite value in [0, 10]) arguments,
    else ValueError."""
    if not isinstance(beam_size, (int, np.integer)) or isinstance(beam_size, bool) or not 1 <= beam_size <= BEAM_MAX:
        raise ValueError(f"beam_size must be an int in 1..{BEAM_MAX}, got {beam_size!r}")
    if length_penalty is not None:
        if isinstance(length_penalty, bool) or not isinstance(length_penalty, (int, float, np.integer, np.floating)) \
                or not math.isfinite(float(length_penalty)) or not 0.0 <= float(length_penalty) <= 10.0:
            raise ValueError(f"length_penalty must be None or a finite value in [0, 10], got {length_penalty!r}")
        length_penalty = float(length_penalty)
    return int(beam_size), length_penalty


def check_repetition(no_repeat_ngram_size, repetition_penalty) -> Tuple[int, float]:
    """The `no_repeat_ngram_size` (an int in 0..16; 0: off) and `repetition_penalty` (a finite value in [1, 10]; 1: off)
    arguments, validated."""
    n = no_repeat_ngram_size
    if not isinstance(n, (int, np.integer)) or isinstance(n, bool) or not 0 <= n <= 16:
        raise ValueError(f"no_repeat_ngram_size must be an int in 0..16, got {n!r}")
    p = repetition_penalty
    if isinstance(p, bool) or not isinstance(p, (int, float, np.integer, np.floating)) or not math.isfinite(float(p)) \
            or not 1.0 <= float(p) <= 10.0:
        raise ValueError(f"repetition_penalty must be a finite value in [1, 10], got {p!r}")
    return int(n), float(p)


def repetition_penalty_option(p: float) -> str:
    """The session option string of a repetition penalty: repr round-trips the double exactly."""
    return "1" if p == 1.0 else repr(float(p))


def length_penalty_option(a: Optional[float]) -> str:
    """The session option string of length penalty a (None: "none")."""
    return "none" if a is None else repr(float(a))


def beam_score(sum_logprob: float, n: int, length_penalty: Optional[float]) -> float:
    """A hypothesis's score: sum / P(n), P(n) = max(n, 1) without a length penalty, else ((5 + n) / 6) ** alpha (the
    library computes it in double from the fp32 sum)."""
    p = float(max(n, 1)) if length_penalty is None else ((5.0 + n) / 6.0) ** length_penalty
    return float(sum_logprob) / p


def rank_hypotheses(hyps: Sequence[Tuple[int, float]], length_penalty: Optional[float]) -> List[int]:
    """Indices of hypotheses (n ids, sum) given in admission order, ranked by (score descending, admission order)."""
    scores = [beam_score(sm, n, length_penalty) for n, sm in hyps]
    return sorted(range(len(hyps)), key=lambda i: (-scores[i], i))


def check_context_ids(context_ids, batch: int, vocab: int) -> Optional[List[Optional[List[int]]]]:
    """The `context_ids` argument: None, or one entry per utterance, each None or a sequence of ints in [0, vocab) (an
    empty one: no context), else ValueError.  Returns None or the entries as lists (None for no context)."""
    if context_ids is None:
        return None
    if isinstance(context_ids, (str, bytes)) or not isinstance(context_ids, Sequence) or len(context_ids) != batch:
        raise ValueError(f"context_ids must be None or one entry per utterance ({batch}), got {context_ids!r}")
    out: List[Optional[List[int]]] = []
    for c in context_ids:
        if c is None:
            out.append(None)
            continue
        if isinstance(c, (str, bytes)) or not isinstance(c, (Sequence, np.ndarray)):
            raise ValueError(f"a context must be None or a sequence of token ids, got {c!r}")
        ids = []
        for i in c:
            if isinstance(i, bool) or not isinstance(i, (int, np.integer)) or not 0 <= int(i) < vocab:
                raise ValueError(f"context ids must be ints in [0, {vocab}), got {i!r}")
            ids.append(int(i))
        out.append(ids or None)
    return out


def temperature_option(t: float) -> str:
    """The session option string of temperature t (a decimal the library parses exactly back to t)."""
    return "0" if t == 0.0 else repr(float(t))


def needs_fallback(token_logprobs: Sequence[float], eos_logprob: Optional[float],
                   logprob_threshold: Optional[float]) -> bool:
    """Whisper's fallback test without the compression-ratio criterion: the attempt stopped at max_new_tokens without EOS
    (eos_logprob None: a repetition loop, typically), or its avg_logprob is below the threshold (None: no such test)."""
    if eos_logprob is None:
        return True
    lp = avg_logprob(token_logprobs, eos_logprob)
    return logprob_threshold is not None and lp is not None and lp < logprob_threshold


def temperature_fallback(run: Callable[[List[int], float], "TranscribeIds"], n: int, temperatures: Sequence[float],
                         logprob_threshold: Optional[float]):
    """Temperature fallback over n utterances.  `run(indices, t)` decodes the utterances `indices` (ascending, one batch)
    at temperature t with the log-probability record on, and returns their TranscribeIds in that order.  All utterances
    run at temperatures[0]; those that need fallback (needs_fallback) run again, as one batch in their original order, at
    the next temperature, and so on.  Each utterance keeps its first accepted attempt, else its last one.
    Returns (per utterance (TranscribeIds, index in it), per utterance the temperature of the kept attempt, the runs)."""
    kept: List[Optional[Tuple["TranscribeIds", int]]] = [None] * n
    temps: List[Optional[float]] = [None] * n
    runs = []
    pending = list(range(n))
    for t in temperatures:
        if not pending:
            break
        r = run(pending, t)
        runs.append(r)
        retry = []
        for j, b in enumerate(pending):
            kept[b], temps[b] = (r, j), t
            if needs_fallback(r.logprobs[j], r.eos_logprobs[j], logprob_threshold):
                retry.append(b)
        pending = retry
    return kept, temps, runs


def _max_len(rows) -> int:
    """Length of the longest of `rows` (None entries count 0; None: 0)."""
    return max((len(r) for r in rows if r is not None), default=0) if rows is not None else 0


def check_segmenting(max_segment_s, search_s) -> Tuple[int, int]:
    """The `max_segment_s` / `search_s` arguments of transcribe_long as 16 kHz sample counts: each a whole number of
    10 ms, with max_segment_s >= 5 and 2 <= search_s <= max_segment_s / 2, else ValueError."""
    out = []
    for name, v in (("max_segment_s", max_segment_s), ("search_s", search_s)):
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(float(v)):
            raise ValueError(f"{name} must be a finite number of seconds, got {v!r}")
        n = int(round(float(v) * MEL_SAMPLE_RATE))
        if n % 160 or abs(n - float(v) * MEL_SAMPLE_RATE) > 1e-6 * max(1.0, n):
            raise ValueError(f"{name} must be a whole number of 10 ms, got {v!r}")
        out.append(n)
    max_seg, search = out
    if max_seg < 5 * MEL_SAMPLE_RATE or search < 2 * MEL_SAMPLE_RATE or 2 * search > max_seg:
        raise ValueError(f"need max_segment_s >= 5 and 2 <= search_s <= max_segment_s / 2, got {max_segment_s!r}, {search_s!r}")
    return max_seg, search


def default_search_s(max_segment_s: float) -> float:
    """The search window transcribe() and the CLI use with `max_segment_s`: 5 s, or half of it in whole 10 ms when
    that is shorter."""
    return min(5.0, math.floor(float(max_segment_s) * 100 / 2) / 100)


_PCM_FMT = {"int16": 0, "float32": 1, "int32": 2}


def _pcm_arrays(pcms) -> List[np.ndarray]:
    """PCM arrays as contiguous [frames, channels] of a supported dtype, else ValueError."""
    arrs = [np.ascontiguousarray(a if a.ndim == 2 else a.reshape(-1, 1)) for a in pcms]
    for a in arrs:
        if a.dtype.name not in _PCM_FMT:
            raise ValueError(f"PCM dtype must be int16 / int32 / float32, got {a.dtype}")
    return arrs


def _pcm_args(arrs: Sequence[np.ndarray], rates: Sequence[int]):
    """The per-file arrays of asrb_ingest_pcm / asrb_ingest_long: data pointers, frames, channels, rates, formats."""
    B = len(arrs)
    return ((C.c_void_p * B)(*[a.ctypes.data for a in arrs]), (C.c_int64 * B)(*[a.shape[0] for a in arrs]),
            (C.c_int32 * B)(*[a.shape[1] for a in arrs]), (C.c_int32 * B)(*[int(r) for r in rates]),
            (C.c_int32 * B)(*[_PCM_FMT[a.dtype.name] for a in arrs]))


# the library's value of every per-call session option (include/asr_b200.h)
_OPTION_DEFAULTS = {"logprobs": "0", "top_logprobs": "0", "temperature": "0", "seed": "0", "beam_size": "1",
                    "length_penalty": "none", "no_repeat_ngram_size": "0", "repetition_penalty": "1"}


def _decode_options(logprobs: bool, top_logprobs: int, temperature: Optional[float], seed: int,
                    beam: Optional[Tuple[int, Optional[float]]], rep: Tuple[int, float]) -> Dict[str, str]:
    """The session options of one decode call, in the order they are set: the records asked for, temperature and seed
    when sampling (temperature not None), beam_size and, for K > 1, length_penalty (beam = (K, length penalty); None:
    neither), and the repetition controls rep = (N, penalty)."""
    opts = {}
    if logprobs:
        opts["logprobs"] = "1"
    if top_logprobs:
        opts["top_logprobs"] = str(top_logprobs)
    if temperature is not None:
        opts.update(temperature=temperature_option(temperature), seed=str(seed))
    if beam is not None:
        opts["beam_size"] = str(beam[0])
        if beam[0] > 1:
            opts["length_penalty"] = length_penalty_option(beam[1])
    opts.update(no_repeat_ngram_size=str(rep[0]), repetition_penalty=repetition_penalty_option(rep[1]))
    return opts


@dataclass
class _Audio:
    """The audio of one call's items, in one of three forms, so that the transcribe, score and align bodies need not
    know which: "ids" = host f32 clips at 16 kHz; "ingested" = PCM arrays at `rates`, brought to mono 16 kHz on the GPU
    (asrb_ingest_pcm); "segments" = (file, start, end) views into the session's long-audio buffer.  `lang` / `ctx`: per
    item its language ids and its context (for a segment, those of its file; None: none for every item)."""
    form: str
    items: list
    rates: Optional[list] = None
    lang: Optional[list] = None
    ctx: Optional[list] = None

    def __len__(self) -> int:
        return len(self.items)

    def subset(self, idx: Sequence[int]) -> "_Audio":
        """The items `idx`, in that order."""
        pick = (lambda xs: None if xs is None else [xs[i] for i in idx])
        return _Audio(self.form, pick(self.items), pick(self.rates), pick(self.lang), pick(self.ctx))

    def prepare(self, eng: "AsrInference", slots: int, max_new: int):
        """Make the engine's session ready for these items and return it.  Clips and PCM grow it to max(items, slots)
        KV slots and `max_new` ids, and PCM is ingested; segment views keep the session as it is, since re-creating it
        would drop the long-audio buffer."""
        B = len(self.items)
        langs, lptrs, llens, mx = eng._pack_lang(self.lang, B)
        if self.form == "ids":
            arrs, ptrs, lens = eng._pack_samples(self.items)
            s = eng._ensure_session(max(B, slots), max(a.shape[0] for a in arrs), mx, max_new, _max_len(self.ctx))
            lead = (ptrs, lens, B)
        elif self.form == "ingested":
            s, arrs, _ = eng._ingest(self.items, self.rates, mx, max_new, slots, _max_len(self.ctx))
            lead = ()
        else:
            s, arrs = eng._session, None
            lead = (B, (C.c_int32 * B)(*[f for f, _, _ in self.items]), (C.c_int64 * B)(*[a for _, a, _ in self.items]),
                    (C.c_int64 * B)(*[b for _, _, b in self.items]))
        self._keep = (arrs, langs)                   # the host arrays the pointers below refer to
        self._args = (s, *lead, lptrs, llens)
        return s

    def call(self, lib, family: str, *rest) -> int:
        """asrb_<family>_<form> (family: transcribe, score or align) on the prepared items; returns its status."""
        return getattr(lib, f"asrb_{family}_{self.form}")(*self._args, *rest)


def _concat_runs(runs: Sequence["TranscribeIds"]) -> "TranscribeIds":
    """The TranscribeIds of consecutive waves as one: per-utterance fields concatenated, times and counters summed."""
    if len(runs) == 1:
        return runs[0]
    r = TranscribeIds(sum((x.ids for x in runs), []), {}, sum(x.kernels_launched for x in runs),
                      sum(x.decode_steps for x in runs))
    for x in runs:
        for name, ms in x.stage_ms.items():
            r.stage_ms[name] = r.stage_ms.get(name, 0.0) + ms
    for field in ("logprobs", "eos_logprobs", "top_logprobs", "eos_top_logprobs", "nbest"):
        if getattr(runs[0], field) is not None:
            setattr(r, field, sum((getattr(x, field) for x in runs), []))
    return r


@dataclass
class TranscribeResult:           # inference.rs:270-274
    text: str
    language: str
    raw_output: str
    ids: List[int]
    token_logprobs: Optional[List[float]] = None    # transcribe(logprobs=True): log p of each id
    avg_logprob: Optional[float] = None             # avg_logprob(token_logprobs, EOS log p)
    # transcribe(top_logprobs=k): per id, the k best candidates of its step as (id, log p), best first (entry 0 = the id)
    top_logprobs: Optional[List[List[Tuple[int, float]]]] = None
    eos_top_logprobs: Optional[List[Tuple[int, float]]] = None   # ... of the step that selected EOS (None: stopped by the cap)
    temperature: Optional[float] = None             # transcribe(temperature=...): that of the kept attempt
    nbest: Optional[List[Tuple[str, float]]] = None   # transcribe(beam_size=K > 1): the K hypotheses as (text, score), ranked
    # transcribe(max_segment_s=...): the segments as (start_s, end_s, text), in time order
    segments: Optional[List[Tuple[float, float, str]]] = None
    # transcribe(word_timestamps=True): the words of the transcript with their times (text.Word), in order
    words: Optional[List["Word"]] = None


@dataclass
class LongSegment:
    """One segment of a long recording (transcribe_long): its time span, ids and the per-utterance fields of
    TranscribeIds for it."""
    start_s: float
    end_s: float
    ids: List[int]
    logprobs: Optional[List[float]] = None
    eos_logprob: Optional[float] = None
    top_logprobs: Optional[List[List[Tuple[int, float]]]] = None
    eos_top_logprobs: Optional[List[Tuple[int, float]]] = None
    temperature: Optional[float] = None
    nbest: Optional[List[Tuple[List[int], float, float, int]]] = None
    words: Optional[List["Word"]] = None            # word_timestamps=True: times absolute in the file


@dataclass
class LongResult:
    files: List[List[LongSegment]]   # per file, its segments in time order
    stage_ms: Dict[str, float]       # device time per stage, summed over the waves
    kernels_launched: int
    decode_steps: int
    n_segments: int
    n_waves: int                     # asrb_transcribe_segments calls, fallback re-runs included


@dataclass
class TranscribeIds:
    ids: List[List[int]]          # generated ids per utterance, EOS excluded
    stage_ms: Dict[str, float]    # device time per stage (CUDA events)
    kernels_launched: int
    decode_steps: int
    logprobs: Optional[List[List[float]]] = None         # logprobs=True: natural-log probability of each id
    eos_logprobs: Optional[List[Optional[float]]] = None  # ... of the EOS id that ended the utterance (None: stopped at max_new_tokens)
    # top_logprobs=k: per utterance, per id, the k best candidates of the step that selected it as (id, log p), best first
    top_logprobs: Optional[List[List[List[Tuple[int, float]]]]] = None
    # ... of the step that selected the EOS ending the utterance (None: stopped at max_new_tokens)
    eos_top_logprobs: Optional[List[Optional[List[Tuple[int, float]]]]] = None
    # temperature=T or a schedule: per utterance, the temperature of the attempt kept (None for a plain greedy call)
    temperatures: Optional[List[float]] = None
    # beam_size=K > 1: per utterance, its K hypotheses ranked as (ids, sum_logprob, score, eos_id; -1 = stopped by the
    # cap); entry 0 is `ids` (None for an attempt that sampled)
    nbest: Optional[List[Optional[List[Tuple[List[int], float, float, int]]]]] = None


@dataclass
class ScoredCandidate:
    """One scored continuation: `logprobs[i]` = log p(ids[i] | prompt, ids[:i]); with top_logprobs = k, the k best
    (id, log p) of every position and `greedy_prefix`, the number of leading ids that are the top-1 of their position."""
    ids: List[int]
    logprobs: List[float]
    sum_logprob: float
    top_logprobs: Optional[List[List[Tuple[int, float]]]] = None
    greedy_prefix: Optional[int] = None


def check_candidates(candidates, batch: int, vocab: int) -> List[List[List[int]]]:
    """candidates[b]: a non-empty list of non-empty id lists per utterance, every id in [0, vocab)."""
    if len(candidates) != batch:
        raise ValueError(f"need one candidate list per utterance: {len(candidates)} for {batch}")
    out = []
    for b, cands in enumerate(candidates):
        if not cands:
            raise ValueError(f"utterance {b} has no candidate")
        rows = []
        for c in cands:
            ids = [int(i) for i in c]
            if not ids:
                raise ValueError(f"utterance {b}: an empty candidate")
            if any(i < 0 or i >= vocab for i in ids):
                raise ValueError(f"utterance {b}: candidate id out of [0, {vocab})")
            rows.append(ids)
        out.append(rows)
    return out


@dataclass
class Alignment:
    """Word-timing alignment of one utterance (asrb_align_ids): entry k is id text_from + k of the aligned ids, its start
    and end in 10 ms mel frames (the end is the next id's start, the last id's the utterance's frame count)."""
    text_from: int
    start_frames: List[int]
    end_frames: List[int]

    @property
    def start_s(self) -> List[float]:
        return [f * FRAME_S for f in self.start_frames]

    @property
    def end_s(self) -> List[float]:
        return [f * FRAME_S for f in self.end_frames]


FRAME_S = 0.01                  # one mel frame: 160 samples at 16 kHz


def check_align_ids(ids, text_from, batch: int, vocab: int) -> Tuple[List[List[int]], List[int]]:
    """ids[b]: a non-empty id list per utterance, every id in [0, vocab); text_from: None (all 0) or one int per
    utterance in [0, len(ids[b]) - 1]."""
    if len(ids) != batch:
        raise ValueError(f"need one id list per utterance: {len(ids)} for {batch}")
    rows = [[int(i) for i in r] for r in ids]
    for b, r in enumerate(rows):
        if not r:
            raise ValueError(f"utterance {b}: no ids to align")
        if any(i < 0 or i >= vocab for i in r):
            raise ValueError(f"utterance {b}: id out of [0, {vocab})")
    tf = [0] * batch if text_from is None else [int(f) for f in text_from]
    if len(tf) != batch or any(not 0 <= f < len(r) for f, r in zip(tf, rows)):
        raise ValueError("text_from must be None or one index per utterance in [0, len(ids[b]) - 1]")
    return rows, tf


def check_alignment_heads(heads, layers: int, nq: int) -> List[Tuple[int, int]]:
    """None -> [] (the library's default: every head of the second half of the layers); else distinct (layer, head)
    pairs inside the model."""
    if heads is None:
        return []
    out = [(int(l), int(h)) for l, h in heads]
    if not out:
        raise ValueError("alignment_heads must be None or a non-empty list of (layer, head) pairs")
    if any(not (0 <= l < layers and 0 <= h < nq) for l, h in out) or len(set(out)) != len(out):
        raise ValueError(f"alignment_heads: distinct (layer, head) pairs with layer < {layers} and head < {nq}")
    return out


def text_start(ids: Sequence[int], asr_text_id: Optional[int]) -> int:
    """Index of the first transcript id: just after the <asr_text> id when it occurs, else 0."""
    if asr_text_id is not None and asr_text_id in ids:
        return list(ids).index(asr_text_id) + 1
    return 0


def score_waves(n_cand: Sequence[int], slots: int) -> List[List[int]]:
    """Utterance indices per call: whole utterances in order, at most max(slots, the largest n_cand) candidates each."""
    cap = max([slots] + list(n_cand))
    waves, cur, used = [], [], 0
    for b, n in enumerate(n_cand):
        if cur and used + n > cap:
            waves.append(cur)
            cur, used = [], 0
        cur.append(b)
        used += n
    if cur:
        waves.append(cur)
    return waves


class AsrInference:
    """``AsrInference`` of the reference, hot path only, batch-capable."""

    def __init__(self, cfg: AsrConfig, ctx, model):
        self.config = cfg
        self._lib = _lib.load_library()
        self._ctx, self._model = ctx, model
        self._session = None
        self._cap = None
        self._options: Dict[str, str] = {}
        self.tokenizer = None     # text.AsrTokenizer when model_dir has tokenizer.json

    # ---- construction ------------------------------------------------------------
    @staticmethod
    def _init_ctx(device: int):
        lib = _lib.load_library()
        ctx = C.c_void_p()
        _lib.check(lib.asrb_init(int(device), C.byref(ctx)))
        return lib, ctx

    @classmethod
    def load(cls, model_dir: str, device: int = 0) -> "AsrInference":
        """AsrInference::load (inference.rs:30-86): config.json + safetensors from ``model_dir``."""
        lib, ctx = cls._init_ctx(device)
        model = C.c_void_p()
        _lib.check(lib.asrb_model_load(ctx, os.fsencode(model_dir), C.byref(model)))
        d = _lib.AsrbDims()
        _lib.check(lib.asrb_model_dims(model, C.byref(d)))
        cfg = AsrConfig.from_file(os.path.join(model_dir, "config.json"))
        eng = cls(cfg, ctx, model)
        if os.path.exists(os.path.join(model_dir, "tokenizer.json")):
            from .text import AsrTokenizer
            eng.tokenizer = AsrTokenizer.from_dir(model_dir)
        return eng

    @classmethod
    def from_weights(cls, cfg: AsrConfig, weights: Dict[str, "object"], device: int = 0) -> "AsrInference":
        """Build from in-memory tensors (name -> torch tensor or numpy array) -- what load()
        does after reading safetensors (weights.rs:62-120).  bf16 torch tensors pass through
        bit-exactly."""
        lib, ctx = cls._init_ctx(device)
        model = C.c_void_p()
        dims = _dims_struct(cfg)
        _lib.check(lib.asrb_model_create(ctx, C.byref(dims), C.byref(model)))
        for name, t in weights.items():
            if hasattr(t, "detach"):          # torch tensor
                import torch
                t = t.detach().cpu().contiguous()
                if t.dtype == torch.bfloat16:
                    arr, code = t.view(torch.int16).numpy(), 1
                elif t.dtype == torch.float16:
                    arr, code = t.view(torch.int16).numpy(), 2
                else:
                    arr, code = t.to(torch.float32).numpy(), 0
            else:
                arr = np.ascontiguousarray(t, dtype=np.float32)
                code = 0
            shape = (C.c_int64 * arr.ndim)(*arr.shape)
            _lib.check(lib.asrb_model_set_tensor(model, name.encode(), code, shape, arr.ndim,
                                                 arr.ctypes.data_as(C.c_void_p)))
        _lib.check(lib.asrb_model_finalize(model))
        return cls(cfg, ctx, model)

    def close(self) -> None:
        if self._session is not None:
            self._lib.asrb_session_free(self._session)
            self._session = None
        if self._model is not None:
            self._lib.asrb_model_free(self._model)
            self._model = None
        if self._ctx is not None:
            self._lib.asrb_ctx_free(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- session management ----------------------------------------------------------
    def set_option(self, key: str, value: str) -> None:
        self._options[key] = value
        if self._session is not None:
            _lib.check(self._lib.asrb_session_set_option(self._session, key.encode(), value.encode()))

    def device_ids(self):
        """(ids_ptr, lens_ptr, row_stride, batch): device addresses of the last generated ids (asrb_session_device_ids)."""
        ids, lens = C.c_void_p(), C.c_void_p()
        stride, batch = C.c_int(), C.c_int()
        _lib.check(self._lib.asrb_session_device_ids(self._session, C.byref(ids), C.byref(lens), C.byref(stride), C.byref(batch)))
        return ids.value, lens.value, stride.value, batch.value

    def stats(self) -> Dict[str, int]:
        """Decoder-forward / GEMM path counters (asrb_session_stats): fallbacks are visible, never silent."""
        out = (C.c_int64 * 8)()
        if self._session is None:
            return {}
        _lib.check(self._lib.asrb_session_stats(self._session, out, 8))
        return dict(zip(("decode_batch_steps", "decode_fused_steps", "decode_phase_steps", "gemm_simt_fallbacks",
                         "gemm_tc_launches", "lmhead_rows_recomputed", "lmhead_step_max_recomputed",
                         "lmhead_full_fallbacks"), [int(v) for v in out]))

    def _ensure_session(self, batch: int, max_samples: int, max_lang: int, max_new: int, max_context: int = 0):
        cap = self._cap
        if cap is None or batch > cap[0] or max_samples > cap[1] or max_lang > cap[2] or max_new > cap[3] \
                or max_context > cap[4]:
            if self._session is not None:
                _lib.check(self._lib.asrb_session_free(self._session))
                self._session, self._cap = None, None        # a refused create below leaves no session, not a stale capacity
            new_cap = (max(batch, cap[0] if cap else 0), max(max_samples, cap[1] if cap else 0),
                       max(max_lang, cap[2] if cap else 0), max(max_new, cap[3] if cap else 0),
                       max(max_context, cap[4] if cap else 0))
            s = C.c_void_p()
            _lib.check(self._lib.asrb_session_create_ex(self._model, new_cap[0], new_cap[1], new_cap[2], new_cap[4],
                                                        new_cap[3], C.byref(s)))
            self._session, self._cap = s, new_cap
            for k, v in self._options.items():
                _lib.check(self._lib.asrb_session_set_option(s, k.encode(), v.encode()))
        return self._session

    @staticmethod
    def _pack_samples(clips: Sequence[np.ndarray]):
        arrs = [np.ascontiguousarray(c, dtype=np.float32) for c in clips]
        ptrs = (C.POINTER(C.c_float) * len(arrs))(*[a.ctypes.data_as(C.POINTER(C.c_float)) for a in arrs])
        lens = (C.c_int64 * len(arrs))(*[a.shape[0] for a in arrs])
        return arrs, ptrs, lens

    @staticmethod
    def _pack_lang(language_ids, batch):
        if language_ids is None:
            return None, None, None, 0
        keep, ptrs, lens, mx = [], [], [], 0
        for ids in language_ids:
            if ids is None:
                ptrs.append(C.POINTER(C.c_int64)())
                lens.append(0)
            else:
                a = np.ascontiguousarray(ids, dtype=np.int64)
                keep.append(a)
                ptrs.append(a.ctypes.data_as(C.POINTER(C.c_int64)))
                lens.append(len(a))
                mx = max(mx, len(a))
        return keep, (C.POINTER(C.c_int64) * batch)(*ptrs), (C.c_int32 * batch)(*lens), mx

    # ---- context biasing (asrb_session_set_context) ------------------------------------------------------
    def set_context(self, context_ids) -> None:
        """asrb_session_set_context on the current session: None clears the contexts; else one entry per utterance of
        the next runs (None or an empty sequence: no context), or a single entry for all of them.  For the stage-level
        calls; transcribe_ids / transcribe_pcm / transcribe set their own contexts for the call."""
        if not context_ids:
            _lib.check(self._lib.asrb_session_set_context(self._session, 0, None, None))
            return
        keep, ptrs, lens, _ = self._pack_lang(context_ids, len(context_ids))
        _lib.check(self._lib.asrb_session_set_context(self._session, len(context_ids), ptrs, lens))

    @contextmanager
    def _call_scope(self, s, options: Dict[str, str], context_ids=None):
        """One call on session s with `options` and, unless None, `context_ids` (as set_context).  An option is set
        only where it differs from the engine's configured value (the library default when none is configured), since
        setting one drops the captured per-phase step graph.  On exit, also on an exception, the context is cleared
        and every option set goes back to that value.  Results that depend on the options are read inside the scope."""
        undo = []
        try:
            for key, val in options.items():
                conf = self._options.get(key, _OPTION_DEFAULTS[key])
                if conf != val:
                    _lib.check(self._lib.asrb_session_set_option(s, key.encode(), val.encode()))
                    undo.append((key, conf))
            if context_ids is not None:
                keep, ptrs, lens, _ = self._pack_lang(context_ids, len(context_ids))
                _lib.check(self._lib.asrb_session_set_context(s, len(context_ids), ptrs, lens))
            yield
        finally:
            if context_ids is not None:
                _lib.check(self._lib.asrb_session_set_context(s, 0, None, None))
            for key, conf in undo:
                _lib.check(self._lib.asrb_session_set_option(s, key.encode(), conf.encode()))

    def _last_batch(self) -> Tuple[int, int]:
        """(the session's batch capacity, the utterances of its last run) for the asrb_last_* reads; AsrbError
        (ASRB_ERR_STATE) before anything has run."""
        if self._session is None:
            raise _lib.AsrbError(4, "no session: nothing has run yet")
        return self._cap[0], getattr(self, "_B", self._cap[0])

    def last_prefill_stats(self) -> Dict[str, int]:
        """asrb_last_prefill_stats: rows computed, rows taken from a leader's shared context, KV bytes fanned out."""
        out = (C.c_int64 * 3)()
        _lib.check(self._lib.asrb_last_prefill_stats(self._session, out, 3))
        return dict(zip(("rows_computed", "rows_shared", "fanout_kv_bytes"), [int(v) for v in out]))

    # ---- per-token log-probabilities (session option "logprobs") ----------------------------
    def last_logprobs(self, max_new_tokens: int):
        """asrb_last_logprobs: (per-utterance log-probabilities of the ids of the last run, EOS log-probability or None).
        Raises AsrbError (ASRB_ERR_STATE) when the last run did not record them."""
        cap, B = self._last_batch()                          # the library writes one row per utterance of the last run
        lp = np.full((cap, max_new_tokens), np.nan, dtype=np.float32)
        eos = np.full(cap, np.nan, dtype=np.float32)
        _lib.check(self._lib.asrb_last_logprobs(self._session, int(max_new_tokens), lp.ctypes.data_as(C.POINTER(C.c_float)),
                                                eos.ctypes.data_as(C.POINTER(C.c_float))))
        rows = []
        for r in lp[:B]:                                     # each row: the finite prefix (NaN from the utterance's length on)
            nan = np.flatnonzero(np.isnan(r))
            rows.append([float(v) for v in r[: nan[0] if len(nan) else len(r)]])
        return rows, [None if np.isnan(e) else float(e) for e in eos[:B]]

    # ---- top-k alternatives (session option "top_logprobs") ------------------------------------
    def last_top_logprobs(self, max_new_tokens: int, k: int):
        """asrb_last_top_logprobs: (per utterance, per id of the last run, the k best candidates of its step as
        (id, log p) pairs, best first; per utterance the same for the step that selected the ending EOS, or None).
        Raises AsrbError: ASRB_ERR_STATE when the last run did not record them, ASRB_ERR_INVALID when k is outside
        [1, the recorded top_logprobs]."""
        cap, B = self._last_batch()
        ids = np.full((cap, max_new_tokens, max(k, 1)), -1, dtype=np.int32)
        lp = np.full(ids.shape, np.nan, dtype=np.float32)
        eids = np.full((cap, max(k, 1)), -1, dtype=np.int32)
        elp = np.full(eids.shape, np.nan, dtype=np.float32)
        _lib.check(self._lib.asrb_last_top_logprobs(
            self._session, int(max_new_tokens), int(k), ids.ctypes.data_as(C.POINTER(C.c_int32)),
            lp.ctypes.data_as(C.POINTER(C.c_float)), eids.ctypes.data_as(C.POINTER(C.c_int32)),
            elp.ctypes.data_as(C.POINTER(C.c_float))))
        rows = []
        for b in range(B):                                   # the rows before the utterance's length (-1 from there on)
            n = int(np.count_nonzero(ids[b, :, 0] >= 0))
            rows.append([[(int(i), float(v)) for i, v in zip(ids[b, t], lp[b, t])] for t in range(n)])
        eos = [None if eids[b, 0] < 0 else [(int(i), float(v)) for i, v in zip(eids[b], elp[b])] for b in range(B)]
        return rows, eos

    # ---- beam search (session options "beam_size" / "length_penalty") ------------------------------------------
    def last_nbest(self, max_new_tokens: int, k: int):
        """asrb_last_nbest: per utterance of the last beam run, its k best hypotheses ranked as (ids, sum_logprob,
        score, eos_id; -1 = stopped by the cap).  Raises AsrbError: ASRB_ERR_STATE when the last run was not a beam
        run, ASRB_ERR_INVALID when k is outside [1, beam_size]."""
        _, B = self._last_batch()
        kk = max(int(k), 1)
        ids = np.full((B, kk, max_new_tokens), -1, dtype=np.int32)
        lens = np.zeros((B, kk), dtype=np.int32)
        sums = np.zeros((B, kk), dtype=np.float32)
        scores = np.zeros((B, kk), dtype=np.float32)
        eos = np.zeros((B, kk), dtype=np.int32)
        P = C.POINTER
        _lib.check(self._lib.asrb_last_nbest(self._session, int(max_new_tokens), int(k), ids.ctypes.data_as(P(C.c_int32)),
                                             lens.ctypes.data_as(P(C.c_int32)), sums.ctypes.data_as(P(C.c_float)),
                                             scores.ctypes.data_as(P(C.c_float)), eos.ctypes.data_as(P(C.c_int32))))
        return [[(ids[b, j, : lens[b, j]].tolist(), float(sums[b, j]), float(scores[b, j]), int(eos[b, j])) for j in range(kk)]
                for b in range(B)]

    def last_beam_stats(self) -> Dict[str, int]:
        """asrb_last_beam_stats: counters of the last beam run."""
        out = (C.c_int64 * 4)()
        _lib.check(self._lib.asrb_last_beam_stats(self._session, out, 4))
        return dict(zip(("beam_steps", "slots_reassigned", "expand_kv_bytes", "reorder_kv_bytes"), [int(v) for v in out]))

    def _finish(self, s, B: int, ids, n, max_new_tokens: int, logprobs: bool, top_logprobs: int = 0,
                beam_size: int = 1) -> TranscribeIds:
        ms = (C.c_float * 6)()
        k, st = C.c_int64(), C.c_int64()
        _lib.check(self._lib.asrb_last_timings(s, ms, C.byref(k), C.byref(st)))
        names = ("h2d", "mel", "encoder", "prefill", "decode", "total")
        r = TranscribeIds([ids[b, : n[b]].tolist() for b in range(B)], dict(zip(names, ms)), k.value, st.value)
        self._B = B
        if logprobs or top_logprobs:
            r.logprobs, r.eos_logprobs = self.last_logprobs(max_new_tokens)
        if top_logprobs:
            r.top_logprobs, r.eos_top_logprobs = self.last_top_logprobs(max_new_tokens, top_logprobs)
        if beam_size > 1:
            r.nbest = self.last_nbest(max_new_tokens, beam_size)
        return r

    # ---- seeded temperature sampling (session options "temperature" / "seed") ---------------------------
    def _sampled(self, B: int, once, temperature, seed, logprob_threshold, logprobs: bool, top_logprobs: int,
                 beam_size: int = 1, length_penalty: Optional[float] = None) -> TranscribeIds:
        """One call of transcribe_ids / transcribe_pcm.  `once(indices, logprobs, top_logprobs, t, beam)` runs the
        utterances `indices` at temperature t (None: the session's configured options) with beam = (K, length penalty)
        (None: greedy or sampling).  With a schedule, attempts at t = 0 run the beam search and attempts at t > 0
        sample, as in Whisper."""
        top_logprobs = check_top_logprobs(top_logprobs)
        temps = check_temperature(temperature)
        seed = check_seed(seed)
        beam_size, length_penalty = check_beam(beam_size, length_penalty)
        schedule = isinstance(temperature, (list, tuple))
        if top_logprobs and any(t > 0.0 for t in temps):
            raise ValueError("temperature > 0 cannot be combined with top_logprobs")
        if beam_size > 1 and top_logprobs:
            raise ValueError("beam_size > 1 cannot be combined with top_logprobs")
        if beam_size > 1 and not schedule and temps[0] > 0.0:
            raise ValueError("beam_size > 1 cannot be combined with temperature > 0 (a schedule runs the beam at t = 0)")
        beam = (beam_size, length_penalty) if beam_size > 1 else None
        if not schedule and temps[0] == 0.0:                 # plain greedy / beam call: the session's options as configured
            return once(list(range(B)), logprobs, top_logprobs, None, beam)
        if not schedule:
            r = once(list(range(B)), logprobs, 0, temps[0], None)
            r.temperatures = [temps[0]] * B
            return r
        kept, used, runs = temperature_fallback(lambda idx, t: once(idx, True, 0, t, beam if t == 0.0 else None), B, temps,
                                                logprob_threshold)
        r = TranscribeIds([k[0].ids[k[1]] for k in kept], {}, sum(x.kernels_launched for x in runs),
                          sum(x.decode_steps for x in runs))
        for x in runs:
            for name, ms in x.stage_ms.items():
                r.stage_ms[name] = r.stage_ms.get(name, 0.0) + ms
        r.logprobs = [k[0].logprobs[k[1]] for k in kept]
        r.eos_logprobs = [k[0].eos_logprobs[k[1]] for k in kept]
        r.temperatures = used
        if beam is not None:
            r.nbest = [k[0].nbest[k[1]] if k[0].nbest is not None else None for k in kept]
        return r

    # ---- the hot path ----------------------------------------------------------------
    def transcribe_ids(self, clips: Sequence[np.ndarray], language_ids: Optional[Sequence] = None,
                       max_new_tokens: int = MAX_NEW_TOKENS, logprobs: bool = False, top_logprobs: int = 0,
                       temperature: Union[float, Sequence[float]] = 0.0, seed: int = 0,
                       logprob_threshold: Optional[float] = -1.0, beam_size: int = 1,
                       length_penalty: Optional[float] = None, context_ids: Optional[Sequence] = None,
                       no_repeat_ngram_size: int = 0, repetition_penalty: float = 1.0) -> TranscribeIds:
        """transcribe() steps 2-8 for a batch: host f32 samples in, host token ids out (and, with `logprobs`, the
        log-probability of every id and of the ending EOS, from the kernels that selected them; with `top_logprobs` = k
        in 1..8, also the k best candidates of each of those steps, and the log-probabilities as with `logprobs`).
        `temperature` T > 0 samples every id with the seeded Gumbel-max draw of the kernels (ids are a pure function of
        the inputs, `seed`, T and the batch order); a sequence of temperatures is a fallback schedule
        (temperature_fallback) with the log-probability record on and `logprob_threshold` (None: off).
        `beam_size` K in 2..6 decodes every utterance with beam search (the session holds batch x K slots; `nbest`
        holds the K ranked hypotheses, `ids` the best) scored with `length_penalty` (None: sum / length); with a
        schedule, only the attempts at t = 0 use it.  `context_ids`: None, or per utterance None or the token ids of
        its context, placed in the prompt's system turn; utterances with identical contexts share its prefill.
        `no_repeat_ngram_size` N >= 1 bans every id that would repeat an N-gram of the ids generated so far, and
        `repetition_penalty` > 1 divides the positive (multiplies the negative) logits of ids generated so far, in every
        attempt, beam and path (include/asr_b200.h); the prompt and context never count."""
        return self._transcribe(_Audio("ids", clips, None, language_ids), max_new_tokens, logprobs, top_logprobs,
                                temperature, seed, logprob_threshold, beam_size, length_penalty, context_ids,
                                no_repeat_ngram_size, repetition_penalty)

    def _transcribe(self, src: _Audio, max_new_tokens: int, logprobs: bool, top_logprobs: int, temperature, seed: int,
                    logprob_threshold: Optional[float], beam_size: int, length_penalty: Optional[float], context_ids,
                    no_repeat_ngram_size: int, repetition_penalty: float) -> TranscribeIds:
        """transcribe_ids / transcribe_pcm on the items of `src`."""
        src = replace(src, ctx=check_context_ids(context_ids, len(src), self.config.text.vocab_size))
        rep = check_repetition(no_repeat_ngram_size, repetition_penalty)
        return self._sampled(len(src), lambda idx, lp, k, t, beam: self._run(src.subset(idx), max_new_tokens, lp, k, t,
                                                                             seed, beam, rep),
                             temperature, seed, logprob_threshold, logprobs, top_logprobs, beam_size, length_penalty)

    def _run(self, src: _Audio, max_new_tokens: int, logprobs: bool, top_logprobs: int, temperature: Optional[float],
             seed: int, beam, rep: Tuple[int, float]) -> TranscribeIds:
        """One decode call of the items of `src` at `temperature` (None: the session's configured options) with
        beam = (K, length penalty) (None: greedy or sampling) and rep = (N, penalty)."""
        B, K = len(src), beam[0] if beam else 1
        s = src.prepare(self, B * K, max_new_tokens)
        ids = np.zeros((B, max_new_tokens), dtype=np.int32)
        n = np.zeros(B, dtype=np.int32)
        with self._call_scope(s, _decode_options(logprobs, top_logprobs, temperature, seed, beam or (1, None), rep),
                              src.ctx):
            _lib.check(src.call(self._lib, "transcribe", int(max_new_tokens), ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                n.ctypes.data_as(C.POINTER(C.c_int32))))
            return self._finish(s, B, ids, n, max_new_tokens, logprobs, top_logprobs, K)

    # ---- streaming (asrb_stream_*) ------------------------------------------------------------------------------------
    def open_streams(self, n: int, max_seconds: float, language: Optional[str] = None, context: Optional[str] = None,
                     rollback: int = 5, unfixed_pushes: int = 2, max_new_tokens: int = 32, language_ids=None,
                     context_ids=None, logprobs: bool = False, top_logprobs: int = 0, temperature: float = 0.0,
                     seed: int = 0, no_repeat_ngram_size: int = 0, repetition_penalty: float = 1.0):
        """n live streams of up to `max_seconds` each (stream.StreamSet): push(samples_per_stream, final=...) returns
        every stream's hypothesis of the audio received so far, decoded with the previous hypothesis less its last
        `rollback` ids forced as a prefix (after `unfixed_pushes` pushes); `max_new_tokens` per push.  `language` /
        `context` need tokenizer.json; `language_ids` / `context_ids` give the ids directly.  The session's
        max_lang_ids is the language ids plus a forced prefix of stream.PREFIX_IDS_PER_SECOND ids per second of
        `max_seconds` plus max_new_tokens (stream.stream_max_lang_ids); a push whose language ids and prefix outgrow it
        is refused (ASRB_ERR_INVALID, the streams intact: finish the stream and open the next).  Any other
        call on this engine ends the streams."""
        from .stream import StreamSet
        from .text import context_prompt_ids, language_prompt_ids
        if self._options.get("beam_size", "1") != "1":
            raise ValueError("beam search is not available on streams (the engine's beam_size option is set)")
        lang = language_ids if language_ids is not None else language_prompt_ids(self.tokenizer, language)
        ctx = context_ids if context_ids is not None else context_prompt_ids(self.tokenizer, context)
        return StreamSet(self, int(n), float(max_seconds), lang, ctx, int(rollback), int(unfixed_pushes), int(max_new_tokens),
                         logprobs, top_logprobs, temperature, seed, no_repeat_ngram_size, repetition_penalty)

    # ---- teacher-forced scoring (asrb_score_ids) --------------------------------------------------------------------
    def score_ids(self, clips: Sequence[np.ndarray], candidates: Sequence[Sequence[Sequence[int]]],
                  language_ids: Optional[Sequence] = None, context_ids: Optional[Sequence] = None,
                  top_logprobs: int = 0) -> List[List[ScoredCandidate]]:
        """Log-probability of every id of every candidate continuation, from one teacher-forced prefill per call:
        `candidates[b]` lists id sequences for clip b, each scored after the prompt transcribe_ids builds (language ids
        and context included).  The candidates of a clip share its prompt's prefill.  With `top_logprobs` = k in 1..8,
        also the k best ids of every position and the greedy prefix.  More candidates than SCORE_SLOTS run in several
        calls of whole utterances."""
        return self._score_waves(_Audio("ids", clips, None, language_ids), candidates, context_ids, top_logprobs)

    def score_pcm(self, pcms: Sequence, rates: Sequence[int], candidates: Sequence[Sequence[Sequence[int]]],
                  language_ids: Optional[Sequence] = None, context_ids: Optional[Sequence] = None,
                  top_logprobs: int = 0) -> List[List[ScoredCandidate]]:
        """score_ids with step 1 on the GPU: raw PCM in (as transcribe_pcm)."""
        return self._score_waves(_Audio("ingested", pcms, rates, language_ids), candidates, context_ids, top_logprobs)

    def _score_waves(self, src: _Audio, candidates, context_ids, top_logprobs: int) -> List[List[ScoredCandidate]]:
        """score_ids / score_pcm on the items of `src`: one _score call per wave of whole utterances."""
        B = len(src)
        cands = check_candidates(candidates, B, self.config.text.vocab_size)
        k = check_top_logprobs(top_logprobs)
        src = replace(src, ctx=check_context_ids(context_ids, B, self.config.text.vocab_size))
        out: List[List[ScoredCandidate]] = [None] * B
        for wave in score_waves([len(c) for c in cands], SCORE_SLOTS):
            for b, r in zip(wave, self._score(src.subset(wave), [cands[b] for b in wave], k)):
                out[b] = r
        return out

    def _score(self, src: _Audio, cands: List[List[List[int]]], k: int) -> List[List[ScoredCandidate]]:
        """One scoring call: cands[b] = the candidates of item b of `src`."""
        flat = [c for cs in cands for c in cs]
        N = len(flat)
        max_new = max(len(c) for c in flat)
        s = src.prepare(self, N, max_new)
        n_cand = (C.c_int32 * len(cands))(*[len(cs) for cs in cands])
        arrs = [np.ascontiguousarray(c, dtype=np.int64) for c in flat]
        cptrs = (C.POINTER(C.c_int64) * N)(*[a.ctypes.data_as(C.POINTER(C.c_int64)) for a in arrs])
        clens = (C.c_int32 * N)(*[len(c) for c in flat])
        lp = np.empty((N, max_new), dtype=np.float32)
        tid = np.empty((N, max_new, max(k, 1)), dtype=np.int32)
        tlp = np.empty((N, max_new, max(k, 1)), dtype=np.float32)
        with self._call_scope(s, {"top_logprobs": str(k)} if k else {}, src.ctx):
            _lib.check(src.call(self._lib, "score", n_cand, cptrs, clens, int(max_new),
                                lp.ctypes.data_as(C.POINTER(C.c_float)),
                                tid.ctypes.data_as(C.POINTER(C.c_int32)) if k else None,
                                tlp.ctypes.data_as(C.POINTER(C.c_float)) if k else None))
        res, q = [], 0
        for cs in cands:
            row = []
            for c in cs:
                n = len(c)
                lps = [float(v) for v in lp[q, :n]]
                sc = ScoredCandidate(ids=list(c), logprobs=lps, sum_logprob=float(np.sum(np.asarray(lps, np.float64))))
                if k:
                    sc.top_logprobs = [[(int(tid[q, i, j]), float(tlp[q, i, j])) for j in range(k)] for i in range(n)]
                    g = 0
                    while g < n and sc.top_logprobs[g][0][0] == c[g]:
                        g += 1
                    sc.greedy_prefix = g
                row.append(sc)
                q += 1
            res.append(row)
        return res

    def score(self, audio_path: str, texts: Sequence[str], language: Optional[str] = None, context: Optional[str] = None,
              eos: bool = True, top_logprobs: int = 0) -> List[ScoredCandidate]:
        """Score transcripts of one WAV file: each text is tokenised (tokenizer.json) and, with `eos`, followed by
        <|im_end|>, so that its log-probability includes ending there.  `language` / `context`: the prompt of
        transcribe(language=..., context=...)."""
        from .audio import read_wav_pcm
        from .text import context_prompt_ids, language_prompt_ids
        if self.tokenizer is None:
            raise ValueError("scoring text needs tokenizer.json")
        lang_ids = language_prompt_ids(self.tokenizer, language)
        ctx_ids = context_prompt_ids(self.tokenizer, context)
        cands = [self.tokenizer.encode(t) + ([EOS_ID] if eos else []) for t in texts]
        pcm, rate = read_wav_pcm(audio_path)
        return self.score_pcm([pcm], [rate], [cands], language_ids=[lang_ids] if lang_ids is not None else None,
                              context_ids=[ctx_ids] if ctx_ids else None, top_logprobs=top_logprobs)[0]

    def detect_language(self, audio_path: str, languages: Sequence[str] = None) -> List[Tuple[str, float]]:
        """Language identification over a closed set: every `language_prompt_ids(tok, name)` continuation ("language
        Xxx") is one candidate of the one utterance, all sharing its prompt's prefill.  Returns (name, probability)
        best first, the probabilities a softmax over the candidates' summed log-probabilities.  The sums are
        comparable without a terminator token only because no name of the set is a prefix of another (true of
        text.LANGUAGES): a name that prefixed another would score its own ids and not its ending."""
        from .audio import read_wav_pcm
        from .text import LANGUAGES, language_probabilities, language_prompt_ids
        names = list(LANGUAGES if languages is None else languages)
        if self.tokenizer is None:
            raise ValueError("language identification needs tokenizer.json")
        cands = [language_prompt_ids(self.tokenizer, n) for n in names]
        pcm, rate = read_wav_pcm(audio_path)
        r = self.score_pcm([pcm], [rate], [cands])[0]
        return language_probabilities(names, [c.sum_logprob for c in r])

    # ---- word-timing alignment (asrb_align_ids, DESIGN.md 4.10) ---------------------------------------------------
    def align_ids(self, clips: Sequence[np.ndarray], ids: Sequence[Sequence[int]], text_from: Optional[Sequence[int]] = None,
                  language_ids: Optional[Sequence] = None, context_ids: Optional[Sequence] = None,
                  alignment_heads: Optional[Sequence[Tuple[int, int]]] = None) -> List[Alignment]:
        """Start and end of every id ids[b][text_from[b]:] in clip b, from the decoder's attention over the audio in one
        teacher-forced pass over the prompt transcribe_ids builds (language ids and context included) and ids[b]
        (normally the decoded ids followed by EOS).  `alignment_heads`: (layer, query head) pairs, None = every head of
        the second half of the layers.  More clips than SCORE_SLOTS run in several calls."""
        return self._align_checked(_Audio("ids", clips, None, language_ids), ids, text_from, context_ids, alignment_heads)

    def align_pcm(self, pcms: Sequence, rates: Sequence[int], ids: Sequence[Sequence[int]],
                  text_from: Optional[Sequence[int]] = None, language_ids: Optional[Sequence] = None,
                  context_ids: Optional[Sequence] = None,
                  alignment_heads: Optional[Sequence[Tuple[int, int]]] = None) -> List[Alignment]:
        """align_ids with step 1 on the GPU: raw PCM in (as transcribe_pcm)."""
        return self._align_checked(_Audio("ingested", pcms, rates, language_ids), ids, text_from, context_ids,
                                   alignment_heads)

    def _align_checked(self, src: _Audio, ids, text_from, context_ids, alignment_heads) -> List[Alignment]:
        """align_ids / align_pcm on the items of `src`, SCORE_SLOTS per call."""
        t = self.config.text
        rows, tf = check_align_ids(ids, text_from, len(src), t.vocab_size)
        heads = check_alignment_heads(alignment_heads, t.num_hidden_layers, t.num_attention_heads)
        src = replace(src, ctx=check_context_ids(context_ids, len(src), t.vocab_size))
        return self._align_waves(src, rows, tf, heads, SCORE_SLOTS)

    def _align_waves(self, src: _Audio, rows: List[List[int]], tf: List[int], heads: List[Tuple[int, int]],
                     per_call: int) -> List[Alignment]:
        """Alignments of the items of `src` (ids rows[b] from tf[b] on), in calls of `per_call` items."""
        out: List[Alignment] = []
        for w0 in range(0, len(rows), per_call):
            wrows, wtf = rows[w0:w0 + per_call], tf[w0:w0 + per_call]
            sub = src.subset(range(w0, w0 + len(wrows)))
            s = sub.prepare(self, len(wrows), max(len(r) for r in wrows))
            out += self._align(s, wrows, wtf, heads, sub.ctx, lambda *a: sub.call(self._lib, "align", *a))
        return out

    def _align(self, s, rows: List[List[int]], tf: List[int], heads: List[Tuple[int, int]], context_ids,
               call) -> List[Alignment]:
        """One alignment call on session s: `call(ids, n_ids, text_from, heads, n_heads, max_ids, start, end)`."""
        B = len(rows)
        max_ids = max(len(r) for r in rows)
        arrs = [np.ascontiguousarray(r, dtype=np.int64) for r in rows]
        iptrs = (C.POINTER(C.c_int64) * B)(*[a.ctypes.data_as(C.POINTER(C.c_int64)) for a in arrs])
        n_ids = (C.c_int32 * B)(*[len(r) for r in rows])
        tfa = (C.c_int32 * B)(*tf)
        harr = np.ascontiguousarray(np.array(heads, dtype=np.int32).reshape(-1, 2))
        st = np.empty((B, max_ids), dtype=np.int32)
        en = np.empty((B, max_ids), dtype=np.int32)
        with self._call_scope(s, {}, context_ids):
            _lib.check(call(iptrs, n_ids, tfa, harr.ctypes.data_as(C.POINTER(C.c_int32)) if heads else None, len(heads),
                            int(max_ids), st.ctypes.data_as(C.POINTER(C.c_int32)), en.ctypes.data_as(C.POINTER(C.c_int32))))
        self._B = B
        return [Alignment(f, [int(v) for v in st[b, f:len(r)]], [int(v) for v in en[b, f:len(r)]])
                for b, (r, f) in enumerate(zip(rows, tf))]

    def last_align_matrix(self, b: int) -> np.ndarray:
        """M [N_b][T_b] of utterance b of the last alignment call (asrb_align_matrix_read): the head-mean of the
        normalised, filtered audio attention that the DTW ran on.  For choosing alignment heads on a checkpoint."""
        n, t = C.c_int32(), C.c_int32()
        _lib.check(self._lib.asrb_last_align_dims(self._session, int(b), C.byref(n), C.byref(t)))
        a = np.empty((n.value, t.value), dtype=np.float32)
        _lib.check(self._lib.asrb_align_matrix_read(self._session, int(b), a.ctypes.data_as(C.POINTER(C.c_float))))
        return a

    def _asr_text_id(self) -> Optional[int]:
        return self.tokenizer.token_to_id("<asr_text>") if self.tokenizer is not None else None

    def _decode_fn(self):
        return self.tokenizer.decode if self.tokenizer is not None else (lambda ids: "".join(f" {i}" for i in ids))

    def _word_language(self, ids: List[int], language: Optional[str]) -> Optional[str]:
        """The language that decides the word split: the tag the decoded ids carry, else `language`."""
        if self.tokenizer is not None:
            from .text import parse_asr_output
            tag = parse_asr_output(self.tokenizer.decode(ids), False)[0]
            if tag != "unknown":
                return tag
        return language

    def _words(self, ids: List[int], al: Alignment, logprobs: Optional[List[float]], language: Optional[str],
               offset_s: float = 0.0) -> List[Word]:
        """Words of a decoded id list whose ids + [EOS] were aligned from al.text_from on."""
        f = al.text_from
        text = ids[f:]
        lp = logprobs[f:] if logprobs is not None else None
        return build_words(self._decode_fn(), text, al.start_s[:len(text)], al.start_s[len(text)], lp, language, offset_s)

    # ---- GPU-side audio ingest (step 1, src/audio.rs:162-245) -------------------------------------------
    def _ingest(self, pcms: Sequence, rates: Sequence[int], max_lang: int, max_new: int, slots: int = 0,
                max_context: int = 0):
        arrs = _pcm_arrays(pcms)
        B = len(arrs)
        n_out = [-(-a.shape[0] * MEL_SAMPLE_RATE // int(r)) for a, r in zip(arrs, rates)]
        s = self._ensure_session(max(B, slots), max(n_out), max_lang, max_new, max_context)
        n = (C.c_int64 * B)()
        _lib.check(self._lib.asrb_ingest_pcm(s, *_pcm_args(arrs, rates), B, n))
        return s, arrs, list(n)

    def ingest_pcm(self, pcms: Sequence, rates: Sequence[int]) -> List[np.ndarray]:
        """asrb_ingest_pcm + read-back (tests): interleaved PCM arrays [frames, channels] -> mono f32 @ 16 kHz, on the GPU."""
        s, _keep, n = self._ingest(pcms, rates, 16, 64)
        out = []
        for b in range(len(pcms)):
            a = np.empty(n[b], dtype=np.float32)
            _lib.check(self._lib.asrb_ingested_read(s, b, a.ctypes.data_as(C.POINTER(C.c_float))))
            out.append(a)
        return out

    def transcribe_pcm(self, pcms: Sequence, rates: Sequence[int], language_ids: Optional[Sequence] = None,
                       max_new_tokens: int = MAX_NEW_TOKENS, logprobs: bool = False, top_logprobs: int = 0,
                       temperature: Union[float, Sequence[float]] = 0.0, seed: int = 0,
                       logprob_threshold: Optional[float] = -1.0, beam_size: int = 1,
                       length_penalty: Optional[float] = None, context_ids: Optional[Sequence] = None,
                       no_repeat_ngram_size: int = 0, repetition_penalty: float = 1.0) -> TranscribeIds:
        """transcribe() steps 1-8 for a batch with step 1 on the GPU: raw PCM in, token ids out (`logprobs`,
        `top_logprobs`, `temperature`, `seed`, `logprob_threshold`, `beam_size`, `length_penalty`, `context_ids`,
        `no_repeat_ngram_size`, `repetition_penalty`: as in transcribe_ids)."""
        return self._transcribe(_Audio("ingested", pcms, rates, language_ids), max_new_tokens, logprobs, top_logprobs,
                                temperature, seed, logprob_threshold, beam_size, length_penalty, context_ids,
                                no_repeat_ngram_size, repetition_penalty)

    # ---- long-form audio: cut at low-energy points on the GPU, decode the pieces in waves -----------------------
    def ingest_long(self, pcms: Sequence, rates: Sequence[int]) -> List[np.ndarray]:
        """asrb_ingest_long + asrb_long_read (tests): interleaved PCM arrays [frames, channels] -> mono f32 @ 16 kHz in
        the session's long-audio buffer, read back."""
        s, n = self._ingest_long(pcms, rates, self._ensure_session(1, 16000, 0, 1))
        self._long_files = len(n)
        out = []
        for f, m in enumerate(n):
            a = np.empty(m, dtype=np.float32)
            _lib.check(self._lib.asrb_long_read(s, f, a.ctypes.data_as(C.POINTER(C.c_float))))
            out.append(a)
        return out

    def _ingest_long(self, pcms: Sequence, rates: Sequence[int], s):
        arrs = _pcm_arrays(pcms)
        n = (C.c_int64 * len(arrs))()
        _lib.check(self._lib.asrb_ingest_long(s, *_pcm_args(arrs, rates), len(arrs), n))
        return s, list(n)

    def segment_long(self, max_segment_samples: int, search_samples: int) -> List[List[Tuple[int, int]]]:
        """asrb_segment_long on the files of the last ingest: per file, its segments as (start, end) sample offsets."""
        s = self._session
        n_files = self._long_files
        cap = 64 * n_files
        while True:
            nseg = (C.c_int32 * n_files)()
            st, en = (C.c_int64 * cap)(), (C.c_int64 * cap)()
            code = self._lib.asrb_segment_long(s, int(max_segment_samples), int(search_samples), cap, nseg, st, en)
            if code == 1 and sum(nseg) > cap:                # did not fit: the counts are filled, retry with room
                cap = sum(nseg)
                continue
            _lib.check(code)
            break
        out, o = [], 0
        for f in range(n_files):
            out.append([(int(st[o + k]), int(en[o + k])) for k in range(nseg[f])])
            o += nseg[f]
        return out

    def transcribe_long(self, pcms: Sequence, rates: Sequence[int], max_segment_s: float = 30.0, search_s: float = 5.0,
                        batch: int = 16, language_ids: Optional[Sequence] = None, max_new_tokens: int = MAX_NEW_TOKENS,
                        logprobs: bool = False, top_logprobs: int = 0,
                        temperature: Union[float, Sequence[float]] = 0.0, seed: int = 0,
                        logprob_threshold: Optional[float] = -1.0, beam_size: int = 1,
                        length_penalty: Optional[float] = None, context_ids: Optional[Sequence] = None,
                        no_repeat_ngram_size: int = 0, repetition_penalty: float = 1.0, word_timestamps: bool = False,
                        alignment_heads: Optional[Sequence[Tuple[int, int]]] = None,
                        language: Optional[str] = None) -> "LongResult":
        """Long recordings: ingest the files (raw PCM, as transcribe_pcm) into the long-audio buffer, cut them on the GPU
        into segments of at most `max_segment_s` at the quietest 100 ms window of the last `search_s` before each limit
        (asrb_segment_long), and decode the segments as views of that buffer (asrb_transcribe_segments) in waves of
        `batch` segments in (file, time) order, `batch // beam_size` with a beam.  `max_new_tokens` applies per segment.
        Every other keyword is that of transcribe_pcm, per segment: the language ids and context of a file apply to each
        of its segments; temperature fallback re-runs only the failing segments, in waves of their own.
        `word_timestamps`: also align every segment's decoded ids + EOS in place (asrb_align_segments, waves of `batch`)
        and fill LongSegment.words with times absolute in the file; it records log-probabilities for the word
        probabilities.  `alignment_heads` as in align_ids; `language`: the forced language's name, which decides how
        words are split (text.split_words) when the ids carry no language tag.
        Returns per file its segments in time order."""
        max_seg, search = check_segmenting(max_segment_s, search_s)
        n_files = len(pcms)
        if len(rates) != n_files or n_files < 1:
            raise ValueError("pcms and rates must be non-empty and of equal length")
        if isinstance(batch, bool) or not isinstance(batch, (int, np.integer)) or batch < 1:
            raise ValueError(f"batch must be an int >= 1, got {batch!r}")
        tk = check_top_logprobs(top_logprobs)
        check_temperature(temperature)
        check_seed(seed)
        K, _ = check_beam(beam_size, length_penalty)
        rep = check_repetition(no_repeat_ngram_size, repetition_penalty)
        if batch // K < 1:
            raise ValueError(f"batch ({batch}) must be >= beam_size ({K})")
        ctx = check_context_ids(context_ids, n_files, self.config.text.vocab_size)
        arrs = _pcm_arrays(pcms)
        if language_ids is not None and len(language_ids) != n_files:
            raise ValueError("language_ids must be None or one entry per file")
        longest = max(-(-a.shape[0] * MEL_SAMPLE_RATE // int(r)) for a, r in zip(arrs, rates))
        mx = _max_len(language_ids)
        # word timestamps align the decoded ids and the EOS: one id more than the decode's cap
        s = self._ensure_session(batch, min(max_seg, max(longest, 201)), mx, max_new_tokens + int(bool(word_timestamps)),
                                 _max_len(ctx))
        s, n = self._ingest_long(arrs, rates, s)
        self._long_files = n_files
        cuts = self.segment_long(max_seg, search)
        segs = [(f, a, b) for f in range(n_files) for a, b in cuts[f]]
        src = _Audio("segments", segs, None, None if language_ids is None else [language_ids[f] for f, _, _ in segs],
                     None if ctx is None else [ctx[f] for f, _, _ in segs])
        n_waves = 0

        def once(idx, lp, k, t, beam):
            nonlocal n_waves
            W = batch // (beam[0] if beam else 1)
            runs = []
            for w0 in range(0, len(idx), W):
                runs.append(self._run(src.subset(idx[w0:w0 + W]), max_new_tokens, lp, k, t, seed, beam, rep))
                n_waves += 1
            return _concat_runs(runs)
        heads = check_alignment_heads(alignment_heads, self.config.text.num_hidden_layers,
                                      self.config.text.num_attention_heads) if word_timestamps else []
        r = self._sampled(len(segs), once, temperature, seed, logprob_threshold, logprobs or word_timestamps, tk, beam_size,
                          length_penalty)
        als: List[Alignment] = []
        if word_timestamps:
            asr_text = self._asr_text_id()
            als = self._align_waves(src, [ids + [EOS_ID] for ids in r.ids], [text_start(ids, asr_text) for ids in r.ids],
                                    heads, batch)
        out: List[List[LongSegment]] = [[] for _ in range(n_files)]
        for i, (f, a, b) in enumerate(segs):
            seg = LongSegment(a / MEL_SAMPLE_RATE, b / MEL_SAMPLE_RATE, r.ids[i])
            if r.logprobs is not None:
                seg.logprobs, seg.eos_logprob = r.logprobs[i], r.eos_logprobs[i]
            if r.top_logprobs is not None:
                seg.top_logprobs, seg.eos_top_logprobs = r.top_logprobs[i], r.eos_top_logprobs[i]
            if r.temperatures is not None:
                seg.temperature = r.temperatures[i]
            if r.nbest is not None:
                seg.nbest = r.nbest[i]
            if word_timestamps:
                seg.words = self._words(r.ids[i], als[i], r.logprobs[i], self._word_language(r.ids[i], language),
                                        a / MEL_SAMPLE_RATE)
            out[f].append(seg)
        return LongResult(out, r.stage_ms, r.kernels_launched, r.decode_steps, len(segs), n_waves)

    def transcribe(self, audio_path: str, language: Optional[str] = None,
                   max_new_tokens: int = MAX_NEW_TOKENS, gpu_ingest: bool = True, logprobs: bool = False,
                   top_logprobs: int = 0, temperature: Union[float, Sequence[float]] = 0.0, seed: int = 0,
                   logprob_threshold: Optional[float] = -1.0, beam_size: int = 1,
                   length_penalty: Optional[float] = None, context: Optional[str] = None,
                   max_segment_s: Optional[float] = None, no_repeat_ngram_size: int = 0,
                   repetition_penalty: float = 1.0, word_timestamps: bool = False,
                   alignment_heads: Optional[Sequence[Tuple[int, int]]] = None) -> TranscribeResult:
        """AsrInference::transcribe (inference.rs:89-213): step 1 (WAV payload -> mono 16 kHz; on the GPU by default,
        `gpu_ingest=False` = the host loader) -> steps 2-8 on the GPU -> step 9 (detokenise + parse, host; needs
        tokenizer.json, else raw_output is the id list as text).  `logprobs`: also fill token_logprobs / avg_logprob;
        `top_logprobs` = k in 1..8: also fill top_logprobs (and token_logprobs / avg_logprob); `temperature`, `seed`,
        `logprob_threshold`, `beam_size`, `length_penalty`, `no_repeat_ngram_size`, `repetition_penalty`: as in
        transcribe_ids, and `temperature` of the result is that
        of the kept attempt; `nbest` holds the beam's hypotheses as (text, score).  `context`: text placed in the prompt's
        system turn to bias recognition (keywords, names, related text; needs tokenizer.json; "" = none).
        `max_segment_s`: None decodes the file in one pass; a number of seconds runs transcribe_long with it (search
        window min(5 s, half of it, in whole 10 ms)) and `max_new_tokens` per segment: see _long_result.
        `word_timestamps`: also fill `words` (text.Word: start, end, text, probability) by aligning the kept
        hypothesis + EOS from just after its <asr_text> id (align_ids; per segment with `max_segment_s`), with
        `alignment_heads` as in align_ids; it records log-probabilities for the word probabilities."""
        from .audio import load_wav, read_wav_pcm
        from .text import context_prompt_ids, language_prompt_ids, parse_asr_output
        lang_ids = language_prompt_ids(self.tokenizer, language)
        ctx_ids = context_prompt_ids(self.tokenizer, context)
        lang = [lang_ids] if lang_ids is not None else None
        ctx = [ctx_ids] if ctx_ids else None
        sampling = dict(temperature=temperature, seed=seed, logprob_threshold=logprob_threshold, beam_size=beam_size,
                        length_penalty=length_penalty, context_ids=ctx, no_repeat_ngram_size=no_repeat_ngram_size,
                        repetition_penalty=repetition_penalty)
        # checked before the file is read; transcribe_long checks them after its own arguments
        heads = check_alignment_heads(alignment_heads, self.config.text.num_hidden_layers,
                                      self.config.text.num_attention_heads) if word_timestamps and max_segment_s is None else None
        pcm, rate = read_wav_pcm(audio_path) if gpu_ingest else (load_wav(audio_path, MEL_SAMPLE_RATE), MEL_SAMPLE_RATE)
        if max_segment_s is not None:
            lr = self.transcribe_long([pcm], [rate], max_segment_s=max_segment_s, search_s=default_search_s(max_segment_s),
                                      language_ids=lang, max_new_tokens=max_new_tokens, logprobs=logprobs,
                                      top_logprobs=top_logprobs, word_timestamps=word_timestamps,
                                      alignment_heads=alignment_heads, language=language, **sampling)
            return self._long_result(lr.files[0], language, logprobs, top_logprobs)
        src = _Audio("ingested", [pcm], [rate], lang) if gpu_ingest else _Audio("ids", [pcm], None, lang)
        r = self._transcribe(src, max_new_tokens=max_new_tokens, logprobs=logprobs or word_timestamps,
                             top_logprobs=top_logprobs, **sampling)
        ids = r.ids[0]
        al = None
        if word_timestamps:
            al = self._align_checked(src, [ids + [EOS_ID]], [text_start(ids, self._asr_text_id())], ctx, heads or None)[0]

        def parse(ids):
            raw = self.tokenizer.decode(ids) if self.tokenizer is not None else " ".join(str(i) for i in ids)
            return raw, (parse_asr_output(raw, language is not None) if self.tokenizer is not None else ("unknown", raw))
        raw, (lang, text) = parse(ids)
        res = TranscribeResult(text=text, language=lang, raw_output=raw, ids=ids)
        if r.nbest is not None and r.nbest[0] is not None:
            res.nbest = [(parse(h[0])[1][1], h[2]) for h in r.nbest[0]]
        if r.temperatures is not None:
            res.temperature = r.temperatures[0]
        if (logprobs or top_logprobs or r.temperatures is not None) and r.logprobs is not None:
            res.token_logprobs = r.logprobs[0]
            res.avg_logprob = avg_logprob(r.logprobs[0], r.eos_logprobs[0])
        if top_logprobs:
            res.top_logprobs = r.top_logprobs[0]
            res.eos_top_logprobs = r.eos_top_logprobs[0]
        if al is not None:
            res.words = self._words(ids, al, r.logprobs[0], language if language is not None else lang)
        return res

    def _long_result(self, segs: List[LongSegment], language: Optional[str], logprobs: bool,
                     top_logprobs: int) -> TranscribeResult:
        """The TranscribeResult of one segmented file: `segments` = (start_s, end_s, text) per segment; `text` = the
        non-empty segment texts joined by text.join_segment_texts; `language` = the most frequent language of the
        segments with text (of all segments when none has text), or "forced"; `raw_output` = the segments' raw outputs,
        one per line; `ids`, `token_logprobs` and `top_logprobs` = the segments' concatenated; `avg_logprob` over all
        ids and each segment's EOS; `eos_top_logprobs` = the last segment's; `temperature` = the highest kept one;
        no `nbest` (a beam's hypotheses are per segment: transcribe_long returns them)."""
        from .text import join_segment_texts, majority_language, parse_asr_output
        parsed = []
        for sg in segs:
            raw = self.tokenizer.decode(sg.ids) if self.tokenizer is not None else " ".join(str(i) for i in sg.ids)
            lang, text = parse_asr_output(raw, language is not None) if self.tokenizer is not None else ("unknown", raw)
            parsed.append((raw, lang, text))
        if language is not None:
            lang = "forced"
            join_lang = language
        else:
            with_text = [p[1] for p in parsed if p[2]]
            lang = join_lang = majority_language(with_text or [p[1] for p in parsed])
        res = TranscribeResult(text=join_segment_texts([p[2] for p in parsed], join_lang), language=lang,
                               raw_output="\n".join(p[0] for p in parsed), ids=sum((sg.ids for sg in segs), []))
        res.segments = [(sg.start_s, sg.end_s, p[2]) for sg, p in zip(segs, parsed)]
        temps = [sg.temperature for sg in segs if sg.temperature is not None]
        if temps:
            res.temperature = max(temps)
        if (logprobs or top_logprobs or temps) and segs[0].logprobs is not None:
            res.token_logprobs = sum((sg.logprobs for sg in segs), [])
            vals = res.token_logprobs + [sg.eos_logprob for sg in segs if sg.eos_logprob is not None]
            res.avg_logprob = sum(vals) / len(vals) if vals else None
        if top_logprobs:
            res.top_logprobs = sum((sg.top_logprobs for sg in segs), [])
            res.eos_top_logprobs = segs[-1].eos_top_logprobs
        if segs[0].words is not None:
            res.words = sum((sg.words for sg in segs), [])
        return res

    # ---- stage-level calls (the calls transcribe() makes; used by the parity tests) ----
    def mel(self, clips: Sequence[np.ndarray], max_new_tokens: int = 64, max_lang: int = 16,
            max_context: int = 0) -> List[np.ndarray]:
        """WhisperFeatureExtractor::extract (mel.rs:49-96) -> [128, F] per utterance."""
        B = len(clips)
        arrs, ptrs, lens = self._pack_samples(clips)
        s = self._ensure_session(B, max(a.shape[0] for a in arrs), max_lang, max_new_tokens, max_context)
        frames = (C.c_int64 * B)()
        _lib.check(self._lib.asrb_mel(s, ptrs, lens, B, frames))
        out = []
        nm = self.config.audio.num_mel_bins
        for b in range(B):
            a = np.empty((nm, frames[b]), dtype=np.float32)
            _lib.check(self._lib.asrb_mel_read(s, b, a.ctypes.data_as(C.POINTER(C.c_float))))
            out.append(a)
        self._B = B
        return out

    def encode(self) -> List[np.ndarray]:
        """AudioEncoder::forward (audio_encoder.rs:79-169) on the mel of the last mel() call."""
        B = self._B
        toks = (C.c_int64 * B)()
        _lib.check(self._lib.asrb_encode(self._session, toks))
        out = []
        for b in range(B):
            a = np.empty((toks[b], self.config.audio.output_dim), dtype=np.float32)
            _lib.check(self._lib.asrb_encode_read(self._session, b, a.ctypes.data_as(C.POINTER(C.c_float))))
            out.append(a)
        return out

    def prefill(self, language_ids: Optional[Sequence] = None, want_logits: bool = True):
        """prompt + embed/inject + MRoPE + prefill (inference.rs:105-149) -> (seq_lens, last-row logits)."""
        B = self._B
        keep, lptrs, llens, mx = self._pack_lang(language_ids, B)
        seq = (C.c_int64 * B)()
        logits = np.empty((B, self.config.text.vocab_size), dtype=np.float32) if want_logits else None
        _lib.check(self._lib.asrb_prefill(self._session, lptrs, llens, seq,
                                          logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None))
        return list(seq), logits

    def decode_step(self, want_logits: bool = True):
        """One greedy iteration (inference.rs:160-200) -> (next ids, logits after the forward)."""
        B = self._B
        nxt = (C.c_int64 * B)()
        logits = np.empty((B, self.config.text.vocab_size), dtype=np.float32) if want_logits else None
        _lib.check(self._lib.asrb_decode_step(self._session, nxt,
                                              logits.ctypes.data_as(C.POINTER(C.c_float)) if want_logits else None))
        return list(nxt), logits

    def generate(self, max_new_tokens: int) -> List[List[int]]:
        B = self._B
        ids = np.zeros((B, max_new_tokens), dtype=np.int32)
        n = np.zeros(B, dtype=np.int32)
        _lib.check(self._lib.asrb_generate(self._session, int(max_new_tokens),
                                           ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                           n.ctypes.data_as(C.POINTER(C.c_int32))))
        return [ids[b, : n[b]].tolist() for b in range(B)]
