"""Streaming transcription (asrb_stream_*, DESIGN.md 4.9): live audio pushed per stream, each push answered with the
hypothesis of everything received so far.  The library re-encodes only the encoder windows whose mel may have changed
and keeps the prompt K/V before the first of them; this module holds the Python side of it."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Union

import numpy as np

from . import _lib

# forced-prefix bound: a stream's prefix holds at most this many ids per second of audio, plus one push's
# max_new_tokens (speech runs at about 3-5 tokens per second)
PREFIX_IDS_PER_SECOND = 8


def stream_max_lang_ids(max_seconds: float, n_lang: int, max_new_tokens: int) -> int:
    """The session's max_lang_ids for streams of up to `max_seconds`: the language ids, then the forced prefix."""
    return n_lang + math.ceil(PREFIX_IDS_PER_SECOND * max_seconds) + max_new_tokens


def next_prefix(hyp: Sequence[int], k: int, rollback: int, unfixed_pushes: int, final: bool) -> List[int]:
    """The forced prefix after push k (0-based) with hypothesis `hyp` (include/asr_b200.h): all of it on the final push,
    else all but the last `rollback` ids once k + 1 >= `unfixed_pushes`, else nothing."""
    if final:
        return list(hyp)
    if k + 1 < unfixed_pushes:
        return []
    return list(hyp[: max(0, len(hyp) - rollback)])


def stream_tokens(n_samples: int, n_window: int = 50) -> int:
    """Encoder output rows of n_samples: chunks of 2 * n_window mel frames, three stride-2 convolutions each."""
    frames, cf, out = -(-n_samples // 160), 2 * n_window, 0
    for k in range(0, frames, cf):
        f = min(cf, frames - k)
        for _ in range(3):
            f = (f - 1) // 2 + 1
        out += f
    return out


def prompt_rows_kept(n_context: int, tokens_before_first_reencoded: int, first_push: bool) -> int:
    """P_b: the prompt positions whose K/V a push keeps (head, context and the audio pads of the windows before the first
    re-encoded one), 0 on a stream's first push."""
    return 0 if first_push else 9 + n_context + tokens_before_first_reencoded


@dataclass
class StreamHypothesis:
    ids: List[int]                       # the hypothesis h = p + g of everything received so far
    fixed: int                           # its first `fixed` ids are forced into every later hypothesis
    text: Optional[str] = None           # with a tokenizer: h and its fixed part as text
    fixed_text: Optional[str] = None
    logprobs: Optional[List[float]] = None           # of g's ids (this push's run), with logprobs / top_logprobs
    top_logprobs: Optional[List[List[tuple]]] = None


class StreamSet:
    """n streams on the engine's session, opened by AsrInference.open_streams.  Any other call on the engine ends
    them (push then raises AsrbError with ASRB_ERR_STATE)."""

    def __init__(self, eng, n: int, max_seconds: float, lang_ids: Optional[List[int]], context_ids: Optional[List[int]],
                 rollback: int, unfixed_pushes: int, max_new_tokens: int, logprobs: bool, top_logprobs: int,
                 temperature: float, seed: int, no_repeat_ngram_size: int, repetition_penalty: float):
        from .inference import _decode_options, check_repetition, check_seed, check_temperature, check_top_logprobs
        if n < 1:
            raise ValueError("n must be >= 1")
        if max_seconds <= 0:
            raise ValueError("max_seconds must be > 0")
        if rollback < 0 or unfixed_pushes < 0:
            raise ValueError("rollback and unfixed_pushes must be >= 0")
        self._eng, self.n = eng, n
        self._lang = list(lang_ids) if lang_ids else []
        self._ctx = [list(context_ids)] if context_ids else None     # one context for every stream (set_context)
        self._max_new = int(max_new_tokens)
        self._top = check_top_logprobs(top_logprobs)
        self._logprobs = bool(logprobs) or self._top > 0
        temps = check_temperature(temperature)
        if len(temps) != 1:
            raise ValueError("streams take one temperature, not a fallback schedule")
        t, seed = temps[0], check_seed(seed)
        if self._top and t > 0.0:
            raise ValueError("temperature > 0 cannot be combined with top_logprobs")
        # a push's session options: the records, sampling at t > 0 and the repetition controls (no beam on streams)
        self._push_options = _decode_options(self._logprobs, self._top, t if t > 0.0 else None, seed, None,
                                             check_repetition(no_repeat_ngram_size, repetition_penalty))
        self.max_samples = int(round(max_seconds * 16000))
        max_lang = stream_max_lang_ids(max_seconds, len(self._lang), self._max_new)
        self._max_ids = max_lang + self._max_new          # h = p + g
        s = eng._ensure_session(n, max(self.max_samples, 201), max_lang, self._max_new, len(self._ctx[0]) if self._ctx else 0)
        self._s = s
        self._n = [0] * n                  # samples pushed per stream
        with eng._call_scope(s, {}, self._ctx):
            _lib.check(eng._lib.asrb_stream_open(s, n, int(rollback), int(unfixed_pushes)))

    def _session(self):
        if self._eng._session is not self._s:
            raise _lib.AsrbError(4, "the streams ended: the engine's session was replaced")
        return self._s

    def push(self, samples_per_stream: Sequence[Optional[np.ndarray]], final: Union[bool, Sequence[bool]] = False
             ) -> List[StreamHypothesis]:
        """One push: `samples_per_stream[b]` = new 16 kHz samples of stream b (None or empty: idle); `final` = True (all
        streams) or per stream.  Returns every stream's hypothesis after the push."""
        if len(samples_per_stream) != self.n:
            raise ValueError(f"need one entry per stream ({self.n})")
        s, eng, lib, n = self._session(), self._eng, self._eng._lib, self.n
        fin = [bool(final)] * n if isinstance(final, (bool, np.bool_)) else [bool(f) for f in final]
        if len(fin) != n:
            raise ValueError(f"need one final flag per stream ({self.n})")
        arrs = [np.ascontiguousarray(x if x is not None else np.zeros(0), dtype=np.float32) for x in samples_per_stream]
        ptrs = (C.POINTER(C.c_float) * n)(*[a.ctypes.data_as(C.POINTER(C.c_float)) for a in arrs])
        lens = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        fins = (C.c_int32 * n)(*fin)
        keep, lptrs, llens, _ = eng._pack_lang([self._lang] * n if self._lang else None, n)
        hyp = np.zeros((n, self._max_ids), dtype=np.int32)
        hl, fl = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
        P = C.POINTER
        with eng._call_scope(s, self._push_options):
            _lib.check(lib.asrb_stream_push(s, n, ptrs, lens, fins, lptrs, llens, self._max_new, self._max_ids,
                                            hyp.ctypes.data_as(P(C.c_int32)), hl.ctypes.data_as(P(C.c_int32)),
                                            fl.ctypes.data_as(P(C.c_int32))))
            eng._B = n
            for b in range(n):
                self._n[b] += arrs[b].shape[0]
            out = [StreamHypothesis(hyp[b, : hl[b]].tolist(), int(fl[b])) for b in range(n)]
            active = [a.shape[0] > 0 or f for a, f in zip(arrs, fin)]
            if self._logprobs:
                lp, _ = eng.last_logprobs(self._max_new)
                for b in range(n):
                    out[b].logprobs = lp[b] if active[b] else None
            if self._top:
                tk, _ = eng.last_top_logprobs(self._max_new, self._top)
                for b in range(n):
                    out[b].top_logprobs = tk[b] if active[b] else None
        if eng.tokenizer is not None:
            from .text import parse_asr_output
            forced = bool(self._lang)
            for h in out:
                h.text = parse_asr_output(eng.tokenizer.decode(h.ids), forced)[1]
                h.fixed_text = parse_asr_output(eng.tokenizer.decode(h.ids[: h.fixed]), forced)[1]
        return out

    def reset(self, b: int) -> None:
        """Stream b back to its start (no samples, empty prefix), open again after a final push."""
        s = self._session()
        with self._eng._call_scope(s, {}, self._ctx):
            _lib.check(self._eng._lib.asrb_stream_reset(s, int(b)))
        self._n[b] = 0

    def stats(self) -> Dict[str, int]:
        """asrb_last_stream_stats: the last push's windows and prompt rows, computed versus reused."""
        out = (C.c_int64 * 5)()
        _lib.check(self._eng._lib.asrb_last_stream_stats(self._session(), out, 5))
        return dict(zip(("windows_encoded", "windows_reused", "windows_floor_moved", "prompt_rows_computed",
                         "prompt_rows_kept"), [int(v) for v in out]))

    def mel(self, b: int) -> np.ndarray:
        """asrb_stream_mel_read: stream b's mel [128][F] after its last push."""
        n = self._stream_samples(b)
        out = np.zeros((self._eng.config.audio.num_mel_bins, (n + 159) // 160), dtype=np.float32)
        _lib.check(self._eng._lib.asrb_stream_mel_read(self._session(), int(b), out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def encoder_output(self, b: int) -> np.ndarray:
        """asrb_stream_encode_read: stream b's encoder output [tokens][output_dim] after its last push."""
        a = self._eng.config.audio
        out = np.zeros((stream_tokens(self._stream_samples(b), a.n_window), a.output_dim), dtype=np.float32)
        _lib.check(self._eng._lib.asrb_stream_encode_read(self._session(), int(b), out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def _stream_samples(self, b: int) -> int:
        if not 0 <= b < self.n or self._n[b] == 0:
            raise ValueError(f"stream {b} has no pushed audio")
        return self._n[b]
