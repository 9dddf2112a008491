"""The per-call option protocol of the Python engine, against a recording stand-in for the library (no GPU): a call
sets only the session options that differ from the engine's configured values, puts them back afterwards, also when
the library refuses the call, and sets and clears its context around it."""
import ctypes as C

import numpy as np
import pytest

from qwen3_asr_rs_b200 import _lib, config_tiny
from qwen3_asr_rs_b200.inference import AsrInference

REFUSED = 2


class RecordingLib:
    """Records every asrb_* call as (name, its int and string arguments); returns REFUSED from the calls in `refuse`."""

    def __init__(self, refuse=()):
        self.calls, self.refuse = [], set(refuse)

    def asrb_last_error(self):
        return b"refused"

    def __getattr__(self, name):
        if not name.startswith("asrb_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name,) + tuple(a.decode() if isinstance(a, bytes) else a for a in args
                                              if isinstance(a, (bytes, int))))
            return REFUSED if name in self.refuse else 0
        return call

    def traffic(self, main):
        """(option and context calls before `main`, `main` calls, those after it)."""
        keep = [c for c in self.calls if c[0] in ("asrb_session_set_option", "asrb_session_set_context", main)]
        i = [c[0] for c in keep].index(main)
        return keep[:i], [c for c in keep if c[0] == main], keep[i + 1:]


def engine(monkeypatch, options=(), refuse=()):
    lib = RecordingLib(refuse)
    monkeypatch.setattr(_lib, "load_library", lambda: lib)
    eng = AsrInference.__new__(AsrInference)
    eng.config, eng._lib, eng._options, eng.tokenizer = config_tiny(), lib, dict(options), None
    eng._ctx = eng._model = None
    eng._session, eng._cap = C.c_void_p(1), (8, 1 << 20, 64, 64, 64)   # big enough: no session is created
    return eng, lib


def opt(key, value):
    return ("asrb_session_set_option", key, value)


CLIP = np.zeros(1600, np.float32)


def test_options_equal_to_the_configured_values_are_not_set(monkeypatch):
    eng, lib = engine(monkeypatch, {"logprobs": "1", "top_logprobs": "3", "repetition_penalty": "1.5"})
    eng.transcribe_ids([CLIP], max_new_tokens=4, logprobs=True, top_logprobs=3, repetition_penalty=1.5)
    before, main, after = lib.traffic("asrb_transcribe_ids")
    assert before == [] and len(main) == 1 and after == []


def test_options_that_differ_are_set_and_restored(monkeypatch):
    eng, lib = engine(monkeypatch, {"repetition_penalty": "1.5"})
    eng.transcribe_ids([CLIP], max_new_tokens=4, temperature=0.7, seed=5, repetition_penalty=1.2)
    before, _, after = lib.traffic("asrb_transcribe_ids")
    assert before == [opt("temperature", "0.7"), opt("seed", "5"), opt("repetition_penalty", "1.2")]
    # back to the configured value, or to the library default where none is configured
    assert sorted(after) == sorted([opt("temperature", "0"), opt("seed", "0"), opt("repetition_penalty", "1.5")])


def test_options_are_restored_when_the_call_is_refused(monkeypatch):
    eng, lib = engine(monkeypatch, refuse=("asrb_transcribe_ids",))
    with pytest.raises(_lib.AsrbError) as e:
        eng.transcribe_ids([CLIP], max_new_tokens=4, beam_size=3, length_penalty=0.6)
    assert e.value.code == REFUSED
    before, _, after = lib.traffic("asrb_transcribe_ids")
    assert before == [opt("beam_size", "3"), opt("length_penalty", "0.6")]
    assert sorted(after) == sorted([opt("beam_size", "1"), opt("length_penalty", "none")])

    eng, lib = engine(monkeypatch, refuse=("asrb_score_ids",))
    with pytest.raises(_lib.AsrbError):
        eng.score_ids([CLIP], [[[1, 2]]], top_logprobs=2)
    assert lib.traffic("asrb_score_ids")[::2] == ([opt("top_logprobs", "2")], [opt("top_logprobs", "0")])


def test_context_is_set_and_cleared_around_the_call(monkeypatch):
    for refuse in ((), ("asrb_align_ids",)):
        eng, lib = engine(monkeypatch, refuse=refuse)
        try:
            eng.align_ids([CLIP, CLIP], [[1, 2], [3]], context_ids=[[5, 6], None])
        except _lib.AsrbError:
            assert refuse
        before, main, after = lib.traffic("asrb_align_ids")
        assert before == [("asrb_session_set_context", 2)] and len(main) == 1
        assert after == [("asrb_session_set_context", 0)]


def test_stream_open_and_push(monkeypatch):
    eng, lib = engine(monkeypatch)
    ss = eng.open_streams(2, 1.0, context_ids=[7, 8], logprobs=True, max_new_tokens=4)
    assert lib.traffic("asrb_stream_open")[::2] == ([("asrb_session_set_context", 1)], [("asrb_session_set_context", 0)])
    lib.calls.clear()
    ss.push([CLIP, None])
    assert lib.traffic("asrb_stream_push")[::2] == ([opt("logprobs", "1")], [opt("logprobs", "0")])
