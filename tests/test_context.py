"""Context biasing: caller-supplied ids in the prompt's system turn, prefilled once per batch when shared.

The oracle's prompt (oracle.build_prompt, the reference's fixed layout) has an empty system turn; `context_prompt`
below inserts a context after `system\\n`, which is where the model takes it.  Every oracle used here (greedy, the
float64 beam of test_beam.py, the Philox sampler of test_sampling.py) builds its prompt through oracle.build_prompt,
so each runs on the context prompt inside `context_prompt`."""
import contextlib
import ctypes as C
import json

import numpy as np
import pytest

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth

LOGIT_RTOL = 2e-3                  # as test_gpu_parity.py
MARGIN_FLOOR_REL = 4 * 1.5e-5      # as test_gpu_parity.py: exact ids are meaningful above this top-1/top-2 gap
HEAD = [151644, 8948, 198]         # <|im_start|>system\n


def ctx_ids(seed, n, hi=150000):
    return [int(v) for v in np.random.default_rng(seed).integers(0, hi, n)]


@contextlib.contextmanager
def context_prompt(ctx):
    """oracle.build_prompt with `ctx` inserted after `<|im_start|>system\\n`, for the duration of the block."""
    orig = O.build_prompt

    def build(num_audio_tokens, language_ids=None):
        toks, a0 = orig(num_audio_tokens, language_ids)
        ctx_l = list(ctx or [])
        return toks[:3] + ctx_l + toks[3:], a0 + len(ctx_l)
    O.build_prompt = build
    try:
        yield
    finally:
        O.build_prompt = orig


def oracle_ids(model, x, ctx, max_new_tokens, language_ids=None, **kw):
    with context_prompt(ctx):
        return O.transcribe_ids(model, x, language_ids=language_ids, max_new_tokens=max_new_tokens, **kw)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_prompt_layout_with_and_without_context():
    base, a0 = O.build_prompt(5, [7, 8])
    with context_prompt([11, 12, 13]):
        got, g0 = O.build_prompt(5, [7, 8])
    assert got == HEAD + [11, 12, 13] + [151645, 198, 151644, 872, 198, 151669] + [151676] * 5 + \
        [151670, 151645, 198, 151644, 77091, 198] + [7, 8]
    assert g0 == a0 + 3 and got[g0:g0 + 5] == [151676] * 5
    for empty in (None, []):
        with context_prompt(empty):
            assert O.build_prompt(5, [7, 8]) == (base, a0)       # no context: today's ids, id for id
    assert O.build_prompt(5, [7, 8]) == (base, a0)               # restored


def test_check_context_ids():
    from qwen3_asr_rs_b200.inference import check_context_ids
    assert check_context_ids(None, 3, 100) is None
    assert check_context_ids([[1, 2], None, []], 3, 100) == [[1, 2], None, None]
    assert check_context_ids([np.array([5, 99], dtype=np.int64)], 1, 100) == [[5, 99]]
    assert check_context_ids(((0,),), 1, 100) == [[0]]
    for bad in ([[1]], [[1], [2], [3]], "abc", [["a"]], [[100]], [[-1]], [[1.0]], [[True]], [7, 8], ["t5 t9", None]):
        with pytest.raises(ValueError):
            check_context_ids(bad, 2, 100)


def test_cli_context_flags(tmp_path):
    from qwen3_asr_rs_b200.__main__ import USAGE, split_context
    assert split_context(["m", "a.wav"]) == (["m", "a.wav"], None)
    assert split_context(["--context", "Qwen ASR", "m", "a.wav", "en"]) == (["m", "a.wav", "en"], "Qwen ASR")
    assert split_context(["m", "--context=kw1 kw2", "a.wav"]) == (["m", "a.wav"], "kw1 kw2")
    f = tmp_path / "ctx.txt"
    f.write_text("Zürich, Grüezi", encoding="utf-8")
    assert split_context(["m", "a.wav", "--context-file", str(f)]) == (["m", "a.wav"], "Zürich, Grüezi")
    assert split_context(["--context-file=" + str(f), "m", "a.wav"]) == (["m", "a.wav"], "Zürich, Grüezi")
    (tmp_path / "bad.txt").write_bytes(b"\xff\xfe\x00")
    for bad in (["m", "a.wav", "--context"], ["m", "a.wav", "--context-file"],
                ["m", "a.wav", "--context-file", str(tmp_path / "missing.txt")],
                ["m", "a.wav", "--context-file", str(tmp_path / "bad.txt")],
                ["m", "a.wav", "--context", "x", "--context-file", str(f)]):
        assert split_context(bad) is None, bad
    assert "--context TEXT" in USAGE and "--context-file PATH" in USAGE


def test_cli_usage_error_on_bad_context_flag(capsys):
    from qwen3_asr_rs_b200.__main__ import main
    assert main(["m", "a.wav", "--context"]) == 1
    assert "Usage" in capsys.readouterr().err


def test_set_context_null_session_is_a_status():
    from qwen3_asr_rs_b200 import _lib
    lib = _lib.load_library()
    ids = (C.c_int64 * 2)(1, 2)
    rows = (C.POINTER(C.c_int64) * 1)(C.cast(ids, C.POINTER(C.c_int64)))
    n = (C.c_int32 * 1)(2)
    assert lib.asrb_session_set_context(None, 1, rows, n) != 0
    assert lib.asrb_session_set_context(None, 0, None, None) != 0
    assert lib.asrb_last_prefill_stats(None, (C.c_int64 * 3)(), 3) != 0
    assert lib.asrb_session_create_ex(None, 1, 16000, 0, 16, 8, None) != 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx_engine(tiny):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    yield eng
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_ctx", [1, 37, 300])
def test_one_utterance_context_parity(tiny, ctx_engine, report, n_ctx):
    """Batch 1: prefill last-row logits within LOGIT_RTOL of the oracle's on the context prompt, and ids equal the
    oracle's on the fused and the per-phase path."""
    _, _, model = tiny
    eng = ctx_engine
    x = synth.make_clip(610 + n_ctx, 3.3)
    ctx = ctx_ids(n_ctx, n_ctx)
    n_new = 16
    ref = oracle_ids(model, x, ctx, n_new, keep_logits=True)
    eng.mel([x], max_new_tokens=n_new, max_context=n_ctx)
    eng.encode()
    eng.set_context([ctx])
    try:
        seq, logits = eng.prefill()
    finally:
        eng.set_context(None)
    assert seq[0] == 15 + n_ctx + ref.audio_embeds.shape[0]          # seq_lens_out: the whole prompt, context included
    report[f"context_{n_ctx}_prefill_logits_rel_err"] = _rel(logits[0], ref.prefill_logits.numpy())
    assert report[f"context_{n_ctx}_prefill_logits_rel_err"] <= LOGIT_RTOL
    for mode in ("mega", "phases"):
        eng.set_option("decode", mode)       # (drops the captured per-phase graph: the next capture is counted)
        try:
            s0 = _steps(eng.stats())
            got = eng.transcribe_ids([x], max_new_tokens=n_new, context_ids=[ctx])
            s1 = _steps(eng.stats())
        finally:
            eng.set_option("decode", "mega")
        assert got.ids[0] == ref.ids, mode
        moved = {k: s1[k] - s0[k] for k in s0}
        if mode == "mega":
            assert moved == {"decode_batch_steps": 0, "decode_fused_steps": got.decode_steps, "decode_phase_steps": 0}
        else:                                # graph replays are not counted, the capture is
            assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0 and moved["decode_phase_steps"] >= 1


@pytest.mark.gpu
def test_ragged_batch_shared_and_distinct_contexts(tiny, ctx_engine, report):
    """Contexts [A, A, None, B, A] with forced-language ids on two utterances: ids equal the oracle per utterance; the
    prefill computes sum(S_b) - 2 P_A rows, takes 2 P_A from the leader and fans out their KV."""
    cfg, _, model = tiny
    eng = ctx_engine
    A, Bc = ctx_ids(1, 23), ctx_ids(2, 41)
    ctxs = [A, list(A), None, Bc, list(A)]
    langs = [None, [9, 10], None, [11], None]
    clips = [synth.make_clip(620 + i, s) for i, s in enumerate([2.1, 4.7, 1.3, 3.0, 6.2])]
    n_new = 14
    got = eng.transcribe_ids(clips, language_ids=langs, max_new_tokens=n_new, context_ids=ctxs)
    st = eng.last_prefill_stats()
    S = []
    for b, (c, ctx, lang) in enumerate(zip(clips, ctxs, langs)):
        ref = oracle_ids(model, c, ctx, n_new, language_ids=lang)
        assert got.ids[b] == ref.ids, b
        S.append(15 + len(ctx or []) + ref.audio_embeds.shape[0] + len(lang or []))
    P_A = len(A) + 9
    bpp = 2 * cfg.text.num_hidden_layers * cfg.text.num_key_value_heads * cfg.text.head_dim * 4
    assert st == {"rows_computed": sum(S) - 2 * P_A, "rows_shared": 2 * P_A, "fanout_kv_bytes": 2 * P_A * bpp}
    report["context_ragged_prefill_stats"] = st


@pytest.mark.gpu
def test_no_context_is_no_change(tiny):
    """A run after set_context with all rows empty and a run after clearing give the ids, logprobs (bitwise) and kernel
    count of a session that never had a context; nothing is shared."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    clips = [synth.make_clip(640 + i, s) for i, s in enumerate([2.4, 5.1, 1.7])]
    plain = AsrInference.from_weights(config_tiny(), w, device=0)
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    try:
        ref = plain.transcribe_ids(clips, max_new_tokens=12, logprobs=True)
        eng.transcribe_ids(clips, max_new_tokens=12, context_ids=[[5, 6], None, [7]])    # a session with context room
        runs = [eng.transcribe_ids(clips, max_new_tokens=12, logprobs=True, context_ids=[None, [], None])]
        assert eng.last_prefill_stats()["rows_shared"] == 0
        eng.set_context(None)
        runs.append(eng.transcribe_ids(clips, max_new_tokens=12, logprobs=True))
        assert eng.last_prefill_stats()["rows_shared"] == 0
    finally:
        plain.close()
        eng.close()
    for r in runs:
        assert r.ids == ref.ids
        assert np.array_equal(np.array(sum(r.logprobs, []), np.float32), np.array(sum(ref.logprobs, []), np.float32))
        assert r.eos_logprobs == ref.eos_logprobs
        assert r.kernels_launched == ref.kernels_launched


@pytest.mark.gpu
def test_sharing_equals_not_sharing(ctx_engine):
    """A batch of 8 with one shared context gives each utterance the ids it gets alone, at batch 1, with that context."""
    eng = ctx_engine
    ctx = ctx_ids(8, 64)
    clips = [synth.make_clip(660 + i, s) for i, s in enumerate([1.2, 3.4, 2.2, 5.5, 0.9, 4.1, 2.8, 3.7])]
    got = eng.transcribe_ids(clips, max_new_tokens=12, context_ids=[ctx] * 8)
    st = eng.last_prefill_stats()
    assert st["rows_shared"] == 7 * (len(ctx) + 9)
    for b, c in enumerate(clips):
        assert eng.transcribe_ids([c], max_new_tokens=12, context_ids=[ctx]).ids[0] == got.ids[b], b


def _min_rel_margin(ref):
    ls = [ref.prefill_logits] + ref.step_logits[:-1]
    gaps = [float(l.topk(2).values[0] - l.topk(2).values[1]) for l in ls]
    mx = max(float(l.abs().max()) for l in ls)
    return min(gaps) / mx


@pytest.mark.gpu
def test_full_size_0p6b_batch8_shared_context(report):
    """Qwen3-ASR-0.6B dims, peaked untied head, batch 8 x 30 s, one shared 200-id context, 64 new tokens: exact ids on
    the batch-aware fused step, no phase steps, no SIMT GEMM fallbacks."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 1, peaked_head=True)
    model = O.OracleModel(cfg, w)
    ctx = ctx_ids(2005, 200)
    # clips whose oracle-side worst top-1/top-2 gap with this context is >= 3e-4 of max|logit| (scanned on the CPU)
    clips = [synth.make_clip(i, 30.0) for i in CLIPS_0P6B]
    refs = [oracle_ids(model, c, ctx, 64, keep_logits=True, lm_head_all_rows=False) for c in clips]
    report["context_full_b8_min_rel_margin"] = min(_min_rel_margin(r) for r in refs)
    assert report["context_full_b8_min_rel_margin"] >= 5 * MARGIN_FLOOR_REL
    ecfg = config_0p6b()
    ecfg.text.tie_word_embeddings = False
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        eng.transcribe_ids(clips, max_new_tokens=64, context_ids=[ctx] * 8)          # session, warm-up
        before = eng.stats()
        got = eng.transcribe_ids(clips, max_new_tokens=64, context_ids=[ctx] * 8)
        st = eng.stats()
        report["context_full_b8_prefill_stats"] = eng.last_prefill_stats()
        report["context_full_b8_stage_ms"] = got.stage_ms
    finally:
        eng.close()
    assert st["decode_batch_steps"] - before["decode_batch_steps"] == 63
    assert st["decode_phase_steps"] == before["decode_phase_steps"] and st["gemm_simt_fallbacks"] == 0
    for b in range(8):
        assert got.ids[b] == refs[b].ids, b


CLIPS_0P6B = (1, 3, 4, 6, 7, 8, 10, 17)


@pytest.mark.gpu
def test_beam_and_sampling_with_shared_context(tiny, report):
    """Beam search and seeded sampling with one context shared by the batch match the float64 oracle beam of
    test_beam.py and the Philox reference of test_sampling.py run on the context prompt."""
    import test_beam as TB
    import test_sampling as TS
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    cfg, w, model = tiny
    ctx = ctx_ids(31, 29)
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    try:
        with context_prompt(ctx):
            picked = TB.pick_clips(model, TB.POOL, 3, 3, 8)
        clips, refs = [p[0] for p in picked], [p[1] for p in picked]
        got = eng.transcribe_ids(clips, max_new_tokens=8, beam_size=3, context_ids=[ctx] * 3)
        TB._check(got, refs, eng.last_beam_stats(), cfg, report, "context_b3k3")
        assert eng.last_prefill_stats()["rows_shared"] == 2 * (len(ctx) + 9)

        sclips = [synth.make_clip(680 + i, s) for i, s in enumerate([2.6, 1.4, 3.8])]
        with context_prompt(ctx):
            seed, srefs, _ = TS.pick_seed(model, sclips, 1.0, 10)
        sgot = eng.transcribe_ids(sclips, max_new_tokens=10, temperature=1.0, seed=seed, context_ids=[ctx] * 3)
        for b, r in enumerate(srefs):
            assert sgot.ids[b] == r.ids, b
    finally:
        eng.close()


@pytest.mark.gpu
def test_context_crossing_fused_limit(tiny, ctx_engine):
    """A context long enough that prompt + generation crosses the fused step's 1152 keys mid-run: the run hands over
    to the per-phase path (counted) and its ids equal the oracle's."""
    _, _, model = tiny
    eng = ctx_engine
    x = synth.make_clip(700, 2.0)
    ctx = ctx_ids(1100, 1100)
    n_new = 40
    ref = oracle_ids(model, x, ctx, n_new)
    S = 15 + len(ctx) + ref.audio_embeds.shape[0]
    assert S < 1152 < S + len(ref.ids) - 1                     # the keys of the last forwards exceed the limit
    eng.transcribe_ids([x], max_new_tokens=n_new, context_ids=[ctx])   # grows the session (its counters restart)
    eng.set_option("decode", "mega")         # drops the captured per-phase graph: the next capture is counted
    s0 = _steps(eng.stats())
    got = eng.transcribe_ids([x], max_new_tokens=n_new, context_ids=[ctx])
    s1 = _steps(eng.stats())
    assert got.ids[0] == ref.ids
    fused = s1["decode_fused_steps"] - s0["decode_fused_steps"]
    assert 0 < fused < got.decode_steps                         # fused up to the limit, per-phase beyond it
    assert s1["decode_phase_steps"] > s0["decode_phase_steps"]


@pytest.mark.gpu
def test_context_refusals(tiny, ctx_engine, tmp_path):
    """Refused at set_context: too long, out of vocabulary, any context on a session without context room; refused at
    prefill, before any state change: a row count that is neither the batch nor 1.  transcribe(context=...) encodes the
    text with the tokenizer."""
    from qwen3_asr_rs_b200 import AsrInference, _lib
    cfg, w, model = tiny
    eng = ctx_engine
    x = synth.make_clip(720, 1.5)
    eng.mel([x, x], max_new_tokens=8, max_context=16)
    eng.encode()
    cap = eng._cap[4]
    for bad in ([[1] * (cap + 1)], [[cfg.text.vocab_size]], [[-1]]):
        with pytest.raises(_lib.AsrbError) as e:
            eng.set_context(bad)
        assert e.value.code == 1
    eng.set_context([[1, 2], [3], [4]])                  # 3 rows, batch of 2
    with pytest.raises(_lib.AsrbError) as e:
        eng.prefill(want_logits=False)
    assert e.value.code == 1
    eng.set_context([[1, 2]])                            # one row: every utterance
    seq, _ = eng.prefill(want_logits=False)              # the stage was still "encoded"
    assert eng.last_prefill_stats()["rows_shared"] == 11
    eng.set_context(None)

    s = C.c_void_p()
    lib = _lib.load_library()
    _lib.check(lib.asrb_session_create(eng._model, 1, 32000, 0, 8, C.byref(s)))
    try:
        ids = (C.c_int64 * 1)(5)
        rows = (C.POINTER(C.c_int64) * 1)(C.cast(ids, C.POINTER(C.c_int64)))
        assert lib.asrb_session_set_context(s, 1, rows, (C.c_int32 * 1)(1)) == 1
        assert lib.asrb_session_set_context(s, 1, rows, (C.c_int32 * 1)(0)) == 0     # empty rows are allowed
        assert lib.asrb_session_set_context(s, 0, None, None) == 0
    finally:
        lib.asrb_session_free(s)

    import wave
    d = tmp_path / "model"
    synth.write_checkpoint(str(d), cfg, w)
    vocab = {f"t{i}": i for i in range(cfg.text.vocab_size)}
    tok = {"version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": None,
           "pre_tokenizer": {"type": "Whitespace"}, "post_processor": None, "decoder": None,
           "model": {"type": "WordLevel", "vocab": vocab, "unk_token": "t0"}}
    (d / "tokenizer.json").write_text(json.dumps(tok))
    pcm = (synth.make_clip(77, 2.0) * 32767).astype("<i2")
    wav = tmp_path / "clip.wav"
    with wave.open(str(wav), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(pcm.tobytes())
    from qwen3_asr_rs_b200.audio import load_wav
    ref = oracle_ids(model, load_wav(str(wav)), [5, 9], 8)
    fe = AsrInference.load(str(d), device=0)
    try:
        r = fe.transcribe(str(wav), max_new_tokens=8, context="t5 t9")
        plain = fe.transcribe(str(wav), max_new_tokens=8, context="")
    finally:
        fe.close()
    assert r.ids == ref.ids
    assert plain.ids == O.transcribe_ids(model, load_wav(str(wav)), max_new_tokens=8).ids
