"""Per-token log-probabilities (session option "logprobs", asrb_last_logprobs): recorded beside the greedy argmax by
every decode path, from the same fp32 logits that select the ids.

Reference: log_softmax in float64 of the oracle's logits behind each id (prefill_logits behind ids[0], step_logits[i-1]
behind ids[i], and the logits after the last appended id behind the EOS that ended the sequence).
Tolerance: |lp - lp_ref| <= 2e-4 * max|logit|.  The logits themselves deviate by ~1.5e-5 * max|logit| (summation order),
and a log-probability moves by at most twice the largest logit error.
"""
import ctypes as C
import math

import numpy as np
import pytest

LP_RTOL = 2e-4
EOS = (151643, 151645)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: host-side rules
# ---------------------------------------------------------------------------------------------------------------------
def test_avg_logprob_rule():
    from qwen3_asr_rs_b200.inference import avg_logprob
    assert avg_logprob([-0.5, -1.5], None) == pytest.approx(-1.0)           # stopped at max_new_tokens: tokens only
    assert avg_logprob([-0.5, -1.5], -0.1) == pytest.approx(-0.7)           # ended on EOS: EOS counts as a token
    assert avg_logprob([], -0.3) == pytest.approx(-0.3)                     # EOS right after the prompt
    assert avg_logprob([], None) is None                                    # nothing to average


def test_cli_logprobs_flag_parsing():
    from qwen3_asr_rs_b200.__main__ import parse_args, main
    assert parse_args(["m", "a.wav"]) == ("m", "a.wav", None, False)
    assert parse_args(["m", "a.wav", "english"]) == ("m", "a.wav", "english", False)
    assert parse_args(["m", "a.wav", "--logprobs"]) == ("m", "a.wav", None, True)        # never the language
    assert parse_args(["--logprobs", "m", "a.wav", "english"]) == ("m", "a.wav", "english", True)
    assert parse_args(["m", "a.wav", "english", "--logprobs"]) == ("m", "a.wav", "english", True)
    assert parse_args(["m", "--logprobs"]) is None
    assert main(["--logprobs"]) == 1


def test_transcribe_result_fields_default_to_none():
    from qwen3_asr_rs_b200.inference import TranscribeIds, TranscribeResult
    r = TranscribeIds([[1]], {}, 0, 0)
    assert r.logprobs is None and r.eos_logprobs is None
    t = TranscribeResult("t", "l", "r", [1])
    assert t.token_logprobs is None and t.avg_logprob is None


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _ref_lps(ref, max_new):
    """(per-token reference log-probs, EOS log-prob or None, max|logit| over the logits involved) from an oracle run."""
    import torch
    ls = [ref.prefill_logits] + ref.step_logits
    lps, mx = [], 0.0
    for i, t in enumerate(ref.ids):
        l = ls[i].double()
        lps.append(float(torch.log_softmax(l, -1)[t]))
        mx = max(mx, float(l.abs().max()))
    eos = None
    if len(ref.ids) < max_new:
        l = ls[len(ref.ids)].double()
        tok = int(l.argmax())
        assert tok in EOS
        eos = float(torch.log_softmax(l, -1)[tok])
        mx = max(mx, float(l.abs().max()))
    return lps, eos, mx


def _check_vs_ref(got_lp, got_eos, ref, max_new):
    """max |lp - lp_ref| / max|logit| over tokens and EOS of one utterance."""
    lps, eos, mx = _ref_lps(ref, max_new)
    assert len(got_lp) == len(lps)
    assert all(v <= 0.0 and math.isfinite(v) for v in got_lp)
    err = max([abs(a - b) for a, b in zip(got_lp, lps)] + [0.0])
    if eos is None:
        assert got_eos is None
    else:
        assert got_eos is not None and got_eos <= 0.0
        err = max(err, abs(got_eos - eos))
    return err / mx


def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


@pytest.fixture(scope="module")
def lp_engine(tiny):
    """Own engine (the shared tiny_engine's options stay untouched)."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    yield eng
    eng.close()


def _run_paths(eng, clips, n_new, options):
    """Option off, then on (each after a warm-up run: session sized, per-phase graph captured), then on again:
    (result off, result on, result on again, step counters moved off / on)."""
    for k, v in options.items():
        eng.set_option(k, v)
    try:
        eng.set_option("logprobs", "0")
        eng.transcribe_ids(clips, max_new_tokens=n_new)
        s0 = _steps(eng.stats())
        off = eng.transcribe_ids(clips, max_new_tokens=n_new)
        s1 = _steps(eng.stats())
        eng.set_option("logprobs", "1")
        eng.transcribe_ids(clips, max_new_tokens=n_new)
        s2 = _steps(eng.stats())
        on = eng.transcribe_ids(clips, max_new_tokens=n_new, logprobs=True)
        s3 = _steps(eng.stats())
        on2 = eng.transcribe_ids(clips, max_new_tokens=n_new, logprobs=True)
    finally:
        eng.set_option("logprobs", "0")
        for k in options:
            eng.set_option(k, {"decode": "mega", "batch_step": "1"}[k])
    moved_off = {k: s1[k] - s0[k] for k in s0}
    moved_on = {k: s3[k] - s2[k] for k in s0}
    return off, on, on2, moved_off, moved_on


def _check_path(r, moved, path):
    """The decode path that ran: fused counters advance once per step; the per-phase path replays a captured graph
    (its counter moves at capture only), so it shows as more than two kernels per step."""
    if path == "decode_phase_steps":
        assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0
        assert r.kernels_launched > 2 * r.decode_steps
    else:
        assert moved[path] == r.decode_steps and moved["decode_phase_steps"] == 0


# (label, clips (index, seconds), new tokens, options, path whose counter must move)
PATHS = [
    ("fused_single", [(70, 4.0)], 48, {}, "decode_fused_steps"),
    ("fused_per_seq_b5", [(80 + i, s) for i, s in enumerate([2.5, 9.1, 5.0, 1.2, 3.3])], 16, {"batch_step": "0"}, "decode_fused_steps"),
    ("batched_nb8", [(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])], 14, {}, "decode_batch_steps"),
    ("batched_nb16", [(200 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9, 5.3, 1.4, 2.8])], 10, {}, "decode_batch_steps"),
    ("phases", [(71, 12.3), (72, 0.8)], 24, {"decode": "phases"}, "decode_phase_steps"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("label,sel,n_new,options,path", PATHS, ids=[p[0] for p in PATHS])
def test_logprobs_on_every_path(tiny, lp_engine, report, label, sel, n_new, options, path):
    """Ids unchanged and equal to the oracle's, the same path taken, log-probs within tolerance and bitwise deterministic."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    clips = [synth.make_clip(i, s) for i, s in sel]
    off, on, on2, moved_off, moved_on = _run_paths(lp_engine, clips, n_new, options)
    assert on.ids == off.ids
    assert moved_on == moved_off
    _check_path(on, moved_on, path)
    assert off.logprobs is None
    assert on.logprobs == on2.logprobs and on.eos_logprobs == on2.eos_logprobs        # bitwise (float equality)
    worst = 0.0
    for b, c in enumerate(clips):
        ref = O.transcribe_ids(model, c, max_new_tokens=n_new, keep_logits=True)
        assert on.ids[b] == ref.ids, b
        worst = max(worst, _check_vs_ref(on.logprobs[b], on.eos_logprobs[b], ref, n_new))
    report[f"logprobs_{label}_max_rel_err"] = worst
    assert worst <= LP_RTOL


@pytest.mark.gpu
def test_logprobs_across_fused_step_limit(tiny, lp_engine, report):
    """60 s prompt + 400 tokens: the fused step hands over to the per-phase path mid-generation; the record continues."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    x = synth.make_clip(302, 60.0)
    n_new = 400
    off, on, on2, moved_off, moved_on = _run_paths(lp_engine, [x], n_new, {})
    assert on.ids == off.ids and moved_on == moved_off
    assert moved_on["decode_fused_steps"] > 0 and on.kernels_launched > 2 * on.decode_steps
    assert on.logprobs == on2.logprobs
    ref = O.transcribe_ids(model, x, max_new_tokens=n_new, keep_logits=True)
    assert on.ids[0] == ref.ids and len(ref.ids) == n_new
    err = _check_vs_ref(on.logprobs[0], on.eos_logprobs[0], ref, n_new)
    report["logprobs_long_crossing_max_rel_err"] = err
    assert err <= LP_RTOL


@pytest.mark.gpu
def test_logprobs_self_consistent_with_returned_logits(lp_engine, report):
    """Per-phase path through the stage calls: each recorded log-prob equals the float64 log-softmax of the logits the
    GPU itself returned for that step."""
    import torch
    from qwen3_asr_rs_b200 import synth
    eng = lp_engine
    x = synth.make_clip(60, 6.2)
    eng.set_option("logprobs", "1")
    try:
        eng.mel([x])
        eng.encode()
        _, lg = eng.prefill()
        logits = [lg[0]]
        ids = []
        for _ in range(5):
            nxt, lg = eng.decode_step()
            ids.append(nxt[0])
            logits.append(lg[0])
        lps, eos = eng.last_logprobs(8)
    finally:
        eng.set_option("logprobs", "0")
    n = len(lps[0])
    assert n == 6 or (n >= 5 and eos[0] is not None)
    worst = 0.0
    for i, l in enumerate(logits[: n + (eos[0] is not None)]):
        ld = torch.from_numpy(l.astype(np.float64))
        if i < 5:
            assert int(ld.argmax()) == ids[i]
        ref = float(ld.max() - torch.logsumexp(ld, -1))
        worst = max(worst, abs((lps[0][i] if i < n else eos[0]) - ref))
    report["logprobs_self_consistency_max_abs_err"] = worst
    assert worst <= 1e-5


@pytest.mark.gpu
def test_logprobs_agree_across_paths(tiny, lp_engine, report):
    """The same clips through the fused single-sequence, batched and per-phase paths give the same ids and log-probs."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    eng = lp_engine
    clips = [synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])]
    n_new = 14
    mx = max(_ref_lps(O.transcribe_ids(model, c, max_new_tokens=n_new, keep_logits=True), n_new)[2] for c in clips)
    single = [eng.transcribe_ids([c], max_new_tokens=n_new, logprobs=True) for c in clips]
    batched = eng.transcribe_ids(clips, max_new_tokens=n_new, logprobs=True)
    eng.set_option("decode", "phases")
    try:
        phases = eng.transcribe_ids(clips, max_new_tokens=n_new, logprobs=True)
    finally:
        eng.set_option("decode", "mega")
    worst = 0.0
    for b in range(len(clips)):
        assert single[b].ids[0] == batched.ids[b] == phases.ids[b]
        for other in (batched, phases):
            a, o = single[b].logprobs[0], other.logprobs[b]
            worst = max([worst] + [abs(u - v) for u, v in zip(a, o)])
            ea, eo = single[b].eos_logprobs[0], other.eos_logprobs[b]
            assert (ea is None) == (eo is None)
            if ea is not None:
                worst = max(worst, abs(ea - eo))
    report["logprobs_cross_path_max_rel_diff"] = worst / mx
    assert worst <= LP_RTOL * mx


def _eos_model(tiny, k, scale=1.5):
    """The EOS-row construction of test_eos_stops_generation: EOS embedding row = scale x that of the k-th generated id
    of clip 90 (tied lm_head), which makes EOS the argmax right after that id's predecessor."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    cfg, w, base = tiny
    x = synth.make_clip(90, 1.5)
    r = O.transcribe_ids(base, x, max_new_tokens=6)
    e = w["thinker.model.embed_tokens.weight"].float().clone()
    e[151645] = e[r.ids[k]] * scale
    w2 = dict(w)
    w2["thinker.model.embed_tokens.weight"] = e.bfloat16()
    return w2, O.OracleModel(cfg, w2), x


@pytest.mark.gpu
def test_eos_right_after_prefill(tiny, report):
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    w2, model, x = _eos_model(tiny, 0)
    ref = O.transcribe_ids(model, x, max_new_tokens=12, keep_logits=True)
    assert len(ref.ids) == 0
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    try:
        got = eng.transcribe_ids([x], max_new_tokens=12, logprobs=True)
    finally:
        eng.close()
    assert got.ids == [[]] and got.logprobs == [[]]
    assert got.eos_logprobs[0] is not None and math.isfinite(got.eos_logprobs[0])
    err = _check_vs_ref(got.logprobs[0], got.eos_logprobs[0], ref, 12)
    report["logprobs_eos_after_prefill_rel_err"] = err
    assert err <= LP_RTOL


@pytest.mark.gpu
def test_eos_mid_generation_and_cap(tiny, report):
    """Clip 90 with the EOS row from its 3rd id: the oracle emits 2 ids, then EOS (top-1 gap 0.33 of max|logit|, scanned
    on the CPU); clip 92 (3 s) runs into the cap of 12 under the same weights.  Fused single-sequence and batched paths."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    w2, model, x = _eos_model(tiny, 2)
    y = synth.make_clip(92, 3.0)
    n_new = 12
    rx = O.transcribe_ids(model, x, max_new_tokens=n_new, keep_logits=True)
    ry = O.transcribe_ids(model, y, max_new_tokens=n_new, keep_logits=True)
    assert len(rx.ids) >= 2 and len(rx.ids) < n_new and len(ry.ids) == n_new
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    try:
        batched = eng.transcribe_ids([x, y], max_new_tokens=n_new, logprobs=True)   # (first run: fresh counters)
        moved = _steps(eng.stats())
        # the raw record: NaN at and beyond each length, also past the run's max_new_tokens
        lp = np.zeros((2, n_new + 4), np.float32)
        eos = np.zeros(2, np.float32)
        from qwen3_asr_rs_b200 import _lib
        _lib.check(eng._lib.asrb_last_logprobs(eng._session, n_new + 4, lp.ctypes.data_as(C.POINTER(C.c_float)),
                                               eos.ctypes.data_as(C.POINTER(C.c_float))))
        single = eng.transcribe_ids([x], max_new_tokens=n_new, logprobs=True)
    finally:
        eng.close()
    assert moved["decode_batch_steps"] > 0 and moved["decode_phase_steps"] == 0
    assert single.ids[0] == rx.ids and batched.ids == [rx.ids, ry.ids]
    worst = max(_check_vs_ref(single.logprobs[0], single.eos_logprobs[0], rx, n_new),
                _check_vs_ref(batched.logprobs[0], batched.eos_logprobs[0], rx, n_new),
                _check_vs_ref(batched.logprobs[1], batched.eos_logprobs[1], ry, n_new))
    report["logprobs_eos_mid_generation_rel_err"] = worst
    assert worst <= LP_RTOL
    assert batched.eos_logprobs[1] is None                                  # stopped by the cap
    assert np.isnan(lp[0, len(rx.ids):]).all() and np.isfinite(lp[0, :len(rx.ids)]).all()
    assert np.isnan(lp[1, n_new:]).all() and np.isfinite(lp[1, :n_new]).all()
    assert np.isfinite(eos[0]) and np.isnan(eos[1])


@pytest.mark.gpu
def test_last_logprobs_states(tiny, lp_engine):
    """ASRB_ERR_STATE before any run, after a run with the option off, and after switching it between prefill and
    generate (both ways)."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    from qwen3_asr_rs_b200._lib import AsrbError
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    x = synth.make_clip(301, 1.7)
    try:
        with pytest.raises(AsrbError):
            eng.last_logprobs(8)                                            # no session yet
        eng.mel([x])                                                        # session, nothing decoded
        with pytest.raises(AsrbError) as e:
            eng.last_logprobs(8)
        assert e.value.code == 4
        eng.transcribe_ids([x], max_new_tokens=8)                           # option off
        with pytest.raises(AsrbError) as e:
            eng.last_logprobs(8)
        assert e.value.code == 4
        for first, then in (("1", "0"), ("0", "1")):
            eng.set_option("logprobs", first)
            eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
            eng.set_option("logprobs", then)
            eng.generate(8)
            with pytest.raises(AsrbError) as e:
                eng.last_logprobs(8)
            assert e.value.code == 4
        eng.set_option("logprobs", "1")                                     # on throughout: readable
        eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
        ids = eng.generate(8)
        lps, _ = eng.last_logprobs(8)
        assert len(lps[0]) == len(ids[0])
        with pytest.raises(AsrbError):
            eng.set_option("logprobs", "yes")
    finally:
        eng.close()


@pytest.mark.gpu
def test_cli_prints_avg_logprob(tiny, tmp_path, capsys):
    """`python -m qwen3_asr_rs_b200 <model_dir> <wav> --logprobs` on a synthetic checkpoint directory."""
    import json
    import wave
    from qwen3_asr_rs_b200 import synth
    from qwen3_asr_rs_b200.__main__ import main
    cfg, w, _ = tiny
    d = tmp_path / "model"
    synth.write_checkpoint(str(d), cfg, w)
    vocab = {f"t{i}": i for i in range(cfg.text.vocab_size)}
    tok = {"version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": None,
           "pre_tokenizer": {"type": "Whitespace"}, "post_processor": None, "decoder": None,
           "model": {"type": "WordLevel", "vocab": vocab, "unk_token": "t0"}}
    (d / "tokenizer.json").write_text(json.dumps(tok))
    x = synth.make_clip(77, 2.0)
    wav = tmp_path / "clip.wav"
    with wave.open(str(wav), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes((x * 32767).astype("<i2").tobytes())
    assert main([str(d), str(wav), "--logprobs"]) == 0
    out = capsys.readouterr().out.splitlines()
    assert out[0].startswith("Language: ") and out[1].startswith("Text: ")
    assert out[2].startswith("Avg logprob: ")
    assert float(out[2].split(": ")[1]) <= 0.0


# ---------------------------------------------------------------------------------------------------------------------
# full-size dims (synthetic peaked untied head, clips vetted in test_gpu_parity.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full_peaked_lp():
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth
    cfg = O.cfg_0p6b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 1, peaked_head=True)
    ecfg = config_0p6b()
    ecfg.text.tie_word_embeddings = False
    eng = AsrInference.from_weights(ecfg, w, device=0)
    yield O.OracleModel(cfg, w), eng
    eng.close()


@pytest.mark.gpu
def test_full_size_0p6b_logprobs(full_peaked_lp, report):
    """0.6B dims: batch 1 x 30 s (fused single-sequence step) and batch 8 x 30 s (batched step), 32 new tokens."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    model, eng = full_peaked_lp
    n_new = 32
    clips = [synth.make_clip(i, 30.0) for i in (1, 3, 4, 6, 7, 8, 10, 17)]
    refs = [O.transcribe_ids(model, c, max_new_tokens=n_new, keep_logits=True, lm_head_all_rows=False) for c in clips]
    s0 = _steps(eng.stats())                      # batch 8 first: the batch-1 run then reuses its session (same counters)
    eight = eng.transcribe_ids(clips, max_new_tokens=n_new, logprobs=True)
    s1 = _steps(eng.stats())
    one = eng.transcribe_ids(clips[:1], max_new_tokens=n_new, logprobs=True)
    s2 = _steps(eng.stats())
    assert s1["decode_batch_steps"] - s0["decode_batch_steps"] == eight.decode_steps and s1["decode_phase_steps"] == s0["decode_phase_steps"]
    assert s2["decode_fused_steps"] - s1["decode_fused_steps"] == one.decode_steps and s2["decode_phase_steps"] == s1["decode_phase_steps"]
    assert one.ids[0] == refs[0].ids
    worst = _check_vs_ref(one.logprobs[0], one.eos_logprobs[0], refs[0], n_new)
    report["logprobs_full_0p6b_b1_rel_err"] = worst
    w8 = 0.0
    for b in range(8):
        assert eight.ids[b] == refs[b].ids, b
        w8 = max(w8, _check_vs_ref(eight.logprobs[b], eight.eos_logprobs[b], refs[b], n_new))
    report["logprobs_full_0p6b_b8_rel_err"] = w8
    assert worst <= LP_RTOL and w8 <= LP_RTOL


@pytest.mark.gpu
def test_full_size_1p7b_logprobs(report):
    """1.7B dims (K = 2048 lm_head: the generic GEMV form of the fused step), seed 3, clip 7, 32 new tokens."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_1p7b, synth
    cfg = O.cfg_1p7b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 3, peaked_head=True)
    ecfg = config_1p7b()
    ecfg.text.tie_word_embeddings = False
    x = synth.make_clip(7, 30.0)
    n_new = 32
    ref = O.transcribe_ids(O.OracleModel(cfg, w), x, max_new_tokens=n_new, keep_logits=True, lm_head_all_rows=False)
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        got = eng.transcribe_ids([x], max_new_tokens=n_new, logprobs=True)
        st = eng.stats()
    finally:
        eng.close()
    assert st["decode_phase_steps"] == 0 and st["decode_fused_steps"] == got.decode_steps
    assert got.ids[0] == ref.ids
    err = _check_vs_ref(got.logprobs[0], got.eos_logprobs[0], ref, n_new)
    report["logprobs_full_1p7b_rel_err"] = err
    assert err <= LP_RTOL
