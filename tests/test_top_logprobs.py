"""Top-k alternatives (session option "top_logprobs", asrb_last_top_logprobs): the k best candidates of every greedy
step, kept beside the argmax by every decode path, from the same fp32 logits that select the ids.

Reference: the oracle's float64 logits behind each id (prefill_logits behind ids[0], step_logits[i-1] behind ids[i], and
the logits after the last appended id behind the EOS that ended the sequence), ranked by (logit descending, id
ascending), with log_softmax for the values.  delta = 2e-4 * max|logit|, the bound of the per-token log-probabilities:
the logits deviate by ~1.5e-5 * max|logit| (summation order), so a candidate's value moves by at most twice that, and
a rank's id is pinned only where the oracle's gaps on both sides of it exceed delta.
"""
import ctypes as C
import math

import numpy as np
import pytest

LP_RTOL = 2e-4
EOS = (151643, 151645)
K = 8


# ---------------------------------------------------------------------------------------------------------------------
# CPU: host-side rules
# ---------------------------------------------------------------------------------------------------------------------
def test_top_logprobs_argument_validation():
    from qwen3_asr_rs_b200.inference import check_top_logprobs
    for k in range(9):
        assert check_top_logprobs(k) == k
    assert check_top_logprobs(np.int64(3)) == 3
    for bad in (9, -1, "x", "3", 2.0, True, None):
        with pytest.raises(ValueError):
            check_top_logprobs(bad)


def test_cli_top_logprobs_flag_parsing():
    from qwen3_asr_rs_b200.__main__ import main, parse_args, split_top_logprobs
    assert split_top_logprobs(["m", "a.wav"]) == (["m", "a.wav"], 0)
    assert split_top_logprobs(["m", "a.wav", "--top-logprobs", "3"]) == (["m", "a.wav"], 3)
    assert split_top_logprobs(["--top-logprobs", "8", "m", "a.wav", "english"]) == (["m", "a.wav", "english"], 8)
    assert split_top_logprobs(["m", "a.wav", "--top-logprobs=5", "--logprobs"]) == (["m", "a.wav", "--logprobs"], 5)
    for bad in (["m", "a.wav", "--top-logprobs"], ["m", "a.wav", "--top-logprobs", "9"],
                ["m", "a.wav", "--top-logprobs", "0"], ["m", "a.wav", "--top-logprobs", "x"],
                ["m", "a.wav", "--top-logprobs=-1"]):
        assert split_top_logprobs(bad) is None, bad
    # the flag's value is never taken for the language, and parse_args keeps its 4-tuple
    rest, k = split_top_logprobs(["m", "a.wav", "--top-logprobs", "2", "english", "--logprobs"])
    assert k == 2 and parse_args(rest) == ("m", "a.wav", "english", True)
    assert main(["m", "a.wav", "--top-logprobs", "9"]) == 1
    assert main(["--top-logprobs", "3", "m"]) == 1


def test_top_logprobs_fields_default_to_none():
    from qwen3_asr_rs_b200.inference import TranscribeIds, TranscribeResult
    r = TranscribeIds([[1]], {}, 0, 0)
    assert r.top_logprobs is None and r.eos_top_logprobs is None
    t = TranscribeResult("t", "l", "r", [1])
    assert t.top_logprobs is None and t.eos_top_logprobs is None


def test_cli_formats_candidates():
    from qwen3_asr_rs_b200.__main__ import format_candidates
    line = format_candidates([(5, -0.01), (7, -2.5)], lambda ids: f"t{ids[0]}")
    assert line == "'t5' -0.0100  't7' -2.5000"


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _ranked(l, n):
    """The n best (ids, logits) of float64 logits `l` under (logit descending, id ascending)."""
    top = np.argpartition(-l, n + 8)[: n + 8]
    order = top[np.lexsort((top, -l[top]))][:n]
    return order, l[order]


def _logsoftmax(l):
    m = l.max()
    return l - m - math.log(np.exp(l - m).sum())


class Stats:
    """Worst relative deviations and exact-id counts over the rows checked."""
    def __init__(self):
        self.val = 0.0          # max |value - reference log p at that id| / max|logit|
        self.rank = 0.0         # max |oracle logit of the rank-r id - oracle's r-th largest logit| / max|logit|
        self.exact = 0          # ranks whose id equals the oracle's rank-r id
        self.total = 0
        self.pinned = 0         # ranks whose oracle gaps exceed delta on both sides (id must match)

    def add(self, o):
        self.val = max(self.val, o.val); self.rank = max(self.rank, o.rank)
        self.exact += o.exact; self.total += o.total; self.pinned += o.pinned
        return self


def _check_row(cands, tok, l, mx, st):
    """One step: the k candidates (id, logprob) against float64 logits `l` (numpy), selected id `tok`."""
    k = len(cands)
    ids = [i for i, _ in cands]
    vals = [v for _, v in cands]
    assert ids[0] == tok
    assert len(set(ids)) == k and all(0 <= i < len(l) for i in ids)
    assert all(math.isfinite(v) and v <= 0.0 for v in vals)
    assert all(vals[j] >= vals[j + 1] for j in range(k - 1))
    delta = LP_RTOL * mx
    lsm = _logsoftmax(l)
    ref_ids, ref_l = _ranked(l, k + 1)
    for r in range(k):
        st.val = max(st.val, abs(vals[r] - lsm[ids[r]]) / mx)
        st.rank = max(st.rank, abs(l[ids[r]] - ref_l[r]) / mx)
        st.total += 1
        st.exact += int(ids[r] == ref_ids[r])
        if (r == 0 or ref_l[r - 1] - ref_l[r] > delta) and ref_l[r] - ref_l[r + 1] > delta:
            st.pinned += 1
            assert ids[r] == ref_ids[r], (r, ids, list(ref_ids))


def _check_vs_ref(rows, eos_row, ref, max_new, k=K):
    """All rows of one utterance against the oracle run `ref` (keep_logits=True)."""
    ls = [ref.prefill_logits] + ref.step_logits
    n = len(ref.ids)
    used = [ls[i].double().numpy() for i in range(n + (n < max_new))]
    mx = max(float(np.abs(l).max()) for l in used)
    st = Stats()
    assert len(rows) == n
    for i, t in enumerate(ref.ids):
        assert len(rows[i]) == k
        _check_row(rows[i], t, used[i], mx, st)
    if n < max_new:
        assert eos_row is not None and len(eos_row) == k
        tok = int(np.argmax(used[n]))
        assert tok in EOS
        _check_row(eos_row, tok, used[n], mx, st)
    else:
        assert eos_row is None
    assert st.val <= LP_RTOL and st.rank <= LP_RTOL
    return st


def _check_against_logprobs(r, b):
    """Entry 0 of every row is the generated id, and its value bitwise the per-token log-probability record."""
    assert [row[0][0] for row in r.top_logprobs[b]] == r.ids[b]
    assert [row[0][1] for row in r.top_logprobs[b]] == r.logprobs[b]
    e = r.eos_top_logprobs[b]
    assert (e is None) == (r.eos_logprobs[b] is None)
    if e is not None:
        assert e[0][0] in EOS and e[0][1] == r.eos_logprobs[b]


def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


def _report(report, key, st):
    report[f"top_logprobs_{key}_max_rel_err"] = st.val
    report[f"top_logprobs_{key}_rank_logit_max_rel_err"] = st.rank
    report[f"top_logprobs_{key}_exact_id_fraction"] = st.exact / max(st.total, 1)
    report[f"top_logprobs_{key}_pinned_ranks"] = st.pinned


@pytest.fixture(scope="module")
def tk_engine(tiny):
    """Own engine (the shared tiny_engine's options stay untouched)."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    yield eng
    eng.close()


def _run_paths(eng, clips, n_new, options):
    """Option off, then k = 8 (each after a warm-up run: session sized, per-phase graph captured), then k = 8 again:
    (result off, result on, result on again, step counters moved off / on)."""
    for k, v in options.items():
        eng.set_option(k, v)
    try:
        eng.transcribe_ids(clips, max_new_tokens=n_new)
        s0 = _steps(eng.stats())
        off = eng.transcribe_ids(clips, max_new_tokens=n_new)
        s1 = _steps(eng.stats())
        eng.set_option("top_logprobs", str(K))                              # configured: no per-call switching
        eng.transcribe_ids(clips, max_new_tokens=n_new, top_logprobs=K)
        s2 = _steps(eng.stats())
        on = eng.transcribe_ids(clips, max_new_tokens=n_new, top_logprobs=K)
        s3 = _steps(eng.stats())
        on2 = eng.transcribe_ids(clips, max_new_tokens=n_new, top_logprobs=K)
    finally:
        eng.set_option("top_logprobs", "0")
        for k in options:
            eng.set_option(k, {"decode": "mega", "batch_step": "1"}[k])
    moved_off = {k: s1[k] - s0[k] for k in s0}
    moved_on = {k: s3[k] - s2[k] for k in s0}
    return off, on, on2, moved_off, moved_on


def _check_path(r, moved, path):
    """The decode path that ran: fused counters advance once per step; the per-phase path replays a captured graph."""
    if path == "decode_phase_steps":
        assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0
        assert r.kernels_launched > 2 * r.decode_steps
    else:
        assert moved[path] == r.decode_steps and moved["decode_phase_steps"] == 0


# (label, clips (index, seconds), new tokens, options, path whose counter must move): those of test_logprobs.py
PATHS = [
    ("fused_single", [(70, 4.0)], 48, {}, "decode_fused_steps"),
    ("fused_per_seq_b5", [(80 + i, s) for i, s in enumerate([2.5, 9.1, 5.0, 1.2, 3.3])], 16, {"batch_step": "0"}, "decode_fused_steps"),
    ("batched_nb8", [(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])], 14, {}, "decode_batch_steps"),
    ("batched_nb16", [(200 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9, 5.3, 1.4, 2.8])], 10, {}, "decode_batch_steps"),
    ("phases", [(71, 12.3), (72, 0.8)], 24, {"decode": "phases"}, "decode_phase_steps"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("label,sel,n_new,options,path", PATHS, ids=[p[0] for p in PATHS])
def test_top_logprobs_on_every_path(tiny, tk_engine, report, label, sel, n_new, options, path):
    """Ids and path unchanged, records bitwise deterministic, entry 0 = the id and its log-probability, candidates
    against the oracle."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    clips = [synth.make_clip(i, s) for i, s in sel]
    off, on, on2, moved_off, moved_on = _run_paths(tk_engine, clips, n_new, options)
    assert on.ids == off.ids
    assert moved_on == moved_off
    _check_path(on, moved_on, path)
    assert off.top_logprobs is None
    assert on.top_logprobs == on2.top_logprobs and on.eos_top_logprobs == on2.eos_top_logprobs     # bitwise
    st = Stats()
    for b, c in enumerate(clips):
        _check_against_logprobs(on, b)
        ref = O.transcribe_ids(model, c, max_new_tokens=n_new, keep_logits=True)
        assert on.ids[b] == ref.ids, b
        st.add(_check_vs_ref(on.top_logprobs[b], on.eos_top_logprobs[b], ref, n_new))
    _report(report, label, st)


@pytest.mark.gpu
def test_top_logprobs_across_fused_step_limit(tiny, tk_engine, report):
    """60 s prompt + 400 tokens: the fused step hands over to the per-phase path mid-generation; the record continues."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    x = synth.make_clip(302, 60.0)
    n_new = 400
    off, on, on2, moved_off, moved_on = _run_paths(tk_engine, [x], n_new, {})
    assert on.ids == off.ids and moved_on == moved_off
    assert moved_on["decode_fused_steps"] > 0 and on.kernels_launched > 2 * on.decode_steps
    assert on.top_logprobs == on2.top_logprobs
    _check_against_logprobs(on, 0)
    ref = O.transcribe_ids(model, x, max_new_tokens=n_new, keep_logits=True)
    assert on.ids[0] == ref.ids and len(ref.ids) == n_new
    _report(report, "long_crossing", _check_vs_ref(on.top_logprobs[0], on.eos_top_logprobs[0], ref, n_new))


@pytest.mark.gpu
def test_top_logprobs_self_consistent_with_returned_logits(tk_engine, report):
    """Per-phase path through the stage calls: each row is the exact top k of the logits the GPU itself returned for
    that step under (value descending, id ascending), with values within 1e-5 of their float64 log-softmax."""
    from qwen3_asr_rs_b200 import synth
    eng = tk_engine
    x = synth.make_clip(60, 6.2)
    eng.set_option("top_logprobs", str(K))
    try:
        eng.mel([x])
        eng.encode()
        _, lg = eng.prefill()
        logits = [lg[0]]
        for _ in range(5):
            _, lg = eng.decode_step()
            logits.append(lg[0])
        rows, eos = eng.last_top_logprobs(8, K)
        lps, eos_lp = eng.last_logprobs(8)
    finally:
        eng.set_option("top_logprobs", "0")
    n = len(rows[0])
    assert n == 6 or (n >= 5 and eos[0] is not None)
    worst = 0.0
    for i, l in enumerate(logits[: n + (eos[0] is not None)]):
        row = rows[0][i] if i < n else eos[0]
        l32 = l.astype(np.float32)
        order = np.lexsort((np.arange(len(l32)), -l32))[:K]              # exact, ties by ascending id
        assert [c[0] for c in row] == [int(j) for j in order], i
        lsm = _logsoftmax(l32.astype(np.float64))
        worst = max([worst] + [abs(v - lsm[j]) for j, v in row])
        assert row[0][1] == (lps[0][i] if i < n else eos_lp[0])
    report["top_logprobs_self_consistency_max_abs_err"] = worst
    assert worst <= 1e-5


@pytest.mark.gpu
def test_top_logprobs_agree_across_paths(tiny, tk_engine, report):
    """The same clips through the fused single-sequence, batched and per-phase paths: values within delta, ids equal
    wherever the candidates' own gaps exceed delta."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    eng = tk_engine
    clips = [synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])]
    n_new = 14
    mx = 0.0
    for c in clips:
        ref = O.transcribe_ids(model, c, max_new_tokens=n_new, keep_logits=True)
        mx = max([mx] + [float(l.abs().max()) for l in [ref.prefill_logits] + ref.step_logits])
    delta = LP_RTOL * mx
    single = [eng.transcribe_ids([c], max_new_tokens=n_new, top_logprobs=K) for c in clips]
    batched = eng.transcribe_ids(clips, max_new_tokens=n_new, top_logprobs=K)
    eng.set_option("decode", "phases")
    try:
        phases = eng.transcribe_ids(clips, max_new_tokens=n_new, top_logprobs=K)
    finally:
        eng.set_option("decode", "mega")
    worst = 0.0
    for b in range(len(clips)):
        assert single[b].ids[0] == batched.ids[b] == phases.ids[b]
        a_rows = single[b].top_logprobs[0] + ([single[b].eos_top_logprobs[0]] if single[b].eos_top_logprobs[0] else [])
        for other in (batched, phases):
            o_rows = other.top_logprobs[b] + ([other.eos_top_logprobs[b]] if other.eos_top_logprobs[b] else [])
            assert len(a_rows) == len(o_rows)
            for ra, ro in zip(a_rows, o_rows):
                va = [v for _, v in ra]
                for r in range(K):
                    worst = max(worst, abs(ra[r][1] - ro[r][1]))
                    if (r == 0 or va[r - 1] - va[r] > 2 * delta) and (r == K - 1 or va[r] - va[r + 1] > 2 * delta):
                        assert ra[r][0] == ro[r][0]
    report["top_logprobs_cross_path_max_rel_diff"] = worst / mx
    assert worst <= LP_RTOL * mx


def _eos_model(tiny, k, scale=1.5):
    """The EOS-row construction of test_logprobs.py: EOS embedding row = scale x that of the k-th generated id of clip 90
    (tied lm_head), which makes EOS the argmax right after that id's predecessor."""
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


def _raw_top(eng, max_new, k, B):
    from qwen3_asr_rs_b200 import _lib
    ids = np.zeros((B, max_new, k), np.int32)
    lp = np.zeros((B, max_new, k), np.float32)
    eids = np.zeros((B, k), np.int32)
    elp = np.zeros((B, k), np.float32)
    _lib.check(eng._lib.asrb_last_top_logprobs(eng._session, max_new, k, ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                               lp.ctypes.data_as(C.POINTER(C.c_float)), eids.ctypes.data_as(C.POINTER(C.c_int32)),
                                               elp.ctypes.data_as(C.POINTER(C.c_float))))
    return ids, lp, eids, elp


@pytest.mark.gpu
def test_top_logprobs_eos_right_after_prefill(tiny, report):
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    w2, model, x = _eos_model(tiny, 0)
    ref = O.transcribe_ids(model, x, max_new_tokens=12, keep_logits=True)
    assert len(ref.ids) == 0
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    try:
        got = eng.transcribe_ids([x], max_new_tokens=12, top_logprobs=K)
        ids, lp, eids, elp = _raw_top(eng, 12, K, 1)
    finally:
        eng.close()
    assert got.ids == [[]] and got.top_logprobs == [[]]
    assert got.eos_top_logprobs[0] is not None
    _check_against_logprobs(got, 0)
    _report(report, "eos_after_prefill", _check_vs_ref(got.top_logprobs[0], got.eos_top_logprobs[0], ref, 12))
    assert (ids == -1).all() and np.isnan(lp).all()
    assert (eids[0] >= 0).all() and np.isfinite(elp[0]).all()


@pytest.mark.gpu
def test_top_logprobs_eos_mid_generation_and_cap(tiny, report):
    """Clip 90 with the EOS row from its 3rd id ends on EOS after 2 ids; clip 92 runs into the cap of 12.  Batched and
    fused single-sequence paths; the raw ABI arrays hold -1 / NaN at and beyond each length."""
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
        batched = eng.transcribe_ids([x, y], max_new_tokens=n_new, top_logprobs=K)
        moved = _steps(eng.stats())
        ids, lp, eids, elp = _raw_top(eng, n_new + 4, 3, 2)                  # k < recorded, rows past max_new_tokens
        single = eng.transcribe_ids([x], max_new_tokens=n_new, top_logprobs=K)
    finally:
        eng.close()
    assert moved["decode_batch_steps"] > 0 and moved["decode_phase_steps"] == 0
    assert single.ids[0] == rx.ids and batched.ids == [rx.ids, ry.ids]
    st = Stats()
    st.add(_check_vs_ref(single.top_logprobs[0], single.eos_top_logprobs[0], rx, n_new))
    st.add(_check_vs_ref(batched.top_logprobs[0], batched.eos_top_logprobs[0], rx, n_new))
    st.add(_check_vs_ref(batched.top_logprobs[1], batched.eos_top_logprobs[1], ry, n_new))
    _check_against_logprobs(single, 0)
    for b in range(2):
        _check_against_logprobs(batched, b)
    _report(report, "eos_mid_generation", st)
    assert batched.eos_top_logprobs[1] is None                              # stopped by the cap
    for b, n in ((0, len(rx.ids)), (1, n_new)):
        assert (ids[b, n:] == -1).all() and np.isnan(lp[b, n:]).all()
        assert (ids[b, :n] >= 0).all() and np.isfinite(lp[b, :n]).all()
        assert [[i for i, _ in row[:3]] for row in batched.top_logprobs[b]] == ids[b, :n].tolist()
    assert (eids[0] >= 0).all() and np.isfinite(elp[0]).all()
    assert (eids[1] == -1).all() and np.isnan(elp[1]).all()


@pytest.mark.gpu
def test_last_top_logprobs_states(tiny):
    """ASRB_ERR_STATE before any run, after a run with the option off, after switching k between the prefill and
    generate; ASRB_ERR_INVALID for k = 0, for k above the recorded value and for option values outside 0..8."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    from qwen3_asr_rs_b200._lib import AsrbError
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    x = synth.make_clip(301, 1.7)
    try:
        with pytest.raises(AsrbError):
            eng.last_top_logprobs(8, 1)                                     # no session yet
        eng.mel([x])                                                        # session, nothing decoded
        with pytest.raises(AsrbError) as e:
            eng.last_top_logprobs(8, 1)
        assert e.value.code == 4
        for bad in ("9", "-1", "x", "", "10", "1.0"):
            with pytest.raises(AsrbError) as e:
                eng.set_option("top_logprobs", bad)
            assert e.value.code == 1
        eng.set_option("top_logprobs", "0")                                 # the engine replays its options
        eng.transcribe_ids([x], max_new_tokens=8)                           # option off
        with pytest.raises(AsrbError) as e:
            eng.last_top_logprobs(8, 1)
        assert e.value.code == 4
        for first, then in (("3", "0"), ("0", "3"), ("3", "5")):
            eng.set_option("top_logprobs", first)
            eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
            eng.set_option("top_logprobs", then)
            eng.generate(8)
            with pytest.raises(AsrbError) as e:
                eng.last_top_logprobs(8, 1)
            assert e.value.code == 4, (first, then)
        eng.set_option("top_logprobs", "3")                                 # on throughout: readable
        eng.set_option("logprobs", "0")
        eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
        ids = eng.generate(8)
        for bad_k in (0, 4):
            with pytest.raises(AsrbError) as e:
                eng.last_top_logprobs(8, bad_k)
            assert e.value.code == 1
        rows3, _ = eng.last_top_logprobs(8, 3)
        rows1, _ = eng.last_top_logprobs(8, 1)
        lps, _ = eng.last_logprobs(8)                                       # recorded too, with "logprobs" off
        assert [[c[0] for c in r] for r in rows1[0]] == [[t] for t in ids[0]]
        assert [r[:1] for r in rows3[0]] == rows1[0]
        assert [r[0][1] for r in rows1[0]] == lps[0]
    finally:
        eng.close()


@pytest.mark.gpu
def test_cli_prints_top_logprobs(tiny, tmp_path, capsys):
    """`python -m qwen3_asr_rs_b200 <model_dir> <wav> --top-logprobs 3` on a synthetic checkpoint directory."""
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
    assert main([str(d), str(wav), "--top-logprobs", "3"]) == 0
    out = capsys.readouterr().out.splitlines()
    assert out[0].startswith("Language: ") and out[1].startswith("Text: ")
    assert out[2] == "Top logprobs:"
    lines = out[3:]
    assert lines and all(l.startswith("  [") for l in lines)
    for l in lines:
        parts = l.split("] ", 1)[1].split("  ")                            # "'t123' -0.0123" per candidate
        vals = [float(p.rsplit(" ", 1)[1]) for p in parts]
        assert len(vals) == 3 and all(v <= 0.0 for v in vals) and vals == sorted(vals, reverse=True)
        assert all(p.startswith("'t") for p in parts)


# ---------------------------------------------------------------------------------------------------------------------
# full-size dims (synthetic peaked untied head, clips vetted in test_gpu_parity.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_size_0p6b_top_logprobs(report):
    """0.6B dims: batch 1 x 30 s (fused single-sequence step) and batch 8 x 30 s (batched step), 16 new tokens; ids
    and path counters identical with the option off."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth
    cfg = O.cfg_0p6b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 1, peaked_head=True)
    ecfg = config_0p6b()
    ecfg.text.tie_word_embeddings = False
    model = O.OracleModel(cfg, w)
    n_new = 16
    clips = [synth.make_clip(i, 30.0) for i in (1, 3, 4, 6, 7, 8, 10, 17)]
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        runs = {}
        for key, sel in (("b8", clips), ("b1", clips[:1])):
            for k in (0, K):
                s0 = _steps(eng.stats())
                r = eng.transcribe_ids(sel, max_new_tokens=n_new, top_logprobs=k)
                s1 = _steps(eng.stats())
                runs[key, k] = (r, {m: s1[m] - s0[m] for m in s0})
    finally:
        eng.close()
    for key, path in (("b8", "decode_batch_steps"), ("b1", "decode_fused_steps")):
        (off, m_off), (on, m_on) = runs[key, 0], runs[key, K]
        assert on.ids == off.ids and m_on == m_off
        assert m_on[path] == on.decode_steps and m_on["decode_phase_steps"] == 0
    st = {"b1": Stats(), "b8": Stats()}
    for b, c in enumerate(clips):
        ref = O.transcribe_ids(model, c, max_new_tokens=n_new, keep_logits=True, lm_head_all_rows=False)
        for key in (("b1", "b8") if b == 0 else ("b8",)):
            r = runs[key, K][0]
            assert r.ids[b] == ref.ids, (key, b)
            _check_against_logprobs(r, b)
            st[key].add(_check_vs_ref(r.top_logprobs[b], r.eos_top_logprobs[b], ref, n_new))
    _report(report, "full_0p6b_b1", st["b1"])
    _report(report, "full_0p6b_b8", st["b8"])


@pytest.mark.gpu
def test_full_size_1p7b_top_logprobs(report):
    """1.7B dims (K = 2048 lm_head: the generic GEMV form of the fused step), seed 3, clip 7, 16 new tokens."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_1p7b, synth
    cfg = O.cfg_1p7b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 3, peaked_head=True)
    ecfg = config_1p7b()
    ecfg.text.tie_word_embeddings = False
    x = synth.make_clip(7, 30.0)
    n_new = 16
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        off = eng.transcribe_ids([x], max_new_tokens=n_new)
        s0 = eng.stats()
        got = eng.transcribe_ids([x], max_new_tokens=n_new, top_logprobs=K)
        st = eng.stats()
    finally:
        eng.close()
    assert got.ids == off.ids
    assert st["decode_phase_steps"] == s0["decode_phase_steps"] == 0
    assert st["decode_fused_steps"] - s0["decode_fused_steps"] == got.decode_steps
    ref = O.transcribe_ids(O.OracleModel(cfg, w), x, max_new_tokens=n_new, keep_logits=True, lm_head_all_rows=False)
    assert got.ids[0] == ref.ids
    _check_against_logprobs(got, 0)
    _report(report, "full_1p7b", _check_vs_ref(got.top_logprobs[0], got.eos_top_logprobs[0], ref, n_new))
