"""Precision against a float64 oracle: every output's error is bounded by that of an fp32 implementation.

DESIGN.md section 2 promises that activations behave like fp32.  For each output Y of a path this file measures

    e_gpu = err(Y_gpu, Y_64)        e_32 = err(Y_oracle_fp32, Y_64)

with Y_64 the same computation in float64 (oracle.OracleModel(dtype=torch.float64): bf16 weights widened exactly,
f32 samples widened, rope and position tables kept in f64), and passes when e_gpu <= R * max(e_32, floor).  The fp32
calibration uses the same inputs and, for decode, the same ids (oracle.score_ids in fp32 on the GPU's own ids), so
the bound calibrates itself.  err is max|y - y64| / max|y64| for stage outputs (mel, encoder output, logits; at least
one whole encoder output or vocabulary row), and max|y - y64| in nats for recorded log-probabilities (every entry of
every step).  The floor is the fp32 rounding of the output itself: 2^-23 relative, or the fp32 ulp of the largest
|log-probability|.

R = 4.  On an H100 the real build's worst output sits at about 3 x e_32 (prefill logits), the decode records at
0.8-1.5 x.  The planes=2 and planes=1 sessions below (encoder and prefill GEMMs fed with fewer bf16 planes) are committed
negative controls that must FAIL the rule, which shows the rule can see one lost plane: planes=2 measured 4.4-7.7 x,
planes=1 thousands.  The planes=2 margin is small because the GEMM producers split round-to-nearest (split3 in
common.cuh): hi + mid then carries about 17 significant bits, and dropping lo costs only ~2^-17 per activation.  The
same loss simulated in the fp32 oracle (every Linear and conv input kept as two bf16 planes, tiny config, clip 60 of
6.2 s) gives 7.7 x (encoder) / 5.4 x (prefill) with a round-to-nearest split, the GPU's 7.7 x / 5.3 x, and 36 x / 28 x
with a truncating split, which keeps ~16 bits with a one-sided error.  So a small planes=2 ratio is what the kernels'
split predicts, not a weak metric.  Each check writes e_gpu, e_32, the floor and the ratio into the report.
"""
import contextlib
import gc

import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth

R = 4.0
EPS32 = 2.0 ** -23
K = 8                                   # top_logprobs recorded per step
EOS = (151643, 151645)


# ---------------------------------------------------------------------------------------------------------------------
# the rule
# ---------------------------------------------------------------------------------------------------------------------
class Err:
    """Running maxima over many values of one output: |y - y64|, |y32 - y64| and |y64| (for relative errors).
    Every value must be finite: a NaN would otherwise vanish from a running maximum (nan > x is False)."""

    def __init__(self, relative: bool):
        self.relative, self.d_gpu, self.d_32, self.scale, self.n = relative, 0.0, 0.0, 0.0, 0

    def add(self, y, y32, y64):
        y, y32, y64 = (np.asarray(a, np.float64) for a in (y, y32, y64))
        assert y.shape == y32.shape == y64.shape, (y.shape, y32.shape, y64.shape)
        for name, a in (("output", y), ("fp32 reference", y32), ("fp64 reference", y64)):
            assert np.isfinite(a).all(), f"{np.count_nonzero(~np.isfinite(a))} non-finite values in the {name}"
        self.d_gpu = max(self.d_gpu, float(np.abs(y - y64).max()))
        self.d_32 = max(self.d_32, float(np.abs(y32 - y64).max()))
        self.scale = max(self.scale, float(np.abs(y64).max()))
        self.n += y64.size
        return self

    def merge(self, o: "Err"):
        self.d_gpu, self.d_32, self.scale = max(self.d_gpu, o.d_gpu), max(self.d_32, o.d_32), max(self.scale, o.scale)
        self.n += o.n
        return self

    def result(self):
        """(e_gpu, e_32, floor)."""
        if self.relative:
            s = max(self.scale, 1e-30)
            return self.d_gpu / s, self.d_32 / s, EPS32
        return self.d_gpu, self.d_32, float(np.spacing(np.float32(self.scale)))


def ratio(report, key, err: Err, min_values: int = 300) -> float:
    """e_gpu / max(e_32, floor), written with its parts into the report."""
    assert err.n >= min_values, (key, err.n)
    e_gpu, e_32, floor = err.result()
    r = e_gpu / max(e_32, floor)
    report[f"fp64_{key}"] = {"e_gpu": e_gpu, "e_32": e_32, "floor": floor, "ratio": r, "values": err.n}
    return r


def check(report, key, err: Err) -> None:
    r = ratio(report, key, err)
    assert r <= R, (key, report[f"fp64_{key}"])


def rel_err(y, y64) -> float:
    y64 = np.asarray(y64, np.float64)
    return float(np.abs(np.asarray(y, np.float64) - y64).max() / np.abs(y64).max())


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle itself
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny64(tiny):
    cfg, w, _ = tiny
    return O.OracleModel(cfg, w, dtype=torch.float64)


def test_score_ids_reproduces_greedy_logits(tiny):
    """fp32 score_ids on the oracle's own greedy ids: argmax of every row is the id, and the logits are those of the
    KV-cache loop of transcribe_ids to 1e-5 of max|logit|."""
    _, _, model = tiny
    x = synth.make_clip(60, 6.2)
    ref = O.transcribe_ids(model, x, max_new_tokens=12, keep_logits=True)
    got = O.score_ids(model, x, ref.ids)
    want = torch.stack([ref.prefill_logits] + ref.step_logits)
    assert got.dtype == torch.float32 and got.shape == want.shape == (len(ref.ids) + 1, model.cfg.text.vocab_size)
    assert got[: len(ref.ids)].argmax(-1).tolist() == ref.ids
    assert rel_err(got.numpy(), want.numpy()) <= 1e-5


def test_score_ids_with_language_suffix(tiny):
    _, _, model = tiny
    x = synth.make_clip(81, 2.5)
    lang = [11528, 6364]
    ref = O.transcribe_ids(model, x, language_ids=lang, max_new_tokens=6, keep_logits=True)
    got = O.score_ids(model, x, ref.ids, language_ids=lang)
    assert got[: len(ref.ids)].argmax(-1).tolist() == ref.ids
    assert rel_err(got.numpy(), torch.stack([ref.prefill_logits] + ref.step_logits).numpy()) <= 1e-5


def test_fp32_oracle_error_against_fp64(tiny, tiny64, report):
    """The fp32 oracle sits at the fp32 level of the fp64 one (about 1e-6 relative on the tiny config): far below the
    existing tolerances, and far above what float64 itself would show (a failed widening would read 0 or ~1e-16)."""
    _, _, m32 = tiny
    x = synth.make_clip(60, 6.2)
    mel32, mel64 = O.extract_mel(x), O.extract_mel(x, dtype=torch.float64)
    assert mel64.dtype == torch.float64
    enc32, enc64 = m32.encode(mel32), tiny64.encode(mel64)
    assert enc64.dtype == torch.float64
    ids = O.transcribe_ids(m32, x, max_new_tokens=8).ids
    s32, s64 = O.score_ids(m32, x, ids), O.score_ids(tiny64, x, ids)
    assert s64.dtype == torch.float64
    errs = {"mel": rel_err(mel32, mel64), "encoder": rel_err(enc32, enc64), "prefill": rel_err(s32[0], s64[0]),
            "steps": rel_err(s32[1:], s64[1:])}
    report["fp64_cpu_fp32_oracle_rel_err"] = errs
    assert 1e-7 <= errs["encoder"] <= 5e-6 and 1e-7 <= errs["prefill"] <= 5e-6 and 1e-7 <= errs["steps"] <= 5e-6, errs
    assert 1e-7 <= errs["mel"] <= 1e-4, errs           # log10 of small band powers amplifies the FFT's rounding


def test_default_dtype_tables_are_fp32():
    """The f64 tables are the f32 ones before rounding."""
    c32, s32 = O.mrope_cos_sin([[0, 5, 700]] * 3, 128, 1e6, (24, 20, 20), False)
    c64, s64 = O.mrope_cos_sin([[0, 5, 700]] * 3, 128, 1e6, (24, 20, 20), False, dtype=torch.float64)
    assert c32.dtype == torch.float32 and c64.dtype == torch.float64
    assert torch.equal(c64.float(), c32) and torch.equal(s64.float(), s32) and not torch.equal(c64, c32.double())
    p32, p64 = O.sinusoid_table(100, 128), O.sinusoid_table(100, 128, torch.float64)
    assert p32.dtype == torch.float32 and torch.equal(p64.float(), p32)
    assert O.causal_mask(3, 2, torch.float64).dtype == torch.float64 and torch.equal(O.causal_mask(3, 2, torch.float64).float(),
                                                                                     O.causal_mask(3, 2))


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", [0, 1, 2])
def test_rule_rejects_non_finite_values(bad, where):
    """A NaN or inf in the output or in either reference fails the check, wherever it is and whatever came before."""
    rng = np.random.default_rng(0)
    y64 = rng.standard_normal(400)
    good = Err(True).add(y64 + 1e-4, y64 + 1e-4, y64)
    assert ratio({}, "rule_sanity", good) == pytest.approx(1.0)
    arrs = [y64 + 1e-4, y64 + 1e-4, y64.copy()]
    arrs[where][17] = bad
    with pytest.raises(AssertionError, match="non-finite"):
        good.add(*arrs)
    with pytest.raises(AssertionError, match="non-finite"):
        Err(False).add(*arrs)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


@contextlib.contextmanager
def options(eng, **opts):
    """Session options for the block.  Afterwards each key goes back to the engine's configured value; a key that had
    none is dropped and the session freed, so that the next call creates one with the library's own default (its
    ASRB_* environment overrides included).  Blocks nest."""
    from qwen3_asr_rs_b200 import _lib
    prior = {k: eng._options.get(k) for k in opts}
    for k, v in opts.items():
        eng.set_option(k, v)
    try:
        yield
    finally:
        for k, v in prior.items():
            if v is not None:
                eng.set_option(k, v)
            else:
                eng._options.pop(k)
        if None in prior.values() and eng._session is not None:
            _lib.check(eng._lib.asrb_session_free(eng._session))
            eng._session, eng._cap = None, None


@pytest.fixture(scope="module")
def eng(tiny):
    """Own tiny engine (the shared tiny_engine's options stay untouched)."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    e = AsrInference.from_weights(config_tiny(), w, device=0)
    yield e
    e.close()


def stage_run(e, clips, n_steps=5, context=None):
    """GPU stage calls: (mels, encoder outputs, prefill logits [B, V], per step logits [n, B, V], ids [B][n])."""
    mels = e.mel(clips, max_context=max((len(c) for c in context or [] if c), default=0))
    if context is not None:
        e.set_context(context)
    try:
        enc = e.encode()
        _, pre = e.prefill()
        steps, ids = [], [[] for _ in clips]
        for _ in range(n_steps):
            nxt, lg = e.decode_step()
            steps.append(lg)
            for b, t in enumerate(nxt):
                ids[b].append(int(t))
    finally:
        if context is not None:
            e.set_context(None)
    return mels, enc, pre, steps, ids


def stage_errs(m32, m64, clips, got, n_steps=5):
    """Err per stage output, maxima over the batch."""
    mels, enc, pre, steps, ids = got
    out = {k: Err(True) for k in ("mel", "encoder", "prefill", "steps")}
    for b, x in enumerate(clips):
        mel32, mel64 = O.extract_mel(x), O.extract_mel(x, dtype=torch.float64)
        out["mel"].add(mels[b], mel32, mel64)
        out["encoder"].add(enc[b], m32.encode(mel32), m64.encode(mel64))
        s32, s64 = O.score_ids(m32, x, ids[b]).numpy(), O.score_ids(m64, x, ids[b]).numpy()
        out["prefill"].add(pre[b], s32[0], s64[0])
        for i in range(n_steps):
            out["steps"].add(steps[i][b], s32[i + 1], s64[i + 1])
    return out


STAGE_CLIPS = [("single_chunk_0.6s", [(31, 0.6)]), ("tail_chunk_8.5s", [(31, 8.5)]),
               ("windowed_11.55s", [(31, 11.55)]), ("windowed_30s", [(31, 30.0)]),
               ("ragged_b4", [(50 + i, s) for i, s in enumerate([3.3, 12.0, 0.9, 17.5])])]


@pytest.mark.gpu
@pytest.mark.parametrize("label,sel", STAGE_CLIPS, ids=[c[0] for c in STAGE_CLIPS])
def test_stage_outputs_tiny(tiny, tiny64, eng, report, label, sel):
    """Mel, encoder output, prefill logits and 5 per-phase decode_step logits: a single chunk, a tail chunk, more than
    8 chunks (windowed encoder attention), a ragged batch of 4."""
    _, _, m32 = tiny
    clips = [synth.make_clip(i, s) for i, s in sel]
    errs = stage_errs(m32, tiny64, clips, stage_run(eng, clips))
    for k, e in errs.items():
        ratio(report, f"tiny_{label}_{k}", e)
    for k, e in errs.items():
        check(report, f"tiny_{label}_{k}", e)


@pytest.mark.gpu
def test_stage_outputs_simt_gemm(tiny, tiny64, eng, report):
    """Positive control: the in-library SIMT GEMM meets the same bound."""
    _, _, m32 = tiny
    clips = [synth.make_clip(31, 11.55), synth.make_clip(52, 0.9)]
    with options(eng, gemm="simt"):
        eng.mel(clips)                                    # session sized before the counters are read
        tc0 = eng.stats()["gemm_tc_launches"]
        got = stage_run(eng, clips)
        assert eng.stats()["gemm_tc_launches"] == tc0     # no tensor-core GEMM ran
    for k, e in stage_errs(m32, tiny64, clips, got).items():
        check(report, f"tiny_simt_{k}", e)


def _planes_errs(m32, m64, e, clips):
    """(encoder Err, prefill Err) of the GPU run."""
    mels, enc, pre, _, _ = stage_run(e, clips, n_steps=0)
    enc_e, pre_e = Err(True), Err(True)
    for b, x in enumerate(clips):
        mel32, mel64 = O.extract_mel(x), O.extract_mel(x, dtype=torch.float64)
        enc_e.add(enc[b], m32.encode(mel32), m64.encode(mel64))
        pre_e.add(pre[b], O.score_ids(m32, x, [])[0].numpy(), O.score_ids(m64, x, [])[0].numpy())
    return enc_e, pre_e


@pytest.mark.gpu
@pytest.mark.parametrize("planes", ["2", "1"])
def test_negative_control_lost_planes_tiny(tiny, tiny64, eng, report, planes):
    """Encoder and prefill GEMMs fed with 2 or 1 bf16 planes per activation must FAIL the rule."""
    _, _, m32 = tiny
    clips = [synth.make_clip(60, 6.2)]
    with options(eng, planes=planes):
        enc_e, pre_e = _planes_errs(m32, tiny64, eng, clips)
    for name, e in (("encoder", enc_e), ("prefill", pre_e)):
        r = ratio(report, f"tiny_planes{planes}_{name}", e)
        assert r > R, (planes, name, report[f"fp64_tiny_planes{planes}_{name}"])


# ---- shared-context prefill ----------------------------------------------------------------------------------------
@contextlib.contextmanager
def context_prompt(ctx):
    """oracle.build_prompt with `ctx` inserted after `<|im_start|>system\\n` (as test_context.py)."""
    orig = O.build_prompt

    def build(num_audio_tokens, language_ids=None):
        toks, a0 = orig(num_audio_tokens, language_ids)
        return toks[:3] + list(ctx) + toks[3:], a0 + len(ctx)
    O.build_prompt = build
    try:
        yield
    finally:
        O.build_prompt = orig


@pytest.mark.gpu
def test_shared_context_prefill(tiny, tiny64, eng, report):
    """Contexts [A, A] at batch 2: the follower's prefix K/V comes from the leader's fan-out; its prefill logits meet
    the bound as the leader's do."""
    _, _, m32 = tiny
    A = [int(v) for v in np.random.default_rng(5).integers(0, 150000, 37)]
    clips = [synth.make_clip(81, 2.5), synth.make_clip(82, 9.1)]
    _, _, pre, _, _ = stage_run(eng, clips, n_steps=0, context=[A, A])
    st = eng.last_prefill_stats()
    assert st["rows_shared"] == len(A) + 9 and st["fanout_kv_bytes"] > 0
    with context_prompt(A):
        for b, role in ((0, "leader"), (1, "follower")):
            e = Err(True).add(pre[b], O.score_ids(m32, clips[b], [])[0].numpy(), O.score_ids(tiny64, clips[b], [])[0].numpy())
            check(report, f"tiny_context_{role}_prefill", e)


# ---- fused decode records ------------------------------------------------------------------------------------------
def _processed_log_softmax(logits, ids, rep):
    """log_softmax of every row of score_ids([T + 1, V], float64); with rep = (N, theta) != (0, 1), row t first processed
    by the repetition controls with history ids[:t] (test_repetition.process)."""
    if rep == (0, 1.0):
        return torch.log_softmax(logits, -1).numpy()
    from test_repetition import process
    l = logits.numpy()
    return torch.log_softmax(torch.from_numpy(np.stack([process(l[t], ids[:t], *rep) for t in range(len(l))])), -1).numpy()


def record_errs(m32, m64, clips, r, top: bool, rep=(0, 1.0), seqs=None, scores=None):
    """Err of the recorded log-probabilities against log_softmax of score_ids at the GPU's own ids: with `top`, every
    entry (id, lp) of every top-k row, EOS step included; else the log-probability of each id and of the ending EOS.
    rep = (no_repeat_ngram_size, repetition_penalty): against the processed logits.  `seqs`: the sequences checked (all
    by default); `scores(b, ids)`: (fp32, fp64) score_ids of sequence b, for a caller that caches them."""
    err = Err(False)
    for b in range(len(clips)) if seqs is None else seqs:
        x, ids = clips[b], r.ids[b]
        s32, s64 = scores(b, ids) if scores else (O.score_ids(m32, x, ids), O.score_ids(m64, x, ids))
        l32 = _processed_log_softmax(s32.double(), ids, rep)
        l64 = _processed_log_softmax(s64, ids, rep)
        if top:
            rows = list(r.top_logprobs[b]) + ([r.eos_top_logprobs[b]] if r.eos_top_logprobs[b] is not None else [])
            assert len(rows) >= len(ids) and all(row[0][0] == t for row, t in zip(rows, ids))
            for t, row in enumerate(rows):
                cand = np.array([c[0] for c in row])
                err.add(np.array([c[1] for c in row]), l32[t, cand], l64[t, cand])
        else:
            got = list(r.logprobs[b]) + ([r.eos_logprobs[b]] if r.eos_logprobs[b] is not None else [])
            drawn = list(ids)
            if r.eos_logprobs[b] is not None:
                # Which of the two EOS ids the sampler drew is not part of the record.  The nearer one is taken, and
                # only when the two candidates lie 0.01 nats apart (about 1000 x the errors of these tiny-config
                # records), so that the recorded value can be within the bound of at most one of them.
                t = len(ids)
                assert abs(l64[t, EOS[0]] - l64[t, EOS[1]]) >= 1e-2, (b, l64[t, list(EOS)])
                drawn.append(min(EOS, key=lambda i: abs(l64[t, i] - r.eos_logprobs[b])))
            rows = np.arange(len(drawn))
            err.add(np.array(got), l32[rows, drawn], l64[rows, drawn])
    return err


def run_path(e, clips, n_new, opts, path, **kw):
    """Warm-up (session sized, graphs captured), then the measured run; asserts the decode path that ran."""
    with options(e, **opts):
        e.transcribe_ids(clips, max_new_tokens=n_new, **kw)
        s0 = _steps(e.stats())
        r = e.transcribe_ids(clips, max_new_tokens=n_new, **kw)
        s1 = _steps(e.stats())
    moved = {k: s1[k] - s0[k] for k in s0}
    if path == "decode_phase_steps":
        assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0
        assert r.kernels_launched > 2 * r.decode_steps
    elif path == "handover":
        assert moved["decode_fused_steps"] > 0 and r.kernels_launched > 2 * r.decode_steps
    else:
        assert moved[path] == r.decode_steps and moved["decode_phase_steps"] == 0
    return r


# (label, clips (index, seconds), new tokens, options, path whose counter must move): those of test_logprobs.py, and
# the hand-over past the fused step's 1152 keys (60 s prompt, 400 tokens)
PATHS = [
    ("fused_single", [(70, 4.0)], 48, {}, "decode_fused_steps"),
    ("fused_per_seq_b5", [(80 + i, s) for i, s in enumerate([2.5, 9.1, 5.0, 1.2, 3.3])], 16, {"batch_step": "0"}, "decode_fused_steps"),
    ("batched_nb8", [(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])], 14, {}, "decode_batch_steps"),
    ("batched_nb16", [(200 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9, 5.3, 1.4, 2.8])], 10, {}, "decode_batch_steps"),
    ("phases", [(71, 12.3), (72, 0.8)], 24, {"decode": "phases"}, "decode_phase_steps"),
    ("handover_60s", [(302, 60.0)], 400, {}, "handover"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("label,sel,n_new,opts,path", PATHS, ids=[p[0] for p in PATHS])
def test_top_logprobs_records_tiny(tiny, tiny64, eng, report, label, sel, n_new, opts, path):
    _, _, m32 = tiny
    clips = [synth.make_clip(i, s) for i, s in sel]
    r = run_path(eng, clips, n_new, opts, path, top_logprobs=K)
    check(report, f"tiny_top{K}_{label}", record_errs(m32, tiny64, clips, r, top=True))


@pytest.mark.gpu
@pytest.mark.parametrize("label", ["fused_single", "batched_nb8"])
def test_sampled_logprobs_tiny(tiny, tiny64, eng, report, label):
    """temperature 0.7: the record is the temperature-1 log-probability of the drawn id (raw-logit merge).  The fused
    single-sequence step runs 7 clips one at a time, the batched step 8 clips at once: 48 tokens each."""
    _, _, m32 = tiny
    clips = [synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])]
    kw = dict(temperature=0.7, seed=1234, logprobs=True)
    if label == "fused_single":
        err = Err(False)
        for x in clips[:7]:
            r = run_path(eng, [x], 48, {}, "decode_fused_steps", **kw)
            err.merge(record_errs(m32, tiny64, [x], r, top=False))
    else:
        err = record_errs(m32, tiny64, clips, run_path(eng, clips, 48, {}, "decode_batch_steps", **kw), top=False)
    check(report, f"tiny_sampled_T0.7_{label}", err)


# ---------------------------------------------------------------------------------------------------------------------
# GPU, Qwen3-ASR-0.6B dims (synthetic weights, peaked untied head): split-K GEMMs, conv implicit GEMM at real channel
# counts, the fused steps' 0.6B instantiations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    """(fp32 oracle, fp64 oracle, engine); the fp64 weights (about 8 GB of host memory) are freed after the module."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 1, peaked_head=True)
    ecfg = config_0p6b()
    ecfg.text.tie_word_embeddings = False
    e = AsrInference.from_weights(ecfg, w, device=0)
    m32, m64 = O.OracleModel(cfg, w), O.OracleModel(cfg, w, dtype=torch.float64)
    del w
    yield m32, m64, e
    e.close()
    del m32, m64
    gc.collect()


FULL_CLIP = (9, 10.0)
FULL_B8 = [(600 + i, s) for i, s in enumerate([2.1, 3.4, 1.3, 4.0, 2.7, 0.9, 3.1, 1.8])]


@pytest.mark.gpu
def test_stage_outputs_0p6b(full, report):
    m32, m64, e = full
    clips = [synth.make_clip(*FULL_CLIP)]
    for k, err in stage_errs(m32, m64, clips, stage_run(e, clips)).items():
        check(report, f"0p6b_b1_{k}", err)


@pytest.mark.gpu
def test_prefill_logits_0p6b_ragged_b8(full, report):
    m32, m64, e = full
    clips = [synth.make_clip(i, s) for i, s in FULL_B8]
    _, _, pre, _, _ = stage_run(e, clips, n_steps=0)
    err = Err(True)
    for b, x in enumerate(clips):
        err.add(pre[b], O.score_ids(m32, x, [])[0].numpy(), O.score_ids(m64, x, [])[0].numpy())
    check(report, "0p6b_b8_prefill", err)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 8])
def test_top_logprobs_records_0p6b(full, report, batch):
    """Fused single-sequence step (batch 1) and batched step (batch 8), 64 new tokens."""
    m32, m64, e = full
    clips = [synth.make_clip(*FULL_CLIP)] if batch == 1 else [synth.make_clip(i, s) for i, s in FULL_B8]
    r = run_path(e, clips, 64, {}, "decode_fused_steps" if batch == 1 else "decode_batch_steps", top_logprobs=K)
    steps = [len(rows) + (eos is not None) for rows, eos in zip(r.top_logprobs, r.eos_top_logprobs)]
    assert min(steps) >= 64, steps                   # every sequence contributes 64 recorded steps
    check(report, f"0p6b_top{K}_b{batch}", record_errs(m32, m64, clips, r, top=True))


@pytest.mark.gpu
@pytest.mark.parametrize("planes", ["2", "1"])
def test_negative_control_lost_planes_0p6b(full, report, planes):
    m32, m64, e = full
    clips = [synth.make_clip(*FULL_CLIP)]
    with options(e, planes=planes):
        enc_e, pre_e = _planes_errs(m32, m64, e, clips)
    for name, err in (("encoder", enc_e), ("prefill", pre_e)):
        r = ratio(report, f"0p6b_planes{planes}_{name}", err)
        assert r > R, (planes, name, report[f"fp64_0p6b_planes{planes}_{name}"])
