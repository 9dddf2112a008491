"""Every record variant of the decode steps, at every width they are compiled for, under DESIGN.md section 2's rule.

The fused steps are compiled per model width and per record variant: decode_step_kernel (decode_mega.cu, one launch per
sequence) for the tiny, 0.6B and 1.7B widths, decode_batch_kernel (decode_batch.cu) for the tiny and 0.6B widths at
NB = 8 and 16, each in ten variants (greedy, log-probability record, top-8 candidates, sampling, sampling with the
log-probability record; each with or without the repetition controls).  The per-phase path (decode.cu) walks
sub-batches of 8 and the batched step passes of 16; both offset every buffer and the sampling draw's row by the
sub-batch's first sequence.  The MATRIX below runs the ten variants on each (model, row), and test_every_instantiation
_has_a_cell derives the instantiation list from the sources so that a new one without a row fails on a CPU host.

The kernel a model runs is chosen by (hidden, q_dim, intermediate) alone, and the fused steps take up to 32 layers, so
the models here keep the production widths and vocabulary with 4 encoder and 4 decoder layers: they run exactly the
production kernels with a cheap oracle.  Each has an untied peaked head (synth.make_weights) so that ids can be pinned.

Per cell: the ids of every sequence equal the oracle's selection (test_repetition.rep_oracle: the argmax, or the
Philox/Gumbel draw at the sequence's global row, of the processed float64-widened logits) on every step whose gap clears
GAP_FLOOR, and at least half of each row's steps are so pinned; the record variants select bitwise the ids of the
variant without the record; top-8 entry 0 is bitwise the log-probability record; the log-probability, top-8 and sampled
log-probability records meet R = 4 against float64 (processed with the repetition controls on) at the GPU's own ids, on
the sequences at the pass and sub-batch boundaries; with the controls on, no output repeats an N-gram, no candidate is a
banned id, and some sequence's ids differ from the run without them.

The CPU tests show that the checks can fail: an oracle that loses the pass / sub-batch row offset of the draw selects
other pinned ids, and records computed from unprocessed logits or, for sampled ids, with the greedy formula -log S
fail the rule.
"""
import gc
import os
import re
import resource
import time
from contextlib import contextmanager
from dataclasses import dataclass
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth
from test_precision_fp64 import R, Err, _planes_errs, _steps, check, options, ratio, record_errs, stage_errs, stage_run
from test_repetition import assert_pinned, process, rep_oracle, repeated_ngrams
from test_sampling import gumbel
from test_top_logprobs import _check_against_logprobs

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "qwen3_asr_rs_b200", "csrc")
T = 0.7
REP_GREEDY = (3, 1.3)           # (no_repeat_ngram_size, repetition_penalty) of the greedy variants
REP_SAMPLE = (2, 1.2)           # and of the sampling ones (test_repetition.py's values)
MIN_RECORDS = 20


# ---------------------------------------------------------------------------------------------------------------------
# models, rows, variants
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Model:
    """A production configuration (or the tiny one) cut to `layers` encoder and decoder layers, untied peaked head."""
    base: str
    seed: int
    layers: int = 0

    def configs(self):
        """(oracle config, engine config) from the one description."""
        from qwen3_asr_rs_b200 import config_0p6b, config_1p7b, config_tiny
        ocfg, ecfg = {"0p6b": (O.cfg_0p6b, config_0p6b), "1p7b": (O.cfg_1p7b, config_1p7b),
                      "tiny": (O.cfg_tiny, config_tiny)}[self.base]
        ocfg, ecfg = ocfg(), ecfg()
        for cfg in (ocfg, ecfg):
            cfg.text.tie_word_embeddings = False
            if self.layers:
                cfg.text.num_hidden_layers = cfg.audio.encoder_layers = self.layers
        for part in ("audio", "text"):
            o, e = getattr(ocfg, part), getattr(ecfg, part)
            assert all(getattr(o, k) == getattr(e, k) for k in o.__dataclass_fields__), (self, part)
        return ocfg, ecfg

    def dims(self):
        t = self.configs()[0].text
        return t.hidden_size, t.num_attention_heads * t.head_dim, t.intermediate_size


MODELS = {"w0p6b": Model("0p6b", 1, 4), "w1p7b": Model("1p7b", 3, 4), "tiny": Model("tiny", 7)}


def _clips(first: int, n: int):
    """n clips of 0.7 .. 3 s."""
    return [(first + i, round(0.7 + (0.37 * i * 7) % 2.3, 2)) for i in range(n)]


# row -> (clips (index, seconds), new tokens, session options, path whose counter must move, launches of the step per
# decode step or None)
ROWS = {
    "fused_single": (_clips(700, 1), 48, {}, "decode_fused_steps", 1),
    "fused_per_seq_b3": (_clips(710, 3), 32, {}, "decode_fused_steps", 3),           # 1.7B has no batched step
    "batched_nb8": (_clips(720, 5), 32, {}, "decode_batch_steps", 1),
    "batched_nb16": (_clips(730, 12), 24, {}, "decode_batch_steps", 1),
    "batched_b20": (_clips(750, 20), 24, {}, "decode_batch_steps", 2),               # an NB 16 pass, then an NB 8 pass
    "phases_b11": (_clips(780, 11), 24, {"decode": "phases"}, "decode_phase_steps", None),   # sub-batches 8 + 3
    "handover": ([(790, 60.0)], 280, {}, "handover", None),    # 60 s prompt + 280 ids: past the fused step's 1024 keys
}
MATRIX = [("tiny", "fused_single"), ("w0p6b", "fused_single"), ("w1p7b", "fused_single"),
          ("w1p7b", "fused_per_seq_b3"),
          ("w0p6b", "batched_nb8"),
          ("w0p6b", "batched_nb16"), ("tiny", "batched_nb16"),
          ("w0p6b", "batched_b20"), ("tiny", "batched_b20"),
          ("w0p6b", "phases_b11"), ("w1p7b", "phases_b11"), ("tiny", "phases_b11"),
          ("w0p6b", "handover"), ("w1p7b", "handover")]
# the sampling seed of each cell: picked on the CPU so that at least half of the row's steps are pinned
SEEDS = {cell: 5 for cell in MATRIX}
SEEDS["w1p7b", "handover"] = 1          # seed 5 pins only the first 116 of 300 sampled steps
# sequences whose records are checked: the pass (16) and sub-batch (8) boundaries; every sequence in the other rows
RECORD_SEQS = {"batched_b20": [0, 7, 8, 15, 16, 19], "phases_b11": [0, 7, 8, 10], "batched_nb16": [0, 8, 11]}

# (name, transcribe_ids options, (LP, TK, SM) of the kernel step_fn / batch_fn select for them)
VARIANTS = [("greedy", {}, (False, False, False)),
            ("logprob", {"logprobs": True}, (True, False, False)),
            ("top8", {"top_logprobs": 8}, (True, True, False)),
            ("sample", {"temperature": T}, (False, False, True)),
            ("sample_logprob", {"temperature": T, "logprobs": True}, (True, False, True))]


def variant_kw(name: str, rep: bool, seed: int) -> dict:
    kw = dict(next(v[1] for v in VARIANTS if v[0] == name))
    sampling = "temperature" in kw
    if sampling:
        kw["seed"] = seed
    if rep:
        kw["no_repeat_ngram_size"], kw["repetition_penalty"] = REP_SAMPLE if sampling else REP_GREEDY
    return kw


def rep_of(name: str, rep: bool):
    return (REP_SAMPLE if name.startswith("sample") else REP_GREEDY) if rep else (0, 1.0)


def cell_instantiations(model: str, row: str):
    """The fused-step instantiations (kernel, dims, NB) a cell runs: NB 0 is the single-sequence step."""
    d = MODELS[model].dims()
    path, n = ROWS[row][3], len(ROWS[row][0])
    if path in ("decode_fused_steps", "handover"):
        return {("decode_step_kernel", d, 0)}
    if path == "decode_batch_steps":
        return {("decode_batch_kernel", d, 8 if min(16, n - b0) <= 8 else 16) for b0 in range(0, n, 16)}
    return set()


# ---------------------------------------------------------------------------------------------------------------------
# oracles and engines, built once per module; oracle results cached by (model, clip, ids / selection)
# ---------------------------------------------------------------------------------------------------------------------
class Zoo:
    def __init__(self):
        self.oracle, self.engines, self.traj, self.score, self.clip = {}, {}, {}, {}, {}

    def oracles(self, name):
        if name not in self.oracle:
            ocfg, _ = MODELS[name].configs()
            w = synth.make_weights(ocfg, MODELS[name].seed, peaked_head=True)
            self.oracle[name] = (O.OracleModel(ocfg, w), O.OracleModel(ocfg, w, dtype=torch.float64), w)
        return self.oracle[name][:2]

    def engine(self, name):
        if name not in self.engines:
            from qwen3_asr_rs_b200 import AsrInference
            self.oracles(name)
            self.engines[name] = AsrInference.from_weights(MODELS[name].configs()[1], self.oracle[name][2], device=0)
        return self.engines[name]

    def samples(self, sel):
        if sel not in self.clip:
            self.clip[sel] = synth.make_clip(*sel)
        return self.clip[sel]

    def trajectory(self, name, sel, rep, n_new, temperature=0.0, seed=0, row=0):
        """rep_oracle on the fp32 oracle: the processed argmax (temperature 0) or the draw at global row `row`."""
        key = (name, sel, rep, n_new, temperature, seed if temperature else 0, row if temperature else 0)
        if key not in self.traj:
            self.traj[key] = rep_oracle(self.oracles(name)[0], self.samples(sel), *rep, n_new, temperature=temperature,
                                        seed=seed, row=row)
        return self.traj[key]

    def scores(self, name, sel, ids):
        key = (name, sel, tuple(ids))
        if key not in self.score:
            m32, m64 = self.oracles(name)
            x = self.samples(sel)
            with torch.no_grad():
                self.score[key] = (O.score_ids(m32, x, ids), O.score_ids(m64, x, ids))
        return self.score[key]

    def close(self):
        for e in self.engines.values():
            e.close()
        self.oracle, self.engines, self.traj, self.score = {}, {}, {}, {}
        gc.collect()


@pytest.fixture(scope="module")
def zoo():
    z = Zoo()
    yield z
    z.close()


@contextmanager
def collect(fails, label):
    """Run a check; a failed assertion is kept (with `label`) and the cell goes on, so that one run reports every
    failing variant."""
    try:
        yield
    except AssertionError as ex:
        fails.append(f"{label}: {ex}")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: coverage of the compiled variants
# ---------------------------------------------------------------------------------------------------------------------
def _body(src: str, signature: str) -> str:
    i = src.index(signature)
    return src[i:src.index("\n}\n", i)]


def compiled_instantiations():
    """{(kernel, (hidden, q_dim, intermediate), NB, (LP, TK, SM, RP))} as step_fn_dims / batch_fn_dims and the variant
    branches of step_fn / batch_fn select them (NB 0: the single-sequence step)."""
    out = set()
    for fname, kernel, dims_fn, var_fn, launch in (
            ("decode_mega.cu", "decode_step_kernel", "static const void* step_fn_dims(", "static const void* step_fn(",
             "void launch_decode_step_mega("),
            ("decode_batch.cu", "decode_batch_kernel", "static const void* batch_fn_dims(", "static const void* batch_fn(",
             "void launch_decode_step_batch(")):
        with open(os.path.join(CSRC, fname)) as f:
            src = f.read()
        nb = r", (\d+)" if kernel == "decode_batch_kernel" else ""
        insts = re.findall(kernel + r"<(\d+), (\d+), (\d+)" + nb + r", [^<>]*LP, TK, SM, RP>", _body(src, dims_fn))
        fn = var_fn.split()[-1].rstrip("(")
        variants = re.findall(fn + r"_dims<(true|false), (true|false), (true|false), RP>", _body(src, var_fn))
        reps = re.findall(r"\b" + fn + r"<(true|false)>", _body(src, launch))
        assert insts and len(variants) == 5 and sorted(reps) == ["false", "true"], (fname, insts, variants, reps)
        for inst in insts:
            d, n = tuple(int(v) for v in inst[:3]), int(inst[3]) if nb else 0
            for v in variants:
                for rp in reps:
                    out.add((kernel, d, n, tuple(s == "true" for s in v) + (rp == "true",)))
    return out


def test_every_instantiation_has_a_cell():
    compiled = compiled_instantiations()
    assert len(compiled) >= (3 + 4) * 10, sorted(compiled)       # the parse found at least today's instances
    covered = {inst + (flags + (rep,),) for model, row in MATRIX for inst in cell_instantiations(model, row)
               for _name, _kw, flags in VARIANTS for rep in (False, True)}
    missing = sorted(compiled - covered)
    assert not missing, f"compiled decode-step variants no cell of MATRIX runs: {missing}"


def test_matrix_rows_run_their_paths():
    """Each row's instantiation comes from its batch size: b20 takes an NB 16 then an NB 8 pass, the 1.7B rows the
    single-sequence step only."""
    assert cell_instantiations("w0p6b", "batched_b20") == {("decode_batch_kernel", (1024, 2048, 3072), 16),
                                                           ("decode_batch_kernel", (1024, 2048, 3072), 8)}
    assert cell_instantiations("tiny", "batched_nb16") == {("decode_batch_kernel", (256, 512, 512), 16)}
    assert cell_instantiations("w1p7b", "fused_per_seq_b3") == {("decode_step_kernel", (2048, 2048, 6144), 0)}
    for model, row in MATRIX:
        assert all(0.7 <= s <= 3.0 for _i, s in ROWS[row][0]) or row == "handover", (model, row)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the checks can fail (tiny model)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row,first", [("batched_b20", 16), ("phases_b11", 8)])
def test_negative_control_lost_row_offset(zoo, row, first):
    """The draw of sequence b >= `first` taken at row b - first (what row0 = 0 in the pass / sub-batch launch gives)
    selects other pinned ids than the draw at the global row b."""
    sel, n_new = ROWS[row][0], ROWS[row][1]
    seed = SEEDS["tiny", row]
    diff = 0
    for b in range(first, len(sel)):
        ref = zoo.trajectory("tiny", sel[b], (0, 1.0), n_new, T, seed, b)
        k = ref.pinned()
        bad = zoo.trajectory("tiny", sel[b], (0, 1.0), n_new, T, seed, b - first)
        diff += bad.ids[:k] != ref.ids[:k]
    assert diff > 0


def _oracle_records(zoo, name, sel, ids, rep):
    """fp32-oracle log-probabilities of ids (processed with `rep`), as a recording kernel would write them."""
    s32, _ = zoo.scores(name, sel, ids)
    lsm = torch.log_softmax(torch.from_numpy(np.stack([process(s32[t].double().numpy(), ids[:t], *rep)
                                                       for t in range(len(ids))])), -1).numpy()
    return lsm


def _rule_ratio(zoo, name, sel, ids, values, rep):
    m32, m64 = zoo.oracles(name)
    r = SimpleNamespace(ids=[ids], logprobs=[list(values)], eos_logprobs=[None])
    return ratio({}, "control", record_errs(m32, m64, [zoo.samples(sel)], r, False, rep=rep,
                                            scores=lambda b, i: zoo.scores(name, sel, i)), min_values=MIN_RECORDS)


def test_negative_control_unprocessed_records(zoo):
    """REP + LOGPROB records taken from the unprocessed logits fail the rule; the processed ones pass it."""
    sel, n_new = ROWS["fused_single"][0][0], ROWS["fused_single"][1]
    ids = zoo.trajectory("tiny", sel, REP_GREEDY, n_new).ids
    rows = np.arange(len(ids))
    good = _oracle_records(zoo, "tiny", sel, ids, REP_GREEDY)[rows, ids]
    bad = _oracle_records(zoo, "tiny", sel, ids, (0, 1.0))[rows, ids]
    assert _rule_ratio(zoo, "tiny", sel, ids, good, REP_GREEDY) <= R
    assert _rule_ratio(zoo, "tiny", sel, ids, bad, REP_GREEDY) > R


def test_negative_control_greedy_formula_on_sampled_records(zoo):
    """SAMPLE + LOGPROB records written as -log S (the greedy formula, which drops l_sel - M) fail the rule: the seed
    draws ids other than the argmax, and on those steps the two differ."""
    sel, n_new = ROWS["fused_single"][0][0], ROWS["fused_single"][1]
    seed = SEEDS["tiny", "fused_single"]
    ref = zoo.trajectory("tiny", sel, (0, 1.0), n_new, T, seed, 0)
    ids = ref.ids
    lsm = _oracle_records(zoo, "tiny", sel, ids, (0, 1.0))
    s64 = zoo.scores("tiny", sel, ids)[1].numpy()
    for t in range(ref.pinned()):           # the trajectory is the draw: argmax of l / T + g at row 0
        assert int(np.argmax(s64[t] / T + gumbel(seed, 0, t, s64.shape[1]))) == ids[t]
    off_argmax = [t for t in range(len(ids)) if ids[t] != int(np.argmax(s64[t]))]
    assert len(off_argmax) > 0
    rows = np.arange(len(ids))
    assert _rule_ratio(zoo, "tiny", sel, ids, lsm[rows, ids], (0, 1.0)) <= R
    assert _rule_ratio(zoo, "tiny", sel, ids, lsm.max(-1), (0, 1.0)) > R


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the matrix
# ---------------------------------------------------------------------------------------------------------------------
def _run(e, clips, n_new, opts, path, **kw):
    """Warm-up (session sized, graphs captured), then the measured run; asserts the decode path that ran (as
    test_precision_fp64.run_path, with the hand-over's per-phase steps counted as captures)."""
    with options(e, **opts):
        e.transcribe_ids(clips, max_new_tokens=n_new, **kw)
        s0 = _steps(e.stats())
        r = e.transcribe_ids(clips, max_new_tokens=n_new, **kw)
        s1 = _steps(e.stats())
        prefill_only = e.transcribe_ids(clips, max_new_tokens=1, **kw)      # the same call without decode steps
    moved = {k: s1[k] - s0[k] for k in s0}
    if path == "decode_phase_steps":
        assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0, moved
        assert r.kernels_launched > 2 * r.decode_steps
    elif path == "handover":
        assert moved["decode_fused_steps"] > 0 and moved["decode_batch_steps"] == 0, moved
        assert r.kernels_launched > 2 * r.decode_steps
    else:
        assert moved[path] == r.decode_steps and moved["decode_phase_steps"] == 0, moved
    return r, r.kernels_launched - prefill_only.kernels_launched


@pytest.mark.gpu
@pytest.mark.parametrize("model,row", MATRIX, ids=[f"{m}-{r}" for m, r in MATRIX])
def test_decode_variants(zoo, report, model, row):
    t0 = time.time()
    sel, n_new, opts, path, per_step = ROWS[row]
    m32, m64 = zoo.oracles(model)
    e = zoo.engine(model)
    clips = [zoo.samples(s) for s in sel]
    seed = SEEDS[model, row]
    key = f"variants_{model}_{row}"
    runs, fails = {}, []
    for rep in (False, True):
        for name, _kw, _flags in VARIANTS:
            r, decode_launches = _run(e, clips, n_new, opts, path, **variant_kw(name, rep, seed))
            if per_step is not None:         # the launcher's launches per step: one per pass of 16 / per sequence
                with collect(fails, f"{name} rep={rep} launches"):
                    assert decode_launches == per_step * r.decode_steps, (decode_launches, r.decode_steps)
            runs[name, rep] = r
    pins = {}
    for rep in (False, True):
        tag = "_rep" if rep else ""
        g, lp, tk, s, slp = (runs[v[0], rep] for v in VARIANTS)
        with collect(fails, f"selection{tag}"):
            assert lp.ids == g.ids and tk.ids == g.ids, "a record variant selected other ids than greedy"
            assert slp.ids == s.ids, "sampling with the record selected other ids than without"
        for b in range(len(clips)):
            with collect(fails, f"top8 entry 0{tag} seq {b}"):
                _check_against_logprobs(tk, b)
        for kind, r, T_ in (("greedy", g, 0.0), ("sample", s, T)):
            pinned = total = 0
            for b in range(len(clips)):
                ref = zoo.trajectory(model, sel[b], rep_of(kind, rep), n_new, T_, seed, b)
                total += len(ref.gaps)
                with collect(fails, f"{kind}{tag} ids seq {b}"):
                    pinned += assert_pinned(r.ids[b], ref, (model, row, kind, rep, b))
            pins[kind + tag] = [pinned, total]
            with collect(fails, f"{kind}{tag} pinned"):
                assert 2 * pinned >= total, (pinned, total)
        if rep:
            for name, r in zip((v[0] for v in VARIANTS), (g, lp, tk, s, slp)):
                N = rep_of(name, rep)[0]
                with collect(fails, f"{name}{tag} repeated n-grams"):
                    assert all(repeated_ngrams(ids, N) == 0 for ids in r.ids)
            with collect(fails, f"top8{tag} banned candidates"):
                assert all(np.isfinite(v) for rows in tk.top_logprobs for cands in rows for _c, v in cands)
        for name, r, top in (("logprob", lp, False), ("top8", tk, True), ("sample_logprob", slp, False)):
            with collect(fails, f"{name}{tag} records"):
                err = record_errs(m32, m64, clips, r, top, rep=rep_of(name, rep), seqs=RECORD_SEQS.get(row),
                                  scores=lambda b, ids: zoo.scores(model, sel[b], ids))
                q = ratio(report, f"{key}_{name}{tag}", err, min_values=MIN_RECORDS)
                assert q <= R, report[f"fp64_{key}_{name}{tag}"]
    for kind in ("greedy", "sample"):
        with collect(fails, f"{kind} repetition controls acted"):
            assert runs[kind, True].ids != runs[kind, False].ids
    report[f"{key}_pinned_steps"] = pins
    report[f"{key}_wall_s"] = time.time() - t0
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: stage outputs at the full 1.7B depth (24 encoder, 28 decoder layers)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full1p7b(zoo):
    """(fp32 oracle, fp64 oracle, engine) of cfg_1p7b(); the cut models are freed first, and the fp64 weights (about
    18 GB of host memory) after the module."""
    from qwen3_asr_rs_b200 import AsrInference, config_1p7b
    zoo.close()
    cfg, ecfg = O.cfg_1p7b(), config_1p7b()
    cfg.text.tie_word_embeddings = ecfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 3, peaked_head=True)
    e = AsrInference.from_weights(ecfg, w, device=0)
    m32, m64 = O.OracleModel(cfg, w), O.OracleModel(cfg, w, dtype=torch.float64)
    del w
    yield m32, m64, e
    e.close()
    del m32, m64
    gc.collect()


FULL_1P7B_CLIP = (31, 8.5)           # one tail chunk


@pytest.mark.gpu
def test_stage_outputs_1p7b_full_depth(full1p7b, report):
    """Mel, encoder output (d_model 1024, ffn 4096), prefill logits (GEMMs up to N = 12288 and K = 6144) and 5
    decode_step logits (the per-phase GEMVs at K = 2048 and 6144: decode_step returns logits) under R = 4."""
    m32, m64, e = full1p7b
    clips = [synth.make_clip(*FULL_1P7B_CLIP)]
    errs = stage_errs(m32, m64, clips, stage_run(e, clips))
    for k, err in errs.items():
        ratio(report, f"1p7b_full_b1_{k}", err)
    report["1p7b_full_peak_host_rss_gb"] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    for k, err in errs.items():
        check(report, f"1p7b_full_b1_{k}", err)


@pytest.mark.gpu
def test_negative_control_lost_planes_1p7b_full_depth(full1p7b, report):
    m32, m64, e = full1p7b
    with options(e, planes="2"):
        enc_e, pre_e = _planes_errs(m32, m64, e, [synth.make_clip(*FULL_1P7B_CLIP)])
    for name, err in (("encoder", enc_e), ("prefill", pre_e)):
        r = ratio(report, f"1p7b_full_planes2_{name}", err)
        assert r > R, (name, report[f"fp64_1p7b_full_planes2_{name}"])
