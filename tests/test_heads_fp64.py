"""Kernel-level precision of the two output heads: the wgmma score head (csrc/score.cu, DESIGN.md 4.8) and the
alignment probability / z-score / median kernels (csrc/align.cu, DESIGN.md 4.10), each against a float64 reference of
the same operation.

The model-level tests (test_score.py, test_align.py) reach these kernels only at the shapes their clips produce: the
score head never sees a second M tile, a CTA with a second work item or fewer than 64 column slices, and the alignment
kernels rarely see a second row tile.  This file drives them through the test probes (csrc/probe.h) at shapes chosen
for those paths: M tiles past the first (rows 1 .. 4100), persistent CTAs walking several (M tile, slice) items (grid
caps 1 and 7, 192 items on 132 SMs), 1 .. 64 slices of equal and unequal width, ragged last vocabulary tiles, targets
at slice edges and at the lane split of each 32-column group, planted top-8 ties; softmax rows across 16-row tiles,
keys across 32-key tiles, the median's pass-through and mirror padding, GQA groups and ragged batches.

Every GPU case first asserts the plan the probe reports, then applies the rule of test_precision_fp64.py
(e_gpu <= R * max(e_32, floor), R = 4) against a float64 reference built from the same fp32 inputs and exact bf16
weights and an fp32 reference of the same operation in torch.  Log-probabilities are compared in absolute nats (floor:
the fp32 ulp of the largest |lp|), alignment stages by relative max error.  e_gpu, e_32 and the ratio go into the
report.  The CPU tests restate the score head's plan and show that the rule rejects a dropped slice partial, M-tile rows
shifted by one tile, a target logit taken from the wrong lane half, a softmax row tile off by one and a median without
mirror padding.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_align import head_mean, median7, zscore
from test_kernels_fp64 import SMS_PCIE, SMS_SXM, bf16_rne, bf16_to_f32, probe, ptr, sms_of_device, split3_np
from test_precision_fp64 import R, Err, ratio

BM, BN = 128, 128                # score head: M tile, lm_head tile (columns)
SLICES = 64                      # SCORE_SLICES
TK = 8                           # TK_MAX
MARGIN = 3e-4                    # a float64 gap the rule's errors cannot reorder (as test_score.py)
PROB_ROWS = 16                   # align_probs_kernel rows per CTA
DEV = "cuda"                     # the score references run on the GPU (fp64 and true fp32 GEMMs: TF32 off)


# ---------------------------------------------------------------------------------------------------------------------
# bindings of the probes (csrc/probe.h)
# ---------------------------------------------------------------------------------------------------------------------
class ScoreArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("rows", "n_hid", "H", "V")] + [
        ("hid", C.c_void_p), ("src", C.c_void_p), ("norm_w", C.c_void_p), ("eps", C.c_float), ("lm_head", C.c_void_p),
        ("target", C.c_void_p), ("nplanes", C.c_int), ("topk", C.c_int), ("grid_cap", C.c_int),
        ("lp_out", C.c_void_p), ("tk_ids_out", C.c_void_p), ("tk_lp_out", C.c_void_p)]


class AlignArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("B", "hd", "group", "nheads", "count")] + [
        (n, C.c_void_p) for n in ("heads", "qrow0", "N", "T", "a0", "slot")] + [
        ("q", C.c_void_p), ("q_rows", C.c_int64), ("ldq", C.c_int),
        ("k", C.c_void_p), ("k_elems", C.c_int64), ("seg_stride", C.c_int64), ("head_stride", C.c_int64),
        ("M_in", C.c_void_p), ("P_out", C.c_void_p), ("Z_out", C.c_void_p), ("M_out", C.c_void_p)]


_bound = False


def heads_probe():
    global _bound
    lib = probe()
    if not _bound:
        i32, vp = C.c_int, C.c_void_p
        for name, args in {"asrbt_score_plan": [i32] * 5 + [vp], "asrbt_score_head": [C.POINTER(ScoreArgs), vp],
                           "asrbt_align": [C.POINTER(AlignArgs)]}.items():
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = C.c_int
        _bound = True
    return lib


def _ok(code):
    from qwen3_asr_rs_b200 import _lib
    _lib.check(code)


SCORE_PLAN_KEYS = ("tiles_m", "tiles_n", "nslices", "grid", "items_per_cta", "slice_min", "slice_max")


def score_plan(rows, V, H=1024, sms=SMS_SXM, cap=0):
    out = np.zeros(len(SCORE_PLAN_KEYS), np.int32)
    _ok(heads_probe().asrbt_score_plan(rows, V, H, sms, cap, ptr(out)))
    return dict(zip(SCORE_PLAN_KEYS, out.tolist()))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the score head's plan
# ---------------------------------------------------------------------------------------------------------------------
def slice_tiles(tiles_n, nslices):
    """[t0, t1) of every slice: slice s takes tiles s * tiles_n / nslices .. (s + 1) * tiles_n / nslices."""
    return [(s * tiles_n // nslices, (s + 1) * tiles_n // nslices) for s in range(nslices)]


def score_plan_py(rows, V, sms=SMS_SXM, cap=0):
    """The score head's launch restated: 128-row M tiles, 128-column lm_head tiles, min(64, tiles_n) slices, work item
    (M tile, slice), persistent grid min(items, SMs), capped by grid_cap when > 0."""
    tiles_m, tiles_n = -(-rows // BM), -(-V // BN)
    nslices = min(SLICES, tiles_n)
    items = tiles_m * nslices
    grid = min(items, sms) if cap == 0 else min(items, sms, cap)
    w = [t1 - t0 for t0, t1 in slice_tiles(tiles_n, nslices)]
    return dict(tiles_m=tiles_m, tiles_n=tiles_n, nslices=nslices, grid=grid, items_per_cta=-(-items // grid),
                slice_min=min(w), slice_max=max(w))


PLAN_ROWS = [1, 127, 128, 129, 255, 256, 257, 300, 1000, 4100, 8193]
PLAN_V = [1, 9, 127, 128, 129, 1000, 8192, 8193, 8320, 8448, 16384, 151936, 151937, 151944, 152064]


@pytest.mark.parametrize("sms", [SMS_SXM, SMS_PCIE])
def test_score_plan_matches_restatement(sms):
    """asrbt_score_plan (the function the launcher itself calls) against score_plan_py over rows x vocabulary x grid
    cap; and the outcomes the GPU cases rely on are reached: one slice, fewer than 64, exactly 64, unequal slice
    widths, >= 3 M tiles, and CTAs with >= 2 items both at the launcher's grid and under a cap."""
    seen = set()
    for rows in PLAN_ROWS:
        for V in PLAN_V:
            for cap in (0, 1, 7, 200):
                got, want = score_plan(rows, V, 1024, sms, cap), score_plan_py(rows, V, sms, cap)
                assert got == want, (rows, V, cap, got, want)
                seen.add(("slices", 1 if got["nslices"] == 1 else (64 if got["nslices"] == 64 else "mid")))
                if got["slice_min"] != got["slice_max"]:
                    seen.add("uneven")
                if got["tiles_m"] >= 3:
                    seen.add("tiles_m>=3")
                if got["items_per_cta"] >= 2:
                    seen.add(("multi", cap))
    want = {("slices", 1), ("slices", "mid"), ("slices", 64), "uneven", "tiles_m>=3", ("multi", 0), ("multi", 1),
            ("multi", 7)}
    assert want <= seen, want - seen


def test_score_plan_production_shapes():
    """The production vocabulary: 1187 tiles in 64 slices of 18 or 19 tiles; 300 rows give 3 M tiles and 192 items,
    so on 132 SMs (and 114) some CTAs take two; a language-ID call of ~100 rows is one M tile, one item per CTA."""
    p = score_plan(300, 151936)
    assert p == dict(tiles_m=3, tiles_n=1187, nslices=64, grid=132, items_per_cta=2, slice_min=18, slice_max=19)
    assert score_plan(300, 151936, sms=SMS_PCIE)["items_per_cta"] == 2
    assert score_plan(100, 151936)["items_per_cta"] == 1
    assert score_plan(129, 8320)["slice_min"] == 1 and score_plan(129, 8320)["slice_max"] == 2


def test_score_plan_refuses_bad_dims():
    from qwen3_asr_rs_b200 import _lib
    out = np.zeros(len(SCORE_PLAN_KEYS), np.int32)
    for a in ((0, 100, 1024, 132, 0), (1, 0, 1024, 132, 0), (1, 100, 1000, 132, 0), (1, 100, 1024, 0, 0),
              (1, 100, 1024, 132, -1)):
        assert heads_probe().asrbt_score_plan(*a, ptr(out)) == 1, a          # ASRB_ERR_INVALID
    assert _lib.load_library().asrb_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def score_logits(hid, w_norm, eps, W, dtype):
    """RMSNorm(hid) * w_norm @ W^T in `dtype` (torch tensors on one device; W holds exact bf16 values)."""
    x = hid.to(dtype)
    y = x * (1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + eps)) * w_norm.to(dtype)
    return y @ W.to(dtype).T


def score_rows(hid, w_norm, eps, W, dtype):
    return torch.log_softmax(score_logits(hid, w_norm, eps, W, dtype), -1)


def rule_ratio(y_bad, y32, y64, relative):
    return ratio({}, "control", Err(relative).add(y_bad, y32, y64), min_values=1)


def _cpu_score_setup(rows=300, V=1000, H=256, seed=0):
    rng = np.random.default_rng(seed)
    hid = torch.from_numpy(rng.standard_normal((rows, H)).astype(np.float32))
    w_norm = torch.from_numpy((1 + 0.1 * rng.standard_normal(H)).astype(np.float32))
    W = torch.from_numpy(bf16_to_f32(bf16_rne(rng.standard_normal((V, H)) * 2 / math.sqrt(H))))
    tgt = rng.integers(0, V, rows)
    l64, l32 = (score_rows(hid, w_norm, 1e-6, W, dt).numpy() for dt in (torch.float64, torch.float32))
    return l64, l32, tgt


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rule sees each way the score head could go wrong
# ---------------------------------------------------------------------------------------------------------------------
def test_rule_sees_a_dropped_slice_partial():
    """One slice's (max, sum) partial left out of a row's log-sum-exp (V = 1000: 8 slices of one tile)."""
    l64, l32, tgt = _cpu_score_setup()
    r = np.arange(len(tgt))
    logits32 = l32                                   # log-softmax rows differ from logits by a per-row constant
    for s in (0, 3, 7):
        keep = np.ones(l32.shape[1], bool)
        keep[s * BN:(s + 1) * BN] = False
        lse = torch.logsumexp(torch.from_numpy(logits32[:, keep]), -1).numpy()
        bad = np.where(keep[tgt], logits32[r, tgt] - lse, l32[r, tgt])
        assert rule_ratio(bad, l32[r, tgt], l64[r, tgt], False) > R


def test_rule_sees_m_tile_rows_shifted():
    """Rows of the second and third M tiles written with the results of the rows one tile earlier."""
    l64, l32, tgt = _cpu_score_setup()
    r = np.arange(len(tgt))
    want32, want64 = l32[r, tgt], l64[r, tgt]
    bad = want32.copy()
    bad[BM:] = want32[:-BM]
    assert rule_ratio(bad, want32, want64, False) > R


def test_rule_sees_the_wrong_lane_half():
    """The target logit taken from the other lane's 16 columns of its 32-column group (column n ^ 16)."""
    l64, l32, tgt = _cpu_score_setup()
    r = np.arange(len(tgt))
    other = tgt ^ 16
    ok = other < l32.shape[1]
    bad = l32[r[ok], other[ok]]
    assert rule_ratio(bad, l32[r[ok], tgt[ok]], l64[r[ok], tgt[ok]], False) > R


def head_emulation(x, w, chunk, p=26):
    """CPU model of the score head's accumulation: test_kernels_fp64.wgmma_emulation with the chunk length as a
    parameter.  Per k-block of 64 the hi, mid and lo planes of x each issue 4 m64n128k16 steps into one accumulator; a
    step aligns its 16 exact products and the accumulator to the largest exponent, truncates each below p bits, sums
    exactly and rounds toward zero to fp32; every `chunk` k-blocks (1 in the head, 4 in gemm_tc.cu) the accumulator is
    added into a second fp32 sum with round-to-nearest.  Returns the fp32 sums [rows][len(w)]."""
    pl = split3_np(np.asarray(x, np.float32).ravel()).reshape(3, *x.shape)
    planes = [bf16_to_f32(pl[i]).astype(np.float64) for i in range(3)]
    K = x.shape[1]
    wd = np.asarray(w, np.float64)
    acc, tot = np.zeros((x.shape[0], wd.shape[0])), np.zeros((x.shape[0], wd.shape[0]), np.float32)
    for kb in range(K // 64):
        if kb % chunk == 0:
            acc[:] = 0.0
        for a in planes:
            for k in range(4):
                sl = slice(kb * 64 + 16 * k, kb * 64 + 16 * k + 16)
                terms = np.concatenate([a[:, None, sl] * wd[None, :, sl], acc[:, :, None]], -1)
                mx = np.abs(terms).max(-1, keepdims=True)
                q = 2.0 ** (np.floor(np.log2(np.where(mx > 0, mx, 1.0))) - p + 1)
                v = np.trunc(terms / q).sum(-1) * q[..., 0]
                m, e = np.frexp(v)
                acc = np.trunc(m * 2.0 ** 24) * 2.0 ** (e - 24)
        if kb % chunk == chunk - 1 or kb == K // 64 - 1:
            tot = tot + acc.astype(np.float32)
    return tot


def test_head_emulation_is_the_gemm_model_at_chunk_4():
    """At chunk 4 the model above is test_kernels_fp64.wgmma_emulation, bit for bit."""
    from test_kernels_fp64 import wgmma_emulation
    rng = np.random.default_rng(3)
    x = rng.standard_normal((3, 640)).astype(np.float32)
    w = bf16_to_f32(bf16_rne(rng.standard_normal((40, 640)) * 0.05))
    assert np.array_equal(head_emulation(x, w, 4), wgmma_emulation(x, w))


def test_score_head_accumulation_model():
    """A row with one dominant logit (the row is the lm_head row scaled, so every product of that dot product has one
    sign) at H = 2048.  The tensor core truncates its running sum toward zero at every k16 step; with 4 k-blocks per
    accumulation (48 truncations before a round-to-nearest add, as gemm_tc.cu) the CPU model of that accumulation
    (head_emulation) puts the row's log-probabilities far over R, as the score head measured on an H100 (up to 12 x)
    while it used 4-block chunks.  With one k-block per accumulation, as the head now does, the model's error drops
    by more than half."""
    rng = np.random.default_rng(17)
    H, V, d = 2048, 1000, 333
    W = bf16_to_f32(bf16_rne(rng.standard_normal((V, H)) * 2 / math.sqrt(H)))
    u = bf16_to_f32(bf16_rne(rng.standard_normal(H) * 40.0 / H))
    W[d] = u
    w_norm = (1 + 0.1 * rng.standard_normal(H)).astype(np.float32)
    x = torch.from_numpy(u[None, :].copy())
    y32 = (x * (1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + 1e-6)) * torch.from_numpy(w_norm)).numpy()
    l64 = score_logits(x, torch.from_numpy(w_norm), 1e-6, torch.from_numpy(W), torch.float64)[0]
    l32 = score_logits(x, torch.from_numpy(w_norm), 1e-6, torch.from_numpy(W), torch.float32)[0].double()
    assert int(l64.argmax()) == d and float(l64[d]) > 30
    cols = torch.topk(l64, TK).indices.numpy()
    want64, want32 = torch.log_softmax(l64, -1).numpy()[cols], torch.log_softmax(l32, -1).numpy()[cols]
    err = {}
    for chunk in (4, 1):
        lm = torch.from_numpy(head_emulation(y32, W, chunk)[0].astype(np.float64))
        got = torch.log_softmax(lm, -1).numpy()[cols]
        err[chunk] = float(np.abs(got - want64).max())
        if chunk == 4:
            assert rule_ratio(got, want32, want64, False) > R
    assert err[1] < 0.5 * err[4], err


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rule sees each way the alignment kernels could go wrong; the z-score of a column of equal values
# ---------------------------------------------------------------------------------------------------------------------
def align_ref(q, k, dtype):
    """Softmax over the keys of q [N][hd] . k [T][hd] / sqrt(hd), in `dtype` (torch, CPU)."""
    qt, kt = torch.from_numpy(q).to(dtype), torch.from_numpy(k).to(dtype)
    return torch.softmax((qt @ kt.T) / math.sqrt(q.shape[1]), -1).numpy()


def test_rule_sees_a_softmax_row_tile_off_by_one():
    """The second and later 16-row tiles computed from the q rows one row earlier."""
    rng = np.random.default_rng(5)
    q, k = rng.standard_normal((50, 128)).astype(np.float32), rng.standard_normal((65, 128)).astype(np.float32)
    p64, p32 = align_ref(q, k, torch.float64), align_ref(q, k, torch.float32)
    qb = q.copy()
    qb[PROB_ROWS:] = q[PROB_ROWS - 1:-1]
    assert rule_ratio(align_ref(qb, k, torch.float32), p32, p64, True) > R


def test_rule_sees_a_median_without_mirror_padding():
    """The width-7 median with the edge value repeated (or zeros) in place of the mirror at both ends."""
    rng = np.random.default_rng(6)
    planes = [align_ref(rng.standard_normal((33, 128)).astype(np.float32), rng.standard_normal((40, 128)).astype(np.float32),
                        torch.float64) for _ in range(2)]
    m64 = head_mean(planes)
    m32 = head_mean([p.astype(np.float32) for p in planes])

    def bad_median(z, mode):
        p = np.pad(z, ((0, 0), (3, 3)), mode=mode)
        return np.median(np.lib.stride_tricks.sliding_window_view(p, 7, axis=1), axis=-1).astype(z.dtype)
    for mode in ("edge", "constant"):
        bad = sum(bad_median(zscore(p.astype(np.float32)), mode) for p in planes) / np.float32(2)
        assert rule_ratio(bad, m32, m64, True) > R


def _zscore_kernel_f32(col, shifted):
    """align_zscore_kernel's arithmetic on one column in float32: the mean as a plain sum / N (before) or as
    P[0] + sum(P - P[0]) / N (now), then the population variance by fmaf and z = (P - mean) / std, 0 where std = 0."""
    f = np.float32
    p0 = col[0] if shifted else f(0)
    s = f(0)
    for v in col:
        s = f(s + f(v - p0))
    mean = f(p0 + f(s / f(len(col))))
    var = f(0)
    for v in col:
        d = f(v - mean)
        var = f(np.float64(d) * np.float64(d) + np.float64(var))        # fmaf: one rounding
    sd = f(np.sqrt(f(var / f(len(col)))))
    return np.array([f(f(v - mean) / sd) if sd > 0 else f(0) for v in col], np.float32)


def test_zscore_of_a_column_of_equal_values_model():
    """A column whose rows hold one value has std 0, so z = 0 (include/asr_b200.h).  With the mean as a plain fp32
    sum / N, the sum of N equal values rounds for about half of all values and N, the deviations are then all equal
    and nonzero, and z came out +-1; the shifted mean gives exactly 0."""
    rng = np.random.default_rng(7)
    wrong = 0
    for N in (2, 3, 5, 17, 33, 200):
        for _ in range(40):
            col = np.full(N, np.float32(rng.random() * 0.3), np.float32)
            assert not _zscore_kernel_f32(col, True).any()
            wrong += bool(_zscore_kernel_f32(col, False).any())
    assert wrong > 60, wrong
    # and on ordinary columns the shifted mean agrees with float64 as closely as the plain one
    for N in (2, 17, 200):
        col = (rng.random(N) * 0.3).astype(np.float32)
        z64 = zscore(col[:, None].astype(np.float64))[:, 0]
        assert np.abs(_zscore_kernel_f32(col, True) - z64).max() < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the score head
# ---------------------------------------------------------------------------------------------------------------------
def check_tf32_off():
    assert not torch.backends.cuda.matmul.allow_tf32 and torch.get_float32_matmul_precision() == "highest"


def lane_edge_columns(V):
    """Columns at n % 32 in {15, 16, 31} (the two lanes of a row split every 32-column group at 16) at the start, the
    middle and the end of the vocabulary."""
    out = []
    for base in (0, 32 * (V // 64), 32 * ((V - 1) // 32) - 32):
        out += [base + o for o in (15, 16, 31)]
    return sorted({c for c in out if 0 <= c < V})


def special_targets(V, plan):
    """Ids 0 and V - 1, the first and last column of every slice, the lane edges and the lone column of a ragged last
    tile (V % 128 == 1)."""
    t = [0, V - 1]
    for t0, t1 in slice_tiles(plan["tiles_n"], plan["nslices"]):
        t += [t0 * BN, min(t1 * BN, V) - 1]
    t += lane_edge_columns(V)
    if V % BN == 1:
        t.append(V - 1)
    return list(dict.fromkeys(t))


def tie_groups(V, plan):
    """Two groups of duplicated lm_head rows placed across the first slice boundary and the lane split (the first
    group's rows weigh 1, the second's 1/2): (group a, group b)."""
    t0, t1 = slice_tiles(plan["tiles_n"], plan["nslices"])[0]
    cb = t1 * BN if plan["nslices"] > 1 else V // 2
    a = sorted({c for c in (cb - 1, cb, cb + 15, cb + 16) if 0 <= c < V})
    b = sorted({c for c in (15, 16, V - 1) if 0 <= c < V and c not in a})
    return a, b


def run_score(hid, src, w_norm, eps, wbits, target, nplanes=3, topk=True, cap=0):
    rows, H = len(target), hid.shape[1]
    hid, w_norm = np.ascontiguousarray(hid, np.float32), np.ascontiguousarray(w_norm, np.float32)
    wbits = np.ascontiguousarray(wbits, np.uint16)
    target = np.ascontiguousarray(target, np.int32)
    srcc = None if src is None else np.ascontiguousarray(src, np.int32)
    a = ScoreArgs()
    a.rows, a.n_hid, a.H, a.V = rows, hid.shape[0], H, wbits.shape[0]
    a.hid, a.src, a.norm_w, a.eps, a.lm_head, a.target = ptr(hid), ptr(srcc), ptr(w_norm), eps, ptr(wbits), ptr(target)
    a.nplanes, a.topk, a.grid_cap = nplanes, int(topk), cap
    lp = np.zeros(rows, np.float32)
    ids = np.zeros((rows, TK), np.int32)
    tlp = np.zeros((rows, TK), np.float32)
    a.lp_out, a.tk_ids_out, a.tk_lp_out = ptr(lp), ptr(ids), ptr(tlp)
    plan = np.zeros(len(SCORE_PLAN_KEYS), np.int32)
    _ok(heads_probe().asrbt_score_head(C.byref(a), ptr(plan)))
    return lp, ids, tlp, dict(zip(SCORE_PLAN_KEYS, plan.tolist()))


def make_score_case(rows, V, H, seed, planted=True, gather=True, logit_scale=1.0):
    """Inputs of one score case (lm_head exact bf16, on `DEV`).  With `planted`, row 0 is all zeros, row 1
    has one dominant logit (id V // 3), rows 2-3 score the two tie groups, and the special targets go to the first rows;
    the remaining rows are random with random targets."""
    dev = DEV
    rng = np.random.default_rng(seed)
    g = torch.Generator(device=dev).manual_seed(seed)
    W = (torch.randn(V, H, device=dev, generator=g) * (2.0 / math.sqrt(H))).to(torch.bfloat16)
    n_hid = rows + 3 if gather else rows
    hid = rng.standard_normal((n_hid, H)).astype(np.float32)
    src = rng.permutation(n_hid)[:rows].astype(np.int32) if gather else None
    w_norm = (logit_scale * (1 + 0.1 * rng.standard_normal(H))).astype(np.float32)
    plan = score_plan_py(rows, V, sms_of_device())
    target = rng.integers(0, V, rows).astype(np.int32)
    info = {"zero": None, "dominant": None, "ties": None}
    sp = special_targets(V, plan)
    if planted and rows >= 4:
        def set_row(r, vec):
            hid[r if src is None else src[r]] = vec
        set_row(0, 0.0)
        info["zero"] = 0
        u = torch.from_numpy(bf16_to_f32(bf16_rne(rng.standard_normal(H) * 40.0 / H))).to(dev)
        d = V // 3
        W[d] = u.to(torch.bfloat16)
        set_row(1, u.cpu().numpy())
        info["dominant"] = (1, d)
        if V >= 1000:
            ga, gb = tie_groups(V, plan)
            t = torch.from_numpy(bf16_to_f32(bf16_rne(rng.standard_normal(H) * 30.0 / H))).to(dev)
            for c in ga:
                W[c] = t.to(torch.bfloat16)
            for c in gb:
                W[c] = (0.5 * t).to(torch.bfloat16)
            set_row(2, t.cpu().numpy())
            set_row(3, -t.cpu().numpy())                 # the same rows as the least likely ids
            info["ties"] = (2, ga, gb)
    for i, c in enumerate(sp[:rows]):
        target[i] = c
    return dict(hid=hid, src=src, w_norm=w_norm, eps=1e-6, W=W, target=target, info=info, plan=plan,
                specials=sp, n_special=min(len(sp), rows))


def model_rows_check(report, key, cs, lp, ids, tlp, rows64, held):
    """Rows held to the CPU model of the head's accumulation instead of R: the model (head_emulation with one k-block
    per accumulation, on the normed rows exactly as the GPU's RMSNorm producer rounds them) must explain the GPU's
    error, agreeing with it to within a quarter of that error against float64."""
    from test_kernels_fp64 import run_norm
    x = cs["hid"] if cs["src"] is None else cs["hid"][cs["src"]]
    Wf = cs["W"].float().cpu().numpy()
    d_model = d_64 = 0.0
    for row in held:
        y = run_norm(1, x[row:row + 1], cs["w_norm"], cs["w_norm"], cs["eps"]).astype(np.float32)
        lm = torch.log_softmax(torch.from_numpy(head_emulation(y, Wf, 1)[0].astype(np.float64)), -1).numpy()
        cols = np.concatenate([[cs["target"][row]], ids[row]])
        got = np.concatenate([[lp[row]], tlp[row]]).astype(np.float64)
        d_model = max(d_model, float(np.abs(got - lm[cols]).max()))
        d_64 = max(d_64, float(np.abs(got - rows64[row][torch.from_numpy(cols).long().to(DEV)].cpu().numpy()).max()))
    report[f"fp64_{key}"].update(model_rows=list(held), max_abs_diff_to_model=d_model, max_abs_err_model_rows=d_64)
    assert d_model <= 0.25 * d_64, (key, d_model, d_64)


def score_case(report, key, rows, V, H, cap=0, seed=0, nplanes=3, topk=True, planted=True, gather=True, logit_scale=1.0,
               need_exact=None, model_rows=()):
    """One score head call against float64 / fp32 log-softmax rows computed on the GPU; returns (ratio, plan).  Rows in
    `model_rows` are held to the accumulation model (model_rows_check) and left out of the rule."""
    check_tf32_off()
    cs = make_score_case(rows, V, H, seed, planted, gather, logit_scale)
    wbits = cs["W"].view(torch.int16).cpu().numpy().view(np.uint16)
    lp, ids, tlp, plan = run_score(cs["hid"], cs["src"], cs["w_norm"], cs["eps"], wbits, cs["target"], nplanes, topk, cap)
    want = score_plan_py(rows, V, sms_of_device(), cap)
    assert plan == want, (key, plan, want)
    x = torch.from_numpy(cs["hid"] if cs["src"] is None else cs["hid"][cs["src"]]).to(DEV)
    wn = torch.from_numpy(cs["w_norm"]).to(DEV)
    r = torch.arange(rows, device=DEV)
    tg = torch.from_numpy(cs["target"]).long().to(DEV)
    err, exact, info = Err(False), 0, cs["info"]
    # the float64 and fp32 rows one at a time, so that only one [rows][V] table is held
    rows64 = score_rows(x, wn, cs["eps"], cs["W"], torch.float64)
    rows32 = score_rows(x, wn, cs["eps"], cs["W"], torch.float32).double()
    keep = np.setdiff1d(np.arange(rows), np.array(model_rows, int))
    err.add(lp[keep], rows32[r, tg].cpu().numpy()[keep], rows64[r, tg].cpu().numpy()[keep])
    if topk:
        ti = torch.from_numpy(ids).long().to(DEV)
        assert ((ids >= 0) & (ids < V)).all(), key
        assert all(len(set(row)) == TK for row in ids.tolist()), key
        assert (np.diff(tlp, axis=1) <= 0).all(), key
        err.add(tlp[keep], torch.gather(rows32, 1, ti).cpu().numpy()[keep], torch.gather(rows64, 1, ti).cpu().numpy()[keep])
        planted_rows = {v if not isinstance(v, tuple) else v[0] for v in info.values() if v is not None}
        if info["ties"]:
            planted_rows.add(3)
        tv, tix = (a.cpu().numpy() for a in torch.topk(rows64, min(V, 2 * TK + 1), dim=1))
        for row in range(rows):
            if row in planted_rows:
                continue
            order = np.lexsort((tix[row], -tv[row]))[:TK + 1]       # (value descending, id ascending)
            i9, v9 = tix[row][order], tv[row][order]
            if (-np.diff(v9) >= MARGIN).all():
                assert ids[row].tolist() == i9[:TK].tolist(), (key, row, ids[row], i9)
                exact += 1
        if info["zero"] is not None:
            z = info["zero"]                              # every logit 0: lp = -log V, the 8 smallest ids in order
            assert ids[z].tolist() == list(range(TK)), (key, ids[z])
            assert (tlp[z] == tlp[z][0]).all() and abs(tlp[z][0] + math.log(V)) <= 4 * np.spacing(np.float32(math.log(V)))
        if info["dominant"] is not None:
            row, d = info["dominant"]
            assert ids[row][0] == d, (key, ids[row])
        if info["ties"]:
            row, ga, gb = info["ties"]
            got = ids[row].tolist()
            assert got[:len(ga) + len(gb)] == ga + gb, (key, got, ga, gb)
            tie_equal = all(len(set(tlp[row][s].tolist())) == 1 for s in (slice(0, len(ga)), slice(len(ga), len(ga) + len(gb))))
            report.setdefault(f"fp64_{key}_ties", {})["bitwise_equal"] = tie_equal
            assert tie_equal, (key, "duplicated lm_head rows gave different logits", tlp[row])
            bounds = slice_tiles(plan["tiles_n"], plan["nslices"])
            slices_of = {next(s for s, (t0, t1) in enumerate(bounds) if t0 <= c // BN < t1) for c in ga}
            assert len(slices_of) == 2, (key, ga, bounds[:2])             # the top-8 straddles a slice boundary
        n_need = need_exact if need_exact is not None else min(10, max(1, (rows - len(planted_rows)) // 2))
        assert exact >= n_need, (key, exact, n_need)
    rr = ratio(report, key, err, min_values=min(300, err.n))
    if model_rows:
        model_rows_check(report, key, cs, lp, ids, tlp, rows64, model_rows)
    report[f"fp64_{key}"].update(plan, rows=rows, V=V, H=H, cap=cap, nplanes=nplanes, top_exact=exact,
                                 specials=cs["n_special"])
    del rows64, rows32, cs, x, wn, r, tg
    torch.cuda.empty_cache()                             # the lm_head and the reference tables go back to the device
    return rr, plan


# rows, V, H, grid cap: every rows value of the issue, nslices 1 / 2 / 8 / 64 / 65 tiles (uneven), ragged last tiles,
# and the production vocabulary with at most ~300 rows
# (rows, V, H): rows held to the accumulation model.  At H = 2048 the row whose logit is a one-signed dot product of
# 2048 terms (row 1, the dominant logit) and the tie row (2) still sit at ~4.2 x the fp32 error with one k-block per
# accumulation (12 truncations toward zero before each round-to-nearest add): the model gives the same, while every
# other row of the case meets R
MODEL_ROWS = {(255, 1000, 2048): (1, 2)}

SCORE_CASES = [
    (300, 151936, 1024, 0),     # tiles_m 3, 192 items: CTAs take two on 132 (and 114) SMs
    (257, 151944, 2048, 7),     # ragged last tile of 8 columns, 7 CTAs walk 192 items
    (129, 151937, 256, 0),      # lone column in the last tile
    (1, 151936, 1024, 0),
    (4100, 9, 256, 0),          # one slice of one ragged tile, 33 M tiles
    (1000, 129, 1024, 1),       # 2 slices, one CTA walks all 16 items (kg wraps the 3 stages 85 times)
    (255, 1000, 2048, 0),       # 8 slices
    (127, 8192, 1024, 0),       # exactly 64 tiles
    (128, 8320, 256, 1),        # 65 tiles in 64 slices: one slice of 2 tiles
    (300, 8320, 1024, 7),
]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,V,H,cap", SCORE_CASES, ids=[f"r{r}_v{v}_h{h}_cap{c}" for r, v, h, c in SCORE_CASES])
def test_score_head(report, rows, V, H, cap):
    """Planted rows (all-zero, one dominant logit, ties), special targets and random rows at each shape.  The dominant
    and tie rows failed the rule (4.6 to 12 x) while the head added 4 k-blocks per tensor-core accumulation into its
    fp32 sums; see test_score_head_accumulation_model."""
    key = f"kernel_score_r{rows}_v{V}_h{H}_cap{cap}"
    r, plan = score_case(report, key, rows, V, H, cap, seed=rows + V + H + cap, model_rows=MODEL_ROWS.get((rows, V, H), ()))
    assert r <= R, (key, report[f"fp64_{key}"])


@pytest.mark.gpu
def test_score_head_plans_reach_the_targets():
    """The cases above, planned on this GPU, include a CTA with >= 2 items at the launcher's own grid, tiles_m >= 3,
    nslices < 64, uneven slices and all of nslices 1, 2, 8 and 64."""
    sms = sms_of_device()
    plans = [score_plan_py(r, v, sms, c) for r, v, _, c in SCORE_CASES]
    assert any(p["items_per_cta"] >= 2 for p, (_, _, _, c) in zip(plans, SCORE_CASES) if c == 0)
    assert any(p["tiles_m"] >= 3 and p["tiles_n"] == 1187 for p in plans)
    assert {1, 2, 8, 64} <= {p["nslices"] for p in plans}
    assert any(p["slice_min"] != p["slice_max"] for p in plans)


@pytest.mark.gpu
def test_score_head_large_logits(report):
    """Logits of |l| ~ 100 (the norm weight scaled by 50): log-sum-exp dominated by a few columns, lp of most ids in
    the hundreds of nats."""
    key = "kernel_score_large_logits"
    r, _ = score_case(report, key, 300, 8320, 1024, seed=11, logit_scale=50.0, planted=False)
    assert r <= R, (key, report[f"fp64_{key}"])


@pytest.mark.gpu
def test_score_head_identity_gather_no_topk(report):
    """No gather map (row r reads hid[r]) and no top-8: the TOPK = false kernel."""
    key = "kernel_score_no_topk"
    r, _ = score_case(report, key, 300, 151936, 1024, seed=12, topk=False, gather=False)
    assert r <= R, (key, report[f"fp64_{key}"])


@pytest.mark.gpu
def test_score_head_negative_control_two_planes(report):
    """nplanes = 2 (the lo plane of the normed rows dropped) must FAIL the rule."""
    key = "kernel_score_planes2"
    r, _ = score_case(report, key, 300, 1000, 256, seed=13, nplanes=2, logit_scale=8.0, planted=False)
    assert r > R, report[f"fp64_{key}"]


@pytest.mark.gpu
def test_score_ids_past_two_m_tiles(tiny, report):
    """The product path: AsrInference.score_ids on the tiny model with 3 clips x 3 candidates of 32 ids (288 rows in
    one score head call: 3 M tiles), top-8 on, against oracle.score_ids in float64 under the rule."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    from test_score import add_errs, oracle_rows
    cfg, w, m32 = tiny
    m64 = O.OracleModel(cfg, w, dtype=torch.float64)
    clips = [synth.make_clip(140 + i, s) for i, s in enumerate((1.2, 2.5, 4.0))]
    rng = np.random.default_rng(21)
    cands = [[[int(v) for v in rng.integers(0, cfg.text.vocab_size, 32)] for _ in range(3)] for _ in clips]
    assert sum(len(c) for cs in cands for c in cs) > 2 * BM
    e = AsrInference.from_weights(config_tiny(), w, device=0)
    try:
        res = e.score_ids(clips, cands, top_logprobs=TK)
    finally:
        e.close()
    err = Err(False)
    for b, x in enumerate(clips):
        for sc in res[b]:
            l32, l64 = oracle_rows(m32, m64, x, sc.ids)
            add_errs(err, sc, l32, l64)
    assert getattr(err, "top_exact", 0) >= 100, getattr(err, "top_exact", 0)
    r = ratio(report, "kernel_score_ids_288_rows", err)
    assert r <= R, report["fp64_kernel_score_ids_288_rows"]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the alignment kernels
# ---------------------------------------------------------------------------------------------------------------------
def run_align(q, k, heads, group, utts, count, M_in=None):
    """utts: [(qrow0, N, T, a0, slot)]; q [q_rows][ldq]; k [slots][G][ctx][hd].  Returns (P, Z, M) as lists of
    per-utterance arrays: P and Z [nheads][N][T], M [N][T]."""
    q, k = np.ascontiguousarray(q, np.float32), np.ascontiguousarray(k, np.float32)
    hd = k.shape[3]
    cols = [np.ascontiguousarray([u[i] for u in utts], np.int32) for i in range(5)]
    hs = np.ascontiguousarray(heads, np.int32)
    total = sum(u[1] * u[2] for u in utts)
    P, Z = np.zeros((len(heads), total), np.float32), np.zeros((len(heads), total), np.float32)
    M = np.zeros(total, np.float32)
    Min = None if M_in is None else np.ascontiguousarray(np.concatenate([m.ravel() for m in M_in]), np.float32)
    a = AlignArgs()
    a.B, a.hd, a.group, a.nheads, a.count = len(utts), hd, group, len(heads), count
    a.heads = ptr(hs)
    a.qrow0, a.N, a.T, a.a0, a.slot = (ptr(c) for c in cols)
    a.q, a.q_rows, a.ldq = ptr(q), q.shape[0], q.shape[1]
    a.k, a.k_elems, a.seg_stride, a.head_stride = ptr(k), k.size, k[0].size, k[0, 0].size
    a.M_in, a.P_out, a.Z_out, a.M_out = ptr(Min), ptr(P), ptr(Z), ptr(M)
    _ok(heads_probe().asrbt_align(C.byref(a)))
    out, off = [], 0
    for (_, N, T, _, _) in utts:
        n = N * T
        out.append((P[:, off:off + n].reshape(-1, N, T), Z[:, off:off + n].reshape(-1, N, T), M[off:off + n].reshape(N, T)))
        off += n
    return out


def align_inputs(rng, utts, Hq, G, hd):
    q_rows = max(u[0] + u[1] for u in utts) + 2
    ctx = max(u[3] + u[2] for u in utts) + 3
    slots = max(u[4] for u in utts) + 1
    return (rng.standard_normal((q_rows, Hq * hd)).astype(np.float32),
            rng.standard_normal((slots, G, ctx, hd)).astype(np.float32))


def align_refs(q, k, heads, group, u, dtype):
    """Per listed head, P [N][T] of utterance u = (qrow0, N, T, a0, slot) in `dtype`."""
    q0, N, T, a0, slot = u
    hd = k.shape[3]
    return [align_ref(q[q0:q0 + N, h * hd:(h + 1) * hd], k[slot, h // group, a0:a0 + T], dtype) for h in heads]


def fold_ref(planes, M_in, count):
    """M_in + the width-7 medians of the planes' z-scores in list order, divided by count when > 0 (the dtype of the
    planes throughout)."""
    acc = M_in.astype(planes[0].dtype) if M_in is not None else np.zeros_like(planes[0])
    for p in planes:
        acc = acc + median7(zscore(p))
    return acc / acc.dtype.type(count) if count > 0 else acc


def align_errs(got, q, k, heads, group, utts, count, M_in=None):
    """(Err of P, Err of Z, Err of M) over the batch; M_in per utterance as (fp32, fp64) pairs or None."""
    eP, eZ, eM = Err(True), Err(True), Err(True)
    for b, u in enumerate(utts):
        P, Z, M = got[b]
        p64 = align_refs(q, k, heads, group, u, torch.float64)
        p32 = align_refs(q, k, heads, group, u, torch.float32)
        eP.add(P, np.stack(p32), np.stack(p64))
        eZ.add(Z, np.stack([zscore(p) for p in p32]), np.stack([zscore(p) for p in p64]))
        m32 = fold_ref(p32, None if M_in is None else M_in[b][0], count)
        m64 = fold_ref(p64, None if M_in is None else M_in[b][1], count)
        eM.add(M, m32, m64)
    return eP, eZ, eM


def check_align(report, key, errs, path):
    for stage, e in zip(("P", "Z", "M"), errs):
        k = f"{key}_{stage}"
        r = ratio(report, k, e, min_values=min(300, e.n))
        report[f"fp64_{k}"]["path"] = path
        assert r <= R, (k, report[f"fp64_{k}"])


ALIGN_N = [1, 15, 16, 17, 33, 200]
ALIGN_T = [1, 2, 3, 4, 5, 7, 31, 32, 33, 64, 65, 390]


@pytest.mark.gpu
@pytest.mark.parametrize("N", ALIGN_N)
def test_align_shapes(report, N):
    """Rows around the 16-row tile (1 .. 13 tiles) x keys around the 32-key tile, the median's pass-through (T <= 3)
    and its mirror padding at T = 4 .. 7; one utterance with nonzero qrow0 / a0 / slot, hd 128, two listed heads of
    different kv groups (out of order), one layer dividing by 2."""
    for T in ALIGN_T:
        rng = np.random.default_rng(1000 * N + T)
        utts = [(3, N, T, 5, 1)]
        heads = [3, 0]
        q, k = align_inputs(rng, utts, 4, 2, 128)
        got = run_align(q, k, heads, 2, utts, 2)
        if T <= 3:
            for b, u in enumerate(utts):                  # the median passes z through: M = mean of the z planes
                assert np.allclose(got[b][2], got[b][1].sum(0) / 2, rtol=0, atol=1e-6)
        if N == 1:
            assert not got[0][1].any()                    # one row: std 0, z = 0
        check_align(report, f"kernel_align_N{N}_T{T}", align_errs(got, q, k, heads, 2, utts, 2),
                    {"row_tiles": -(-N // PROB_ROWS), "key_tiles": -(-T // 32), "median": "identity" if T <= 3 else "mirror"})


@pytest.mark.gpu
@pytest.mark.parametrize("group", [1, 2, 4, 8])
def test_align_gqa_groups(report, group):
    """Query heads per kv head 1 / 2 / 4 / 8 at hd 128 (G = 2 kv heads): listed heads from both kv groups, in an order
    that is not ascending."""
    rng = np.random.default_rng(group)
    Hq = 2 * group
    heads = sorted(range(Hq), key=lambda h: (h * 7 + 3) % Hq)[: min(Hq, 5)]
    assert heads != sorted(heads) or len(heads) == 1
    if group == 1:
        heads = [1, 0]
    assert {h // group for h in heads} == {0, 1}
    utts = [(0, 33, 65, 7, 0)]
    q, k = align_inputs(rng, utts, Hq, 2, 128)
    got = run_align(q, k, heads, group, utts, len(heads))
    check_align(report, f"kernel_align_group{group}", align_errs(got, q, k, heads, group, utts, len(heads)),
                {"group": group, "heads": heads})


@pytest.mark.gpu
def test_align_ragged_batch_two_layers(report):
    """Three utterances of different N / T with distinct slots and nonzero qrow0 / a0 in one launch, then a second
    layer call: the first adds its medians into M (count 0), the second adds into that M and divides by the 5 listed
    heads of both layers.  Also a batch of one of the utterances gives the same bits as its place in the batch."""
    rng = np.random.default_rng(31)
    Hq, G, hd = 8, 2, 128
    utts = [(2, 17, 390, 9, 2), (40, 200, 33, 1, 0), (300, 5, 7, 30, 3)]
    q1, k1 = align_inputs(rng, utts, Hq, G, hd)
    q2, k2 = align_inputs(rng, utts, Hq, G, hd)
    h1, h2 = [6, 1, 4], [2, 7]
    got1 = run_align(q1, k1, h1, Hq // G, utts, 0)
    check_align(report, "kernel_align_ragged_layer1", align_errs(got1, q1, k1, h1, Hq // G, utts, 0),
                {"B": 3, "layer": 1, "count": 0})
    m_in = [g[2] for g in got1]
    got2 = run_align(q2, k2, h2, Hq // G, utts, 5, M_in=m_in)
    # the reference M: both layers' planes folded from zero in (layer, head) order
    eM = Err(True)
    for b, u in enumerate(utts):
        p = {dt: align_refs(q1, k1, h1, Hq // G, u, dt) + align_refs(q2, k2, h2, Hq // G, u, dt)
             for dt in (torch.float32, torch.float64)}
        eM.add(got2[b][2], fold_ref(p[torch.float32], None, 5), fold_ref(p[torch.float64], None, 5))
    eP, eZ, _ = align_errs(got2, q2, k2, h2, Hq // G, utts, 5,
                           M_in=[(m, m.astype(np.float64)) for m in m_in])
    check_align(report, "kernel_align_ragged_layer2", (eP, eZ, eM), {"B": 3, "layer": 2, "count": 5})
    alone = run_align(q1, k1, h1, Hq // G, [utts[1]], 0)[0]
    for a, b in zip(alone, got1[1]):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_align_column_of_equal_values(report):
    """Every aligned row of an utterance has the same q: each column of P holds one value (bitwise, whatever the row
    tile), its std is 0 and every z-score must be exactly 0, so M = M_in / count exactly.  Before the shifted mean in
    align_zscore_kernel about half of such columns came back at z = +-1.  T = 1 (every P = 1) likewise."""
    rng = np.random.default_rng(41)
    utts = [(0, 33, 65, 3, 0), (40, 17, 1, 0, 1), (60, 3, 40, 2, 2)]
    q, k = align_inputs(rng, utts, 4, 2, 128)
    for q0, N, _, _, _ in utts:
        q[q0:q0 + N] = q[q0]
    m_in = [rng.standard_normal((u[1], u[2])).astype(np.float32) for u in utts]
    got = run_align(q, k, [2, 1], 2, utts, 4, M_in=m_in)
    for b, u in enumerate(utts):
        P, Z, M = got[b]
        assert (P == P[:, :1, :]).all(), b
        assert not any(zscore(p.astype(np.float64)).any() for p in P)    # the spec in float64 on these P
        assert not Z.any(), (b, np.count_nonzero(Z), Z.size)
        assert np.array_equal(M, m_in[b] / np.float32(4)), b
    eP = Err(True)
    for b, u in enumerate(utts):
        eP.add(got[b][0], np.stack(align_refs(q, k, [2, 1], 2, u, torch.float32)),
               np.stack(align_refs(q, k, [2, 1], 2, u, torch.float64)))
    r = ratio(report, "kernel_align_equal_columns_P", eP)
    assert r <= R


@pytest.mark.gpu
def test_align_probe_refusals():
    """Shapes the probe must refuse before any launch: a head outside the q row, keys past the K cache, N = 0."""
    rng = np.random.default_rng(51)
    utts = [(0, 4, 8, 0, 0)]
    q, k = align_inputs(rng, utts, 2, 1, 64)
    from qwen3_asr_rs_b200 import _lib
    for heads, bad in (([2], utts), ([0], [(0, 4, k.shape[2] + 1, 0, 0)]), ([0], [(0, 0, 8, 0, 0)]),
                       ([0], [(q.shape[0], 4, 8, 0, 0)])):
        with pytest.raises(_lib.AsrbError):
            run_align(q, k, heads, 2, bad, 1)
    run_align(q, k, [1], 2, utts, 1)                      # and the probe still runs
