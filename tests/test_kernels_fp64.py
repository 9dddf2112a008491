"""Kernel-level precision: each encoder / prefill kernel against a float64 reference of the same operation.

The model-level suite (test_precision_fp64.py and the files built on it) reaches the kernels only through the shapes
its clips happen to produce.  This file drives the kernels one at a time through the library's test probes
(csrc/probe.h) at activation shapes chosen for the code paths inside them: the wgmma GEMM's k-split factors, its
persistent work items, its tile edges and its two SIMT fall-backs; the fp32 attention kernel's causal tile pairing,
query offsets, GQA groups and ragged segments; the split3 producers at the edges of their domain.

Every GPU case applies the rule of test_precision_fp64.py (e_gpu <= R * max(e_32, floor), R = 4) with a float64
reference computed from the same fp32 inputs and exact bf16 weights, and an fp32 reference of the same operation in
plain torch on the CPU.  Each case first asserts the path the probe reports, so that a case that drifted off its
target fails instead of passing on an easier path.  The path, e_gpu, e_32 and the ratio go into the report.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_precision_fp64 import R, Err, ratio

BM = BN = 128                    # wgmma GEMM output tile
BK = 64                          # its k-block
SPLITK_WS_FLOATS = 4 * 64 * 128 * 128
EPI = {"plain": 0, "swiglu": 1, "conv_parity": 2, "conv_feat": 3, "convout": 4}
SMS_SXM, SMS_PCIE = 132, 114     # H100 SXM5 / PCIe SM counts
OVERFLOW_BITS = 0x7F7F8000       # |x| at or above: bf16 round-to-nearest of x is infinite


# ---------------------------------------------------------------------------------------------------------------------
# bindings of the probes (csrc/probe.h)
# ---------------------------------------------------------------------------------------------------------------------
class GemmArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("impl", "a_mode", "epi", "M", "N", "K", "nplanes")] + [
        ("x", C.c_void_p)] + [(n, C.c_int) for n in ("OH", "OW", "Hh", "Wh", "cpad")] + [
        ("w", C.c_void_p), ("bias", C.c_void_p), ("gelu", C.c_int), ("residual", C.c_void_p), ("row_map", C.c_void_p),
        ("pos", C.c_void_p), ("pos_period", C.c_int), ("use_splitk", C.c_int),
        ("out_f32", C.c_void_p), ("out_f32_rows", C.c_int64), ("ldo", C.c_int),
        ("out_planes", C.c_void_p), ("out_plane_elems", C.c_int64), ("lds", C.c_int),
        ("Hh2", C.c_int), ("Wh2", C.c_int), ("cpad2", C.c_int)]


class AttnArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("hd", "nseg", "nheads", "group", "causal", "keys_in_rows", "max_len")] + [
        ("seg_q0", C.c_void_p), ("seg_len", C.c_void_p), ("seg_pos0", C.c_void_p),
        ("buf", C.c_void_p), ("buf_elems", C.c_int64), ("q_off", C.c_int64), ("k_off", C.c_int64), ("v_off", C.c_int64),
        ("ldq", C.c_int), ("ldk", C.c_int), ("seg_stride", C.c_int64), ("head_stride", C.c_int64),
        ("out_planes", C.c_void_p), ("out_rows", C.c_int64), ("ldo", C.c_int)]


_probe = None


def probe():
    global _probe
    if _probe is None:
        from qwen3_asr_rs_b200 import _lib
        lib = _lib.load_library()
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
        sig = {"asrbt_split3": [vp, i64, vp], "asrbt_norm_s3": [i32, vp, vp, vp, i32, i32, f32, vp],
               "asrbt_gemm_plan": [i32] * 10 + [vp], "asrbt_gemm": [C.POINTER(GemmArgs), vp],
               "asrbt_attention": [C.POINTER(AttnArgs)]}
        for name, args in sig.items():
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = C.c_int
        _probe = lib
    return _probe


def _ok(code):
    from qwen3_asr_rs_b200 import _lib
    _lib.check(code)


def ptr(a):
    return None if a is None else a.ctypes.data


def c32(a):
    return np.ascontiguousarray(a, np.float32)


def planes_value(p):
    """float64 hi + mid + lo of 3 stacked bf16 planes (exact: three bf16 values sum exactly in float64)."""
    v = bf16_to_f32(p).astype(np.float64)
    return v[0] + v[1] + v[2]


PLAN_KEYS = ("tc", "splits", "tiles_m", "tiles_n", "grid", "items_per_cta", "simt_fallbacks", "box_h")


def gemm_plan(M, N, K, mode=0, epi="plain", sms=SMS_SXM, splitk=True, OH=0, OW=0, cpad=0):
    out = np.zeros(8, np.int32)
    _ok(probe().asrbt_gemm_plan(M, N, K, mode, EPI[epi], sms, int(splitk), OH, OW, cpad, ptr(out)))
    return dict(zip(PLAN_KEYS, out.tolist()))


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatement of split3 (common.cuh): hi = bf16_rn(x), mid = bf16_rn(x - hi), lo = bf16_rn(x - hi - mid)
# ---------------------------------------------------------------------------------------------------------------------
def bf16_rne(x):
    """float32 -> bf16 bits, round to nearest even (cvt.rn.bf16.f32); NaN -> the canonical 0x7FFF."""
    x = np.asarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r[np.isnan(x)] = 0x7FFF
    return r


def bf16_to_f32(b):
    return (np.asarray(b, np.uint16).astype(np.uint32) << 16).view(np.float32)


def split3_np(x):
    """[3, n] bf16 bits of (hi, mid, lo), fp32 arithmetic as on the GPU (IEEE, no flush to zero)."""
    x = np.asarray(x, np.float32)
    with np.errstate(all="ignore"):
        hi = bf16_rne(x)
        r = x - bf16_to_f32(hi)
        mid = bf16_rne(r)
        lo = bf16_rne(r - bf16_to_f32(mid))
    return np.stack([hi, mid, lo])


def torch_bf16_bits(x):
    return torch.from_numpy(np.asarray(x, np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def split3_values():
    """Random full-mantissa values over every exponent, subnormals, +-0, powers of two, bf16 halfway cases (ties to
    even both ways), the last values below the overflow threshold, +-FLT_MAX, +-inf and NaN."""
    rng = np.random.default_rng(3)
    parts = [rng.integers(0, 0x7F800000, 200000, dtype=np.uint32),                 # any finite positive
             rng.integers(1, 1 << 23, 20000, dtype=np.uint32),                      # subnormals
             np.array([0, 1, 2, 0x7FFFFF, 1 << 23, 0x7FFFFFE, 0x8000000], np.uint32),
             (np.arange(1, 255, dtype=np.uint32) << 23),                            # powers of two
             (rng.integers(1, 254, 4000, dtype=np.uint32) << 23) | (rng.integers(0, 128, 4000, dtype=np.uint32) << 16) | 0x8000,
             (rng.integers(1, 254, 4000, dtype=np.uint32) << 23) | (rng.integers(0, 1 << 23, 4000, dtype=np.uint32) & ~np.uint32(0xFF)) | 0x80,
             np.array([OVERFLOW_BITS - 1, OVERFLOW_BITS, OVERFLOW_BITS + 1, 0x7F7FFFFF, 0x7F800000, 0x7FC00000, 0x7FFFFFFF], np.uint32)]
    u = np.concatenate(parts)
    return np.concatenate([u, u | np.uint32(0x80000000)]).view(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: split3
# ---------------------------------------------------------------------------------------------------------------------
def test_split3_restatement_matches_torch_bf16_rounding():
    """Each plane of the restatement is torch's bf16 round-to-nearest-even of the fp32 remainder, bitwise, for every
    non-NaN input (NaN planes are NaN in both; the bit pattern of a NaN is not part of the claim)."""
    x = split3_values()
    got = split3_np(x)
    with np.errstate(all="ignore"):
        r1 = x - bf16_to_f32(torch_bf16_bits(x))
        r2 = r1 - bf16_to_f32(torch_bf16_bits(r1))
    want = np.stack([torch_bf16_bits(x), torch_bf16_bits(r1), torch_bf16_bits(r2)])
    gv, wv = bf16_to_f32(got), bf16_to_f32(want)
    assert np.array_equal(np.isnan(gv), np.isnan(wv))
    keep = ~np.isnan(wv)
    assert np.array_equal(got[keep], want[keep])
    # ties: a value exactly halfway between two bf16 values rounds to the even one
    assert bf16_rne(np.array([1.0 + 2 ** -8], np.float32))[0] == 0x3F80
    assert bf16_rne(np.array([1.0 + 3 * 2 ** -8], np.float32))[0] == 0x3F82


def _split3_domain(x):
    """(finite sum error, non-finite sums) of the restatement over x."""
    p = split3_np(x)
    with np.errstate(all="ignore"):
        s = planes_value(p)
        return s, np.abs(s - x.astype(np.float64))


def test_split3_domain_statement():
    """hi + mid + lo == x exactly for 2^-110 <= |x| < 0x7F7F8000 (bits), and to 1 ulp for 2^-111 <= |x| < 2^-110;
    below 2^-111 the lo plane cannot hold the last bits (bf16's smallest subnormal is 2^-133), so the error exceeds
    1 ulp there but stays <= 2^-134 absolute, far below anything an activation carries into a GEMM; at and above 0x7F7F8000 hi rounds to infinity and the sum is NaN
    or infinite, never a wrong finite value; inf and NaN inputs give non-finite sums.  Checked on the value set, on
    every mantissa of the exponents around each edge, and on every subnormal with an odd stride."""
    rng = np.random.default_rng(11)
    sets = [split3_values(), (np.arange(1, 1 << 23, 7, dtype=np.uint32)).view(np.float32)]
    for e in (0, 1, 2, 15, 16, 17, 18, 127, 200, 253, 254):      # biased exponents: subnormals, 2^-111, 2^-110, 1, top
        m = np.arange(0, 1 << 23, 1 if e in (16, 17) else 7, dtype=np.uint32)
        sets.append(((np.uint32(e) << 23) | m).view(np.float32))
    sets.append(rng.integers(0, 0xFFFFFFFF, 500000, dtype=np.uint32, endpoint=True).view(np.float32))
    for x in sets:
        x = np.concatenate([x, -x])
        s, err = _split3_domain(x)
        bits = np.abs(x).view(np.uint32)
        fin = np.isfinite(x) & (bits < OVERFLOW_BITS)
        assert np.isfinite(s[fin]).all()
        with np.errstate(all="ignore"):
            ulp = np.spacing(np.abs(x)).astype(np.float64)
        exact = fin & (np.abs(x) >= 2.0 ** -110)
        assert (err[exact] == 0).all(), x[exact][err[exact] != 0][:5]
        one_ulp = fin & (np.abs(x) >= 2.0 ** -111)
        assert (err[one_ulp] <= ulp[one_ulp]).all()
        assert (err[fin & ~one_ulp] <= 2.0 ** -134).all()
        over = ~np.isfinite(x) | (bits >= OVERFLOW_BITS)
        assert not np.isfinite(s[over]).any()
    # the edges themselves
    s, _ = _split3_domain(np.array([OVERFLOW_BITS - 1, OVERFLOW_BITS], np.uint32).view(np.float32))
    assert np.isfinite(s[0]) and np.isnan(s[1])
    x = np.array([2.0 ** -148, 2.0 ** -120 + 2.0 ** -140], np.float32)
    s, err = _split3_domain(x)
    assert (err > np.spacing(x)).all() and (err <= 2.0 ** -134).all(), err


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the GEMM launch plan
# ---------------------------------------------------------------------------------------------------------------------
def plan_py(M, N, K, mode=0, epi="plain", sms=SMS_SXM, splitk=True, OH=0, OW=0, cpad=0):
    """The wgmma GEMM's launch decision restated: the shape limits that send a GEMM to the SIMT kernel, the k-split
    factor (plain / conv_out epilogues with a workspace, <= 64 tiles, the most of 4, 3, 2 splits that divides the
    k-blocks, leaves >= 6 k-blocks per split and keeps the items within ~1.1 waves) and the persistent grid."""
    simt = dict(tc=0, splits=1, tiles_m=0, tiles_n=0, grid=0, items_per_cta=0, simt_fallbacks=0, box_h=0)
    e = EPI[epi]
    if K % BK or M <= 0 or N <= 0 or N % 8:
        return simt
    splits, box_h = 1, 0
    tiles_n = -(-N // BN)
    if mode == 0:
        if e not in (0, 1, 4):
            return simt
        tiles_m = -(-M // BM)
        tiles, kb = tiles_m * tiles_n, K // BK
        if e in (0, 4) and splitk and tiles <= 64 and 4 * M * N <= SPLITK_WS_FLOATS:
            for sp in (4, 3, 2):
                if kb % sp == 0 and kb // sp >= 6 and tiles * sp <= sms + sms // 12:
                    splits = sp
                    break
    else:
        if cpad % BK or OW > BM or OW <= 0 or OH <= 0 or e not in (2, 3):
            return simt
        box_h = min(OH, BM // OW)
        tiles_m = (M // (OH * OW)) * -(-OH // box_h)
    items = tiles_m * tiles_n * splits
    grid = min(items, sms)
    if grid <= 0:
        return simt
    return dict(tc=1, splits=splits, tiles_m=tiles_m, tiles_n=tiles_n, grid=grid, items_per_cta=-(-items // grid),
                simt_fallbacks=0, box_h=box_h)


PLAN_M = [1, 64, 127, 128, 129, 256, 384, 513, 640, 700, 767, 1024, 1025, 2048, 4100]
PLAN_N = [8, 120, 136, 896, 1000, 1001, 1024, 2048, 3584, 6144]
PLAN_K = [64, 192, 200, 768, 896, 1024, 1152, 1536, 2048, 3072, 3584, 4608, 7680]


@pytest.mark.parametrize("sms", [SMS_SXM, SMS_PCIE])
def test_gemm_plan_matches_restatement(sms):
    """asrbt_gemm_plan (the function launch_gemm_tc itself calls) against plan_py over M x N x K x epilogue x
    workspace, plain and conv; and every outcome the rule allows is reached: splits 1-4, a CTA with >= 2 work items
    with and without split, and both SIMT fall-backs."""
    seen = set()
    for M in PLAN_M:
        for N in PLAN_N:
            for K in PLAN_K:
                for epi in ("plain", "swiglu", "convout", "conv_parity"):
                    for ws in (True, False):
                        got, want = gemm_plan(M, N, K, 0, epi, sms, ws), plan_py(M, N, K, 0, epi, sms, ws)
                        assert got == want, (M, N, K, epi, ws, got, want)
                        seen.add(("split", got["splits"]) if got["tc"] else ("simt", N % 8 != 0, K % BK != 0))
                        if got["tc"] and got["items_per_cta"] >= 2:
                            seen.add(("multi", got["splits"] > 1))
    for (OH, OW) in ((32, 25), (16, 13), (32, 20), (16, 10), (4, 130)):
        for chunks in (1, 3, 55):
            for epi in ("conv_parity", "conv_feat", "plain"):
                for cpad in (128, 512, 480):
                    a = (chunks * OH * OW, 480, 9 * cpad, 1, epi, sms, True, OH, OW, cpad)
                    assert gemm_plan(*a) == plan_py(*a), a
    want = {("split", 1), ("split", 2), ("split", 3), ("split", 4), ("simt", True, False), ("simt", False, True),
            ("multi", True), ("multi", False)}
    assert want <= seen, want - seen


def test_gemm_plan_production_shapes():
    """The split factors named in the plan's own comment and in the model's shapes (0.6B: d_model 896, hidden 1024,
    intermediate 3072, q_dim 2048; 132 SMs)."""
    assert gemm_plan(700, 1024, 2048)["splits"] == 2                     # o_proj, 513..1024 prompt rows
    assert gemm_plan(1025, 1024, 2048)["splits"] == 1
    assert gemm_plan(600, 1024, 3072)["splits"] == 3                     # down_proj, 513..640 rows
    assert gemm_plan(700, 1024, 3072)["splits"] == 2
    assert gemm_plan(1025, 1024, 3072)["splits"] == 1
    assert gemm_plan(55 * 13, 896, 7680, epi="convout")["splits"] == 3   # conv_out, ~50-59 chunks
    assert gemm_plan(55 * 13, 896, 7680, epi="convout", splitk=False)["splits"] == 1
    assert gemm_plan(32, 1024, 2048, epi="swiglu")["splits"] == 1        # only plain / conv_out epilogues split


def test_gemm_plan_workspace_cap_is_implied_by_the_tile_limit():
    """The workspace condition 4 M N <= SPLITK_WS_FLOATS never decides: <= 64 tiles of 128 x 128 already bound M N by
    64 * 128^2, which is the cap over 4.  So a workspace of SPLITK_WS_FLOATS is always enough for a split GEMM; the
    condition guards a later change of either constant."""
    for M in range(1, 64 * BM + 1, 37):
        for N in range(8, 64 * BN + 1, 8 * 13):
            if -(-M // BM) * -(-N // BN) <= 64:
                assert 4 * M * N <= SPLITK_WS_FLOATS
    assert 4 * (64 * BM) * BN == SPLITK_WS_FLOATS


# ---------------------------------------------------------------------------------------------------------------------
# references (plain torch on the CPU) and "the rule sees it" controls
# ---------------------------------------------------------------------------------------------------------------------
def gemm_ref(x, w, dtype, bias=None, gelu=False, residual=None):
    """x [M][K] fp32, w [N][K] exact bf16 values: y = x w^T (+ bias, GELU, + residual) in `dtype`."""
    t = lambda a: torch.from_numpy(np.asarray(a)).to(dtype)
    y = t(x) @ t(w).T
    if bias is not None:
        y = y + t(bias)
    if gelu:
        y = torch.nn.functional.gelu(y)
    if residual is not None:
        y = y + t(residual)
    return y.numpy()


def attn_ref(q, k, v, dtype, causal, pos0=0, extra_keys=0, boundary_shift=0):
    """One segment, all heads: q [L][H][hd], k, v [keys][G][hd] (G kv heads); query i at position pos0 + i sees keys
    0..pos0 + i (causal) or all of its first `pos0 + L` keys.  extra_keys / boundary_shift are mutations for the
    controls (padded keys left unmasked, an off-by-one causal boundary)."""
    L, H, hd = q.shape
    G = k.shape[1]
    nk = pos0 + L + extra_keys
    qt = torch.from_numpy(q).to(dtype).permute(1, 0, 2)
    kt = torch.from_numpy(k[:nk]).to(dtype).permute(1, 0, 2).repeat_interleave(H // G, 0)
    vt = torch.from_numpy(v[:nk]).to(dtype).permute(1, 0, 2).repeat_interleave(H // G, 0)
    s = (qt @ kt.transpose(1, 2)) / math.sqrt(hd)
    if causal:
        j = torch.arange(nk)[None, :]
        i = torch.arange(L)[:, None]
        s = s.masked_fill(j > pos0 + i + boundary_shift, float("-inf"))
    return (torch.softmax(s, -1) @ vt).permute(1, 0, 2).numpy()


def _rule_ratio(y_bad, y32, y64):
    return ratio({}, "control", Err(True).add(y_bad, y32, y64))


def test_rule_sees_a_dropped_k_block():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((129, 768)).astype(np.float32)
    w = bf16_to_f32(bf16_rne(rng.standard_normal((136, 768)) * 0.05))
    y64, y32 = gemm_ref(x, w, torch.float64), gemm_ref(x, w, torch.float32)
    for kb in (0, 5, 11):
        keep = np.ones(768, bool)
        keep[kb * BK:(kb + 1) * BK] = False
        assert _rule_ratio(gemm_ref(x[:, keep], w[:, keep], torch.float32), y32, y64) > R


def test_rule_sees_a_dropped_tail_row():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((129, 192)).astype(np.float32)
    w = bf16_to_f32(bf16_rne(rng.standard_normal((136, 192)) * 0.05))
    y64, y32 = gemm_ref(x, w, torch.float64), gemm_ref(x, w, torch.float32)
    bad = y32.copy()
    bad[-1] = 0.0                       # the row of the M tail's only row left unwritten (zero-initialised output)
    assert _rule_ratio(bad, y32, y64) > R


def _attn_inputs(rng, L, H, G, hd, nkeys):
    return (rng.standard_normal((L, H, hd)).astype(np.float32), rng.standard_normal((nkeys, G, hd)).astype(np.float32),
            rng.standard_normal((nkeys, G, hd)).astype(np.float32))


def test_rule_sees_attention_mutations():
    """Off-by-one causal boundary (either way), the query offset ignored, one padded key left unmasked: each is far
    over R against fp32 attention."""
    rng = np.random.default_rng(4)
    q, k, v = _attn_inputs(rng, 97, 4, 2, 64, 300 + 97 + 1)
    y64, y32 = attn_ref(q, k, v, torch.float64, True), attn_ref(q, k, v, torch.float32, True)
    for shift in (1, -1):
        bad = attn_ref(q, k, v, torch.float32, True, boundary_shift=shift)
        if shift == -1:
            bad[0] = y32[0]             # row 0 would have no key at all
        assert _rule_ratio(bad, y32, y64) > R
    y64o, y32o = attn_ref(q, k, v, torch.float64, True, pos0=300), attn_ref(q, k, v, torch.float32, True, pos0=300)
    assert _rule_ratio(attn_ref(q, k, v, torch.float32, True, pos0=0), y32o, y64o) > R
    y64n, y32n = attn_ref(q, k, v, torch.float64, False), attn_ref(q, k, v, torch.float32, False)
    assert _rule_ratio(attn_ref(q, k, v, torch.float32, False, extra_keys=1), y32n, y64n) > R


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def run_split3(x):
    x = c32(x)
    out = np.zeros((3, x.size), np.uint16)
    _ok(probe().asrbt_split3(ptr(x), x.size, ptr(out)))
    return out


def bf16_weights(rng, N, K, scale=None, positive=False):
    w = rng.standard_normal((N, K)) * (scale if scale is not None else 1.0 / math.sqrt(K))
    if positive:
        w = np.abs(w)
    bits = bf16_rne(w.astype(np.float32))
    return bits, bf16_to_f32(bits)


def run_gemm(x, wbits, N, K, impl=1, epi="plain", nplanes=3, bias=None, gelu=False, residual=None, row_map=None,
             pos=None, out_rows=None, ldo=None, planes_elems=0, lds=0, conv=None, splitk=True):
    """(fp32 output or None, planes or None, path report)."""
    x = c32(x)
    wbits = np.ascontiguousarray(wbits, np.uint16)
    a = GemmArgs()
    a.impl, a.epi, a.N, a.K, a.nplanes, a.gelu, a.use_splitk = impl, EPI[epi], N, K, nplanes, int(gelu), int(splitk)
    keep = [x, wbits]
    if conv is None:
        a.a_mode, a.M = 0, x.shape[0]
    else:
        a.a_mode, a.M = 1, conv["M"]
        a.OH, a.OW, a.Hh, a.Wh, a.cpad = conv["OH"], conv["OW"], conv["Hh"], conv["Wh"], conv["cpad"]
        a.Hh2, a.Wh2, a.cpad2 = conv.get("Hh2", 0), conv.get("Wh2", 0), conv.get("cpad2", 0)
    a.x, a.w = ptr(x), ptr(wbits)
    for name, arr, dt in (("bias", bias, np.float32), ("residual", residual, np.float32), ("row_map", row_map, np.int32),
                          ("pos", pos, np.float32)):
        if arr is not None:
            arr = np.ascontiguousarray(arr, dt)
            keep.append(arr)
            setattr(a, name, ptr(arr))
    if pos is not None:
        a.pos_period = pos.shape[0]
    out = planes = None
    if ldo:
        out = np.zeros((out_rows, ldo), np.float32)
        a.out_f32, a.out_f32_rows, a.ldo = ptr(out), out_rows, ldo
    if planes_elems:
        planes = np.zeros((3, planes_elems), np.uint16)
        a.out_planes, a.out_plane_elems, a.lds = ptr(planes), planes_elems, lds
    plan = np.zeros(8, np.int32)
    _ok(probe().asrbt_gemm(C.byref(a), ptr(plan)))
    return out, planes, dict(zip(PLAN_KEYS, plan.tolist()))


def sms_of_device():
    return torch.cuda.get_device_properties(0).multi_processor_count


def record(report, key, err, path):
    r = ratio(report, key, err)
    report[f"fp64_{key}"]["path"] = path
    return r


def check_path(report, key, err, path):
    record(report, key, err, path)
    assert report[f"fp64_{key}"]["ratio"] <= R, (key, report[f"fp64_{key}"])


def find_shape(sms, want, Ms=(128, 256, 384, 512, 640, 768, 1024), Ns=(128, 256, 384, 512, 640, 896, 1024, 1152),
               Ks=(768, 1152, 1536, 2304, 3072, 4608), epi="plain"):
    """The cheapest (M, N, K) whose plan on this GPU satisfies want(plan)."""
    best = None
    for M in Ms:
        for N in Ns:
            for K in Ks:
                p = gemm_plan(M, N, K, epi=epi, sms=sms)
                if want(p) and (best is None or M * N * K < best[0]):
                    best = (M * N * K, (M, N, K))
    assert best is not None, "no shape reaches the target on this GPU"
    return best[1]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: split3 and the norm producers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_split3_gpu_matches_restatement_bitwise():
    x = split3_values()
    got, want = run_split3(x), split3_np(x)
    gv = bf16_to_f32(got)
    nan = np.isnan(bf16_to_f32(want))
    assert np.array_equal(np.isnan(gv), nan)
    assert np.array_equal(got[~nan], want[~nan]), np.argwhere(got != want)[:5]


def norm_ref(x, w, b, eps, kind, dtype):
    t = lambda a: torch.from_numpy(np.asarray(a)).to(dtype)
    x = t(x)
    if kind == 0:
        mean = x.mean(-1, keepdim=True)
        var = ((x - mean) ** 2).mean(-1, keepdim=True)
        return ((x - mean) / torch.sqrt(var + eps) * t(w) + t(b)).numpy()
    return (x * (1.0 / torch.sqrt((x * x).mean(-1, keepdim=True) + eps)) * t(w)).numpy()


def run_norm(kind, x, w, b, eps):
    x = c32(x)
    rows, dim = x.shape
    out = np.zeros((3, rows * dim), np.uint16)
    w, b = c32(w), c32(b)
    _ok(probe().asrbt_norm_s3(kind, ptr(x), ptr(w), ptr(b), rows, dim, eps, ptr(out)))
    return planes_value(out).reshape(rows, dim)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [192, 320, 896, 1024, 2048])
@pytest.mark.parametrize("kind", [0, 1], ids=["layernorm", "rmsnorm"])
def test_norm_producers(report, kind, dim):
    """Rows of ordinary scale, rows with mean 1e3 and std 1, tiny rows (std 1e-4 and 1e-20: eps dominates) and
    constant rows.  A constant row of exactly representable value has a zero centred row: LayerNorm gives b exactly."""
    rng = np.random.default_rng(dim + kind)
    eps = 1e-5 if kind == 0 else 1e-6
    w = (1.0 + 0.1 * rng.standard_normal(dim)).astype(np.float32)
    b = (0.1 * rng.standard_normal(dim)).astype(np.float32)
    groups = {"plain": rng.standard_normal((16, dim)), "mean1e3": 1e3 + rng.standard_normal((16, dim)),
              "tiny1e-4": 1e-4 * rng.standard_normal((8, dim)), "tiny1e-20": 1e-20 * rng.standard_normal((8, dim)),
              "const": np.repeat(np.array([[0.75], [-3.0], [1024.0], [0.0]]), dim, 1)}
    for name, x in groups.items():
        x = x.astype(np.float32)
        y = run_norm(kind, x, w, b, eps)
        y64, y32 = norm_ref(x, w, b, eps, kind, torch.float64), norm_ref(x, w, b, eps, kind, torch.float32)
        if name == "const" and kind == 0:
            assert np.array_equal(y, np.broadcast_to(b.astype(np.float64), y.shape))
        if name == "const" and kind == 1:
            assert np.array_equal(y[3], np.zeros(dim))          # the zero row stays zero
            x, y, y64, y32 = x[:3], y[:3], y64[:3], y32[:3]
        check_path(report, f"kernel_norm_{['ln', 'rms'][kind]}_d{dim}_{name}",
                   Err(True).add(y, y32, y64), {"kernel": ["layernorm_s3", "rmsnorm_s3"][kind], "rows": len(x)})


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the GEMM
# ---------------------------------------------------------------------------------------------------------------------
def plain_case(report, key, M, N, K, impl=1, seed=0, epi="plain", bias=True, gelu=False, residual=True, planes_out=False,
               nplanes=3, x=None, wpair=None, expect=None, splitk=True):
    """One plain GEMM through the probe against fp32 / fp64 references; returns (ratio, path, output)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((M, K)).astype(np.float32) if x is None else x
    wbits, w = bf16_weights(rng, N, K) if wpair is None else wpair
    bb = (0.1 * rng.standard_normal(N)).astype(np.float32) if bias else None
    res = rng.standard_normal((M, N)).astype(np.float32) if residual else None
    if epi == "swiglu":
        out, planes, path = run_gemm(x, wbits, N, K, impl, "swiglu", nplanes, out_rows=M, ldo=N // 2,
                                     planes_elems=M * (N // 2) if planes_out else 0, lds=N // 2, splitk=splitk)
        t = {dt: torch.from_numpy(gemm_ref(x, w, dt)) for dt in (torch.float32, torch.float64)}
        ref = {dt: (torch.nn.functional.silu(a[:, 0::2]) * a[:, 1::2]).numpy() for dt, a in t.items()}
    else:
        out, planes, path = run_gemm(x, wbits, N, K, impl, epi, nplanes, bias=bb, gelu=gelu, residual=res,
                                     out_rows=M if not planes_out else None, ldo=N if not planes_out else 0,
                                     planes_elems=M * N if planes_out else 0, lds=N, splitk=splitk)
        ref = {dt: gemm_ref(x, w, dt, bb, gelu, res) for dt in (torch.float32, torch.float64)}
    y = planes_value(planes).reshape(M, -1) if planes_out else out
    if expect:
        for k, v in expect.items():
            assert v(path[k]) if callable(v) else path[k] == v, (key, k, path)
    err = Err(True).add(y, ref[torch.float32], ref[torch.float64])
    r = record(report, key, err, dict(path, M=M, N=N, K=K, impl=["simt", "tc"][impl], epi=epi, nplanes=nplanes))
    return r, path, y


SHAPES = [(1, 1000, 64), (127, 8, 192), (128, 1000, 768), (129, 3584, 192), (1025, 136, 3072), (129, 1000, 7680),
          (1025, 1000, 768), (128, 136, 7680)]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["tc", "simt"])
@pytest.mark.parametrize("M,N,K", SHAPES, ids=[f"{m}x{n}x{k}" for m, n, k in SHAPES])
def test_gemm_tile_edges(report, impl, M, N, K):
    """M in {1, 127, 128, 129, 1025} (M % 128 = 1, 127, 0), N in {8, 136, 1000, 3584}, K in {64, 192, 768, 3072, 7680}
    with bias and in-place residual, on the wgmma GEMM (split or not, as the plan decides on this GPU) and the SIMT
    GEMM.  The SIMT GEMM's long-K cases failed the rule (10x at K = 7680) while it summed all of K in one running fp32
    register; it now adds 256-wide chunks like the wgmma kernel."""
    sms = sms_of_device()
    want = plan_py(M, N, K, sms=sms)
    expect = {"tc": 1, "splits": want["splits"], "grid": want["grid"], "simt_fallbacks": 0} if impl else {"tc": 0}
    r, _, _ = plain_case(report, f"kernel_gemm_{['simt', 'tc'][impl]}_{M}x{N}x{K}", M, N, K, impl, seed=M + N + K,
                           expect=expect)
    assert r <= R


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 2, 3, 4])
def test_gemm_every_split_factor(report, splits):
    """EPI_PLAIN + bias + in-place residual at the cheapest shape whose plan on this GPU splits the k-range in
    `splits`; also the same call twice is bitwise equal (the partial tiles are summed in a fixed order)."""
    sms = sms_of_device()
    M, N, K = find_shape(sms, lambda p: p["tc"] and p["splits"] == splits)
    key = f"kernel_gemm_tc_split{splits}_{M}x{N}x{K}"
    r, path, y = plain_case(report, key, M, N, K, seed=splits, expect={"tc": 1, "splits": splits})
    _, _, y2 = plain_case({}, key, M, N, K, seed=splits)
    assert np.array_equal(y, y2)
    assert r <= R


@pytest.mark.gpu
@pytest.mark.parametrize("split", [False, True], ids=["nosplit", "split"])
def test_gemm_cta_with_several_items(report, split):
    """Persistent CTAs taking >= 2 (tile, split) items, so the TMA ring's stage counter carries across items: more
    tiles than SMs without split; with split, tiles * splits between the SM count and its 1.1-wave limit."""
    sms = sms_of_device()
    if split:
        M, N, K = find_shape(sms, lambda p: p["tc"] and p["splits"] > 1 and p["items_per_cta"] >= 2,
                             Ms=(256, 384, 512, 640, 768, 896, 1024), Ns=(384, 512, 640, 768, 896, 1024, 1152, 1280))
    else:
        M, N, K = 1025, 3584, 192
    key = f"kernel_gemm_tc_items_{'split' if split else 'nosplit'}"
    r, path, _ = plain_case(report, key, M, N, K, seed=7, expect={"tc": 1, "items_per_cta": lambda v: v >= 2,
                                                                    "splits": (lambda v: v > 1) if split else 1})
    assert r <= R


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["tc", "simt"])
def test_gemm_swiglu_and_gelu_planes(report, impl):
    """SwiGLU (interleaved gate / up rows) to fp32 and to split3 planes, and bias + GELU to planes (encoder fc1)."""
    for M, N, K in ((129, 1024, 896),):
        for planes_out in (False, True):
            key = f"kernel_gemm_{['simt', 'tc'][impl]}_swiglu_{M}x{N}x{K}_{'planes' if planes_out else 'f32'}"
            r, _, _ = plain_case(report, key, M, N, K, impl, seed=M, epi="swiglu", planes_out=planes_out,
                                   expect={"tc": impl, "splits": 1})
            assert r <= R
    key = f"kernel_gemm_{['simt', 'tc'][impl]}_gelu_planes_1025x3584x896"
    r, _, _ = plain_case(report, key, 1025, 3584, 896, impl, seed=3, gelu=True, residual=False, planes_out=True,
                           expect={"tc": impl})
    assert r <= R


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["0p6b_conv_out", "small_split"])
@pytest.mark.parametrize("impl", [1, 0], ids=["tc", "simt"])
def test_gemm_convout(report, impl, which):
    """conv_out: + bias + positional row (m % tokens per chunk), valid rows gathered through row_map (tail chunks keep
    fewer tokens).  The 0.6B shape (d_model 896, K = 480 x 16 = 7680) at 55 chunks splits in 3 on an H100 SXM; a small
    shape splits in 2.  The tensor-core path is asserted to split (the row_map gather is in the split-K reduction)."""
    rng = np.random.default_rng(5)
    tpc = 13
    if which == "0p6b_conv_out":
        chunks, N, K = 55, 896, 7680
    else:
        chunks, N, K = 10, 256, 768
    M = chunks * tpc
    valid = [tpc] * chunks
    valid[-1], valid[chunks // 2] = 4, 1
    row_map = np.full(M, -1, np.int32)
    tok = 0
    for c, n in enumerate(valid):
        row_map[c * tpc:c * tpc + n] = np.arange(tok, tok + n)
        tok += n
    x = rng.standard_normal((M, K)).astype(np.float32)
    wbits, w = bf16_weights(rng, N, K)
    bias = (0.1 * rng.standard_normal(N)).astype(np.float32)
    pos = rng.standard_normal((tpc, N)).astype(np.float32)
    out, _, path = run_gemm(x, wbits, N, K, impl, "convout", bias=bias, row_map=row_map, pos=pos, out_rows=tok, ldo=N)
    if impl:
        assert path["tc"] == 1 and path["splits"] == plan_py(M, N, K, epi="convout", sms=sms_of_device())["splits"]
        assert path["splits"] > 1 or which == "0p6b_conv_out", path
    sel = row_map >= 0
    ref = {}
    for dt in (torch.float32, torch.float64):
        y = gemm_ref(x, w, dt, bias)
        ref[dt] = (torch.from_numpy(y) + torch.from_numpy(pos).to(dt)[torch.arange(M) % tpc]).numpy()[sel]
    assert np.array_equal(np.argsort(row_map[sel]), np.arange(tok))
    key = f"kernel_gemm_{['simt', 'tc'][impl]}_convout_{which}"
    check_path(report, key, Err(True).add(out, ref[torch.float32], ref[torch.float64]),
               dict(path, M=M, N=N, K=K, chunks=chunks))


CONV_GEOMS = {   # n_window 50 (default) and 40: conv2 / conv3 output extents (OH, OW) and the next conv's halves
    "default_conv2": dict(OH=32, OW=25, Hh=32, Wh=25, Hh2=16, Wh2=13, in_hw=(64, 50), epi="conv_parity"),
    "default_conv3": dict(OH=16, OW=13, Hh=16, Wh=13, in_hw=(32, 25), epi="conv_feat"),
    "window40_conv2": dict(OH=32, OW=20, Hh=32, Wh=20, Hh2=16, Wh2=10, in_hw=(64, 40), epi="conv_parity"),
    "window40_conv3": dict(OH=16, OW=10, Hh=16, Wh=10, in_hw=(32, 20), epi="conv_feat"),
}


def conv_image(rng, chunks, g, dsh, cpad):
    """[chunks][2 Hh][2 Wh][cpad] channels-last input: the real channels (< dsh) over the image's real extent (the
    previous conv's output, e.g. 32 x 25 before conv3, in a 32 x 26 parity buffer) are post-GELU values; the rest is
    zero, as the session's parity buffers hold it."""
    x = np.zeros((chunks, 2 * g["Hh"], 2 * g["Wh"], cpad), np.float32)
    H, W = g["in_hw"]
    x[:, :H, :W, :dsh] = torch.nn.functional.gelu(torch.from_numpy(rng.standard_normal((chunks, H, W, dsh)))).numpy()
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["tc", "simt"])
@pytest.mark.parametrize("geom", list(CONV_GEOMS))
def test_gemm_conv(report, impl, geom):
    """Implicit 3x3 / stride 2 / pad 1 conv GEMM + bias + GELU at the conv2 / conv3 geometries of the default and
    window40 dims: a TMA box of box_h < OH output rows (the last box partial), the top / left padding taps (TMA
    zero fill), the right / bottom ones (zeros in the buffer), padding channels (dsh 120 of cpad 128), written to the
    next conv's parity layout (conv2) or the transposed conv_out feature rows (conv3)."""
    g = CONV_GEOMS[geom]
    rng = np.random.default_rng(len(geom))
    chunks, dsh, cpad = 3, 120, 128
    K = 9 * cpad
    x = conv_image(rng, chunks, g, dsh, cpad)
    wconv = np.zeros((dsh, 3, 3, cpad), np.float32)
    wconv[..., :dsh] = rng.standard_normal((dsh, 3, 3, dsh)) / math.sqrt(9 * dsh)
    wbits = bf16_rne(wconv.reshape(dsh, K))
    w = bf16_to_f32(wbits)
    bias = (0.1 * rng.standard_normal(dsh)).astype(np.float32)
    M = chunks * g["OH"] * g["OW"]
    conv = dict(M=M, OH=g["OH"], OW=g["OW"], Hh=g["Hh"], Wh=g["Wh"], cpad=cpad)
    ref = {}
    for dt in (torch.float32, torch.float64):
        xt = torch.from_numpy(x).to(dt).permute(0, 3, 1, 2)
        wt = torch.from_numpy(w.reshape(dsh, 3, 3, cpad)).to(dt).permute(0, 3, 1, 2)
        y = torch.nn.functional.conv2d(xt, wt, torch.from_numpy(bias).to(dt), stride=2, padding=1)
        ref[dt] = torch.nn.functional.gelu(y[:, :, :g["OH"], :g["OW"]]).permute(0, 2, 3, 1).numpy()   # [c][oh][ow][n]
    if g["epi"] == "conv_parity":
        Hh2, Wh2 = g["Hh2"], g["Wh2"]
        conv.update(Hh2=Hh2, Wh2=Wh2, cpad2=cpad)
        elems = chunks * 4 * Hh2 * Wh2 * cpad
        _, planes, path = run_gemm(x, wbits, dsh, K, impl, "conv_parity", bias=bias, conv=conv, planes_elems=elems)
        y = planes_value(planes).reshape(chunks, 2, 2, Hh2, Wh2, cpad)
        oh, ow = np.arange(g["OH"]), np.arange(g["OW"])
        got = y[:, oh[:, None] & 1, ow[None, :] & 1, oh[:, None] >> 1, ow[None, :] >> 1, :]   # [c][oh][ow][cpad]
        assert not got[..., dsh:].any()                     # padding channels untouched
        mask = np.ones(y.shape, bool)
        mask[:, oh[:, None] & 1, ow[None, :] & 1, oh[:, None] >> 1, ow[None, :] >> 1, :] = False
        assert not y[mask].any()                            # the parity layout's padding slots untouched
        got = got[..., :dsh]
    else:
        feat = dsh * g["OH"]
        _, planes, path = run_gemm(x, wbits, dsh, K, impl, "conv_feat", bias=bias, conv=conv,
                                   planes_elems=chunks * g["OW"] * feat, lds=feat)
        y = planes_value(planes).reshape(chunks, g["OW"], g["OH"], dsh)       # [c][ow][oh * N + n]
        got = y.transpose(0, 2, 1, 3)
    if impl:
        want = plan_py(M, dsh, K, 1, g["epi"], sms_of_device(), OH=g["OH"], OW=g["OW"], cpad=cpad)
        assert path["tc"] == 1 and path["box_h"] == want["box_h"] and path["tiles_m"] == want["tiles_m"], path
        assert path["box_h"] < g["OH"]
    check_path(report, f"kernel_gemm_{['simt', 'tc'][impl]}_{geom}",
               Err(True).add(got, ref[torch.float32], ref[torch.float64]), dict(path, M=M, N=dsh, K=K))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["n_not_multiple_of_8", "k_not_multiple_of_64"])
def test_gemm_fallbacks(report, case):
    """A tensor-core request the wgmma kernel cannot take runs the SIMT GEMM, moves the fall-back counter, and still
    meets the rule."""
    M, N, K = (129, 1001, 768) if case == "n_not_multiple_of_8" else (129, 1000, 200)
    r, path, _ = plain_case(report, f"kernel_gemm_fallback_{case}", M, N, K, impl=1, seed=9,
                              expect={"tc": 0, "simt_fallbacks": 1})
    assert r <= R


@pytest.mark.gpu
@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("impl", [1, 0], ids=["tc", "simt"])
def test_gemm_negative_control_two_planes(report, impl, K):
    """nplanes = 2 (the lo plane dropped) must FAIL the rule at small K.  At large K the fp32 reference's own
    accumulation error grows past the ~2^-17 relative loss of one plane, so the control stays at small K."""
    key = f"kernel_gemm_{['simt', 'tc'][impl]}_planes2_K{K}"
    r, _, _ = plain_case(report, key, 256, 256, K, impl, seed=K, residual=False, nplanes=2, expect={"tc": impl})
    assert r > R


@pytest.mark.gpu
@pytest.mark.parametrize("K", [768, 3072, 7680])
def test_gemm_same_sign_operands(report, K):
    """Post-GELU activations (almost all >= 0) against positive weights: every product has one sign, so a biased
    accumulator would show here first.  The wgmma kernel accumulates 4 k-blocks (K = 256) at a time inside the tensor
    core and adds each chunk into fp32 registers with round-to-nearest (gemm_tc.cu), so the bias is confined to sums
    of 256 products."""
    rng = np.random.default_rng(K)
    M, N = 256, 512
    x = torch.nn.functional.gelu(torch.from_numpy(rng.standard_normal((M, K)).astype(np.float32))).numpy()
    wpair = bf16_weights(rng, N, K, positive=True)
    key = f"kernel_gemm_tc_same_sign_K{K}"
    r, _, _ = plain_case(report, key, M, N, K, 1, x=x, wpair=wpair, bias=False, residual=False, expect={"tc": 1})
    assert r <= R


def wgmma_emulation(x, w, p=26):
    """CPU model of the wgmma GEMM's accumulation (gemm_tc.cu, wgmma.cuh consume_k_blocks): per k-block of 64 the hi,
    mid and lo planes each issue 4 m64n128k16 steps into one accumulator; a step adds its 16 exact products to the
    accumulator by aligning all 17 terms to the largest exponent, truncating each below p bits, summing exactly and
    rounding the sum toward zero to fp32; every 4 k-blocks the accumulator is added into a second fp32 sum
    (round-to-nearest).  With p = 26 this model reproduces the H100's measured errors."""
    pl = split3_np(np.asarray(x, np.float32).ravel()).reshape(3, *x.shape)
    planes = [bf16_to_f32(pl[i]).astype(np.float64) for i in range(3)]
    M, K = x.shape
    wd = np.asarray(w, np.float64)
    acc, tot = np.zeros((M, wd.shape[0])), np.zeros((M, wd.shape[0]), np.float32)
    for kb in range(K // BK):
        if kb % 4 == 0:
            acc[:] = 0.0
        for a in planes:
            for k in range(BK // 16):
                sl = slice(kb * BK + 16 * k, kb * BK + 16 * k + 16)
                terms = np.concatenate([a[:, None, sl] * wd[None, :, sl], acc[:, :, None]], -1)
                mx = np.abs(terms).max(-1, keepdims=True)
                q = 2.0 ** (np.floor(np.log2(np.where(mx > 0, mx, 1.0))) - p + 1)
                v = np.trunc(terms / q).sum(-1) * q[..., 0]
                m, e = np.frexp(v)
                acc = np.trunc(m * 2.0 ** 24) * 2.0 ** (e - 24)
        if kb % 4 == 3 or kb == K // BK - 1:
            tot = tot + acc.astype(np.float32)
    return tot


def _swiglu(a, dt):
    t = torch.from_numpy(np.asarray(a)).to(dt)
    return (torch.nn.functional.silu(t[:, 0::2]) * t[:, 1::2]).numpy()


def _short_k_row(seed=1):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((1, 192)).astype(np.float32)
    wbits, w = bf16_weights(rng, 1024, 192)
    return x, wbits, w


def test_wgmma_emulation_of_the_short_k_row():
    """The tensor core's truncating accumulation alone puts one SwiGLU row at K = 192 far over R (about 14 x: the fp32
    reference's error there is at the rounding floor, while each of the 36 k16 steps truncates against the running
    sum), and a 129-row SwiGLU at K = 896 under it."""
    x, _, w = _short_k_row()
    y = _swiglu(wgmma_emulation(x, w), torch.float32)
    r = ratio({}, "emulation", Err(True).add(y, _swiglu(gemm_ref(x, w, torch.float32), torch.float32),
                                             _swiglu(gemm_ref(x, w, torch.float64), torch.float64)))
    assert r > 3 * R, r


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["tc", "simt"])
def test_gemm_short_k_single_row_swiglu(report, impl):
    """One SwiGLU row at K = 192.  The SIMT GEMM meets R.  The wgmma GEMM does NOT: on an H100 it measured 14 x the
    fp32 error, and the CPU model of its accumulation (wgmma_emulation, p = 26) gives the same 14 x.  So the excess is
    the tensor core's round-toward-zero accumulation inside each k16 step, not a defect of this kernel's indexing or
    epilogue.  For this case alone the wgmma GEMM is held to the model instead of R: its output must agree with the
    emulation to within a tenth of its own error against float64."""
    x, wbits, w = _short_k_row()
    out, _, path = run_gemm(x, wbits, 1024, 192, impl, "swiglu", out_rows=1, ldo=512)
    assert path["tc"] == impl and path["simt_fallbacks"] == 0
    y64, y32 = _swiglu(gemm_ref(x, w, torch.float64), torch.float64), _swiglu(gemm_ref(x, w, torch.float32), torch.float32)
    key = f"kernel_gemm_{['simt', 'tc'][impl]}_swiglu_1x1024x192"
    r = record(report, key, Err(True).add(out, y32, y64), dict(path, M=1, N=1024, K=192, epi="swiglu"))
    if not impl:
        assert r <= R
        return
    emu = _swiglu(wgmma_emulation(x, w), torch.float32)
    d_model, d_64 = float(np.abs(out - emu).max()), float(np.abs(out - y64).max())
    report[f"fp64_{key}"].update(emulation_ratio=ratio({}, "emu", Err(True).add(emu, y32, y64)),
                                 max_abs_diff_to_emulation=d_model)
    assert d_model <= 0.1 * d_64, (d_model, d_64)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: attention
# ---------------------------------------------------------------------------------------------------------------------
def run_prefill_attn(segs, H, G, hd, rng, pos0=None, q_scale=1.0, k_const=False):
    """Causal prefill layout: queries packed by segment [rows][H * hd]; K / V in cache slots [seg][G][max_ctx][hd]
    (slot positions past each segment's keys hold random values that must stay masked).  Returns (got, [(q, k, v)])."""
    lens = np.array(segs, np.int32)
    p0 = np.zeros(len(segs), np.int32) if pos0 is None else np.array(pos0, np.int32)
    max_ctx = int((lens + p0).max()) + 40
    rows = int(lens.sum())
    q = (q_scale * rng.standard_normal((rows, H, hd))).astype(np.float32)
    kc = rng.standard_normal((len(segs), G, max_ctx, hd)).astype(np.float32)
    if k_const:
        kc[:] = kc[:, :, :1, :]
    vc = rng.standard_normal((len(segs), G, max_ctx, hd)).astype(np.float32)
    buf = np.concatenate([q.ravel(), kc.ravel(), vc.ravel()])
    q0 = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
    a = AttnArgs()
    a.hd, a.nseg, a.nheads, a.group, a.causal, a.keys_in_rows, a.max_len = hd, len(segs), H, H // G, 1, 0, int(lens.max())
    a.seg_q0, a.seg_len, a.seg_pos0 = ptr(q0), ptr(lens), ptr(p0) if pos0 is not None else None
    a.buf, a.buf_elems, a.q_off, a.k_off, a.v_off = ptr(buf), buf.size, 0, q.size, q.size + kc.size
    a.ldq, a.ldk, a.seg_stride, a.head_stride = H * hd, hd, G * max_ctx * hd, max_ctx * hd
    out = np.zeros((3, rows * H * hd), np.uint16)
    a.out_planes, a.out_rows, a.ldo = ptr(out), rows, H * hd
    _ok(probe().asrbt_attention(C.byref(a)))
    got = planes_value(out).reshape(rows, H, hd)
    parts = [(q[q0[s]:q0[s] + lens[s]], kc[s].transpose(1, 0, 2), vc[s].transpose(1, 0, 2), int(p0[s]))
             for s in range(len(segs))]
    return got, q0, lens, parts


def attn_check(report, key, got, q0, lens, parts, causal, path):
    err = Err(True)
    for s, (q, k, v, p0) in enumerate(parts):
        y64, y32 = (attn_ref(q, k, v, dt, causal, pos0=p0) for dt in (torch.float64, torch.float32))
        err.add(got[q0[s]:q0[s] + lens[s]], y32, y64)
    check_path(report, key, err, path)


CAUSAL_LENS = [1, 31, 32, 33, 64, 65, 97, 405, 1200]


@pytest.mark.gpu
@pytest.mark.parametrize("hd", [64, 128])
def test_attention_causal_lengths(report, hd):
    """One segment per launch at lengths around the 32-query tile and the 64-key tile: 1..38 query tiles, odd and even
    counts (CTA x runs tiles x and nqt-1-x)."""
    for L in CAUSAL_LENS:
        rng = np.random.default_rng(L)
        got, q0, lens, parts = run_prefill_attn([L], 8, 4, hd, rng)
        nqt = -(-L // 32)
        attn_check(report, f"kernel_attn_causal_hd{hd}_L{L}", got, q0, lens, parts, True,
                   {"kernel": "attn_f32", "query_tiles": nqt, "ctas_x": (nqt + 1) // 2, "odd_tiles": nqt % 2 == 1})


@pytest.mark.gpu
@pytest.mark.parametrize("pos0", [1, 63, 64, 300])
def test_attention_query_offset(report, pos0):
    """seg_pos0 (shared-context followers, score candidates): query i at position pos0 + i, keys from slot position 0,
    offsets either side of the 64-key tile; two segments with different offsets in one launch."""
    rng = np.random.default_rng(pos0)
    got, q0, lens, parts = run_prefill_attn([33, 97], 8, 2, 128, rng, pos0=[pos0, pos0 // 2 + 5])
    attn_check(report, f"kernel_attn_pos0_{pos0}", got, q0, lens, parts, True, {"kernel": "attn_f32", "pos0": pos0})


@pytest.mark.gpu
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("group", [1, 2, 3, 8])
def test_attention_gqa_groups(report, group, hd):
    rng = np.random.default_rng(group * hd)
    G = 2
    got, q0, lens, parts = run_prefill_attn([70, 5], G * group, G, hd, rng)
    attn_check(report, f"kernel_attn_gqa{group}_hd{hd}", got, q0, lens, parts, True, {"kernel": "attn_f32", "group": group})


@pytest.mark.gpu
def test_attention_mixed_segments(report):
    """Short and long causal segments in one launch (grid sized by the longest; short segments' extra CTAs idle),
    with and without query offsets."""
    rng = np.random.default_rng(8)
    segs = [1, 700, 33, 2, 129, 64]
    got, q0, lens, parts = run_prefill_attn(segs, 16, 8, 128, rng)
    attn_check(report, "kernel_attn_mixed", got, q0, lens, parts, True, {"kernel": "attn_f32", "segs": segs})
    got, q0, lens, parts = run_prefill_attn(segs, 16, 8, 128, rng, pos0=[0, 7, 64, 500, 1, 31])
    attn_check(report, "kernel_attn_mixed_pos0", got, q0, lens, parts, True, {"kernel": "attn_f32", "segs": segs})


@pytest.mark.gpu
@pytest.mark.parametrize("hd", [64, 128])
def test_attention_encoder_windows(report, hd):
    """Encoder layout: one [T][3 d_model] qkv buffer, keys at the window's own rows, non-causal windows of 1..104
    rows in one launch."""
    rng = np.random.default_rng(hd)
    H = 896 // hd if hd == 64 else 7
    dm = H * hd
    wins = [104, 1, 13, 31, 32, 33, 63, 64, 65, 100, 2, 104]
    T = sum(wins)
    qkv = rng.standard_normal((T, 3 * dm)).astype(np.float32)
    q0 = np.concatenate([[0], np.cumsum(wins)[:-1]]).astype(np.int32)
    lens = np.array(wins, np.int32)
    a = AttnArgs()
    a.hd, a.nseg, a.nheads, a.group, a.causal, a.keys_in_rows, a.max_len = hd, len(wins), H, 1, 0, 1, max(wins)
    a.seg_q0, a.seg_len, a.seg_pos0 = ptr(q0), ptr(lens), None
    a.buf, a.buf_elems, a.q_off, a.k_off, a.v_off = ptr(qkv), qkv.size, 0, dm, 2 * dm
    a.ldq, a.ldk, a.seg_stride, a.head_stride = 3 * dm, 3 * dm, 0, hd
    out = np.zeros((3, T * dm), np.uint16)
    a.out_planes, a.out_rows, a.ldo = ptr(out), T, dm
    _ok(probe().asrbt_attention(C.byref(a)))
    got = planes_value(out).reshape(T, H, hd)
    r = qkv.reshape(T, 3, H, hd)
    parts = [(r[q0[s]:q0[s] + wins[s], 0], r[q0[s]:q0[s] + wins[s], 1], r[q0[s]:q0[s] + wins[s], 2], 0)
             for s in range(len(wins))]
    attn_check(report, f"kernel_attn_encoder_hd{hd}", got, q0, lens, parts, False, {"kernel": "attn_f32", "windows": wins})


@pytest.mark.gpu
def test_attention_score_extremes(report):
    """Near-one-hot scores (queries scaled so that the best key leads by tens of nats) and all-equal scores (every
    key identical: uniform weights, the output is the mean of V)."""
    rng = np.random.default_rng(12)
    got, q0, lens, parts = run_prefill_attn([97, 405], 4, 2, 128, rng, q_scale=12.0)
    attn_check(report, "kernel_attn_one_hot", got, q0, lens, parts, True, {"kernel": "attn_f32", "q_scale": 12.0})
    got, q0, lens, parts = run_prefill_attn([97, 405], 4, 2, 128, rng, k_const=True)
    attn_check(report, "kernel_attn_equal_scores", got, q0, lens, parts, True, {"kernel": "attn_f32", "k_const": True})
