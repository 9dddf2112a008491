"""The greedy fused step's lm_head from its int8 copy (DESIGN.md section 4.1, "lm_head from its int8 copy").

The default (greedy) instantiation of decode_step_kernel streams an int8 copy of the lm_head with one scale s_r and one
bound constant C_r per row (model.cu quantize_head_kernel), keeps the rows whose interval [a_r - B_r, a_r + B_r] reaches
the CTA's best lower bound, and recomputes those rows from bf16 with the arithmetic of the full read.  Its ids must be
those of the LOGPROB instantiation, which reads every bf16 row.

CPU: a numpy restatement of the quantization and of the bound holds the float64 logit and the fp32 logit in the
kernel's order (two FMA chains of K / 64 terms per lane, one add, a 5-level butterfly) for random rows, rows with an
outlier, rows with all-equal entries and an x with a wide dynamic range.

GPU (tiny, and the 0.6B and 1.7B widths cut to 2 layers, untied heads): the greedy ids equal the LOGPROB ids at every
step for a random head, a head whose rows all come in duplicates (exact ties, which must resolve to the lower id, inside
one CTA and across CTAs), and a near-flat head whose candidate lists overflow, so that the CTAs recompute their whole
slices.  The session counters show which of these ran.

The bound itself is held tight on the GPU by the "tight" head (TIGHT_K below): with the final norm weight one-hot at
element k the normed x is x_k e_k, and rows whose only quantization residual sits at k have |f_r - a_r| = |x_k| times
the residual, within a relative 5e-4 of B_r.  Two such rows are arranged so that the one with the smaller a_r has the
larger logit; a C_r short by more than about 12 % drops that row from the candidates, and the greedy ids then differ
from the LOGPROB ids.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth

U = 2.0 ** -24


def gamma(k):
    return k * U / (1 - k * U)


def quantize(w):
    """model.cu quantize_head_kernel: (q int8 [R, K], s fp32 [R], C fp32 [R], rounded up)."""
    w = np.asarray(w, np.float32)
    K = w.shape[1]
    n = K // 64 + 6
    s = (np.abs(w).max(1) / np.float32(127)).astype(np.float32)
    safe = np.where(s > 0, s, np.float32(1))
    q = np.where(s[:, None] > 0, np.clip(np.rint(w / safe[:, None]), -127, 127), 0).astype(np.int8)
    w64, s64, q64 = w.astype(np.float64), s.astype(np.float64), q.astype(np.float64)
    rho = np.linalg.norm(w64 - s64[:, None] * q64, axis=1)
    C = (rho + gamma(n) * np.linalg.norm(w64, axis=1) + gamma(n + 1) * s64 * np.linalg.norm(q64, axis=1)) * (1 + 1e-9)
    Cf = C.astype(np.float32)
    Cf = np.where(Cf.astype(np.float64) < C, np.nextafter(Cf, np.float32(np.inf)), Cf)
    return q, s, Cf


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def kernel_dot(w, x):
    """fp32 row sums in the order of row_dot4 / row_dot / row_dot4_q (decode_mega.cu): lane l, chunk c holds elements
    (c * 32 + l) * 8 + e; chain 0 takes e = 0, 2, 4, 6 and chain 1 e = 1, 3, 5, 7; then chain 0 + chain 1 and the
    butterfly over lanes ^16, ^8, ^4, ^2, ^1."""
    R, K = w.shape
    wr = np.asarray(w, np.float32).reshape(R, K // 256, 32, 8)
    xr = np.asarray(x, np.float32).reshape(K // 256, 32, 8)
    a0 = np.zeros((R, 32), np.float32)
    a1 = np.zeros((R, 32), np.float32)
    for c in range(K // 256):
        for e in (0, 2, 4, 6):
            a0 = _fma(wr[:, c, :, e], xr[c, :, e], a0)
            a1 = _fma(wr[:, c, :, e + 1], xr[c, :, e + 1], a1)
    s = (a0 + a1).astype(np.float32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = (s + s[:, lanes ^ o]).astype(np.float32)
    return s[:, 0]


def interval(q, s, C, x):
    """(a, B) as consume_head_q forms them: a = s * sum q x in the kernel order, B = |x| (1 + 2^-12) C + 2^-100."""
    g = kernel_dot(q.astype(np.float32), x)
    a = (g * s).astype(np.float32)
    nx = np.float32(np.sqrt(np.sum(np.asarray(x, np.float64) ** 2)) * (1 + 2 ** -12))
    B = nx.astype(np.float64) * C.astype(np.float64) + 2.0 ** -100
    return a.astype(np.float64), B


# the "tight" head: rows 0 (A) and 1 (B), and their negatives for x_k < 0 at rows 2 / 3.
# Each row holds 127 s_r at element TIGHT_J (which sets s_r to a power of two) and its value at TIGHT_K (a multiple of
# 2^-10, exact in bf16): A = 20.625 s_A with s_A = 2^-7 rounds up to q = 21, B = 10.375 s_B with s_B = 2^-6 rounds
# down to q = 10.  So f_B - f_A = 2^-10 x_k > 0, while a_A - a_B = 2^-7 x_k, and B is a candidate only if
# a_B + B_B >= a_A - B_A, that is only if C_A + C_B >= 7/8 of the residuals' sum (0.375 + 0.75) 2^-7.  They come
# first, in the first turn of CTA 0's first warp, so that T passes every other row's upper bound from there on.  Every
# other row holds a single value 0.01 N(0, 1) at TIGHT_K (no residual, |f| < 0.07 |x_k| against 0.16 |x_k|): its
# interval is a few ulps wide, so no CTA's list overflows.
TIGHT_K, TIGHT_J, TIGHT_ROW = 5, 200, 0
TIGHT_ROWS = ((2.0 ** -7, 20.625), (2.0 ** -6, 10.375))


def _tight(V, H):
    w = torch.zeros(V, H)
    w[:, TIGHT_K] = 0.01 * torch.randn(V, generator=torch.Generator().manual_seed(13))
    w[TIGHT_ROW: TIGHT_ROW + 4] = 0.0
    for i, (s, v) in enumerate(TIGHT_ROWS):
        w[TIGHT_ROW + i, TIGHT_J] = 127 * s
        w[TIGHT_ROW + i, TIGHT_K] = v * s
    w[TIGHT_ROW + 2: TIGHT_ROW + 4] = -w[TIGHT_ROW: TIGHT_ROW + 2]
    return w.to(torch.bfloat16)


def test_tight_rows_need_the_full_bound():
    """The tight rows under numpy's quantize: the full C keeps row B, the issue's C x 0.1 (and C x 0.85) drops it."""
    H = 256
    w = _tight(TIGHT_ROW + 4, H).float().numpy()[TIGHT_ROW:]
    x = np.zeros(H, np.float32)
    for xk in (1.7, -0.6):
        x[TIGHT_K] = xk
        q, s, C = quantize(w)
        f = kernel_dot(w, x)
        best = int(np.argmax(f))
        assert best == (1 if xk > 0 else 3)
        for scale, kept in ((1.0, True), (0.85, False), (0.1, False)):
            a, B = interval(q, s, (C * scale).astype(np.float32), x)
            assert np.all(np.abs(f - a) <= B) == kept
            assert ((a + B)[best] >= np.max(a - B)) == kept, (xk, scale)


def _bf16(a):
    return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16).float().numpy()


def _rows(kind, R, K, rng):
    if kind == "random":
        return _bf16(rng.standard_normal((R, K)) * 0.1)
    if kind == "outlier":
        w = rng.standard_normal((R, K)) * 0.02
        w[np.arange(R), rng.integers(0, K, R)] *= 200.0
        return _bf16(w)
    if kind == "equal":
        return _bf16(np.repeat(rng.uniform(-0.2, 0.2, (R, 1)), K, axis=1))
    raise ValueError(kind)


@pytest.mark.parametrize("K", [256, 1024, 2048])
@pytest.mark.parametrize("rows", ["random", "outlier", "equal"])
@pytest.mark.parametrize("xkind", ["normal", "wide"])
def test_bound_contains_fp64_and_kernel_logits(K, rows, xkind):
    rng = np.random.default_rng(K + len(rows) * 7 + len(xkind))
    w = _rows(rows, 64, K, rng)
    x = rng.standard_normal(K)
    if xkind == "wide":                                     # entries from 1e-6 to 1e3
        x = x * 10.0 ** rng.uniform(-6, 3, K)
    x = x.astype(np.float32)
    q, s, C = quantize(w)
    a, B = interval(q, s, C, x)
    f64 = w.astype(np.float64) @ x.astype(np.float64)
    f32 = kernel_dot(w, x).astype(np.float64)
    assert np.all(np.abs(f64 - a) <= B), np.max(np.abs(f64 - a) / B)
    assert np.all(np.abs(f32 - a) <= B), np.max(np.abs(f32 - a) / B)
    if rows == "equal":                                     # no quantization residual: C is the rounding terms alone
        assert np.all(C < (2 * (K // 64 + 6) + 4) * U * np.linalg.norm(w.astype(np.float64), axis=1) + 1e-30)


def test_selection_rule_keeps_every_maximum():
    """The rule (T = max lower bound, candidates = upper bound >= T) keeps every row that attains the maximum,
    duplicated rows included, and the lower-id fold over them gives the full read's (value, id)."""
    rng = np.random.default_rng(3)
    K = 1024
    base = _bf16(rng.standard_normal((300, K)) * 0.1)
    w = np.concatenate([base, base[::-1], base])                 # every row three times, in two orders
    x = rng.standard_normal(K).astype(np.float32)
    q, s, C = quantize(w)
    a, B = interval(q, s, C, x)
    T = np.max(a - B)
    cand = np.nonzero(a + B >= T)[0]
    f = kernel_dot(w, x)
    best = np.flatnonzero(f == f.max())
    assert set(best) <= set(cand) and len(best) == 3
    fc = f[cand]
    assert cand[np.flatnonzero(fc == fc.max())].min() == best.min() == int(np.argmax(f))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the greedy (int8) instantiation against the LOGPROB one (full bf16 read)
# ---------------------------------------------------------------------------------------------------------------------
_WEIGHTS = {}


def _model(base):
    from qwen3_asr_rs_b200 import config_0p6b, config_1p7b, config_tiny
    ocfg, ecfg = {"0p6b": (O.cfg_0p6b, config_0p6b), "1p7b": (O.cfg_1p7b, config_1p7b),
                  "tiny": (O.cfg_tiny, config_tiny)}[base]
    ocfg, ecfg = ocfg(), ecfg()
    for cfg in (ocfg, ecfg):
        cfg.text.tie_word_embeddings = False
        if base != "tiny":
            cfg.text.num_hidden_layers = cfg.audio.encoder_layers = 2
    if base not in _WEIGHTS:
        _WEIGHTS.clear()
        _WEIGHTS[base] = synth.make_weights(ocfg, 5)
    return ecfg, _WEIGHTS[base]


def _head(kind, head):
    V, H = head.shape
    g = torch.Generator().manual_seed(11)
    if kind == "random":
        return head
    if kind == "ties":                  # rows 2k + 1 = rows 2k, and the second half repeats the first
        half = head[: V // 2].clone()
        half[1::2] = half[0::2]
        return torch.cat([half, half])
    if kind == "tight":
        return _tight(V, H)
    if kind == "flat":                  # one row plus a perturbation far inside every row's bound: every list overflows
        w0 = head[:1].float()
        e = torch.randn(V, H, generator=g) * 1e-4 * w0.abs().max()
        return (w0 + e).to(torch.bfloat16)
    raise ValueError(kind)


def _hq(st):
    return np.array([st.get(k, 0) for k in ("lmhead_rows_recomputed", "lmhead_full_fallbacks", "decode_fused_steps")])


@pytest.mark.gpu
@pytest.mark.parametrize("base", ["tiny", "0p6b", "1p7b"])
@pytest.mark.parametrize("kind", ["random", "ties", "flat", "tight"])
def test_greedy_int8_head_selects_full_read_ids(base, kind):
    from qwen3_asr_rs_b200 import AsrInference
    ecfg, w = _model(base)
    w = dict(w)
    w["thinker.lm_head.weight"] = _head(kind, w["thinker.lm_head.weight"])
    if kind == "tight":                 # x = x_k e_k after the final norm
        nw = torch.zeros_like(w["thinker.model.norm.weight"])
        nw[TIGHT_K] = 1.0
        w["thinker.model.norm.weight"] = nw
    clip = synth.make_clip(1, 4.0)
    n_new = 24
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        s0 = _hq(eng.stats())
        got = eng.transcribe_ids([clip], max_new_tokens=n_new)
        s1 = _hq(eng.stats())
        ref = eng.transcribe_ids([clip], max_new_tokens=n_new, logprobs=True)
        s2 = _hq(eng.stats())
    finally:
        eng.close()
    assert got.ids[0] == ref.ids[0], (base, kind, got.ids[0], ref.ids[0])
    steps = s1[2] - s0[2]
    assert steps >= len(got.ids[0]) - 1 >= 1                 # every step after the prefill's token ran on the fused kernel
    recomputed, fallbacks = s1[0] - s0[0], s1[1] - s0[1]
    assert np.all(s2[:2] == s1[:2])                          # the LOGPROB instantiation reads every bf16 row
    assert recomputed >= steps                               # each step recomputes at least the selected row
    if kind == "ties":
        V = w["thinker.lm_head.weight"].shape[0]
        assert all(t % 2 == 0 and t < V // 2 for t in got.ids[0]), got.ids[0]
        assert len(got.ids[0]) == n_new
    if kind == "tight":                 # row B (or its negative) every step: the bound kept it
        assert set(got.ids[0]) <= {TIGHT_ROW + 1, TIGHT_ROW + 3} and len(got.ids[0]) == n_new, got.ids[0]
    if kind == "flat":
        assert fallbacks >= steps                            # at least one CTA per step recomputed its whole slice
    else:
        assert fallbacks == 0
