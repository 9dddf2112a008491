"""Word timestamps (asrb_align_ids, DESIGN.md 4.10): a numpy statement of the alignment spec in include/asr_b200.h,
checked on the CPU against scipy and brute force; on the GPU, the head-mean matrix M against the spec applied to the
float64 oracle's teacher-forced attention under DESIGN.md section 2's rule (test_precision_fp64.py), two negative
controls that must fail it, the DTW bit for bit against numpy float32, the asrbt_dtw probe, the call's state rules and
refusals, and the end-to-end word times.  CPU tests also cover the frame mapping, word splitting and the CLI flag."""
import contextlib
import ctypes as C
import gc
import math

import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth
from qwen3_asr_rs_b200.inference import Alignment, check_align_ids, check_alignment_heads, text_start
from qwen3_asr_rs_b200.text import build_words, merge_punctuation, split_words
from test_precision_fp64 import R, Err, context_prompt, options, ratio

EOS = 151645
ASRB_ERR_INVALID, ASRB_ERR_STATE = 1, 4


# ---------------------------------------------------------------------------------------------------------------------
# the spec in numpy (any float dtype)
# ---------------------------------------------------------------------------------------------------------------------
def median7(z):
    """Width-7 median along the last axis with mirror padding (x[-1] = x[1]); the identity when T <= 3."""
    if z.shape[-1] <= 3:
        return z.copy()
    p = np.pad(z, ((0, 0), (3, 3)), mode="reflect")
    return np.median(np.lib.stride_tricks.sliding_window_view(p, 7, axis=1), axis=-1).astype(z.dtype)


def zscore(P):
    mean = P.mean(0)
    sd = P.std(0)
    return np.where(sd > 0, (P - mean) / np.where(sd > 0, sd, 1), 0).astype(P.dtype)


def head_mean(planes):
    """M from the per-head probability planes [N][T], in list order."""
    acc = np.zeros_like(planes[0])
    for P in planes:
        acc = acc + median7(zscore(P))
    return acc / acc.dtype.type(len(planes))


def dtw_f32(M):
    """DTW on X = -M in float32 (Whisper's dtw_cpu, ties included) -> start column of every row."""
    X = -np.asarray(M, np.float32)
    N, T = X.shape
    cost = np.full((N + 1, T + 1), np.inf, np.float32)
    trace = np.full((N + 1, T + 1), -1, np.int8)
    cost[0, 0] = 0
    for j in range(1, T + 1):
        for i in range(1, N + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c1 < c0 and c1 < c2:
                c, t = c1, 1
            else:
                c, t = c2, 2
            cost[i, j] = X[i - 1, j - 1] + c
            trace[i, j] = t
    start = [-1] * N
    i, j = N, T
    while i > 0 and j > 0:
        start[i - 1] = j - 1
        t = trace[i, j]
        if t == 0:
            i, j = i - 1, j - 1
        elif t == 1:
            i -= 1
        else:
            j -= 1
    assert i == 0 and j == 0
    return start


def token_frames(F, n_window):
    """Start frame of every audio token: token t of chunk k at k * 2 * n_window + 8 t, the chunks' valid tokens as the
    encoder keeps them."""
    cf = 2 * n_window
    out = []
    for k in range(-(-F // cf)):
        fr = min(cf, F - k * cf)
        valid = O.feat_extract_output_length(fr)
        out += [k * cf + 8 * t for t in range(valid)]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_median_matches_scipy():
    from scipy.ndimage import median_filter
    rng = np.random.default_rng(0)
    for T in (4, 5, 7, 13, 40):
        z = rng.standard_normal((6, T))
        assert np.array_equal(median7(z), median_filter(z, size=(1, 7), mode="mirror"))
    for T in (1, 2, 3):
        z = rng.standard_normal((4, T))
        assert np.array_equal(median7(z), z)


def test_zscore_std_zero():
    P = np.array([[0.5, 0.1, 0.2], [0.5, 0.3, 0.2]], np.float32)
    z = zscore(P)
    assert np.all(np.isfinite(z)) and z[0, 0] == 0 and z[1, 0] == 0 and z[0, 2] == 0
    assert abs(z[0, 1] + 1) < 1e-6 and abs(z[1, 1] - 1) < 1e-6


def _paths(N, T):
    """Every monotone path from (0, 0) to (N, T) with diagonal / up / left steps, as the cells it enters."""
    def walk(i, j):
        if (i, j) == (N, T):
            yield []
            return
        for di, dj in ((1, 1), (1, 0), (0, 1)):
            a, b = i + di, j + dj
            if a <= N and b <= T and a >= 1 and b >= 1:
                for rest in walk(a, b):
                    yield [(a, b)] + rest
    return list(walk(0, 0))


def test_dtw_optimal_against_brute_force():
    rng = np.random.default_rng(1)
    for N, T in ((1, 1), (2, 3), (3, 2), (3, 4), (4, 4), (2, 6)):
        for _ in range(5):
            M = rng.standard_normal((N, T)).astype(np.float32)
            X = -M.astype(np.float64)
            best = min(sum(X[a - 1, b - 1] for a, b in p) for p in _paths(N, T))
            start = dtw_f32(M)
            # the DTW path's cost, rebuilt from the start columns (the path walks each row from its start to the next
            # row's start, diagonally between rows when the start moves)
            cells = []
            for p in _paths(N, T):
                rows = {}
                for a, b in p:
                    rows.setdefault(a - 1, b - 1)
                if [rows[r] for r in range(N)] == start:
                    cells.append(sum(X[a - 1, b - 1] for a, b in p))
            assert cells and min(cells) <= best + 1e-5, (N, T, start, best, cells)
            assert start[0] == 0 and all(start[r] <= start[r + 1] for r in range(N - 1))


def test_dtw_tie_rule_hand_cases():
    # constant matrix: every interior step ties and the rule takes left, so the path runs left along the last row and
    # enters column 1 (where up beats the +inf border) -- every row starts at column 0, whatever N > T, T > N, N or T = 1
    for shape in ((3, 3), (1, 5), (4, 1), (4, 2), (2, 5), (5, 2)):
        assert dtw_f32(np.zeros(shape, np.float32)) == [0] * shape[0], shape
    # planted diagonal blocks: row i is strong on columns 3i .. 3i + 2, every other cell costs
    M = -np.ones((3, 9), np.float32)
    for i in range(3):
        M[i, 3 * i:3 * i + 3] = 1
    assert dtw_f32(M) == [0, 3, 6]
    # zero off the blocks: entering row 1 at column 2 (up, a zero cell) ties with the diagonal into column 3
    M[M < 0] = 0
    assert dtw_f32(M) == [0, 2, 5]


def test_frame_mapping():
    # n_window 50: chunks of 100 frames, 13 tokens each; a tail chunk of 35 frames keeps 5 tokens
    f = token_frames(235, 50)
    assert f[:13] == [8 * t for t in range(13)] and f[13] == 100 and f[26] == 200
    assert len(f) == 13 + 13 + O.feat_extract_output_length(35) == 31
    # n_window 40: chunks of 80 frames, 10 tokens
    f = token_frames(170, 40)
    assert f[:10] == [8 * t for t in range(10)] and f[10] == 80 and f[20] == 160 and len(f) == 10 + 10 + 2


class StubTok:
    """Token id -> bytes, decoded as a byte-level BPE tokenizer decodes (an incomplete character decodes to U+FFFD)."""

    def __init__(self, table):
        self.table = table

    def decode(self, ids):
        raw = b"".join(self.table[i] for i in ids)
        return raw.decode("utf-8", errors="replace")


EN = StubTok({1: b" Hello", 2: b",", 3: b" wor", 4: b"ld", 5: b" \"", 6: b"yes", 7: b"\"", 8: b".", 9: b" (", 10: b"a", 11: b")"})
ZH = StubTok({1: "你".encode(), 2: "好".encode()[:2], 3: "好".encode()[2:], 4: "。".encode(), 5: "世界".encode()})


def test_word_splitting_spaces_and_punctuation():
    w = split_words(EN.decode, [1, 2, 3, 4, 5, 6, 7, 8], "English")
    assert [t for t, _ in w] == [" Hello,", " world", " \"yes\"."]
    assert [ix for _, ix in w] == [[0, 1], [2, 3], [4, 5, 6, 7]]
    w = split_words(EN.decode, [9, 10, 11], None)
    assert [t for t, _ in w] == [" (a)"]
    assert merge_punctuation([(" \"", [0]), ("x", [1])]) == [(" \"x", [0, 1])]


def test_word_splitting_no_space_language():
    w = split_words(ZH.decode, [1, 2, 3, 4, 5], "Chinese")
    assert [t for t, _ in w] == ["你", "好。", "世界"]
    assert [ix for _, ix in w] == [[0], [1, 2, 3], [4]]


def test_build_words_times_and_probability():
    starts = [0.0, 0.1, 0.3, 0.4, 0.6, 0.7, 0.8, 0.9]
    lp = [math.log(0.5), math.log(1.0), -1.0, -2.0, 0.0, 0.0, 0.0, 0.0]
    ws = build_words(EN.decode, [1, 2, 3, 4, 5, 6, 7, 8], starts, 1.5, lp, "English", offset_s=10.0)
    assert [(w.start_s, w.end_s) for w in ws] == [(10.0, 10.3), (10.3, 10.6), (10.6, 11.5)]
    assert abs(ws[0].probability - 0.75) < 1e-12
    assert abs(ws[1].probability - (math.exp(-1) + math.exp(-2)) / 2) < 1e-12


def test_host_checks():
    assert check_align_ids([[1, 2]], None, 1, 10) == ([[1, 2]], [0])
    for ids, tf, msg in (([[1]], [1], "text_from"), ([[]], None, "no ids"), ([[10]], None, "out of"), ([[1], [2]], None, "one id")):
        with pytest.raises(ValueError, match=msg):
            check_align_ids(ids, tf, 1, 10)
    assert check_alignment_heads(None, 3, 4) == []
    assert check_alignment_heads([(0, 1), (2, 3)], 3, 4) == [(0, 1), (2, 3)]
    for bad in ([], [(3, 0)], [(0, 4)], [(1, 1), (1, 1)]):
        with pytest.raises(ValueError):
            check_alignment_heads(bad, 3, 4)
    assert text_start([5, 7, 9, 1], 9) == 3 and text_start([5, 7], 9) == 0 and text_start([5], None) == 0
    a = Alignment(1, [0, 8], [8, 20])
    assert a.start_s == [0.0, 0.08] and a.end_s == [0.08, 0.2]


def test_cli_flag():
    from qwen3_asr_rs_b200.__main__ import USAGE, main, split_word_timestamps
    assert split_word_timestamps(["m", "a.wav"]) == (["m", "a.wav"], False)
    assert split_word_timestamps(["m", "--word-timestamps", "a.wav", "English"]) == (["m", "a.wav", "English"], True)
    assert "--word-timestamps" in USAGE
    for extra in (["--stream", "2"], ["--score", "hi"], ["--detect-language"]):
        assert main(["m", "a.wav", "--word-timestamps"] + extra) == 1


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def capture_rope():
    """Record the post-RoPE q and k of every decoder layer that oracle.score_ids runs (apply_rotary is called for q,
    then k, once per layer)."""
    orig, got = O.apply_rotary, []

    def rec(x, cos, sin):
        y = orig(x, cos, sin)
        got.append(y)
        return y
    O.apply_rotary = rec
    try:
        yield got
    finally:
        O.apply_rotary = orig


def oracle_planes(model, x, ids, f, heads, lang=None, ctx=None, rows_shift=0, all_keys=False):
    """Per listed head, P [N][T] in the model's dtype from its teacher-forced pass over prompt + ids.  rows_shift and
    all_keys are the negative controls: rows at the token's own position, softmax over every causal key."""
    t = model.cfg.text
    cm = context_prompt(ctx) if ctx else contextlib.nullcontext()
    with cm, capture_rope() as got:
        O.score_ids(model, x, ids, language_ids=lang)
        prompt, a0 = O.build_prompt(0, lang)
    qk = got[: 2 * t.num_hidden_layers]
    n = len(ids)
    S = qk[0].shape[2] - n                 # score_ids runs prompt + every id
    T = S - len(prompt)
    rows = [S - 1 + i + rows_shift for i in range(f, n)]
    group = t.num_attention_heads // t.num_key_value_heads
    out = []
    for l, h in heads:
        q, k = qk[2 * l][0, h], qk[2 * l + 1][0, h // group]
        s = (q[rows] @ k.transpose(0, 1)) / math.sqrt(t.head_dim)
        if all_keys:
            mask = torch.full_like(s, float("-inf"))
            for r, row in enumerate(rows):
                mask[r, : row + 1] = 0
            p = torch.softmax(s + mask, -1)[:, a0:a0 + T]
        else:
            p = torch.softmax(s[:, a0:a0 + T], -1)
        out.append(p.numpy())
    return out, T


def default_heads(t):
    return [(l, h) for l in range(t.num_hidden_layers // 2, t.num_hidden_layers) for h in range(t.num_attention_heads)]


def gpu_ids(e, clips, lang=None, n=12):
    with options(e, logprobs="0"):
        r = e.transcribe_ids(clips, language_ids=lang, max_new_tokens=n)
    return [ids + [EOS] for ids in r.ids]


def m_errs(e, m32, m64, clips, rows, tf, heads, lang=None, ctx=None, **ctl):
    """Err of M over the batch (relative), and the per-utterance (M_gpu, M_64)."""
    err, mats = Err(True), []
    e.align_ids(clips, rows, text_from=tf, language_ids=lang, context_ids=ctx,
                alignment_heads=None if heads is None else heads)
    hs = heads if heads is not None else default_heads(m32.cfg.text)
    for b, x in enumerate(clips):
        lb = None if lang is None else lang[b]
        cb = None if ctx is None else ctx[b]
        got = e.last_align_matrix(b)
        p32, _ = oracle_planes(m32, x, rows[b], tf[b], hs, lb, cb, **ctl)
        p64, _ = oracle_planes(m64, x, rows[b], tf[b], hs, lb, cb, **ctl)
        M32, M64 = head_mean([p.astype(np.float32) for p in p32]), head_mean([p.astype(np.float64) for p in p64])
        assert got.shape == M64.shape, (got.shape, M64.shape)
        err.add(got, M32, M64)
        mats.append((got, M64))
    return err, mats


@pytest.fixture(scope="module")
def eng(tiny):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    e = AsrInference.from_weights(config_tiny(), w, device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def tiny64(tiny):
    cfg, w, _ = tiny
    return O.OracleModel(cfg, w, dtype=torch.float64)


CLIPS = {"sub_chunk": (11, 0.7), "tail_chunk": (12, 2.35), "past_window": (13, 9.5)}


# ---------------------------------------------------------------------------------------------------------------------
# GPU: M under the float64 rule, negative controls, DTW exactness
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("clip", sorted(CLIPS))
def test_matrix_fp64_tiny(tiny, tiny64, eng, report, clip):
    _, _, m32 = tiny
    x = synth.make_clip(*CLIPS[clip])
    rows = gpu_ids(eng, [x])
    t = m32.cfg.text
    for name, heads in (("default", None), ("explicit", [(0, 1), (1, 3), (t.num_hidden_layers - 1, 0)])):
        err, mats = m_errs(eng, m32, tiny64, [x], rows, [0], heads)
        r = ratio(report, f"align_tiny_{clip}_{name}", err, min_values=1)
        assert r <= R, report[f"fp64_align_tiny_{clip}_{name}"]


@pytest.mark.gpu
def test_matrix_fp64_ragged_batch(tiny, tiny64, eng, report):
    _, _, m32 = tiny
    clips = [synth.make_clip(21, 1.6), synth.make_clip(22, 3.3), synth.make_clip(23, 0.9)]
    lang = [None, [11528, 6364, 151704], None]
    ctx = [None, None, [9707, 11, 1879, 13]]
    rows = []
    for b, x in enumerate(clips):
        with options(eng, logprobs="0"):
            r = eng.transcribe_ids([x], language_ids=None if lang[b] is None else [lang[b]], max_new_tokens=10,
                                   context_ids=None if ctx[b] is None else [ctx[b]])
        rows.append(r.ids[0] + [EOS])
    tf = [min(2, len(rows[0]) - 1), 0, min(1, len(rows[2]) - 1)]
    for name, heads in (("default", None), ("explicit", [(0, 0), (2, 3)])):
        err, _ = m_errs(eng, m32, tiny64, clips, rows, tf, heads, lang=lang, ctx=ctx)
        r = ratio(report, f"align_tiny_ragged_{name}", err, min_values=1)
        assert r <= R, report[f"fp64_align_tiny_ragged_{name}"]


@pytest.mark.gpu
def test_negative_controls(tiny, tiny64, eng, report):
    """Rows at the token's own position, and the softmax over all causal keys, must fail the rule."""
    _, _, m32 = tiny
    x = synth.make_clip(*CLIPS["tail_chunk"])
    rows = gpu_ids(eng, [x])
    eng.align_ids([x], rows)
    got = eng.last_align_matrix(0)
    hs = default_heads(m32.cfg.text)
    for name, ctl in (("rows_off_by_one", dict(rows_shift=1)), ("all_causal_keys", dict(all_keys=True))):
        p32, _ = oracle_planes(m32, x, rows[0], 0, hs, **ctl)
        p64, _ = oracle_planes(tiny64, x, rows[0], 0, hs, **ctl)
        M32 = head_mean([p.astype(np.float32) for p in p32])
        M64 = head_mean([p.astype(np.float64) for p in p64])
        err = Err(True).add(got, M32, M64)
        r = ratio(report, f"align_negative_{name}", err, min_values=1)
        assert r > R, report[f"fp64_align_negative_{name}"]


@pytest.mark.gpu
def test_dtw_exact_on_gpu_matrix(tiny, tiny64, eng, report):
    _, _, m32 = tiny
    clips = [synth.make_clip(*CLIPS[k]) for k in sorted(CLIPS)]
    rows = gpu_ids(eng, clips, n=16)
    al = eng.align_ids(clips, rows)
    agree = []
    for b, x in enumerate(clips):
        M = eng.last_align_matrix(b)
        F = -(-len(x) // 160)
        frames = token_frames(F, 50)
        assert M.shape == (len(rows[b]), len(frames))
        start = dtw_f32(M)
        assert [frames[j] for j in start] == al[b].start_frames
        assert al[b].end_frames == al[b].start_frames[1:] + [F]
        # against the DTW of M_64
        p64, _ = oracle_planes(tiny64, x, rows[b], 0, default_heads(m32.cfg.text))
        s64 = dtw_f32(head_mean([p.astype(np.float64) for p in p64]))
        agree.append(s64 == start)
    report["align_dtw_agrees_with_M64"] = agree


# ---------------------------------------------------------------------------------------------------------------------
# GPU: depth-cut model at the 0.6B widths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cut06():
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    cfg.text.num_hidden_layers, cfg.audio.encoder_layers = 4, 2
    w = synth.make_weights(cfg, 3)
    ecfg = config_0p6b()
    ecfg.text.num_hidden_layers, ecfg.audio.encoder_layers = 4, 2
    e = AsrInference.from_weights(ecfg, w, device=0)
    m32, m64 = O.OracleModel(cfg, w), O.OracleModel(cfg, w, dtype=torch.float64)
    del w
    yield m32, m64, e
    e.close()
    del m32, m64
    gc.collect()


@pytest.mark.gpu
def test_matrix_fp64_0p6b_widths(cut06, report):
    m32, m64, e = cut06
    x = synth.make_clip(31, 4.2)
    rows = gpu_ids(e, [x], n=20)
    for name, heads in (("default", None), ("explicit", [(0, 5), (3, 15)])):
        err, _ = m_errs(e, m32, m64, [x], rows, [0], heads)
        r = ratio(report, f"align_0p6b_cut_{name}", err, min_values=1)
        assert r <= R, report[f"fp64_align_0p6b_cut_{name}"]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the DTW probe
# ---------------------------------------------------------------------------------------------------------------------
def probe_dtw(M):
    from qwen3_asr_rs_b200 import _lib
    lib = _lib.load_library()
    fn = lib.asrbt_dtw
    fn.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.POINTER(C.c_int32)]
    fn.restype = C.c_int
    M = np.ascontiguousarray(M, np.float32)
    out = np.full(M.shape[0], -7, np.int32)
    _lib.check(fn(M.ctypes.data_as(C.POINTER(C.c_float)), M.shape[0], M.shape[1], out.ctypes.data_as(C.POINTER(C.c_int32))))
    return out.tolist()


@pytest.mark.gpu
def test_dtw_probe():
    rng = np.random.default_rng(5)
    planted = np.zeros((5, 20), np.float32)
    for i in range(5):
        planted[i, 4 * i:4 * i + 4] = 1
    cases = [planted, np.zeros((6, 6), np.float32), np.zeros((7, 3), np.float32), np.zeros((1, 9), np.float32),
             np.zeros((8, 1), np.float32), rng.standard_normal((37, 101)).astype(np.float32),
             rng.standard_normal((120, 390)).astype(np.float32),
             np.round(rng.standard_normal((30, 50)), 1).astype(np.float32)]      # many exact ties
    for M in cases:
        assert probe_dtw(M) == dtw_f32(M), M.shape
    big = rng.standard_normal((700, 1400)).astype(np.float32)   # 2-bit trace of 245 KB: past shared memory
    assert probe_dtw(big) == dtw_f32(big)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: calls and state
# ---------------------------------------------------------------------------------------------------------------------
def _raw_align(e, clips, rows, tf=None, heads=(), max_ids=None, n_ids=None):
    """asrb_align_ids straight through the C ABI -> status."""
    from qwen3_asr_rs_b200 import _lib
    B = len(clips)
    arrs, ptrs, lens = e._pack_samples(clips)
    ia = [np.ascontiguousarray(r, np.int64) for r in rows]
    ip = (C.POINTER(C.c_int64) * B)(*[a.ctypes.data_as(C.POINTER(C.c_int64)) for a in ia])
    nn = (C.c_int32 * B)(*(n_ids or [len(r) for r in rows]))
    tfa = (C.c_int32 * B)(*(tf or [0] * B))
    h = np.ascontiguousarray(np.array(heads, np.int32).reshape(-1, 2))
    m = max_ids or max(len(r) for r in rows)
    st, en = np.zeros((B, m), np.int32), np.zeros((B, m), np.int32)
    return e._lib.asrb_align_ids(e._session, ptrs, lens, B, None, None, ip, nn, tfa,
                                 h.ctypes.data_as(C.POINTER(C.c_int32)) if len(heads) else None, len(heads), m,
                                 st.ctypes.data_as(C.POINTER(C.c_int32)), en.ctypes.data_as(C.POINTER(C.c_int32)))


@pytest.mark.gpu
def test_calls_and_state(eng):
    from qwen3_asr_rs_b200 import _lib
    clips = [synth.make_clip(41, 2.2), synth.make_clip(42, 1.1)]
    rows = gpu_ids(eng, clips)
    a = eng.align_ids(clips, rows, text_from=[1, 0])
    Ms = [eng.last_align_matrix(b) for b in range(2)]
    b_ = eng.align_ids(clips, rows, text_from=[1, 0])
    assert a == b_ and all(np.array_equal(M, eng.last_align_matrix(i)) for i, M in enumerate(Ms))
    with options(eng, temperature="0.8", seed="9", no_repeat_ngram_size="2", repetition_penalty="1.3"):
        c = eng.align_ids(clips, rows, text_from=[1, 0])
        assert c == a and all(np.array_equal(M, eng.last_align_matrix(i)) for i, M in enumerate(Ms))
    # after an alignment call no run is pending (the options block above freed its session: align on a new one)
    assert eng.align_ids(clips, rows, text_from=[1, 0]) == a
    ids = np.zeros((2, 4), np.int32)
    n = np.zeros(2, np.int32)
    assert eng._lib.asrb_generate(eng._session, 4, ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                  n.ctypes.data_as(C.POINTER(C.c_int32))) == ASRB_ERR_STATE
    # refusals, each leaving the session usable
    V = eng.config.text.vocab_size
    L, H = eng.config.text.num_hidden_layers, eng.config.text.num_attention_heads
    bad = [dict(n_ids=[0, len(rows[1])]), dict(max_ids=len(rows[0]) - 1), dict(tf=[len(rows[0]), 0]),
           dict(tf=[-1, 0]), dict(heads=[(L, 0)]), dict(heads=[(0, H)]), dict(heads=[(1, 1), (1, 1)])]
    for kw in bad:
        assert _raw_align(eng, clips, rows, **kw) == ASRB_ERR_INVALID, kw
        assert eng.align_ids(clips, rows, text_from=[1, 0]) == a
    assert _raw_align(eng, clips, [rows[0], rows[1][:-1] + [V]]) == ASRB_ERR_INVALID
    assert _raw_align(eng, clips, [rows[0] * 40, rows[1]]) == ASRB_ERR_INVALID     # past the session's max_new_tokens
    assert eng.align_ids(clips, rows, text_from=[1, 0]) == a


@pytest.mark.gpu
def test_segments_view_equals_copy(eng):
    """asrb_align_segments on a view of the long-audio buffer is bitwise asrb_align_ids on the samples copied out."""
    x = np.concatenate([synth.make_clip(51, 3.0), synth.make_clip(52, 2.0)])
    lr = eng.transcribe_long([x], [16000], max_segment_s=5.0, search_s=2.0, batch=4, word_timestamps=True)
    cuts = eng.segment_long(80000, 32000)[0]
    a, b = cuts[0]
    ids = lr.files[0][0].ids + [EOS]
    s = eng._session
    fl, st, en = (C.c_int32 * 1)(0), (C.c_int64 * 1)(a), (C.c_int64 * 1)(b)
    view = eng._align(s, [ids], [0], [], None, lambda *q: eng._lib.asrb_align_segments(s, 1, fl, st, en, None, None, *q))[0]
    Mv = eng.last_align_matrix(0)
    copy = eng.align_ids([x[a:b]], [ids])[0]
    assert view == copy and np.array_equal(Mv, eng.last_align_matrix(0))
    w = lr.files[0][0].words
    assert [round(q.start_s - a / 16000, 6) for q in w] == [round(f * 0.01, 6) for f in
                                                           [copy.start_frames[k] for k in range(len(copy.start_frames))]][:len(w)] or w == []


@pytest.mark.gpu
def test_end_to_end_times(eng):
    x = synth.make_clip(61, 6.0)
    r = eng.transcribe_ids([x], max_new_tokens=24)
    al = eng.align_ids([x], [r.ids[0] + [EOS]])[0]
    F = -(-len(x) // 160)
    assert al.start_frames == sorted(al.start_frames) and al.end_frames[-1] == F
    assert all(0 <= s <= e <= F for s, e in zip(al.start_frames, al.end_frames))
    ws = eng._words(r.ids[0], al, None, None)
    assert [w.start_s for w in ws] == sorted(w.start_s for w in ws)
    # long form: monotone, inside the segment and the file
    y = np.concatenate([synth.make_clip(62, 4.0), synth.make_clip(63, 4.0), synth.make_clip(64, 3.0)])
    lr = eng.transcribe_long([y], [16000], max_segment_s=5.0, search_s=2.0, batch=2, word_timestamps=True)
    dur = len(y) / 16000
    prev = 0.0
    for sg in lr.files[0]:
        assert sg.words is not None
        for w in sg.words:
            assert sg.start_s - 1e-9 <= w.start_s <= w.end_s <= sg.start_s + math.ceil((sg.end_s - sg.start_s) * 100) / 100 + 1e-9
            assert w.start_s >= prev - 1e-9 and w.end_s <= dur + 0.01
            prev = w.start_s
