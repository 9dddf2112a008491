"""Long-form transcription: cut points on the GPU (asrb_segment_long), segment views decoded in place
(asrb_transcribe_segments), AsrInference.transcribe_long, the text join rule and the CLI flag.

`ref_energy` / `ref_segments` below are the cut rule in float64 numpy; the package has no host copy of it."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth

SR = 16000
MARGIN_FLOOR_REL = 4 * 1.5e-5      # as test_gpu_parity.py: exact ids are meaningful above this top-1/top-2 gap


# ---------------------------------------------------------------------------------------------------------------------
# the reference rule
# ---------------------------------------------------------------------------------------------------------------------
def ref_energy(x):
    """e[j] = sum x[i]^2, i in [160 j, 160 j + 1600), in float64, for every window inside the signal."""
    x = np.asarray(x, dtype=np.float64)
    nb = len(x) // 160
    if nb < 10:
        return np.zeros(0)
    blk = (x[: nb * 160].reshape(nb, 160) ** 2).sum(1)
    return np.lib.stride_tricks.sliding_window_view(blk, 10).sum(1)


def ref_candidates(e, N, c, max_seg, search):
    """Window indices j whose centre 160 j + 800 may follow cut c."""
    lo, hi = c + max_seg - search, min(c + max_seg, N - SR)
    return np.arange((lo - 800) // 160, (hi - 800) // 160 + 1)


def ref_segments(x, max_seg, search, e=None):
    N = len(x)
    e = ref_energy(x) if e is None else e
    cuts, c = [0], 0
    while N - c > max_seg:
        j = ref_candidates(e, N, c, max_seg, search)
        v = e[j]
        c = 160 * int(j[np.flatnonzero(v == v.min())[-1]]) + 800
        cuts.append(c)
    return list(zip(cuts, cuts[1:] + [N]))


def gap_file(index, pieces, gap_s=0.6, sr=SR, gap_amp=1e-4):
    """make_clip pieces of the given lengths separated by near-silent gaps; returns (signal, gap centres in samples)."""
    rng = np.random.default_rng(9000 + index)
    parts, centres, pos = [], [], 0
    for i, s in enumerate(pieces):
        if i:
            g = int(gap_s * sr)
            parts.append((rng.standard_normal(g) * gap_amp).astype(np.float32))
            centres.append(pos + g // 2)
            pos += g
        clip = synth.make_clip(index * 100 + i, s, sr)
        parts.append(clip)
        pos += len(clip)
    return np.concatenate(parts), centres


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_reference_rule_cuts_in_quiet_gaps():
    x, centres = gap_file(1, [9.0, 7.5, 9.3, 8.0, 6.0])
    segs = ref_segments(x, 10 * SR, 5 * SR)
    assert len(segs) == 5
    for (a, b), c in zip(segs[1:], centres):
        assert abs(a - c) <= 0.25 * SR, (a, c)           # the 100 ms window sits inside the 0.6 s gap
    assert segs[0][0] == 0 and segs[-1][1] == len(x)
    assert all(b == a2 for (_, b), (a2, _) in zip(segs, segs[1:]))


@pytest.mark.parametrize("max_s,search_s", [(5, 2), (10, 5), (30, 5), (12.5, 6.25)])
def test_reference_rule_bounds(max_s, search_s):
    max_seg, search = int(max_s * SR), int(search_s * SR)
    rng = np.random.default_rng(int(max_s * 10))
    for n in (max_seg + 1, max_seg + SR, 3 * max_seg + 12345, 7 * max_seg - 77):
        x = rng.standard_normal(n).astype(np.float32)
        segs = ref_segments(x, max_seg, search)
        assert all(b - a <= max_seg for a, b in segs)
        assert segs[-1][1] - segs[-1][0] >= SR
        assert all(a % 160 == 0 for a, _ in segs)


def test_reference_rule_all_zero_gives_longest_pieces():
    max_seg, search = 10 * SR, 5 * SR
    x = np.zeros(47 * SR + 321, dtype=np.float32)
    segs = ref_segments(x, max_seg, search)
    assert [b - a for a, b in segs[:-1]] == [max_seg] * (len(segs) - 1)
    assert segs == [(0, 160000), (160000, 320000), (320000, 480000), (480000, 640000), (640000, len(x))]


def test_reference_rule_short_file_is_one_segment():
    for n in (201, SR, 10 * SR):
        x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
        assert ref_segments(x, 10 * SR, 5 * SR) == [(0, n)]


def test_check_segmenting():
    from qwen3_asr_rs_b200.inference import check_segmenting, default_search_s
    assert check_segmenting(30.0, 5.0) == (480000, 80000)
    assert check_segmenting(5, 2.5) == (80000, 40000)
    assert check_segmenting(7.77, 2.0) == (124320, 32000)
    for bad in ((4.99, 2.0), (10.0, 1.99), (10.0, 5.01), (30.005, 5.0), (30.0, 5.001), (float("nan"), 5.0),
                (True, 5.0), ("30", 5.0), (30.0, None)):
        with pytest.raises(ValueError):
            check_segmenting(*bad)
    assert default_search_s(30.0) == 5.0 and default_search_s(8.0) == 4.0 and default_search_s(8.01) == 4.0


def test_join_rule_and_majority_language():
    from qwen3_asr_rs_b200.text import join_segment_texts, majority_language
    assert join_segment_texts(["Hello there.", "", "General Kenobi."], "English") == "Hello there. General Kenobi."
    assert join_segment_texts(["你好", "", "世界"], "Chinese") == "你好世界"
    assert join_segment_texts(["こんにちは", "世界"], "japanese") == "こんにちは世界"
    assert join_segment_texts(["a", "b"], "Cantonese") == "ab"
    assert join_segment_texts(["a", "b"], None) == "a b"
    assert join_segment_texts(["", ""], "English") == ""
    assert majority_language(["English", "Chinese", "Chinese", "English"]) == "English"      # first on ties
    assert majority_language(["English", "Chinese", "Chinese"]) == "Chinese"
    assert majority_language([]) == "unknown"


def test_cli_max_segment_flag(capsys):
    from qwen3_asr_rs_b200.__main__ import USAGE, format_segment, main, split_max_segment
    assert split_max_segment(["m", "a.wav"]) == (["m", "a.wav"], None)
    assert split_max_segment(["--max-segment", "30", "m", "a.wav", "en"]) == (["m", "a.wav", "en"], 30.0)
    assert split_max_segment(["m", "--max-segment=12.5", "a.wav"]) == (["m", "a.wav"], 12.5)
    for bad in (["m", "a.wav", "--max-segment"], ["m", "a.wav", "--max-segment", "x"],
                ["m", "a.wav", "--max-segment", "4"], ["m", "a.wav", "--max-segment", "30.001"]):
        assert split_max_segment(bad) is None, bad
    assert "--max-segment S" in USAGE
    assert format_segment(0.0, 29.87, "hello") == "  [0.00 - 29.87] hello"
    assert main(["m", "a.wav", "--max-segment", "2"]) == 1
    assert "Usage" in capsys.readouterr().err


def test_transcribe_long_argument_validation_before_gpu_work():
    from qwen3_asr_rs_b200.inference import AsrInference
    eng = AsrInference.__new__(AsrInference)          # no library / GPU: every check runs before either is touched
    from qwen3_asr_rs_b200 import config_tiny
    eng.config = config_tiny()
    pcm = [np.zeros(SR, np.float32)]
    for kw in (dict(max_segment_s=4.0), dict(search_s=1.0), dict(batch=0), dict(batch=2, beam_size=3),
               dict(top_logprobs=9), dict(temperature=-1.0), dict(context_ids=[[1], [2]]), dict(language_ids=[[1], [2]])):
        with pytest.raises(ValueError):
            eng.transcribe_long(pcm, [SR], **kw)
    with pytest.raises(ValueError):
        eng.transcribe_long(pcm, [SR, SR])


def test_segment_symbols_null_session_is_a_status():
    from qwen3_asr_rs_b200 import _lib
    lib = _lib.load_library()
    n = (C.c_int32 * 1)()
    se, en = (C.c_int64 * 4)(), (C.c_int64 * 4)()
    assert lib.asrb_segment_long(None, 160000, 80000, 4, n, se, en) != 0
    assert lib.asrb_long_read(None, 0, (C.c_float * 1)()) != 0
    assert lib.asrb_transcribe_segments(None, 1, (C.c_int32 * 1)(), se, en, None, None, 8, (C.c_int32 * 8)(),
                                        (C.c_int32 * 1)()) != 0
    assert lib.asrb_ingest_long(None, None, None, None, None, None, 1, None) != 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _check_cuts(x, got, max_seg, search):
    """`got` segments follow the rule on x: each cut is a candidate after the previous one with the least energy, an
    equal-energy later one (to 1e-12 relative) being accepted in its place.  Returns the number of such ties."""
    N = len(x)
    e = ref_energy(x)
    ties, c = 0, 0
    assert got[0][0] == 0 and got[-1][1] == N
    assert all(b == a2 for (_, b), (a2, _) in zip(got, got[1:]))
    for a, b in got[1:]:
        assert N - c > max_seg
        j = ref_candidates(e, N, c, max_seg, search)
        v = e[j]
        ref = 160 * int(j[np.flatnonzero(v == v.min())[-1]]) + 800
        if a != ref:
            jj = (a - 800) // 160
            assert a % 160 == 0 and j[0] <= jj <= j[-1], (a, c)
            assert abs(e[jj] - v.min()) <= 1e-12 * max(abs(v.min()), 1e-300), (a, ref, e[jj], v.min())
            ties += 1
        c = a
    assert N - c <= max_seg and N - c >= min(N, SR)
    return ties


def make_long_files(sr):
    """Two files of make_clip pieces with near-silent gaps (~62 s and ~195 s), 90 s of noise, 70 s of zeros."""
    return [gap_file(2, [8.0, 11.0, 6.5, 9.7, 12.0, 7.3], sr=sr)[0],
            gap_file(3, [14.0, 3.0, 22.0, 9.0, 17.5, 28.0, 6.0, 19.0, 25.0, 21.0, 24.0], sr=sr)[0],
            (np.random.default_rng(5).standard_normal(90 * sr) * 0.1).astype(np.float32),
            np.zeros(70 * sr + 77, dtype=np.float32)]


@pytest.fixture(scope="module")
def long_files():
    return make_long_files(SR)


@pytest.mark.gpu
@pytest.mark.parametrize("max_s,search_s", [(30.0, 5.0), (10.0, 5.0), (5.0, 2.0)])
def test_cuts_match_reference(tiny_engine, long_files, report, max_s, search_s):
    """asrb_segment_long on files ingested at 16 kHz f32 and at 44.1 kHz s16 gives the reference rule's cuts on the
    samples asrb_long_read returns."""
    from qwen3_asr_rs_b200.inference import check_segmenting
    eng = tiny_engine
    max_seg, search = check_segmenting(max_s, search_s)
    ties = 0
    for rate in (16000, 44100):
        pcms = long_files if rate == 16000 else [(f * 32767).astype(np.int16) for f in make_long_files(rate)]
        xs = eng.ingest_long(pcms, [rate] * len(pcms))
        got = eng.segment_long(max_seg, search)
        for x, g in zip(xs, got):
            ties += _check_cuts(x, g, max_seg, search)
    report[f"longform_cut_ties_{max_s}_{search_s}"] = ties
    zero = got[3]            # all-zero file: longest pieces (the one before the last may be shortened to keep 1 s last)
    assert [b - a for a, b in zero[:-2]] == [max_seg] * (len(zero) - 2)


@pytest.mark.gpu
def test_segment_long_capacity_retry_and_refusals(tiny_engine, long_files):
    from qwen3_asr_rs_b200 import _lib
    eng = tiny_engine
    eng.ingest_long(long_files[:2], [SR, SR])
    s, lib = eng._session, eng._lib
    n = (C.c_int32 * 2)()
    st, en = (C.c_int64 * 64)(), (C.c_int64 * 64)()
    assert lib.asrb_segment_long(s, 160000, 80000, 3, n, st, en) == 1         # does not fit: counts still filled
    want = [len(ref_segments(x, 160000, 80000)) for x in eng.ingest_long(long_files[:2], [SR, SR])]
    assert list(n) == want
    assert lib.asrb_segment_long(s, 160000, 80000, sum(want), n, st, en) == 0
    for bad in ((160001, 80000), (160000, 80001), (79840, 32000), (160000, 31840), (160000, 80160)):
        assert lib.asrb_segment_long(s, bad[0], bad[1], 64, n, st, en) == 1, bad
    with pytest.raises(_lib.AsrbError):
        eng.ingest_long([np.zeros((0, 1), np.float32)], [SR])
    assert lib.asrb_segment_long(s, 160000, 80000, 64, n, st, en) == 4         # a failed ingest leaves nothing


def _host_clips(eng, pcms, rates, max_seg, search):
    xs = eng.ingest_long(pcms, rates)
    segs = eng.segment_long(max_seg, search)
    return [(f, a, b, xs[f][a:b].copy()) for f in range(len(xs)) for a, b in segs[f]]


def _flat(rows):
    return np.array([v for r in rows for v in r], dtype=np.float32)


def _compare(long_res, ref_runs, with_lp=False, with_top=False, with_nbest=False):
    segs = [sg for f in long_res.files for sg in f]
    ids = [i for r in ref_runs for i in r.ids]
    assert [sg.ids for sg in segs] == ids
    if with_lp:
        lp = [x for r in ref_runs for x in r.logprobs]
        assert np.array_equal(_flat([sg.logprobs for sg in segs]), _flat(lp))
        assert [sg.eos_logprob for sg in segs] == [x for r in ref_runs for x in r.eos_logprobs]
    if with_top:
        assert [sg.top_logprobs for sg in segs] == [x for r in ref_runs for x in r.top_logprobs]
    if with_nbest:
        assert [sg.nbest for sg in segs] == [x for r in ref_runs for x in r.nbest]


def _views_equal_copies(eng, pcms, rates, max_s, search_s, batch, n_new, report, tag, ctx=None):
    from qwen3_asr_rs_b200.inference import check_segmenting
    max_seg, search = check_segmenting(max_s, search_s)
    cl = _host_clips(eng, pcms, rates, max_seg, search)
    clips = [c[3] for c in cl]
    sctx = None if ctx is None else [ctx[c[0]] for c in cl]

    def waves(W, **kw):
        out = []
        for w0 in range(0, len(clips), W):
            c = None if sctx is None else sctx[w0:w0 + W]
            out.append(eng.transcribe_ids(clips[w0:w0 + W], max_new_tokens=n_new, context_ids=c, **kw))
        return out
    common = dict(max_segment_s=max_s, search_s=search_s, batch=batch, max_new_tokens=n_new, context_ids=ctx)
    got = eng.transcribe_long(pcms, rates, **common)
    _compare(got, waves(batch))
    report[f"longform_{tag}_segments"] = got.n_segments
    got = eng.transcribe_long(pcms, rates, logprobs=True, **common)
    _compare(got, waves(batch, logprobs=True), with_lp=True)
    got = eng.transcribe_long(pcms, rates, top_logprobs=8, **common)
    _compare(got, waves(batch, top_logprobs=8), with_lp=True, with_top=True)
    got = eng.transcribe_long(pcms, rates, logprobs=True, temperature=0.8, seed=77, **common)
    _compare(got, waves(batch, logprobs=True, temperature=0.8, seed=77), with_lp=True)
    assert all(sg.temperature == 0.8 for f in got.files for sg in f)
    got = eng.transcribe_long(pcms, rates, beam_size=3, **common)
    _compare(got, waves(batch // 3, beam_size=3), with_nbest=True)
    assert got.n_waves == -(-len(clips) // (batch // 3))
    return cl


@pytest.mark.gpu
def test_views_equal_copies_tiny(tiny_engine, report):
    """transcribe_long (views of the long buffer) equals transcribe_ids on the same samples cut out on the host, in the
    same batch order: ids, log-probability records, top-8 records, sampled ids, beam n-best lists; and with a context
    per file, each file's segments share its prefill."""
    eng = tiny_engine
    a, _ = gap_file(11, [4.0, 3.5, 4.4, 2.9, 4.1, 3.3])
    b, _ = gap_file(12, [2.0, 4.8, 3.9])
    c, _ = gap_file(13, [4.2, 3.1, 4.7, 2.6])
    pcms, rates = [a, (b * 32767).astype(np.int16), c], [SR, SR, SR]
    _views_equal_copies(eng, pcms, rates, 5.0, 2.0, 16, 10, report, "tiny")
    # contexts: file 0 has one, file 1 none, file 2 another; file 0's segments fit in one wave
    ctxs = [[int(v) for v in np.random.default_rng(3).integers(0, 150000, 17)], None,
            [int(v) for v in np.random.default_rng(4).integers(0, 150000, 5)]]
    cl = _views_equal_copies(eng, [a], [SR], 5.0, 2.0, 16, 10, report, "tiny_ctx", ctx=ctxs[:1])
    eng.transcribe_long([a], [SR], max_segment_s=5.0, search_s=2.0, batch=16, max_new_tokens=10, context_ids=ctxs[:1])
    assert eng.last_prefill_stats()["rows_shared"] == (len(cl) - 1) * (17 + 9)
    _views_equal_copies(eng, pcms, rates, 5.0, 2.0, 16, 10, report, "tiny_ctx3", ctx=ctxs)


@pytest.mark.gpu
def test_views_equal_copies_0p6b_batch16(report):
    """At Qwen3-ASR-0.6B dims, 16 segments per wave: the batch-aware fused step and the beam path on views."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    w = synth.make_weights(cfg, 1)
    eng = AsrInference.from_weights(config_0p6b(), w, device=0)
    try:
        x, _ = gap_file(21, [4.1, 3.0, 4.6, 2.7, 4.4, 3.9, 2.2, 4.8, 3.3, 4.0, 2.5, 4.9, 3.6, 4.2, 2.8, 4.5])
        before = eng.stats()
        cl = _views_equal_copies(eng, [x], [SR], 5.0, 2.0, 16, 12, report, "0p6b")
        st = eng.stats()
        assert len(cl) >= 16
        assert st["decode_batch_steps"] > before.get("decode_batch_steps", 0)
    finally:
        eng.close()


@pytest.mark.gpu
def test_short_file_is_one_segment(tiny_engine):
    eng = tiny_engine
    x = synth.make_clip(31, 7.3)
    pcm = (x * 32767).astype(np.int16)
    got = eng.transcribe_long([pcm], [SR], max_segment_s=10.0, search_s=5.0, max_new_tokens=12, logprobs=True)
    ref = eng.transcribe_pcm([pcm], [SR], max_new_tokens=12, logprobs=True)
    assert len(got.files[0]) == 1 and got.files[0][0].start_s == 0.0 and got.files[0][0].end_s == len(x) / SR
    sg = got.files[0][0]
    assert sg.ids == ref.ids[0]
    assert np.array_equal(np.array(sg.logprobs, np.float32), np.array(ref.logprobs[0], np.float32))
    assert sg.eos_logprob == ref.eos_logprobs[0]


@pytest.mark.gpu
def test_long_file_stays_on_fused_steps(report):
    """A ~3 min file at 0.6B dims: transcribe_long decodes on the batch-aware fused step only, while the same file in
    one pass has a prompt beyond the fused step's 1152 keys and runs per-phase steps."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    w = synth.make_weights(cfg, 1)
    eng = AsrInference.from_weights(config_0p6b(), w, device=0)
    try:
        x, _ = gap_file(41, [26.0, 22.0, 29.0, 18.0, 27.0, 24.0, 28.0], gap_s=0.8)
        assert 170 * SR < len(x) < 190 * SR
        eng.transcribe_long([x], [SR], max_segment_s=30.0, max_new_tokens=8)        # session, warm-up
        s0 = eng.stats()
        got = eng.transcribe_long([x], [SR], max_segment_s=30.0, max_new_tokens=8)
        s1 = eng.stats()
        report["longform_3min_segments"] = got.n_segments
        assert got.n_segments >= 6 and got.n_waves == 1
        assert s1["decode_phase_steps"] == s0["decode_phase_steps"]
        assert s1["decode_fused_steps"] == s0["decode_fused_steps"]
        assert s1["decode_batch_steps"] - s0["decode_batch_steps"] == got.decode_steps == 7
    finally:
        eng.close()
    one_pass = AsrInference.from_weights(config_0p6b(), w, device=0)     # its own session: one row of 3 min
    try:
        p0 = one_pass.stats()
        one = one_pass.transcribe_ids([x], max_new_tokens=8)
        p1 = one_pass.stats()
        assert one.decode_steps == 7 and p1["decode_phase_steps"] > p0.get("decode_phase_steps", 0)
    finally:
        one_pass.close()


@pytest.mark.gpu
def test_transcribe_segments_refusals(tiny):
    """Every refusal of asrb_transcribe_segments returns its status before any work; a following valid call still equals
    transcribe_ids on the cut-out samples."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    try:
        x, _ = gap_file(51, [3.0, 4.0])
        y = synth.make_clip(52, 2.0)
        eng.transcribe_ids([x[:SR]] * 4, max_new_tokens=8)        # a session of 4 rows, 16000 samples, 8 new tokens
        s, lib = eng._session, eng._lib
        ids, lens = (C.c_int32 * (8 * 8))(), (C.c_int32 * 8)()

        def call(files, starts, ends, n=None, max_new=8):
            n = len(files) if n is None else n
            k = max(len(files), 1)
            return lib.asrb_transcribe_segments(s, n, (C.c_int32 * k)(*files), (C.c_int64 * k)(*starts),
                                                (C.c_int64 * k)(*ends), None, None, max_new, ids, lens)
        assert call([0], [0], [1000]) == 4                                   # nothing ingested with asrb_ingest_long
        nseg = (C.c_int32 * 1)()
        assert lib.asrb_segment_long(s, 160000, 80000, 4, nseg, (C.c_int64 * 4)(), (C.c_int64 * 4)()) == 4
        xs = eng.ingest_long([x, y], [SR, SR])
        N1 = len(xs[1])
        steps0 = eng.stats()
        bad = [([2], [0], [1000]), ([-1], [0], [1000]), ([0], [500], [500]), ([0], [600], [500]), ([0], [-1], [1000]),
               ([1], [N1 - 1000], [N1 + 1]), ([0], [0], [200]), ([0], [0], [16001]),
               ([0] * 5, [0] * 5, [1000] * 5)]
        for files, starts, ends in bad:
            assert call(files, starts, ends) == 1, (files, starts, ends)
        assert call([0], [0], [1000], n=0) == 1
        assert call([0], [0], [1000], max_new=9) == 1
        eng.set_option("beam_size", "3")
        try:
            assert call([0, 1], [0, 0], [1000, 1000]) == 1                   # 2 x 3 > 4 rows
        finally:
            eng.set_option("beam_size", "1")
        assert eng.stats() == steps0                                         # no decode work ran
        assert call([0, 1, 0], [0, 100, 16000], [16000, 12100, 16000 + 201]) == 0
        got = [list(ids[b * 8: b * 8 + lens[b]]) for b in range(3)]
        ref = eng.transcribe_ids([xs[0][:16000], xs[1][100:12100], xs[0][16000:16201]], max_new_tokens=8)
        assert got == ref.ids
    finally:
        eng.close()


@pytest.mark.gpu
def test_segment_ids_equal_fp32_oracle(report):
    """Tiny config with the peaked untied head: the ids of every segment whose oracle-side worst top-1/top-2 gap is above
    the noise floor equal the fp32 oracle's on that segment cut out on the host."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    cfg = O.cfg_tiny()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 7, peaked_head=True)
    model = O.OracleModel(cfg, w)
    ecfg = config_tiny()
    ecfg.text.tie_word_embeddings = False
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        x, _ = gap_file(61, [4.0, 9.1, 3.2, 7.7, 5.5, 8.3, 2.4])
        got = eng.transcribe_long([x], [SR], max_segment_s=10.0, search_s=5.0, max_new_tokens=24)
        xs = eng.ingest_long([x], [SR])[0]
    finally:
        eng.close()
    checked, margins = 0, []
    for sg in got.files[0]:
        a, b = int(round(sg.start_s * SR)), int(round(sg.end_s * SR))
        ref = O.transcribe_ids(model, xs[a:b], max_new_tokens=24, keep_logits=True)
        ls = [ref.prefill_logits] + ref.step_logits[:-1]
        m = min(float(l.topk(2).values[0] - l.topk(2).values[1]) for l in ls) / max(float(l.abs().max()) for l in ls)
        margins.append(m)
        if m >= 5 * MARGIN_FLOOR_REL:
            assert sg.ids == ref.ids, (sg.start_s, m)
            checked += 1
    report["longform_oracle_margins"] = margins
    assert checked >= 3, margins
