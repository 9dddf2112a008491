"""Streaming transcription (asrb_stream_*, DESIGN.md 4.9).

CPU: a numpy mirror of the window-reuse rule over growing prefixes reproduces the offline clamped mel of every prefix
bit for bit, on a clip whose floor moves up (silence, then speech) and on one whose loud provisional end frame settles
lower (the floor moves down); the same mirror without the floor condition fails on both.  The host rules (rollback and
unfixed pushes, P_b, the refusals) and the CLI's --stream parsing.

GPU: the stream's mel is bitwise asrb_mel of the prefix after every push, its window counters are the mirror's, its
encoder output is the offline encoder's on the prefix, and its continuation equals transcribe_ids(prefix, lang + p) at
every push; several streams with idle ones and a reset; the lifecycle and its refusals; reproducibility.
"""
import numpy as np
import pytest

from qwen3_asr_rs_b200 import stream as S
from qwen3_asr_rs_b200 import synth

HOP, NFFT = 160, 400
WIN_FRAMES = 800                   # released dims: chunks of 2 * n_window = 100 frames, n_window_infer = 800 frames
PUSH = 16000                       # 1 s pushes


# ---------------------------------------------------------------------------------------------------------------------
# a frame-exact float64 -> float32 raw log-mel: each frame's value depends on that frame's samples only
# ---------------------------------------------------------------------------------------------------------------------
_FB = None


def _fb():
    global _FB
    if _FB is None:
        from oracle import oracle as O
        _FB = O.mel_filterbank(128).astype(np.float64)
    return _FB


def raw_log_mel(x: np.ndarray) -> np.ndarray:
    """Pre-floor log10 mel [128][F] of x, F = ceil(n / 160) (mel.rs: hop zero padding, reflection, Hann, |STFT|^2)."""
    x = np.asarray(x, dtype=np.float32)
    npad = -(-len(x) // HOP) * HOP
    xp = np.zeros(npad, dtype=np.float64)
    xp[: len(x)] = x
    wave = np.pad(xp, (NFFT // 2, NFFT // 2), mode="reflect")
    F = npad // HOP
    idx = np.arange(F)[:, None] * HOP + np.arange(NFFT)[None, :]
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(NFFT) / NFFT)
    mag = np.abs(np.fft.rfft(wave[idx] * win, axis=1)) ** 2          # [F][201], row by row
    fb = _fb()
    acc = np.zeros((128, F))
    for k in range(fb.shape[1]):                                     # fixed summation order per (mel, frame)
        acc += fb[:, k: k + 1] * mag[None, :, k]
    return np.log10(np.maximum(acc, 1e-10)).astype(np.float32)


def offline_mel(raw: np.ndarray) -> np.ndarray:
    phi = np.float32(raw.max()) - np.float32(8.0)
    return ((np.maximum(raw, phi) + np.float32(4.0)) / np.float32(4.0)).astype(np.float32)


def final_frames(n: int, final: bool) -> int:
    F = -(-n // HOP)
    return F if final else min(F, (n - 200) // HOP + 1 if n >= 200 else 0)


def mirror(x: np.ndarray, pushes, win_frames: int = WIN_FRAMES, floor_rule: bool = True):
    """The reuse rule of session_stream_push over the pushes' prefixes.  Yields per push (n, assembled clamped mel,
    counters {encoded, reused, floor_moved}, tokens-before-first-re-encoded in frames).  A reused window keeps the
    clamped values it was encoded with; without `floor_rule` a finished window is reused whatever the floor did."""
    raw_store = None
    fin_max, Ffin = -np.inf, 0
    wmin, wphi, wfinal, clamped = {}, {}, {}, {}
    for j, n in enumerate(pushes):
        final = j == len(pushes) - 1
        raw = raw_log_mel(x[:n])
        F = raw.shape[1]
        if raw_store is not None:                                    # final frames never change
            assert np.array_equal(raw[:, :Ffin], raw_store[:, :Ffin])
        raw_store = raw
        f_new = final_frames(n, final)
        if f_new > Ffin:
            fin_max = max(fin_max, float(raw[:, Ffin:f_new].max()))
            for w in range(Ffin // win_frames, -(-f_new // win_frames)):
                a, b = max(Ffin, w * win_frames), min(f_new, (w + 1) * win_frames)
                wmin[w] = min(wmin.get(w, np.inf), float(raw[:, a:b].min()))
        tail = float(raw[:, f_new:].max()) if F > f_new else -np.inf
        Ffin = f_new
        phi = np.float32(max(fin_max, tail)) - np.float32(8.0)
        counts = dict(encoded=0, reused=0, floor_moved=0)
        first_re = None
        out = np.empty_like(raw)
        for w in range(-(-F // win_frames)):
            a, b = w * win_frames, min(F, (w + 1) * win_frames)
            finished = b <= Ffin
            ok = (phi == wphi.get(w) or wmin.get(w, -np.inf) >= max(phi, wphi.get(w, phi))) if floor_rule else True
            if finished and wfinal.get(w) and ok:
                counts["reused"] += 1
            else:
                if finished and wfinal.get(w):
                    counts["floor_moved"] += 1
                counts["encoded"] += 1
                clamped[w] = ((np.maximum(raw[:, a:b], phi) + np.float32(4.0)) / np.float32(4.0)).astype(np.float32)
                wphi[w], wfinal[w] = phi, finished
                first_re = w if first_re is None else first_re
            out[:, a:b] = clamped[w]
        yield n, out, counts, first_re


def clip_floor_up(seconds_quiet: float = 10.0, seconds_loud: float = 8.0) -> np.ndarray:
    rng = np.random.default_rng(7)
    quiet = (rng.normal(0, 1e-3, int(seconds_quiet * 16000))).astype(np.float32)
    return np.concatenate([quiet, synth.make_clip(3, seconds_loud)]).astype(np.float32)


def clip_floor_down(seconds: float = 14.0, end: int = 9 * PUSH) -> np.ndarray:
    """Low noise with a short loud tone burst ending 141 samples before a push boundary.  While it is near the end of
    the audio, the end frame (its window reflected at the last sample) holds the clip's maximum; one push later that
    frame is final and lower, and no new frame reaches it: the floor moves down (found by a seeded search)."""
    rng = np.random.default_rng(11)
    x = rng.normal(0, 1e-3, int(seconds * 16000)).astype(np.float32)
    L, off = 31, 141
    t = np.arange(L) / 16000.0
    x[end - off - L: end - off] += (0.5 * np.sin(2 * np.pi * 1161.273157308735 * t + 0.4442515599503922)
                                    * np.hanning(L)).astype(np.float32)
    return x


def pushes_of(n: int, step: int = PUSH):
    return [min(a + step, n) for a in range(0, n, step)]


CLIPS = {"floor_up": clip_floor_up, "floor_down": clip_floor_down}


@pytest.mark.parametrize("name", sorted(CLIPS))
def test_reuse_rule_reproduces_offline_mel(name):
    x = CLIPS[name]()
    pushes = pushes_of(len(x))
    moved, phis = 0, []
    for n, got, counts, _ in mirror(x, pushes):
        raw = raw_log_mel(x[:n])
        phis.append(float(np.float32(raw.max()) - np.float32(8.0)))
        assert np.array_equal(got.view(np.int32), offline_mel(raw).view(np.int32)), n
        moved += counts["floor_moved"]
    assert moved >= 1                                             # the floor condition was exercised
    if name == "floor_down":
        assert any(b < a for a, b in zip(phis, phis[1:]))          # and the floor did move down


@pytest.mark.parametrize("name", sorted(CLIPS))
def test_reuse_rule_without_floor_condition_fails(name):
    """Negative control: reusing every finished window whatever the floor did gives another mel on these clips."""
    x = CLIPS[name]()
    bad = 0
    for n, got, _, _ in mirror(x, pushes_of(len(x)), floor_rule=False):
        bad += not np.array_equal(got.view(np.int32), offline_mel(raw_log_mel(x[:n])).view(np.int32))
    assert bad >= 1


def test_next_prefix_rollback_and_unfixed():
    h = list(range(10, 22))
    assert S.next_prefix(h, 0, 5, 2, False) == []                  # k + 1 < U: nothing fixed yet
    assert S.next_prefix(h, 1, 5, 2, False) == h[:7]
    assert S.next_prefix(h, 1, 20, 2, False) == []                 # rollback longer than h
    assert S.next_prefix(h, 0, 5, 0, False) == h[:7]
    assert S.next_prefix(h, 0, 5, 2, True) == h                    # final: no rollback
    assert S.next_prefix(h, 3, 0, 1, False) == h


def test_prompt_rows_kept():
    assert S.prompt_rows_kept(0, 104, first_push=True) == 0
    assert S.prompt_rows_kept(0, 0, first_push=False) == 9
    assert S.prompt_rows_kept(5, 208, first_push=False) == 9 + 5 + 208


def test_max_lang_ids_bound():
    assert S.stream_max_lang_ids(60.0, 0, 8) == 480 + 8
    assert S.stream_max_lang_ids(1.5, 3, 32) == 3 + 12 + 32


def test_cli_stream_parsing():
    from qwen3_asr_rs_b200 import __main__ as M
    assert M.split_stream(["m", "a.wav"]) == (["m", "a.wav"], None)
    assert M.split_stream(["m", "--stream", "1", "a.wav"]) == (["m", "a.wav"], 1.0)
    assert M.split_stream(["m", "a.wav", "--stream=0.5"]) == (["m", "a.wav"], 0.5)
    for bad in (["--stream"], ["--stream", "x"], ["--stream", "0"], ["--stream", "0.005"], ["--stream", "31"]):
        assert M.split_stream(["m", "a.wav"] + bad) is None
    assert M.stream_pushes(40000, 1.0) == [(0, 16000, False), (16000, 32000, False), (32000, 40000, True)]
    parts = M.stream_pushes(75 * 16000, 10.0)                      # a long recording: streams of 30 s, then the rest
    assert [p[2] for p in parts] == [False, False, True, False, False, True, False, True]
    assert parts[3][0] == 30 * 16000 and parts[-1][1] == 75 * 16000
    for bad in (["--logprobs"], ["--top-logprobs", "2"], ["--score", "x"], ["--detect-language"], ["--beam-size", "2"],
                ["--temperature", "0,0.4"]):
        assert M.main(["m", "a.wav", "--stream", "1"] + bad) == 1
    assert M.main(["m", "a.wav", "--stream", "1", "--max-segment", "30"]) == 1


def test_refusals_before_any_session():
    from qwen3_asr_rs_b200.stream import StreamSet

    class Eng:                                                    # never reached: the arguments are refused first
        _options = {}
    for kw in (dict(n=0), dict(max_seconds=0.0), dict(rollback=-1), dict(unfixed_pushes=-1), dict(temperature=[0.0, 0.2]),
               dict(temperature=0.5, top_logprobs=2)):
        args = dict(n=1, max_seconds=5.0, lang_ids=None, context_ids=None, rollback=5, unfixed_pushes=2, max_new_tokens=8,
                    logprobs=False, top_logprobs=0, temperature=0.0, seed=0, no_repeat_ngram_size=0, repetition_penalty=1.0)
        args.update(kw)
        with pytest.raises(ValueError):
            StreamSet(Eng(), **args)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _tiny_engine(seed=3):
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    return AsrInference.from_weights(config_tiny(), synth.make_weights(O.cfg_tiny(), seed), device=0)


def _run_schedule(eng, x_list, schedule, max_new=8, lang=None, **kw):
    """Streams x_list[b] pushed per `schedule` (a list of pushes, each a list of sample counts per stream, 0 = idle; the
    last nonzero count of a stream ends it with final).  Returns per push the (prefix used, hypotheses) and stats."""
    n = len(x_list)
    ss = eng.open_streams(n, max(len(x) for x in x_list) / 16000.0 + 1.0, max_new_tokens=max_new, language_ids=lang, **kw)
    R, U = kw.get("rollback", 5), kw.get("unfixed_pushes", 2)
    k = [0] * n
    pos = [0] * n
    recs = []
    prefix = [[] for _ in range(n)]
    for step in schedule:
        chunks, fin = [], []
        for b, c in enumerate(step):
            chunks.append(x_list[b][pos[b]: pos[b] + c] if c else None)
            pos[b] += c
            fin.append(bool(c) and pos[b] >= len(x_list[b]))
        before = [list(p) for p in prefix]
        hyps = ss.push(chunks, final=fin)
        recs.append(dict(n=list(pos), active=[bool(c) for c in step], prefix=before, hyps=hyps, stats=ss.stats(),
                         mel=[ss.mel(b) if step[b] else None for b in range(n)]))
        for b in range(n):
            if step[b]:                                             # the library's rollback and U rule
                assert hyps[b].ids[: hyps[b].fixed] == S.next_prefix(hyps[b].ids, k[b], R, U, fin[b]), (b, k[b])
                prefix[b] = hyps[b].ids[: hyps[b].fixed]
                k[b] += 1
    return ss, recs


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CLIPS))
def test_gpu_mel_bitwise_and_window_counters(name):
    x = CLIPS[name]()
    pushes = pushes_of(len(x))
    eng = _tiny_engine()
    try:
        steps = [[b - a] for a, b in zip([0] + pushes, pushes)]
        _, recs = _run_schedule(eng, [x], steps)
        pred = list(mirror(x, pushes))
        for r, (n, _, counts, _) in zip(recs, pred):
            st = r["stats"]
            assert (st["windows_encoded"], st["windows_reused"], st["windows_floor_moved"]) == \
                (counts["encoded"], counts["reused"], counts["floor_moved"]), n
        offline = [eng.mel([x[:n]])[0] for n in pushes]
        for r, ref in zip(recs, offline):
            assert np.array_equal(r["mel"][0].view(np.int32), ref.view(np.int32)), r["n"]
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_ids_equal_offline_with_forced_prefix():
    """g of every push equals transcribe_ids(prefix audio, lang + p); the prompt rows kept are P_b; the encoder output
    meets the offline encoder's on the prefix; the final push equals the offline transcription with lang + p."""
    x = synth.make_clip(5, 19.3)
    lang = [151700, 151701]
    eng = _tiny_engine()
    try:
        pushes = pushes_of(len(x))
        steps = [[b - a] for a, b in zip([0] + pushes, pushes)]
        _, recs = _run_schedule(eng, [x], steps, max_new=8, lang=lang)
        assert recs[-1]["hyps"][0].fixed == len(recs[-1]["hyps"][0].ids)
        pred = list(mirror(x, pushes))
        for j, (r, (n, _, _, first_re)) in enumerate(zip(recs, pred)):
            kept = S.prompt_rows_kept(0, n_tokens(first_re * 800), first_push=j == 0)
            S_b = 9 + n_tokens(-(-n // 160)) + 6 + len(lang) + len(r["prefix"][0])
            assert (r["stats"]["prompt_rows_kept"], r["stats"]["prompt_rows_computed"]) == (kept, S_b - kept), n
        assert any(r["stats"]["prompt_rows_kept"] >= 9 + 104 for r in recs)     # a finished window's pads were kept
        for r in recs:
            n, p, h = r["n"][0], r["prefix"][0], r["hyps"][0]
            got = eng.transcribe_ids([x[:n]], language_ids=[lang + p], max_new_tokens=8).ids[0]
            assert h.ids == p + got, (n, p, h.ids, got)
    finally:
        eng.close()


def n_tokens(frames: int) -> int:
    """Encoder tokens of `frames` mel frames: chunks of 100 frames, three stride-2 convolutions each."""
    out = 0
    for k in range(0, frames, 100):
        f = min(100, frames - k)
        for _ in range(3):
            f = (f - 1) // 2 + 1
        out += f
    return out


@pytest.mark.gpu
def test_gpu_several_streams_idle_and_reset():
    xs = [synth.make_clip(20 + b, s) for b, s in enumerate((9.5, 6.2, 12.0))]
    sched = [[16000, 16000, 0], [16000, 0, 16000], [0, 16000, 16000], [16000, 16000, 16000], [16000, 0, 16000]]
    eng = _tiny_engine()
    try:
        _, multi = _run_schedule(eng, xs, sched)
        for r_prev, r in zip(multi, multi[1:]):                     # idle streams: hypotheses unchanged, bitwise
            for b in range(3):
                if not r["active"][b]:
                    assert r["hyps"][b].ids == r_prev["hyps"][b].ids and r["hyps"][b].fixed == r_prev["hyps"][b].fixed
        for b in range(3):                                          # each stream alone on the same schedule
            own = [[st[b]] for st in sched if st[b]]
            _, single = _run_schedule(eng, [xs[b]], own)
            got = [r["hyps"][b].ids for r in multi if r["active"][b]]
            assert got == [r["hyps"][0].ids for r in single], b
        # reset in the middle: stream 1 starts over and then matches a fresh stream
        ss = eng.open_streams(2, 13.0, max_new_tokens=8)
        ss.push([xs[0][:16000], xs[1][:16000]])
        ss.reset(1)
        h1 = ss.push([None, xs[2][:20000]])[1]
        _, fresh = _run_schedule(eng, [xs[2]], [[20000]])
        assert h1.ids == fresh[0]["hyps"][0].ids
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_lifecycle_refusals_and_reproducibility():
    from qwen3_asr_rs_b200._lib import AsrbError
    x = synth.make_clip(9, 6.0)
    eng = _tiny_engine()
    try:
        runs = []
        for _ in range(2):
            _, recs = _run_schedule(eng, [x], [[16000]] * 6)
            runs.append([r["hyps"][0].ids for r in recs])
        assert runs[0] == runs[1]                                   # bitwise reproducible
        final = recs[-1]["hyps"][0]
        off = eng.transcribe_ids([x], language_ids=[recs[-1]["prefix"][0]], max_new_tokens=8).ids[0]
        assert final.ids == recs[-1]["prefix"][0] + off
        ss = eng.open_streams(2, 3.0, max_new_tokens=8)
        ss.push([x[:16000], None], final=[True, False])
        with pytest.raises(AsrbError) as e:                         # closed until reset
            ss.push([x[16000:20000], None])
        assert e.value.code == 4
        with pytest.raises(AsrbError) as e:                         # past max_samples: refused, streams intact
            ss.push([None, np.zeros(eng._cap[1] + 1, np.float32)])
        assert e.value.code == 1
        closed = ss.push([None, None])[0]
        h = ss.push([None, x[:16000]])
        assert h[1].ids and h[0].ids == closed.ids                   # the refusals left both streams usable
        ss.reset(0)
        ss.push([x[:16000], None])
        eng.transcribe_ids([x[:16000]], max_new_tokens=4)            # a non-stream call ends the streams
        with pytest.raises(AsrbError) as e:
            ss.push([x[16000:20000], None])
        assert e.value.code == 4
        eng.set_option("beam_size", "2")
        with pytest.raises(ValueError):
            eng.open_streams(1, 3.0)
        eng.set_option("beam_size", "1")
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_prefix_overflow_and_beam_refusals_leave_streams_usable():
    """|lang| + |p| past max_lang_ids and beam_size > 1 on push are refused with ASRB_ERR_INVALID before any work: the
    hypotheses are unchanged and the streams take further pushes."""
    from qwen3_asr_rs_b200._lib import AsrbError
    x = synth.make_clip(12, 3.0)
    eng = _tiny_engine()
    try:
        ss = eng.open_streams(1, 2.0, max_new_tokens=8, rollback=0, unfixed_pushes=0)
        cap = eng._cap[2]                                           # max_lang_ids = 8 x 2 s + 8
        assert cap == S.stream_max_lang_ids(2.0, 0, 8)
        pos, last = 0, None
        while True:                                                 # the prefix grows by 8 ids per push
            before = last
            try:
                last = ss.push([x[pos: pos + 4000]])[0]
            except AsrbError as e:
                assert e.code == 1 and before is not None
                assert len(before.ids) > cap                        # refused exactly when |p| > max_lang_ids
                break
            pos += 4000
            assert len(last.ids) == last.fixed                      # rollback 0, U 0: all of h is fixed
        assert ss.push([None])[0].ids == before.ids                 # unchanged by the refusal
        ss.reset(0)
        h = ss.push([x[:4000]])[0]
        assert len(h.ids) == 8
        eng.set_option("beam_size", "2")
        with pytest.raises(AsrbError) as e:                         # the library refuses beams on streams
            ss.push([x[4000:8000]])
        assert e.value.code == 1
        eng.set_option("beam_size", "1")
        assert ss.push([None])[0].ids == h.ids
        assert len(ss.push([x[4000:8000]])[0].ids) == 16
    finally:
        eng.close()
