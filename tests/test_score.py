"""Teacher-forced scoring (asrb_score_ids, AsrInference.score_ids / detect_language): the per-token log-probabilities and
top-8 records of the wgmma score head against log_softmax of the float64 oracle's score_ids, under DESIGN.md section 2's
rule (test_precision_fp64.py); prompt sharing, independence from the decode options, refusals, waves and language
identification.  CPU tests: the host helpers and the CLI flags."""
import ctypes as C
import wave

import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth
from qwen3_asr_rs_b200.inference import check_candidates, score_waves
from qwen3_asr_rs_b200.text import LANGUAGES, language_probabilities
from test_precision_fp64 import R, Err, check, context_prompt, options, ratio

EOS = 151645
K = 8
ASRB_ERR_INVALID, ASRB_ERR_STATE = 1, 4


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_check_candidates():
    assert check_candidates([[[1, 2], [3]]], 1, 10) == [[[1, 2], [3]]]
    for bad, msg in (([[[1]], [[2]]], "one candidate list"), ([[]], "no candidate"), ([[[]]], "empty candidate"),
                     ([[[10]]], "out of"), ([[[-1]]], "out of")):
        with pytest.raises(ValueError, match=msg):
            check_candidates(bad, 1, 10)


def test_score_waves():
    assert score_waves([1, 1, 1], 32) == [[0, 1, 2]]
    assert score_waves([2, 2, 2], 4) == [[0, 1], [2]]
    assert score_waves([5, 1, 1], 2) == [[0], [1, 2]]         # an utterance larger than the cap gets a call of its own
    assert score_waves([1, 6, 1], 3) == [[0], [1], [2]]


def test_language_softmax():
    r = language_probabilities(["a", "b", "c"], [-1.0, -3.0, -1.0 - np.log(3.0)])
    assert [n for n, _ in r] == ["a", "c", "b"]
    assert abs(sum(p for _, p in r) - 1.0) < 1e-12
    assert abs(r[0][1] / r[1][1] - 3.0) < 1e-9
    with pytest.raises(ValueError):
        language_probabilities(["a"], [])


def test_language_set_has_no_prefixes():
    assert len(LANGUAGES) == 30 == len(set(LANGUAGES))
    assert not [(a, b) for a in LANGUAGES for b in LANGUAGES if a != b and b.startswith(a)]


def test_cli_flags():
    from qwen3_asr_rs_b200.__main__ import USAGE, split_score
    assert split_score(["m", "a.wav"]) == (["m", "a.wav"], None, False)
    assert split_score(["m", "a.wav", "--score", "hello there"]) == (["m", "a.wav"], "hello there", False)
    assert split_score(["m", "--detect-language", "a.wav"]) == (["m", "a.wav"], None, True)
    assert split_score(["m", "a.wav", "--score"]) is None
    assert split_score(["m", "a.wav", "--score", "x", "--detect-language"]) is None
    assert "--score TEXT" in USAGE and "--detect-language" in USAGE


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def oracle_rows(m32, m64, x, ids, lang=None, ctx=None):
    """(fp32, fp64) log_softmax rows [len(ids)][V] of the teacher-forced oracle, in float64."""
    out = []
    for m in (m32, m64):
        if ctx:
            with context_prompt(ctx):
                s = O.score_ids(m, x, ids, language_ids=lang)
        else:
            s = O.score_ids(m, x, ids, language_ids=lang)
        out.append(torch.log_softmax(s.double(), -1).numpy()[: len(ids)])
    return out


MARGIN = 3e-4                          # DESIGN.md section 2: a gap the rule's errors cannot reorder


def oracle_top(l64_row, k=K + 1):
    """The k best ids of a float64 row under (logit descending, id ascending), and their values."""
    part = np.argpartition(-l64_row, k)[: k + 8]
    order = part[np.lexsort((part, -l64_row[part]))][:k]
    return order, l64_row[order]


def add_errs(err, sc, l32, l64, top=True):
    """Err of one scored candidate: its log-probabilities and, with `top`, every (id, lp) of its top-8 rows.  Each top-8
    row is in (lp descending) order, and where the oracle's 9 best are separated by at least MARGIN it is exactly the
    oracle's 8 best in their order (counted in err.top_exact)."""
    n = len(sc.ids)
    rows = np.arange(n)
    err.add(np.array(sc.logprobs), l32[rows, sc.ids], l64[rows, sc.ids])
    if top:
        for t, row in enumerate(sc.top_logprobs):
            cand = np.array([c[0] for c in row])
            lps = np.array([c[1] for c in row])
            assert len(set(cand.tolist())) == K
            assert (np.diff(lps) <= 0).all(), (t, lps)
            err.add(lps, l32[t, cand], l64[t, cand])
            ids9, v9 = oracle_top(l64[t])
            if (-np.diff(v9) >= MARGIN).all():
                assert cand.tolist() == ids9[:K].tolist(), (t, cand, ids9)
                err.top_exact = getattr(err, "top_exact", 0) + 1
    return err


def candidates_for(eng, x, n_new, vocab, seed, lang=None):
    """The greedy ids + EOS, random ids, length 1, and length n_new."""
    g = eng.transcribe_ids([x], language_ids=[lang] if lang else None, max_new_tokens=n_new - 1).ids[0]
    rng = np.random.default_rng(seed)
    return [list(g) + [EOS], [int(v) for v in rng.integers(0, vocab, 5)], [int(rng.integers(0, vocab))],
            [int(v) for v in rng.integers(0, vocab, n_new)]]


CLIPS = [(31, 0.6), (32, 8.5), (33, 13.1)]       # under one chunk, a tail chunk, past one attention window (11.55 s)


def precision_case(eng, m32, m64, vocab, setup, n_new=12):
    clips = [synth.make_clip(i, s) for i, s in CLIPS]
    lang = [11528, 6364] if setup == "lang" else None
    ctx = [int(v) for v in np.random.default_rng(3).integers(0, 150000, 23)] if setup == "context" else None
    cands = [candidates_for(eng, x, n_new, vocab, 40 + b, lang) if ctx is None else
             [[int(v) for v in np.random.default_rng(50 + b).integers(0, vocab, 12)] + [EOS], [EOS]] for b, x in enumerate(clips)]
    r = eng.score_ids(clips, cands, language_ids=[lang] * 3 if lang else None, context_ids=[ctx] * 3 if ctx else None,
                      top_logprobs=K)
    err = Err(False)
    for b, x in enumerate(clips):
        for sc in r[b]:
            l32, l64 = oracle_rows(m32, m64, x, sc.ids, lang, ctx)
            add_errs(err, sc, l32, l64)
    assert getattr(err, "top_exact", 0) >= 10, "too few top-8 rows with separated oracle logits to check their ids"
    return err


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


# ---------------------------------------------------------------------------------------------------------------------
# GPU: precision
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("setup", ["plain", "lang", "context"])
def test_score_precision_tiny(tiny, tiny64, eng, report, setup):
    cfg, _, m32 = tiny
    check(report, f"score_tiny_{setup}", precision_case(eng, m32, tiny64, cfg.text.vocab_size, setup))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["vocab_odd", "vocab_x8"])
def test_score_precision_ragged_vocab(report, name):
    """Vocabularies of 1185 x 128 + 1 and + 8 with the largest head rows in the ragged tail."""
    from qwen3_asr_rs_b200 import AsrInference
    from test_dims_grid_fp64 import GRID
    ent = GRID[name]
    ocfg, ecfg = ent.configs()
    w = ent.weights(ocfg)
    m32, m64 = O.OracleModel(ocfg, w), O.OracleModel(ocfg, w, dtype=torch.float64)
    e = AsrInference.from_weights(ecfg, w, device=0)
    try:
        err = precision_case(e, m32, m64, ocfg.text.vocab_size, "plain")
    finally:
        e.close()
    check(report, f"score_{name}", err)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["0p6b", "1p7b"])
def test_score_precision_full_width_4_layers(report, size):
    """The 0.6B and 1.7B widths (hidden 1024 / 2048, vocab 151936, untied peaked head), cut to 4 decoder layers."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, config_1p7b
    cfg = O.cfg_0p6b() if size == "0p6b" else O.cfg_1p7b()
    ecfg = config_0p6b() if size == "0p6b" else config_1p7b()
    for c in (cfg, ecfg):
        c.text.tie_word_embeddings = False
        c.text.num_hidden_layers = 4
    w = synth.make_weights(cfg, 1, peaked_head=True)
    m32, m64 = O.OracleModel(cfg, w), O.OracleModel(cfg, w, dtype=torch.float64)
    e = AsrInference.from_weights(ecfg, w, device=0)
    try:
        x = synth.make_clip(9, 6.0)
        cands = candidates_for(e, x, 32, cfg.text.vocab_size, 7)
        r = e.score_ids([x], [cands], top_logprobs=K)[0]
    finally:
        e.close()
    err = Err(False)
    for sc in r:
        l32, l64 = oracle_rows(m32, m64, x, sc.ids)
        add_errs(err, sc, l32, l64)
    check(report, f"score_{size}_4layers", err)


@pytest.mark.gpu
def test_score_negative_control_planes2(tiny, tiny64, eng, report):
    """The score head and prefill fed two bf16 planes per activation must FAIL the rule."""
    cfg, _, m32 = tiny
    with options(eng, planes="2"):
        err = precision_case(eng, m32, tiny64, cfg.text.vocab_size, "plain")
    assert ratio(report, "score_tiny_planes2", err) > R


# ---------------------------------------------------------------------------------------------------------------------
# GPU: agreement with decoding, sharing, independence
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_score_agrees_with_greedy_decoding(tiny, tiny64, eng, report):
    _, _, m32 = tiny
    clips = [synth.make_clip(i, s) for i, s in ((70, 4.0), (71, 2.2))]
    run = eng.transcribe_ids(clips, max_new_tokens=40, logprobs=True)
    err = Err(False)
    for b, x in enumerate(clips):
        ids = list(run.ids[b]) + [EOS]                  # the run's ids, then ending there
        sc = eng.score_ids([x], [[ids]], top_logprobs=K)[0][0]
        l32, l64 = oracle_rows(m32, tiny64, x, ids)
        add_errs(err, sc, l32, l64)
        top2 = np.sort(l64, axis=1)[:, -2:]
        margin = top2[:, 1] - top2[:, 0] >= 3e-4
        for t in np.nonzero(margin[: len(ids) - 1])[0]:
            assert sc.top_logprobs[t][0][0] == ids[t], (b, t)
        if margin[: len(ids) - 1].all():
            assert sc.greedy_prefix >= len(run.ids[b])
    check(report, "score_tiny_greedy_agreement", err)


@pytest.mark.gpu
def test_score_sharing(tiny, tiny64, eng, report):
    cfg, _, m32 = tiny
    clips = [synth.make_clip(81, 2.5), synth.make_clip(82, 9.1)]
    rng = np.random.default_rng(9)
    cands = [[[int(v) for v in rng.integers(0, cfg.text.vocab_size, n)] for n in (4, 1, 7, 1, 3)], [[EOS, 11]]]
    shared = eng.score_ids(clips, cands)
    st = eng.last_prefill_stats()
    alone = eng.score_ids([clips[0]], [[cands[0][2]]])[0][0]
    e_sh, e_al = Err(False), Err(False)
    l32, l64 = oracle_rows(m32, tiny64, clips[0], cands[0][2])
    add_errs(e_sh, shared[0][2], l32, l64, top=False)
    add_errs(e_al, alone, l32, l64, top=False)
    for b, x in enumerate(clips):
        for sc in shared[b]:
            a32, a64 = oracle_rows(m32, tiny64, x, sc.ids)
            add_errs(e_sh, sc, a32, a64, top=False)
    for key, e in (("score_tiny_shared_among_5", e_sh), ("score_tiny_alone", e_al)):   # few values: min_values lowered
        assert ratio(report, key, e, min_values=7) <= R, report[f"fp64_{key}"]
    # rows computed / shared / fanned out: sum S_b + sum (len - 1), sum (n_cand - 1) S_b, rows shared x KV bytes.  S_b
    # is what a single length-1 candidate computes
    n_tok = []
    for x in clips:
        eng.score_ids([x], [[[EOS]]])
        n_tok.append(eng.last_prefill_stats()["rows_computed"])
    want_rows = sum(n_tok) + sum(len(c) - 1 for cs in cands for c in cs)
    t = cfg.text
    kv = 2 * t.num_hidden_layers * t.num_key_value_heads * t.head_dim * 4
    assert st == {"rows_computed": want_rows, "rows_shared": 4 * n_tok[0], "fanout_kv_bytes": 4 * n_tok[0] * kv}
    # a length-1 follower adds no row
    eng.score_ids([clips[0]], [[[5, 6, 7], [EOS]]])
    assert eng.last_prefill_stats()["rows_computed"] == n_tok[0] + 2


@pytest.mark.gpu
def test_score_bitwise_independent_of_decode_options(tiny, eng):
    cfg, _, _ = tiny
    clips = [synth.make_clip(90, 3.0), synth.make_clip(91, 5.5)]
    rng = np.random.default_rng(2)
    cands = [[[int(v) for v in rng.integers(0, cfg.text.vocab_size, 6)] for _ in range(3)], [[EOS]]]

    def flat(r):
        return [(sc.logprobs, sc.top_logprobs) for cs in r for sc in cs]
    a = flat(eng.score_ids(clips, cands, top_logprobs=K))
    assert flat(eng.score_ids(clips, cands, top_logprobs=K)) == a
    with options(eng, temperature="0.7", seed="5", beam_size="2", length_penalty="1.0", no_repeat_ngram_size="2",
                 repetition_penalty="1.5"):
        assert flat(eng.score_ids(clips, cands, top_logprobs=K)) == a


@pytest.mark.gpu
def test_score_refusals_and_state(tiny, eng):
    from qwen3_asr_rs_b200 import _lib
    cfg, _, _ = tiny
    x = synth.make_clip(95, 2.0)
    eng.transcribe_ids([x, x], max_new_tokens=8)           # session: 2 slots, 8 new tokens
    s, lib = eng._session, eng._lib
    samples = (C.POINTER(C.c_float) * 1)(x.ctypes.data_as(C.POINTER(C.c_float)))
    n_s = (C.c_int64 * 1)(x.shape[0])

    def call(cands, n_cand, max_new=8):
        keep = [np.ascontiguousarray(c, dtype=np.int64) for c in cands]
        ptrs = (C.POINTER(C.c_int64) * max(len(keep), 1))(*[a.ctypes.data_as(C.POINTER(C.c_int64)) for a in keep])
        lens = (C.c_int32 * max(len(keep), 1))(*[len(c) for c in cands])
        out = np.zeros((max(len(keep), 1), max_new), np.float32)
        return lib.asrb_score_ids(s, samples, n_s, 1, None, None, (C.c_int32 * 1)(n_cand), ptrs, lens, max_new,
                                  out.ctypes.data_as(C.POINTER(C.c_float)), None, None)
    assert call([[1], [2], [3]], 3) == ASRB_ERR_INVALID                  # more candidates than max_batch
    assert call([[]], 1) == ASRB_ERR_INVALID                             # length 0
    assert call([list(range(9))], 1) == ASRB_ERR_INVALID                 # longer than max_new_tokens
    assert call([[1, 2], [2]], 2, max_new=9) == ASRB_ERR_INVALID         # max_new_tokens above the session's
    assert call([[cfg.text.vocab_size]], 1) == ASRB_ERR_INVALID          # id out of range
    assert call([[-1]], 1) == ASRB_ERR_INVALID
    assert call([], 0) == ASRB_ERR_INVALID                               # an utterance with no candidate
    assert call([[1, 2], [EOS]], 2) == 0                                 # the session is usable
    ids, n = np.zeros((2, 8), np.int32), np.zeros(2, np.int32)
    assert lib.asrb_generate(s, 8, ids.ctypes.data_as(C.POINTER(C.c_int32)), n.ctypes.data_as(C.POINTER(C.c_int32))) == ASRB_ERR_STATE
    lp = np.zeros((2, 8), np.float32)
    assert lib.asrb_last_logprobs(s, 8, lp.ctypes.data_as(C.POINTER(C.c_float)), None) == ASRB_ERR_STATE
    with pytest.raises(_lib.AsrbError):
        _lib.check(lib.asrb_decode_step(s, None, None))
    assert eng.transcribe_ids([x], max_new_tokens=8).ids[0]                  # and decodes again


@pytest.mark.gpu
def test_score_waves_equal_smaller_calls(tiny, eng, monkeypatch):
    from qwen3_asr_rs_b200 import inference
    cfg, _, _ = tiny
    clips = [synth.make_clip(100 + i, s) for i, s in enumerate([1.5, 4.0, 2.2])]
    rng = np.random.default_rng(4)
    cands = [[[int(v) for v in rng.integers(0, cfg.text.vocab_size, n)] for n in ns] for ns in ((3, 2), (4,), (1, 5, 2))]
    whole = eng.score_ids(clips, cands)
    monkeypatch.setattr(inference, "SCORE_SLOTS", 2)
    waves = eng.score_ids(clips, cands)
    singles = [eng.score_ids([x], [c])[0] for x, c in zip(clips, cands)]
    for r in (waves, singles):
        for a, b in zip([sc for cs in whole for sc in cs], [sc for cs in r for sc in cs]):
            assert a.ids == b.ids and np.abs(np.array(a.logprobs) - np.array(b.logprobs)).max() <= 1e-4


class StubTokenizer:
    """Maps "language Xxx" to [11528, 3000 + index of Xxx, 4000 + index] (distinct, none a prefix of another)."""

    def encode(self, text):
        name = text.split(" ", 1)[1]
        i = LANGUAGES.index(name)
        return [11528, 3000 + i, 4000 + i]

    def decode(self, ids):
        return " ".join(map(str, ids))


@pytest.mark.gpu
def test_detect_language(tiny, tiny64, eng, tmp_path):
    _, _, m32 = tiny
    x = synth.make_clip(120, 3.0)
    pcm = np.clip(np.round(x * 32767.0), -32768, 32767).astype("<i2")
    path = str(tmp_path / "clip.wav")
    with wave.open(path, "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000); w.writeframes(pcm.tobytes())
    tok = StubTokenizer()
    eng.tokenizer = tok
    try:
        r = eng.detect_language(path)
    finally:
        eng.tokenizer = None
    assert len(r) == 30 and abs(sum(p for _, p in r) - 1.0) < 1e-6
    xs = pcm.astype(np.float32) / 32768.0
    sums = {}
    for name in LANGUAGES:
        ids = tok.encode(f"language {name}")
        l64 = torch.log_softmax(O.score_ids(tiny64, xs, ids).double(), -1).numpy()
        sums[name] = float(sum(l64[t, i] for t, i in enumerate(ids)))
    best = sorted(sums.values())
    if best[-1] - best[-2] >= 1e-3:
        assert r[0][0] == max(sums, key=sums.get)
