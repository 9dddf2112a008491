"""Repetition controls (session options "no_repeat_ngram_size" / "repetition_penalty").

The rule (include/asr_b200.h, common.cuh): for sequence b at step n the history is ids[0 .. n), the ids the run generated.
Before any use of the step's logits, a logit l_v of an id in the history becomes l_v * theta (l_v < 0) or l_v / theta
(fp32), and with N >= 1 every id that would complete an N-gram already in the history becomes -inf.

Reference: rep_oracle below, the fp32 oracle's logits widened to float64 and processed along the trajectory the float64
processed logits select.  An id is pinned while every step's processed top-1 / top-2 gap exceeds GAP_FLOOR times the
fp32 noise of a GPU logit (test_sampling.py's floor); the log-probability and top-8 records are held to DESIGN 2's
precision rule (R = 4 against the fp32 oracle's processed values) at the GPU's own ids.
"""
import numpy as np
import pytest

EOS = (151643, 151645)
LOGIT_NOISE = 1.5e-5          # fp32 logits vs the oracle, relative to max|logit|
G_NOISE = 4e-6                # fp32 g vs float64 g, absolute (sampling)
GAP_FLOOR = 20.0
R_RULE = 4.0


# ---------------------------------------------------------------------------------------------------------------------
# numpy reference of the rule
# ---------------------------------------------------------------------------------------------------------------------
def banned_ids(hist, N: int):
    """Ids that would complete an N-gram of `hist` (HF's NoRepeatNGramLogitsProcessor on the history)."""
    n = len(hist)
    if N < 1 or n < N:
        return set()
    suffix = list(hist[n - N + 1:]) if N > 1 else []
    return {int(hist[i + N - 1]) for i in range(n - N + 1) if list(hist[i:i + N - 1]) == suffix}


def process(logits, hist, N: int, theta: float):
    """The processed logits l' of one step: the penalty in the logits' own dtype (fp32 multiply / divide for float32
    input), then the bans."""
    l = np.array(logits, copy=True)
    th = l.dtype.type(np.float32(theta))
    h = np.unique(np.asarray(hist, dtype=np.int64))
    if theta != 1.0 and h.size:
        v = l[h]
        l[h] = np.where(v < 0, v * th, v / th)
    for u in banned_ids(hist, N):
        l[u] = -np.inf
    return l


def repeated_ngrams(ids, N: int) -> int:
    grams = [tuple(ids[i:i + N]) for i in range(len(ids) - N + 1)]
    return len(grams) - len(set(grams))


class Run:
    def __init__(self, temperature: float = 0.0):
        self.ids, self.gaps = [], []     # gaps[i]: the processed top-1 / top-2 key gap of the step that selected ids[i] (or EOS)
        self.maxabs = 0.0
        self.eos = False
        self.temperature = temperature

    def pinned(self) -> int:
        """Steps whose selection is pinned: all of them up to the first gap under the floor (test_sampling.py's: the
        logit noise over T, plus the noise of g when sampling)."""
        t = self.temperature
        fl = GAP_FLOOR * (LOGIT_NOISE * self.maxabs / (t if t > 0.0 else 1.0) + (G_NOISE if t > 0.0 else 0.0))
        for i, g in enumerate(self.gaps):
            if not g > fl:
                return i
        return len(self.gaps)


def context_prompt(num_audio_tokens: int, context=None):
    """The library's prompt (session.cu): the context ids inside the system turn."""
    from oracle import oracle as O
    toks, a0 = O.build_prompt(num_audio_tokens)
    if not context:
        return toks, a0
    return toks[:3] + list(context) + toks[3:], a0 + len(context)


def rep_oracle(model, samples, N: int, theta: float, max_new_tokens: int, history_of=None, temperature: float = 0.0,
               seed: int = 0, row: int = 0, context=None):
    """oracle.transcribe_ids selecting on the processed float64 logits (temperature > 0: the seeded draw of
    test_sampling.py on them), with `context` ids in the system turn.  `history_of(prompt, ids)` restates what counts
    as history (negative controls)."""
    import torch
    from oracle import oracle as O
    from test_sampling import gumbel
    t = model.cfg.text
    mel = O.extract_mel(samples, model.cfg.audio.num_mel_bins)
    audio = model.encode(mel)
    prompt, a0 = context_prompt(audio.shape[0], context)
    S = len(prompt)
    hidden = model.embed(prompt).unsqueeze(0)
    hidden[0, a0:a0 + audio.shape[0], :] = audio
    pos = list(range(S))
    cos, sin = O.mrope_cos_sin([pos, pos, pos], t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved)
    cache = [None] * t.num_hidden_layers
    r = Run(temperature)
    with torch.no_grad():
        nxt = model.decoder_forward(hidden, cos, sin, cache, O.causal_mask(S, 0), last_only=True)[:, -1, :]
        cur = S
        for n in range(max_new_tokens):
            hist = r.ids if history_of is None else history_of(prompt, r.ids)
            l = process(nxt[0].double().numpy(), hist, N, theta)
            key = l if temperature == 0.0 else l / temperature + gumbel(seed, row, n, len(l))
            top = np.argpartition(-key, 2)[:2]
            top = top[np.argsort(-key[top])]
            tok = int(top[0])
            r.gaps.append(float(key[top[0]] - key[top[1]]))
            r.maxabs = max(r.maxabs, float(np.abs(l[np.isfinite(l)]).max()))
            if tok in EOS:
                r.eos = True
                break
            r.ids.append(tok)
            h = model.embed([tok]).unsqueeze(0)
            c1, s1 = O.mrope_cos_sin([[cur]] * 3, t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved)
            past = cache[0][0].shape[2]
            nxt = model.decoder_forward(h, c1, s1, cache, O.causal_mask(1, past))[:, 0, :]
            cur += 1
    return r


def assert_pinned(got_ids, ref: Run, label=""):
    k = ref.pinned()
    assert list(got_ids[:k]) == ref.ids[:k], (label, k)
    if k == len(ref.gaps):                     # every step pinned, the EOS-selecting one included
        assert list(got_ids) == ref.ids, label
    return k


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rule
# ---------------------------------------------------------------------------------------------------------------------
def test_ban_hand_cases():
    h = [5, 6, 7, 5, 6]
    assert banned_ids(h, 0) == set()
    assert banned_ids(h, 1) == {5, 6, 7}                    # every id already generated
    assert banned_ids(h, 2) == {7}                          # suffix (6): 6 -> 7 seen
    assert banned_ids(h, 3) == {7}                          # suffix (5, 6): (5, 6) -> 7 seen
    assert banned_ids(h, 4) == set()                        # suffix (7, 5, 6) never seen before
    assert banned_ids(h, 6) == set()                        # fewer ids than N
    assert banned_ids([1, 1, 1], 2) == {1}                  # overlapping matches: (1,1) at 0 and 1
    assert banned_ids([3, 1, 3, 2, 3], 2) == {1, 2}         # both continuations of 3
    assert banned_ids([9, 4, 9, 4, 9], 3) == {4}            # overlapping 3-grams (9,4,9), (4,9,4), (9,4,9)
    assert banned_ids([8, 8], 1) == {8}                     # the id just generated
    assert banned_ids([2, 8], 2) == set() and banned_ids([8, 2, 8], 2) == {2}


def test_penalty_is_fp32_arithmetic():
    rng = np.random.default_rng(0)
    l = (rng.standard_normal(64) * 7).astype(np.float32)
    l[:3] = [0.0, -0.0, 3.0]
    hist = [0, 1, 2, 10, 11, 40, 63, 10]
    for theta in (1.2, 1.3, 10.0):
        got = process(l, hist, 0, theta)
        th = np.float32(theta)
        for v in range(64):
            want = (l[v] * th if l[v] < 0 else l[v] / th) if v in hist else l[v]
            assert got[v].tobytes() == np.float32(want).tobytes(), (theta, v)
        assert got[0] == 0.0 and got[1] == 0.0                      # zero stays zero
    assert process(l, hist, 0, 1.0).tobytes() == l.tobytes()
    # the ban comes after the penalty and wins
    got = process(l, [4, 5, 4], 2, 1.3)
    assert got[5] == -np.inf and got[4].tobytes() == (l[4] * np.float32(1.3) if l[4] < 0 else l[4] / np.float32(1.3)).tobytes()


def test_rule_sees_generated_ids_only():
    l = np.zeros(16, dtype=np.float32) + 1.0
    prompt_like = [3, 7, 4]
    assert np.isfinite(process(l, [], 1, 2.0)).all() and (process(l, [], 1, 2.0) == l).all()
    got = process(l, [7], 2, 2.0)                           # one generated id: penalised, nothing banned at N = 2
    assert got[7] == np.float32(0.5) and np.isfinite(got).all()
    assert banned_ids(prompt_like + [7], 2) == {4}          # what counting the prompt would ban: not the rule
    assert banned_ids([7], 2) == set()


def test_argument_validation():
    from qwen3_asr_rs_b200.inference import check_repetition, repetition_penalty_option
    assert check_repetition(0, 1.0) == (0, 1.0) and check_repetition(16, 10) == (16, 10.0)
    assert check_repetition(np.int64(3), np.float32(1.5)) == (3, 1.5)
    for n, p in ((-1, 1.0), (17, 1.0), (3.0, 1.0), (True, 1.0), ("3", 1.0), (None, 1.0),
                 (0, 0.99), (0, 10.5), (0, float("nan")), (0, float("inf")), (0, True), (0, "1.2"), (0, None)):
        with pytest.raises(ValueError):
            check_repetition(n, p)
    for p in (1.0, 1.2, 1.3, 9.75):
        assert float(repetition_penalty_option(p)) == p
    assert repetition_penalty_option(1.0) == "1"


def test_cli_flag_parsing():
    from qwen3_asr_rs_b200.__main__ import main, split_repetition
    assert split_repetition(["m", "a.wav"]) == (["m", "a.wav"], 0, 1.0)
    assert split_repetition(["m", "--no-repeat-ngram", "3", "a.wav", "--repetition-penalty=1.2"]) == (["m", "a.wav"], 3, 1.2)
    for bad in (["m", "a.wav", "--no-repeat-ngram"], ["m", "a.wav", "--repetition-penalty"],
                ["m", "a.wav", "--no-repeat-ngram", "17"], ["m", "a.wav", "--no-repeat-ngram", "-1"],
                ["m", "a.wav", "--no-repeat-ngram", "x"], ["m", "a.wav", "--repetition-penalty", "0.5"],
                ["m", "a.wav", "--repetition-penalty", "nan"], ["m", "a.wav", "--repetition-penalty", "11"]):
        assert split_repetition(bad) is None, bad
    assert main(["m", "a.wav", "--no-repeat-ngram", "99"]) == 1
    assert main(["--repetition-penalty", "0", "m", "a.wav"]) == 1


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle on the peaked tiny model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def peaked():
    """(fp32 oracle, weights) of the tiny config with an untied peaked head, seed 7: its greedy output loops."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    cfg = O.cfg_tiny()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 7, peaked_head=True)
    return O.OracleModel(cfg, w), w


CLIPS = [(0, 4.0), (1, 4.0), (2, 4.0)]


def test_oracle_breaks_the_loops(peaked):
    from qwen3_asr_rs_b200 import synth
    model, _ = peaked
    for i, s in CLIPS:
        x = synth.make_clip(i, s)
        off = rep_oracle(model, x, 0, 1.0, 48)
        on = rep_oracle(model, x, 3, 1.0, 48)
        assert repeated_ngrams(off.ids, 3) > 0, i
        assert repeated_ngrams(on.ids, 3) == 0 and on.ids != off.ids, i


def test_negative_control_n_minus_one(peaked):
    """A restatement that bans with N - 1 selects other pinned ids on the clips.  (Counting the prompt as history
    changes no id of these clips, whose outputs never contain a prompt id: test_rule_sees_generated_ids_only shows on a
    hand case that it bans other ids.)"""
    from qwen3_asr_rs_b200 import synth
    model, _ = peaked
    diff_n = 0
    for i, s in CLIPS:
        x = synth.make_clip(i, s)
        ref = rep_oracle(model, x, 2, 1.3, 32)
        k = ref.pinned()
        assert k > 0
        bad_n = rep_oracle(model, x, 1, 1.3, 32)
        diff_n += bad_n.ids[:k] != ref.ids[:k]
    assert diff_n > 0


def ctx_case(model, i):
    """(clip, context) of clip i: the context holds the first distinct ids the run generates without one, so counting
    the context as history would penalise the ids the run selects."""
    from qwen3_asr_rs_b200 import synth
    x = synth.make_clip(i, 4.0)
    ids = rep_oracle(model, x, 0, 1.0, 12).ids
    return x, list(dict.fromkeys(ids))[:6]


def test_negative_control_context_as_history(peaked):
    """A restatement that counts the context ids as history selects other pinned ids, so the GPU test that pins context
    runs against rep_oracle can tell the two apart."""
    model, _ = peaked
    diff = 0
    for i, _s in CLIPS:
        x, ctx = ctx_case(model, i)
        ref = rep_oracle(model, x, 0, 3.0, 16, context=ctx)
        k = ref.pinned()
        assert k > 0
        bad = rep_oracle(model, x, 0, 3.0, 16, context=ctx, history_of=lambda prompt, ids: ctx + list(ids))
        diff += bad.ids[:k] != ref.ids[:k]
    assert diff > 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


@pytest.fixture(scope="module")
def rep_engine(peaked):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w = peaked
    ecfg = config_tiny()
    ecfg.text.tie_word_embeddings = False
    eng = AsrInference.from_weights(ecfg, w, device=0)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def peaked64(peaked):
    import torch
    from oracle import oracle as O
    model, w = peaked
    return O.OracleModel(model.cfg, w, dtype=torch.float64)


# (label, clips (index, seconds), new tokens, options, path whose counter must move)
PATHS = [
    ("fused_single", [(0, 4.0)], 48, {}, "decode_fused_steps"),
    ("batched_b3", [(0, 4.0), (1, 4.0), (2, 4.0)], 40, {}, "decode_batch_steps"),
    ("batched_b8", [(i, 2.0 + 0.4 * i) for i in range(8)], 24, {}, "decode_batch_steps"),
    ("phases", [(1, 4.0), (2, 3.0)], 32, {"decode": "phases"}, "decode_phase_steps"),
]
RULES = [(3, 1.0), (0, 1.3), (3, 1.3)]
RESET = {"decode": "mega", "batch_step": "1"}


def _run(eng, clips, n_new, options, **kw):
    for k, v in options.items():
        eng.set_option(k, v)
    try:
        s0 = _steps(eng.stats())
        r = eng.transcribe_ids(clips, max_new_tokens=n_new, **kw)
        s1 = _steps(eng.stats())
    finally:
        for k in options:
            eng.set_option(k, RESET[k])
    return r, {k: s1[k] - s0[k] for k in s0}


def _check_path(moved, path, r):
    if path == "decode_phase_steps":
        assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0 and moved[path] > 0
    else:
        assert moved[path] == r.decode_steps and moved["decode_phase_steps"] == 0


def _lsm(l):
    f = np.isfinite(l)
    m = l[f].max()
    return l - (m + np.log(np.exp(l[f] - m).sum()))


def _records_rule(model32, model64, x, ids, lps, tops, N, theta, report, key):
    """DESIGN 2's rule on the log-probability and top-8 records at the GPU's ids: e_gpu <= R * max(e_32, floor)."""
    import torch
    from oracle import oracle as O
    with torch.no_grad():
        l32 = O.score_ids(model32, x, ids).double().numpy()
        l64 = O.score_ids(model64, x, ids).numpy()
    e_gpu = e_32 = mx = 0.0
    for i in range(len(ids)):
        p32 = _lsm(process(l32[i], ids[:i], N, theta))
        p64 = _lsm(process(l64[i], ids[:i], N, theta))
        cand = [ids[i]] if tops is None else [c for c, _ in tops[i]]
        vals = [lps[i]] if tops is None else [v for _, v in tops[i]]
        for c, v in zip(cand, vals):
            assert np.isfinite(v) and np.isfinite(p64[c]), (key, i, c, v)      # a banned id is never a candidate
            e_gpu = max(e_gpu, abs(v - p64[c]))
            e_32 = max(e_32, abs(p32[c] - p64[c]))
            mx = max(mx, abs(p64[c]))
    floor = float(np.finfo(np.float32).eps) * max(mx, 1.0)
    report[key] = {"e_gpu": e_gpu, "e_32": e_32, "ratio": e_gpu / max(e_32, floor)}
    assert e_gpu <= R_RULE * max(e_32, floor), report[key]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PATHS, ids=[p[0] for p in PATHS])
def test_defaults_are_a_no_op(rep_engine, case):
    from qwen3_asr_rs_b200 import synth
    label, sel, n_new, options, path = case
    eng = rep_engine
    clips = [synth.make_clip(i, s) for i, s in sel]
    base, m0 = _run(eng, clips, n_new, options, top_logprobs=8)
    eng.set_option("no_repeat_ngram_size", "0")
    eng.set_option("repetition_penalty", "1")
    try:
        got, m1 = _run(eng, clips, n_new, options, top_logprobs=8)
    finally:
        eng.set_option("no_repeat_ngram_size", "0")
        eng.set_option("repetition_penalty", "1")
    _check_path(m1, path, got)
    assert got.ids == base.ids
    assert np.array_equal(np.array(sum(got.logprobs, []), np.float32).view(np.uint32),
                          np.array(sum(base.logprobs, []), np.float32).view(np.uint32))
    assert got.top_logprobs == base.top_logprobs and got.eos_top_logprobs == base.eos_top_logprobs


@pytest.mark.gpu
@pytest.mark.parametrize("rule", RULES, ids=[f"N{n}-p{p}" for n, p in RULES])
@pytest.mark.parametrize("case", PATHS, ids=[p[0] for p in PATHS])
def test_greedy_rule_on_every_path(peaked, peaked64, rep_engine, report, case, rule):
    from qwen3_asr_rs_b200 import synth
    label, sel, n_new, options, path = case
    N, theta = rule
    model, _ = peaked
    eng = rep_engine
    clips = [synth.make_clip(i, s) for i, s in sel]
    off, _ = _run(eng, clips, n_new, options)
    got, moved = _run(eng, clips, n_new, options, top_logprobs=8, no_repeat_ngram_size=N, repetition_penalty=theta)
    _check_path(moved, path, got)
    pinned = 0
    for b, x in enumerate(clips):
        ids = got.ids[b]
        if N:
            assert repeated_ngrams(ids, N) == 0, (label, b)
        pinned += assert_pinned(ids, rep_oracle(model, x, N, theta, n_new), (label, b))
        if b < 2:
            _records_rule(model, peaked64, x, ids, got.logprobs[b], None, N, theta, report,
                          f"rep_{label}_N{N}_p{theta}_{b}_logprobs")
            _records_rule(model, peaked64, x, ids, None, got.top_logprobs[b], N, theta, report,
                          f"rep_{label}_N{N}_p{theta}_{b}_top8")
    assert got.ids != off.ids
    report[f"rep_{label}_N{N}_p{theta}_pinned_steps"] = pinned


@pytest.mark.gpu
@pytest.mark.parametrize("case", PATHS, ids=[p[0] for p in PATHS])
def test_sampling_rule(peaked, rep_engine, report, case):
    """No banned id is ever drawn, runs repeat bitwise, and the pinned ids are the processed draw's."""
    from qwen3_asr_rs_b200 import synth
    label, sel, n_new, options, path = case
    model, _ = peaked
    eng = rep_engine
    clips = [synth.make_clip(i, s) for i, s in sel]
    kw = dict(temperature=0.7, seed=5, no_repeat_ngram_size=2, repetition_penalty=1.2, logprobs=True)
    got, moved = _run(eng, clips, n_new, options, **kw)
    again, _ = _run(eng, clips, n_new, options, **kw)
    _check_path(moved, path, got)
    assert again.ids == got.ids
    assert np.array_equal(np.array(sum(again.logprobs, []), np.float32), np.array(sum(got.logprobs, []), np.float32))
    pinned = 0
    for b, x in enumerate(clips):
        ids = got.ids[b]
        assert repeated_ngrams(ids, 2) == 0, (label, b)
        ref = rep_oracle(model, x, 2, 1.2, n_new, temperature=0.7, seed=5, row=b)
        pinned += assert_pinned(ids, ref, (label, b))
    report[f"rep_sampling_{label}_pinned_steps"] = pinned


@pytest.mark.gpu
@pytest.mark.parametrize("case", PATHS, ids=[p[0] for p in PATHS])
def test_other_record_variants(peaked, peaked64, rep_engine, report, case):
    """Greedy with the log-probability record only, and sampling without it: the kernel variants the tests above do
    not launch."""
    from qwen3_asr_rs_b200 import synth
    label, sel, n_new, options, path = case
    model, _ = peaked
    eng = rep_engine
    clips = [synth.make_clip(i, s) for i, s in sel]
    got, moved = _run(eng, clips, n_new, options, logprobs=True, no_repeat_ngram_size=3, repetition_penalty=1.3)
    _check_path(moved, path, got)
    smp, moved_s = _run(eng, clips, n_new, options, temperature=0.7, seed=5, no_repeat_ngram_size=2, repetition_penalty=1.2)
    _check_path(moved_s, path, smp)
    for b, x in enumerate(clips):
        assert repeated_ngrams(got.ids[b], 3) == 0 and repeated_ngrams(smp.ids[b], 2) == 0, (label, b)
        assert_pinned(got.ids[b], rep_oracle(model, x, 3, 1.3, n_new), (label, b))
        assert_pinned(smp.ids[b], rep_oracle(model, x, 2, 1.2, n_new, temperature=0.7, seed=5, row=b), (label, b))
        if b < 2:
            _records_rule(model, peaked64, x, got.ids[b], got.logprobs[b], None, 3, 1.3, report,
                          f"rep_{label}_logprobs_only_{b}")


@pytest.mark.gpu
def test_beam_rule(peaked, peaked64, rep_engine, report):
    """Every n-best hypothesis is free of repeated 3-grams, its sum meets DESIGN 2's rule against the processed float64
    oracle's sum along its ids, and slots were reassigned (the ids lineage copy ran)."""
    import torch
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    model, _ = peaked
    eng = rep_engine
    clips = [synth.make_clip(i, 4.0) for i in (0, 1)]
    got = eng.transcribe_ids(clips, max_new_tokens=32, beam_size=4, no_repeat_ngram_size=3, repetition_penalty=1.2)
    stats = eng.last_beam_stats()
    assert stats["slots_reassigned"] > 0

    def processed_sum(m, x, ids, eos):
        with torch.no_grad():
            l = O.score_ids(m, x, ids).double().numpy()
        sm = sum(_lsm(process(l[i], ids[:i], 3, 1.2))[ids[i]] for i in range(len(ids)))
        return sm + (_lsm(process(l[len(ids)], ids, 3, 1.2))[eos] if eos >= 0 else 0.0)
    worst = 0.0
    for b, x in enumerate(clips):
        for ids, sm, _score, eos in got.nbest[b]:
            assert repeated_ngrams(ids, 3) == 0, (b, ids)
            s64, s32 = processed_sum(peaked64, x, ids, eos), processed_sum(model, x, ids, eos)
            floor = float(np.finfo(np.float32).eps) * max(abs(s64), 1.0) * (len(ids) + 1)   # fp32 sum of the terms
            ratio = abs(sm - s64) / max(abs(s32 - s64), floor)
            worst = max(worst, ratio)
            assert ratio <= R_RULE, (b, sm, s64, s32)
    report["rep_beam_worst_ratio"] = worst
    report["rep_beam_slots_reassigned"] = stats["slots_reassigned"]


@pytest.mark.gpu
def test_hand_over_keeps_the_rule(peaked, rep_engine, report):
    """A run that crosses the fused step's key limit mid-generation keeps the rule and the pinned ids."""
    from qwen3_asr_rs_b200 import synth
    model, _ = peaked
    eng = rep_engine
    x = synth.make_clip(3, 60.0)
    eng.transcribe_ids([x], max_new_tokens=400)                 # sizes the session: the counters below are its own
    got, moved = _run(eng, [x], 400, {}, no_repeat_ngram_size=3, repetition_penalty=1.3)
    assert moved["decode_fused_steps"] > 0 and moved["decode_phase_steps"] > 0, moved
    assert repeated_ngrams(got.ids[0], 3) == 0
    report["rep_hand_over_pinned_steps"] = assert_pinned(got.ids[0], rep_oracle(model, x, 3, 1.3, 400))


@pytest.mark.gpu
def test_composition_context(peaked, rep_engine, report):
    """With a shared context (and with one per utterance) the rule holds per utterance and the pinned ids are the
    processed oracle's with the context in its prompt; the context holds ids the run selects, so counting it as history
    would change them (test_negative_control_context_as_history)."""
    from qwen3_asr_rs_b200 import synth
    model, _ = peaked
    eng = rep_engine
    cases = [ctx_case(model, i) for i, _s in CLIPS]
    clips = [x for x, _c in cases]
    pinned = 0
    for shared in (True, False):
        ctxs = [cases[0][1]] * 3 if shared else [c for _x, c in cases]
        got = eng.transcribe_ids(clips, max_new_tokens=16, repetition_penalty=3.0, no_repeat_ngram_size=2, context_ids=ctxs)
        for b, x in enumerate(clips):
            assert repeated_ngrams(got.ids[b], 2) == 0
            pinned += assert_pinned(got.ids[b], rep_oracle(model, x, 2, 3.0, 16, context=ctxs[b]), (shared, b))
    report["rep_context_pinned_steps"] = pinned


@pytest.mark.gpu
def test_composition_segments(peaked, rep_engine, report):
    """transcribe_long's segment views keep the rule: each segment's ids are the processed oracle's on its samples."""
    from qwen3_asr_rs_b200 import synth
    model, _ = peaked
    eng = rep_engine
    pcm = np.concatenate([synth.make_clip(i, 9.0) for i in (4, 5, 6, 7)]).astype(np.float32)
    lr = eng.transcribe_long([pcm[:, None]], [16000], max_segment_s=10.0, batch=4, max_new_tokens=24,
                             no_repeat_ngram_size=3, repetition_penalty=1.2)
    segs = lr.files[0]
    assert len(segs) >= 3
    pinned = 0
    for sg in segs:
        assert repeated_ngrams(sg.ids, 3) == 0
        a, b = round(sg.start_s * 16000), round(sg.end_s * 16000)
        pinned += assert_pinned(sg.ids, rep_oracle(model, pcm[a:b], 3, 1.2, 24), (a, b))
    report["rep_segments_pinned_steps"] = pinned
