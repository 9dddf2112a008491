"""Seeded temperature sampling (session options "temperature" / "seed") and temperature fallback.

The draw (common.cuh): x0 = word 0 of Philox4x32-10 with key (seed lo, seed hi) and counter (token id, step n, row r, 0),
u = ((x0 >> 8) | 1) * 2^-24, g = -log(-log u), key = logit / T + g; the selected id is the argmax of the keys.

Reference: the oracle's float64 logits along the trajectory the float64 keys select (sampled_oracle below: the same
Philox in numpy, the same u, g in float64).  An id is pinned when the step's top-1 / top-2 key gap exceeds GAP_FLOOR
times the noise of a GPU key: the fp32 logits deviate by ~1.5e-5 * max|logit| from the oracle's (summation order),
times inv_t, plus the fp32 rounding of g (|g| < 17).  Seeds are picked from a fixed list so that every step of the
batch is pinned; the test asserts that floor for the seed it uses.
"""
import math

import numpy as np
import pytest

EOS = (151643, 151645)
LP_RTOL = 2e-4
LOGIT_NOISE = 1.5e-5          # fp32 logits vs the oracle, relative to max|logit|
G_NOISE = 4e-6                # fp32 g vs float64 g, absolute
GAP_FLOOR = 20.0
SEEDS = (0, 1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 144)


# ---------------------------------------------------------------------------------------------------------------------
# numpy Philox4x32-10 and the draw
# ---------------------------------------------------------------------------------------------------------------------
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Random123 Philox4x32-10, vectorised: ctr = 4 uint32 arrays (broadcast), key = (k0, k1) -> 4 uint32 arrays."""
    c0, c1, c2, c3 = [np.asarray(c, dtype=np.uint64) & _MASK for c in ctr]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for i in range(10):
        if i:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK
            k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
    return [x.astype(np.uint32) for x in (c0, c1, c2, c3)]


def gumbel_of_x0(x0):
    u = ((np.asarray(x0, dtype=np.uint64) >> np.uint64(8)) | np.uint64(1)).astype(np.float64) * 2.0 ** -24
    return -np.log(-np.log(u))


def gumbel(seed: int, row: int, n: int, vocab: int):
    """float64 g of every token id for (seed, row, step n)."""
    x0 = philox4x32_10((np.arange(vocab), n, row, 0), (seed & 0xFFFFFFFF, seed >> 32))[0]
    return gumbel_of_x0(x0)


class Sampled:
    def __init__(self):
        self.ids, self.logits, self.gaps = [], [], []     # logits[i] / gaps[i]: the step that selected ids[i] (or EOS)
        self.eos = False


def sampled_oracle(model, samples, temperature: float, seed: int, row: int, max_new_tokens: int):
    """oracle.transcribe_ids with the selection of the draw (temperature 0: the argmax): float64 keys l / T + g."""
    import torch
    from oracle import oracle as O
    t = model.cfg.text
    mel = O.extract_mel(samples, model.cfg.audio.num_mel_bins)
    audio = model.encode(mel)
    ids, a0 = O.build_prompt(audio.shape[0])
    S = len(ids)
    hidden = model.embed(ids).unsqueeze(0)
    hidden[0, a0:a0 + audio.shape[0], :] = audio
    pos = list(range(S))
    cos, sin = O.mrope_cos_sin([pos, pos, pos], t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved)
    cache = [None] * t.num_hidden_layers
    with torch.no_grad():
        nxt = model.decoder_forward(hidden, cos, sin, cache, O.causal_mask(S, 0), last_only=True)[:, -1, :]
        r = Sampled()
        cur = S
        for n in range(max_new_tokens):
            l = nxt[0].double().numpy()
            key = l.copy() if temperature == 0.0 else l / temperature + gumbel(seed, row, n, len(l))
            top = np.argpartition(-key, 2)[:2]
            top = top[np.argsort(-key[top])]
            tok = int(top[0])
            r.logits.append(l)
            r.gaps.append(float(key[top[0]] - key[top[1]]))
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


def _floor(refs, temperature):
    mx = max(float(np.abs(l).max()) for r in refs for l in r.logits)
    return GAP_FLOOR * (LOGIT_NOISE * mx / temperature + G_NOISE)


def pick_seed(model, clips, temperature, n_new, seeds=SEEDS):
    """The first seed whose oracle runs (row = index in the batch) have every step's key gap above the floor."""
    for seed in seeds:
        refs = [sampled_oracle(model, c, temperature, seed, b, n_new) for b, c in enumerate(clips)]
        fl = _floor(refs, temperature)
        if min(min(r.gaps) for r in refs) > fl:
            return seed, refs, fl
    raise AssertionError("no seed of the list pins every step")


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        assert tuple(int(w) for w in philox4x32_10(ctr, key)) == want


def test_gumbel_extremes_are_finite():
    g = gumbel_of_x0(np.array([0, 0xffffffff], dtype=np.uint32))
    assert np.isfinite(g).all()
    assert -2.9 < g.min() and g.max() < 16.7
    # the fp32 u of the kernels is exact: 24 significant bits
    u = ((np.array([0, 0xffffffff], np.uint64) >> np.uint64(8)) | np.uint64(1)).astype(np.float32) * np.float32(2.0 ** -24)
    assert u[0] == np.float32(2.0 ** -24) and u[1] == np.float32(1 - 2.0 ** -24)


def test_oracle_tiny_temperature_is_greedy(tiny):
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    x = synth.make_clip(70, 4.0)
    ref = O.transcribe_ids(model, x, max_new_tokens=12, lm_head_all_rows=False)
    got = sampled_oracle(model, x, 1e-6, 5, 0, 12)
    assert got.ids == ref.ids


def test_sampling_argument_validation():
    from qwen3_asr_rs_b200.inference import check_seed, check_temperature, temperature_option
    assert check_temperature(0.0) == (0.0,) and check_temperature(1) == (1.0,)
    assert check_temperature([0.0, 0.5, 1.0]) == (0.0, 0.5, 1.0) and check_temperature((1e-6, 100.0)) == (1e-6, 100.0)
    for bad in (-1.0, 1e-7, 100.5, float("nan"), float("inf"), "1", None, True, [], [0.0, -1.0]):
        with pytest.raises(ValueError):
            check_temperature(bad)
    assert check_seed(0) == 0 and check_seed(2 ** 64 - 1) == 2 ** 64 - 1 and check_seed(np.uint64(7)) == 7
    for bad in (-1, 2 ** 64, 1.0, "3", True, None):
        with pytest.raises(ValueError):
            check_seed(bad)
    for t in (1e-6, 0.3, 1.0, 100.0):
        assert float(temperature_option(t)) == t
    assert temperature_option(0.0) == "0"


class _Fake:
    """A run callable: utterance b at temperature t yields avg_logprob table[b][t] (None: stopped by the cap)."""
    def __init__(self, table):
        self.table, self.calls = table, []

    def __call__(self, idx, t):
        from qwen3_asr_rs_b200.inference import TranscribeIds
        self.calls.append((list(idx), t))
        r = TranscribeIds([[b, int(t * 10)] for b in idx], {"decode": 1.0}, 1, 1)
        r.logprobs = [[self.table[b][t] if self.table[b][t] is not None else -0.1] * 2 for b in idx]
        r.eos_logprobs = [None if self.table[b][t] is None else self.table[b][t] for b in idx]
        return r


def test_fallback_policy():
    from qwen3_asr_rs_b200.inference import temperature_fallback
    table = [{0.0: -0.2, 0.5: -0.1, 1.0: -0.1},     # accepted at once
             {0.0: -1.5, 0.5: -0.3, 1.0: -0.1},     # below the threshold, accepted at 0.5
             {0.0: None, 0.5: None, 1.0: None},     # capped every time: keeps the last attempt
             {0.0: -2.0, 0.5: -1.2, 1.0: -0.5}]     # accepted at 1.0
    f = _Fake(table)
    kept, temps, runs = temperature_fallback(f, 4, (0.0, 0.5, 1.0), -1.0)
    assert f.calls == [([0, 1, 2, 3], 0.0), ([1, 2, 3], 0.5), ([2, 3], 1.0)]
    assert temps == [0.0, 0.5, 1.0, 1.0] and len(runs) == 3
    assert [k[0].ids[k[1]] for k in kept] == [[0, 0], [1, 5], [2, 10], [3, 10]]
    # threshold None: only the capped utterance runs again
    f = _Fake(table)
    kept, temps, _ = temperature_fallback(f, 4, (0.0, 0.5), None)
    assert f.calls == [([0, 1, 2, 3], 0.0), ([2], 0.5)] and temps == [0.0, 0.0, 0.5, 0.0]
    # nothing left to re-run: the schedule stops early
    f = _Fake([{0.0: -0.1, 1.0: -0.1}])
    temperature_fallback(f, 1, (0.0, 1.0), -1.0)
    assert f.calls == [([0], 0.0)]


def test_sampling_fields_default_to_none():
    from qwen3_asr_rs_b200.inference import TranscribeIds, TranscribeResult
    assert TranscribeIds([[1]], {}, 0, 0).temperatures is None
    assert TranscribeResult("t", "l", "r", [1]).temperature is None


def test_cli_sampling_flag_parsing():
    from qwen3_asr_rs_b200.__main__ import main, parse_args, split_sampling, split_top_logprobs
    assert split_sampling(["m", "a.wav"]) == (["m", "a.wav"], None, 0)
    assert split_sampling(["m", "a.wav", "--temperature", "0.7", "--seed", "9"]) == (["m", "a.wav"], 0.7, 9)
    assert split_sampling(["--seed=3", "m", "--temperature=0,0.4,1", "a.wav", "english"]) == \
        (["m", "a.wav", "english"], (0.0, 0.4, 1.0), 3)
    for bad in (["m", "a.wav", "--temperature"], ["m", "a.wav", "--seed"], ["m", "a.wav", "--temperature", "-1"],
                ["m", "a.wav", "--temperature", "x"], ["m", "a.wav", "--temperature", "nan"],
                ["m", "a.wav", "--seed", "-3"], ["m", "a.wav", "--seed", "18446744073709551616"],
                ["m", "a.wav", "--temperature", "0,,1"]):
        assert split_sampling(bad) is None, bad
    rest, t, seed = split_sampling(["m", "a.wav", "--temperature", "1", "english", "--logprobs", "--top-logprobs", "2"])
    rest, k = split_top_logprobs(rest)
    assert (t, seed, k) == (1.0, 0, 2) and parse_args(rest) == ("m", "a.wav", "english", True)
    assert main(["m", "a.wav", "--temperature", "200"]) == 1
    assert main(["--seed", "1", "m"]) == 1


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


@pytest.fixture(scope="module")
def smp_engine(tiny):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    yield eng
    eng.close()


# (label, clips (index, seconds), new tokens, options, path whose counter must move): those of test_top_logprobs.py
PATHS = [
    ("fused_single", [(70, 4.0)], 48, {}, "decode_fused_steps"),
    ("fused_per_seq_b5", [(80 + i, s) for i, s in enumerate([2.5, 9.1, 5.0, 1.2, 3.3])], 16, {"batch_step": "0"}, "decode_fused_steps"),
    ("batched_nb8", [(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9])], 14, {}, "decode_batch_steps"),
    ("batched_nb16", [(200 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9, 5.3, 1.4, 2.8])], 10, {}, "decode_batch_steps"),
    ("phases", [(71, 12.3), (72, 0.8)], 24, {"decode": "phases"}, "decode_phase_steps"),
]
CASES = [(p, 1.0) for p in PATHS] + [(PATHS[0], 0.7), (PATHS[2], 0.7), (PATHS[4], 0.7)]


def _configure(eng, temperature, seed):
    from qwen3_asr_rs_b200.inference import temperature_option
    eng.set_option("temperature", temperature_option(temperature))
    eng.set_option("seed", str(seed))


def _moved(eng, fn):
    s0 = _steps(eng.stats())
    r = fn()
    s1 = _steps(eng.stats())
    return r, {k: s1[k] - s0[k] for k in s0}


@pytest.mark.gpu
@pytest.mark.parametrize("case,temperature", CASES, ids=[f"{c[0]}-T{t}" for c, t in CASES])
def test_sampling_on_every_path(tiny, smp_engine, report, case, temperature):
    """Ids equal the oracle's sampled ids; path counters equal a greedy run's; runs are bitwise repeatable; another
    seed changes at least one utterance."""
    from qwen3_asr_rs_b200 import synth
    label, sel, n_new, options, path = case
    _, _, model = tiny
    eng = smp_engine
    clips = [synth.make_clip(i, s) for i, s in sel]
    seed, refs, floor = pick_seed(model, clips, temperature, n_new)
    for k, v in options.items():
        eng.set_option(k, v)
    try:
        eng.transcribe_ids(clips, max_new_tokens=n_new)                                  # warm-up: session, graphs
        greedy, m_greedy = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=n_new))
        # configured (setting an option drops the captured per-phase graph, whose capture counts one step): the calls
        # below switch nothing
        _configure(eng, temperature, seed)
        eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=temperature, seed=seed)
        got, m_got = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=temperature, seed=seed))
        again = eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=temperature, seed=seed)
        other = eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=temperature, seed=seed + 1000)
    finally:
        _configure(eng, 0.0, 0)
        for k in options:
            eng.set_option(k, {"decode": "mega", "batch_step": "1"}[k])
    assert got.ids == [r.ids for r in refs], (label, seed)
    assert got.temperatures == [temperature] * len(clips) and greedy.temperatures is None
    if [len(i) for i in got.ids] == [len(i) for i in greedy.ids]:
        assert m_got == m_greedy
    if path == "decode_phase_steps":         # the per-phase path replays a captured graph: its counter counts the capture
        assert m_got["decode_fused_steps"] == 0 and m_got["decode_batch_steps"] == 0
        assert got.kernels_launched > 2 * got.decode_steps
    else:
        assert m_got[path] == got.decode_steps and m_got["decode_phase_steps"] == 0
    assert again.ids == got.ids and other.ids != got.ids
    report[f"sampling_{label}_T{temperature}_seed"] = seed
    report[f"sampling_{label}_T{temperature}_min_gap_over_floor"] = min(min(r.gaps) for r in refs) / floor


@pytest.mark.gpu
def test_sampling_path_counters_match_greedy(smp_engine):
    """Same shapes (every utterance runs to the cap): the decode path and its counters are those of a greedy run."""
    from qwen3_asr_rs_b200 import synth
    eng = smp_engine
    clips = [synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7, 4.9])]
    for opts in ({}, {"decode": "phases"}, {"batch_step": "0"}):
        for k, v in opts.items():
            eng.set_option(k, v)
        try:
            eng.transcribe_ids(clips, max_new_tokens=6)
            g, mg = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=6))
            _configure(eng, 1.0, 4)
            eng.transcribe_ids(clips, max_new_tokens=6)
            s, ms = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=6, temperature=1.0, seed=4))
        finally:
            _configure(eng, 0.0, 0)
            for k in opts:
                eng.set_option(k, {"decode": "mega", "batch_step": "1"}[k])
        if [len(i) for i in g.ids] == [len(i) for i in s.ids]:
            assert mg == ms and g.decode_steps == s.decode_steps, opts


@pytest.mark.gpu
def test_sampling_across_fused_step_limit(tiny, smp_engine, report):
    """60 s prompt + 400 tokens: the draw's step index continues across the hand-over to the per-phase path."""
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    x = synth.make_clip(302, 60.0)
    n_new = 400
    seed, refs, floor = pick_seed(model, [x], 1.0, n_new, seeds=SEEDS[:4])
    smp_engine.transcribe_ids([x], max_new_tokens=n_new)          # sizes the session: its counters start at zero
    got, moved = _moved(smp_engine, lambda: smp_engine.transcribe_ids([x], max_new_tokens=n_new, temperature=1.0, seed=seed))
    assert got.ids[0] == refs[0].ids
    if len(got.ids[0]) > 300:
        assert moved["decode_fused_steps"] > 0 and moved["decode_phase_steps"] > 0
    report["sampling_long_crossing_tokens"] = len(got.ids[0])


@pytest.mark.gpu
def test_sampling_tiny_temperature_is_greedy(smp_engine):
    """T = 1e-6 reproduces the greedy ids; a greedy run after sampled runs reproduces ids and logprobs bitwise."""
    from qwen3_asr_rs_b200 import synth
    eng = smp_engine
    for clips, opts in (([synth.make_clip(70, 4.0)], {}), ([synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7])], {}),
                        ([synth.make_clip(71, 12.3), synth.make_clip(72, 0.8)], {"decode": "phases"})):
        for k, v in opts.items():
            eng.set_option(k, v)
        try:
            g = eng.transcribe_ids(clips, max_new_tokens=24, logprobs=True)
            t0 = eng.transcribe_ids(clips, max_new_tokens=24, temperature=1e-6, seed=11)
            eng.transcribe_ids(clips, max_new_tokens=24, temperature=1.0, seed=11, logprobs=True)
            g2 = eng.transcribe_ids(clips, max_new_tokens=24, logprobs=True)
        finally:
            for k in opts:
                eng.set_option(k, "mega")
        assert t0.ids == g.ids
        assert g2.ids == g.ids and g2.logprobs == g.logprobs and g2.eos_logprobs == g.eos_logprobs


@pytest.mark.gpu
def test_sampling_distribution_of_token0(smp_engine, report):
    """Token 0 over 16 rows x 256 seeds (stage API, per-phase lm_head in sub-batches of 8) against softmax(l / T) of the
    GPU's own returned logits: chi-square with bins of expected count < 5 pooled."""
    from scipy.stats import chisquare
    from qwen3_asr_rs_b200 import synth
    eng = smp_engine
    x = synth.make_clip(60, 3.0)
    rows, n_seeds = 16, 256
    eng.mel([x] * rows)
    eng.encode()
    _, lg = eng.prefill()
    l = lg[0].astype(np.float64)
    assert np.array_equal(lg[0], lg[rows - 1])

    def eff(T):                                      # effective number of tokens exp(entropy) of softmax(l / T)
        p = np.exp((l - l.max()) / T); p /= p.sum()
        return math.exp(-(p[p > 0] * np.log(p[p > 0])).sum())
    lo, hi = 1e-3, 100.0
    for _ in range(60):
        mid = math.sqrt(lo * hi)
        lo, hi = (mid, hi) if eff(mid) < 30 else (lo, mid)
    T = hi
    p = np.exp((l - l.max()) / T); p /= p.sum()
    counts = {}
    try:
        eng.set_option("temperature", repr(T))
        for seed in range(n_seeds):
            eng.set_option("seed", str(seed))
            eng.prefill(want_logits=False)
            for ids in eng.generate(1):
                assert len(ids) <= 1
                tok = ids[0] if ids else -1
                counts[tok] = counts.get(tok, 0) + 1
    finally:
        eng.set_option("temperature", "0"); eng.set_option("seed", "0")
    n = rows * n_seeds
    assert sum(counts.values()) == n
    # bins: each non-EOS id with expected count >= 5, one bin for both EOS ids (a sampled EOS appends nothing), the rest
    # pooled
    obs, exp_ = [float(counts.get(-1, 0))], [float(p[list(EOS)].sum() * n)]
    pool_o = pool_e = 0.0
    for v in np.argsort(-p):
        if int(v) in EOS:
            continue
        e, o = p[v] * n, counts.get(int(v), 0)
        if e >= 5:
            obs.append(o); exp_.append(e)
        else:
            pool_o += o; pool_e += e
    obs.append(pool_o); exp_.append(pool_e)
    obs, exp_ = np.array(obs, float), np.array(exp_, float)
    keep = exp_ >= 5
    obs = np.append(obs[keep], obs[~keep].sum()); exp_ = np.append(exp_[keep], exp_[~keep].sum())
    if exp_[-1] < 5:
        obs[-2] += obs[-1]; exp_[-2] += exp_[-1]; obs, exp_ = obs[:-1], exp_[:-1]
    res = chisquare(obs, exp_ * (obs.sum() / exp_.sum()))
    report["sampling_token0_chi2_p"] = float(res.pvalue)
    report["sampling_token0_temperature"] = T
    report["sampling_token0_bins"] = len(obs)
    assert len(obs) >= 10 and res.pvalue > 1e-4


def _eos_model(tiny, k, scale=1.5):
    """The EOS-row construction of test_logprobs.py (EOS embedding row = scale x that of the k-th generated id)."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    cfg, w, base = tiny
    x = synth.make_clip(90, 1.5)
    r = O.transcribe_ids(base, x, max_new_tokens=6)
    e = w["thinker.model.embed_tokens.weight"].float().clone()
    e[151645] = e[r.ids[k]] * scale
    w2 = dict(w)
    w2["thinker.model.embed_tokens.weight"] = e.bfloat16()
    return w2, O.OracleModel(cfg, w2), x


def _lsm(l):
    m = l.max()
    return l - m - math.log(np.exp(l - m).sum())


@pytest.mark.gpu
def test_sampling_logprobs(tiny, report):
    """Under sampling the record holds the model's own log-probability of the sampled id: within 2e-4 * max|logit| of
    the float64 log_softmax at that id, a sampled EOS included; NaN for the EOS of a capped sequence."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    w2, model, x = _eos_model(tiny, 2)
    y = synth.make_clip(92, 3.0)
    n_new = 12
    seed = T = None
    # the first (T, seed) under which x ends on a sampled EOS and y runs into the cap, every step pinned
    for t in (0.5, 0.3, 0.2, 0.1):
        for s in SEEDS:
            rx = sampled_oracle(model, x, t, s, 0, n_new)
            ry = sampled_oracle(model, y, t, s, 1, n_new)
            if rx.eos and not ry.eos and min(rx.gaps + ry.gaps) > _floor([rx, ry], t):
                seed, T = s, t
                break
        if seed is not None:
            break
    assert seed is not None
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    try:
        worst = 0.0
        for opts in ({}, {"decode": "phases"}, {"batch_step": "0"}):
            for k, v in opts.items():
                eng.set_option(k, v)
            got = eng.transcribe_ids([x, y], max_new_tokens=n_new, temperature=T, seed=seed, logprobs=True)
            for k in opts:
                eng.set_option(k, {"decode": "mega", "batch_step": "1"}[k])
            assert got.ids == [rx.ids, ry.ids], opts
            for b, ref in ((0, rx), (1, ry)):
                mx = max(float(np.abs(l).max()) for l in ref.logits)
                want = [_lsm(ref.logits[i])[t] for i, t in enumerate(ref.ids)]
                worst = max([worst] + [abs(a - c) / mx for a, c in zip(got.logprobs[b], want)])
                if ref.eos:
                    tok = int(np.argmax(ref.logits[-1] / T + gumbel(seed, b, len(ref.ids), len(ref.logits[-1]))))
                    worst = max(worst, abs(got.eos_logprobs[b] - _lsm(ref.logits[-1])[tok]) / mx)
                else:
                    assert got.eos_logprobs[b] is None
    finally:
        eng.close()
    report["sampling_logprobs_eos_temperature"] = T
    report["sampling_logprobs_max_rel_err"] = worst
    assert worst <= LP_RTOL


@pytest.mark.gpu
def test_sampling_logprobs_of_non_argmax_ids(tiny, smp_engine, report):
    """T = 1 on the batched path: the record at ids that are not the argmax of their step, (l_sel - M) - log S, within
    2e-4 * max|logit| of the float64 log_softmax at the sampled id."""
    from qwen3_asr_rs_b200 import synth
    _, _, model = tiny
    label, sel, n_new, _, _ = PATHS[2]
    clips = [synth.make_clip(i, s) for i, s in sel]
    seed, refs, _ = pick_seed(model, clips, 1.0, n_new)
    got = smp_engine.transcribe_ids(clips, max_new_tokens=n_new, temperature=1.0, seed=seed, logprobs=True)
    assert got.ids == [r.ids for r in refs]
    worst, off_argmax = 0.0, 0
    for b, ref in enumerate(refs):
        mx = max(float(np.abs(l).max()) for l in ref.logits)
        for i, t in enumerate(ref.ids):
            off_argmax += int(t != int(np.argmax(ref.logits[i])))
            worst = max(worst, abs(got.logprobs[b][i] - _lsm(ref.logits[i])[t]) / mx)
    report["sampling_logprobs_t1_max_rel_err"] = worst
    report["sampling_logprobs_t1_non_argmax_ids"] = off_argmax
    assert off_argmax > 0 and worst <= LP_RTOL


@pytest.mark.gpu
def test_sampling_errors_and_latching(tiny):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    from qwen3_asr_rs_b200._lib import AsrbError
    _, w, model = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    x = synth.make_clip(301, 1.7)
    try:
        eng.mel([x])
        for key, bads in (("temperature", ("-1", "+1", "nan", "inf", "1x", "", " 1", "1e-7", "100.5", "0x1p0")),
                          ("seed", ("-1", "+1", "18446744073709551616", "1.5", "", " 3", "x"))):
            for bad in bads:
                with pytest.raises(AsrbError) as e:
                    eng.set_option(key, bad)
                assert e.value.code == 1, (key, bad)
        eng.set_option("seed", "18446744073709551615"); eng.set_option("seed", "0")
        eng.set_option("temperature", "1"); eng.set_option("top_logprobs", "2")
        with pytest.raises(AsrbError) as e:                  # refused before any work by every prefill call
            eng.transcribe_ids([x], max_new_tokens=4)
        assert e.value.code == 1
        eng.mel([x]); eng.encode()
        with pytest.raises(AsrbError) as e:
            eng.prefill(want_logits=False)
        assert e.value.code == 1
        with pytest.raises(AsrbError) as e:
            eng.transcribe_pcm([(x * 32767).astype(np.int16)], [16000], max_new_tokens=4)
        assert e.value.code == 1
        with pytest.raises(ValueError):
            eng.transcribe_ids([x], max_new_tokens=4, temperature=1.0, top_logprobs=2)
        eng.set_option("top_logprobs", "0"); eng.set_option("temperature", "0")
        # latched at the prefill: a change before generate affects the next run only
        greedy = eng.transcribe_ids([x], max_new_tokens=12)
        eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
        eng.set_option("temperature", "1"); eng.set_option("seed", "3")
        assert eng.generate(12) == greedy.ids
        ref = sampled_oracle(model, x, 1.0, 3, 0, 12)
        eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
        eng.set_option("temperature", "0")
        sampled = eng.generate(12)
        if min(ref.gaps) > _floor([ref], 1.0):
            assert sampled[0] == ref.ids
    finally:
        eng.close()


@pytest.mark.gpu
def test_temperature_fallback_end_to_end(tiny, report):
    """Schedule (0, 1) on a model where clip x ends on EOS and clip y runs into the cap.  Threshold below x's greedy
    avg_logprob: x keeps its greedy ids bitwise, y (capped) falls back and equals a direct T = 1 run of that subset.
    Threshold above it: both fall back, and equal a direct T = 1 run of the batch."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    from qwen3_asr_rs_b200.inference import avg_logprob
    w2, _, x = _eos_model(tiny, 2)
    y = synth.make_clip(92, 3.0)
    clips, n_new = [x, y], 12
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    try:
        g = eng.transcribe_ids(clips, max_new_tokens=n_new, logprobs=True)
        assert g.eos_logprobs[0] is not None and g.eos_logprobs[1] is None
        avg_x = avg_logprob(g.logprobs[0], g.eos_logprobs[0])
        low = eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=(0.0, 1.0), seed=6, logprob_threshold=avg_x - 0.5)
        direct_y = eng.transcribe_ids([y], max_new_tokens=n_new, temperature=1.0, seed=6)
        high = eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=[0.0, 1.0], seed=6, logprob_threshold=avg_x + 0.5)
        direct = eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=1.0, seed=6)
        none = eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=(0.0, 1.0), seed=6, logprob_threshold=None)
    finally:
        eng.close()
    assert low.ids == [g.ids[0], direct_y.ids[0]] and low.temperatures == [0.0, 1.0]
    assert low.logprobs[0] == g.logprobs[0]
    assert high.ids == direct.ids and high.temperatures == [1.0, 1.0]
    assert none.ids == low.ids and none.temperatures == [0.0, 1.0]      # no threshold: only the capped one re-runs
    report["sampling_fallback_avg_logprob_x"] = avg_x


def _full(cfg_fn, ecfg_fn, seed_w):
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    cfg = cfg_fn()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, seed_w, peaked_head=True)
    ecfg = ecfg_fn()
    ecfg.text.tie_word_embeddings = False
    return cfg, w, ecfg, O.OracleModel(cfg, w)


@pytest.mark.gpu
def test_full_size_0p6b_sampling(report):
    """0.6B dims: batch 1 (fused single-sequence step) and batch 8 (batched step), 30 s clips, 8 new tokens."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth
    cfg, w, ecfg, model = _full(O.cfg_0p6b, config_0p6b, 1)
    n_new = 8
    clips = [synth.make_clip(i, 30.0) for i in (1, 3, 4, 6, 7, 8, 10, 17)]
    seed, refs, floor = pick_seed(model, clips, 1.0, n_new, seeds=SEEDS[:3])
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        b8, m8 = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=n_new, temperature=1.0, seed=seed))
        b1, m1 = _moved(eng, lambda: eng.transcribe_ids(clips[:1], max_new_tokens=n_new, temperature=1.0, seed=seed))
    finally:
        eng.close()
    assert m8["decode_batch_steps"] == b8.decode_steps and m1["decode_fused_steps"] == b1.decode_steps
    assert b8.ids == [r.ids for r in refs] and b1.ids[0] == refs[0].ids
    report["sampling_full_0p6b_seed"] = seed


@pytest.mark.gpu
def test_full_size_1p7b_sampling(report):
    """1.7B dims (K = 2048 lm_head form of the fused step), 8 new tokens."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_1p7b, synth
    cfg, w, ecfg, model = _full(O.cfg_1p7b, config_1p7b, 3)
    x = synth.make_clip(7, 30.0)
    n_new = 8
    seed, refs, floor = pick_seed(model, [x], 1.0, n_new, seeds=SEEDS[:3])
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        got, m = _moved(eng, lambda: eng.transcribe_ids([x], max_new_tokens=n_new, temperature=1.0, seed=seed))
    finally:
        eng.close()
    assert m["decode_fused_steps"] == got.decode_steps and m["decode_phase_steps"] == 0
    assert got.ids[0] == refs[0].ids
    report["sampling_full_1p7b_seed"] = seed
