"""Beam search (session options "beam_size" / "length_penalty"), spec in include/asr_b200.h.

Reference: `beam_oracle` below, a float64 beam search on the oracle's logits with one KV cache per hypothesis and the
same walk, slot and ranking rules (`walk` / `assign_slots` / `rank`, also checked on hand-made records).  The GPU sums
differ from the oracle's by fp32 noise (~1.5e-5 * max|logit| per log-probability, accumulated over the steps), so a run
is compared only when every selection boundary clears GAP_FLOOR times that noise: adjacent candidate sums up to and
just past the walk's stop, the K+2 cut of each record, and adjacent final scores.  Clips come from fixed lists; the
test asserts the floor for the ones it uses.  The noise is the worst per-value deviation of the TOPK records, summed
linearly over the steps, so a floor of 2 already bounds the accumulated error twice over; the synthetic models' beam
candidates are too close together for a larger floor to leave clips to test.  Runs too long to pin (the 400-token run,
the 1.7B dims at 24 tokens) check self-consistency instead: sums against the reported log-probabilities, repeatability,
paths.
"""
import math

import numpy as np
import pytest

EOS = (151643, 151645)
LP_RTOL = 2e-4
LOGIT_NOISE = 1.5e-5
GAP_FLOOR = 2.0


# ---------------------------------------------------------------------------------------------------------------------
# the rules (shared by the CPU tests and the oracle)
# ---------------------------------------------------------------------------------------------------------------------
def walk(records, sums, K, nfin):
    """records[r] = [(id, lp), ...] of the alive beam of rank r (best first), sums[r] its sum.  Returns (alive, fresh,
    order, stop): alive = K (parent rank, id, lp, sum), fresh = admitted EOS (parent rank, id, lp, sum) in walk order,
    order = all candidates sorted, stop = number of candidates walked."""
    cands = []
    for r, rec in enumerate(records):
        for j, (i, lp) in enumerate(rec[:K + 2]):
            cands.append((sums[r] + lp, r, j, i, lp))
    cands.sort(key=lambda c: (-c[0], c[1], c[2]))
    alive, new_fin, q = [], [], 0
    while q < len(cands) and len(alive) < K:
        s, r, j, i, lp = cands[q]
        (new_fin if i in EOS else alive).append((r, i, lp, s))
        q += 1
    fresh = new_fin[:max(0, K - nfin)]
    return alive, fresh, cands, q


def assign_slots(parents, K, first=False):
    """parents[r] = beam index of new beam r's parent (all 0 at token 0).  Returns dst[r] = beam index of its slot."""
    has_child = set(parents)
    if first:
        has_child = {0}
    dst, claimed = [None] * K, set()
    for r, p in enumerate(parents):
        if p not in claimed:
            dst[r] = p
            claimed.add(p)
    free = [j for j in range(K) if j not in has_child]
    it = iter(free)
    for r in range(K):
        if dst[r] is None:
            dst[r] = next(it)
    return dst


def score(sm, n, alpha):
    p = float(max(n, 1)) if alpha is None else ((5.0 + n) / 6.0) ** alpha
    return float(sm) / p


def rank(hyps, alpha):
    """hyps in admission order as (n, sum): indices by (score descending, admission order)."""
    sc = [score(s, n, alpha) for n, s in hyps]
    return sorted(range(len(hyps)), key=lambda i: (-sc[i], i))


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_walk_two_eos_at_top_and_token0():
    K = 3
    rec = [(151645, -0.1), (151643, -0.2), (10, -0.3), (11, -0.4), (12, -0.5), (13, -0.6), (14, -0.7), (15, -0.8)]
    alive, fresh, cands, stop = walk([rec], [0.0], K, 0)
    assert [a[1] for a in alive] == [10, 11, 12] and [f[1] for f in fresh] == [151645, 151643]
    assert stop == 5 and len(cands) == K + 2              # only the first K + 2 entries are candidates
    assert assign_slots([0, 0, 0], K, first=True) == [0, 1, 2]
    # a full finished list admits nothing more
    _, fresh, _, _ = walk([rec], [0.0], K, 2)
    assert [f[1] for f in fresh] == [151645]
    _, fresh, _, _ = walk([rec], [0.0], K, 3)
    assert fresh == []


def test_walk_both_eos_on_top_of_every_beam():
    """K = 6 beams whose records all start with both EOS ids: the walk passes 2 * K = 12 EOS candidates before K beams
    are alive, and only the first K - nfin of them are admitted, in walk order."""
    K = 6
    recs = [[(151643, -0.1 - 0.01 * r), (151645, -0.2 - 0.01 * r)] + [(100 + 10 * r + j, -1.0 - 0.01 * r - 0.1 * j)
                                                                      for j in range(6)] for r in range(K)]
    sums = [-1.0 - 0.001 * r for r in range(K)]
    alive, fresh, cands, stop = walk(recs, sums, K, 0)
    walked_eos = [c for c in cands[:stop] if c[3] in EOS]
    assert len(walked_eos) == 2 * K and len(alive) == K
    assert [(f[0], f[1]) for f in fresh] == [(c[1], c[3]) for c in walked_eos[:K]]
    _, fresh, _, _ = walk(recs, sums, K, 4)
    assert [(f[0], f[1]) for f in fresh] == [(c[1], c[3]) for c in walked_eos[:2]]


def test_walk_ties_and_childless_beam():
    K = 3
    recs = [[(1, -1.0), (2, -2.0), (3, -3.0), (4, -4.0), (5, -5.0)],
            [(6, -0.5), (7, -0.6), (8, -9.0), (9, -9.5), (16, -9.6)],
            [(17, -5.0), (18, -6.0), (19, -7.0), (20, -8.0), (21, -9.0)]]
    sums = [-1.0, -1.5, -1.5]
    alive, fresh, cands, _ = walk(recs, sums, K, 0)
    # (rank 0, id 1) sums -2.0, (rank 1, id 6) -2.0: equal sums -> lower parent rank first
    assert [(a[0], a[1]) for a in alive] == [(0, 1), (1, 6), (1, 7)]
    dst = assign_slots([a[0] for a in alive], K)
    assert dst == [0, 1, 2]                                # beam 2 had no child: its slot takes rank 2
    moved = [(p, d) for p, d in zip([a[0] for a in alive], dst) if p != d]
    assert moved == [(1, 2)]
    srcs, dsts = {p for p, _ in moved}, {d for _, d in moved}
    assert not (srcs & dsts)


def test_slot_rule_sources_and_destinations_disjoint():
    rng = np.random.default_rng(0)
    for _ in range(500):
        K = int(rng.integers(2, 7))
        parents = sorted(int(x) for x in rng.integers(0, K, size=K))
        rng.shuffle(parents)
        dst = assign_slots(parents, K)
        assert sorted(dst) == list(range(K))
        best = {}
        for r, p in enumerate(parents):
            best.setdefault(p, r)
        for r, p in enumerate(parents):
            assert (dst[r] == p) == (best[p] == r)
        srcs = {p for r, p in enumerate(parents) if dst[r] != p}
        dsts = {dst[r] for r, p in enumerate(parents) if dst[r] != p}
        assert not (srcs & dsts) and not (dsts & set(parents))


def test_host_ranking_and_length_penalty():
    from qwen3_asr_rs_b200.inference import beam_score, rank_hypotheses
    assert beam_score(-6.0, 3, None) == -2.0 and beam_score(-6.0, 0, None) == -6.0
    assert beam_score(-6.0, 7, 1.0) == -6.0 / 2.0 and beam_score(-3.0, 1, 0.0) == -3.0
    assert math.isclose(beam_score(-4.0, 4, 0.6), -4.0 / (1.5 ** 0.6), rel_tol=0, abs_tol=0)
    hyps = [(2, -2.0), (4, -4.0), (1, -0.5), (3, -9.0)]     # scores -1, -1, -0.5, -3: a tie keeps admission order
    assert rank_hypotheses(hyps, None) == [2, 0, 1, 3] == rank(hyps, None)
    assert rank_hypotheses(hyps, 1.0) == rank(hyps, 1.0)
    assert rank_hypotheses([(0, -1.0), (5, -1.0)], 0.0) == [0, 1]


def test_beam_argument_validation():
    from qwen3_asr_rs_b200.inference import AsrInference, check_beam, length_penalty_option
    assert check_beam(1, None) == (1, None) and check_beam(6, 0) == (6, 0.0) and check_beam(np.int64(3), 10.0) == (3, 10.0)
    for bad in ((0, None), (7, None), (True, None), (2.0, None), ("2", None), (2, -0.1), (2, 10.5), (2, float("nan")),
                (2, True), (2, "1")):
        with pytest.raises(ValueError):
            check_beam(*bad)
    assert length_penalty_option(None) == "none" and float(length_penalty_option(0.6)) == 0.6
    once = lambda *a: pytest.fail("must refuse before any run")   # noqa: E731
    for kw in (dict(temperature=0.5), dict(top_logprobs=2), dict(temperature=(0.0, 1.0), top_logprobs=1)):
        args = dict(temperature=0.0, top_logprobs=0)
        args.update(kw)
        with pytest.raises(ValueError):
            AsrInference._sampled(None, 1, once, args["temperature"], 0, -1.0, False, args["top_logprobs"], 4, None)


def test_cli_beam_flag_parsing():
    from qwen3_asr_rs_b200.__main__ import main, split_beam
    assert split_beam(["m", "a.wav"]) == (["m", "a.wav"], 1, None)
    assert split_beam(["m", "--beam-size", "5", "a.wav", "--length-penalty=0.6"]) == (["m", "a.wav"], 5, 0.6)
    for bad in (["m", "a.wav", "--beam-size"], ["m", "a.wav", "--beam-size", "7"], ["m", "a.wav", "--beam-size", "0"],
                ["m", "a.wav", "--beam-size", "x"], ["m", "a.wav", "--length-penalty", "11"],
                ["m", "a.wav", "--length-penalty"], ["m", "a.wav", "--beam-size", "-2"]):
        assert split_beam(bad) is None, bad
    assert main(["m", "a.wav", "--beam-size", "9"]) == 1
    assert main(["m", "a.wav", "--beam-size", "4", "--temperature", "0.5"]) == 1
    assert main(["m", "a.wav", "--beam-size", "4", "--top-logprobs", "2"]) == 1


def test_nbest_fields_default_to_none():
    from qwen3_asr_rs_b200.inference import TranscribeIds, TranscribeResult
    assert TranscribeIds([[1]], {}, 0, 0).nbest is None
    assert TranscribeResult("t", "l", "r", [1]).nbest is None


# ---------------------------------------------------------------------------------------------------------------------
# float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
class BeamRef:
    def __init__(self):
        self.hyps = []           # ranked (ids, sum, score, eos_id)
        self.gaps = []           # (gap, steps accumulated) of every selection boundary
        self.mx = 0.0            # max |logit| seen
        self.reassigned = 0
        self.reorder_positions = 0
        self.expand_positions = 0
        self.steps = 0           # beam steps (decode steps) executed


def _record(l):
    top = np.argpartition(-l, 8)[:9]
    top = sorted(top.tolist(), key=lambda i: (-l[i], i))
    m = l.max()
    lse = m + math.log(np.exp(l - m).sum())
    return [(int(i), float(l[i] - lse)) for i in top[:8]], [float(l[i]) for i in top]


def beam_oracle(model, samples, K, max_new_tokens, alpha=None):
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
    ref = BeamRef()
    with torch.no_grad():
        l0 = model.decoder_forward(hidden, cos, sin, cache, O.causal_mask(S, 0), last_only=True)[:, -1, :][0].double().numpy()
        # alive beams in rank order: dict(ids, sum, logits, cache, nodes, beam)
        beams = [dict(ids=[], sum=0.0, logits=l0, cache=cache, nodes=[], beam=0)]
        fin = []                 # admission order: (ids, sum, eos)
        node = 0
        first, step = True, 0
        while True:
            recs, cuts = [], []
            for bm in beams:
                rec, lg = _record(bm["logits"])
                recs.append(rec)
                ref.mx = max(ref.mx, float(np.abs(bm["logits"]).max()))
                ref.gaps.append((lg[K + 1] - lg[K + 2], 0))      # the K+2 cut of the record
            alive, fresh, cands, stop = walk(recs, [b["sum"] for b in beams], K, len(fin))
            for q in range(min(stop, len(cands) - 1)):
                ref.gaps.append((cands[q][0] - cands[q + 1][0], step + 1))
            for r, i, lp, s in fresh:
                fin.append((list(beams[r]["ids"]), s, i))
            if len(fin) >= K:
                break
            parents = [beams[r]["beam"] for r, _, _, _ in alive]
            dst = assign_slots(parents, K, first=first)
            new = []
            for (r, i, lp, s), d in zip(alive, dst):
                par = beams[r]
                if d != par["beam"]:
                    if first:
                        ref.expand_positions += S
                    else:
                        old = next(b for b in beams if b["beam"] == d)
                        common = 0
                        while common < len(old["nodes"]) and common < len(par["nodes"]) and old["nodes"][common] == par["nodes"][common]:
                            common += 1
                        ref.reassigned += 1
                        ref.reorder_positions += len(par["nodes"]) - common
                new.append(dict(ids=par["ids"] + [i], sum=s, parent=par, beam=d, nodes=par["nodes"] + [node], tok=i))
                node += 1
            first = False
            if len(new[0]["ids"]) >= max_new_tokens:
                beams = new
                break
            for bm in new:                                       # one forward per hypothesis on its own cache
                c = list(bm["parent"]["cache"])
                cur = S + len(bm["ids"]) - 1
                h = model.embed([bm["tok"]]).unsqueeze(0)
                c1, s1 = O.mrope_cos_sin([[cur]] * 3, t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved)
                past = c[0][0].shape[2]
                bm["logits"] = model.decoder_forward(h, c1, s1, c, O.causal_mask(1, past))[:, 0, :][0].double().numpy()
                bm["cache"] = c
            beams = new
            step += 1
            ref.steps += 1
        for bm in beams:                                         # at the cap: the alive beams fill the list, rank order
            if len(fin) >= K:
                break
            fin.append((list(bm["ids"]), bm["sum"], -1))
    order = rank([(len(h[0]), h[1]) for h in fin], alpha)
    scores = [score(h[1], len(h[0]), alpha) for h in fin]
    ref.hyps = [(fin[i][0], fin[i][1], scores[i], fin[i][2]) for i in order]
    nmax = max(len(h[0]) for h in fin) + 1
    for a, b in zip(order, order[1:]):
        ref.gaps.append((scores[a] - scores[b], nmax))
    return ref


def pinned(ref):
    """The smallest gap over its floor (> 1: every boundary clears GAP_FLOOR x the accumulated noise)."""
    worst = math.inf
    for g, n in ref.gaps:
        fl = GAP_FLOOR * LOGIT_NOISE * ref.mx * (n + 1)
        worst = min(worst, abs(g) / fl)
    return worst


def pick_clips(model, pool, n, K, n_new, alpha=None):
    """The first n clips of `pool` ((index, seconds)) whose oracle runs are pinned."""
    from qwen3_asr_rs_b200 import synth
    got = []
    for i, sec in pool:
        x = synth.make_clip(i, sec)
        ref = beam_oracle(model, x, K, n_new, alpha)
        if pinned(ref) > 1.0:
            got.append((x, ref))
            if len(got) == n:
                return got
    raise AssertionError(f"only {len(got)} of {n} clips of the pool are pinned")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _steps(st):
    return {k: st.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}


def _moved(eng, fn):
    s0 = _steps(eng.stats())
    r = fn()
    s1 = _steps(eng.stats())
    return r, {k: s1[k] - s0[k] for k in s0}


@pytest.fixture(scope="module")
def beam_engine(tiny):
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    yield eng
    eng.close()


def _bytes_per_pos(cfg):
    t = cfg.text
    return 2 * t.num_hidden_layers * t.num_key_value_heads * t.head_dim * 4


POOL = [(500 + i, s) for i, s in enumerate([1.3, 2.2, 0.9, 3.7, 1.8, 2.9, 1.1, 4.4, 0.8, 2.6, 3.1, 1.6, 2.0, 3.4, 1.2,
                                            2.4, 0.7, 3.9, 1.5, 2.7, 1.9, 0.6, 3.3, 2.1, 1.4, 2.8, 1.0, 3.6, 1.7, 2.5])]
# (label, utterances, K, new tokens, options, path whose counter must move)
CASES = [
    ("nb8_b2k4", 2, 4, 8, {}, "decode_batch_steps"),
    ("nb16_b3k5", 3, 5, 6, {}, "decode_batch_steps"),
    ("passes_b4k5", 4, 5, 6, {}, "decode_batch_steps"),
    ("per_seq_b2k2", 2, 2, 8, {"batch_step": "0"}, "decode_fused_steps"),
    ("phases_b2k4", 2, 4, 8, {"decode": "phases"}, "decode_phase_steps"),
    ("b1k6", 1, 6, 8, {}, "decode_batch_steps"),
    ("b1k2", 1, 2, 10, {}, "decode_batch_steps"),
]
_RESET = {"decode": "mega", "batch_step": "1"}


def _check(got, refs, st, cfg, report, label):
    worst = 0.0
    for b, ref in enumerate(refs):
        assert [h[0] for h in got.nbest[b]] == [h[0] for h in ref.hyps], (label, b)
        assert [h[3] for h in got.nbest[b]] == [h[3] for h in ref.hyps], (label, b)
        for (ids, sm, sc, _), (_, rs, _, _) in zip(got.nbest[b], ref.hyps):
            worst = max(worst, abs(sm - rs) / (ref.mx * (len(ids) + 1)))
        assert got.ids[b] == ref.hyps[0][0]
    bpp = _bytes_per_pos(cfg)
    assert st["slots_reassigned"] == sum(r.reassigned for r in refs), label
    assert st["reorder_kv_bytes"] == bpp * sum(r.reorder_positions for r in refs), label
    assert st["expand_kv_bytes"] == bpp * sum(r.expand_positions for r in refs), label
    assert st["beam_steps"] == got.decode_steps
    report[f"beam_{label}_max_rel_sum_err"] = worst
    report[f"beam_{label}_reassigned"] = st["slots_reassigned"]
    assert worst <= LP_RTOL
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_beam_parity_on_every_path(tiny, beam_engine, report, case):
    """All K hypotheses equal the float64 oracle's (ids, EOS ids, sums within LP_RTOL); the beam statistics equal the
    oracle's replay; the path counter moves as a greedy run over B * K sequences; repeated runs are bitwise equal."""
    label, B, K, n_new, options, path = case
    cfg, _, model = tiny
    picked = pick_clips(model, POOL, B, K, n_new)
    clips, refs = [p[0] for p in picked], [p[1] for p in picked]
    eng = beam_engine
    for k, v in options.items():
        eng.set_option(k, v)
    try:
        eng.transcribe_ids(clips, max_new_tokens=n_new, beam_size=K)      # warm-up: session, graphs
        got, moved = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=n_new, beam_size=K, logprobs=True))
        st = eng.last_beam_stats()
        again = eng.transcribe_ids(clips, max_new_tokens=n_new, beam_size=K, logprobs=True)
    finally:
        for k in options:
            eng.set_option(k, _RESET[k])
    _check(got, refs, st, cfg, report, label)
    assert st["slots_reassigned"] > 0 and st["reorder_kv_bytes"] > 0     # these clips move beams: the reorder runs
    assert again.nbest == got.nbest and again.logprobs == got.logprobs and again.eos_logprobs == got.eos_logprobs
    if path == "decode_phase_steps":
        assert moved["decode_fused_steps"] == 0 and moved["decode_batch_steps"] == 0
    else:
        assert moved[path] == got.decode_steps and moved["decode_phase_steps"] == 0
    for b in range(B):                       # the best hypothesis's values: its sum, bitwise
        acc = np.float32(0.0)
        for v in got.logprobs[b] + ([got.eos_logprobs[b]] if got.eos_logprobs[b] is not None else []):
            acc = np.float32(acc + np.float32(v))
        assert float(acc) == got.nbest[b][0][1]
        assert (got.eos_logprobs[b] is None) == (got.nbest[b][0][3] == -1)


@pytest.mark.gpu
def test_beam_length_penalty(tiny, beam_engine, report):
    cfg, _, model = tiny
    picked = pick_clips(model, POOL[5:], 2, 3, 12, alpha=0.6)
    clips, refs = [p[0] for p in picked], [p[1] for p in picked]
    got = beam_engine.transcribe_ids(clips, max_new_tokens=12, beam_size=3, length_penalty=0.6)
    _check(got, refs, beam_engine.last_beam_stats(), cfg, report, "alpha0.6")
    for b in range(2):
        for ids, sm, sc, _ in got.nbest[b]:
            assert math.isclose(sc, score(sm, len(ids), 0.6), rel_tol=1e-6)


def _self_consistent(got):
    """Each utterance's best hypothesis: its sum is the fp32 sequential sum of its reported values and its EOS value,
    bitwise; its ids are `ids`; the n-best is ranked by score."""
    for b in range(len(got.ids)):
        acc = np.float32(0.0)
        for v in got.logprobs[b] + ([got.eos_logprobs[b]] if got.eos_logprobs[b] is not None else []):
            acc = np.float32(acc + np.float32(v))
        assert float(acc) == got.nbest[b][0][1] and got.nbest[b][0][0] == got.ids[b]
        assert (got.eos_logprobs[b] is None) == (got.nbest[b][0][3] == -1)
        sc = [h[2] for h in got.nbest[b]]
        assert sc == sorted(sc, reverse=True)


@pytest.mark.gpu
def test_beam_across_fused_step_limit(beam_engine, report):
    """60 s prompt + 400 tokens, one fused launch per slot (batch_step=0): the search continues across the hand-over to
    the per-phase path."""
    from qwen3_asr_rs_b200 import synth
    x = synth.make_clip(302, 60.0)
    beam_engine.set_option("batch_step", "0")
    try:
        got, moved = _moved(beam_engine, lambda: beam_engine.transcribe_ids([x], max_new_tokens=400, beam_size=2, logprobs=True))
        again = beam_engine.transcribe_ids([x], max_new_tokens=400, beam_size=2, logprobs=True)
    finally:
        beam_engine.set_option("batch_step", "1")
    _self_consistent(got)
    assert again.nbest == got.nbest
    if got.decode_steps > 300:
        assert moved["decode_fused_steps"] > 0 and moved["decode_phase_steps"] > 0
    report["beam_long_steps"] = got.decode_steps
    report["beam_long_reassigned"] = beam_engine.last_beam_stats()["slots_reassigned"]


@pytest.mark.gpu
def test_beam_size_1_is_greedy_and_greedy_after_beam(beam_engine):
    from qwen3_asr_rs_b200 import synth
    eng = beam_engine
    clips = [synth.make_clip(400 + i, s) for i, s in enumerate([1.1, 2.3, 0.7])]
    g, mg = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=16, logprobs=True))
    b1, mb = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=16, logprobs=True, beam_size=1))
    assert b1.ids == g.ids and b1.logprobs == g.logprobs and b1.eos_logprobs == g.eos_logprobs and mb == mg
    assert b1.nbest is None
    eng.transcribe_ids(clips, max_new_tokens=16, beam_size=4, logprobs=True)
    g2, mg2 = _moved(eng, lambda: eng.transcribe_ids(clips, max_new_tokens=16, logprobs=True))
    assert g2.ids == g.ids and g2.logprobs == g.logprobs and g2.eos_logprobs == g.eos_logprobs and mg2 == mg


def _last_hidden(model, x):
    """The oracle's final-normed hidden state of the prompt's last row (what the lm_head multiplies for token 0)."""
    import torch
    from oracle import oracle as O
    t = model.cfg.text
    mel = O.extract_mel(x, model.cfg.audio.num_mel_bins)
    audio = model.encode(mel)
    ids, a0 = O.build_prompt(audio.shape[0])
    S = len(ids)
    hid = model.embed(ids).unsqueeze(0)
    hid[0, a0:a0 + audio.shape[0], :] = audio
    pos = list(range(S))
    cos, sin = O.mrope_cos_sin([pos] * 3, t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved)
    head = model.lm_head_weight
    model.lm_head_weight = lambda: torch.eye(t.hidden_size, dtype=hid.dtype)
    try:
        with torch.no_grad():
            h = model.decoder_forward(hid, cos, sin, [None] * t.num_hidden_layers, O.causal_mask(S, 0), last_only=True)
    finally:
        del model.lm_head_weight
        assert model.lm_head_weight == head
    return h[0, -1].double()


# clip A ends at token 0 under the EOS model below; the others run on (C to the cap, D to EOS at step 3)
EOS_A, EOS_B, EOS_C, EOS_D = (510, 1.9), (511, 1.6), (512, 2.0), (513, 3.4)


def _eos_model():
    """Tiny dims with an untied lm_head whose two EOS rows point along clip A's last hidden state, made orthogonal to
    clip B's: A's token-0 record starts with both EOS ids (logits 0.3 above its best other one, EOS rows 3 % apart), so
    with K = 2 it is done at token 0, while the other clips meet EOS later or never."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import synth
    cfg = O.cfg_tiny()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 7)
    base = O.OracleModel(cfg, w)
    ha, hb = _last_hidden(base, synth.make_clip(*EOS_A)), _last_hidden(base, synth.make_clip(*EOS_B))
    perp = ha - (ha @ hb) / (hb @ hb) * hb
    head = w["thinker.lm_head.weight"].float().clone()
    row = (float((head.double() @ ha).max()) + 0.3) * perp / (perp @ ha)
    head[151643] = row.float()
    head[151645] = (0.97 * row).float()
    w2 = dict(w)
    w2["thinker.lm_head.weight"] = head.bfloat16()
    return cfg, w2, O.OracleModel(cfg, w2)


@pytest.mark.gpu
def test_beam_eos(report):
    """K = 2 on the EOS model, against the oracle:
    - [A, D, C]: A is done at token 0 (EOS among, indeed on top of, token 0's candidates) while D and C stay alive on
      the batched step, after a longer beam run left other positions in those slots; D's hypotheses finish on EOS at
      step 3 and C's stop at the cap (eos_id -1) beside them;
    - [A, D] with a cap of 40: every utterance completes early, so the loop stops at its first all-done check (16)."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    cfg, w2, model = _eos_model()
    cfg_e = config_tiny()
    cfg_e.text.tie_word_embeddings = False
    a, c, d = (synth.make_clip(*x) for x in (EOS_A, EOS_C, EOS_D))
    refs = [beam_oracle(model, y, 2, 12) for y in (a, d, c)]
    refs_early = [beam_oracle(model, y, 2, 40) for y in (a, d)]
    for r in refs + refs_early:
        assert pinned(r) > 1.0
    assert [h[3] != -1 and len(h[0]) == 0 for h in refs[0].hyps] == [True, True]
    assert {len(h[0]) for h in refs[1].hyps if h[3] != -1} and all(h[3] == -1 for h in refs[2].hyps)
    eng = AsrInference.from_weights(cfg_e, w2, device=0)
    try:
        eng.transcribe_ids([synth.make_clip(520, 9.0)] * 3, max_new_tokens=40, beam_size=2)   # positions > A's prompt
        got, moved = _moved(eng, lambda: eng.transcribe_ids([a, d, c], max_new_tokens=12, beam_size=2, logprobs=True))
        _check(got, refs, eng.last_beam_stats(), cfg, report, "eos")
        early = eng.transcribe_ids([a, d], max_new_tokens=40, beam_size=2, logprobs=True)
        _check(early, refs_early, eng.last_beam_stats(), cfg, report, "eos_early")
    finally:
        eng.close()
    assert moved["decode_batch_steps"] == got.decode_steps
    assert got.ids[0] == [] and [h[3] for h in got.nbest[0]] == [151643, 151645] and got.eos_logprobs[0] is not None
    eos_steps = {len(h[0]) for b in range(3) for h in got.nbest[b] if h[3] != -1}
    assert len(eos_steps) >= 2                                       # hypotheses finished at different steps
    assert all(h[3] == -1 for h in got.nbest[2]) and got.eos_logprobs[2] is None
    assert early.decode_steps == 16 < 39                             # early completion, below the cap
    report["beam_eos_lengths"] = sorted(eos_steps)


@pytest.mark.gpu
def test_beam_refusals_through_the_abi(tiny):
    import ctypes as C
    from qwen3_asr_rs_b200 import AsrInference, config_tiny, synth
    from qwen3_asr_rs_b200 import _lib
    from qwen3_asr_rs_b200._lib import AsrbError
    _, w, _ = tiny
    eng = AsrInference.from_weights(config_tiny(), w, device=0)
    x = synth.make_clip(301, 1.7)
    try:
        eng.transcribe_ids([x], max_new_tokens=4)           # a session with max_batch 1
        with pytest.raises(AsrbError) as e:
            eng.last_nbest(4, 1)
        assert e.value.code == 4
        for bad in ("0", "7", "", "2 ", "x"):
            with pytest.raises(AsrbError) as e:
                eng.set_option("beam_size", bad)
            assert e.value.code == 1
        for bad in ("-1", "10.5", "nan", "", "x", " 1"):
            with pytest.raises(AsrbError) as e:
                eng.set_option("length_penalty", bad)
            assert e.value.code == 1
        eng.set_option("length_penalty", "0.6"); eng.set_option("length_penalty", "none")
        eng.set_option("beam_size", "2")
        ids = np.zeros((1, 4), np.int32)
        n = np.zeros(1, np.int32)
        arrs, ptrs, lens = eng._pack_samples([x])
        with pytest.raises(AsrbError) as e:                 # batch 1 x K 2 > max_batch 1
            _lib.check(eng._lib.asrb_transcribe_ids(eng._session, ptrs, lens, 1, None, None, 4,
                                                    ids.ctypes.data_as(C.POINTER(C.c_int32)), n.ctypes.data_as(C.POINTER(C.c_int32))))
        assert e.value.code == 1
        eng.set_option("beam_size", "1")
        eng.transcribe_ids([x, x], max_new_tokens=4)        # max_batch 2
        eng.set_option("beam_size", "2")
        for key, val in (("temperature", "1"), ("top_logprobs", "1")):
            eng.set_option(key, val)
            with pytest.raises(AsrbError) as e:
                eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
            assert e.value.code == 1
            eng.set_option(key, "0")
        eng.mel([x]); eng.encode(); eng.prefill(want_logits=False)
        with pytest.raises(AsrbError) as e:
            eng.decode_step(want_logits=False)
        assert e.value.code == 1
        ids = eng.generate(6)
        assert len(ids) == 1 and len(eng.last_nbest(6, 2)[0]) == 2
        with pytest.raises(AsrbError) as e:                 # finalized: the search does not resume
            eng.generate(12)
        assert e.value.code == 4
        with pytest.raises(AsrbError) as e:
            eng.last_nbest(6, 3)
        assert e.value.code == 1
        eng.set_option("beam_size", "1")
    finally:
        eng.close()


@pytest.mark.gpu
def test_beam_device_ids_and_fallback(tiny, beam_engine):
    """asrb_session_device_ids returns the best hypotheses; a schedule runs the beam at t = 0."""
    import torch
    from qwen3_asr_rs_b200 import synth
    from qwen3_asr_rs_b200.parallel import _DevView
    eng = beam_engine
    clips = [synth.make_clip(500 + i, s) for i, s in enumerate([1.3, 2.2])]
    got = eng.transcribe_ids(clips, max_new_tokens=10, beam_size=3)
    ids_p, lens_p, stride, batch = eng.device_ids()
    assert batch == 2
    ids = torch.as_tensor(_DevView(ids_p, (batch, stride)), device="cuda").cpu()
    lens = torch.as_tensor(_DevView(lens_p, (batch,)), device="cuda").cpu()
    for b in range(2):
        assert int(lens[b]) == len(got.ids[b]) and ids[b, : int(lens[b])].tolist() == got.ids[b]
    fb = eng.transcribe_ids(clips, max_new_tokens=10, beam_size=3, temperature=(0.0, 1.0), logprob_threshold=None)
    direct = eng.transcribe_ids(clips, max_new_tokens=10, beam_size=3)
    for b in range(2):
        if fb.temperatures[b] == 0.0:
            assert fb.ids[b] == direct.ids[b] and fb.nbest[b] == direct.nbest[b]


@pytest.mark.gpu
@pytest.mark.parametrize("dims", ["0p6b", "1p7b"])
def test_full_size_beam(report, dims):
    """Full dims, 30 s clips.  0.6B: batch 3 x beam 5 (15 slots, NB 16) and batch 1 x beam 5, 6 new tokens, against the
    float64 oracle on pinned clips.  1.7B: batch 1 x beam 5, 24 new tokens, self-consistent and repeatable on the
    fused single-sequence step (one launch per slot)."""
    from oracle import oracle as O
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, config_1p7b, synth
    cfg = {"0p6b": O.cfg_0p6b, "1p7b": O.cfg_1p7b}[dims]()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 1, peaked_head=True)
    ecfg = {"0p6b": config_0p6b, "1p7b": config_1p7b}[dims]()
    ecfg.text.tie_word_embeddings = False
    if dims == "0p6b":
        model, n_new, picked = O.OracleModel(cfg, w), 6, []
        for i in (1, 3, 4, 6, 7, 8):
            x = synth.make_clip(i, 30.0)
            r = beam_oracle(model, x, 5, n_new)
            if pinned(r) > 1.0:
                picked.append((x, r))
            if len(picked) == 3:
                break
        assert len(picked) == 3
        clips, refs = [p[0] for p in picked], [p[1] for p in picked]
        # the 15-slot run first: it sizes the session, whose path counters then stay the same object
        runs = [(clips, refs, "decode_batch_steps"), (clips[:1], refs[:1], "decode_batch_steps")]
    else:
        n_new = 24
        runs = [([synth.make_clip(1, 30.0)], None, "decode_fused_steps")]
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        for cl, rf, path in runs:
            got, moved = _moved(eng, lambda: eng.transcribe_ids(cl, max_new_tokens=n_new, beam_size=5, logprobs=True))
            st = eng.last_beam_stats()
            again = eng.transcribe_ids(cl, max_new_tokens=n_new, beam_size=5, logprobs=True)
            _self_consistent(got)
            if rf is not None:
                _check(got, rf, st, cfg, report, f"full_{dims}_b{len(cl)}")
            assert again.nbest == got.nbest and st["beam_steps"] == got.decode_steps
            assert moved[path] == got.decode_steps and moved["decode_phase_steps"] == 0
            assert st["expand_kv_bytes"] > 0
            report[f"beam_full_{dims}_b{len(cl)}_reassigned"] = st["slots_reassigned"]
    finally:
        eng.close()
