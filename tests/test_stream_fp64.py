"""Streams at the tiny, 0.6B and 1.7B widths under DESIGN.md section 2's float64 rule, on every decode path.

The models are test_decode_variants_fp64.MODELS: the production widths and vocabulary cut to 4 encoder and 4 decoder
layers (the tiny one whole), each with an untied peaked head so that ids can be pinned.  Each cell pushes its streams'
audio and checks, at every push, for the checked streams:
  - the encoder output (asrb_stream_encode_read) of the prefix against OracleModel's encoder in fp32 / float64 on the
    prefix's mel: R = 4, on a push whose first window is reused and on the final push;
  - the log-probability and top-8 records of the push's continuation g at the stream's own ids, against log_softmax of
    oracle.score_ids(prefix audio, g, language ids = p) in fp32 / float64: R = 4;
  - g at every step whose float64 top-1 / top-2 gap clears GAP is the float64 argmax, and at least half the steps are
    so pinned; up to the first unpinned step g equals transcribe_ids(prefix audio, lang + p) of the offline path;
and that the cell's decode path ran, from asrb_session_stats: the single-sequence fused step (one stream), the batched
step at NB 8 and NB 16 (5 and 12 streams), the fused step per sequence at 1.7B (no batched step there), and the
per-phase hand-over of a stream whose push passes the fused step's 1152 keys after keeping its first windows' K/V.
"""
import gc

import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth
from test_decode_variants_fp64 import MODELS
from test_precision_fp64 import Err, check

GAP = 1e-2                # float64 logit gap above which an id is pinned (about 1000 x the fp32 errors of these models)

# cell -> (model, clips (index, seconds), push seconds, max_new_tokens, rollback, unfixed pushes, streams checked,
#          path counters that must move)
CELLS = {
    "tiny_single": ("tiny", [(801, 17.3)], 1.0, 24, 20, 2, [0], ("decode_fused_steps",)),
    "w0p6b_single": ("w0p6b", [(802, 17.3)], 1.0, 24, 20, 2, [0], ("decode_fused_steps",)),
    "w1p7b_single": ("w1p7b", [(803, 17.3)], 1.0, 24, 20, 2, [0], ("decode_fused_steps",)),
    "w0p6b_nb8": ("w0p6b", [(810 + i, 9.0 + 0.7 * i) for i in range(5)], 2.0, 20, 10, 2, [0, 2, 4], ("decode_batch_steps",)),
    "w0p6b_nb16": ("w0p6b", [(820 + i, 8.5 + 0.3 * i) for i in range(12)], 2.0, 20, 10, 2, [0, 7, 11],
                   ("decode_batch_steps",)),
    "w1p7b_b3": ("w1p7b", [(840 + i, 9.5 + i) for i in range(3)], 2.0, 20, 10, 2, [0, 1, 2], ("decode_fused_steps",)),
    # 30 s, then the rest to 60 s with 400 new ids: prompt ~800 keys + 8 forced ids, past 1152 keys mid-push
    "w0p6b_handover": ("w0p6b", [(850, 60.0)], 30.0, 400, 392, 1, [0], ("decode_fused_steps", "decode_phase_steps")),
}


class Zoo:
    def __init__(self):
        self.models = {}

    def get(self, name):
        if name not in self.models:
            for k in list(self.models):                  # one width at a time: the oracles hold float64 weights
                self.models.pop(k)[2].close()
            gc.collect()
            from qwen3_asr_rs_b200 import AsrInference
            ocfg, ecfg = MODELS[name].configs()
            w = synth.make_weights(ocfg, MODELS[name].seed, peaked_head=True)
            self.models[name] = (O.OracleModel(ocfg, w), O.OracleModel(ocfg, w, dtype=torch.float64),
                                 AsrInference.from_weights(ecfg, w, device=0))
        return self.models[name]

    def close(self):
        for v in self.models.values():
            v[2].close()
        self.models = {}


@pytest.fixture(scope="module")
def zoo():
    z = Zoo()
    yield z
    z.close()


def _log_softmax(logits):
    return torch.log_softmax(logits.double(), dim=-1).numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("cell", list(CELLS))
def test_stream_records_encoder_ids_and_path(zoo, report, cell):
    name, sel, push_s, max_new, rollback, unfixed, checked, paths = CELLS[cell]
    m32, m64, eng = zoo.get(name)
    xs = [synth.make_clip(*c) for c in sel]
    n = len(xs)
    ss = eng.open_streams(n, max(len(x) for x in xs) / 16000.0 + 0.1, max_new_tokens=max_new, rollback=rollback,
                          unfixed_pushes=unfixed, top_logprobs=8)
    step = int(round(push_s * 16000))
    pos, prefix, pushes = [0] * n, [[] for _ in range(n)], []
    enc_at = {}
    before = after = None
    while any(p < len(x) for p, x in zip(pos, xs)):
        chunks, fin = [], []
        for b, x in enumerate(xs):
            c = x[pos[b]: pos[b] + step] if pos[b] < len(x) else None
            pos[b] += 0 if c is None else len(c)
            chunks.append(c)
            fin.append(c is not None and pos[b] >= len(x))
        last = all(p >= len(x) for p, x in zip(pos, xs))
        if last:
            before = eng.stats()
        hyps = ss.push(chunks, final=fin)
        if last:
            after = eng.stats()
        st = ss.stats()
        for b in checked:
            if chunks[b] is None:
                continue
            pushes.append((b, pos[b], list(prefix[b]), hyps[b]))
            if fin[b] or (st["windows_reused"] > 0 and b not in enc_at):
                enc_at.setdefault(b, []).append((pos[b], ss.encoder_output(b)))
        for b in range(n):
            if chunks[b] is not None:
                prefix[b] = hyps[b].ids[: hyps[b].fixed]
    # ---- the decode path of the cell's last push ----
    for p in paths:
        assert after[p] > before[p], (cell, p, before, after)
    # ---- encoder: float64 rule on the prefix ----
    enc = Err(True)
    for b, outs in enc_at.items():
        for nb, got in outs:
            x = xs[b][:nb]
            with torch.no_grad():
                e32 = m32.encode(O.extract_mel(x)).numpy()
                e64 = m64.encode(O.extract_mel(x, dtype=torch.float64)).numpy()
            enc.add(got, e32, e64)
    check(report, f"stream_{cell}_encoder", enc)
    # ---- records, pinned ids, equality with the offline path ----
    lp_err, tk_err = Err(False), Err(False)
    pinned = steps = 0
    offline = []
    for b, nb, p, h in pushes:
        g = h.ids[len(p):]
        x = xs[b][:nb]
        with torch.no_grad():
            s32 = O.score_ids(m32, x, g, language_ids=p or None)
            s64 = O.score_ids(m64, x, g, language_ids=p or None)
        l32, l64 = _log_softmax(s32), _log_softmax(s64)
        rows = np.arange(len(g))
        lp_err.add(np.array(h.logprobs), l32[rows, g], l64[rows, g])
        for t, row in enumerate(h.top_logprobs):
            cand = np.array([c[0] for c in row])
            assert row[0][0] == g[t]
            tk_err.add(np.array([c[1] for c in row]), l32[t, cand], l64[t, cand])
        first_unpinned = len(g)
        for t, tok in enumerate(g):
            top2 = np.sort(s64[t].numpy())[-2:]
            steps += 1
            if top2[1] - top2[0] > GAP:
                pinned += 1
                assert tok == int(s64[t].argmax()), (cell, b, nb, t)
            else:
                first_unpinned = min(first_unpinned, t)
        offline.append((x, p, g[:first_unpinned]))
    check(report, f"stream_{cell}_logprobs", lp_err)
    check(report, f"stream_{cell}_top8", tk_err)
    assert pinned * 2 >= steps, (cell, pinned, steps)
    for x, p, g in offline:                                           # ends the streams: after every push
        got = eng.transcribe_ids([x], language_ids=[p] if p else None, max_new_tokens=max_new).ids[0]
        assert got[: len(g)] == g, (cell, len(x))
