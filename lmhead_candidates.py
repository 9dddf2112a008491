"""Candidate rows of the greedy fused step's int8 lm_head (DESIGN.md section 4.1), counted on the CPU.

Runs the oracle on the bench workload (synth.make_weights(cfg, 1), make_clip(0), --new-tokens greedy tokens), takes the
final normed hidden vector x of every step, splits the lm_head into the --ctas contiguous row ranges of make_slice and
counts, per CTA and step, the rows whose interval [a_r - B_r, a_r + B_r] reaches the CTA's best lower bound, for two
approximate forms:
  (a) int8 weights dequantized in fp32 FMA (what consume_head_q does): B_r = |x|_2 C_r;
  (b) int8 weights and an int8 per-vector quantization of x contracted with dp4a: B_r gains |x - s_x q_x|_2 s_r |q_r|_2.
C_r is model.cu's (quantize_head_kernel); a_r is evaluated in float64, which moves the counts by rounding only.
Prints one JSON line.  The 0.6B model takes a few minutes and about 10 GB of host memory.

  python lmhead_candidates.py [--model 0p6b|1p7b] [--new-tokens 128] [--ctas 132]
"""
import argparse
import json

import numpy as np

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="0p6b", choices=["0p6b", "1p7b"])
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--ctas", type=int, default=132)
    args = ap.parse_args()
    cfg = O.cfg_0p6b() if args.model == "0p6b" else O.cfg_1p7b()
    xs = []

    class Capture(O.OracleModel):
        def decoder_forward(self, hidden, cos, sin, cache, mask, last_only=False, from_row=0):
            x = hidden
            for i in range(self.cfg.text.num_hidden_layers):
                x = self.decoder_layer(x, i, cos, sin, cache, mask)
            x = O.rms_norm(x, self.w["thinker.model.norm.weight"], self.cfg.text.rms_norm_eps)
            xs.append(x[0, -1].double().numpy())
            return x[:, -1:, :].matmul(self.lm_head_weight().t())

    m = Capture(cfg, synth.make_weights(cfg, 1))
    ids = O.transcribe_ids(m, synth.make_clip(0), max_new_tokens=args.new_tokens, lm_head_all_rows=False).ids
    steps = xs[1:len(ids)]                           # the fused steps: xs[0] is the prefill's row, the last x selects nothing
    W = m.lm_head_weight().float().numpy().astype(np.float64)
    V, K = W.shape
    u = 2.0 ** -24
    n = K // 64 + 6
    gamma = lambda k: k * u / (1 - k * u)            # noqa: E731
    s = (np.abs(W).max(1) / 127).astype(np.float32).astype(np.float64)
    q = np.clip(np.rint(W / np.where(s > 0, s, 1)[:, None]), -127, 127)
    nq = np.linalg.norm(q, axis=1)
    C = np.linalg.norm(W - s[:, None] * q, axis=1) + gamma(n) * np.linalg.norm(W, axis=1) + gamma(n + 1) * s * nq
    G = args.ctas
    bounds = [((c * V) // G, ((c + 1) * V) // G) for c in range(G)]
    counts = {"a": [], "b": []}
    for x in steps:
        nx = np.linalg.norm(x) * (1 + 2 ** -12)
        a, B = s * (q @ x), nx * C
        sx = np.abs(x).max() / 127
        qx = np.rint(x / sx)
        ab, Bb = s * sx * (q @ qx), B + np.linalg.norm(x - sx * qx) * (1 + 2 ** -12) * s * nq
        for form, (aa, bb) in (("a", (a, B)), ("b", (ab, Bb))):
            row = []
            for r0, r1 in bounds:
                T = np.max(aa[r0:r1] - bb[r0:r1])
                row.append(int(np.count_nonzero(aa[r0:r1] + bb[r0:r1] >= T)))
            counts[form].append(row)
    out = {"model": args.model, "tokens": len(ids), "steps": len(steps), "ctas": G, "rows_per_cta": V // G}
    for form, c in counts.items():
        c = np.array(c)
        out[form] = {"per_cta_mean": round(float(c.mean()), 2), "per_cta_max": int(c.max()),
                     "per_step_mean": round(float(c.sum(1).mean()), 1), "per_step_max": int(c.sum(1).max())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
