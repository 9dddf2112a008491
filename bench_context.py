"""Cost of context biasing (asrb_session_set_context) and what sharing a context saves in the prefill.

Runs Qwen3-ASR-0.6B dims (synthetic weights), 30 s clips, 64 new tokens, at batch 1 and 16, three arms alternated in one
process: (a) no context; (b) one 256-id context shared by every utterance (prefilled once, its K/V fanned out);
(c) 256-id contexts that differ per utterance, which computes the rows a non-shared implementation would.  Per arm: the
prefill time (the library's CUDA events, stage_ms["prefill"]), the decode time per executed step, the prefill counters
(asrb_last_prefill_stats), the decoder forwards by path, and the spread over rounds; plus the card's name, power limit
and maximum SM clock, read in the same run.  Prints one JSON line.

    python bench_context.py [--rounds 5] [--warmup 1] [--new-tokens 64] [--context-ids 256]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_logprobs import gpu_info  # noqa: E402

PATHS = ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--new-tokens", type=int, default=64)
    ap.add_argument("--context-ids", type=int, default=256)
    args = ap.parse_args()
    import numpy as np
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    L = args.context_ids
    out = {"metric": f"prefill ms and decode step us: no context / one shared {L}-id context / distinct {L}-id contexts "
                     "(Qwen3-ASR-0.6B dims, 30 s clips)",
           "gpu": gpu_info(0), "shapes": {}}
    try:
        for label, B in (("b1", 1), ("b16", 16)):
            clips = [synth.make_clip(i, 30.0) for i in range(B)]
            rng = np.random.default_rng(0)
            shared = [int(v) for v in rng.integers(0, 150000, L)]
            distinct = [[int(v) for v in rng.integers(0, 150000, L)] for _ in range(B)]
            arms = (("none", None), ("shared", [shared] * B), ("distinct", distinct))

            def run(ctx):
                before = eng.stats()
                r = eng.transcribe_ids(clips, max_new_tokens=args.new_tokens, context_ids=ctx)
                after = eng.stats()
                moved = {k: after[k] - before.get(k, 0) for k in PATHS}
                return r.stage_ms["prefill"], 1e3 * r.stage_ms["decode"] / max(r.decode_steps, 1), r.decode_steps, moved, \
                    eng.last_prefill_stats()

            for _ in range(args.warmup):
                for _, ctx in arms:
                    run(ctx)
            pre = {a: [] for a, _ in arms}
            dec = {a: [] for a, _ in arms}
            steps, moved, pstats = {}, {}, {}
            for _ in range(args.rounds):         # alternated: clock / thermal drift hits all arms alike
                for a, ctx in arms:
                    p, d, steps[a], moved[a], pstats[a] = run(ctx)
                    pre[a].append(p)
                    dec[a].append(d)
            mp = {a: statistics.median(v) for a, v in pre.items()}
            md = {a: statistics.median(v) for a, v in dec.items()}
            out["shapes"][label] = {
                "batch": B, "context_ids": L, "new_tokens": args.new_tokens,
                **{f"prefill_ms_{a}": round(mp[a], 3) for a in mp},
                **{f"prefill_spread_{a}_pct": round(100.0 * (max(v) - min(v)) / mp[a], 3) for a, v in pre.items()},
                **{f"step_us_{a}": round(md[a], 2) for a in md},
                **{f"step_spread_{a}_pct": round(100.0 * (max(v) - min(v)) / md[a], 3) for a, v in dec.items()},
                "prefill_saved_shared_vs_distinct_pct": round(100.0 * (1.0 - mp["shared"] / mp["distinct"]), 3),
                "prefill_stats": pstats, "decode_steps": steps, "steps_by_path": moved,
            }
    finally:
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
