"""Cost of seeded temperature sampling (session options "temperature" / "seed") on the decode step.

Times the decode loop of Qwen3-ASR-0.6B dims (synthetic weights) greedy, at T = 1, and at T = 1 with logprobs, the
three alternated in one process: batch 1 (one 30 s clip, 128 new tokens: single-sequence fused step) and batch 8 (eight
30 s clips, batched fused step).  A sampled run of synthetic weights may select EOS early, so the figure is the decode
time per executed step (the library's CUDA events: stage_ms["decode"] / decode_steps).  Prints one JSON line with the
card's name, power limit and maximum SM clock read in the same run.

    python bench_sampling.py [--rounds 7] [--warmup 2] [--new-tokens 128]
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
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    out = {"metric": "decode step us per executed step, greedy vs T=1 vs T=1+logprobs (Qwen3-ASR-0.6B dims, 30 s clips)",
           "gpu": gpu_info(0), "shapes": {}}
    arms = (("greedy", {}), ("t1", dict(temperature=1.0, seed=1)), ("t1_logprobs", dict(temperature=1.0, seed=1, logprobs=True)))
    try:
        for label, B, path in (("b1", 1, "decode_fused_steps"), ("b8", 8, "decode_batch_steps")):
            clips = [synth.make_clip(i, 30.0) for i in range(B)]

            def step_us(kw):
                before = eng.stats()
                r = eng.transcribe_ids(clips, max_new_tokens=args.new_tokens, **kw)
                after = eng.stats()
                moved = {k: after[k] - before.get(k, 0) for k in PATHS}
                return 1e3 * r.stage_ms["decode"] / max(r.decode_steps, 1), r.decode_steps, moved

            for _ in range(args.warmup):
                for _, kw in arms:
                    step_us(kw)
            times = {a: [] for a, _ in arms}
            steps, moved = {}, {}
            for _ in range(args.rounds):         # alternated: clock / thermal drift hits all arms alike
                for a, kw in arms:
                    t, steps[a], moved[a] = step_us(kw)
                    times[a].append(t)
            med = {a: statistics.median(v) for a, v in times.items()}
            out["shapes"][label] = {
                "batch": B, "new_tokens": args.new_tokens, "expected_path": path,
                **{f"step_us_{a}": round(med[a], 2) for a in med},
                **{f"spread_{a}_pct": round(100.0 * (max(v) - min(v)) / med[a], 3) for a, v in times.items()},
                "overhead_t1_pct": round(100.0 * (med["t1"] / med["greedy"] - 1.0), 3),
                "overhead_t1_logprobs_pct": round(100.0 * (med["t1_logprobs"] / med["greedy"] - 1.0), 3),
                "decode_steps": steps, "steps_by_path": moved,
            }
    finally:
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
