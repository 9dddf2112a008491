"""Cost of the repetition controls (session options "no_repeat_ngram_size" / "repetition_penalty") on the decode step.

Times the decode loop of Qwen3-ASR-0.6B dims (synthetic weights, which do not loop, so the options change little of
the work) with the options off, N = 3, theta = 1.2 and both, the four alternated in one process: batch 1 (one 30 s
clip, 128 new tokens: single-sequence fused step) and batch 8 (eight 30 s clips, batched fused step).  The figure is the
decode time per executed step (the library's CUDA events: stage_ms["decode"] / decode_steps).  A long-history arm
(4 s clip, --long-tokens new tokens: audio + prompt + generation stay within the fused step's 1,152 keys; it asserts
that every step ran fused) shows how the per-step history scan grows with n.  Prints one JSON line with the card's
name, power limit and maximum SM clock read in the same run.

    python bench_repetition.py [--rounds 7] [--warmup 2] [--new-tokens 128] [--long-tokens 900]
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
ARMS = (("off", {}), ("ngram3", dict(no_repeat_ngram_size=3)), ("penalty1.2", dict(repetition_penalty=1.2)),
        ("both", dict(no_repeat_ngram_size=3, repetition_penalty=1.2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--long-tokens", type=int, default=900)
    args = ap.parse_args()
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    out = {"metric": "decode step us per executed step, repetition controls off / N=3 / theta=1.2 / both "
                     "(Qwen3-ASR-0.6B dims)", "gpu": gpu_info(0), "shapes": {}}
    shapes = (("b1", 1, 30.0, args.new_tokens, "decode_fused_steps"), ("b8", 8, 30.0, args.new_tokens, "decode_batch_steps"),
              ("b1_long", 1, 4.0, args.long_tokens, "decode_fused_steps"))
    try:
        for label, B, secs, n_new, path in shapes:
            clips = [synth.make_clip(i, secs) for i in range(B)]

            def step_us(kw):
                before = eng.stats()
                r = eng.transcribe_ids(clips, max_new_tokens=n_new, **kw)
                after = eng.stats()
                moved = {k: after[k] - before.get(k, 0) for k in PATHS}
                return 1e3 * r.stage_ms["decode"] / max(r.decode_steps, 1), r.decode_steps, moved

            for _ in range(args.warmup):
                for _, kw in ARMS:
                    step_us(kw)
            times = {a: [] for a, _ in ARMS}
            steps, moved = {}, {}
            for _ in range(args.rounds):         # alternated: clock / thermal drift hits all arms alike
                for a, kw in ARMS:
                    t, steps[a], moved[a] = step_us(kw)
                    times[a].append(t)
            if label == "b1_long":
                assert all(m["decode_phase_steps"] == 0 and m["decode_fused_steps"] == steps[a] for a, m in moved.items()), moved
            med = {a: statistics.median(v) for a, v in times.items()}
            out["shapes"][label] = {
                "batch": B, "clip_s": secs, "new_tokens": n_new, "expected_path": path,
                **{f"step_us_{a}": round(med[a], 2) for a in med},
                **{f"spread_{a}_pct": round(100.0 * (max(v) - min(v)) / med[a], 3) for a, v in times.items()},
                **{f"overhead_{a}_pct": round(100.0 * (med[a] / med["off"] - 1.0), 3) for a in med if a != "off"},
                "decode_steps": steps, "steps_by_path": moved,
            }
    finally:
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
