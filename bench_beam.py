"""Cost of beam search (session options "beam_size" / "length_penalty") on the decode step.

Times the decode loop of Qwen3-ASR-0.6B dims (synthetic weights), 30 s clips, with the same slot count in both arms so
that the difference is the cost of the selection and the KV reorder: greedy batch 5 against beam 5 x batch 1, and
greedy batch 40 against beam 5 x batch 8, the arms alternated in one process.  A run may end early on EOS, so the figure
is the decode time per executed step (the library's CUDA events: stage_ms["decode"] / decode_steps).  Also reports the
KV bytes the beam runs copied (asrb_last_beam_stats) per step, and the card's name, power limit and maximum SM clock,
read in the same run.  Prints one JSON line.

    python bench_beam.py [--rounds 5] [--warmup 1] [--new-tokens 128]
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
K = 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    out = {"metric": "decode step us per executed step, greedy B*5 vs beam 5 x B (Qwen3-ASR-0.6B dims, 30 s clips)",
           "gpu": gpu_info(0), "shapes": {}}
    try:
        for label, B in (("b1", 1), ("b8", 8)):
            clips = [synth.make_clip(i, 30.0) for i in range(B)]
            arms = (("greedy", clips * K, {}), ("beam", clips, dict(beam_size=K)))

            def run(cl, kw):
                before = eng.stats()
                r = eng.transcribe_ids(cl, max_new_tokens=args.new_tokens, **kw)
                after = eng.stats()
                moved = {k: after[k] - before.get(k, 0) for k in PATHS}
                extra = eng.last_beam_stats() if kw else {}
                return 1e3 * r.stage_ms["decode"] / max(r.decode_steps, 1), r.decode_steps, moved, extra

            for _ in range(args.warmup):
                for _, cl, kw in arms:
                    run(cl, kw)
            times = {a: [] for a, _, _ in arms}
            steps, moved, beam = {}, {}, {}
            for _ in range(args.rounds):         # alternated: clock / thermal drift hits all arms alike
                for a, cl, kw in arms:
                    t, steps[a], moved[a], extra = run(cl, kw)
                    times[a].append(t)
                    if extra:
                        beam = extra
            med = {a: statistics.median(v) for a, v in times.items()}
            n = max(beam.get("beam_steps", 0), 1)
            out["shapes"][label] = {
                "batch": B, "beam": K, "slots": B * K, "new_tokens": args.new_tokens,
                **{f"step_us_{a}": round(med[a], 2) for a in med},
                **{f"spread_{a}_pct": round(100.0 * (max(v) - min(v)) / med[a], 3) for a, v in times.items()},
                "overhead_beam_pct": round(100.0 * (med["beam"] / med["greedy"] - 1.0), 3),
                "reorder_kv_bytes_per_step": round(beam.get("reorder_kv_bytes", 0) / n, 1),
                "slots_reassigned_per_step": round(beam.get("slots_reassigned", 0) / n, 3),
                "expand_kv_bytes": beam.get("expand_kv_bytes", 0),
                "decode_steps": steps, "steps_by_path": moved,
            }
    finally:
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
