"""Cost of per-token log-probabilities (session option "logprobs") and of top-k alternatives (option "top_logprobs")
on the decode step.

Times the greedy decode loop of Qwen3-ASR-0.6B dims (synthetic weights) with the options off, with logprobs on and
with top_logprobs = 5, the three alternated in one process: batch 1 (one 30 s clip, 128 new tokens: the headline shape, single-sequence fused step) and batch 8 (eight 30 s
clips, batched fused step).  The decode time per step comes from the library's CUDA events (stage_ms["decode"] /
decode_steps).  Prints one JSON line with the card's name, power limit and maximum SM clock read in the same run.

    python bench_logprobs.py [--rounds 7] [--warmup 2] [--new-tokens 128]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def gpu_info(device: int):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip()
        name, watts, mhz = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit_w": float(watts), "sm_max_mhz": float(mhz)}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    out = {"metric": "decode step us, logprobs off vs on vs top_logprobs=5 (Qwen3-ASR-0.6B dims, 30 s clips)",
           "gpu": gpu_info(0), "shapes": {}}
    try:
        for label, B, path in (("b1", 1, "decode_fused_steps"), ("b8", 8, "decode_batch_steps")):
            clips = [synth.make_clip(i, 30.0) for i in range(B)]

            def step_us(on: bool, top: int = 0):
                eng.set_option("logprobs", "1" if on else "0")
                eng.set_option("top_logprobs", str(top))
                before = eng.stats()
                r = eng.transcribe_ids(clips, max_new_tokens=args.new_tokens)
                after = eng.stats()
                moved = {k: after[k] - before.get(k, 0) for k in ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")}
                return 1e3 * r.stage_ms["decode"] / max(r.decode_steps, 1), r.ids, moved

            for _ in range(args.warmup):
                step_us(False)
                step_us(True)
                step_us(False, 5)
            off, on, top = [], [], []
            for _ in range(args.rounds):         # alternated: clock / thermal drift hits all arms alike
                t, ids_off, moved_off = step_us(False)
                off.append(t)
                t, ids_on, moved_on = step_us(True)
                on.append(t)
                t, ids_top, moved_top = step_us(False, 5)
                top.append(t)
            m_off, m_on, m_top = statistics.median(off), statistics.median(on), statistics.median(top)
            out["shapes"][label] = {
                "batch": B, "new_tokens": args.new_tokens,
                "step_us_off": round(m_off, 2), "step_us_on": round(m_on, 2),
                "overhead_pct": round(100.0 * (m_on / m_off - 1.0), 3),
                "spread_off_pct": round(100.0 * (max(off) - min(off)) / m_off, 3),
                "spread_on_pct": round(100.0 * (max(on) - min(on)) / m_on, 3),
                "step_us_top5": round(m_top, 2),
                "overhead_top5_pct": round(100.0 * (m_top / m_off - 1.0), 3),
                "spread_top5_pct": round(100.0 * (max(top) - min(top)) / m_top, 3),
                "ids_equal": ids_off == ids_on,
                "ids_equal_top5": ids_off == ids_top,
                "steps_by_path_off": moved_off, "steps_by_path_on": moved_on, "steps_by_path_top5": moved_top,
                "expected_path": path,
            }
    finally:
        eng.set_option("logprobs", "0")
        eng.set_option("top_logprobs", "0")
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
