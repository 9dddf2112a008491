"""Long-form transcription: one pass over a 10 min recording against cutting it at quiet points and decoding the pieces
as batches (AsrInference.transcribe_long).

Runs Qwen3-ASR-0.6B dims (synthetic weights) on a 10 min file of make_clip pieces (8-29 s) separated by 0.4 s near-silent
gaps, as 16 kHz s16 PCM.  Two arms, alternated in one process, each on its own engine (their sessions differ: one row of
10 min against 16 rows of 30 s):
  (a) one pass: transcribe_pcm with max_new_tokens = segments x 128;
  (b) transcribe_long(max_segment_s=30, search_s=5, batch=16) with 128 new tokens per segment.
Synthetic weights never emit EOS, so both arms generate the same number of tokens.  Per arm: wall time (host clock
around the call, which ends in a device synchronise), real-time factor, the spread over rounds, and the decoder forwards
by path.  Also the segment count, the wave count, the time of one asrb_segment_long call (host clock; the call ends in a
stream synchronise and copies the cuts back), and the card's name, power limit and maximum SM clock, read in the same
run.  Prints one JSON line.

    python bench_longform.py [--rounds 3] [--warmup 1] [--minutes 10]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_logprobs import gpu_info  # noqa: E402

PATHS = ("decode_batch_steps", "decode_fused_steps", "decode_phase_steps")
SR = 16000


def make_recording(minutes: float):
    import numpy as np
    from qwen3_asr_rs_b200 import synth
    rng = np.random.default_rng(2026)
    parts, n, i = [], 0, 0
    while n < minutes * 60 * SR:
        clip = synth.make_clip(900 + i, float(rng.uniform(8.0, 29.0)))
        gap = (rng.standard_normal(int(0.4 * SR)) * 1e-4).astype(np.float32)
        parts += [clip, gap]
        n += len(clip) + len(gap)
        i += 1
    x = np.concatenate(parts)[: int(minutes * 60 * SR)]
    return (x * 32767).astype(np.int16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--new-tokens", type=int, default=128)
    args = ap.parse_args()
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    w = synth.make_weights(cfg, 1)
    pcm = make_recording(args.minutes)
    dur = len(pcm) / SR
    one = AsrInference.from_weights(cfg, w, device=0)
    seg = AsrInference.from_weights(cfg, w, device=0)
    out = {"metric": f"wall s and RTF: one pass vs transcribe_long on a {args.minutes:g} min recording "
                     f"(Qwen3-ASR-0.6B dims, {args.new_tokens} new tokens per segment)",
           "gpu": gpu_info(0), "audio_s": round(dur, 3)}
    try:
        seg.ingest_long([pcm], [SR])
        n_seg = len(seg.segment_long(30 * SR, 5 * SR)[0])
        budget = n_seg * args.new_tokens

        def run_one():
            r = one.transcribe_pcm([pcm], [SR], max_new_tokens=budget)
            return r.decode_steps + 1, len(r.ids[0])

        def run_seg():
            r = seg.transcribe_long([pcm], [SR], max_segment_s=30.0, search_s=5.0, batch=16,
                                    max_new_tokens=args.new_tokens)
            return r.n_waves, sum(len(s.ids) for s in r.files[0])

        arms = (("one_pass", one, run_one), ("segmented", seg, run_seg))

        def timed(eng, fn):
            before = eng.stats()
            t0 = time.perf_counter()
            info = fn()
            wall = time.perf_counter() - t0
            after = eng.stats()
            print(f"{fn.__name__}: {wall:.3f} s", file=sys.stderr, flush=True)      # progress of a long run
            return wall, info, {k: after[k] - before.get(k, 0) for k in PATHS}

        for _ in range(args.warmup):
            for _, eng, fn in arms:
                timed(eng, fn)
        walls = {a: [] for a, _, _ in arms}
        info, moved = {}, {}
        for _ in range(args.rounds):         # alternated: clock / thermal drift hits both arms alike
            for a, eng, fn in arms:
                wl, info[a], moved[a] = timed(eng, fn)
                walls[a].append(wl)
        seg.ingest_long([pcm], [SR])
        seg.segment_long(30 * SR, 5 * SR)
        ts = []
        for _ in range(20):
            t0 = time.perf_counter()
            seg.segment_long(30 * SR, 5 * SR)
            ts.append(1e3 * (time.perf_counter() - t0))
        med = {a: statistics.median(v) for a, v in walls.items()}
        out.update({
            "segments": n_seg, "waves": info["segmented"][0],
            "tokens": {"one_pass": info["one_pass"][1], "segmented": info["segmented"][1]},
            **{f"wall_s_{a}": round(m, 4) for a, m in med.items()},
            **{f"rtf_{a}": round(m / dur, 6) for a, m in med.items()},
            **{f"spread_{a}_pct": round(100.0 * (max(v) - min(v)) / med[a], 3) for a, v in walls.items()},
            "speedup_segmented_vs_one_pass": round(med["one_pass"] / med["segmented"], 3),
            "steps_by_path": moved,
            "segment_call_ms_median": round(statistics.median(ts), 4),
        })
    finally:
        one.close()
        seg.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
