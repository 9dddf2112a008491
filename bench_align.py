"""Cost of word-timing alignment (asrb_align_ids) against the transcription it follows.

Qwen3-ASR-0.6B dims, synthetic weights, 30 s clips, 128-id transcripts (127 ids + EOS, default heads: every query head
of layers 14..27), at batch 1 and 8.  Arms, alternated in one process after a warm-up:
  align      asrb_align_ids
  reference  transcribe_ids of the same clips with 128 new tokens
Stage times come from the library's CUDA events (asrb_last_timings): [1] mel, [2] encoder, [3] the decoder layers up to
the last listed one with the probability and fold kernels, [4] DTW, [5] the whole call.  The probability + fold share
of [3] is measured in a separate torch.profiler run (kernel names align_probs_kernel, align_zscore_kernel,
align_median_kernel), which also times align_dtw_kernel alone.  Prints one JSON line with the card's name, power limit
and maximum SM clock read in the same run.

    python bench_align.py [--rounds 7] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench_logprobs import gpu_info  # noqa: E402

EOS = 151645


def last_ms(eng):
    ms = (C.c_float * 6)()
    k, st = C.c_int64(), C.c_int64()
    eng._lib.asrb_last_timings(eng._session, ms, C.byref(k), C.byref(st))
    return list(ms), k.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth

    cfg = config_0p6b()
    t = cfg.text
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    clips = [synth.make_clip(i, 30.0) for i in range(8)]
    rng = np.random.default_rng(0)
    ids = [[int(v) for v in rng.integers(0, 151000, 127)] + [EOS] for _ in clips]

    def arm(name, B):
        if name == "align":
            eng.align_ids(clips[:B], ids[:B])
        else:
            eng.transcribe_ids(clips[:B], max_new_tokens=128)
        return last_ms(eng)

    out = {"metric": "word-timing alignment vs transcription (Qwen3-ASR-0.6B dims, synthetic weights, 30 s clips, "
                     "128-id transcripts, default heads)", "gpu": gpu_info(0), "rounds": args.rounds, "batches": {}}
    for B in (1, 8):
        for _ in range(args.warmup):
            arm("align", B)
            arm("reference", B)
        res = {"align": [], "reference": []}
        for _ in range(args.rounds):
            for n in res:
                res[n].append(arm(n, B))
        med = lambda n, i: round(statistics.median(r[0][i] for r in res[n]), 3)   # noqa: E731
        tot = [r[0][5] for r in res["align"]]
        a = {"mel_ms": med("align", 1), "encoder_ms": med("align", 2), "layers_probs_fold_ms": med("align", 3),
             "dtw_ms": med("align", 4), "total_ms": med("align", 5),
             "spread_total_pct": round(100.0 * (max(tot) - min(tot)) / statistics.median(tot), 2),
             "kernels": res["align"][-1][1], "transcribe_ids_ms": med("reference", 5)}
        a["align_over_transcribe"] = round(a["total_ms"] / a["transcribe_ids_ms"], 4)
        # kernel times of the alignment kernels, in a profiled run of their own
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                arm("align", B)
            torch.cuda.synchronize()
        sums = {}
        for ev in prof.events():
            for k in ("align_probs_kernel", "align_zscore_kernel", "align_median_kernel", "align_dtw_kernel"):
                if k in ev.name:
                    sums[k] = sums.get(k, 0.0) + ev.device_time / 1000.0 / 3
        a["profiled_ms_per_call"] = {k: round(v, 3) for k, v in sorted(sums.items())}
        a["probs_fold_ms"] = round(sum(v for k, v in sums.items() if k != "align_dtw_kernel"), 3)
        out["batches"][str(B)] = a
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
