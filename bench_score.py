"""Cost of teacher-forced scoring (asrb_score_ids) against decoding the same clips.

Qwen3-ASR-0.6B dims, synthetic weights, 30 s clips.  Three arms, alternated in one process after a warm-up:
  score      16 utterances x 1 candidate of 128 ids
  lid        1 utterance x 30 language candidates ("language Xxx" as 3 ids each, all sharing the prompt's prefill)
  reference  transcribe_ids of the same 16 clips with 128 new tokens
Times come from the library's CUDA events (asrb_last_timings): [3] the decoder layers of the prefill, [4] the score head
(gather, final norm, lm_head GEMM with the folding epilogue, merge) or the decode loop.  The head's achieved rate counts
3 planes x 2 x rows x vocab x hidden over [4]; 989 TFLOP/s is the H100 SXM data-sheet dense BF16 figure, printed beside
it for scale, not a measured one.  Prints one JSON line with the card's name, power limit and maximum SM clock read in the
same run.

    python bench_score.py [--rounds 7] [--warmup 2]
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

DATASHEET_BF16_TFLOPS = 989.0


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
    from qwen3_asr_rs_b200.text import LANGUAGES

    cfg = config_0p6b()
    t = cfg.text
    eng = AsrInference.from_weights(cfg, synth.make_weights(cfg, 1), device=0)
    clips = [synth.make_clip(i, 30.0) for i in range(16)]
    rng = np.random.default_rng(0)
    cands16 = [[[int(v) for v in rng.integers(0, t.vocab_size, 128)]] for _ in clips]
    lid = [[[11528, 3000 + i, 4000 + i] for i in range(len(LANGUAGES))]]

    def arm(name):
        if name == "score":
            eng.score_ids(clips, cands16)
            rows = 16 * 128
        elif name == "lid":
            eng.score_ids(clips[:1], lid)
            rows = 3 * len(LANGUAGES)
        else:
            eng.transcribe_ids(clips, max_new_tokens=128)
            rows = None
        ms, kernels = last_ms(eng)
        return ms[3], ms[4], ms[5], rows, kernels

    names = ("score", "lid", "reference")
    for _ in range(args.warmup):
        for n in names:
            arm(n)
    res = {n: [] for n in names}
    for _ in range(args.rounds):                 # alternated: clock / thermal drift hits all arms alike
        for n in names:
            res[n].append(arm(n))
    out = {"metric": "teacher-forced scoring vs decoding (Qwen3-ASR-0.6B dims, synthetic weights, 30 s clips)",
           "gpu": gpu_info(0), "rounds": args.rounds, "arms": {}}
    for n in names:
        pre = [r[0] for r in res[n]]; head = [r[1] for r in res[n]]; tot = [r[2] for r in res[n]]
        a = {"prefill_ms": round(statistics.median(pre), 3), "head_or_decode_ms": round(statistics.median(head), 3),
             "total_ms": round(statistics.median(tot), 3),
             "spread_head_pct": round(100.0 * (max(head) - min(head)) / statistics.median(head), 2),
             "spread_total_pct": round(100.0 * (max(tot) - min(tot)) / statistics.median(tot), 2),
             "kernels": res[n][-1][4]}
        rows = res[n][0][3]
        if rows is not None:
            flop = 3 * 2.0 * rows * t.vocab_size * t.hidden_size
            a.update(rows=rows, rows_per_s=round(rows / (statistics.median(tot) * 1e-3), 1),
                     head_tflops=round(flop / (statistics.median(head) * 1e-3) / 1e12, 1),
                     head_share_of_datasheet_bf16=round(flop / (statistics.median(head) * 1e-3) / 1e12 / DATASHEET_BF16_TFLOPS, 3))
        out["arms"][n] = a
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
