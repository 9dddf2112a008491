"""Streaming transcription: pushes on live streams (AsrInference.open_streams) against decoding the accumulated audio
again at every push.

Runs Qwen3-ASR-0.6B dims (synthetic weights) on 16 concurrent 60 s streams (synth.make_clip), 1 s pushes and
max_new_tokens = 8 per push.  Synthetic weights never emit EOS, so each push's hypothesis is the forced prefix plus 8
ids and the prefix grows by 8 - rollback = 3 ids per push.  Two arms, alternated push by push in one process, each on its
own engine:
  (a) stream: one asrb_stream_push on the 16 streams;
  (b) naive: transcribe_ids on the 16 accumulated prefixes with the same forced prefixes as language ids.
Per push and arm: device time per stage (asrb_last_timings: mel, encoder, prefill, decode) and the encoder windows and
prompt rows computed versus reused (the naive arm reuses nothing: its windows are ceil(chunks / 8) per stream and its
rows the whole prompts).  Also the card's name, power limit and maximum SM clock, read in the same run.  Prints one JSON
line.

    python bench_stream.py [--streams 16] [--seconds 60] [--push 1.0] [--max-new 8]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_logprobs import gpu_info  # noqa: E402

STAGES = ("h2d", "mel", "encoder", "prefill", "decode", "total")


def timings(eng):
    import ctypes as C
    from qwen3_asr_rs_b200 import _lib
    ms = (C.c_float * 6)()
    k, st = C.c_int64(), C.c_int64()
    _lib.check(eng._lib.asrb_last_timings(eng._session, ms, C.byref(k), C.byref(st)))
    return dict(zip(STAGES, [round(float(v), 3) for v in ms]))


def naive_counts(n_samples, prefix_lens):
    """Encoder windows and prompt rows of transcribe_ids on the accumulated audio (released dims, no language ids)."""
    windows = rows = 0
    for n, p in zip(n_samples, prefix_lens):
        F = -(-n // 160)
        C_ = -(-F // 100)
        T = 0
        for k in range(C_):
            f = min(100, F - 100 * k)
            for _ in range(3):
                f = (f - 1) // 2 + 1
            T += f
        windows += -(-C_ // 8)
        rows += 9 + T + 6 + p
    return windows, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--push", type=float, default=1.0)
    ap.add_argument("--max-new", type=int, default=8)
    a = ap.parse_args()
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b, synth
    cfg = config_0p6b()
    w = synth.make_weights(cfg, 1)
    eng_s = AsrInference.from_weights(cfg, w, device=0)
    eng_n = AsrInference.from_weights(cfg, w, device=0)
    del w
    n = a.streams
    xs = [synth.make_clip(500 + b, a.seconds) for b in range(n)]
    step = int(round(a.push * 16000))
    bounds = list(range(step, len(xs[0]) + step, step))
    ss = eng_s.open_streams(n, a.seconds, max_new_tokens=a.max_new)
    per_push = []
    pos, prefixes = 0, [[] for _ in range(n)]
    t0 = time.time()
    for j, end in enumerate(bounds):
        end = min(end, len(xs[0]))
        final = j == len(bounds) - 1
        hyps = ss.push([x[pos:end] for x in xs], final=final)
        rec = {"n_s": round(end / 16000.0, 2), "stream": dict(ms=timings(eng_s), **ss.stats())}
        r = eng_n.transcribe_ids([x[:end] for x in xs], language_ids=[p if p else None for p in prefixes],
                                 max_new_tokens=a.max_new)
        wn, rn = naive_counts([end] * n, [len(p) for p in prefixes])
        rec["naive"] = dict(ms={k: round(float(v), 3) for k, v in r.stage_ms.items()}, windows_encoded=wn,
                            prompt_rows_computed=rn)
        per_push.append(rec)
        prefixes = [h.ids[: h.fixed] for h in hyps]
        pos = end
    wall = time.time() - t0

    def tot(arm, stage):
        return round(sum(p[arm]["ms"][stage] for p in per_push), 2)
    out = {
        "bench": "stream", "streams": n, "seconds": a.seconds, "push_s": a.push, "max_new_tokens": a.max_new,
        "model": "0.6B dims, synthetic weights", "gpu": gpu_info(0), "wall_s": round(wall, 2),
        "stream_total_ms": {s: tot("stream", s) for s in STAGES[1:]},
        "naive_total_ms": {s: tot("naive", s) for s in STAGES[1:]},
        "stream_windows": [sum(p["stream"]["windows_encoded"] for p in per_push), sum(p["stream"]["windows_reused"] for p in per_push)],
        "naive_windows": sum(p["naive"]["windows_encoded"] for p in per_push),
        "stream_rows": [sum(p["stream"]["prompt_rows_computed"] for p in per_push),
                        sum(p["stream"]["prompt_rows_kept"] for p in per_push)],
        "naive_rows": sum(p["naive"]["prompt_rows_computed"] for p in per_push),
        "last_push": per_push[-2] if len(per_push) > 1 else per_push[-1],
        "per_push": per_push,
    }
    print(json.dumps(out))
    eng_s.close()
    eng_n.close()


if __name__ == "__main__":
    main()
