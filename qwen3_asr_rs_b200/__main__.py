"""CLI mirroring the reference's `asr <model_dir> <audio_file> [language]` (/root/reference/src/main.rs:7-81).
`--logprobs` (anywhere on the line) also prints the utterance's average token log-probability.
`--top-logprobs N` (N in 1..8, anywhere on the line) also prints, for every generated token and the ending EOS, the N
best candidates of the step that selected it with their log-probabilities."""
import sys

USAGE = "Usage: python -m qwen3_asr_rs_b200 <model_dir> <audio_file> [language] [--logprobs] [--top-logprobs N]"


def parse_args(argv):
    """-> (model_dir, audio, language or None, logprobs) or None on a usage error."""
    logprobs = "--logprobs" in argv
    pos = [a for a in argv if a != "--logprobs"]
    if len(pos) < 2:
        return None
    return pos[0], pos[1], (pos[2] if len(pos) > 2 else None), logprobs


def split_top_logprobs(argv):
    """Remove `--top-logprobs N` / `--top-logprobs=N` from argv -> (remaining argv, N; 0 when absent), or None when
    the flag has no value or the value is not an integer in 1..8."""
    rest, k, i = [], 0, 0
    while i < len(argv):
        a = argv[i]
        if a == "--top-logprobs" or a.startswith("--top-logprobs="):
            if "=" in a:
                v = a.split("=", 1)[1]
            elif i + 1 < len(argv):
                v = argv[i + 1]
                i += 1
            else:
                return None
            if not v.isdigit() or not 1 <= int(v) <= 8:
                return None
            k = int(v)
        else:
            rest.append(a)
        i += 1
    return rest, k


def format_candidates(cands, decode) -> str:
    """One line of candidates: `'text' -0.0123` pairs, best first; `decode([id])` gives each candidate's text."""
    return "  ".join(f"{decode([i])!r} {lp:.4f}" for i, lp in cands)


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    split = split_top_logprobs(argv)
    args = parse_args(split[0]) if split is not None else None
    if args is None:
        print(USAGE, file=sys.stderr)   # main.rs:18-27
        return 1
    model_dir, audio, language, logprobs = args
    top = split[1]
    from . import AsrInference
    eng = AsrInference.load(model_dir, device=0)
    try:
        r = eng.transcribe(audio, language, logprobs=logprobs, top_logprobs=top)
        decode = eng.tokenizer.decode if eng.tokenizer is not None else (lambda ids: " ".join(str(i) for i in ids))
    finally:
        eng.close()
    print(f"Language: {r.language}")                       # main.rs:77-78
    print(f"Text: {r.text}")
    if logprobs:
        print(f"Avg logprob: {r.avg_logprob:.4f}" if r.avg_logprob is not None else "Avg logprob: n/a")
    if top:
        print("Top logprobs:")
        for t, cands in enumerate(r.top_logprobs):
            print(f"  [{t}] {format_candidates(cands, decode)}")
        if r.eos_top_logprobs is not None:
            print(f"  [eos] {format_candidates(r.eos_top_logprobs, decode)}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
