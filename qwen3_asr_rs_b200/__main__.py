"""CLI mirroring the reference's `asr <model_dir> <audio_file> [language]` (/root/reference/src/main.rs:7-81).
`--logprobs` (anywhere on the line) also prints the utterance's average token log-probability."""
import sys


def parse_args(argv):
    """-> (model_dir, audio, language or None, logprobs) or None on a usage error."""
    logprobs = "--logprobs" in argv
    pos = [a for a in argv if a != "--logprobs"]
    if len(pos) < 2:
        return None
    return pos[0], pos[1], (pos[2] if len(pos) > 2 else None), logprobs


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    args = parse_args(argv)
    if args is None:
        print("Usage: python -m qwen3_asr_rs_b200 <model_dir> <audio_file> [language] [--logprobs]", file=sys.stderr)   # main.rs:18-27
        return 1
    model_dir, audio, language, logprobs = args
    from . import AsrInference
    eng = AsrInference.load(model_dir, device=0)
    try:
        r = eng.transcribe(audio, language, logprobs=logprobs)
    finally:
        eng.close()
    print(f"Language: {r.language}")                       # main.rs:77-78
    print(f"Text: {r.text}")
    if logprobs:
        print(f"Avg logprob: {r.avg_logprob:.4f}" if r.avg_logprob is not None else "Avg logprob: n/a")
    return 0


if __name__ == "__main__":
    sys.exit(main())
