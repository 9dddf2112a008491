"""CLI mirroring the reference's `asr <model_dir> <audio_file> [language]` (/root/reference/src/main.rs:7-81).
`--logprobs` (anywhere on the line) also prints the utterance's average token log-probability.
`--top-logprobs N` (N in 1..8, anywhere on the line) also prints, for every generated token and the ending EOS, the N
best candidates of the step that selected it with their log-probabilities.
`--temperature T[,T...]` samples with temperature T (a list is a fallback schedule), `--seed N` seeds the draw; both
anywhere on the line, and `Temperature: x` reports the temperature of the kept attempt.
`--beam-size N` (N in 1..6) decodes with beam search and prints an `N-best:` block of the ranked hypotheses with their
scores; `--length-penalty A` (A in [0, 10]) scores them with ((5 + n) / 6) ** A instead of the length.
`--context TEXT` or `--context-file PATH` (UTF-8), anywhere on the line, places TEXT in the prompt's system turn to bias
recognition towards its words (names, jargon, a keyword list).
`--no-repeat-ngram N` (N in 0..16) bans every token that would repeat an N-gram of the tokens generated so far, and
`--repetition-penalty P` (P in [1, 10]) penalises the logits of tokens generated so far; both anywhere on the line.
`--max-segment S` (seconds, anywhere on the line) cuts the recording at quiet points into segments of at most S seconds,
decodes them as batches and prints a `Segments:` block of `[start - end] text` lines.
`--stream S` (seconds, anywhere on the line) replays the file as a live stream in pushes of S seconds and prints each
push's fixed and unfixed text (`[t] fixed | unfixed`), then the final transcript.
`--word-timestamps` (anywhere on the line) also prints a `Words:` block of `[start - end] word` lines, from the
decoder's attention over the audio (with `--max-segment` too); not with `--stream`, `--score` or `--detect-language`."""
import sys

USAGE = ("Usage: python -m qwen3_asr_rs_b200 <model_dir> <audio_file> [language] [--logprobs] [--top-logprobs N] "
         "[--temperature T[,T...]] [--seed N] [--beam-size N] [--length-penalty A] [--context TEXT | --context-file PATH] "
         "[--no-repeat-ngram N] [--repetition-penalty P] [--max-segment S | --stream S] [--score TEXT | --detect-language] "
         "[--word-timestamps]")


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


def _take_flag(argv, name):
    """Remove `name V` / `name=V` from argv -> (remaining argv, V or None when absent), or None when it has no value."""
    rest, val, i = [], None, 0
    while i < len(argv):
        a = argv[i]
        if a == name or a.startswith(name + "="):
            if "=" in a:
                val = a.split("=", 1)[1]
            elif i + 1 < len(argv):
                val = argv[i + 1]
                i += 1
            else:
                return None
        else:
            rest.append(a)
        i += 1
    return rest, val


def split_sampling(argv):
    """Remove `--temperature T[,T...]` and `--seed N` from argv -> (remaining argv, temperature, seed), where temperature
    is None when absent, a float, or a tuple for a comma-separated schedule, and seed is 0 when absent; None when a value
    is missing or invalid."""
    from .inference import check_seed, check_temperature
    t = _take_flag(argv, "--temperature")
    if t is None:
        return None
    sd = _take_flag(t[0], "--seed")
    if sd is None:
        return None
    temperature, seed = None, 0
    try:
        if t[1] is not None:
            parts = t[1].split(",")
            vals = check_temperature(tuple(float(v) for v in parts))
            temperature = vals if len(parts) > 1 else vals[0]
        if sd[1] is not None:
            if not sd[1].isdigit():
                return None
            seed = check_seed(int(sd[1]))
    except ValueError:
        return None
    return sd[0], temperature, seed


def split_beam(argv):
    """Remove `--beam-size N` and `--length-penalty A` from argv -> (remaining argv, N; 1 when absent, A; None when
    absent), or None when a value is missing or invalid."""
    from .inference import check_beam
    k = _take_flag(argv, "--beam-size")
    if k is None:
        return None
    a = _take_flag(k[0], "--length-penalty")
    if a is None:
        return None
    try:
        if k[1] is not None and not k[1].isdigit():
            return None
        size, alpha = check_beam(int(k[1]) if k[1] is not None else 1, float(a[1]) if a[1] is not None else None)
    except ValueError:
        return None
    return a[0], size, alpha


def split_repetition(argv):
    """Remove `--no-repeat-ngram N` and `--repetition-penalty P` from argv -> (remaining argv, N; 0 when absent, P; 1.0
    when absent), or None when a value is missing or invalid."""
    from .inference import check_repetition
    n = _take_flag(argv, "--no-repeat-ngram")
    if n is None:
        return None
    p = _take_flag(n[0], "--repetition-penalty")
    if p is None:
        return None
    try:
        if n[1] is not None and not n[1].isdigit():
            return None
        size, penalty = check_repetition(int(n[1]) if n[1] is not None else 0, float(p[1]) if p[1] is not None else 1.0)
    except ValueError:
        return None
    return p[0], size, penalty


def split_context(argv):
    """Remove `--context TEXT` and `--context-file PATH` from argv -> (remaining argv, context text; None when absent),
    or None when a value is missing, both are given, or the file cannot be read as UTF-8."""
    c = _take_flag(argv, "--context")
    if c is None:
        return None
    f = _take_flag(c[0], "--context-file")
    if f is None or (c[1] is not None and f[1] is not None):
        return None
    text = c[1]
    if f[1] is not None:
        try:
            with open(f[1], encoding="utf-8") as fh:
                text = fh.read()
        except (OSError, UnicodeDecodeError):
            return None
    return f[0], text


def split_score(argv):
    """Remove `--score TEXT` and `--detect-language` from argv -> (remaining argv, text to score or None, detect), or
    None when the text is missing or both are given."""
    c = _take_flag(argv, "--score")
    if c is None:
        return None
    rest = [a for a in c[0] if a != "--detect-language"]
    detect = len(rest) != len(c[0])
    if detect and c[1] is not None:
        return None
    return rest, c[1], detect


def split_max_segment(argv):
    """Remove `--max-segment S` from argv -> (remaining argv, S in seconds; None when absent), or None when the value is
    missing or not a valid segment length (a whole number of 10 ms, at least 5 s)."""
    from .inference import check_segmenting, default_search_s
    m = _take_flag(argv, "--max-segment")
    if m is None:
        return None
    if m[1] is None:
        return m[0], None
    try:
        s = float(m[1])
        check_segmenting(s, default_search_s(s))
    except ValueError:
        return None
    return m[0], s


def split_stream(argv):
    """Remove `--stream S` from argv -> (remaining argv, S in seconds; None when absent), or None when the value is
    missing or not a push length in whole 10 ms from 0.1 s to 30 s."""
    m = _take_flag(argv, "--stream")
    if m is None:
        return None
    if m[1] is None:
        return m[0], None
    try:
        s = float(m[1])
    except ValueError:
        return None
    if not (0.1 <= s <= 30.0) or abs(s * 100 - round(s * 100)) > 1e-6:
        return None
    return m[0], s


STREAM_PART_S = 30.0          # a recording is streamed in parts of at most this long, each a stream of its own


def stream_pushes(n_samples: int, push_s: float):
    """(start, end, final) sample ranges of the pushes replaying n_samples in pushes of push_s seconds.  A part's last
    push is final: the stream ends there, and the next part is a new stream."""
    step = int(round(push_s * 16000))
    per_part = max(1, int(STREAM_PART_S * 16000) // step)
    out = []
    for k, a in enumerate(range(0, n_samples, step)):
        b = min(a + step, n_samples)
        out.append((a, b, b == n_samples or (k + 1) % per_part == 0))
    return out


def split_word_timestamps(argv):
    """Remove `--word-timestamps` from argv -> (remaining argv, whether it was there)."""
    rest = [a for a in argv if a != "--word-timestamps"]
    return rest, len(rest) != len(argv)


def format_segment(start_s: float, end_s: float, text: str) -> str:
    """One line of the `Segments:` block."""
    return f"  [{start_s:.2f} - {end_s:.2f}] {text}"


def format_candidates(cands, decode) -> str:
    """One line of candidates: `'text' -0.0123` pairs, best first; `decode([id])` gives each candidate's text."""
    return "  ".join(f"{decode([i])!r} {lp:.4f}" for i, lp in cands)


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    argv, words = split_word_timestamps(argv)
    seg = split_max_segment(argv)
    if seg is None:
        print(USAGE, file=sys.stderr)
        return 1
    argv, max_segment = seg
    sm = split_stream(argv)
    if sm is None or (sm[1] is not None and max_segment is not None):
        print(USAGE, file=sys.stderr)
        return 1
    argv, stream_s = sm
    sc = split_score(argv)
    if sc is None:
        print(USAGE, file=sys.stderr)
        return 1
    argv, score_text, detect = sc
    rep = split_repetition(argv)
    ctx = split_context(rep[0]) if rep is not None else None
    beam = split_beam(ctx[0]) if ctx is not None else None
    sampling = split_sampling(beam[0]) if beam is not None else None
    split = split_top_logprobs(sampling[0]) if sampling is not None else None
    args = parse_args(split[0]) if split is not None else None
    if args is None:
        print(USAGE, file=sys.stderr)   # main.rs:18-27
        return 1
    model_dir, audio, language, logprobs = args
    top = split[1]
    _, beam_size, length_penalty = beam
    temperature = sampling[1]
    if stream_s is not None and (score_text is not None or detect or logprobs or top or beam_size > 1
                                 or isinstance(temperature, tuple)):
        print("--stream cannot be combined with --score, --detect-language, --logprobs, --top-logprobs, --beam-size or "
              "a temperature schedule", file=sys.stderr)
        print(USAGE, file=sys.stderr)
        return 1
    if words and (stream_s is not None or score_text is not None or detect):
        print("--word-timestamps cannot be combined with --stream, --score or --detect-language", file=sys.stderr)
        print(USAGE, file=sys.stderr)
        return 1
    if beam_size > 1 and (top or (temperature is not None and not isinstance(temperature, tuple) and temperature > 0)):
        print("--beam-size > 1 cannot be combined with --top-logprobs or a temperature > 0", file=sys.stderr)
        print(USAGE, file=sys.stderr)
        return 1
    from . import AsrInference
    eng = AsrInference.load(model_dir, device=0)
    if (score_text is not None or detect) and eng.tokenizer is None:
        eng.close()
        print(f"--score / --detect-language need tokenizer.json in {model_dir}", file=sys.stderr)
        return 1
    if stream_s is not None:
        try:
            return _stream_file(eng, audio, language, stream_s, ctx[1] or None, rep, sampling)
        finally:
            eng.close()
    if score_text is not None or detect:
        try:
            if detect:
                for name, p in eng.detect_language(audio)[:5]:
                    print(f"{name}\t{p:.4f}")
            else:
                r = eng.score(audio, [score_text], language=language, context=ctx[1] or None)[0]
                for t, lp in zip(r.ids, r.logprobs):
                    print(f"{t}\t{lp:.6f}")
                print(f"sum\t{r.sum_logprob:.6f}")
        finally:
            eng.close()
        return 0
    try:
        _, temperature, seed = sampling
        kw = {} if temperature is None else dict(temperature=temperature, seed=seed)
        if beam_size > 1:
            kw.update(beam_size=beam_size, length_penalty=length_penalty)
        if ctx[1]:
            kw.update(context=ctx[1])
        if max_segment is not None:
            kw.update(max_segment_s=max_segment)
        if rep[1] or rep[2] != 1.0:
            kw.update(no_repeat_ngram_size=rep[1], repetition_penalty=rep[2])
        if words:
            kw.update(word_timestamps=True)
        r = eng.transcribe(audio, language, logprobs=logprobs, top_logprobs=top, **kw)
        decode = eng.tokenizer.decode if eng.tokenizer is not None else (lambda ids: " ".join(str(i) for i in ids))
    finally:
        eng.close()
    print(f"Language: {r.language}")                       # main.rs:77-78
    print(f"Text: {r.text}")
    if r.temperature is not None:
        print(f"Temperature: {r.temperature:g}")
    if logprobs:
        print(f"Avg logprob: {r.avg_logprob:.4f}" if r.avg_logprob is not None else "Avg logprob: n/a")
    if top:
        print("Top logprobs:")
        for t, cands in enumerate(r.top_logprobs):
            print(f"  [{t}] {format_candidates(cands, decode)}")
        if r.eos_top_logprobs is not None:
            print(f"  [eos] {format_candidates(r.eos_top_logprobs, decode)}")
    if r.nbest is not None:
        print("N-best:")
        for j, (text, score) in enumerate(r.nbest):
            print(f"  [{j}] {score:.4f} {text}")
    if r.segments is not None:
        print("Segments:")
        for start_s, end_s, text in r.segments:
            print(format_segment(start_s, end_s, text))
    if r.words is not None:
        print("Words:")
        for w in r.words:
            print(format_segment(w.start_s, w.end_s, w.text.strip()))
    return 0


def _stream_file(eng, audio: str, language, push_s: float, context, rep, sampling) -> int:
    """--stream: the file's 16 kHz samples (GPU ingest) pushed as live streams of at most STREAM_PART_S each."""
    from .audio import read_wav_pcm
    from .text import join_segment_texts
    _, temperature, seed = sampling
    pcm, rate = read_wav_pcm(audio)
    x = eng.ingest_pcm([pcm], [rate])[0]
    decode = eng.tokenizer.decode if eng.tokenizer is not None else (lambda ids: " ".join(str(i) for i in ids))
    ss, start, texts = None, 0, []
    for a, b, final in stream_pushes(len(x), push_s):
        if ss is None:
            ss = eng.open_streams(1, STREAM_PART_S + 0.02, language=language, context=context, temperature=temperature or 0.0,
                                  seed=seed or 0, no_repeat_ngram_size=rep[1], repetition_penalty=rep[2])
        if final and b < len(x) and len(x) - b <= 160:      # a stream needs > 160 samples: the last bit joins this part
            b = len(x)
        h = ss.push([x[a:b]], final=final)[0]
        fixed = h.fixed_text if h.fixed_text is not None else decode(h.ids[: h.fixed])
        text = h.text if h.text is not None else decode(h.ids)
        print(f"[{b / 16000.0:.2f}] {fixed} | {text[len(fixed):] if text.startswith(fixed) else text}")
        if final:
            texts.append(text)
            ss = None
        if b == len(x):
            break
    print(f"Text: {join_segment_texts(texts, language)}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
