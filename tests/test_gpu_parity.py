"""GPU: the CUDA hot path (through the C ABI) vs the CPU oracle on identical seeded inputs.

Tolerances (floating point; the oracle is fp32 and itself only reproducible to
summation-order noise, e.g. 1.7e-5 between two FFT implementations of the mel --
oracle/pin_against_hf.py):
  mel        max |d| <= 2e-4   (values in [-0.7, 1.4])
  encoder    max |d| <= 1e-3 * max|ref|
  logits     max |d| <= 2e-3 * max|ref|
  token ids  exact equality with the oracle's greedy output
"""
import numpy as np
import pytest

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth

pytestmark = pytest.mark.gpu

MEL_TOL, ENC_RTOL, LOGIT_RTOL = 2e-4, 1e-3, 2e-3


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("seconds", [0.02, 0.5, 1.003, 3.07, 11.55, 30.0])
def test_mel_parity(tiny_engine, report, seconds):
    x = synth.make_clip(11, seconds)
    got = tiny_engine.mel([x])[0]
    ref = O.extract_mel(x).numpy()
    assert got.shape == ref.shape
    err = float(np.abs(got - ref).max())
    report[f"mel_abs_err_{seconds}s"] = err
    assert err <= MEL_TOL


def test_mel_batch_ragged(tiny_engine, report):
    clips = [synth.make_clip(20 + i, s) for i, s in enumerate([2.0, 0.31, 7.77, 1.0])]
    got = tiny_engine.mel(clips)
    for g, c in zip(got, clips):
        ref = O.extract_mel(c).numpy()
        assert g.shape == ref.shape and np.abs(g - ref).max() <= MEL_TOL


def test_mel_pure_noise_and_silence(tiny_engine):
    rng = np.random.default_rng(0)
    noise = (rng.standard_normal(16000) * 0.1).astype(np.float32)
    silence = np.zeros(8000, np.float32)
    got = tiny_engine.mel([noise, silence])
    assert np.abs(got[0] - O.extract_mel(noise).numpy()).max() <= MEL_TOL
    assert np.abs(got[1] - O.extract_mel(silence).numpy()).max() <= MEL_TOL


@pytest.mark.parametrize("seconds", [0.6, 1.0, 5.0, 8.0, 8.5, 11.55, 30.0])
def test_encoder_parity(tiny, tiny_engine, report, seconds):
    """covers: single chunk, tail chunks of assorted lengths, C <= 8 (mask None), C > 8 (windows)."""
    _, _, model = tiny
    x = synth.make_clip(31, seconds)
    tiny_engine.mel([x])
    got = tiny_engine.encode()[0]
    ref = model.encode(O.extract_mel(x)).numpy()
    assert got.shape == ref.shape
    r = _rel(got, ref)
    report[f"enc_rel_err_{seconds}s"] = r
    assert r <= ENC_RTOL


@pytest.mark.parametrize("tail_frames", [1, 2, 7, 8, 9, 16, 17, 33, 50, 64, 65, 99])
def test_encoder_tail_chunk_lengths(tiny, tiny_engine, tail_frames):
    _, _, model = tiny
    n = (100 + tail_frames) * 160 - 37            # ragged sample count inside the last frame
    x = synth.make_clip(40 + tail_frames, n / 16000.0)[:n]
    tiny_engine.mel([x])
    got = tiny_engine.encode()[0]
    ref = model.encode(O.extract_mel(x)).numpy()
    assert got.shape == ref.shape == (13 + O.feat_extract_output_length(tail_frames), 256)
    assert _rel(got, ref) <= ENC_RTOL


def test_encoder_batch_mixed_windows(tiny, tiny_engine):
    _, _, model = tiny
    clips = [synth.make_clip(50 + i, s) for i, s in enumerate([3.3, 12.0, 0.9, 17.5])]
    tiny_engine.mel(clips)
    got = tiny_engine.encode()
    for g, c in zip(got, clips):
        ref = model.encode(O.extract_mel(c)).numpy()
        assert g.shape == ref.shape and _rel(g, ref) <= ENC_RTOL


def test_prefill_and_step_logits(tiny, tiny_engine, report):
    _, _, model = tiny
    x = synth.make_clip(60, 6.2)
    ref = O.transcribe_ids(model, x, max_new_tokens=6, keep_logits=True)
    tiny_engine.mel([x])
    tiny_engine.encode()
    seq, logits = tiny_engine.prefill()
    assert seq[0] == ref.audio_embeds.shape[0] + 15
    r0 = _rel(logits[0], ref.prefill_logits.numpy())
    report["prefill_logits_rel_err"] = r0
    assert r0 <= LOGIT_RTOL
    for i in range(5):
        nxt, lg = tiny_engine.decode_step()
        assert nxt[0] == ref.ids[i]
        r = _rel(lg[0], ref.step_logits[i].numpy())
        report[f"step{i}_logits_rel_err"] = r
        assert r <= LOGIT_RTOL


@pytest.mark.parametrize("decode", ["phases", "mega"])
def test_token_ids_exact_tiny(tiny, tiny_engine, report, decode):
    _, _, model = tiny
    tiny_engine.set_option("decode", decode)
    try:
        for idx, sec, n_new in [(70, 4.0, 48), (71, 12.3, 32), (72, 0.8, 40)]:
            x = synth.make_clip(idx, sec)
            ref = O.transcribe_ids(model, x, max_new_tokens=n_new, keep_logits=True)
            got = tiny_engine.transcribe_ids([x], max_new_tokens=n_new)
            margins = [float(l.topk(2).values[0] - l.topk(2).values[1]) for l in [ref.prefill_logits] + ref.step_logits[:-1]]
            report[f"ids_{decode}_{idx}_min_margin"] = min(margins)
            assert got.ids[0] == ref.ids, (decode, idx, min(margins))
    finally:
        tiny_engine.set_option("decode", "mega")


def test_token_ids_batch_and_forced_language(tiny, tiny_engine):
    _, _, model = tiny
    clips = [synth.make_clip(80 + i, s) for i, s in enumerate([2.5, 9.1, 5.0])]
    lang = [None, [11528, 6364], [11528, 8453, 55]]     # arbitrary in-vocab ids standing in for "language Xxx"
    got = tiny_engine.transcribe_ids(clips, language_ids=lang, max_new_tokens=20)
    for g, c, l in zip(got.ids, clips, lang):
        ref = O.transcribe_ids(model, c, language_ids=l, max_new_tokens=20)
        assert g == ref.ids


def test_eos_stops_generation(tiny):
    """EOS semantics (inference.rs:161-166): a model whose argmax is EOS right after prefill
    generates nothing; built by making the EOS embedding row dominate the tied lm_head."""
    import torch
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    cfg, w, _ = tiny
    w2 = dict(w)
    e = w["thinker.model.embed_tokens.weight"].float().clone()
    x = synth.make_clip(90, 1.5)
    base = O.OracleModel(cfg, w2)
    r = O.transcribe_ids(base, x, max_new_tokens=3)
    # make token r.ids[1]'s successor EOS: copy a scaled version of the 2nd generated token's row direction
    e[151645] = e[r.ids[2]] * 1.5
    w2["thinker.model.embed_tokens.weight"] = e.bfloat16()
    model = O.OracleModel(cfg, w2)
    ref = O.transcribe_ids(model, x, max_new_tokens=12)
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    try:
        got = eng.transcribe_ids([x], max_new_tokens=12)
    finally:
        eng.close()
    assert got.ids[0] == ref.ids
    assert len(ref.ids) < 12          # EOS actually hit


def test_errors_are_statuses(tiny_engine):
    from qwen3_asr_rs_b200._lib import AsrbError
    with pytest.raises(AsrbError):
        tiny_engine.mel([np.zeros(100, np.float32)])           # too short for reflect padding


def test_full_size_0p6b_one_clip(report):
    """Qwen3-ASR-0.6B dims, one 30 s clip (BASELINE.json configs[1] shape), synthetic weights:
    exact ids + logits tolerance against the oracle run on the host cores."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    w = synth.make_weights(cfg, 1)
    x = synth.make_clip(0, 30.0)
    n_new = 24
    ref = O.transcribe_ids(O.OracleModel(cfg, w), x, max_new_tokens=n_new, keep_logits=True, lm_head_all_rows=False)
    eng = AsrInference.from_weights(config_0p6b(), w, device=0)
    try:
        mel = eng.mel([x])[0]
        report["full_mel_abs_err"] = float(np.abs(mel - ref.mel.numpy()).max())
        enc = eng.encode()[0]
        report["full_enc_rel_err"] = _rel(enc, ref.audio_embeds.numpy())
        seq, logits = eng.prefill()
        report["full_prefill_logits_rel_err"] = _rel(logits[0], ref.prefill_logits.numpy())
        assert seq[0] == 405 and enc.shape == (390, 1024)
        got = eng.transcribe_ids([x], max_new_tokens=n_new)
        margins = [float(l.topk(2).values[0] - l.topk(2).values[1]) for l in [ref.prefill_logits] + ref.step_logits[:-1]]
        report["full_min_margin"] = min(margins)
        report["full_stage_ms"] = got.stage_ms
        assert report["full_mel_abs_err"] <= MEL_TOL
        assert report["full_enc_rel_err"] <= ENC_RTOL
        assert report["full_prefill_logits_rel_err"] <= LOGIT_RTOL
        assert got.ids[0] == ref.ids
    finally:
        eng.close()


def test_full_size_1p7b_short_clip(report):
    """Qwen3-ASR-1.7B dims (BASELINE.json configs[3] model; dims as recalled in SURVEY.md section 8), one 10 s clip,
    synthetic weights: exact ids + logits tolerance.  The 6 ids run on the fused single-sequence step's 1.7B
    instantiation; the per-phase path at 1.7B widths is covered by tests/test_decode_variants_fp64.py."""
    from qwen3_asr_rs_b200 import AsrInference, config_1p7b
    cfg = O.cfg_1p7b()
    w = synth.make_weights(cfg, 3)
    x = synth.make_clip(7, 10.0)
    n_new = 6
    ref = O.transcribe_ids(O.OracleModel(cfg, w), x, max_new_tokens=n_new, keep_logits=True, lm_head_all_rows=False)
    eng = AsrInference.from_weights(config_1p7b(), w, device=0)
    try:
        eng.mel([x])
        enc = eng.encode()[0]
        report["full1p7b_enc_rel_err"] = _rel(enc, ref.audio_embeds.numpy())
        seq, logits = eng.prefill()
        report["full1p7b_prefill_logits_rel_err"] = _rel(logits[0], ref.prefill_logits.numpy())
        assert enc.shape == (130, 2048) and seq[0] == 145
        got = eng.transcribe_ids([x], max_new_tokens=n_new)
        report["full1p7b_stage_ms"] = got.stage_ms
        assert report["full1p7b_enc_rel_err"] <= ENC_RTOL
        assert report["full1p7b_prefill_logits_rel_err"] <= LOGIT_RTOL
        assert got.ids[0] == ref.ids
    finally:
        eng.close()


@pytest.mark.parametrize("shards", [1, 3])
def test_model_load_from_directory(tiny, tmp_path, shards):
    """AsrInference::load (inference.rs:30-86): config.json + model.safetensors / sharded index
    (weights.rs:10-58) parsed by the C++ loader must behave exactly like in-memory construction."""
    from qwen3_asr_rs_b200 import AsrInference
    from qwen3_asr_rs_b200._lib import AsrbError
    cfg, w, model = tiny
    d = tmp_path / f"model{shards}"
    synth.write_checkpoint(str(d), cfg, w, shards=shards)
    x = synth.make_clip(95, 3.3)
    ref = O.transcribe_ids(model, x, max_new_tokens=10)
    eng = AsrInference.load(str(d), device=0)
    try:
        assert eng.config.text.hidden_size == 256 and eng.config.audio.d_model == 128
        got = eng.transcribe_ids([x], max_new_tokens=10)
    finally:
        eng.close()
    assert got.ids[0] == ref.ids
    with pytest.raises(AsrbError):
        AsrInference.load(str(tmp_path / "does_not_exist"), device=0)


def test_token_ids_batch_larger_than_8(tiny, tiny_engine):
    """batch 11: the batched fused step at NB = 16 (the per-phase path's sub-batches of 8 are covered by
    tests/test_decode_variants_fp64.py); utterances stay independent (the reference is batch-1, so batch semantics ==
    B independent runs of it)."""
    _, _, model = tiny
    secs = [1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9, 5.3, 1.4, 2.8]
    clips = [synth.make_clip(200 + i, s) for i, s in enumerate(secs)]
    got = tiny_engine.transcribe_ids(clips, max_new_tokens=10)
    for g, c in zip(got.ids, clips):
        assert g == O.transcribe_ids(model, c, max_new_tokens=10).ids


def test_long_generation_beyond_ten_splits(tiny, tiny_engine):
    """A 30 s prompt (405 keys) + 300 new tokens: the fused decode step runs with up to 12 attention splits of 64
    cached keys per kv head (contexts up to 1152 keys are covered by 18 splits)."""
    _, _, model = tiny
    x = synth.make_clip(300, 30.0)
    n_new = 300
    ref = O.transcribe_ids(model, x, max_new_tokens=n_new)
    got = tiny_engine.transcribe_ids([x], max_new_tokens=n_new)
    assert len(ref.ids) == n_new
    assert got.ids[0] == ref.ids
    assert got.decode_steps == n_new - 1


def test_long_generation_crosses_fused_step_limit(tiny, tiny_engine):
    """The fused decode step covers contexts up to 1152 keys; a 60 s prompt (795) + 400 new tokens crosses it
    mid-generation and must continue seamlessly on the per-phase path (same KV cache, same state)."""
    _, _, model = tiny
    x = synth.make_clip(302, 60.0)
    n_new = 400
    ref = O.transcribe_ids(model, x, max_new_tokens=n_new)
    got = tiny_engine.transcribe_ids([x], max_new_tokens=n_new)
    assert len(ref.ids) == n_new
    assert got.ids[0] == ref.ids
    assert got.decode_steps == n_new - 1
    assert got.kernels_launched > 2 * got.decode_steps          # the tail ran as per-phase kernels (fused: 1 launch per step)


def test_max_new_tokens_one(tiny, tiny_engine):
    _, _, model = tiny
    x = synth.make_clip(301, 1.7)
    assert tiny_engine.transcribe_ids([x], max_new_tokens=1).ids[0] == O.transcribe_ids(model, x, max_new_tokens=1).ids


def test_transcribe_file_end_to_end(tiny, tmp_path):
    """AsrInference::{load, transcribe} (inference.rs:30-213) through the public API: model directory with
    config.json + safetensors + tokenizer.json, a 24 kHz stereo WAV on disk -> text.  The tokenizer is a synthetic
    word-level vocabulary (id i <-> "t<i>") so that the decoded string identifies the generated ids."""
    import json
    import wave
    from qwen3_asr_rs_b200 import AsrInference
    from qwen3_asr_rs_b200.audio import load_wav
    cfg, w, model = tiny
    d = tmp_path / "model"
    synth.write_checkpoint(str(d), cfg, w)
    vocab = {f"t{i}": i for i in range(cfg.text.vocab_size)}
    tok = {"version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": None,
           "pre_tokenizer": {"type": "Whitespace"}, "post_processor": None, "decoder": None,
           "model": {"type": "WordLevel", "vocab": vocab, "unk_token": "t0"}}
    (d / "tokenizer.json").write_text(json.dumps(tok))
    x24 = synth.make_clip(77, 2.0, sample_rate=24000)
    pcm = (np.stack([x24, x24], 1) * 32767).astype("<i2")
    wav = tmp_path / "clip.wav"
    with wave.open(str(wav), "wb") as f:
        f.setnchannels(2); f.setsampwidth(2); f.setframerate(24000); f.writeframes(pcm.tobytes())
    samples = load_wav(str(wav))
    ref = O.transcribe_ids(model, samples, max_new_tokens=8)
    eng = AsrInference.load(str(d), device=0)
    try:
        r = eng.transcribe(str(wav), max_new_tokens=8)
        forced = eng.transcribe(str(wav), language="english", max_new_tokens=8)
    finally:
        eng.close()
    assert r.ids == ref.ids
    assert r.raw_output.split() == [f"t{i}" for i in ref.ids]
    assert r.language == "unknown"
    # "language English" -> two unknown words -> unk id 0 twice
    ref_forced = O.transcribe_ids(model, samples, language_ids=[0, 0], max_new_tokens=8)
    assert forced.language == "forced" and forced.ids == ref_forced.ids


# ------------------------------------------------------------------------------------------------------
# batch-aware fused decode step (decode_batch.cu) and full-size batches
# ------------------------------------------------------------------------------------------------------
NOISE_REL = 1.5e-5      # measured logits deviation vs the oracle (summation order), relative to max|logit|
MARGIN_FLOOR_REL = 4 * NOISE_REL   # an exact-id comparison is only meaningful above this top-1/top-2 gap


def _min_rel_margin(ref):
    ls = [ref.prefill_logits] + ref.step_logits[:-1]
    gaps = [float(l.topk(2).values[0] - l.topk(2).values[1]) for l in ls]
    mx = max(float(l.abs().max()) for l in ls)
    return min(gaps) / mx


@pytest.mark.parametrize("secs", [[2.5, 5.0], [2.5, 9.1, 5.0], [1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9],
                                  [1.1, 2.3, 0.7, 4.9, 3.1, 1.9, 2.2, 0.9, 5.3], [12.0] * 16, [30.0, 12.0, 20.0, 3.0, 25.0]])
def test_batch_step_tiny(tiny, tiny_engine, secs):
    """decode_batch.cu (weights streamed once for all sequences): ragged batches of 2..16, NB = 8 and 16 instantiations,
    one and several 64 / 32-key attention splits per sequence -- ids equal the oracle's AND the per-sequence fused step's."""
    _, _, model = tiny
    clips = [synth.make_clip(400 + i, s) for i, s in enumerate(secs)]
    n_new = 14
    try:
        tiny_engine.set_option("batch_step", "1")
        before = tiny_engine.stats()
        got = tiny_engine.transcribe_ids(clips, max_new_tokens=n_new)
        assert got.decode_steps == n_new - 1
        st = tiny_engine.stats()              # (counters restart when the engine re-creates its session for a larger batch)
        fresh = st["decode_batch_steps"] < before.get("decode_batch_steps", 0) + n_new - 1
        base = {} if fresh else before
        assert st["decode_batch_steps"] - base.get("decode_batch_steps", 0) == n_new - 1      # the batched kernel really ran
        assert st["decode_phase_steps"] - base.get("decode_phase_steps", 0) == 0
        got = got.ids
        tiny_engine.set_option("batch_step", "0")
        per_seq = tiny_engine.transcribe_ids(clips, max_new_tokens=n_new).ids
    finally:
        tiny_engine.set_option("batch_step", "1")
    assert got == per_seq
    for g, c in zip(got, clips):
        assert g == O.transcribe_ids(model, c, max_new_tokens=n_new).ids


def test_peaked_untied_head_tiny(report):
    """Untied lm_head (the `thinker.lm_head.weight` key, src/text_decoder.rs:75-79) with peaked logits (synth.make_weights
    peaked_head): exact ids with a top-1/top-2 gap well above summation-order noise, batch 1 (fused step) and batch 5."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    cfg = O.cfg_tiny()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 7, peaked_head=True)
    model = O.OracleModel(cfg, w)
    ecfg = config_tiny()
    ecfg.text.tie_word_embeddings = False
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        # clips picked by their oracle-side worst gap (>= 1.3e-3 of max|logit|; 502 / 504 sit at 2e-5 / 1.4e-4)
        clips = [synth.make_clip(i, s) for i, s in [(500, 4.0), (501, 12.3), (507, 1.5), (503, 7.7), (505, 4.0)]]
        refs = [O.transcribe_ids(model, c, max_new_tokens=40, keep_logits=True) for c in clips]
        report["peaked_tiny_min_rel_margin"] = min(_min_rel_margin(r) for r in refs)
        assert report["peaked_tiny_min_rel_margin"] >= 10 * MARGIN_FLOOR_REL
        assert eng.transcribe_ids(clips[:1], max_new_tokens=40).ids[0] == refs[0].ids
        got = eng.transcribe_ids(clips, max_new_tokens=40).ids
        for g, r in zip(got, refs):
            assert g == r.ids
        assert len({i for r in refs for i in r.ids}) > 20          # not a degenerate one-token model
    finally:
        eng.close()


@pytest.fixture(scope="module")
def full_peaked():
    """Qwen3-ASR-0.6B dims, synthetic weights with the peaked untied head: (oracle model, engine)."""
    from qwen3_asr_rs_b200 import AsrInference, config_0p6b
    cfg = O.cfg_0p6b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 1, peaked_head=True)
    ecfg = config_0p6b()
    ecfg.text.tie_word_embeddings = False
    eng = AsrInference.from_weights(ecfg, w, device=0)
    yield O.OracleModel(cfg, w), eng
    eng.close()


def test_full_size_0p6b_batch8_30s_128_tokens(full_peaked, report):
    """north_star shape: Qwen3-ASR-0.6B, batch 8 x 30 s, 128 new tokens per clip -- exact ids for every clip through the
    batch-aware fused decode step (and the batch-8 encoder / prefill GEMMs), logits within tolerance."""
    model, eng = full_peaked
    # clips whose oracle-side worst top-1/top-2 gap is >= 5e-4 of max|logit| (scanned on the CPU; clips 0, 2, 5, 9 ... sit
    # at 1e-4 .. 6e-7, i.e. inside summation-order noise, where "exact ids" is a coin toss for any implementation)
    clips = [synth.make_clip(i, 30.0) for i in (1, 3, 4, 6, 7, 8, 10, 17)]
    refs = [O.transcribe_ids(model, c, max_new_tokens=128, keep_logits=True, lm_head_all_rows=False) for c in clips]
    report["full_b8_min_rel_margin"] = min(_min_rel_margin(r) for r in refs)
    eng.mel(clips)
    eng.encode()
    _, logits = eng.prefill()
    report["full_b8_prefill_logits_rel_err"] = max(_rel(logits[b], refs[b].prefill_logits.numpy()) for b in range(8))
    before = eng.stats().get("decode_batch_steps", 0)
    got = eng.transcribe_ids(clips, max_new_tokens=128)
    st = eng.stats()
    report["full_b8_stage_ms"] = got.stage_ms
    assert report["full_b8_min_rel_margin"] >= 5 * MARGIN_FLOOR_REL
    assert report["full_b8_prefill_logits_rel_err"] <= LOGIT_RTOL
    assert st["decode_batch_steps"] == before + 127 and st["gemm_simt_fallbacks"] == 0
    for b in range(8):
        assert got.ids[b] == refs[b].ids, b


def test_full_size_0p6b_16_sequences_512_token_kv(full_peaked, report):
    """BASELINE configs[4] per GPU: 16 sequences decoding around a 512-token KV cache (prompts of 300..405 tokens +
    128 new tokens cross 512 for the 30 s ones), ragged lengths -- exact ids for every sequence (NB = 16 instantiation,
    32-key attention splits, up to 17 splits per kv head)."""
    model, eng = full_peaked
    # (clip index, seconds): ragged 20 .. 30 s clips whose oracle-side worst top-1/top-2 gap is >= 4.8e-4 of max|logit|
    # (scanned on the CPU with the same generator; see test_full_size_0p6b_batch8_30s_128_tokens)
    sel = [(102, 27.8), (104, 23.0), (106, 20.1), (109, 24.7), (111, 22.8), (113, 24.5), (116, 30.0), (117, 27.9),
           (118, 26.2), (119, 29.9), (120, 22.2), (122, 26.1), (123, 20.4), (124, 20.4), (125, 25.1), (127, 29.2)]
    clips = [synth.make_clip(i, s) for i, s in sel]
    refs = [O.transcribe_ids(model, c, max_new_tokens=128, keep_logits=True, lm_head_all_rows=False) for c in clips]
    report["full_b16_min_rel_margin"] = min(_min_rel_margin(r) for r in refs)
    got = eng.transcribe_ids(clips, max_new_tokens=128)
    report["full_b16_stage_ms"] = got.stage_ms
    assert report["full_b16_min_rel_margin"] >= 5 * MARGIN_FLOOR_REL
    for b in range(16):
        assert got.ids[b] == refs[b].ids, b


def test_full_size_1p7b_30s_64_tokens(report):
    """BASELINE configs[3] model (1.7B dims as recalled in SURVEY.md section 8), one 30 s clip, 64 new tokens, peaked
    untied head: exact ids on the fused decode step's 1.7B instantiation."""
    from qwen3_asr_rs_b200 import AsrInference, config_1p7b
    cfg = O.cfg_1p7b()
    cfg.text.tie_word_embeddings = False
    w = synth.make_weights(cfg, 3, peaked_head=True)
    ecfg = config_1p7b()
    ecfg.text.tie_word_embeddings = False
    x = synth.make_clip(7, 30.0)
    ref = O.transcribe_ids(O.OracleModel(cfg, w), x, max_new_tokens=64, keep_logits=True, lm_head_all_rows=False)
    report["full1p7b_30s_min_rel_margin"] = _min_rel_margin(ref)
    eng = AsrInference.from_weights(ecfg, w, device=0)
    try:
        got = eng.transcribe_ids([x], max_new_tokens=64)
        st = eng.stats()
    finally:
        eng.close()
    report["full1p7b_30s_stage_ms"] = got.stage_ms
    assert report["full1p7b_30s_min_rel_margin"] >= MARGIN_FLOOR_REL
    assert st["decode_phase_steps"] == 0 and st["gemm_simt_fallbacks"] == 0
    assert got.ids[0] == ref.ids


def test_lossy_f32_matrix_is_rejected(tiny):
    """Matrices are kept in bf16: an f32 matrix that is not bf16-representable must be an error, not silently
    different logits (the reference widens everything to f32, weights.rs:74-89)."""
    import torch
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    from qwen3_asr_rs_b200._lib import AsrbError
    cfg, w, _ = tiny
    w2 = dict(w)
    k = "thinker.model.layers.0.mlp.down_proj.weight"
    w2[k] = w[k].float() + 1e-4          # no longer representable in bf16
    with pytest.raises(AsrbError, match="bf16-representable"):
        AsrInference.from_weights(config_tiny(), w2, device=0)
    w2[k] = w[k].float()                 # f32 container, bf16-exact values: accepted
    eng = AsrInference.from_weights(config_tiny(), w2, device=0)
    eng.close()


def test_bad_config_json_is_a_status_not_a_crash(tiny, tmp_path):
    """config.json with n_window = 0 used to divide by zero inside Dims::derive (SIGFPE)."""
    import json
    from qwen3_asr_rs_b200 import AsrInference
    from qwen3_asr_rs_b200._lib import AsrbError
    cfg, w, _ = tiny
    d = tmp_path / "bad"
    synth.write_checkpoint(str(d), cfg, w)
    j = json.loads((d / "config.json").read_text())
    j["thinker_config"]["audio_config"]["n_window"] = 0
    (d / "config.json").write_text(json.dumps(j))
    with pytest.raises(AsrbError):
        AsrInference.load(str(d), device=0)


@pytest.mark.parametrize("rate,channels,dtype", [(24000, 2, "int16"), (44100, 1, "int16"), (48000, 2, "float32"),
                                                 (8000, 1, "int16"), (16000, 3, "int32"), (22050, 2, "int16")])
def test_gpu_ingest_matches_scipy_resample_poly(tiny_engine, rate, channels, dtype):
    """asrb_ingest_pcm (src/audio.rs:162-245 on the GPU): sample scaling, mono mixdown and the polyphase resampler against
    its own golden, scipy.signal.resample_poly on the f64 mono signal (the host loader of audio.py)."""
    from math import gcd
    from scipy.signal import resample_poly
    rng = np.random.default_rng(rate + channels)
    n = int(rate * 1.37) + 11
    t = np.arange(n) / rate
    sig = np.stack([0.4 * np.sin(2 * np.pi * (220.0 + 90 * c) * t) + 0.05 * rng.standard_normal(n) for c in range(channels)], 1)
    if dtype == "int16":
        pcm = np.clip(np.round(sig * 32767), -32768, 32767).astype(np.int16); f = pcm.astype(np.float32) / 32768.0
    elif dtype == "int32":
        pcm = np.round(sig * 2147483000.0).astype(np.int32); f = pcm.astype(np.float32) / 2147483648.0
    else:
        pcm = sig.astype(np.float32); f = pcm
    mono = f.sum(axis=1, dtype=np.float32) / np.float32(channels) if channels > 1 else f[:, 0]
    g = gcd(rate, 16000)
    ref = mono.astype(np.float32) if rate == 16000 else resample_poly(mono.astype(np.float64), 16000 // g, rate // g).astype(np.float32)
    got = tiny_engine.ingest_pcm([pcm], [rate])[0]
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2e-6


def test_transcribe_pcm_equals_host_ingest(tiny, tiny_engine):
    """steps 1-8 with step 1 on the GPU == host loader + steps 2-8 (same ids), batch of two different formats."""
    from math import gcd
    from scipy.signal import resample_poly
    _, _, model = tiny
    x24 = synth.make_clip(77, 2.0, sample_rate=24000)
    x48 = synth.make_clip(78, 1.3, sample_rate=48000)
    pcm24 = (np.stack([x24, x24], 1) * 32767).astype(np.int16)
    pcm48 = x48.astype(np.float32).reshape(-1, 1)
    host = []
    for pcm, rate in ((pcm24, 24000), (pcm48, 48000)):
        f = pcm.astype(np.float32) / (32768.0 if pcm.dtype == np.int16 else 1.0)
        mono = f.mean(axis=1)
        g = gcd(rate, 16000)
        host.append(resample_poly(mono.astype(np.float64), 16000 // g, rate // g).astype(np.float32))
    want = tiny_engine.transcribe_ids(host, max_new_tokens=10).ids
    got = tiny_engine.transcribe_pcm([pcm24, pcm48], [24000, 48000], max_new_tokens=10).ids
    assert got == want
    assert got[0] == O.transcribe_ids(model, host[0], max_new_tokens=10).ids


def test_ids_gather_reads_device_buffers(tiny_engine):
    """parallel.IdsGather (bench.py's N > 1 path): the ids all_gather reads the session's own device buffers
    (asrb_session_device_ids) -- single-rank NCCL group here, the 2-rank logic is covered on gloo in test_parallel.py."""
    import torch
    import torch.distributed as dist
    from qwen3_asr_rs_b200 import parallel
    own = not dist.is_initialized()
    if own:
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29533", world_size=1, rank=0)
    try:
        clips = [synth.make_clip(90 + i, 1.5 + 0.4 * i) for i in range(3)]
        want = tiny_engine.transcribe_ids(clips, max_new_tokens=9).ids
        g = parallel.IdsGather(1, len(clips), 9, torch.device("cuda", 0))
        assert g(tiny_engine) == want
        want2 = tiny_engine.transcribe_ids(clips[:2], max_new_tokens=5).ids       # smaller batch, shorter rows: no stale ids
        assert g(tiny_engine)[:2] == want2
    finally:
        if own:
            dist.destroy_process_group()
