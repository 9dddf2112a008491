"""The float64 precision rule across the model dimensions the library accepts, and at value edges.

The library takes its dimensions from the caller (asrb_dims or a config.json).  tests/test_precision_fp64.py applies its
rule -- an output passes when its error against the float64 oracle is at most R = 4 times the fp32 oracle's error on the
same inputs -- at the tiny and 0.6B configurations, which are the same point on every axis that selects kernel code:
GQA group 2, encoder head_dim 64, 100-frame chunks in 8-chunk windows, a vocabulary of 1187 x 128 rows.  This file moves
the *model* to the other points.  Each GRID entry is the tiny configuration with one or two fields changed, so that a
failure names an axis; the oracle's and the engine's configurations are built from the one description.  Every entry
is either refused by the library with ASRB_ERR_INVALID before a kernel runs, or passes every check: stage outputs (mel,
encoder, prefill logits, 5 decode_step logits) on a batch of three clips, and the recorded top-8 log-probabilities of
the default decode path (batch 1, ragged batch 3) and of the per-phase path.  The decode path that ran is read from the
session counters, asserted against what the source selects for those dims, and written to the report
(grid_<entry>_path).

Value edges run under the same rule: clipped, nearly silent, offset, silent-then-burst, impulse and white-noise audio
on the tiny configuration, and a checkpoint with outlier channels (entry `outliers`).  The fp32 oracle calibrates the
bound per input, and its own error e_32 is in the report so that a reader sees the input stressed the arithmetic.

CPU tests show that the oracle is generic over the grid (fp32 against float64 stays at the fp32 level) and that the rule
sees the errors these axes exist to catch: a wrong GQA head mapping, an encoder window mask of the wrong size, a dropped
ragged vocabulary tail.
"""
import gc
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from oracle import oracle as O
from qwen3_asr_rs_b200 import synth
from test_precision_fp64 import (K, R, Err, _planes_errs, check, options, ratio, record_errs, rel_err, run_path,
                                 stage_errs, stage_run)

ASRB_ERR_INVALID = 1


# ---------------------------------------------------------------------------------------------------------------------
# the grid
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Entry:
    """The tiny configuration with `audio` / `text` fields replaced.  head: "tied", "untied" (plain untied lm_head) or
    "tail" (untied peaked head whose last vocab % 128 rows are the largest).  outliers: see outlier_weights."""
    name: str
    audio: dict = field(default_factory=dict)
    text: dict = field(default_factory=dict)
    seed: int = 11
    head: str = "tied"
    outliers: bool = False

    def configs(self):
        """(oracle config, engine config) from the one description."""
        from qwen3_asr_rs_b200 import config_tiny
        ocfg, ecfg = O.cfg_tiny(), config_tiny()
        text = dict(self.text, tie_word_embeddings=self.head == "tied")
        for cfg in (ocfg, ecfg):
            for part, over in ((cfg.audio, self.audio), (cfg.text, text)):
                for k, v in over.items():
                    assert hasattr(part, k), (self.name, k)
                    setattr(part, k, v)
        for part in ("audio", "text"):           # the two agree on every field the oracle knows
            o, e = getattr(ocfg, part), getattr(ecfg, part)
            assert all(getattr(o, k) == getattr(e, k) for k in o.__dataclass_fields__), (self.name, part)
        return ocfg, ecfg

    def weights(self, cfg):
        w = synth.make_weights(cfg, self.seed, peaked_head=self.head == "tail")
        if self.head == "tail":
            # x 32 (a power of two: bf16-exact) on the rows past the last full 128-row block: log-normal row norms
            # reach about 9 x the median, so a tail row wins whenever it points along the hidden state
            w["thinker.lm_head.weight"][tail_start(cfg.text.vocab_size):] *= 32.0
        if self.outliers:
            outlier_weights(w)
        return w

    def past_window_s(self) -> float:
        """A clip length with a tail chunk that is past one full encoder attention window (11.55 s by default)."""
        n_infer = self.audio.get("n_window_infer", 800)
        return n_infer / 100.0 + 3.55

    def expected_path(self, batch: int) -> str:
        """The step counter that must move on the default decode path, as decode_batch_supported and
        decode_mega_supported select it: the fused steps are instantiated per (hidden, q_dim, intermediate), the batched
        one only for two query heads per kv head, and neither takes more than 32 layers or a group above 6."""
        t = self.configs()[0].text
        dims = (t.hidden_size, t.num_attention_heads * t.head_dim, t.intermediate_size)
        group = t.num_attention_heads // t.num_key_value_heads
        if t.num_hidden_layers <= 32 and group <= 6:
            if batch >= 2 and group == 2 and dims in ((1024, 2048, 3072), (256, 512, 512)):
                return "decode_batch_steps"
            if dims in ((1024, 2048, 3072), (2048, 2048, 6144), (256, 512, 512)):
                return "decode_fused_steps"
        return "decode_phase_steps"


def tail_start(vocab: int) -> int:
    return 128 * (vocab // 128)


def outlier_weights(w) -> None:
    """Outlier channels as real checkpoints have them, by powers of two so that every value stays bf16-exact: two
    channels of every decoder RMSNorm and encoder LayerNorm weight x 64, one input column of every down_proj and fc2
    x 32, q_norm / k_norm x 4 (attention scores 16 x larger: softmax near one-hot)."""
    for name, t in w.items():
        if name.endswith(("input_layernorm.weight", "post_attention_layernorm.weight", "model.norm.weight",
                          "self_attn_layer_norm.weight", "final_layer_norm.weight", "ln_post.weight")):
            t[[3, t.shape[0] - 7]] *= 64.0
        elif name.endswith(("mlp.down_proj.weight", "fc2.weight")):
            t[:, 5] *= 32.0
        elif name.endswith(("q_norm.weight", "k_norm.weight")):
            t *= 4.0


ENTRIES = [
    # GQA group: 1 and 4 keep (hidden, q_dim, intermediate) = (256, 512, 512) and so run the fused single-sequence step
    Entry("gqa1", text=dict(num_attention_heads=4, num_key_value_heads=4)),
    Entry("gqa4", text=dict(num_attention_heads=4, num_key_value_heads=1)),
    Entry("gqa8", text=dict(num_attention_heads=8, num_key_value_heads=1)),                  # q_dim 1024: per-phase
    Entry("gqa3", text=dict(num_attention_heads=6, num_key_value_heads=2)),                  # odd group, q_dim 768
    Entry("enc_hd128", audio=dict(d_model=256, encoder_attention_heads=2)),                  # non-causal windowed HD 128
    Entry("enc_3heads", audio=dict(d_model=192, encoder_attention_heads=3, encoder_ffn_dim=320)),   # N = 192, 576, 320
    Entry("window40", audio=dict(n_window=40, n_window_infer=400)),      # 80-frame chunks, 10 tokens each, 5 per window
    Entry("window_uneven", audio=dict(n_window=50, n_window_infer=750)),                     # 750 // 100 = 7 chunks
    Entry("window_none", audio=dict(n_window=50, n_window_infer=60)),    # 0 chunks per window: no mask, one window
    Entry("dsh64", audio=dict(downsample_hidden_size=64)),                                   # no channel padding
    Entry("dsh72", audio=dict(downsample_hidden_size=72)),                                   # padded to 128, feat 1152
    Entry("wide", audio=dict(output_dim=512), text=dict(hidden_size=512, intermediate_size=768)),   # K = 768 down_proj
    Entry("vocab_x8", text=dict(vocab_size=151688), head="tail"),                            # 1185 x 128 + 8
    Entry("vocab_odd", text=dict(vocab_size=151681), head="tail"),                           # 1185 x 128 + 1
    Entry("layers33", text=dict(num_hidden_layers=33)),                                      # past the fused steps' 32
    Entry("eps_theta", text=dict(rms_norm_eps=1e-5, rope_theta=1e4)),
    Entry("untied", text=dict(num_attention_heads=4, num_key_value_heads=1), head="untied"),
    Entry("outliers", seed=7, outliers=True),
]
GRID = {e.name: e for e in ENTRIES}
GRID["tiny"] = Entry("tiny", seed=7)               # the base point itself: the audio edges run on it
NAMES = [e.name for e in ENTRIES]


def test_grid_descriptions():
    """Every entry differs from the base, and oracle and engine configurations are one description."""
    base = GRID["tiny"].configs()[0]
    for e in ENTRIES:
        ocfg, _ = e.configs()
        assert ocfg != base or e.outliers, e.name
        assert ocfg.audio.output_dim == ocfg.text.hidden_size
    assert GRID["gqa1"].expected_path(1) == GRID["gqa4"].expected_path(3) == "decode_fused_steps"
    assert GRID["tiny"].expected_path(3) == "decode_batch_steps"
    assert {GRID[n].expected_path(b) for n in ("gqa8", "gqa3", "wide", "layers33") for b in (1, 3)} == {"decode_phase_steps"}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle over the grid, and the rule's resolution on these axes
# ---------------------------------------------------------------------------------------------------------------------
def oracles(ent: Entry):
    cfg, _ = ent.configs()
    w = ent.weights(cfg)
    return O.OracleModel(cfg, w), O.OracleModel(cfg, w, dtype=torch.float64)


@pytest.mark.parametrize("name", NAMES)
def test_fp32_oracle_error_against_fp64_over_grid(name, report):
    """The fp32 oracle stays at the fp32 level of the float64 one at every entry (the band of the tiny configuration;
    wider above for the deliberately ill-conditioned entries), on a clip past one attention window: the oracle is
    generic over the grid, and it reads each description as make_weights does."""
    ent = GRID[name]
    m32, m64 = oracles(ent)
    x = synth.make_clip(60, ent.past_window_s())
    mel32, mel64 = O.extract_mel(x), O.extract_mel(x, dtype=torch.float64)
    enc32, enc64 = m32.encode(mel32), m64.encode(mel64)
    assert enc64.dtype == torch.float64 and enc32.shape == enc64.shape
    ids = O.transcribe_ids(m32, x, max_new_tokens=6, lm_head_all_rows=False).ids
    s32, s64 = O.score_ids(m32, x, ids), O.score_ids(m64, x, ids)
    errs = {"encoder": rel_err(enc32, enc64), "prefill": rel_err(s32[0], s64[0]), "steps": rel_err(s32[1:], s64[1:])}
    report[f"grid_cpu_{name}_fp32_oracle_rel_err"] = errs
    # 33 layers accumulate more rounding than 3; outlier channels and x 32 head rows amplify it
    hi = {"layers33": 2e-5, "outliers": 5e-5}.get(name, 5e-6)
    assert all(1e-7 <= v <= hi for v in errs.values()), errs
    del m32, m64
    gc.collect()


def test_rule_sees_wrong_gqa_head_mapping(report, monkeypatch):
    """Query head h reading kv head h % nkv instead of h // group, at nq = 6, nkv = 2.  (With one kv head, as at gqa4
    and gqa8, the two mappings are the same function: the odd group is the entry that tells them apart.)"""
    m32, m64 = oracles(GRID["gqa3"])
    x = synth.make_clip(60, 3.0)
    good32, good64 = O.score_ids(m32, x, []), O.score_ids(m64, x, [])
    monkeypatch.setattr(O, "repeat_kv", lambda t, n_rep: t.repeat(1, n_rep, 1, 1))
    wrong = O.score_ids(m32, x, [])
    r = ratio(report, "grid_mutation_gqa_head_mapping", Err(True).add(wrong[0], good32[0], good64[0]))
    assert r > 100 * R, r


def test_rule_sees_wrong_window_size(report):
    """The encoder mask built for 8 chunks per window where the configuration says 5 (window40, 11 chunks)."""
    class EightChunkWindows(O.OracleModel):
        def window_mask(self, total, chunk_tokens):
            cfg = self.cfg
            try:
                self.cfg = O.AsrCfg(O.AudioCfg(**{**cfg.audio.__dict__, "n_window_infer": 16 * cfg.audio.n_window}), cfg.text)
                return super().window_mask(total, chunk_tokens)
            finally:
                self.cfg = cfg

    ent = GRID["window40"]
    cfg, _ = ent.configs()
    w = ent.weights(cfg)
    m32, m64, bad = O.OracleModel(cfg, w), O.OracleModel(cfg, w, dtype=torch.float64), EightChunkWindows(cfg, w)
    x = synth.make_clip(60, 8.5)
    mel32, mel64 = O.extract_mel(x), O.extract_mel(x, dtype=torch.float64)
    r = ratio(report, "grid_mutation_window_size", Err(True).add(bad.encode(mel32), m32.encode(mel32), m64.encode(mel64)))
    assert r > 100 * R, r


def test_rule_sees_dropped_vocabulary_tail(report):
    """The last vocab % 128 logits zeroed, as a partition merge that stops at the last full block would leave them."""
    ent = GRID["vocab_x8"]
    m32, m64 = oracles(ent)
    x = synth.make_clip(60, 3.0)
    good32, good64 = O.score_ids(m32, x, [])[0], O.score_ids(m64, x, [])[0]
    wrong = good32.clone()
    wrong[tail_start(m32.cfg.text.vocab_size):] = 0.0
    r = ratio(report, "grid_mutation_vocab_tail", Err(True).add(wrong, good32, good64))
    assert r > 100 * R, r


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def grid(request):
    """(entry, fp32 oracle, fp64 oracle, engine) of the entry named by the (indirect) parameter.  One entry is alive at
    a time: its engine and float64 weights are freed before the next is built."""
    from qwen3_asr_rs_b200 import AsrInference
    ent = GRID[request.param]
    ocfg, ecfg = ent.configs()
    w = ent.weights(ocfg)
    e = AsrInference.from_weights(ecfg, w, device=0)
    m32, m64 = O.OracleModel(ocfg, w), O.OracleModel(ocfg, w, dtype=torch.float64)
    del w
    yield ent, m32, m64, e
    e.close()
    del m32, m64
    gc.collect()


def over(names):
    return pytest.mark.parametrize("grid", names, indirect=True)


@pytest.mark.gpu
@over(NAMES)
def test_grid_stage_outputs(grid, report):
    """Mel, encoder output, prefill logits and 5 decode_step logits of three clips: under one chunk, with a tail chunk,
    past one full attention window of the entry."""
    ent, m32, m64, e = grid
    clips = [synth.make_clip(31, 0.6), synth.make_clip(32, 8.5), synth.make_clip(33, ent.past_window_s())]
    errs = stage_errs(m32, m64, clips, stage_run(e, clips))
    for k, err in errs.items():
        ratio(report, f"grid_{ent.name}_{k}", err)
    for k, err in errs.items():
        check(report, f"grid_{ent.name}_{k}", err)


SHORT = {"decode_fused_steps": "fused", "decode_batch_steps": "batch", "decode_phase_steps": "phases",
         "gemm_simt_fallbacks": "simt_fallbacks", "gemm_tc_launches": "tc_launches"}
B1 = [(70, 4.0)]
B3 = [(80, 2.5), (81, 9.1), (82, 1.2)]


def counted_run(e, sel, n_new, opts, path):
    """run_path (warm-up, measured run, the step counter that must move) with top-8 records; also every session
    counter's movement over both runs."""
    clips = [synth.make_clip(i, s) for i, s in sel]
    with options(e, **opts):
        e.mel(clips, max_new_tokens=n_new)                # session sized before the counters are read
        s0 = e.stats()
        r = run_path(e, clips, n_new, {}, path, top_logprobs=K)
        s1 = e.stats()
    return clips, r, {short: s1[k] - s0[k] for k, short in SHORT.items()}


def tail_rows_err(m32, m64, clips, r, vocab):
    """Err over the recorded candidates with an id in the ragged tail, and how many steps had one."""
    err, steps = Err(False), 0
    for b, x in enumerate(clips):
        l32 = torch.log_softmax(O.score_ids(m32, x, r.ids[b]).double(), -1).numpy()
        l64 = torch.log_softmax(O.score_ids(m64, x, r.ids[b]), -1).numpy()
        rows = list(r.top_logprobs[b]) + ([r.eos_top_logprobs[b]] if r.eos_top_logprobs[b] is not None else [])
        for t, row in enumerate(rows):
            tail = [(i, lp) for i, lp in row if i >= tail_start(vocab)]
            if tail:
                steps += 1
                cand = np.array([i for i, _ in tail])
                assert cand.max() < vocab, row
                err.add(np.array([lp for _, lp in tail]), l32[t, cand], l64[t, cand])
    return err, steps


@pytest.mark.gpu
@over(NAMES)
def test_grid_top_logprobs_default_path(grid, report):
    """Top-8 log-probabilities of every step on the decode path the library picks: batch 1 (40 new tokens) and a ragged
    batch of 3 (16).  The path is asserted: gqa1 and gqa4 must run the fused single-sequence step, or this file does
    not cover what it claims; gqa8, gqa3, wide and layers33 must move only the per-phase counter."""
    ent, m32, m64, e = grid
    total = dict.fromkeys(SHORT.values(), 0)
    tail_err, tail_steps = Err(False), 0
    for label, sel, n_new in (("b1", B1, 40), ("b3", B3, 16)):
        clips, r, moved = counted_run(e, sel, n_new, {}, ent.expected_path(len(sel)))
        for k, v in moved.items():
            total[k] += v
        check(report, f"grid_{ent.name}_top{K}_{label}", record_errs(m32, m64, clips, r, top=True))
        if ent.head == "tail":
            err, n = tail_rows_err(m32, m64, clips, r, m32.cfg.text.vocab_size)
            tail_err.merge(err)
            tail_steps += n
    report[f"grid_{ent.name}_path"] = total
    if ent.name in ("gqa1", "gqa4"):
        assert total["fused"] > 0 and total["batch"] == 0 and total["phases"] == 0, total
    if ent.name in ("gqa8", "gqa3", "wide", "layers33"):
        assert total["phases"] > 0 and total["fused"] == 0 and total["batch"] == 0, total
    if ent.head == "tail":
        # a partition merge that drops the ragged tail fails here on ids, not only on error size
        report[f"grid_{ent.name}_tail_steps"] = tail_steps
        assert tail_steps >= 1, "no recorded top-8 row holds an id of the ragged vocabulary tail"
        assert ratio(report, f"grid_{ent.name}_tail_top{K}", tail_err, min_values=1) <= R


@pytest.mark.gpu
@over(NAMES)
def test_grid_top_logprobs_phases(grid, report):
    """The ragged batch on the per-phase path; whether its ids equal the default path's is reported, not asserted
    (random tied heads have top-1 gaps inside summation noise)."""
    ent, m32, m64, e = grid
    clips, r, _ = counted_run(e, B3, 16, {"decode": "phases"}, "decode_phase_steps")
    check(report, f"grid_{ent.name}_top{K}_b3_phases", record_errs(m32, m64, clips, r, top=True))
    same = e.transcribe_ids(clips, max_new_tokens=16).ids == r.ids
    report[f"grid_{ent.name}_ids_equal_default_vs_phases"] = bool(same)


@pytest.mark.gpu
@over(["enc_hd128", "gqa8"])
def test_grid_negative_control_planes2(grid, report):
    """Encoder and prefill GEMMs fed with two bf16 planes must FAIL the rule at the new shapes as they do on the tiny
    configuration: the rule keeps its resolution there."""
    ent, m32, m64, e = grid
    with options(e, planes="2"):
        enc_e, pre_e = _planes_errs(m32, m64, e, [synth.make_clip(60, 6.2)])
    for name, err in (("encoder", enc_e), ("prefill", pre_e)):
        r = ratio(report, f"grid_{ent.name}_planes2_{name}", err)
        assert r > R, (name, report[f"fp64_grid_{ent.name}_planes2_{name}"])


# ---- refusals ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@over(["gqa8"])
def test_session_refuses_context_beyond_decode_attention(grid):
    """The per-phase decode attention keeps group * (128 + context) scores in shared memory.  A session whose context
    does not fit is refused when it is created, with the numbers, instead of failing in the middle of a decode step;
    the engine then sizes a smaller session as if nothing had happened."""
    from qwen3_asr_rs_b200._lib import AsrbError
    _, _, _, e = grid
    with pytest.raises(AsrbError, match=r"GQA group 8 needs \d+ bytes of shared memory for decode attention") as ei:
        e._ensure_session(1, 30 * 16000, 0, 8000)          # 8 * (128 + 390 + 15 + 8000) * 4 bytes = 273 KB
    assert ei.value.code == ASRB_ERR_INVALID
    assert len(e.transcribe_ids([synth.make_clip(70, 1.0)], max_new_tokens=4).ids) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("field_,value,message", [("text.head_dim", 64, "decoder head_dim must be 128"),
                                                  ("audio.num_mel_bins", 80, "num_mel_bins must be 128")])
def test_unsupported_dims_are_refused(field_, value, message):
    """Decoder head_dim != 128 and num_mel_bins != 128 stay refused, by asrb_model_create or asrb_model_finalize, before
    any tensor is read."""
    from qwen3_asr_rs_b200 import AsrInference, config_tiny
    from qwen3_asr_rs_b200._lib import AsrbError
    cfg = config_tiny()
    part, name = field_.split(".")
    setattr(getattr(cfg, part), name, value)
    with pytest.raises(AsrbError, match=message) as ei:
        AsrInference.from_weights(cfg, {}, device=0)
    assert ei.value.code == ASRB_ERR_INVALID


# ---- value edges ---------------------------------------------------------------------------------------------------
def edge_clips():
    base = synth.make_clip(90, 3.0)
    rng = np.random.default_rng(77)
    burst = np.zeros(3 * 16000, np.float32)
    burst[2 * 16000:] = synth.make_clip(91, 1.0)
    impulse = np.zeros(16000, np.float32)
    impulse[8000] = 1.0
    noise = rng.standard_normal(2 * 16000)
    return [("clipped", np.clip(4.0 * base, -1.0, 1.0).astype(np.float32)),
            ("amplitude_1e-4", (base * 2e-4).astype(np.float32)),                    # peak 0.5 -> 1e-4
            ("dc_offset", (0.3 + 0.02 * base).astype(np.float32)),
            ("silence_then_burst", burst),
            ("impulse", impulse),
            ("white_noise", (0.9 * noise / np.abs(noise).max()).astype(np.float32))]


@pytest.mark.gpu
@over(["tiny"])
def test_audio_value_edges(grid, report):
    """Clipped, nearly silent, offset, silent-then-burst, impulse and white-noise audio as one batch: mel, encoder
    output and prefill logits of each meet the rule (bound calibrated per input), and silence gives no non-finite
    value (Err refuses them)."""
    _, m32, m64, e = grid
    names, clips = zip(*edge_clips())
    mels, enc, pre, _, _ = stage_run(e, list(clips), n_steps=0)
    failed = []
    for b, name in enumerate(names):
        errs = stage_errs(m32, m64, [clips[b]], ([mels[b]], [enc[b]], pre[b:b + 1], [], [[]]), n_steps=0)
        for k in ("mel", "encoder", "prefill"):
            if ratio(report, f"edge_{name}_{k}", errs[k]) > R:
                failed.append((name, k, report[f"fp64_edge_{name}_{k}"]))
    assert not failed, failed
