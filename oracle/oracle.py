"""CPU fp32 restatement of the reference's tch-CPU hot path  --  TEST INFRASTRUCTURE.

This file is the parity oracle for the H100 path.  It is NOT product code: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl
reference`` legs may import it; the product path (``qwen3_asr_rs_b200``) never does and
fails loudly when its CUDA library is missing.

What it restates (reference = second-state/qwen3_asr_rs @ eed686e, paths relative to
/root/reference): ``transcribe()`` steps 2-8 (src/inference.rs:94-200) i.e.
mel (src/mel.rs:49-96,115-187) -> audio encoder (src/audio_encoder.rs:79-301,
src/layers.rs:10-243) -> prompt/inject (src/inference.rs:105-124,215-266) -> MRoPE
(src/layers.rs:471-562) -> prefill + greedy KV-cache decode (src/layers.rs:35-55,249-464,
src/text_decoder.rs:10-131, src/inference.rs:139-200), for the **tch arm** of
src/tensor.rs (:145-488).  The arithmetic of that arm lives in libtorch 2.7.1 via
tch 0.20.0 (Cargo.lock:1279-1281); PyTorch-CPU here dispatches to the same ATen
operators (torch 2.11), op for op, in fp32, as weights.rs:74-89 up-casts every
checkpoint tensor to f32.

PARITY PINNING: the reference ships no unit tests, golden tensors or known-answer
vectors for this path (SURVEY.md section 4/8c) -> "parity unpinned" by the reference
itself.  The Rust crate cannot be built here (no cargo/rustc).  The restatement is
therefore pinned against the model authors' independent HF implementations
(WhisperFeatureExtractor, Qwen3OmniMoeAudioEncoder, Qwen3ForCausalLM) by
``oracle/pin_against_hf.py``; its outputs are committed under ``tests/golden/``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, asdict
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

# Special token ids (src/tokenizer.rs:53-59)
IM_START, IM_END, ENDOFTEXT = 151644, 151645, 151643
AUDIO_START, AUDIO_END, AUDIO_PAD = 151669, 151670, 151676
EOS_IDS = (ENDOFTEXT, IM_END)  # src/inference.rs:154

N_FFT, HOP, SAMPLE_RATE = 400, 160, 16000  # src/inference.rs:16,68-74


# --------------------------------------------------------------------------------------
# Config (src/config.rs:27-113; every default is the 0.6B value)
# --------------------------------------------------------------------------------------
@dataclass
class AudioCfg:
    d_model: int = 896
    encoder_layers: int = 18
    encoder_attention_heads: int = 14
    encoder_ffn_dim: int = 3584
    num_mel_bins: int = 128
    max_source_positions: int = 1500
    n_window: int = 50
    n_window_infer: int = 800
    downsample_hidden_size: int = 480
    output_dim: int = 1024


@dataclass
class TextCfg:
    vocab_size: int = 151936
    hidden_size: int = 1024
    intermediate_size: int = 3072
    num_hidden_layers: int = 28
    num_attention_heads: int = 16
    num_key_value_heads: int = 8
    head_dim: int = 128
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1_000_000.0
    tie_word_embeddings: bool = True
    mrope_section: Tuple[int, ...] = (24, 20, 20)
    mrope_interleaved: bool = False


@dataclass
class AsrCfg:
    audio: AudioCfg = field(default_factory=AudioCfg)
    text: TextCfg = field(default_factory=TextCfg)

    def to_config_json(self) -> dict:
        """HF-style config.json the reference's src/config.rs parses."""
        t = asdict(self.text)
        sec, inter = t.pop("mrope_section"), t.pop("mrope_interleaved")
        t["rope_scaling"] = {"rope_type": "default", "mrope_section": list(sec),
                             "mrope_interleaved": bool(inter)}
        return {"thinker_config": {"audio_config": asdict(self.audio), "text_config": t,
                                   "audio_start_token_id": AUDIO_START,
                                   "audio_end_token_id": AUDIO_END,
                                   "audio_token_id": AUDIO_PAD}}

    @staticmethod
    def from_config_json(d: dict) -> "AsrCfg":
        th = d["thinker_config"]
        a = {k: v for k, v in th.get("audio_config", {}).items() if k in AudioCfg.__dataclass_fields__}
        tj = dict(th.get("text_config", {}))
        rs = tj.pop("rope_scaling", None) or {}
        t = {k: v for k, v in tj.items() if k in TextCfg.__dataclass_fields__}
        if "mrope_section" in rs:
            t["mrope_section"] = tuple(rs["mrope_section"])
        t["mrope_interleaved"] = bool(rs.get("mrope_interleaved", False) or rs.get("interleaved", False))
        return AsrCfg(AudioCfg(**a), TextCfg(**t))


def cfg_0p6b() -> AsrCfg:
    return AsrCfg()


def cfg_1p7b() -> AsrCfg:
    """Dims recalled from the HF card (SURVEY.md section 8) -- verify against a real config.json."""
    return AsrCfg(AudioCfg(d_model=1024, encoder_layers=24, encoder_attention_heads=16,
                           encoder_ffn_dim=4096, output_dim=2048),
                  TextCfg(hidden_size=2048, intermediate_size=6144))


def cfg_tiny(vocab: int = 151936) -> AsrCfg:
    """Small config for fast tests: same structure, every code path exercised."""
    return AsrCfg(AudioCfg(d_model=128, encoder_layers=2, encoder_attention_heads=2,
                           encoder_ffn_dim=256, downsample_hidden_size=32, output_dim=256),
                  TextCfg(vocab_size=vocab, hidden_size=256, intermediate_size=512,
                          num_hidden_layers=3, num_attention_heads=4, num_key_value_heads=2,
                          head_dim=128))


# --------------------------------------------------------------------------------------
# mel  (src/mel.rs)
# --------------------------------------------------------------------------------------
def mel_filterbank(num_mels: int = 128, n_fft: int = N_FFT, sample_rate: int = SAMPLE_RATE) -> np.ndarray:
    """Slaney-scale / slaney-norm triangular filters, f64 -> f32.  src/mel.rs:115-187."""
    n_freqs = n_fft // 2 + 1
    sr = float(sample_rate)
    fmin, fmax = 0.0, sr / 2.0
    f_sp = 200.0 / 3.0
    min_log_hz = 1000.0
    min_log_mel = (min_log_hz - 0.0) / f_sp
    logstep = math.log(6.4) / 27.0

    def hz_to_mel(f):
        return f / f_sp if f < min_log_hz else min_log_mel + math.log(f / min_log_hz) / logstep

    def mel_to_hz(m):
        return f_sp * m if m < min_log_mel else min_log_hz * math.exp(logstep * (m - min_log_mel))

    mel_min, mel_max = hz_to_mel(fmin), hz_to_mel(fmax)
    filter_freqs = [mel_to_hz(mel_min + (mel_max - mel_min) * i / (num_mels + 1)) for i in range(num_mels + 2)]
    all_freqs = [j * sr / n_fft for j in range(n_freqs)]
    f_diff = [filter_freqs[i + 1] - filter_freqs[i] for i in range(num_mels + 1)]
    filters = np.zeros((num_mels, n_freqs), dtype=np.float32)
    for j in range(n_freqs):
        for i in range(num_mels):
            down = (all_freqs[j] - filter_freqs[i]) / f_diff[i]
            up = (filter_freqs[i + 2] - all_freqs[j]) / f_diff[i + 1]
            filters[i, j] = np.float32(max(min(down, up), 0.0))          # `val as f32` (:166)
    for i in range(num_mels):
        enorm = np.float32(2.0 / (filter_freqs[i + 2] - filter_freqs[i]))  # `enorm as f32` (:174)
        filters[i, :] = filters[i, :] * enorm                              # f32 * f32
    return filters


_FB_CACHE: Dict[Tuple[int, int, int], torch.Tensor] = {}


def extract_mel(samples: np.ndarray, num_mels: int = 128, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """f32 samples @16 kHz -> log-mel [num_mels, F], F = ceil(n/160).  src/mel.rs:49-96.
    ``dtype=torch.float64``: the f32 samples and the (f32) filterbank widened exactly, every operation in f64."""
    key = (num_mels, N_FFT, SAMPLE_RATE)
    if key not in _FB_CACHE:
        _FB_CACHE[key] = torch.from_numpy(mel_filterbank(num_mels))
    fb = _FB_CACHE[key].to(dtype)
    x = np.asarray(samples, dtype=np.float32)
    padded_len = ((len(x) + HOP - 1) // HOP) * HOP                        # :51
    xp = np.zeros(padded_len, dtype=np.float32)
    xp[: len(x)] = x
    wave = torch.from_numpy(xp).to(dtype)
    window = torch.hann_window(N_FFT, dtype=dtype)                        # periodic (tensor.rs:215)
    pad = N_FFT // 2
    wave = torch.nn.functional.pad(wave[None, None, :], (pad, pad), mode="reflect")[0, 0]   # :63-65
    stft = torch.stft(wave, N_FFT, hop_length=HOP, win_length=N_FFT, window=window,
                      center=False, normalized=False, onesided=True, return_complex=True)   # :68-76
    mag = stft.abs().square()                                             # :80
    mag = mag[:, :-1]                                                     # :83-84
    mel = fb.matmul(mag)                                                  # :87
    log_mel = mel.clamp_min(1e-10).log10()                                # :90
    mx = log_mel.max()                                                    # :91
    log_mel = torch.maximum(log_mel, mx - 8.0)                            # :92
    return (log_mel + 4.0) / 4.0                                          # :93


# --------------------------------------------------------------------------------------
# NN blocks  (src/layers.rs)
# --------------------------------------------------------------------------------------
def linear(x, w, b=None):
    """x.matmul(W^T) (+ b).  src/layers.rs:74-80."""
    out = x.matmul(w.t())
    return out + b if b is not None else out


def rms_norm(x, w, eps):
    """src/layers.rs:48-54 with rsqrt := sqrt().reciprocal() (src/tensor.rs:323-326)."""
    var = (x * x).mean(dim=-1, keepdim=True)
    return (x * (var + eps).sqrt().reciprocal()) * w


def layer_norm(x, w, b, eps=1e-5):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), w, b, eps)   # layers.rs:25-28


def gelu(x):
    return torch.nn.functional.gelu(x, approximate="none")                # tensor.rs:350-352


def rotate_half(x):
    half = x.shape[-1] // 2                                               # layers.rs:370-375
    return torch.cat([-x[..., half:], x[..., :half]], dim=-1)


def apply_rotary(x, cos, sin):
    return x * cos[None, None] + rotate_half(x) * sin[None, None]         # layers.rs:361-367


def repeat_kv(x, n_rep):
    if n_rep == 1:
        return x
    b, h, s, d = x.shape                                                  # layers.rs:350-358
    return x.unsqueeze(2).expand(b, h, n_rep, s, d).reshape(b, h * n_rep, s, d)


def build_dim_map(sections: Sequence[int], total: int, interleaved: bool) -> List[int]:
    """src/layers.rs:524-562."""
    if not interleaved:
        m: List[int] = []
        for dim, size in enumerate(sections):
            for _ in range(size):
                if len(m) >= total:
                    break
                m.append(dim)
        while len(m) < total:
            m.append(len(sections) - 1)
        return m
    m = []
    counts = [0] * len(sections)
    while len(m) < total:
        prev = len(m)
        for dim in range(len(sections)):
            if len(m) >= total:
                break
            if counts[dim] < sections[dim]:
                m.append(dim)
                counts[dim] += 1
        if len(m) == prev:
            break
    return m


def mrope_cos_sin(position_ids: Sequence[Sequence[int]], head_dim: int, theta: float,
                  sections: Sequence[int], interleaved: bool,
                  dtype: torch.dtype = torch.float32) -> Tuple[torch.Tensor, torch.Tensor]:
    """Host f64 table, duplicated halves, -> [S, head_dim] in ``dtype`` (f32: rounded as the reference does).
    src/layers.rs:471-522."""
    half = head_dim // 2
    inv_freq = np.array([1.0 / (theta ** (2.0 * i / head_dim)) for i in range(half)], dtype=np.float64)
    dim_map = build_dim_map(sections, half, interleaved)
    pos = np.asarray(position_ids, dtype=np.float64)                      # [3, S]
    sel = pos[np.asarray(dim_map), :].T                                    # [S, half]
    ang = sel * inv_freq[None, :]
    npdt = torch.empty(0, dtype=dtype).numpy().dtype
    c, s = np.cos(ang).astype(npdt), np.sin(ang).astype(npdt)
    return (torch.from_numpy(np.concatenate([c, c], axis=1)),
            torch.from_numpy(np.concatenate([s, s], axis=1)))


def sinusoid_table(max_len: int, dim: int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """src/audio_encoder.rs:283-301 (f64 host, sin || cos), returned in ``dtype``."""
    half = dim // 2
    inc = math.log(10000.0) / (half - 1)
    inv = np.exp(-np.arange(half, dtype=np.float64) * inc)
    ang = np.arange(max_len, dtype=np.float64)[:, None] * inv[None, :]
    return torch.from_numpy(np.concatenate([np.sin(ang), np.cos(ang)], axis=1)).to(dtype)


def feat_extract_output_length(frames: int) -> int:
    o = lambda l: (l - 1) // 2 + 1                                        # audio_encoder.rs:263-266
    return o(o(o(frames)))


# --------------------------------------------------------------------------------------
# Model
# --------------------------------------------------------------------------------------
class OracleModel:
    """Holds fp32 weights under the HF names the reference loads (SURVEY.md section 8c).  ``dtype=torch.float64``
    widens the (bf16) weights exactly and runs every stage in f64: the high-precision reference of the same model."""

    def __init__(self, cfg: AsrCfg, weights: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float32):
        self.cfg = cfg
        self.dtype = dtype
        self.w = {k: v.to(dtype) for k, v in weights.items()}             # weights.rs:74-89
        self.pos_emb = sinusoid_table(cfg.audio.max_source_positions, cfg.audio.d_model, dtype)

    # ---- audio encoder (src/audio_encoder.rs:79-169) ----
    def chunk_plan(self, num_frames: int) -> Tuple[int, List[int]]:
        cs = self.cfg.audio.n_window * 2
        full, tail = divmod(num_frames, cs)
        valid = [feat_extract_output_length(cs)] * full
        if tail > 0:
            valid.append(feat_extract_output_length(tail))
        return cs, valid

    def window_mask(self, total: int, chunk_tokens: List[int]) -> Optional[torch.Tensor]:
        """Additive 0/-inf block-diagonal mask; None if C <= chunks_per_window.  :172-260."""
        cs = self.cfg.audio.n_window * 2
        cpw = self.cfg.audio.n_window_infer // cs
        if cpw == 0 or len(chunk_tokens) <= cpw:
            return None
        mask = torch.full((1, 1, total, total), float("-inf"), dtype=self.dtype)
        off = 0
        for w0 in range(0, len(chunk_tokens), cpw):
            n = sum(chunk_tokens[w0:w0 + cpw])
            mask[0, 0, off:off + n, off:off + n] = 0.0
            off += n
        return mask

    def encoder_stem(self, mel: torch.Tensor) -> Tuple[torch.Tensor, List[int]]:
        w, p = self.w, "thinker.audio_tower"
        F_ = mel.shape[1]
        cs, valid = self.chunk_plan(F_)
        C = len(valid)
        padded = torch.zeros(mel.shape[0], C * cs, dtype=self.dtype)
        padded[:, :F_] = mel                                              # :105-121 zero-pad tail
        batched = padded.reshape(mel.shape[0], C, cs).permute(1, 0, 2).unsqueeze(1)   # [C,1,128,cs]
        x = batched
        for name in ("conv2d1", "conv2d2", "conv2d3"):                    # :127-129
            x = gelu(torch.nn.functional.conv2d(x, w[f"{p}.{name}.weight"], w.get(f"{p}.{name}.bias"),
                                                stride=(2, 2), padding=(1, 1)))
        b, c, f, t = x.shape
        x = x.permute(0, 3, 1, 2).contiguous().reshape(b, t, c * f)       # :132-133
        x = linear(x, w[f"{p}.conv_out.weight"], w.get(f"{p}.conv_out.bias"))
        x = x + self.pos_emb[:t].unsqueeze(0)                             # :137-138
        hidden = torch.cat([x[i, :v] for i, v in enumerate(valid)], dim=0)  # :141-149
        return hidden, valid

    def encoder_layer(self, x, i, mask):
        w, p = self.w, f"thinker.audio_tower.layers.{i}"
        nh = self.cfg.audio.encoder_attention_heads
        hd = self.cfg.audio.d_model // nh
        res = x
        h = layer_norm(x, w[f"{p}.self_attn_layer_norm.weight"], w[f"{p}.self_attn_layer_norm.bias"])
        bsz, S, _ = h.shape
        q = linear(h, w[f"{p}.self_attn.q_proj.weight"], w[f"{p}.self_attn.q_proj.bias"]).reshape(bsz, S, nh, hd).permute(0, 2, 1, 3)
        k = linear(h, w[f"{p}.self_attn.k_proj.weight"], w[f"{p}.self_attn.k_proj.bias"]).reshape(bsz, S, nh, hd).permute(0, 2, 1, 3)
        v = linear(h, w[f"{p}.self_attn.v_proj.weight"], w[f"{p}.self_attn.v_proj.bias"]).reshape(bsz, S, nh, hd).permute(0, 2, 1, 3)
        attn = q.matmul(k.transpose(-2, -1)) / math.sqrt(hd)              # layers.rs:161-162
        if mask is not None:
            attn = attn + mask
        attn = attn.softmax(-1)
        out = attn.matmul(v).permute(0, 2, 1, 3).reshape(bsz, S, nh * hd)
        x = linear(out, w[f"{p}.self_attn.out_proj.weight"], w[f"{p}.self_attn.out_proj.bias"]) + res
        res = x
        h = layer_norm(x, w[f"{p}.final_layer_norm.weight"], w[f"{p}.final_layer_norm.bias"])
        h = gelu(linear(h, w[f"{p}.fc1.weight"], w[f"{p}.fc1.bias"]))
        h = linear(h, w[f"{p}.fc2.weight"], w[f"{p}.fc2.bias"])
        return h + res

    def encode(self, mel: torch.Tensor, return_stages: bool = False):
        w, p = self.w, "thinker.audio_tower"
        hidden, valid = self.encoder_stem(mel)
        stages = {"stem": hidden.clone()} if return_stages else None
        T = hidden.shape[0]
        mask = self.window_mask(T, valid)
        x = hidden.unsqueeze(0)
        for i in range(self.cfg.audio.encoder_layers):
            x = self.encoder_layer(x, i, mask)
            if return_stages and i == 0:
                stages["layer0"] = x[0].clone()
        x = layer_norm(x, w[f"{p}.ln_post.weight"], w[f"{p}.ln_post.bias"])   # :163-165
        x = gelu(linear(x, w[f"{p}.proj1.weight"], w[f"{p}.proj1.bias"]))
        x = linear(x, w[f"{p}.proj2.weight"], w[f"{p}.proj2.bias"])
        out = x.squeeze(0)
        return (out, stages) if return_stages else out

    # ---- text decoder (src/text_decoder.rs, src/layers.rs:249-464) ----
    def decoder_layer(self, x, i, cos, sin, cache, mask):
        w, p, t = self.w, f"thinker.model.layers.{i}", self.cfg.text
        nq, nkv, hd, eps = t.num_attention_heads, t.num_key_value_heads, t.head_dim, t.rms_norm_eps
        res = x
        h = rms_norm(x, w[f"{p}.input_layernorm.weight"], eps)
        bsz, S, _ = h.shape
        q = linear(h, w[f"{p}.self_attn.q_proj.weight"]).reshape(bsz, S, nq, hd).transpose(1, 2)
        k = linear(h, w[f"{p}.self_attn.k_proj.weight"]).reshape(bsz, S, nkv, hd).transpose(1, 2)
        v = linear(h, w[f"{p}.self_attn.v_proj.weight"]).reshape(bsz, S, nkv, hd).transpose(1, 2)
        q = rms_norm(q, w[f"{p}.self_attn.q_norm.weight"], eps)           # layers.rs:303-304
        k = rms_norm(k, w[f"{p}.self_attn.k_norm.weight"], eps)
        q = apply_rotary(q, cos, sin)                                      # :307-308
        k = apply_rotary(k, cos, sin)
        if cache[i] is not None:                                           # :311-317
            k = torch.cat([cache[i][0], k], dim=2)
            v = torch.cat([cache[i][1], v], dim=2)
        cache[i] = (k, v)
        kk, vv = repeat_kv(k, nq // nkv), repeat_kv(v, nq // nkv)
        attn = q.matmul(kk.transpose(-2, -1)) / math.sqrt(hd)             # :327-328
        if mask is not None:
            attn = attn + mask
        attn = attn.softmax(-1)
        out = attn.matmul(vv).transpose(1, 2).reshape(bsz, S, nq * hd)
        x = linear(out, w[f"{p}.self_attn.o_proj.weight"]) + res
        res = x
        h = rms_norm(x, w[f"{p}.post_attention_layernorm.weight"], eps)
        g = torch.nn.functional.silu(linear(h, w[f"{p}.mlp.gate_proj.weight"]))   # :396-400
        u = linear(h, w[f"{p}.mlp.up_proj.weight"])
        return linear(g * u, w[f"{p}.mlp.down_proj.weight"]) + res

    def lm_head_weight(self):
        if self.cfg.text.tie_word_embeddings:                              # text_decoder.rs:75-79
            return self.w["thinker.model.embed_tokens.weight"]
        return self.w["thinker.lm_head.weight"]

    def decoder_forward(self, hidden, cos, sin, cache, mask, last_only: bool = False, from_row: int = 0):
        """src/text_decoder.rs:94-113.  ``last_only`` / ``from_row`` skip (unused) lm_head rows -- the
        reference computes all S rows; the values of the rows kept are identical either way."""
        x = hidden
        for i in range(self.cfg.text.num_hidden_layers):
            x = self.decoder_layer(x, i, cos, sin, cache, mask)
        x = rms_norm(x, self.w["thinker.model.norm.weight"], self.cfg.text.rms_norm_eps)
        if last_only:
            x = x[:, -1:, :]
        elif from_row:
            x = x[:, from_row:, :]
        return x.matmul(self.lm_head_weight().t())

    def embed(self, ids: Sequence[int]) -> torch.Tensor:
        return torch.nn.functional.embedding(torch.tensor(list(ids), dtype=torch.int64),
                                             self.w["thinker.model.embed_tokens.weight"])


def causal_mask(seq_len: int, past: int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """full(-inf).triu(past+1) -> [1,1,S,past+S].  src/text_decoder.rs:121-131."""
    m = torch.full((seq_len, past + seq_len), float("-inf"), dtype=dtype)
    return m.triu(past + 1)[None, None]


def build_prompt(num_audio_tokens: int, language_ids: Optional[Sequence[int]] = None) -> Tuple[List[int], int]:
    """src/inference.rs:215-257.  ``language_ids`` = tokenizer.encode("language Xxx") when forced."""
    toks = [IM_START, 8948, 198, IM_END, 198, IM_START, 872, 198, AUDIO_START]
    audio_start = len(toks)
    toks += [AUDIO_PAD] * num_audio_tokens
    toks += [AUDIO_END, IM_END, 198, IM_START, 77091, 198]
    if language_ids is not None:
        toks += list(language_ids)
    return toks, audio_start


@dataclass
class OracleResult:
    ids: List[int]
    mel: torch.Tensor
    audio_embeds: torch.Tensor
    prefill_logits: torch.Tensor          # [V] last row
    step_logits: List[torch.Tensor]       # [V] per generated step (logits that produced ids[i+1])
    timings: Dict[str, float]


def transcribe_ids(model: OracleModel, samples: np.ndarray, language_ids: Optional[Sequence[int]] = None,
                   max_new_tokens: int = 4096, keep_logits: bool = False,
                   lm_head_all_rows: bool = True) -> OracleResult:
    """transcribe() steps 2-8, src/inference.rs:94-200: samples -> generated token ids."""
    import time
    t, tm, dt = model.cfg.text, {}, model.dtype
    t0 = time.perf_counter()
    mel = extract_mel(samples, model.cfg.audio.num_mel_bins, dt)          # step 2
    tm["mel"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    audio = model.encode(mel)                                             # step 3
    tm["encoder"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    ids, a0 = build_prompt(audio.shape[0], language_ids)                  # step 4
    S = len(ids)
    hidden = model.embed(ids).unsqueeze(0)                                # step 5
    hidden[0, a0:a0 + audio.shape[0], :] = audio                          # == T slice_scatter calls (:115-124)
    pos = list(range(S))                                                  # build_position_ids :259-266
    cos, sin = mrope_cos_sin([pos, pos, pos], t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved, dt)
    cache = [None] * t.num_hidden_layers
    logits = model.decoder_forward(hidden, cos, sin, cache, causal_mask(S, 0, dt),
                                   last_only=not lm_head_all_rows)         # step 7
    nxt = logits[:, -1, :]
    tm["prefill"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    prefill_logits = nxt[0].clone()
    out: List[int] = []
    step_logits: List[torch.Tensor] = []
    cur = S
    for _ in range(max_new_tokens):                                       # step 8 (:160-200)
        tok = int(nxt.argmax(-1)[0])
        if tok in EOS_IDS:
            break
        out.append(tok)
        h = model.embed([tok]).unsqueeze(0)
        c1, s1 = mrope_cos_sin([[cur]] * 3, t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved, dt)
        past = cache[0][0].shape[2]
        nxt = model.decoder_forward(h, c1, s1, cache, causal_mask(1, past, dt))[:, 0, :]
        if keep_logits:
            step_logits.append(nxt[0].clone())
        cur += 1
    tm["decode"] = time.perf_counter() - t0
    return OracleResult(out, mel, audio, prefill_logits, step_logits, tm)


def score_ids(model: OracleModel, samples: np.ndarray, ids: Sequence[int],
              language_ids: Optional[Sequence[int]] = None) -> torch.Tensor:
    """Teacher-forced scoring: ONE causal forward over prompt + ``ids`` (positions 0..S + len(ids) - 1), in the
    model's dtype -> logits [len(ids) + 1, V].  Row i is what the greedy loop of transcribe_ids computes before
    choosing ids[i] (row 0: the prefill's last row); the last row follows the last id.  This makes the reference a
    function of any implementation's own ids, so comparisons do not depend on it reproducing the oracle's."""
    t, dt = model.cfg.text, model.dtype
    mel = extract_mel(samples, model.cfg.audio.num_mel_bins, dt)
    audio = model.encode(mel)
    prompt, a0 = build_prompt(audio.shape[0], language_ids)
    S = len(prompt)
    toks = list(prompt) + [int(i) for i in ids]
    hidden = model.embed(toks).unsqueeze(0)
    hidden[0, a0:a0 + audio.shape[0], :] = audio
    pos = list(range(len(toks)))
    cos, sin = mrope_cos_sin([pos, pos, pos], t.head_dim, t.rope_theta, t.mrope_section, t.mrope_interleaved, dt)
    logits = model.decoder_forward(hidden, cos, sin, [None] * t.num_hidden_layers, causal_mask(len(toks), 0, dt),
                                   from_row=S - 1)
    return logits[0]
