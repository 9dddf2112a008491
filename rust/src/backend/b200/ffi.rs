//! Raw bindings of `include/asr_b200.h` (libasr_b200.so).  Same idiom as `src/backend/mlx/ffi.rs:60-110`:
//! every function returns an `int` status (0 = ok), results come back through out-parameters, handles are opaque.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_longlong, c_void};

pub const ASRB_OK: c_int = 0;
pub const ASRB_ERR_INVALID: c_int = 1;
pub const ASRB_ERR_CUDA: c_int = 2;
pub const ASRB_ERR_IO: c_int = 3;
pub const ASRB_ERR_STATE: c_int = 4;

pub const ASRB_DT_F32: c_int = 0;
pub const ASRB_DT_BF16: c_int = 1;
pub const ASRB_DT_F16: c_int = 2;

#[repr(C)] pub struct asrb_ctx { _private: [u8; 0] }
#[repr(C)] pub struct asrb_model { _private: [u8; 0] }
#[repr(C)] pub struct asrb_session { _private: [u8; 0] }

/// `asrb_dims`: the fields of `src/config.rs:27-113`.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct AsrbDims {
    pub d_model: i32, pub encoder_layers: i32, pub encoder_attention_heads: i32, pub encoder_ffn_dim: i32,
    pub num_mel_bins: i32, pub max_source_positions: i32, pub n_window: i32, pub n_window_infer: i32,
    pub downsample_hidden_size: i32, pub output_dim: i32,
    pub vocab_size: i32, pub hidden_size: i32, pub intermediate_size: i32, pub num_hidden_layers: i32,
    pub num_attention_heads: i32, pub num_key_value_heads: i32, pub head_dim: i32,
    pub tie_word_embeddings: i32,
    pub rms_norm_eps: f64, pub rope_theta: f64,
}

extern "C" {
    pub fn asrb_init(device: c_int, out: *mut *mut asrb_ctx) -> c_int;
    pub fn asrb_ctx_free(ctx: *mut asrb_ctx) -> c_int;
    pub fn asrb_last_error() -> *const c_char;
    pub fn asrb_version() -> *const c_char;

    pub fn asrb_dims_default(d: *mut AsrbDims) -> c_int;
    pub fn asrb_model_load(ctx: *mut asrb_ctx, model_dir: *const c_char, out: *mut *mut asrb_model) -> c_int;
    pub fn asrb_model_create(ctx: *mut asrb_ctx, dims: *const AsrbDims, out: *mut *mut asrb_model) -> c_int;
    pub fn asrb_model_set_tensor(m: *mut asrb_model, name: *const c_char, dtype: c_int, shape: *const i64, ndim: c_int, host_data: *const c_void) -> c_int;
    pub fn asrb_model_finalize(m: *mut asrb_model) -> c_int;
    pub fn asrb_model_dims(m: *const asrb_model, out: *mut AsrbDims) -> c_int;
    pub fn asrb_model_lossy_tensors(m: *const asrb_model, count: *mut c_int) -> c_int;
    pub fn asrb_model_free(m: *mut asrb_model) -> c_int;

    pub fn asrb_session_create(m: *mut asrb_model, max_batch: c_int, max_samples: i64, max_lang_ids: c_int, max_new_tokens: c_int, out: *mut *mut asrb_session) -> c_int;
    pub fn asrb_session_create_ex(m: *mut asrb_model, max_batch: c_int, max_samples: i64, max_lang_ids: c_int, max_context_ids: c_int, max_new_tokens: c_int, out: *mut *mut asrb_session) -> c_int;
    pub fn asrb_session_free(s: *mut asrb_session) -> c_int;
    pub fn asrb_session_set_context(s: *mut asrb_session, n_rows: c_int, ids: *const *const i64, n_ids: *const i32) -> c_int;
    pub fn asrb_last_prefill_stats(s: *mut asrb_session, out: *mut i64, n: c_int) -> c_int;

    pub fn asrb_transcribe_ids(s: *mut asrb_session, samples: *const *const f32, n_samples: *const i64, batch: c_int, lang_ids: *const *const i64, n_lang_ids: *const i32, max_new_tokens: c_int, ids_out: *mut i32, lens_out: *mut i32) -> c_int;

    pub fn asrb_mel(s: *mut asrb_session, samples: *const *const f32, n_samples: *const i64, batch: c_int, n_frames_out: *mut i64) -> c_int;
    pub fn asrb_mel_read(s: *mut asrb_session, b: c_int, out: *mut f32) -> c_int;
    pub fn asrb_encode(s: *mut asrb_session, n_tokens_out: *mut i64) -> c_int;
    pub fn asrb_encode_read(s: *mut asrb_session, b: c_int, out: *mut f32) -> c_int;
    pub fn asrb_prefill(s: *mut asrb_session, lang_ids: *const *const i64, n_lang_ids: *const i32, seq_lens_out: *mut i64, last_logits: *mut f32) -> c_int;
    pub fn asrb_decode_step(s: *mut asrb_session, next_ids_out: *mut i64, logits: *mut f32) -> c_int;
    pub fn asrb_generate(s: *mut asrb_session, max_new_tokens: c_int, ids_out: *mut i32, lens_out: *mut i32) -> c_int;

    pub fn asrb_last_timings(s: *mut asrb_session, ms_out6: *mut f32, kernels_launched: *mut i64, decode_steps: *mut i64) -> c_int;
    pub fn asrb_ingest_pcm(s: *mut asrb_session, pcm: *const *const c_void, n_frames: *const i64, channels: *const i32, sample_rate: *const i32, format: *const i32, batch: c_int, n_samples_out: *mut i64) -> c_int;
    pub fn asrb_ingested_read(s: *mut asrb_session, b: c_int, out: *mut f32) -> c_int;
    pub fn asrb_transcribe_ingested(s: *mut asrb_session, lang_ids: *const *const i64, n_lang_ids: *const i32, max_new_tokens: c_int, ids_out: *mut i32, lens_out: *mut i32) -> c_int;
    pub fn asrb_ingest_long(s: *mut asrb_session, pcm: *const *const c_void, n_frames: *const i64, channels: *const i32, sample_rate: *const i32, format: *const i32, n_files: c_int, n_samples_out: *mut i64) -> c_int;
    pub fn asrb_long_read(s: *mut asrb_session, file: c_int, out: *mut f32) -> c_int;
    pub fn asrb_segment_long(s: *mut asrb_session, max_segment_samples: i64, search_samples: i64, max_segments: c_int, n_segments_out: *mut i32, start_out: *mut i64, end_out: *mut i64) -> c_int;
    pub fn asrb_transcribe_segments(s: *mut asrb_session, n: c_int, file: *const i32, start: *const i64, end: *const i64, lang_ids: *const *const i64, n_lang_ids: *const i32, max_new_tokens: c_int, ids_out: *mut i32, lens_out: *mut i32) -> c_int;
    pub fn asrb_score_ids(s: *mut asrb_session, samples: *const *const f32, n_samples: *const i64, batch: c_int,
                          lang_ids: *const *const i64, n_lang_ids: *const i32, n_cand: *const i32, cand_ids: *const *const i64,
                          cand_len: *const i32, max_new_tokens: c_int, logprob_out: *mut f32, top_ids_out: *mut i32,
                          top_lp_out: *mut f32) -> c_int;
    pub fn asrb_score_ingested(s: *mut asrb_session, lang_ids: *const *const i64, n_lang_ids: *const i32, n_cand: *const i32,
                               cand_ids: *const *const i64, cand_len: *const i32, max_new_tokens: c_int, logprob_out: *mut f32,
                               top_ids_out: *mut i32, top_lp_out: *mut f32) -> c_int;
    pub fn asrb_align_ids(s: *mut asrb_session, samples: *const *const f32, n_samples: *const i64, batch: c_int,
                          lang_ids: *const *const i64, n_lang_ids: *const i32, ids: *const *const i64, n_ids: *const i32,
                          text_from: *const i32, heads: *const i32, n_heads: c_int, max_ids: c_int,
                          start_frame_out: *mut i32, end_frame_out: *mut i32) -> c_int;
    pub fn asrb_align_ingested(s: *mut asrb_session, lang_ids: *const *const i64, n_lang_ids: *const i32, ids: *const *const i64,
                               n_ids: *const i32, text_from: *const i32, heads: *const i32, n_heads: c_int, max_ids: c_int,
                               start_frame_out: *mut i32, end_frame_out: *mut i32) -> c_int;
    pub fn asrb_align_segments(s: *mut asrb_session, n: c_int, file: *const i32, start: *const i64, end: *const i64,
                               lang_ids: *const *const i64, n_lang_ids: *const i32, ids: *const *const i64, n_ids: *const i32,
                               text_from: *const i32, heads: *const i32, n_heads: c_int, max_ids: c_int,
                               start_frame_out: *mut i32, end_frame_out: *mut i32) -> c_int;
    pub fn asrb_last_align_dims(s: *mut asrb_session, b: c_int, n_rows_out: *mut i32, n_tokens_out: *mut i32) -> c_int;
    pub fn asrb_align_matrix_read(s: *mut asrb_session, b: c_int, out: *mut f32) -> c_int;
    pub fn asrb_session_device_ids(s: *mut asrb_session, ids_dev: *mut *const i32, lens_dev: *mut *const i32, row_stride: *mut c_int, batch: *mut c_int) -> c_int;
    pub fn asrb_session_stats(s: *mut asrb_session, out: *mut i64, n: c_int) -> c_int;
    pub fn asrb_session_set_option(s: *mut asrb_session, key: *const c_char, value: *const c_char) -> c_int;
    pub fn asrb_last_logprobs(s: *mut asrb_session, max_new_tokens: c_int, logprobs_out: *mut f32, eos_logprob_out: *mut f32) -> c_int;
    pub fn asrb_last_top_logprobs(s: *mut asrb_session, max_new_tokens: c_int, k: c_int, ids_out: *mut i32, logprobs_out: *mut f32,
                                  eos_ids_out: *mut i32, eos_logprobs_out: *mut f32) -> c_int;
    pub fn asrb_last_nbest(s: *mut asrb_session, max_new_tokens: c_int, k: c_int, ids_out: *mut i32, lens_out: *mut i32,
                           sum_logprob_out: *mut f32, score_out: *mut f32, eos_id_out: *mut i32) -> c_int;
    pub fn asrb_last_beam_stats(s: *mut asrb_session, out: *mut i64, n: c_int) -> c_int;
    pub fn asrb_stream_open(s: *mut asrb_session, n_streams: c_int, rollback_ids: c_int, unfixed_pushes: c_int) -> c_int;
    pub fn asrb_stream_reset(s: *mut asrb_session, stream: c_int) -> c_int;
    pub fn asrb_stream_push(s: *mut asrb_session, n_streams: c_int, samples: *const *const f32, n_samples: *const i64,
                            is_final: *const i32, lang_ids: *const *const i64, n_lang_ids: *const i32, max_new_tokens: c_int,
                            max_ids: c_int, hyp_out: *mut i32, hyp_len_out: *mut i32, fixed_len_out: *mut i32) -> c_int;
    pub fn asrb_stream_mel_read(s: *mut asrb_session, stream: c_int, out: *mut f32) -> c_int;
    pub fn asrb_stream_encode_read(s: *mut asrb_session, stream: c_int, out: *mut f32) -> c_int;
    pub fn asrb_last_stream_stats(s: *mut asrb_session, out: *mut i64, n: c_int) -> c_int;
    pub fn asrb_debug_mega_timeline(out: *mut c_longlong, cap: c_int) -> c_int;
}
