// c_api.cu -- the extern "C" boundary (include/asr_b200.h).  Exceptions never cross it: every
// entry point returns a status int and records a thread-local message (idiom of the reference's
// own FFI layer, /root/reference/src/backend/mlx/ffi.rs:60-110).
#include <cstring>
#include <functional>
#include "internal.h"

namespace asrb {
struct Session;
void model_set_tensor(Model* m, const char* name, int dtype, const int64_t* shape, int ndim, const void* host);
void model_finalize(Model* m);
void model_load_dir(Ctx* ctx, const char* dir, Model** out);
Session* session_create(Model* m, int max_batch, int64_t max_samples, int max_lang, int max_context, int max_new);
void session_free(Session* s);
void session_mel(Session* s, const float* const* samples, const int64_t* n_samples, int batch, int64_t* n_frames_out);
void session_mel_read(Session* s, int b, float* out);
void session_encode(Session* s, int64_t* n_tokens_out);
void session_encode_read(Session* s, int b, float* out);
void session_prefill(Session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, int64_t* seq_lens_out, float* last_logits);
void session_decode_step(Session* s, int64_t* next_ids_out, float* logits);
void session_generate(Session* s, int max_new_tokens, int32_t* ids_out, int32_t* lens_out);
void session_transcribe_ids(Session* s, const float* const* samples, const int64_t* n_samples, int batch,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                            int32_t* ids_out, int32_t* lens_out);
void session_last_timings(Session* s, float* ms6, int64_t* kernels, int64_t* steps);
void session_set_option(Session* s, const char* key, const char* value);
void session_stats(Session* s, int64_t* out, int n);
void session_last_logprobs(Session* s, int max_new_tokens, float* out, float* eos_out);
void session_last_top_logprobs(Session* s, int max_new_tokens, int k, int32_t* ids_out, float* lp_out, int32_t* eos_ids_out,
                               float* eos_lp_out);
void session_ingest_pcm(Session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels, const int32_t* rate,
                        const int32_t* format, int batch, int64_t* n_samples_out);
void session_ingested_read(Session* s, int b, float* out);
void session_ingest_long(Session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels, const int32_t* rate,
                         const int32_t* format, int n_files, int64_t* n_samples_out);
void session_long_read(Session* s, int f, float* out);
void session_segment_long(Session* s, int64_t max_seg, int64_t search, int max_segments, int32_t* n_seg_out, int64_t* start_out,
                          int64_t* end_out);
void session_transcribe_segments(Session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                                 const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                                 int32_t* ids_out, int32_t* lens_out);
void session_device_ids(Session* s, const int32_t** ids, const int32_t** lens, int* stride, int* batch);
void session_last_nbest(Session* s, int max_new_tokens, int k, int32_t* ids_out, int32_t* lens_out, float* sum_out,
                        float* score_out, int32_t* eos_out);
void session_last_beam_stats(Session* s, int64_t* out, int n);
void session_set_context(Session* s, int n_rows, const int64_t* const* ids, const int32_t* n_ids);
void session_last_prefill_stats(Session* s, int64_t* out, int n);
void session_score_ids(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* const* lang_ids,
                       const int32_t* n_lang_ids, const int32_t* n_cand, const int64_t* const* cand_ids, const int32_t* cand_len,
                       int max_new_tokens, float* logprob_out, int32_t* top_ids_out, float* top_lp_out);
void session_align_ids(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* const* lang_ids,
                       const int32_t* n_lang_ids, const int64_t* const* ids, const int32_t* n_ids, const int32_t* text_from,
                       const int32_t* heads, int n_heads, int max_ids, int32_t* start_out, int32_t* end_out);
void session_align_segments(Session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                            const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids,
                            int32_t* start_out, int32_t* end_out);
void session_last_align_dims(Session* s, int b, int32_t* n_rows, int32_t* n_tokens);
void session_align_matrix_read(Session* s, int b, float* out);
void session_stream_open(Session* s, int n_streams, int rollback, int unfixed);
void session_stream_reset(Session* s, int b);
void session_stream_push(Session* s, int nst, const float* const* samples, const int64_t* n_samples, const int32_t* is_final,
                         const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens, int max_ids,
                         int32_t* hyp_out, int32_t* hyp_len_out, int32_t* fixed_len_out);
void session_stream_mel_read(Session* s, int b, float* out);
void session_stream_encode_read(Session* s, int b, float* out);
void session_last_stream_stats(Session* s, int64_t* out, int n);
int decode_mega_debug_timeline(long long* out, int cap);
int decode_batch_debug_timeline(long long* out, int cap);
}  // namespace asrb

using namespace asrb;

namespace asrb {
// shared by asrb_model_create and the config.json loader: anything that would divide by zero or index out of bounds later
void validate_dims(const asrb_dims& d) {
    ASRB_REQUIRE(d.num_mel_bins == 128, ASRB_ERR_INVALID, "num_mel_bins must be 128");
    ASRB_REQUIRE(d.n_window > 0 && d.n_window_infer > 0 && d.d_model > 0 && d.encoder_layers > 0 && d.encoder_attention_heads > 0 &&
                     d.d_model % d.encoder_attention_heads == 0 && d.encoder_ffn_dim > 0 && d.downsample_hidden_size > 0 && d.output_dim > 0,
                 ASRB_ERR_INVALID, "bad audio encoder dims");
    ASRB_REQUIRE(d.hidden_size > 0 && d.intermediate_size > 0 && d.num_hidden_layers > 0 && d.num_attention_heads > 0 &&
                     d.num_key_value_heads > 0 && d.num_attention_heads % d.num_key_value_heads == 0 && d.head_dim > 0 && d.head_dim % 2 == 0,
                 ASRB_ERR_INVALID, "bad text decoder dims");
    ASRB_REQUIRE(d.vocab_size > 151676, ASRB_ERR_INVALID, "bad dims (vocab must contain the prompt special tokens)");
    ASRB_REQUIRE(d.rms_norm_eps > 0 && d.rope_theta > 1.0, ASRB_ERR_INVALID, "bad rms_norm_eps / rope_theta");
}
}  // namespace asrb

static thread_local std::string g_last_error;

template <typename F> static int guarded(F&& f) {
    try { f(); return ASRB_OK; }
    catch (const Error& e) { g_last_error = e.what(); return e.code; }
    catch (const std::bad_alloc&) { g_last_error = "host out of memory"; return ASRB_ERR_INVALID; }
    catch (const std::exception& e) { g_last_error = e.what(); return ASRB_ERR_INVALID; }
    catch (...) { g_last_error = "unknown error"; return ASRB_ERR_INVALID; }
}
#define NONNULL(p) ASRB_REQUIRE((p) != nullptr, ASRB_ERR_INVALID, "null pointer: " #p)

namespace asrb {
// the same status / message convention for the test probes (probe.cu)
int run_guarded(const std::function<void()>& f) { return guarded(f); }
}  // namespace asrb

struct asrb_ctx { Ctx c; };
struct asrb_model { Model m; };
struct asrb_session { Session* s; };

extern "C" {

const char* asrb_last_error(void) { return g_last_error.c_str(); }
const char* asrb_version(void) { return "qwen3_asr_rs_b200 0.1 (sm_90a)"; }

int asrb_init(int device, asrb_ctx** out) {
    return guarded([&] {
        NONNULL(out);
        int n = 0;
        ASRB_CUDA_CHECK(cudaGetDeviceCount(&n));
        ASRB_REQUIRE(device >= 0 && device < n, ASRB_ERR_INVALID, "no such CUDA device");
        ASRB_CUDA_CHECK(cudaSetDevice(device));
        cudaDeviceProp p;
        ASRB_CUDA_CHECK(cudaGetDeviceProperties(&p, device));
        ASRB_REQUIRE(p.major == 9 && p.minor == 0, ASRB_ERR_INVALID,
                     "this library is built for sm_90a (H100) only; found compute capability " +
                         std::to_string(p.major) + "." + std::to_string(p.minor));
        asrb_ctx* c = new asrb_ctx();
        c->c.device = device; c->c.sm_count = p.multiProcessorCount; c->c.smem_optin = p.sharedMemPerBlockOptin;
        *out = c;
    });
}
int asrb_ctx_free(asrb_ctx* ctx) { return guarded([&] { delete ctx; }); }

int asrb_dims_default(asrb_dims* d) {
    return guarded([&] {
        NONNULL(d);
        // src/config.rs:52-62, 90-99
        d->d_model = 896; d->encoder_layers = 18; d->encoder_attention_heads = 14; d->encoder_ffn_dim = 3584;
        d->num_mel_bins = 128; d->max_source_positions = 1500; d->n_window = 50; d->n_window_infer = 800;
        d->downsample_hidden_size = 480; d->output_dim = 1024;
        d->vocab_size = 151936; d->hidden_size = 1024; d->intermediate_size = 3072; d->num_hidden_layers = 28;
        d->num_attention_heads = 16; d->num_key_value_heads = 8; d->head_dim = 128; d->tie_word_embeddings = 1;
        d->rms_norm_eps = 1e-6; d->rope_theta = 1000000.0;
    });
}

int asrb_model_create(asrb_ctx* ctx, const asrb_dims* dims, asrb_model** out) {
    return guarded([&] {
        NONNULL(ctx); NONNULL(dims); NONNULL(out);
        validate_dims(*dims);
        ASRB_CUDA_CHECK(cudaSetDevice(ctx->c.device));
        asrb_model* m = new asrb_model();
        m->m.ctx = &ctx->c; m->m.d.c = *dims; m->m.d.derive();
        *out = m;
    });
}
int asrb_model_set_tensor(asrb_model* m, const char* name, int dtype, const int64_t* shape, int ndim, const void* host) {
    return guarded([&] { NONNULL(m); NONNULL(shape); ASRB_CUDA_CHECK(cudaSetDevice(m->m.ctx->device)); model_set_tensor(&m->m, name, dtype, shape, ndim, host); });
}
int asrb_model_finalize(asrb_model* m) {
    return guarded([&] { NONNULL(m); ASRB_CUDA_CHECK(cudaSetDevice(m->m.ctx->device)); model_finalize(&m->m); });
}
int asrb_model_load(asrb_ctx* ctx, const char* model_dir, asrb_model** out) {
    return guarded([&] {
        NONNULL(ctx); NONNULL(model_dir); NONNULL(out);
        ASRB_CUDA_CHECK(cudaSetDevice(ctx->c.device));
        asrb_model* m = new asrb_model();
        m->m.ctx = &ctx->c;
        try {
            Model* mp = &m->m;
            model_load_dir(&ctx->c, model_dir, &mp);
        } catch (...) { delete m; throw; }
        *out = m;
    });
}
int asrb_model_dims(const asrb_model* m, asrb_dims* out) { return guarded([&] { NONNULL(m); NONNULL(out); *out = m->m.d.c; }); }
int asrb_model_lossy_tensors(const asrb_model* m, int* count) { return guarded([&] { NONNULL(m); NONNULL(count); *count = m->m.lossy_count; }); }
int asrb_model_free(asrb_model* m) { return guarded([&] { if (m) { cudaSetDevice(m->m.ctx->device); delete m; } }); }

int asrb_session_create_ex(asrb_model* m, int max_batch, int64_t max_samples, int max_lang_ids, int max_context_ids,
                           int max_new_tokens, asrb_session** out) {
    return guarded([&] {
        NONNULL(m); NONNULL(out);
        asrb_session* s = new asrb_session();
        try { s->s = session_create(&m->m, max_batch, max_samples, max_lang_ids, max_context_ids, max_new_tokens); }
        catch (...) { delete s; throw; }
        *out = s;
    });
}
int asrb_session_create(asrb_model* m, int max_batch, int64_t max_samples, int max_lang_ids, int max_new_tokens, asrb_session** out) {
    return asrb_session_create_ex(m, max_batch, max_samples, max_lang_ids, 0, max_new_tokens, out);
}
int asrb_session_set_context(asrb_session* s, int n_rows, const int64_t* const* ids, const int32_t* n_ids) {
    return guarded([&] { NONNULL(s); session_set_context(s->s, n_rows, ids, n_ids); });
}
int asrb_last_prefill_stats(asrb_session* s, int64_t* out, int n) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_last_prefill_stats(s->s, out, n); });
}
int asrb_session_free(asrb_session* s) { return guarded([&] { if (s) { session_free(s->s); delete s; } }); }

int asrb_transcribe_ids(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch,
                        const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                        int32_t* ids_out, int32_t* lens_out) {
    return guarded([&] { NONNULL(s); NONNULL(samples); NONNULL(n_samples);
                         session_transcribe_ids(s->s, samples, n_samples, batch, lang_ids, n_lang_ids, max_new_tokens, ids_out, lens_out); });
}
int asrb_mel(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch, int64_t* n_frames_out) {
    return guarded([&] { NONNULL(s); NONNULL(samples); NONNULL(n_samples); session_mel(s->s, samples, n_samples, batch, n_frames_out); });
}
int asrb_mel_read(asrb_session* s, int b, float* out) { return guarded([&] { NONNULL(s); NONNULL(out); session_mel_read(s->s, b, out); }); }
int asrb_encode(asrb_session* s, int64_t* n_tokens_out) { return guarded([&] { NONNULL(s); session_encode(s->s, n_tokens_out); }); }
int asrb_encode_read(asrb_session* s, int b, float* out) { return guarded([&] { NONNULL(s); NONNULL(out); session_encode_read(s->s, b, out); }); }
int asrb_prefill(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, int64_t* seq_lens_out, float* last_logits) {
    return guarded([&] { NONNULL(s); session_prefill(s->s, lang_ids, n_lang_ids, seq_lens_out, last_logits); });
}
int asrb_decode_step(asrb_session* s, int64_t* next_ids_out, float* logits) {
    return guarded([&] { NONNULL(s); session_decode_step(s->s, next_ids_out, logits); });
}
int asrb_generate(asrb_session* s, int max_new_tokens, int32_t* ids_out, int32_t* lens_out) {
    return guarded([&] { NONNULL(s); NONNULL(ids_out); NONNULL(lens_out); session_generate(s->s, max_new_tokens, ids_out, lens_out); });
}
int asrb_last_timings(asrb_session* s, float* ms_out6, int64_t* kernels_launched, int64_t* decode_steps) {
    return guarded([&] { NONNULL(s); session_last_timings(s->s, ms_out6, kernels_launched, decode_steps); });
}
int asrb_ingest_pcm(asrb_session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels,
                    const int32_t* sample_rate, const int32_t* format, int batch, int64_t* n_samples_out) {
    return guarded([&] { NONNULL(s); NONNULL(pcm); NONNULL(n_frames); NONNULL(channels); NONNULL(sample_rate); NONNULL(format);
                         session_ingest_pcm(s->s, pcm, n_frames, channels, sample_rate, format, batch, n_samples_out); });
}
int asrb_ingested_read(asrb_session* s, int b, float* out) { return guarded([&] { NONNULL(s); NONNULL(out); session_ingested_read(s->s, b, out); }); }
int asrb_transcribe_ingested(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                             int32_t* ids_out, int32_t* lens_out) {
    return guarded([&] { NONNULL(s); session_transcribe_ids(s->s, nullptr, nullptr, 0, lang_ids, n_lang_ids, max_new_tokens, ids_out, lens_out); });
}
int asrb_ingest_long(asrb_session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels,
                     const int32_t* sample_rate, const int32_t* format, int n_files, int64_t* n_samples_out) {
    return guarded([&] { NONNULL(s); NONNULL(pcm); NONNULL(n_frames); NONNULL(channels); NONNULL(sample_rate); NONNULL(format);
                         session_ingest_long(s->s, pcm, n_frames, channels, sample_rate, format, n_files, n_samples_out); });
}
int asrb_long_read(asrb_session* s, int file, float* out) { return guarded([&] { NONNULL(s); NONNULL(out); session_long_read(s->s, file, out); }); }
int asrb_segment_long(asrb_session* s, int64_t max_segment_samples, int64_t search_samples, int max_segments,
                      int32_t* n_segments_out, int64_t* start_out, int64_t* end_out) {
    return guarded([&] { NONNULL(s); NONNULL(n_segments_out); NONNULL(start_out); NONNULL(end_out);
                         session_segment_long(s->s, max_segment_samples, search_samples, max_segments, n_segments_out, start_out, end_out); });
}
int asrb_transcribe_segments(asrb_session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                             const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                             int32_t* ids_out, int32_t* lens_out) {
    return guarded([&] { NONNULL(s); NONNULL(file); NONNULL(start); NONNULL(end); NONNULL(ids_out); NONNULL(lens_out);
                         session_transcribe_segments(s->s, n, file, start, end, lang_ids, n_lang_ids, max_new_tokens, ids_out, lens_out); });
}
int asrb_session_device_ids(asrb_session* s, const int32_t** ids_dev, const int32_t** lens_dev, int* row_stride, int* batch) {
    return guarded([&] { NONNULL(s); NONNULL(ids_dev); NONNULL(lens_dev); NONNULL(row_stride); NONNULL(batch);
                         session_device_ids(s->s, ids_dev, lens_dev, row_stride, batch); });
}
int asrb_session_stats(asrb_session* s, int64_t* out, int n) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_stats(s->s, out, n); });
}
int asrb_session_set_option(asrb_session* s, const char* key, const char* value) {
    return guarded([&] { NONNULL(s); session_set_option(s->s, key, value); });
}
int asrb_last_logprobs(asrb_session* s, int max_new_tokens, float* logprobs_out, float* eos_logprob_out) {
    return guarded([&] { NONNULL(s); NONNULL(logprobs_out); session_last_logprobs(s->s, max_new_tokens, logprobs_out, eos_logprob_out); });
}
int asrb_last_top_logprobs(asrb_session* s, int max_new_tokens, int k, int32_t* ids_out, float* logprobs_out,
                           int32_t* eos_ids_out, float* eos_logprobs_out) {
    return guarded([&] {
        NONNULL(s); NONNULL(ids_out); NONNULL(logprobs_out);
        session_last_top_logprobs(s->s, max_new_tokens, k, ids_out, logprobs_out, eos_ids_out, eos_logprobs_out);
    });
}
int asrb_last_nbest(asrb_session* s, int max_new_tokens, int k, int32_t* ids_out, int32_t* lens_out, float* sum_logprob_out,
                    float* score_out, int32_t* eos_id_out) {
    return guarded([&] {
        NONNULL(s); NONNULL(ids_out); NONNULL(lens_out);
        session_last_nbest(s->s, max_new_tokens, k, ids_out, lens_out, sum_logprob_out, score_out, eos_id_out);
    });
}
int asrb_last_beam_stats(asrb_session* s, int64_t* out, int n) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_last_beam_stats(s->s, out, n); });
}
int asrb_score_ids(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch,
                   const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int32_t* n_cand,
                   const int64_t* const* cand_ids, const int32_t* cand_len, int max_new_tokens, float* logprob_out,
                   int32_t* top_ids_out, float* top_lp_out) {
    return guarded([&] { NONNULL(s); NONNULL(samples); NONNULL(n_samples);
                         session_score_ids(s->s, samples, n_samples, batch, lang_ids, n_lang_ids, n_cand, cand_ids, cand_len,
                                           max_new_tokens, logprob_out, top_ids_out, top_lp_out); });
}
int asrb_score_ingested(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int32_t* n_cand,
                        const int64_t* const* cand_ids, const int32_t* cand_len, int max_new_tokens, float* logprob_out,
                        int32_t* top_ids_out, float* top_lp_out) {
    return guarded([&] { NONNULL(s);
                         session_score_ids(s->s, nullptr, nullptr, 0, lang_ids, n_lang_ids, n_cand, cand_ids, cand_len,
                                           max_new_tokens, logprob_out, top_ids_out, top_lp_out); });
}

int asrb_align_ids(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch,
                   const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids, const int32_t* n_ids,
                   const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids, int32_t* start_frame_out,
                   int32_t* end_frame_out) {
    return guarded([&] { NONNULL(s); NONNULL(samples); NONNULL(n_samples);
                         session_align_ids(s->s, samples, n_samples, batch, lang_ids, n_lang_ids, ids, n_ids, text_from, heads,
                                           n_heads, max_ids, start_frame_out, end_frame_out); });
}
int asrb_align_ingested(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                        const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids,
                        int32_t* start_frame_out, int32_t* end_frame_out) {
    return guarded([&] { NONNULL(s);
                         session_align_ids(s->s, nullptr, nullptr, 0, lang_ids, n_lang_ids, ids, n_ids, text_from, heads,
                                           n_heads, max_ids, start_frame_out, end_frame_out); });
}
int asrb_align_segments(asrb_session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                        const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                        const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids,
                        int32_t* start_frame_out, int32_t* end_frame_out) {
    return guarded([&] { NONNULL(s); NONNULL(file); NONNULL(start); NONNULL(end);
                         session_align_segments(s->s, n, file, start, end, lang_ids, n_lang_ids, ids, n_ids, text_from, heads,
                                                n_heads, max_ids, start_frame_out, end_frame_out); });
}
int asrb_last_align_dims(asrb_session* s, int b, int32_t* n_rows_out, int32_t* n_tokens_out) {
    return guarded([&] { NONNULL(s); session_last_align_dims(s->s, b, n_rows_out, n_tokens_out); });
}
int asrb_align_matrix_read(asrb_session* s, int b, float* out) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_align_matrix_read(s->s, b, out); });
}

int asrb_stream_open(asrb_session* s, int n_streams, int rollback_ids, int unfixed_pushes) {
    return guarded([&] { NONNULL(s); session_stream_open(s->s, n_streams, rollback_ids, unfixed_pushes); });
}
int asrb_stream_reset(asrb_session* s, int stream) { return guarded([&] { NONNULL(s); session_stream_reset(s->s, stream); }); }
int asrb_stream_push(asrb_session* s, int n_streams, const float* const* samples, const int64_t* n_samples, const int32_t* is_final,
                     const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens, int max_ids,
                     int32_t* hyp_out, int32_t* hyp_len_out, int32_t* fixed_len_out) {
    return guarded([&] { NONNULL(s); NONNULL(n_samples); NONNULL(hyp_out); NONNULL(hyp_len_out); NONNULL(fixed_len_out);
                         session_stream_push(s->s, n_streams, samples, n_samples, is_final, lang_ids, n_lang_ids, max_new_tokens,
                                             max_ids, hyp_out, hyp_len_out, fixed_len_out); });
}
int asrb_stream_mel_read(asrb_session* s, int stream, float* out) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_stream_mel_read(s->s, stream, out); });
}
int asrb_stream_encode_read(asrb_session* s, int stream, float* out) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_stream_encode_read(s->s, stream, out); });
}
int asrb_last_stream_stats(asrb_session* s, int64_t* out, int n) {
    return guarded([&] { NONNULL(s); NONNULL(out); session_last_stream_stats(s->s, out, n); });
}

int asrb_debug_mega_timeline(long long* out, int cap) {
    int n = 0;
    guarded([&] { n = (getenv("ASRB_MEGA_DEBUG") && std::string(getenv("ASRB_MEGA_DEBUG")) == "batch") ? decode_batch_debug_timeline(out, cap)
                                                                                                            : decode_mega_debug_timeline(out, cap); });
    return n;
}

}  // extern "C"
