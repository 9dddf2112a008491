/*
 * asr_b200.h -- C ABI of the H100-native (sm_90a) Qwen3-ASR hot path.
 *
 * Drop-in boundary for second-state/qwen3_asr_rs (reference paths relative to
 * /root/reference).  The reference has no backend trait: its seam is the cfg-switched
 * `struct Tensor` (src/tensor.rs:120-126) that the three hot modules call
 * (src/mel.rs, src/audio_encoder.rs, src/text_decoder.rs) from
 * `AsrInference::transcribe` (src/inference.rs:89-213).  This library replaces the
 * span steps 2-8 of that function (src/inference.rs:94-200) -- f32 samples in host
 * memory -> generated token ids in host memory -- with hand-written sm_90a kernels.
 * A third `#[cfg(feature = "b200")]` arm binds these symbols (INTEGRATION.md).
 *
 * Conventions follow the reference's own FFI idiom (src/backend/mlx/ffi.rs:60-110):
 * every function returns an int status (0 = ok), results come back through
 * out-parameters, handles are opaque, every handle has an explicit _free.  Nothing
 * throws or aborts across this boundary; asrb_last_error() returns a thread-local
 * message for the last non-zero status.  No torch / C++ types appear in signatures.
 *
 * Threading: one CUDA stream per session; distinct sessions may be driven from
 * distinct threads; a single session is not re-entrant (the reference is
 * single-threaded and synchronous, src/inference.rs:89).
 */
#ifndef ASR_B200_H
#define ASR_B200_H

#include <stdint.h>

#if defined(__GNUC__)
#define ASRB_API __attribute__((visibility("default")))
#else
#define ASRB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define ASRB_OK 0
#define ASRB_ERR_INVALID 1   /* bad argument / shape / missing tensor            */
#define ASRB_ERR_CUDA 2      /* CUDA runtime or driver error                      */
#define ASRB_ERR_IO 3        /* model directory / safetensors / config.json       */
#define ASRB_ERR_STATE 4     /* call order (e.g. encode before mel)               */

typedef struct asrb_ctx asrb_ctx;         /* one per device                              */
typedef struct asrb_model asrb_model;     /* immutable weights, shareable by sessions   */
typedef struct asrb_session asrb_session; /* KV cache, scratch, streams for ONE batch   */

/* dtype codes for asrb_model_set_tensor (safetensors dtypes the reference accepts,
 * src/weights.rs:74-117) */
#define ASRB_DT_F32 0
#define ASRB_DT_BF16 1
#define ASRB_DT_F16 2

/* Model hyper-parameters: the fields of src/config.rs:27-113, defaults = 0.6B. */
typedef struct asrb_dims {
    /* audio encoder (AudioEncoderConfig, src/config.rs:27-62) */
    int32_t d_model, encoder_layers, encoder_attention_heads, encoder_ffn_dim;
    int32_t num_mel_bins, max_source_positions, n_window, n_window_infer;
    int32_t downsample_hidden_size, output_dim;
    /* text decoder (TextDecoderConfig, src/config.rs:66-113) */
    int32_t vocab_size, hidden_size, intermediate_size, num_hidden_layers;
    int32_t num_attention_heads, num_key_value_heads, head_dim;
    int32_t tie_word_embeddings;
    double rms_norm_eps, rope_theta;
} asrb_dims;

/* ---- context --------------------------------------------------------------------- */
/* replaces the device pick of src/main.rs:51-58 */
ASRB_API int asrb_init(int device, asrb_ctx** out);
ASRB_API int asrb_ctx_free(asrb_ctx* ctx);
ASRB_API const char* asrb_last_error(void);
ASRB_API const char* asrb_version(void);

/* ---- model ----------------------------------------------------------------------- */
/* fills *d with src/config.rs defaults (Qwen3-ASR-0.6B) */
ASRB_API int asrb_dims_default(asrb_dims* d);
/* AsrInference::load (src/inference.rs:30-86): config.json + model.safetensors or
 * model.safetensors.index.json + shards (src/weights.rs:10-58).  bf16 stays bf16. */
ASRB_API int asrb_model_load(asrb_ctx* ctx, const char* model_dir, asrb_model** out);
/* Incremental construction (what load() does internally; also used by tests to
 * build models in memory): create -> set_tensor for every HF name -> finalize. */
ASRB_API int asrb_model_create(asrb_ctx* ctx, const asrb_dims* dims, asrb_model** out);
ASRB_API int asrb_model_set_tensor(asrb_model* m, const char* name, int dtype,
                          const int64_t* shape, int ndim, const void* host_data);
ASRB_API int asrb_model_finalize(asrb_model* m);
ASRB_API int asrb_model_dims(const asrb_model* m, asrb_dims* out);
/* Matrices are kept in bf16 (lossless for the released bf16 checkpoints; the reference widens them to f32,
 * src/weights.rs:74-89).  An F32/F16 matrix that is not bf16-representable is REJECTED by set_tensor / load unless
 * ASRB_ALLOW_LOSSY_WEIGHTS=1; *count = number of matrices that were rounded under that override (0 = exact). */
ASRB_API int asrb_model_lossy_tensors(const asrb_model* m, int* count);
ASRB_API int asrb_model_free(asrb_model* m);

/* ---- session --------------------------------------------------------------------- */
/* Capacity: up to max_batch utterances of up to max_samples samples each, prompt
 * suffix of up to max_lang_ids forced-language ids, up to max_new_tokens generated
 * ids (the reference caps at 4096, src/inference.rs:153).
 * ASRB_ERR_INVALID when the context (audio tokens + prompt + max_new_tokens positions) exceeds the RoPE table, or when
 * group * (128 + context) fp32 values (group = num_attention_heads / num_key_value_heads) do not fit the shared memory a
 * block may opt in to: the per-phase decode attention keeps one score per (query head of a group, key) there. */
ASRB_API int asrb_session_create(asrb_model* m, int max_batch, int64_t max_samples,
                        int max_lang_ids, int max_new_tokens, asrb_session** out);
/* asrb_session_create with room for up to max_context_ids context ids per utterance (asrb_session_set_context);
 * asrb_session_create is this call with max_context_ids = 0.  Every prompt, the KV cache and the RoPE-table check
 * (prompt + max_new_tokens positions) include them. */
ASRB_API int asrb_session_create_ex(asrb_model* m, int max_batch, int64_t max_samples, int max_lang_ids,
                                    int max_context_ids, int max_new_tokens, asrb_session** out);
ASRB_API int asrb_session_free(asrb_session* s);

/* Whole hot path, the call `transcribe()` makes once per file (src/inference.rs:94-200)
 * generalised to a batch of independent utterances:
 *   samples[b]        f32 mono 16 kHz (src/mel.rs:49), n_samples[b] of them
 *   lang_ids[b]       NULL, or the ids of tokenizer.encode("language Xxx")
 *                     (src/inference.rs:246-250) appended to the prompt
 *   ids_out           [batch][max_new_tokens] generated ids (EOS excluded)
 *   lens_out          [batch] number of ids generated
 * Greedy argmax; stops a sequence at EOS {151643,151645} (src/inference.rs:154,163)
 * or at max_new_tokens. */
ASRB_API int asrb_transcribe_ids(asrb_session* s, const float* const* samples, const int64_t* n_samples,
                        int batch, const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                        int max_new_tokens, int32_t* ids_out, int32_t* lens_out);

/* ---- GPU-side audio ingest (step 1 of transcribe(), load_audio_wav + resample, src/audio.rs:162-245) ----------- */
/* Raw interleaved PCM of `batch` utterances (hound samples: s16 / s32 scaled by 2^-(bits-1), or f32; src/audio.rs:181-189)
 * -> mono mixdown (mean over channels, :193-206) -> 16 kHz (:209-213) ON THE GPU, written straight into the session's
 * sample buffer: the payload crosses PCIe once in its native format.  The resampler is the polyphase FIR of
 * scipy.signal.resample_poly (the reference's rubato / swresample interpolators are not reproducible here); this stage
 * is outside the parity point of the hot path and is pinned by its own golden (tests/test_gpu_parity.py).
 * n_samples_out[b] = number of 16 kHz samples produced.  Follow with asrb_transcribe_ingested (or asrb_mel with
 * samples == NULL). */
#define ASRB_PCM_S16 0
#define ASRB_PCM_F32 1
#define ASRB_PCM_S32 2
ASRB_API int asrb_ingest_pcm(asrb_session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels,
                    const int32_t* sample_rate, const int32_t* format, int batch, int64_t* n_samples_out);
ASRB_API int asrb_ingested_read(asrb_session* s, int b, float* out /* [n_samples[b]] */);
/* asrb_transcribe_ids on the utterances ingested by the last asrb_ingest_pcm */
ASRB_API int asrb_transcribe_ingested(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                             int max_new_tokens, int32_t* ids_out, int32_t* lens_out);

/* ---- long-form audio: cut recordings at low-energy points, decode the pieces as one batch -------------------------- */
/* asrb_ingest_pcm's ingest (same arguments, same kernels) into a separate long-audio buffer that the session grows on
 * demand: files are not bounded by max_samples, and what asrb_ingest_pcm / asrb_transcribe_ingested consume is left as
 * it is.  File f keeps n_samples_out[f] 16 kHz samples until the next asrb_ingest_long; a failed call leaves none. */
ASRB_API int asrb_ingest_long(asrb_session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels,
                              const int32_t* sample_rate, const int32_t* format, int n_files, int64_t* n_samples_out);
ASRB_API int asrb_long_read(asrb_session* s, int file, float* out /* [n_samples[file]] */);
/* Cut points of every ingested file, on the GPU.  Window energy e[j] = sum x[i]^2, i in [160 j, 160 j + 1600) (100 ms
 * every 10 ms, f32 samples accumulated in fp64, deterministic).  For a file of N samples: c_0 = 0; while
 * N - c_k > max_segment_samples, c_{k+1} is the window centre p = 160 j + 800 with the least e[j] among
 *   c_k + max_segment_samples - search_samples <= p <= min(c_k + max_segment_samples, N - 16000),
 * ties to the largest p.  The segments are [c_k, c_{k+1}) and [c_K, N): each at most max_segment_samples, the last at
 * least 1 s; a file of at most max_segment_samples is the one segment [0, N).
 *   n_segments_out   [n_files] segments per file
 *   start_out/end_out [max_segments] sample offsets within the file, in (file, time) order
 * ASRB_ERR_INVALID: max_segment_samples / search_samples not multiples of 160, max_segment_samples < 80000 (5 s),
 * search_samples < 32000 (2 s) or > max_segment_samples / 2; or more segments than max_segments, in which case
 * n_segments_out is still filled so the caller can retry.  ASRB_ERR_STATE if nothing was ingested. */
ASRB_API int asrb_segment_long(asrb_session* s, int64_t max_segment_samples, int64_t search_samples, int max_segments,
                               int32_t* n_segments_out, int64_t* start_out, int64_t* end_out);
/* asrb_transcribe_ids on n views [start[i], end[i]) of ingested file file[i] as one batch of n utterances, read in place
 * by the mel (no copy).  The views may come from asrb_segment_long or from the caller (their own VAD).  Everything that
 * applies to asrb_transcribe_ids applies unchanged: options, contexts, asrb_last_logprobs / _top_logprobs / _nbest /
 * _timings / _prefill_stats, asrb_session_device_ids; the sampling row r is the view's position in this call.
 * ASRB_ERR_INVALID before any work: a file index out of range, start >= end, end past the file, a view longer than
 * max_samples or shorter than 201 samples, n < 1, or n (x beam_size) > max_batch.  ASRB_ERR_STATE if nothing was
 * ingested with asrb_ingest_long. */
ASRB_API int asrb_transcribe_segments(asrb_session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                                      const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                                      int32_t* ids_out, int32_t* lens_out);

/* Stage entry points = the calls transcribe() makes (each runs on the session stream;
 * *_read functions synchronise and copy to host, for parity tests). */
/* WhisperFeatureExtractor::extract, src/mel.rs:49-96 (called at src/inference.rs:95) */
ASRB_API int asrb_mel(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch,
             int64_t* n_frames_out);
ASRB_API int asrb_mel_read(asrb_session* s, int b, float* out /* [num_mel_bins * n_frames[b]] */);
/* AudioEncoder::forward, src/audio_encoder.rs:79-169 (src/inference.rs:100) */
ASRB_API int asrb_encode(asrb_session* s, int64_t* n_tokens_out);
ASRB_API int asrb_encode_read(asrb_session* s, int b, float* out /* [n_tokens[b] * output_dim] */);
/* build_prompt + embed + inject + MRoPE + prefill, src/inference.rs:105-149; writes the
 * last-row logits [batch][vocab] if last_logits != NULL (parity mode) */
ASRB_API int asrb_prefill(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                 int64_t* seq_lens_out, float* last_logits);
/* one greedy iteration, src/inference.rs:160-200: argmax of the pending logits ->
 * next_ids_out[b] (-1 when b already hit EOS) -> embed -> decoder forward with S=1;
 * logits [batch][vocab] if non-NULL */
ASRB_API int asrb_decode_step(asrb_session* s, int64_t* next_ids_out, float* logits);
/* remaining iterations with no per-token host sync */
ASRB_API int asrb_generate(asrb_session* s, int max_new_tokens, int32_t* ids_out, int32_t* lens_out);

/* ---- introspection for bench / tests ---------------------------------------------- */
/* per-stage device milliseconds of the last asrb_transcribe_ids (CUDA events on the session
 * stream): [0]=h2d of samples [1]=mel [2]=encoder [3]=prefill [4]=decode loop [5]=total;
 * plus counters (kernels launched, decoder forward steps) */
ASRB_API int asrb_last_timings(asrb_session* s, float* ms_out6, int64_t* kernels_launched,
                      int64_t* decode_steps);
/* Device-resident results of the last asrb_generate / asrb_transcribe_ids (valid until the next call on this
 * session; the session stream has been synchronised): ids [max_batch][max_new_tokens] int32 and lens [max_batch]
 * int32 in HBM.  This is what the multi-GPU gather (the path's only collective: one all-gather of ids over
 * NCCL / NVLink, SURVEY.md section 8e) reads directly, with no host staging. */
ASRB_API int asrb_session_device_ids(asrb_session* s, const int32_t** ids_dev, const int32_t** lens_dev,
                            int* row_stride, int* batch);
/* Path counters since session creation -- silent fallbacks made visible (bench.py asserts the fallback ones are 0):
 *   [0] decoder forwards on the batch-aware fused step   [1] on the single-sequence fused step
 *   [2] on the per-phase kernels (fallback: logits requested, unsupported dims, context beyond the fused limit)
 *   [3] GEMMs that fell back from wgmma to the SIMT kernel (process-wide)   [4] wgmma GEMM launches (process-wide)
 *   greedy single-sequence fused step, lm_head read from its int8 copy (DESIGN.md section 4.1):
 *   [5] rows recomputed from bf16 as candidates for the argmax   [6] most rows recomputed in one step
 *   [7] CTA slices recomputed in full (candidate list overflow or a non-finite bound)
 * writes min(n, 8) values (n > 5 waits for the session's stream) */
ASRB_API int asrb_session_stats(asrb_session* s, int64_t* out, int n);
/* knobs: "gemm" = "tc"|"simt", "decode" = "mega"|"phases", "batch_step" = "1"|"0", "planes" = "1"|"2"|"3",
 * "resident" = "1"|"0" (1: the samples uploaded by the previous call are reused, no H2D),
 * "logprobs" = "1"|"0" (1: every greedy step also records the log-probability of the token it selects, read with
 * asrb_last_logprobs; same ids, same decode paths; the value in effect at the prefill applies to the whole run),
 * "top_logprobs" = "0".."8" (k >= 1: every greedy step also records its k best candidates, read with
 * asrb_last_top_logprobs, and the log-probabilities asrb_last_logprobs reads; same ids, same decode paths; the value in
 * effect at the prefill applies to the whole run),
 * "temperature" = a decimal string, "0" (default: greedy) or a finite value in [1e-6, 100]: every step samples its
 * token by the Gumbel-max draw below instead of taking the argmax, on every decode path,
 * "seed" = a decimal unsigned 64-bit integer (default "0") seeding that draw.
 * Both are latched at the prefill and apply to the whole run.  The draw for sequence row r (0-based in the call's
 * batch), step n (ids already generated for that sequence when the step selects; 0 after the prefill) and token id v:
 * x0 = word 0 of Philox4x32-10 (Random123 constants) with key (seed & 0xffffffff, seed >> 32) and counter (v, n, r, 0),
 * u = (float)((x0 >> 8) | 1) * 2^-24, g = -logf(-logf(u)), key = fmaf(logit, (float)(1.0 / T), g); the selected id is
 * the argmax of the keys under (key descending, id ascending).  Ids are bitwise deterministic for a given (inputs, seed,
 * temperature, batch order).  With "logprobs" the record holds the model's own log-probability of the sampled id.
 * temperature > 0 with top_logprobs >= 1 is refused with ASRB_ERR_INVALID by asrb_prefill, asrb_transcribe_ids and
 * asrb_transcribe_ingested, before any work.
 * "beam_size" = "1".."6" (default "1": greedy, exactly the code above) and "length_penalty" = "none" (default) or a
 * decimal in [0, 10]; both latched at the prefill.  With beam_size = K > 1 every utterance runs this beam search
 * (Whisper's BeamSearchDecoder with patience 1, exact and deterministic):
 *   1. candidates: each alive beam contributes the first K + 2 entries of its step's top-8 record (logit descending, id
 *      ascending; two EOS ids exist, so at least K are not EOS), with sum = sum_parent + lp, one fp32 add;
 *   2. walk: all candidates of the utterance in (sum descending, parent rank ascending, position in the record
 *      ascending) order; an EOS candidate joins the newly finished, any other becomes the next alive beam (its rank is
 *      the count so far); stop at K alive beams; then admit the newly finished in walk order while the utterance has
 *      fewer than K finished hypotheses;
 *   3. token 0: the walk runs on the prefill's single record;
 *   4. slots: utterance b uses K slots, beam j in slot j * batch + b; a beam's best-ranked child keeps its parent's slot,
 *      the other children take, in rank order, the slots of childless beams in ascending slot order;
 *   5. a slot handed to a child of another slot gets only the KV cache positions after the last common ancestor of its
 *      old and new lineage (the earlier ones are bitwise equal already);
 *   6. an utterance is done at K finished hypotheses; at max_new_tokens its alive beams, in rank order, fill the list up
 *      to K as "no EOS";
 *   7. score = sum / P(n), n = ids (EOS excluded), the sum including the EOS log-probability; P(n) = max(n, 1) with
 *      "none", else ((5 + n) / 6) ** length_penalty, in double; ranked by (score descending, admission order).
 * Rank 0 of each utterance is the result: ids_out / lens_out, asrb_session_device_ids ([batch] rows) and, with
 * "logprobs", asrb_last_logprobs (its per-token values and its EOS value).  Read all K with asrb_last_nbest.
 * Refused with ASRB_ERR_INVALID before any work: beam_size > 1 with temperature > 0, with top_logprobs >= 1, or with
 * batch * beam_size > max_batch; asrb_decode_step in a beam run.  A beam run takes one asrb_generate per prefill (its
 * end writes the result rows, which are also beam 0's slots); a second one returns ASRB_ERR_STATE.
 * "no_repeat_ngram_size" = "0" (default: off) or N in "1".."16", and "repetition_penalty" = "1" (default: off) or a
 * decimal in [1, 10], parsed in double and converted once to the fp32 theta; both latched at the prefill and applied to
 * the whole run, on every decode path.  For sequence b at step n the history is ids[b][0 .. n), the ids this run
 * generated for it: never the prompt, context, audio pad or forced-language ids, and never EOS.  Before any use of the
 * step's logits every path replaces each logit l_v by l'_v:
 *   1. penalty: v in the history: l'_v = l_v < 0 ? l_v * theta : l_v / theta (IEEE fp32 multiply and round-to-nearest
 *      divide, the rule of HF's RepetitionPenaltyLogitsProcessor); otherwise l'_v = l_v;
 *   2. ban: N >= 1 and some i in [0, n - N] with ids[i .. i+N-2] == ids[n-N+1 .. n-1]: l'_{ids[i+N-1]} = -inf (HF's
 *      NoRepeatNGramLogitsProcessor restricted to the history; N = 1 bans every id already generated).
 * Every use then sees l': the greedy argmax, the sampling keys fmaf(l', 1 / T, g), "logprobs" (log-probabilities under
 * softmax(l')), the top-8 records, the beam candidates and their sums, and the logits asrb_decode_step returns.  Token 0
 * has an empty history (l' = l).  A banned id is never selected: the vocabulary keeps more than 8 finite logits.  With
 * both at their defaults the ids, records and kernels are exactly those above.  An invalid value is refused with
 * ASRB_ERR_INVALID and the previous value is kept. */
ASRB_API int asrb_session_set_option(asrb_session* s, const char* key, const char* value);

/* Per-token log-probabilities of the last run (asrb_generate / asrb_transcribe_ids / asrb_transcribe_ingested, or
 * asrb_prefill + asrb_decode_step), recorded when the option "logprobs" was "1" for its prefill and every step:
 *   logprobs_out      [batch][max_new_tokens]: log p(ids[b][i]) = logit - logsumexp(logits) under the fp32 logits
 *                     that selected the token (<= 0); NaN at and beyond lens_out[b]
 *   eos_logprob_out   [batch] or NULL: the same for the EOS token that ended sequence b, NaN if it stopped at
 *                     max_new_tokens
 * Returns ASRB_ERR_STATE when the last run did not record them (option off, or switched after the prefill). */
ASRB_API int asrb_last_logprobs(asrb_session* s, int max_new_tokens, float* logprobs_out, float* eos_logprob_out);

/* Top-k alternatives of the last run, recorded when the option "top_logprobs" was k_rec >= 1 for its prefill and every
 * step.  Candidates are the best logits of the step under (logit descending, id ascending), the order the greedy argmax
 * uses; candidate j's value is its log-probability under the same fp32 logits: (l_j - max) + lp_0, where lp_0 is the
 * value asrb_last_logprobs reports for the selected token.
 *   ids_out / logprobs_out          [batch][max_new_tokens][k]: candidates of the step that selected ids[b][i], best first
 *                                   (entry 0 = ids[b][i]); -1 / NaN at and beyond lens_out[b]
 *   eos_ids_out / eos_logprobs_out  [batch][k] or NULL: the same for the step that selected the EOS ending sequence b
 *                                   (entry 0 = that EOS id); -1 / NaN if it stopped at max_new_tokens
 * ASRB_ERR_STATE when the last run did not record them; ASRB_ERR_INVALID when k < 1 or k > k_rec. */
ASRB_API int asrb_last_top_logprobs(asrb_session* s, int max_new_tokens, int k, int32_t* ids_out, float* logprobs_out,
                                    int32_t* eos_ids_out, float* eos_logprobs_out);

/* The k (1..beam_size) best hypotheses of each utterance of the last beam run, ranked (entry 0 = the result):
 *   ids_out          [batch][k][max_new_tokens], -1 at and beyond the length
 *   lens_out         [batch][k] ids (EOS excluded)
 *   sum_logprob_out  [batch][k] or NULL: the fp32 running sum of the ids' log-probabilities and the EOS one
 *   score_out        [batch][k] or NULL: sum / P(n) (option "length_penalty")
 *   eos_id_out       [batch][k] or NULL: the EOS id that ended it, -1 when stopped by max_new_tokens
 * ASRB_ERR_STATE if the last run was not a beam run; ASRB_ERR_INVALID when k is outside [1, beam_size]. */
ASRB_API int asrb_last_nbest(asrb_session* s, int max_new_tokens, int k, int32_t* ids_out, int32_t* lens_out,
                             float* sum_logprob_out, float* score_out, int32_t* eos_id_out);
/* Counters of the last beam run: [0] beam steps  [1] slots reassigned  [2] KV bytes copied by the prompt expansion
 * [3] KV bytes copied by reorders; writes min(n, 4) values.  ASRB_ERR_STATE if the last run was not a beam run. */
ASRB_API int asrb_last_beam_stats(asrb_session* s, int64_t* out, int n);

/* Context biasing: ids placed as the content of the prompt's system turn (a keyword list, names, related text; the
 * model's own `context`).  Utterance b with context ids c_b (length L_b >= 0) gets the prompt
 *   [151644, 8948, 198] + c_b + [151645, 198, 151644, 872, 198, 151669] + audio pads + tail + language ids
 * at positions 0..S_b-1, S_b = 15 + L_b + audio tokens + language ids; with L_b = 0 it is the prompt without context.
 *   n_rows = 0          clears the contexts
 *   n_rows = 1          ids[0] (n_ids[0] of them) applies to every utterance of later runs
 *   any other n_rows    one context per utterance; a NULL row or n_ids[b] = 0 means no context for utterance b
 * The ids are copied and kept until the next call; like the options, they are latched at the prefill.
 * ASRB_ERR_INVALID here, with the previous contexts kept: an id outside [0, vocab), or a row longer than the session's
 * max_context_ids (so any context on a session made by asrb_session_create).  ASRB_ERR_INVALID from asrb_prefill,
 * asrb_transcribe_ids and asrb_transcribe_ingested, before any work or state change: a batch that is neither n_rows
 * nor covered by n_rows = 1.
 * Shared contexts: utterances of one call whose contexts are identical and non-empty have the same first P = L + 9
 * prompt ids at the same positions, hence the same K/V.  The lowest-indexed one (the leader) computes those rows and
 * writes their K/V into the others' caches; the others compute their rows from position P on.  Utterances without a
 * context never share.  asrb_prefill's seq_lens_out stays S_b, context included.  A context lengthens every
 * sequence's KV: a run that crosses the fused decode step's key limit continues on the per-phase kernels, counted in
 * asrb_session_stats [2]. */
ASRB_API int asrb_session_set_context(asrb_session* s, int n_rows, const int64_t* const* ids, const int32_t* n_ids);
/* Counters of the last prefill: [0] prompt rows computed  [1] prompt rows taken from a leader instead of computed
 * [2] KV bytes fanned out to followers; writes min(n, 3) values. */
ASRB_API int asrb_last_prefill_stats(asrb_session* s, int64_t* out, int n);

/* Teacher-forced scoring of caller-given continuations.  Utterance b (prompt S_b ids exactly as asrb_transcribe_ids
 * builds it: context and lang_ids included) has n_cand[b] >= 1 candidates; candidate c (flattened over utterances in
 * order) is cand_len[c] ids cand_ids[c][0..len).  Id i of candidate c sits at position S_b + i.
 *   logprob_out  [n_total][max_new_tokens]  log p(ids[i] | prompt, ids[0..i)) = l - logsumexp(l) under the model's raw fp32
 *                                          logits; NaN at and beyond cand_len[c]
 *   top_ids_out / top_lp_out  [n_total][max_new_tokens][k] or NULL: with option "top_logprobs" = k >= 1, the k best ids
 *                                          of that position under (logit descending, id ascending) and their
 *                                          log-probabilities; -1 / NaN beyond the length
 * Independent of the decode options: temperature, seed, beam_size, length_penalty, no_repeat_ngram_size and
 * repetition_penalty are not consulted, and the results are bitwise equal whatever they are set to.  Bitwise
 * deterministic for a given call.  Each candidate takes one KV slot; the first candidate of an utterance computes its
 * prompt, the others take the prompt's K/V from it (asrb_last_prefill_stats: rows computed = sum_b S_b +
 * sum_c (len_c - 1), rows shared = sum_b (n_cand[b] - 1) * S_b, KV bytes fanned out = rows shared x the K/V bytes of one
 * position).  asrb_last_timings: [3] the decoder layers of the prefill, [4] the score head, [5] the whole call.
 * ASRB_ERR_INVALID before any work: n_total = sum n_cand > max_batch, n_cand[b] < 1, cand_len[c] outside
 * [1, max_new_tokens], an id outside [0, vocab), a hidden size the wgmma score head cannot take (not a multiple of 64),
 * plus everything asrb_transcribe_ids refuses.  A scoring call ends any pending run: asrb_generate / asrb_decode_step /
 * asrb_last_logprobs / _top_logprobs / _nbest return ASRB_ERR_STATE until the next prefill. */
ASRB_API int asrb_score_ids(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                            const int32_t* n_cand, const int64_t* const* cand_ids, const int32_t* cand_len,
                            int max_new_tokens, float* logprob_out, int32_t* top_ids_out, float* top_lp_out);
/* the same on the utterances of the last asrb_ingest_pcm */
ASRB_API int asrb_score_ingested(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                                 const int32_t* n_cand, const int64_t* const* cand_ids, const int32_t* cand_len,
                                 int max_new_tokens, float* logprob_out, int32_t* top_ids_out, float* top_lp_out);

/* ---- word timestamps: alignment from the decoder's audio attention (DESIGN.md 4.10) ----
 * Utterance b has its prompt of S_b ids exactly as asrb_transcribe_ids builds it (context and lang_ids included), its
 * T_b audio tokens at positions a_b .. a_b + T_b - 1 with a_b = 9 + L_b (L_b = its context length), caller-given ids
 * x_0 .. x_{n_b - 1} = ids[b][0 .. n_ids[b]) (normally the decoded ids followed by EOS 151645), and f_b = text_from[b]:
 * the ids before f_b (for example "language English<asr_text>") are context and are not aligned.
 *   Rows: row i, f_b <= i < n_b, is the query at position S_b - 1 + i, the row that predicts x_i in one causal forward
 *     over prompt + ids; N_b = n_b - f_b rows.
 *   Heads: heads[k] = {layer, query head}, n_heads pairs; n_heads = 0 means every query head of the layers
 *     num_hidden_layers / 2 .. num_hidden_layers - 1.  Query head h reads kv head h / (nq / nkv).
 *   Weights: per head and row, P[i][j] = softmax_j(q_i . k_j / sqrt(head_dim)) over the audio keys only, 0 <= j < T_b,
 *     in fp32.
 *   Normalise: per head and column j, z[i][j] = (P[i][j] - mean) / std over the N_b rows, std the population std;
 *     z = 0 where std = 0.
 *   Filter: per head and row, the median of width 7 along j with mirror padding (x[-1] = x[1]); none when T_b <= 3.
 *   Head mean: M[i][j] = the sum over the heads in (layer, head) ascending order, divided by their count.
 *   DTW on X = -M: C is (N + 1) x (T + 1) fp32, C[0][0] = 0 and the rest of row 0 and column 0 +inf;
 *     C[i][j] = X[i-1][j-1] + c, where the step is diagonal (c = C[i-1][j-1]) when C[i-1][j-1] is less than both other
 *     predecessors, else up (c = C[i-1][j]) when C[i-1][j] is less than both, else left (c = C[i][j-1]).  The path is
 *     traced back from (N, T) to (0, 0); start_tok[i] = the least j on the path in row i.
 *   Frames (10 ms each): audio token j, at in-chunk index t of encoder chunk k, starts at frame k * 2 * n_window + 8 t.
 *     start_frame_out[b][i] = the frame of start_tok of row i, end_frame_out[b][i] = the next row's start frame, the
 *     last row's = F_b, the utterance's mel frame count.  Both are [batch][max_ids] by id position; -1 outside
 *     [f_b, n_b).
 * Bitwise deterministic for a given call, and independent of the decode options (temperature, seed, beam_size,
 * length_penalty and the repetition controls are not consulted).  The context of asrb_session_set_context applies,
 * latched as in scoring.  An alignment call ends any pending run, as a scoring call does.  asrb_last_timings: [3] the
 * decoder layers up to the last listed one with the probability and fold kernels, [4] the DTW, [5] the whole call.
 * ASRB_ERR_INVALID before any work, the session as it was: batch outside [1, max_batch], n_ids[b] < 1 or greater than
 * max_ids or the session's max_new_tokens, an id outside [0, vocab), text_from[b] outside [0, n_ids[b] - 1], a head
 * outside the model or listed twice, plus everything asrb_transcribe_ids refuses (language ids, context rows). */
ASRB_API int asrb_align_ids(asrb_session* s, const float* const* samples, const int64_t* n_samples, int batch,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                            const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids,
                            int32_t* start_frame_out, int32_t* end_frame_out);
/* the same on the utterances of the last asrb_ingest_pcm */
ASRB_API int asrb_align_ingested(asrb_session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                                 const int64_t* const* ids, const int32_t* n_ids, const int32_t* text_from,
                                 const int32_t* heads, int n_heads, int max_ids, int32_t* start_frame_out,
                                 int32_t* end_frame_out);
/* the same on n views [start, end) of the long-audio files, read in place and checked as asrb_transcribe_segments
 * reads and checks them; frames count from each view's start */
ASRB_API int asrb_align_segments(asrb_session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                                 const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                                 const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads,
                                 int max_ids, int32_t* start_frame_out, int32_t* end_frame_out);
/* N_b (rows) and T_b (audio tokens) of utterance b of the last alignment call (either pointer may be NULL), and its
 * M [N_b][T_b]; ASRB_ERR_STATE when that call had no utterance b */
ASRB_API int asrb_last_align_dims(asrb_session* s, int b, int32_t* n_rows_out, int32_t* n_tokens_out);
ASRB_API int asrb_align_matrix_read(asrb_session* s, int b, float* out);

/* ---- streaming transcription (DESIGN.md 4.9) ----
 * A streaming run uses an ordinary session (asrb_session_create_ex).  Stream b lives in KV slot b,
 * 0 <= b < n_streams <= max_batch.  It owns its 16 kHz f32 samples x[0..n), its forced prefix p (ids, empty at the
 * start) and a push counter k.  Push k on stream b with new samples, and optionally `final`:
 *   1. appends the samples; n may not exceed max_samples;
 *   2. computes the hypothesis h = p + g, where g is the greedy (or sampled, per the session options) continuation of
 *      the prompt asrb_transcribe_ids builds for x[0..n) with lang_ids = the push's language ids + p.  The context of
 *      asrb_session_set_context is latched when the stream starts (asrb_stream_open / asrb_stream_reset).  g stops at
 *      EOS or at the push's max_new_tokens;
 *   3. sets the next prefix p' = h[0 .. max(0, |h| - R)) when k + 1 >= U, else empty; R = rollback_ids (default 5),
 *      U = unfixed_pushes (default 2).  |p'| is returned as the hypothesis' fixed length;
 *   4. on a final push every frame counts as final and there is no rollback (p' = h); the stream is then closed and a
 *      later push on it returns ASRB_ERR_STATE until asrb_stream_reset.
 * A stream that gets no samples (and is not final) in a push is idle: it is not prefilled or decoded and its
 * hypothesis is unchanged.  k counts the pushes that gave the stream samples.
 * Equivalence: the stream's mel after any push is bitwise asrb_mel(x[0..n)); its encoder output, prefill and decode
 * records follow the project's float64 rule against the oracle on x[0..n) with the same prompt; its g equals
 * asrb_transcribe_ids(x[0..n), lang + p) on clips whose decisions have a margin; for a given push schedule, samples and
 * options the results are bitwise reproducible.  They are NOT promised bitwise equal to an offline call: windows and K/V
 * reused from earlier pushes were computed under other GEMM shapes (split-K choice).
 * Reuse: a finished encoder window (all frames final: frame f is final once 160 f + 200 <= n) is not encoded again when
 * its clamped mel cannot have changed; the decoder keeps the K/V of positions < P_b = 9 + L_b + (tokens of the windows
 * before the first re-encoded one), and P_b = 0 on a stream's first push after open / reset.
 * Any non-stream call that starts a run (asrb_transcribe*, asrb_score*, asrb_mel, asrb_prefill) or asrb_stream_open
 * ends all streams: asrb_stream_push then returns ASRB_ERR_STATE.
 * Refused with ASRB_ERR_INVALID before any work, leaving all stream state intact: beam_size > 1 (streams own their
 * slots), n_streams > max_batch, samples past max_samples, |lang| + |p| > max_lang_ids, a stream's first push with
 * <= 160 samples, max_ids < |p| + max_new_tokens, and the option conflicts asrb_transcribe_ids refuses. */
ASRB_API int asrb_stream_open(asrb_session* s, int n_streams, int rollback_ids, int unfixed_pushes);
/* stream b back to its start (no samples, empty prefix, k = 0, open), the context re-latched */
ASRB_API int asrb_stream_reset(asrb_session* s, int stream);
/* one push on all n_streams streams (n_streams as opened):
 *   samples[b] / n_samples[b]  new samples of stream b (n_samples[b] = 0: none)
 *   is_final[b]                NULL or nonzero: stream b's last push
 *   lang_ids[b] / n_lang_ids   as asrb_transcribe_ids
 *   hyp_out [n_streams][max_ids], hyp_len_out / fixed_len_out [n_streams]: every stream's hypothesis after the push
 * asrb_last_logprobs / _top_logprobs / asrb_last_timings / asrb_session_stats describe the push's run, one row per
 * stream (idle streams: no ids). */
ASRB_API int asrb_stream_push(asrb_session* s, int n_streams, const float* const* samples, const int64_t* n_samples,
                              const int32_t* is_final, const int64_t* const* lang_ids, const int32_t* n_lang_ids,
                              int max_new_tokens, int max_ids, int32_t* hyp_out, int32_t* hyp_len_out,
                              int32_t* fixed_len_out);
/* stream b's mel [128][F] (F = ceil(n / 160)) and encoder output [T][output_dim] after its last push */
ASRB_API int asrb_stream_mel_read(asrb_session* s, int stream, float* out);
ASRB_API int asrb_stream_encode_read(asrb_session* s, int stream, float* out);
/* counters of the last push, summed over its streams: [0] windows encoded  [1] windows reused  [2] windows re-encoded
 * because the mel floor moved  [3] prompt rows computed  [4] prompt rows kept from earlier pushes */
ASRB_API int asrb_last_stream_stats(asrb_session* s, int64_t* out, int n);

/* debug (ASRB_MEGA_DEBUG=1): clock64 timeline of the last fused decode step, CTA 0 then CTA G-1;
 * returns the number of slots per CTA (0 if disabled) */
ASRB_API int asrb_debug_mega_timeline(long long* out, int cap);

#ifdef __cplusplus
}
#endif
#endif /* ASR_B200_H */
