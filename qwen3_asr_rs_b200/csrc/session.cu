// session.cu -- host driver: restates AsrInference::transcribe steps 2-8
// (/root/reference/src/inference.rs:94-200) for a BATCH of independent utterances on one GPU.
// Control flow (prompt layout, position ids, greedy loop, EOS) is the reference's; all arithmetic
// is in the kernels.  Everything is varlen: rows of all utterances are concatenated and described
// by small index arrays uploaded once per call.
#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include "internal.h"

namespace asrb {

void model_set_tensor(Model* m, const char* name, int dtype, const int64_t* shape, int ndim, const void* host);
void model_finalize(Model* m);
struct IngestState;
IngestState* ingest_state_new();
void ingest_state_free(IngestState* st);
void ingest_pcm(IngestState* st, cudaStream_t stream, const void* const* pcm, const int64_t* n_frames, const int32_t* channels,
                const int32_t* rate, const int32_t* format, int batch, float* d_samples, int64_t max_samples_per_utt,
                int64_t* n_out, int64_t* soff_out);

// token ids of the fixed prompt (inference.rs:215-257) and special tokens (tokenizer.rs:53-59)
static const int kPromptHead[9] = {151644, 8948, 198, 151645, 198, 151644, 872, 198, 151669};
static const int kPromptTail[6] = {151670, 151645, 198, 151644, 77091, 198};
static const int kAudioPad = 151676;
// the prompt's layout (build_prompt): 3 head ids, the context, 6 more head ids, the audio pads, the tail, the language
// ids, the forced ids
static int audio_start(int ctx) { return 3 + ctx + 6; }
static int prompt_len(int ctx, int T, int nl, int nforced) { return audio_start(ctx) + T + 6 + nl + nforced; }
// audio tokens of a chunk of `frames` mel frames: three stride-2 convolutions (feat_extract_output_length)
static int chunk_tokens(int frames) { return conv_out_len(conv_out_len(conv_out_len(frames))); }

struct Session {
    Model* m = nullptr;
    cudaStream_t st = nullptr;
    int max_batch = 0, max_lang = 0, max_new = 0, max_context = 0;
    int64_t max_samples = 0, max_npad = 0;
    int maxF = 0, maxC = 0, maxT = 0, maxS = 0, max_ctx = 0;
    int gemm_impl = GEMM_TC;
    int decode_mode = 1;   // 1 = fused step when available, 0 = per-phase kernels
    bool batch_step = true;   // batch >= 2: the batch-aware fused step (decode_batch.cu); false = one fused launch per sequence
    int64_t n_batch_steps = 0, n_mega_steps = 0, n_phase_steps = 0;   // decoder forwards by path since session creation
    int nplanes = 3;
    // ---- current batch plan (host) ----
    int stage = 0;         // 0 idle, 1 mel, 2 encoded, 3 prefilled
    int B = 0;
    std::vector<int64_t> n, npad, F, foff, soff;
    std::vector<int> C, T, toff, S;
    int totF = 0, totC = 0, totT = 0, maxlenS = 0, maxwin = 0, nwin = 0;
    // ---- buffers: device (cudaMalloc) and pinned host (cudaMallocHost) memory, freed with the session ----
    std::vector<void*> owned, owned_host;
    float *h_samples = nullptr, *d_samples = nullptr, *d_mel = nullptr;
    int64_t* d_i64 = nullptr;      // soff | n | npad | foff | frames  (5 * max_batch)
    int64_t* h_i64 = nullptr;
    int *d_int = nullptr, *h_int = nullptr; size_t int_cap = 0, enc_int_cap = 0;   // [encoder plan | prefill plan]
    int* d_maxkey = nullptr;
    bf16 *act1 = nullptr, *act2 = nullptr, *feat = nullptr; size_t act1_ps = 0, act2_ps = 0, feat_ps = 0;
    float *x_enc = nullptr, *enc_qkv = nullptr, *audio = nullptr;
    bf16 *enc_h = nullptr, *enc_attn = nullptr, *enc_ff = nullptr; size_t ench_ps = 0, encff_ps = 0;
    float *hid = nullptr, *dqkv = nullptr, *qrot = nullptr;
    bf16 *dh = nullptr, *dattn = nullptr, *dact = nullptr; size_t dh_ps = 0, dattn_ps = 0, dact_ps = 0;
    float *kcache = nullptr, *vcache = nullptr; size_t cache_layer_stride = 0, cache_seq_stride = 0;
    DecodeBufs db{};
    float* splitk_ws = nullptr;   // fp32 partial tiles of split-K GEMMs (gemm_tc.cu)
    MegaBufs mega{};
    int sx_nb = 0;             // NB instantiation the exchange words were last armed for (decode_batch.cu)
    unsigned mega_steps = 1;   // host mirror of the device epoch (upper bound): see launch_decode_step_mega
    int* d_lastrow = nullptr;
    int *h_done = nullptr, *h_ids = nullptr, *h_nout = nullptr, *h_next = nullptr;
    // int-plan offsets (into d_int)
    int *d_chunk_clip = nullptr, *d_chunk_f0 = nullptr, *d_rowmap = nullptr, *d_win_q0 = nullptr, *d_win_len = nullptr;
    int *d_ids = nullptr, *d_audio_row = nullptr, *d_row_seq = nullptr, *d_row_pos = nullptr, *d_seq_q0 = nullptr, *d_seq_len = nullptr;
    // decode graph
    cudaGraphExec_t step_graph = nullptr; int graph_B = 0; int graph_mode = -1;
    // stats
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    float last_ms[6] = {0, 0, 0, 0, 0, 0};
    bool resident = false, timing = false;
    IngestState* ingest = nullptr;      // GPU-side audio ingest (ingest.cu)
    std::vector<int64_t> ingested_n;    // 16 kHz samples per utterance produced by the last asrb_ingest_pcm (empty: none pending)
    int64_t launches = 0, decode_steps = 0;
    int greedy_done = 0;   // greedy applications since prefill (tokens appended or EOS), bounds max_new
    // per-token log-probabilities: option "logprobs" (db.logprobs selects the kernel variants); lp_valid = the prefill
    // and every step since ran with it on, i.e. db.lp_out / db.eos_lp describe the current run
    bool lp_valid = false;
    // top-k alternatives: option "top_logprobs" (top_k >= 1 sets db.topk and db.logprobs); tk_valid = the k the prefill
    // and every step since ran with (0: none), i.e. db.tk_* describe the current run for k <= tk_valid
    bool opt_logprobs = false; int top_k = 0, tk_valid = 0;
    // seeded temperature sampling: options "temperature" (0 = greedy) and "seed", latched at the prefill into db.sample
    // and the device-resident db.smp, so they apply to the whole run
    double temperature = 0.0; uint64_t seed = 0;
    SampleParams* d_smp = nullptr;
    // repetition controls: options "no_repeat_ngram_size" (0 = off) and "repetition_penalty" (1 = off), latched at the
    // prefill into db.rep and the device-resident db.rep_params, so they apply to the whole run
    int ngram = 0; double rep_penalty = 1.0;
    RepParams* d_rep = nullptr;
    // beam search: options "beam_size" (1 = greedy) and "length_penalty" (< 0: none), latched at the prefill into run_k /
    // run_alpha.  A beam run decodes nslots = B * run_k slots; B stays the number of utterances.
    int beam_k = 1, run_k = 1, nslots = 0;
    double length_penalty = -1.0, run_alpha = -1.0;
    BeamArgs beam{};                    // device buffers (allocated on the first beam run) and the run's geometry
    int* d_hyp = nullptr; float* d_best_eos = nullptr;   // finalize input: ranked (depth, slot) per hypothesis, rank 0's EOS lp
    bool nbest_valid = false;           // the last run was a beam run and has been finalized
    std::vector<float> nb_sum; std::vector<double> nb_score; std::vector<int> nb_eos, nb_n;   // [B][run_k], ranked
    int64_t beam_steps = 0, beam_reassigned = 0, beam_expand_bytes = 0, beam_reorder_bytes = 0;
    // context biasing (asrb_session_set_context): ids placed in the system turn, latched at the prefill.  ctx_rows = 0:
    // none; 1: ctx[0] for every utterance; else one row per utterance (empty: no context)
    int ctx_rows = 0;
    std::vector<std::vector<int>> ctx;
    int64_t pf_rows = 0, pf_shared_rows = 0, pf_fan_bytes = 0;   // last prefill: rows computed / taken from a leader, KV bytes fanned out
    // long-form audio (asrb_ingest_long): file f holds long_n[f] samples at d_long + long_off[f], zero padded to a
    // multiple of 160; not bounded by max_samples, grown on demand.  Segment views of it are decoded in place.
    float* d_long = nullptr; size_t long_cap = 0;
    std::vector<int64_t> long_n, long_off;
    double* d_seg_blk = nullptr; size_t seg_blk_cap = 0;      // asrb_segment_long scratch: 160-sample block energies
    int64_t* d_seg_i64 = nullptr; size_t seg_i64_cap = 0;     // ... its plan, cut counts and cuts
    size_t act_rows = 0;                // rows the decoder activations hold (hid, dqkv, qrot, dh, dattn, dact)
    // teacher-forced scoring (asrb_score_ids): allocated, and grown, by the scoring calls that need them; a scoring call
    // whose prefill has more rows than act_rows (the candidates' own rows beside the prompts) widens the activations
    struct ScoreBufs {
        int rows_cap = 0;                       // score rows the head's scratch holds
        float* gathered = nullptr; bf16* planes = nullptr; ScorePart* part = nullptr;
        float* lp = nullptr; int* tk_ids = nullptr; float* tk_lp = nullptr;
        int* h_int = nullptr; int* d_int = nullptr; size_t int_cap = 0;   // row plan | per-slot arrays | score rows
    } sc;
    // word-timing alignment (asrb_align_ids, DESIGN.md 4.10): scratch allocated, and grown, all or none by the alignment
    // calls; the last call's M and dims stay readable (asrb_align_matrix_read / asrb_last_align_dims) until the next one
    struct AlignBufs {
        size_t p_cap = 0, m_cap = 0, trace_cap = 0, start_cap = 0;   // floats / floats / words / ints
        float *P = nullptr, *M = nullptr; uint32_t* trace = nullptr; int* start = nullptr;
        std::vector<int> N, T; std::vector<long long> moff;   // of the last alignment call (empty: none)
    } al;
    // streaming (asrb_stream_*, DESIGN.md 4.9): stream b lives in KV slot b; its buffers are allocated by the first open
    struct Stream {
        int64_t n = 0;                  // samples received, in str_samples row b
        int k = 0;                      // pushes that gave it samples
        bool closed = false;            // its final push is done
        std::vector<int> p, hyp, ctx;   // forced prefix, last hypothesis, context latched when the stream started
        int fixed = 0;                  // fixed length of hyp (= |p|)
        int Ffin = 0;                   // final mel frames, folded into stats row b
        float phi = 0.f;                // mel floor of the last push
        int T = 0;                      // audio tokens in token-store row b
        int kv_valid = 0;               // prompt positions whose K/V in slot b are those of the stream's current audio
        std::vector<float> win_phi;     // per encoder window: the floor it was last encoded under
        std::vector<char> win_final;    //   and whether all its frames were final then
    };
    std::vector<Stream> streams;
    bool streams_open = false;
    bool stream_run = false;            // the last run was a push: the stage-level reads describe no offline batch
    int str_rollback = 5, str_unfixed = 2, str_maxW = 0, str_stats_ld = 0;
    float* str_samples = nullptr;       // [max_batch][max_npad] 16 kHz samples
    float* str_raw = nullptr;           // [max_batch][n_mels][maxF] raw (pre-floor) log-mel
    float* str_tok = nullptr;           // [max_batch][maxT][output_dim] encoder output
    float* str_stats = nullptr;         // [max_batch][2 + maxW] fold results (mel_stream_fold_kernel)
    float* h_str_stats = nullptr;
    int *str_int = nullptr, *h_str_int = nullptr; size_t str_int_cap = 0;   // fold plan | first frames | staging plan
    int64_t str_counts[5] = {0, 0, 0, 0, 0};   // last push: windows encoded / reused / re-encoded for the floor, rows computed / kept
    ~Session();
};

Session::~Session() {
    if (step_graph) cudaGraphExecDestroy(step_graph);
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    for (void* p : owned) cudaFree(p);
    for (void* p : owned_host) cudaFreeHost(p);
    if (ingest) ingest_state_free(ingest);
    if (st) cudaStreamDestroy(st);
}

template <typename T> static T* salloc(Session* s, size_t n, bool zero = false) {
    T* p = nullptr;
    ASRB_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
    s->owned.push_back(p);
    if (zero) ASRB_CUDA_CHECK(cudaMemset(p, 0, std::max<size_t>(n, 1) * sizeof(T)));
    return p;
}
template <typename T> static T* halloc(Session* s, size_t n) {     // pinned host memory
    T* p = nullptr;
    ASRB_CUDA_CHECK(cudaMallocHost(&p, std::max<size_t>(n, 1) * sizeof(T)));
    s->owned_host.push_back(p);
    return p;
}
// frees a buffer of the session's (device or pinned host); null or not the session's: nothing
static void release_owned(Session* s, void* p) {
    for (auto* list : {&s->owned, &s->owned_host}) {
        auto it = std::find(list->begin(), list->end(), p);
        if (it == list->end()) continue;
        if (list == &s->owned) cudaFree(p); else cudaFreeHost(p);
        list->erase(it);
        return;
    }
}

Session* session_create(Model* m, int max_batch, int64_t max_samples, int max_lang, int max_context, int max_new) {
    ASRB_REQUIRE(m && m->finalized, ASRB_ERR_STATE, "model not finalized");
    ASRB_REQUIRE(max_batch >= 1 && max_samples > 200 && max_new >= 1 && max_lang >= 0 && max_context >= 0, ASRB_ERR_INVALID,
                 "bad session capacity");
    ASRB_CUDA_CHECK(cudaSetDevice(m->ctx->device));
    Session* s = new Session();
    try {
        const Dims& d = m->d; const asrb_dims& c = d.c;
        if (const char* e = getenv("ASRB_GEMM")) s->gemm_impl = (std::string(e) == "simt") ? GEMM_SIMT : GEMM_TC;     // debug overrides
        if (const char* e = getenv("ASRB_DECODE")) s->decode_mode = (std::string(e) == "phases") ? 0 : 1;
        if (const char* e = getenv("ASRB_PLANES")) s->nplanes = std::min(3, std::max(1, atoi(e)));
        s->m = m; s->max_batch = max_batch; s->max_samples = max_samples; s->max_lang = max_lang; s->max_new = max_new;
        s->max_context = max_context;
        s->max_npad = ((max_samples + 159) / 160) * 160;
        s->maxF = (int)(s->max_npad / 160);
        s->maxC = (s->maxF + d.chunk_frames - 1) / d.chunk_frames;
        s->maxT = s->maxC * d.tok_per_chunk;
        s->maxS = prompt_len(max_context, s->maxT, max_lang, 0);
        s->max_ctx = s->maxS + max_new;
        ASRB_REQUIRE(s->max_ctx <= m->rope_max_pos, ASRB_ERR_INVALID, "context exceeds RoPE table");
        // the per-phase decode step (asrb_decode_step with logits, any model or context the fused steps decline) holds a
        // score per (query head of a GQA group, key) in shared memory: refuse here what its launch would refuse mid-decode
        ASRB_REQUIRE(dec_attn_smem_bytes(*m, s->max_ctx) <= m->ctx->smem_optin, ASRB_ERR_INVALID,
                     "session context of " + std::to_string(s->max_ctx) + " positions (audio tokens + prompt + max_new_tokens) with GQA group " +
                         std::to_string(c.num_attention_heads / c.num_key_value_heads) + " needs " +
                         std::to_string(dec_attn_smem_bytes(*m, s->max_ctx)) + " bytes of shared memory for decode attention, the device offers " +
                         std::to_string(m->ctx->smem_optin) + ": lower max_samples or max_new_tokens");
        ASRB_CUDA_CHECK(cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking));
        for (auto& e : s->ev) ASRB_CUDA_CHECK(cudaEventCreate(&e));
        const size_t Bm = max_batch;
        s->h_samples = halloc<float>(s, Bm * s->max_npad);
        s->d_samples = salloc<float>(s, Bm * s->max_npad);
        s->d_mel = salloc<float>(s, Bm * c.num_mel_bins * s->maxF);
        s->h_i64 = halloc<int64_t>(s, 5 * Bm);
        s->d_i64 = salloc<int64_t>(s, 5 * Bm);
        s->d_maxkey = salloc<int>(s, Bm);
        const size_t totC = Bm * s->maxC, totT = Bm * s->maxT, totS = Bm * s->maxS;
        s->enc_int_cap = 2 * totC + totC * d.tok_per_chunk + 2 * (totC + Bm) + 16;
        s->int_cap = s->enc_int_cap + 4 * totS + 10 * Bm;   // rows, per-sequence plan and fan-out, lastrow | pos0 | done0
        s->h_int = halloc<int>(s, s->int_cap);
        s->d_int = salloc<int>(s, s->int_cap);
        // encoder activations
        s->act1_ps = totC * 4 * d.conv_h[2] * d.conv_w[2] * d.cpad;
        s->act2_ps = totC * 4 * d.conv_h[3] * d.conv_w[3] * d.cpad;
        s->feat_ps = totC * d.tok_per_chunk * (size_t)d.feat;
        s->act1 = salloc<bf16>(s, 3 * s->act1_ps, true);     // zero: channel padding / odd-parity pad column
        s->act2 = salloc<bf16>(s, 3 * s->act2_ps, true);
        s->feat = salloc<bf16>(s, 3 * s->feat_ps);
        s->x_enc = salloc<float>(s, totT * c.d_model);
        s->enc_qkv = salloc<float>(s, totT * 3 * c.d_model);
        s->audio = salloc<float>(s, totT * c.output_dim);
        s->ench_ps = totT * c.d_model; s->encff_ps = totT * c.encoder_ffn_dim;
        s->enc_h = salloc<bf16>(s, 3 * s->ench_ps);
        s->enc_attn = salloc<bf16>(s, 3 * s->ench_ps);
        s->enc_ff = salloc<bf16>(s, 3 * s->encff_ps);
        s->splitk_ws = salloc<float>(s, SPLITK_WS_FLOATS);
        // decoder activations
        s->hid = salloc<float>(s, totS * c.hidden_size);
        s->dqkv = salloc<float>(s, totS * d.qkv_dim);
        s->qrot = salloc<float>(s, totS * d.q_dim);
        s->dh_ps = totS * c.hidden_size; s->dattn_ps = totS * d.q_dim; s->dact_ps = totS * c.intermediate_size;
        s->act_rows = totS;
        s->dh = salloc<bf16>(s, 3 * s->dh_ps);
        s->dattn = salloc<bf16>(s, 3 * s->dattn_ps);
        s->dact = salloc<bf16>(s, 3 * s->dact_ps);
        s->cache_seq_stride = (size_t)c.num_key_value_heads * s->max_ctx * c.head_dim;
        s->cache_layer_stride = Bm * s->cache_seq_stride;
        s->kcache = salloc<float>(s, c.num_hidden_layers * s->cache_layer_stride);
        s->vcache = salloc<float>(s, c.num_hidden_layers * s->cache_layer_stride);
        // decode state
        DecodeBufs& b = s->db;
        b.x = salloc<float>(s, Bm * c.hidden_size);
        b.qkv = salloc<float>(s, Bm * d.qkv_dim);
        b.attn = salloc<float>(s, Bm * d.q_dim);
        b.act = salloc<float>(s, Bm * c.intermediate_size);
        b.logits = salloc<float>(s, Bm * c.vocab_size);
        b.n_part = m->ctx->sm_count * 2;
        b.part_val = salloc<float>(s, Bm * b.n_part);
        b.part_idx = salloc<int>(s, Bm * b.n_part);
        b.pos = salloc<int>(s, Bm); b.done = salloc<int>(s, Bm); b.next_id = salloc<int>(s, Bm);
        b.ids_out = salloc<int>(s, Bm * max_new); b.n_out = salloc<int>(s, Bm);
        b.max_new = max_new;
        s->d_smp = salloc<SampleParams>(s, 1, true);
        b.smp = s->d_smp;
        s->d_rep = salloc<RepParams>(s, 1, true);
        b.rep_params = s->d_rep; b.rep_words = (c.vocab_size + 31) / 32;   // per-phase bit arrays: the whole vocabulary
        s->d_lastrow = salloc<int>(s, Bm);
        s->mega.bar = salloc<unsigned>(s, 4, true);
        { const unsigned one = 1; ASRB_CUDA_CHECK(cudaMemcpy(s->mega.bar + 1, &one, sizeof(one), cudaMemcpyHostToDevice)); }   // epoch 1
        const size_t part_floats = std::max(decode_mega_part_floats(*m), decode_batch_part_floats(*m));
        s->mega.part = salloc<float>(s, part_floats, true);   // zero = tag 0 = never written
        s->mega.part_bytes = part_floats * sizeof(float);
        s->mega.steps_issued = &s->mega_steps;
        if (max_batch >= 2) {   // batch-aware fused step: self-validating exchange words, all "not written yet" (0xFFFFFFFF)
            s->mega.sx_bytes = decode_batch_sx_bytes(*m);
            s->mega.sx = (uint32_t*)salloc<uint8_t>(s, s->mega.sx_bytes);
            ASRB_CUDA_CHECK(cudaMemset(s->mega.sx, 0xFF, s->mega.sx_bytes));
            s->mega.sx_nb = &s->sx_nb;
            // keep them L2-resident between steps (2-3 GB of weights and KV stream through L2 every step): persisting
            // access window on the session stream; best effort (ignored if the device refuses the set-aside)
            int maxwin = 0, maxpersist = 0;
            cudaDeviceGetAttribute(&maxwin, cudaDevAttrMaxAccessPolicyWindowSize, m->ctx->device);
            cudaDeviceGetAttribute(&maxpersist, cudaDevAttrMaxPersistingL2CacheSize, m->ctx->device);
            if (maxwin > 0 && maxpersist > 0) {
                const size_t want = std::min<size_t>({s->mega.sx_bytes, (size_t)maxwin, (size_t)maxpersist});
                if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) {
                    cudaStreamAttrValue av{};
                    av.accessPolicyWindow.base_ptr = s->mega.sx; av.accessPolicyWindow.num_bytes = want;
                    av.accessPolicyWindow.hitRatio = 1.0f; av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
                    av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
                    if (cudaStreamSetAttribute(s->st, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();
                } else cudaGetLastError();
            }
        }
        {   // single-sequence fused step (batch 1 included): self-validating exchange words, all "not written yet"
            const size_t bytes = decode_mega_sx_bytes(*m);
            s->mega.sx_seq = (uint32_t*)salloc<uint8_t>(s, bytes);
            ASRB_CUDA_CHECK(cudaMemset(s->mega.sx_seq, 0xFF, bytes));
        }
        s->mega.hq_stats = salloc<unsigned long long>(s, 4, true);
        if (getenv("ASRB_MEGA_DEBUG")) s->mega.dbg = salloc<long long>(s, decode_mega_dbg_slots(), true);
        s->h_done = halloc<int>(s, Bm); s->h_nout = halloc<int>(s, Bm); s->h_next = halloc<int>(s, Bm);
        s->h_ids = halloc<int>(s, Bm * max_new);
        ASRB_CUDA_CHECK(cudaDeviceSynchronize());
    } catch (...) { delete s; throw; }
    return s;
}

void session_free(Session* s) { delete s; }

// -------------------------------------------------------------------------------------------------
// step 2: mel  (inference.rs:95)
// -------------------------------------------------------------------------------------------------
// view_off != nullptr: utterance b is the view of n_samples[b] samples at d_long + view_off[b] (asrb_transcribe_segments),
// read in place by the mel kernel, which reads sample j only for j < n
static void mel_impl(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* view_off,
                     int64_t* n_frames_out) {
    ASRB_REQUIRE(batch >= 1 && batch <= s->max_batch, ASRB_ERR_INVALID, "batch exceeds session capacity");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    const bool views = view_off != nullptr;
    const bool ingested = (samples == nullptr) && !views;   // samples already in HBM, written by asrb_ingest_pcm
    if (ingested) ASRB_REQUIRE((int)s->ingested_n.size() == batch, ASRB_ERR_STATE, "no ingested audio for this batch");
    s->B = batch; s->stage = 0;
    s->streams_open = false; s->stream_run = false;     // every call that starts from audio ends the streams
    s->n.assign(batch, 0); s->npad.assign(batch, 0); s->F.assign(batch, 0); s->foff.assign(batch, 0); s->soff.assign(batch, 0);
    int64_t so = 0, fo = 0; int maxF = 0;
    for (int b = 0; b < batch; ++b) {
        int64_t n = ingested ? s->ingested_n[b] : n_samples[b];
        ASRB_REQUIRE((ingested || views || samples[b]) && n > 0 && n <= s->max_samples, ASRB_ERR_INVALID, "n_samples out of session capacity");
        int64_t np = ((n + 159) / 160) * 160;                                       // mel.rs:51
        ASRB_REQUIRE(np > 200, ASRB_ERR_INVALID, "utterance too short for reflect padding (needs > 200 samples)");
        s->n[b] = n; s->npad[b] = np; s->F[b] = np / 160; s->soff[b] = views ? view_off[b] : so; s->foff[b] = fo;
        if (!s->resident && !ingested && !views) {
            memcpy(s->h_samples + so, samples[b], n * sizeof(float));
            if (np > n) memset(s->h_samples + so + n, 0, (np - n) * sizeof(float));
        }
        so += np; fo += np / 160; maxF = std::max<int>(maxF, (int)(np / 160));
    }
    s->totF = (int)fo;
    int64_t* h = s->h_i64; const int Bm = s->max_batch;
    for (int b = 0; b < batch; ++b) { h[b] = s->soff[b]; h[Bm + b] = s->n[b]; h[2 * Bm + b] = s->npad[b]; h[3 * Bm + b] = s->foff[b]; h[4 * Bm + b] = s->F[b]; }
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_i64, h, 5 * Bm * sizeof(int64_t), cudaMemcpyHostToDevice, s->st));
    if (!s->resident && !ingested && !views)
        ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_samples, s->h_samples, so * sizeof(float), cudaMemcpyHostToDevice, s->st));
    if (ingested) s->ingested_n.clear();                 // consumed
    if (s->timing) ASRB_CUDA_CHECK(cudaEventRecord(s->ev[1], s->st));
    launch_mel(*s->m, views ? s->d_long : s->d_samples, s->d_i64, s->d_i64 + Bm, s->d_i64 + 2 * Bm, s->d_i64 + 3 * Bm, batch,
               maxF, s->d_mel, s->d_maxkey, s->st);
    s->launches += 3;
    if (n_frames_out) for (int b = 0; b < batch; ++b) n_frames_out[b] = s->F[b];
    s->stage = 1;
}
void session_mel(Session* s, const float* const* samples, const int64_t* n_samples, int batch, int64_t* n_frames_out) {
    mel_impl(s, samples, n_samples, batch, nullptr, n_frames_out);
}

// step 1 on the GPU (src/audio.rs:162-245): raw interleaved PCM -> mono 16 kHz f32 in the session's sample buffer
void session_ingest_pcm(Session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels, const int32_t* rate,
                        const int32_t* format, int batch, int64_t* n_samples_out) {
    ASRB_REQUIRE(batch >= 1 && batch <= s->max_batch, ASRB_ERR_INVALID, "batch exceeds session capacity");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    if (!s->ingest) s->ingest = ingest_state_new();
    std::vector<int64_t> n((size_t)batch), so((size_t)batch);
    ingest_pcm(s->ingest, s->st, pcm, n_frames, channels, rate, format, batch, s->d_samples, s->max_samples, n.data(), so.data());
    s->ingested_n = n;
    s->stage = 0;
    if (n_samples_out) for (int b = 0; b < batch; ++b) n_samples_out[b] = n[b];
}
void session_ingested_read(Session* s, int b, float* out) {
    ASRB_REQUIRE(b >= 0 && b < (int)s->ingested_n.size(), ASRB_ERR_STATE, "ingested_read: nothing ingested for this index");
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    int64_t so = 0;
    for (int i = 0; i < b; ++i) so += ((s->ingested_n[i] + 159) / 160) * 160;
    ASRB_CUDA_CHECK(cudaMemcpy(out, s->d_samples + so, (size_t)s->ingested_n[b] * sizeof(float), cudaMemcpyDeviceToHost));
}

// (re)allocate a session scratch buffer to at least `n` elements; its contents are not kept.  The old buffer is freed
// first: the long-audio buffer can take hundreds of MB
template <typename T> static void grow(Session* s, T** p, size_t* cap, size_t n) {
    if (n <= *cap && *p) return;
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));      // the old buffer may still be read
    release_owned(s, *p); *p = nullptr; *cap = 0;
    *p = salloc<T>(s, n);
    *cap = n;
}

// asrb_ingest_long: the ingest of asrb_ingest_pcm into the long-audio buffer; a failed call leaves nothing ingested
void session_ingest_long(Session* s, const void* const* pcm, const int64_t* n_frames, const int32_t* channels, const int32_t* rate,
                         const int32_t* format, int n_files, int64_t* n_samples_out) {
    ASRB_REQUIRE(n_files >= 1, ASRB_ERR_INVALID, "n_files must be >= 1");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    s->long_n.clear(); s->long_off.clear();
    size_t total = 0;
    for (int f = 0; f < n_files; ++f) {
        ASRB_REQUIRE(n_frames[f] > 0 && rate[f] >= 1000 && rate[f] <= 768000, ASRB_ERR_INVALID, "ingest: bad PCM description");
        const int64_t nout = (n_frames[f] * 16000 + rate[f] - 1) / rate[f];       // = ingest_pcm's output length
        total += (size_t)((nout + 159) / 160) * 160;
    }
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));      // the ingest staging buffers may still be in use
    grow(s, &s->d_long, &s->long_cap, total);
    if (!s->ingest) s->ingest = ingest_state_new();
    std::vector<int64_t> n((size_t)n_files), so((size_t)n_files);
    ingest_pcm(s->ingest, s->st, pcm, n_frames, channels, rate, format, n_files, s->d_long, std::numeric_limits<int64_t>::max(),
               n.data(), so.data());
    s->long_n = n; s->long_off = so;
    if (n_samples_out) for (int f = 0; f < n_files; ++f) n_samples_out[f] = n[f];
}
void session_long_read(Session* s, int f, float* out) {
    ASRB_REQUIRE(f >= 0 && f < (int)s->long_n.size(), ASRB_ERR_STATE, "long_read: nothing ingested for this index");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    ASRB_CUDA_CHECK(cudaMemcpy(out, s->d_long + s->long_off[f], (size_t)s->long_n[f] * sizeof(float), cudaMemcpyDeviceToHost));
}

// asrb_segment_long: the cut rule of segment.cu on every long-audio file; segments in (file, time) order
void session_segment_long(Session* s, int64_t max_seg, int64_t search, int max_segments, int32_t* n_seg_out, int64_t* start_out,
                          int64_t* end_out) {
    ASRB_REQUIRE(!s->long_n.empty(), ASRB_ERR_STATE, "segment_long: nothing ingested with asrb_ingest_long");
    ASRB_REQUIRE(max_seg % 160 == 0 && search % 160 == 0 && max_seg >= 80000 && search >= 32000 && 2 * search <= max_seg,
                 ASRB_ERR_INVALID, "segment_long: need multiples of 160 with max_segment >= 80000 and 32000 <= search <= max_segment / 2");
    ASRB_REQUIRE(max_segments >= 0, ASRB_ERR_INVALID, "max_segments must be >= 0");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    const int F = (int)s->long_n.size();
    std::vector<int64_t> plan((size_t)4 * F + 1);         // off | n | boff[F + 1] | coff
    int64_t* off = plan.data(); int64_t* n = off + F; int64_t* boff = n + F; int64_t* coff = boff + F + 1;
    int64_t nblk = 0, ncut = 0;
    for (int f = 0; f < F; ++f) {
        off[f] = s->long_off[f]; n[f] = s->long_n[f];
        boff[f] = nblk; nblk += n[f] / 160;
        coff[f] = ncut; ncut += n[f] / (max_seg - search) + 1;   // each cut advances by >= max_seg - search
    }
    boff[F] = nblk;
    grow(s, &s->d_seg_blk, &s->seg_blk_cap, (size_t)nblk);
    grow(s, &s->d_seg_i64, &s->seg_i64_cap, plan.size() + F + ncut);
    int64_t* d_ncuts = s->d_seg_i64 + plan.size(); int64_t* d_cuts = d_ncuts + F;
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_seg_i64, plan.data(), plan.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s->st));
    launch_segment(s->d_long, s->d_seg_i64, F, nblk, max_seg, search, s->d_seg_blk, d_cuts, d_ncuts, s->m->ctx->sm_count, s->st);
    std::vector<int64_t> res((size_t)F + ncut);
    ASRB_CUDA_CHECK(cudaMemcpyAsync(res.data(), d_ncuts, res.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    int64_t total = 0;
    for (int f = 0; f < F; ++f) { total += res[f] + 1; if (n_seg_out) n_seg_out[f] = (int32_t)(res[f] + 1); }
    ASRB_REQUIRE(total <= max_segments, ASRB_ERR_INVALID,
                 "segment_long: " + std::to_string(total) + " segments do not fit in max_segments (n_segments_out holds the counts)");
    int64_t o = 0;
    for (int f = 0; f < F; ++f) {
        const int64_t* c = res.data() + F + coff[f];
        for (int64_t k = 0; k <= res[f]; ++k, ++o) {
            start_out[o] = k == 0 ? 0 : c[k - 1];
            end_out[o] = k == res[f] ? n[f] : c[k];
        }
    }
}

void session_mel_read(Session* s, int b, float* out) {
    ASRB_REQUIRE(s->stage >= 1 && !s->stream_run && b >= 0 && b < s->B, ASRB_ERR_STATE, "mel_read: no mel for this index");
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    const int nm = s->m->d.c.num_mel_bins;
    ASRB_CUDA_CHECK(cudaMemcpy(out, s->d_mel + (size_t)nm * s->foff[b], (size_t)nm * s->F[b] * sizeof(float), cudaMemcpyDeviceToHost));
}

// -------------------------------------------------------------------------------------------------
// step 3: audio encoder  (inference.rs:100 -> audio_encoder.rs:79-169)
// -------------------------------------------------------------------------------------------------
static GemmA plainA(const bf16* a, size_t ps, int M, int K, int nplanes) {
    GemmA A; A.mode = A_PLAIN; A.a = a; A.plane_stride = ps; A.M = M; A.K = K; A.lda = K; A.nplanes = nplanes; return A;
}

void session_encode(Session* s, int64_t* n_tokens_out) {
    ASRB_REQUIRE(s->stage >= 1 && !s->stream_run, ASRB_ERR_STATE, "encode called before mel");
    Model& m = *s->m; const Dims& d = m.d; const asrb_dims& c = d.c;
    const int B = s->B, tpc = d.tok_per_chunk, cf = d.chunk_frames;
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    // ---- plan: chunks, valid tokens, windows (audio_encoder.rs:83-121,141-152,172-209) ----
    s->C.assign(B, 0); s->T.assign(B, 0); s->toff.assign(B, 0);
    int totC = 0, totT = 0;
    for (int b = 0; b < B; ++b) { s->C[b] = (int)((s->F[b] + cf - 1) / cf); totC += s->C[b]; }
    int* hi = s->h_int;
    int* chunk_clip = hi; int* chunk_f0 = chunk_clip + totC; int* rowmap = chunk_f0 + totC;
    int* win_q0 = rowmap + (size_t)totC * tpc; int* win_len = win_q0 + (totC + B);
    int ci = 0, nwin = 0, maxwin = 0;
    for (int b = 0; b < B; ++b) {
        s->toff[b] = totT;
        int wtok = 0, wq0 = totT;
        for (int k = 0; k < s->C[b]; ++k, ++ci) {
            chunk_clip[ci] = b; chunk_f0[ci] = k * cf;
            int frames = (int)std::min<int64_t>(cf, s->F[b] - (int64_t)k * cf);
            int valid = chunk_tokens(frames);
            for (int t = 0; t < tpc; ++t) rowmap[(size_t)ci * tpc + t] = t < valid ? totT + t : -1;
            totT += valid; wtok += valid;
            bool close = d.chunks_per_window > 0 && ((k + 1) % d.chunks_per_window == 0);
            if (close || k == s->C[b] - 1) {
                if (d.chunks_per_window == 0) { /* mask None: one window per utterance */ if (k != s->C[b] - 1) continue; }
                win_q0[nwin] = wq0; win_len[nwin] = wtok; maxwin = std::max(maxwin, wtok); ++nwin;
                wq0 = totT; wtok = 0;
            }
        }
        s->T[b] = totT - s->toff[b];
    }
    s->totC = totC; s->totT = totT; s->nwin = nwin; s->maxwin = maxwin;
    const size_t nint = (size_t)(win_len + (totC + B) - hi);
    ASRB_REQUIRE(nint <= s->enc_int_cap, ASRB_ERR_INVALID, "plan exceeds session capacity");
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_int, hi, nint * sizeof(int), cudaMemcpyHostToDevice, s->st));
    s->d_chunk_clip = s->d_int; s->d_chunk_f0 = s->d_int + (chunk_f0 - hi); s->d_rowmap = s->d_int + (rowmap - hi);
    s->d_win_q0 = s->d_int + (win_q0 - hi); s->d_win_len = s->d_int + (win_len - hi);
    const int Bm = s->max_batch; const int np = s->nplanes; cudaStream_t st = s->st;

    // ---- conv stem ----
    launch_conv1(m, s->d_mel, s->d_chunk_clip, s->d_chunk_f0, s->d_i64 + 3 * Bm, s->d_i64 + 4 * Bm, totC, s->act1, s->act1_ps, st);
    {   // conv2d2: implicit GEMM  M = C*32*25, N = dsh, K = 9*cpad
        GemmA A; A.mode = A_CONV; A.a = s->act1; A.plane_stride = s->act1_ps; A.nplanes = np;
        A.OH = d.conv_h[2]; A.OW = d.conv_w[2]; A.Hh = d.conv_h[2]; A.Wh = d.conv_w[2]; A.cpad = d.cpad;
        A.M = totC * A.OH * A.OW; A.K = 9 * d.cpad; A.lda = A.K;
        GemmEpi E; E.mode = EPI_CONV_PARITY; E.bias = m.conv2_b; E.out_s3 = s->act2; E.s3_plane_stride = s->act2_ps;
        E.OH = A.OH; E.OW = A.OW; E.Hh2 = d.conv_h[3]; E.Wh2 = d.conv_w[3]; E.cpad = d.cpad;
        launch_gemm(A, m.conv2_w, c.downsample_hidden_size, E, s->gemm_impl, st);
    }
    {   // conv2d3
        GemmA A; A.mode = A_CONV; A.a = s->act2; A.plane_stride = s->act2_ps; A.nplanes = np;
        A.OH = d.conv_h[3]; A.OW = d.conv_w[3]; A.Hh = d.conv_h[3]; A.Wh = d.conv_w[3]; A.cpad = d.cpad;
        A.M = totC * A.OH * A.OW; A.K = 9 * d.cpad; A.lda = A.K;
        GemmEpi E; E.mode = EPI_CONV_FEAT; E.bias = m.conv3_b; E.out_s3 = s->feat; E.s3_plane_stride = s->feat_ps;
        E.OH = A.OH; E.OW = A.OW; E.lds = d.feat;
        launch_gemm(A, m.conv3_w, c.downsample_hidden_size, E, s->gemm_impl, st);
    }
    {   // conv_out + positional embedding + valid-token gather -> x_enc [totT][d_model]
        GemmA A = plainA(s->feat, s->feat_ps, totC * tpc, d.feat, np);
        GemmEpi E; E.mode = EPI_CONVOUT; E.bias = m.conv_out_b; E.out_f32 = s->x_enc; E.ldo = c.d_model;
        E.splitk_ws = s->splitk_ws; E.extra_launches = &s->launches;
        E.row_map = s->d_rowmap; E.pos = m.pos_emb; E.pos_period = tpc;
        launch_gemm(A, m.conv_out_w, c.d_model, E, s->gemm_impl, st);
    }
    s->launches += 4;
    // ---- transformer layers (layers.rs:230-242) ----
    const int dm = c.d_model;
    for (int l = 0; l < c.encoder_layers; ++l) {
        const EncLayerW& w = m.enc[l];
        launch_layernorm_s3(s->x_enc, w.ln1_w, w.ln1_b, totT, dm, 1e-5f, s->enc_h, s->ench_ps, st);
        { GemmA A = plainA(s->enc_h, s->ench_ps, totT, dm, np);
          GemmEpi E; E.bias = w.bqkv; E.out_f32 = s->enc_qkv; E.ldo = 3 * dm;
          launch_gemm(A, w.wqkv, 3 * dm, E, s->gemm_impl, st); }
        { AttnParams p{}; p.q = s->enc_qkv; p.ldq = 3 * dm; p.k = s->enc_qkv + dm; p.v = s->enc_qkv + 2 * dm;
          p.head_stride = d.enc_hd; p.ldk = 3 * dm; p.seg_stride = 0; p.keys_in_rows = 1;
          p.seg_q0 = s->d_win_q0; p.seg_len = s->d_win_len; p.nseg = nwin; p.nheads = c.encoder_attention_heads; p.group = 1;
          p.causal = 0; p.max_len = maxwin; p.out_s3 = s->enc_attn; p.plane_stride = s->ench_ps; p.ldo = dm;
          launch_attention(p, d.enc_hd, st); }
        { GemmA A = plainA(s->enc_attn, s->ench_ps, totT, dm, np);
          GemmEpi E; E.bias = w.bo; E.residual = s->x_enc; E.ldr = dm; E.out_f32 = s->x_enc; E.ldo = dm; E.splitk_ws = s->splitk_ws; E.extra_launches = &s->launches;
          launch_gemm(A, w.wo, dm, E, s->gemm_impl, st); }
        launch_layernorm_s3(s->x_enc, w.ln2_w, w.ln2_b, totT, dm, 1e-5f, s->enc_h, s->ench_ps, st);
        { GemmA A = plainA(s->enc_h, s->ench_ps, totT, dm, np);
          GemmEpi E; E.bias = w.b1; E.act = 1; E.out_s3 = s->enc_ff; E.s3_plane_stride = s->encff_ps; E.lds = c.encoder_ffn_dim;
          launch_gemm(A, w.fc1, c.encoder_ffn_dim, E, s->gemm_impl, st); }
        { GemmA A = plainA(s->enc_ff, s->encff_ps, totT, c.encoder_ffn_dim, np);
          GemmEpi E; E.bias = w.b2; E.residual = s->x_enc; E.ldr = dm; E.out_f32 = s->x_enc; E.ldo = dm; E.splitk_ws = s->splitk_ws; E.extra_launches = &s->launches;
          launch_gemm(A, w.fc2, dm, E, s->gemm_impl, st); }
        s->launches += 7;
    }
    // ---- ln_post -> proj1 + GELU -> proj2  (audio_encoder.rs:163-165) ----
    launch_layernorm_s3(s->x_enc, m.lnpost_w, m.lnpost_b, totT, dm, 1e-5f, s->enc_h, s->ench_ps, st);
    { GemmA A = plainA(s->enc_h, s->ench_ps, totT, dm, np);
      GemmEpi E; E.bias = m.proj1_b; E.act = 1; E.out_s3 = s->enc_attn; E.s3_plane_stride = s->ench_ps; E.lds = dm;
      launch_gemm(A, m.proj1, dm, E, s->gemm_impl, st); }
    { GemmA A = plainA(s->enc_attn, s->ench_ps, totT, dm, np);
      GemmEpi E; E.bias = m.proj2_b; E.out_f32 = s->audio; E.ldo = c.output_dim; E.splitk_ws = s->splitk_ws; E.extra_launches = &s->launches;
      launch_gemm(A, m.proj2, c.output_dim, E, s->gemm_impl, st); }
    s->launches += 3;
    if (n_tokens_out) for (int b = 0; b < B; ++b) n_tokens_out[b] = s->T[b];
    s->stage = 2;
}

void session_encode_read(Session* s, int b, float* out) {
    ASRB_REQUIRE(s->stage >= 2 && !s->stream_run && b >= 0 && b < s->B, ASRB_ERR_STATE, "encode_read: nothing encoded for this index");
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    const int od = s->m->d.c.output_dim;
    ASRB_CUDA_CHECK(cudaMemcpy(out, s->audio + (size_t)s->toff[b] * od, (size_t)s->T[b] * od * sizeof(float), cudaMemcpyDeviceToHost));
}

// -------------------------------------------------------------------------------------------------
// steps 4-7: prompt, embed + inject, positions, prefill  (inference.rs:105-149)
// -------------------------------------------------------------------------------------------------
// sampling with the top-k candidate lists is not offered, nor beam search with either; a beam run needs batch * K slots.
// Refused by every call that runs a prefill, before any work.
static void check_sampling_options(const Session* s, int batch) {
    ASRB_REQUIRE(!(s->temperature > 0.0 && s->top_k > 0), ASRB_ERR_INVALID, "temperature > 0 cannot be combined with top_logprobs");
    if (s->beam_k > 1) {
        ASRB_REQUIRE(s->temperature == 0.0, ASRB_ERR_INVALID, "beam_size > 1 cannot be combined with temperature > 0");
        ASRB_REQUIRE(s->top_k == 0, ASRB_ERR_INVALID, "beam_size > 1 cannot be combined with top_logprobs");
        ASRB_REQUIRE((int64_t)batch * s->beam_k <= s->max_batch, ASRB_ERR_INVALID,
                     "beam search needs batch * beam_size <= the session's max_batch");
    }
}

static void ensure_beam_bufs(Session* s) {
    BeamArgs& a = s->beam;
    if (a.u) return;
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    const size_t Bm = s->max_batch, hist = (size_t)s->max_new * Bm, nb = Bm * BEAM_MAX * s->max_new;
    a.u = salloc<BeamUtt>(s, Bm, true);
    a.hist_tok = salloc<int>(s, hist); a.hist_par = salloc<int>(s, hist); a.hist_lp = salloc<float>(s, hist);
    a.cp_src = salloc<int>(s, Bm); a.cp_p0 = salloc<int>(s, Bm); a.cp_n = salloc<int>(s, Bm, true);
    a.nb_ids = salloc<int>(s, nb); a.nb_lp = salloc<float>(s, nb);
    s->d_hyp = salloc<int>(s, Bm * BEAM_MAX * 2);
    s->d_best_eos = salloc<float>(s, Bm);
}

// the run's geometry and the current decode buffers (the record buffers may have been allocated since the last call)
static const BeamArgs& beam_args(Session* s) {
    const Dims& d = s->m->d; const asrb_dims& c = d.c; const DecodeBufs& db = s->db;
    BeamArgs& a = s->beam;
    a.B = s->B; a.K = s->run_k; a.max_new = s->max_new; a.hidden = c.hidden_size; a.ldh = s->max_batch;
    a.bytes_per_pos = 2LL * c.num_hidden_layers * c.num_key_value_heads * c.head_dim * (long long)sizeof(float);
    a.tk_ids = db.tk_ids; a.tk_lp = db.tk_lp; a.tk_eos_ids = db.tk_eos_ids; a.tk_eos_lp = db.tk_eos_lp;
    a.done = db.done; a.pos = db.pos; a.next_id = db.next_id; a.n_out = db.n_out; a.ids_out = db.ids_out;
    a.x = db.x; a.embed = s->m->embed; a.lp_out = db.lp_out; a.eos_lp = db.eos_lp;
    a.kcache = s->kcache; a.vcache = s->vcache; a.layers = c.num_hidden_layers; a.nkv = c.num_key_value_heads;
    a.head_dim = c.head_dim; a.max_ctx = s->max_ctx; a.layer_stride = s->cache_layer_stride; a.seq_stride = s->cache_seq_stride;
    return a;
}

static void ensure_sample_bufs(Session* s) {     // sampling with logprobs: the raw records beside the keys
    DecodeBufs& b = s->db;
    if (b.sample && b.logprobs && !b.part_max) {
        ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
        b.part_max = salloc<float>(s, (size_t)s->max_batch * b.n_part);
        b.part_sel = salloc<float>(s, (size_t)s->max_batch * b.n_part);
    }
}

// contexts: set by asrb_session_set_context, checked against the run's batch by every call that runs a prefill, before
// any work
static void check_context(const Session* s, int batch) {
    ASRB_REQUIRE(s->ctx_rows <= 1 || s->ctx_rows == batch, ASRB_ERR_INVALID,
                 "the contexts set with asrb_session_set_context have neither 1 row nor one row per utterance of this batch");
}
static const std::vector<int>& context_of(const Session* s, int b) {
    static const std::vector<int> none;
    return s->ctx_rows == 0 ? none : s->ctx[s->ctx_rows == 1 ? 0 : b];
}

void session_set_context(Session* s, int n_rows, const int64_t* const* ids, const int32_t* n_ids) {
    ASRB_REQUIRE(n_rows >= 0, ASRB_ERR_INVALID, "n_rows must be >= 0");
    ASRB_REQUIRE(n_rows == 0 || n_ids, ASRB_ERR_INVALID, "null pointer: n_ids");
    std::vector<std::vector<int>> rows((size_t)n_rows);
    for (int b = 0; b < n_rows; ++b) {
        const int n = (ids && ids[b]) ? n_ids[b] : 0;
        ASRB_REQUIRE(n >= 0 && n <= s->max_context, ASRB_ERR_INVALID, "context exceeds the session's max_context_ids");
        rows[b].resize(n);
        for (int i = 0; i < n; ++i) {
            const int64_t id = ids[b][i];
            ASRB_REQUIRE(id >= 0 && id < s->m->d.c.vocab_size, ASRB_ERR_INVALID, "context id out of vocabulary");
            rows[b][i] = (int)id;
        }
    }
    s->ctx = std::move(rows); s->ctx_rows = n_rows;
}

// [0] prompt rows computed  [1] prompt rows taken from a leader  [2] KV bytes fanned out to followers
void session_last_prefill_stats(Session* s, int64_t* out, int n) {
    const int64_t v[3] = {s->pf_rows, s->pf_shared_rows, s->pf_fan_bytes};
    for (int i = 0; i < n && i < 3; ++i) out[i] = v[i];
}

// language ids of utterance b: their count (0 when none are given), checked against the session's max_lang less
// `reserved` (a stream's forced prefix) and against the vocabulary
static int lang_count(const Session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, int b, int reserved = 0,
                      const char* over = "language prompt exceeds session capacity") {
    const int nl = (lang_ids && lang_ids[b] && n_lang_ids) ? n_lang_ids[b] : 0;
    ASRB_REQUIRE(nl >= 0 && nl + reserved <= s->max_lang, ASRB_ERR_INVALID, over);
    for (int i = 0; i < nl; ++i)
        ASRB_REQUIRE(lang_ids[b][i] >= 0 && lang_ids[b][i] < s->m->d.c.vocab_size, ASRB_ERR_INVALID, "language id out of vocabulary");
    return nl;
}

// a whole prompt, position by position: ids, and the audio row of each audio position (-1 elsewhere).  Head, context,
// end of the system turn and start of the user turn, T audio pads reading rows arow0 .. arow0 + T - 1, the tail, the nl
// language ids, then the forced prefix of a stream
static void build_prompt(const std::vector<int>& ctx, int T, int arow0, const int64_t* lang, int nl, const std::vector<int>& forced,
                         std::vector<int>& pid, std::vector<int>& parow) {
    pid.clear(); parow.clear();
    for (int i = 0; i < 3; ++i) { pid.push_back(kPromptHead[i]); parow.push_back(-1); }
    for (int id : ctx) { pid.push_back(id); parow.push_back(-1); }
    for (int i = 3; i < 9; ++i) { pid.push_back(kPromptHead[i]); parow.push_back(-1); }
    for (int t = 0; t < T; ++t) { pid.push_back(kAudioPad); parow.push_back(arow0 + t); }
    for (int i = 0; i < 6; ++i) { pid.push_back(kPromptTail[i]); parow.push_back(-1); }
    for (int i = 0; i < nl; ++i) { pid.push_back((int)lang[i]); parow.push_back(-1); }
    for (int id : forced) { pid.push_back(id); parow.push_back(-1); }
}
// utterance b's prompt of the current offline batch, with its nl language ids
static void build_prompt(const Session* s, int b, const int64_t* const* lang_ids, int nl, std::vector<int>& pid, std::vector<int>& parow) {
    build_prompt(context_of(s, b), s->T[b], s->toff[b], nl > 0 ? lang_ids[b] : nullptr, nl, {}, pid, parow);
}

// one sequence (KV slot) of a prefill: all its positions (ids, and audio rows as build_prompt gives them), the first one
// it computes, and the slot whose K/V holds positions [0, from): an earlier slot, a leader that fans them out to this
// follower as it computes them; this slot itself, which kept them from an earlier call; or none (-1, from = 0)
struct PrefillSeq {
    std::vector<int> pid, parow;
    int from = 0, lead = -1;
};
struct PrefillPlan {
    int totS = 0, nseq = 0, maxrows = 0;      // rows, sequences, most rows of one sequence
    std::vector<int> srow0;                   // first row of each sequence
    bool fan = false; FanOut fan_plan{};      // fan: some sequence follows a leader
    const int* d_qpos0 = nullptr;             // first computed position per sequence; null: no sequence has a lead
    const int* d_tail = nullptr;              // the caller's ints behind the plan
};
// the row plan of a prefill, sequence-major, in the int region (hi, di) of `cap` ints: ids | arow | rseq | rpos per row,
// sq0 | slen | qpos0 | fan_n | fan_off | fan_P per sequence, the follower slots grouped by leader, then `extra` ints of
// the caller's that fill_tail(tail, plan) writes.  Uploads it, points the session's row arrays at it and records the
// prefill stats
template <typename FillTail>
static PrefillPlan plan_prefill(Session* s, const std::vector<PrefillSeq>& seq, int* hi, int* di, size_t cap, int extra,
                                FillTail fill_tail) {
    const asrb_dims& c = s->m->d.c;
    PrefillPlan p;
    const int N = (int)seq.size();
    p.nseq = N; p.srow0.assign(N, 0);
    int nf = 0; int64_t shared = 0; bool led = false;
    for (int q = 0; q < N; ++q) {
        const int rows = (int)seq[q].pid.size() - seq[q].from;
        p.srow0[q] = p.totS; p.totS += rows; p.maxrows = std::max(p.maxrows, rows);
        led = led || seq[q].lead >= 0;
        if (seq[q].lead >= 0 && seq[q].lead != q) { ++nf; shared += seq[q].from; }
    }
    const int totS = p.totS;
    const size_t nint = 4 * (size_t)totS + 6 * (size_t)N + std::max(nf, 1) + extra;
    ASRB_REQUIRE(nint <= cap, ASRB_ERR_INVALID, "plan exceeds session capacity");
    int* ids = hi; int* arow = ids + totS; int* rseq = arow + totS; int* rpos = rseq + totS;
    int* sq0 = rpos + totS; int* slen = sq0 + N; int* qpos0 = slen + N;
    int* fan_n = qpos0 + N; int* fan_off = fan_n + N; int* fan_P = fan_off + N; int* fan_slots = fan_P + N;
    int* tail = fan_slots + std::max(nf, 1);
    for (int q = 0, r = 0, f = 0; q < N; ++q) {
        const PrefillSeq& x = seq[q];
        // position = index in the prompt (build_position_ids, inference.rs:259-266)
        for (int i = x.from; i < (int)x.pid.size(); ++i, ++r) { ids[r] = x.pid[i]; arow[r] = x.parow[i]; rseq[r] = q; rpos[r] = i; }
        sq0[q] = p.srow0[q]; slen[q] = (int)x.pid.size() - x.from; qpos0[q] = x.from;
        fan_off[q] = f; fan_n[q] = 0; fan_P[q] = 0;
        for (int b = q + 1; b < N; ++b)
            if (seq[b].lead == q) { fan_slots[f++] = b; ++fan_n[q]; fan_P[q] = seq[b].from; }
    }
    fill_tail(tail, p);
    s->pf_rows = totS; s->pf_shared_rows = shared;
    s->pf_fan_bytes = shared * 2LL * c.num_hidden_layers * c.num_key_value_heads * c.head_dim * (int64_t)sizeof(float);
    ASRB_CUDA_CHECK(cudaMemcpyAsync(di, hi, nint * sizeof(int), cudaMemcpyHostToDevice, s->st));
    s->d_ids = di; s->d_audio_row = di + (arow - hi); s->d_row_seq = di + (rseq - hi);
    s->d_row_pos = di + (rpos - hi); s->d_seq_q0 = di + (sq0 - hi); s->d_seq_len = di + (slen - hi);
    p.fan = nf > 0;
    p.fan_plan = FanOut{di + (fan_n - hi), di + (fan_off - hi), di + (fan_P - hi), di + (fan_slots - hi)};
    p.d_qpos0 = led ? di + (qpos0 - hi) : nullptr;   // none: the kernels of a call without contexts
    p.d_tail = di + (tail - hi);
    return p;
}

// an alignment call's work inside the prefill: run(l) after layer l's q / k normalisation and RoPE, while s->qrot
// holds that layer's q and the K cache that layer's keys
struct LayerHook {
    virtual void run(int layer) = 0;
    virtual ~LayerHook() = default;
};

// embed + inject and the decoder layers over the rows of plan `pf` (sequence q's rows are its segment of the attention,
// in KV slot q); audio rows are read from `audio`.  n_layers < 0: every layer; else the layers 0 .. n_layers - 1, the
// last of them stopping after `hook` (an alignment call, which needs no later work)
static void prefill_layers(Session* s, const PrefillPlan& pf, const float* audio, int n_layers = -1, LayerHook* hook = nullptr) {
    Model& m = *s->m; const Dims& d = m.d; const asrb_dims& c = d.c;
    cudaStream_t st = s->st; const int np = s->nplanes;
    const int totS = pf.totS;
    const FanOut* fan = pf.fan ? &pf.fan_plan : nullptr;
    launch_embed_inject(m.embed, c.hidden_size, s->d_ids, s->d_audio_row, audio, totS, s->hid, st);
    s->launches += 1;
    const int H = c.hidden_size; const float eps = (float)c.rms_norm_eps;
    const int L = n_layers < 0 ? c.num_hidden_layers : n_layers;
    for (int l = 0; l < L; ++l) {
        const DecLayerW& w = m.dec[l];
        float* kc = s->kcache + (size_t)l * s->cache_layer_stride;
        float* vc = s->vcache + (size_t)l * s->cache_layer_stride;
        launch_rmsnorm_s3(s->hid, w.ln_in, totS, H, eps, s->dh, s->dh_ps, st);
        { GemmA A = plainA(s->dh, s->dh_ps, totS, H, np);
          GemmEpi E; E.out_f32 = s->dqkv; E.ldo = d.qkv_dim;
          launch_gemm(A, w.wqkv, d.qkv_dim, E, s->gemm_impl, st); }
        launch_qk_norm_rope(s->dqkv, totS, s->d_row_seq, s->d_row_pos, w.qnorm, w.knorm, eps, m.rope_cos, m.rope_sin,
                            c.num_attention_heads, c.num_key_value_heads, c.head_dim, s->qrot, kc, vc, s->cache_seq_stride,
                            s->max_ctx, st, fan);
        if (hook) {
            hook->run(l);
            if (l == L - 1) { s->launches += 3; break; }
        }
        { AttnParams p{}; p.q = s->qrot; p.ldq = d.q_dim; p.k = kc; p.v = vc; p.seg_stride = s->cache_seq_stride;
          p.head_stride = (size_t)s->max_ctx * c.head_dim; p.ldk = c.head_dim; p.keys_in_rows = 0;
          p.seg_q0 = s->d_seq_q0; p.seg_len = s->d_seq_len; p.nseg = pf.nseq; p.nheads = c.num_attention_heads;
          p.group = c.num_attention_heads / c.num_key_value_heads; p.causal = 1; p.max_len = pf.maxrows; p.seg_pos0 = pf.d_qpos0;
          p.out_s3 = s->dattn; p.plane_stride = s->dattn_ps; p.ldo = d.q_dim;
          launch_attention(p, c.head_dim, st); }
        { GemmA A = plainA(s->dattn, s->dattn_ps, totS, d.q_dim, np);
          GemmEpi E; E.residual = s->hid; E.ldr = H; E.out_f32 = s->hid; E.ldo = H; E.splitk_ws = s->splitk_ws; E.extra_launches = &s->launches;
          launch_gemm(A, w.wo, H, E, s->gemm_impl, st); }
        launch_rmsnorm_s3(s->hid, w.ln_post, totS, H, eps, s->dh, s->dh_ps, st);
        { GemmA A = plainA(s->dh, s->dh_ps, totS, H, np);
          GemmEpi E; E.mode = EPI_SWIGLU; E.out_s3 = s->dact; E.s3_plane_stride = s->dact_ps; E.lds = c.intermediate_size;
          launch_gemm(A, w.wgu, 2 * c.intermediate_size, E, s->gemm_impl, st); }
        { GemmA A = plainA(s->dact, s->dact_ps, totS, c.intermediate_size, np);
          GemmEpi E; E.residual = s->hid; E.ldr = H; E.out_f32 = s->hid; E.ldo = H; E.splitk_ws = s->splitk_ws; E.extra_launches = &s->launches;
          launch_gemm(A, w.wdown, H, E, s->gemm_impl, st); }
        s->launches += 8;
    }
}

static void begin_run(Session* s, int B, const int* d_start);
static void first_token(Session* s, int B, bool write_logits, const int* pos0);

void session_prefill(Session* s, const int64_t* const* lang_ids, const int32_t* n_lang_ids, int64_t* seq_lens_out,
                     float* last_logits) {
    ASRB_REQUIRE(s->stage >= 2 && !s->stream_run, ASRB_ERR_STATE, "prefill called before encode");
    check_sampling_options(s, s->B);
    s->streams_open = false;                        // the prefill overwrites the streams' K/V slots
    check_context(s, s->B);
    Model& m = *s->m; const asrb_dims& c = m.d.c;
    const int B = s->B; cudaStream_t st = s->st;
    std::vector<int> nl((size_t)B);
    for (int b = 0; b < B; ++b) nl[b] = lang_count(s, lang_ids, n_lang_ids, b);
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    s->run_k = s->beam_k; s->run_alpha = s->length_penalty; s->nslots = B * s->run_k; s->nbest_valid = false;
    if (s->run_k > 1) { ensure_beam_bufs(s); s->beam_steps = 0; }
    // shared contexts: an utterance whose non-empty context equals that of an earlier leader follows it; its positions
    // before the audio (head, context, end of the system turn, user turn up to the audio start) are the leader's
    std::vector<PrefillSeq> seq((size_t)B);
    s->S.assign(B, 0); s->maxlenS = 0;
    for (int b = 0; b < B; ++b) {
        build_prompt(s, b, lang_ids, nl[b], seq[b].pid, seq[b].parow);
        s->S[b] = (int)seq[b].pid.size(); s->maxlenS = std::max(s->maxlenS, s->S[b]);
        const std::vector<int>& cb = context_of(s, b);
        if (cb.empty()) continue;
        for (int a = 0; a < b; ++a)
            if (seq[a].lead < 0 && context_of(s, a) == cb) { seq[b].lead = a; seq[b].from = audio_start((int)cb.size()); break; }
    }
    // separate region: the encoder plan upload may still be in flight
    const PrefillPlan pf = plan_prefill(s, seq, s->h_int + s->enc_int_cap, s->d_int + s->enc_int_cap, s->int_cap - s->enc_int_cap,
                                        3 * B, [&](int* t, const PrefillPlan& p) {   // lastrow | pos0 | done0
        for (int b = 0; b < B; ++b) { t[b] = p.srow0[b] + s->S[b] - seq[b].from - 1; t[B + b] = s->S[b] - 1; t[2 * B + b] = 0; }
    });
    begin_run(s, B, pf.d_tail);
    prefill_layers(s, pf, s->audio);
    first_token(s, B, last_logits != nullptr, pf.d_tail + B);
    if (seq_lens_out) for (int b = 0; b < B; ++b) seq_lens_out[b] = s->S[b];
    if (last_logits) {
        ASRB_CUDA_CHECK(cudaStreamSynchronize(st));
        ASRB_CUDA_CHECK(cudaMemcpy(last_logits, s->db.logits, (size_t)B * c.vocab_size * sizeof(float), cudaMemcpyDeviceToHost));
    }
    s->stage = 3;
}

// the run's B sequences started from the device ints lastrow | pos0 | done0 at d_start (each sequence's last prefill row,
// its decode position and whether it is done from the start), its result rows reset and its record, sampling and
// top-k options latched; before the prefill
static void begin_run(Session* s, int B, const int* d_start) {
    cudaStream_t st = s->st;
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_lastrow, d_start, B * sizeof(int), cudaMemcpyDeviceToDevice, st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->db.pos, d_start + B, B * sizeof(int), cudaMemcpyDeviceToDevice, st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->db.done, d_start + 2 * B, B * sizeof(int), cudaMemcpyDeviceToDevice, st));
    ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.n_out, 0, B * sizeof(int), st));
    s->lp_valid = s->opt_logprobs || s->top_k > 0;   // latched here: a run records log-probabilities only if it starts with the option on
    if (s->db.logprobs) {                  // all NaN (0xFFFFFFFF): no EOS seen, nothing appended
        ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.eos_lp, 0xFF, B * sizeof(float), st));
        ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.lp_out, 0xFF, (size_t)B * s->max_new * sizeof(float), st));
    }
    s->db.sample = s->temperature > 0.0;   // latched: the whole run samples with this run's temperature and seed
    if (s->db.sample) {
        const SampleParams hp{(float)(1.0 / s->temperature), (uint32_t)(s->seed & 0xffffffffu), (uint32_t)(s->seed >> 32)};
        ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_smp, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
        ensure_sample_bufs(s);
    }
    s->db.rep = false;                     // token 0 has no history: the prefill's lm_head folds the raw logits
    s->tk_valid = s->top_k;
    if (s->db.topk) {                      // ids -1, values NaN (0xFFFFFFFF): nothing recorded yet
        const size_t rows = (size_t)B * s->max_new * TK_MAX;
        ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.tk_ids, 0xFF, rows * sizeof(int), st));
        ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.tk_lp, 0xFF, rows * sizeof(float), st));
        ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.tk_eos_ids, 0xFF, (size_t)B * TK_MAX * sizeof(int), st));
        ASRB_CUDA_CHECK(cudaMemsetAsync(s->db.tk_eos_lp, 0xFF, (size_t)B * TK_MAX * sizeof(float), st));
    }
}

// token 0 of every sequence from its last prefill row (s->d_lastrow), then the repetition rule latched for the steps;
// pos0: the prompt lengths minus one, for the beam run's token-0 walk
static void first_token(Session* s, int B, bool write_logits, const int* pos0) {
    Model& m = *s->m; cudaStream_t st = s->st;
    // final norm + lm_head on the last row of each utterance only (the reference computes all S rows,
    // text_decoder.rs:111-112, and uses row S-1, inference.rs:156)
    launch_lmhead_argmax(m, s->hid, s->d_lastrow, B, s->db, write_logits, st, &s->launches);
    // greedy bookkeeping for token 0 (inference.rs:161-170): argmax, EOS check, append, embed
    launch_greedy(m, s->db, B, st, &s->launches);
    // beam search: the token-0 walk on each utterance's record, then its prompt KV copied into its other K - 1 slots
    if (s->run_k > 1) launch_beam_step(beam_args(s), true, pos0, st, &s->launches);
    s->greedy_done = 1;
    s->db.rep = s->ngram > 0 || s->rep_penalty != 1.0;   // latched: every decode step of the run applies this run's rule
    if (s->db.rep) {
        const RepParams hp{(float)s->rep_penalty, s->ngram};
        ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_rep, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
        if (!s->db.rep_mask)                // per-phase: [max_batch][2][vocab words]; fused steps: [G][up to 16][2][CTA words]
            s->db.rep_mask = salloc<uint32_t>(s, std::max((size_t)s->max_batch * 2 * s->db.rep_words,
                                                          (size_t)m.ctx->sm_count * 16 * 2 * rep_cta_words(m.d.c, m.ctx->sm_count)));
    }
}

// -------------------------------------------------------------------------------------------------
// step 8: greedy loop  (inference.rs:160-200)
// -------------------------------------------------------------------------------------------------
bool decode_mega_supported(const Model& m, int B, int max_ctx);
bool decode_batch_supported(const Model& m, int B, int max_ctx);
size_t decode_batch_part_floats(const Model& m);
void launch_decode_step_batch(const Model& m, const DecodeBufs& b, int B, float* kcache, float* vcache,
                              size_t cache_layer_stride, size_t cache_seq_stride, int max_ctx, int ctx_now, const MegaBufs& mb,
                              cudaStream_t st, int64_t* launches);
void launch_decode_step_mega(const Model& m, const DecodeBufs& b, int B, float* kcache, float* vcache,
                             size_t cache_layer_stride, size_t cache_seq_stride, int max_ctx, int ctx_now, const MegaBufs& mb,
                             cudaStream_t st, int64_t* launches);
size_t decode_mega_part_floats(const Model& m);
int decode_mega_dbg_slots();
static void apply_record_options(Session* s);

// one iteration of the loop body: decoder forward on the pending token, then the greedy bookkeeping
// that selects / appends / embeds the next one.  (The fused kernel does both.)
// upper bound of (position + 1) for the next forward: prompt length + tokens appended so far
static int ctx_bound(const Session* s) { return std::min(s->max_ctx, s->maxlenS + s->greedy_done); }
// the decode rows are the nslots sequences of the run: the utterances, or their beam slots
static bool use_batch(Session* s, bool write_logits) {     // batch >= 2: weights streamed once for all sequences
    return s->decode_mode == 1 && s->batch_step && !write_logits && s->nslots >= 2 && decode_batch_supported(*s->m, s->nslots, ctx_bound(s));
}
static bool use_mega(Session* s, bool write_logits) {
    return use_batch(s, write_logits) ||
           (s->decode_mode == 1 && !write_logits && decode_mega_supported(*s->m, s->nslots, ctx_bound(s)));
}
static void forward_step(Session* s, bool write_logits) {
    Model& m = *s->m;
    const int R = s->nslots;
    if (use_batch(s, write_logits)) {
        launch_decode_step_batch(m, s->db, R, s->kcache, s->vcache, s->cache_layer_stride, s->cache_seq_stride, s->max_ctx,
                                 ctx_bound(s), s->mega, s->st, &s->launches);
        s->n_batch_steps += 1;
    } else if (use_mega(s, write_logits)) {
        launch_decode_step_mega(m, s->db, R, s->kcache, s->vcache, s->cache_layer_stride, s->cache_seq_stride, s->max_ctx,
                                ctx_bound(s), s->mega, s->st, &s->launches);
        s->n_mega_steps += 1;
    } else {
        s->n_phase_steps += 1;
        if (s->db.rep) launch_rep_mask(s->db, R, s->st, &s->launches);     // the fused steps build their own bits
        launch_decode_step_phases(m, s->db, R, s->kcache, s->vcache, s->cache_layer_stride, s->cache_seq_stride, s->max_ctx,
                                  write_logits, s->st, &s->launches);
        launch_greedy(m, s->db, R, s->st, &s->launches);
    }
}

// end of a beam run: the finished hypotheses (filled up to K with the alive beams, "no EOS", at the cap) ranked by
// (sum / P(n) descending, admission order) with P(n) = max(n, 1), or ((5 + n) / 6) ** alpha with a length penalty, in
// double; then the kernel backtracks them and writes rank 0 into the result rows 0..B-1
static void beam_finalize(Session* s) {
    const int B = s->B, K = s->run_k;
    std::vector<BeamUtt> u((size_t)B);
    ASRB_CUDA_CHECK(cudaMemcpyAsync(u.data(), s->beam.u, B * sizeof(BeamUtt), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    std::vector<int> hyp((size_t)B * K * 2);
    std::vector<float> best_eos((size_t)B);
    s->nb_sum.assign((size_t)B * K, 0.f); s->nb_score.assign((size_t)B * K, 0.0);
    s->nb_eos.assign((size_t)B * K, -1); s->nb_n.assign((size_t)B * K, 0);
    s->beam_reassigned = s->beam_expand_bytes = s->beam_reorder_bytes = 0;
    const float nan = std::numeric_limits<float>::quiet_NaN();
    for (int b = 0; b < B; ++b) {
        const BeamUtt& x = u[b];
        struct H { int depth, slot, eos; float eos_lp, sum; double score; };
        std::vector<H> h;
        for (int f = 0; f < x.nfin && f < K; ++f) h.push_back({x.fin_depth[f], x.fin_slot[f], x.fin_eos[f], x.fin_eos_lp[f], x.fin_sum[f], 0.0});
        for (int r = 0; (int)h.size() < K; ++r) h.push_back({x.t - 1, x.slot_of_rank[r], -1, nan, x.sum_of_rank[r], 0.0});
        for (H& e : h) {
            const int n = e.depth + 1;
            const double p = s->run_alpha < 0.0 ? (double)std::max(n, 1) : std::pow((5.0 + n) / 6.0, s->run_alpha);
            e.score = (double)e.sum / p;
        }
        std::stable_sort(h.begin(), h.end(), [](const H& p, const H& q) { return p.score > q.score; });
        for (int k = 0; k < K; ++k) {
            const size_t o = (size_t)b * K + k;
            hyp[o * 2] = h[k].depth; hyp[o * 2 + 1] = h[k].slot;
            s->nb_sum[o] = h[k].sum; s->nb_score[o] = h[k].score; s->nb_eos[o] = h[k].eos; s->nb_n[o] = h[k].depth + 1;
        }
        best_eos[b] = h[0].eos_lp;
        s->beam_reassigned += x.reassigned; s->beam_expand_bytes += x.expand_bytes; s->beam_reorder_bytes += x.reorder_bytes;
    }
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_hyp, hyp.data(), hyp.size() * sizeof(int), cudaMemcpyHostToDevice, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_best_eos, best_eos.data(), best_eos.size() * sizeof(float), cudaMemcpyHostToDevice, s->st));
    launch_beam_finalize(beam_args(s), s->d_hyp, s->d_best_eos, s->st, &s->launches);
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));     // the host vectors above are pageable
    s->nbest_valid = true;
}

void session_decode_step(Session* s, int64_t* next_ids_out, float* logits) {
    ASRB_REQUIRE(s->stage >= 3, ASRB_ERR_STATE, "decode_step called before prefill");
    ASRB_REQUIRE(s->run_k == 1, ASRB_ERR_INVALID, "decode_step is not available in a beam run (beam_size > 1): use generate");
    Model& m = *s->m; const int B = s->B;
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    s->lp_valid = s->lp_valid && s->db.logprobs;
    if (s->tk_valid != s->top_k) s->tk_valid = 0;
    // the id selected by the previous greedy application is the one this iteration consumes
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_next, s->db.next_id, B * sizeof(int), cudaMemcpyDeviceToHost, s->st));
    forward_step(s, logits != nullptr);
    s->decode_steps += 1; s->greedy_done += 1;
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    if (next_ids_out) for (int b = 0; b < B; ++b) next_ids_out[b] = s->h_next[b];
    if (logits) ASRB_CUDA_CHECK(cudaMemcpy(logits, s->db.logits, (size_t)B * m.d.c.vocab_size * sizeof(float), cudaMemcpyDeviceToHost));
}

void session_generate(Session* s, int max_new_tokens, int32_t* ids_out, int32_t* lens_out) {
    ASRB_REQUIRE(s->stage >= 3, ASRB_ERR_STATE, "generate called before prefill");
    ASRB_REQUIRE(max_new_tokens >= 1 && max_new_tokens <= s->max_new, ASRB_ERR_INVALID, "max_new_tokens exceeds session capacity");
    Model& m = *s->m; const int B = s->B, R = s->nslots; cudaStream_t st = s->st;
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    s->lp_valid = s->lp_valid && (s->opt_logprobs || s->top_k > 0);   // switched off after the prefill: this run's record is incomplete
    if (s->tk_valid != s->top_k) s->tk_valid = 0;    // top_logprobs changed after the prefill: likewise
    const bool beam = s->run_k > 1;
    // finalize wrote the result rows, which are also the beam-0 slots: the search cannot resume after it
    ASRB_REQUIRE(!(beam && s->nbest_valid), ASRB_ERR_STATE, "generate: a beam run takes one generate per prefill");
    struct Restore { Session* s; bool on; ~Restore() { if (on) try { apply_record_options(s); } catch (...) {} } } restore{s, beam};
    if (beam) { s->db.topk = true; s->db.logprobs = true; }   // the search reads the records, whatever the options now say
    // Token 0 was selected at the end of prefill; each further token costs one forward + greedy.  The
    // reference also runs `forward` after the last appended token and discards its logits
    // (inference.rs:160-200); that wasted forward is not issued here.
    const int steps = std::max(0, max_new_tokens - s->greedy_done);
    auto ensure_graph = [&]() {   // per-phase path: ~142 launches per step -> replay them as one CUDA graph
        const int mode_key = (((((int)s->db.rep * 2 + (int)s->db.sample) * 2 + (int)s->db.topk) * 2 + (int)s->db.logprobs) * 2 + s->decode_mode) * (s->max_batch + 1) + R;   // unique per (rep, sample, topk, logprobs, mode, decode rows)
        if (s->step_graph == nullptr || s->graph_mode != mode_key) {
            if (s->step_graph) { cudaGraphExecDestroy(s->step_graph); s->step_graph = nullptr; }
            cudaGraph_t g = nullptr;
            int64_t before = s->launches;
            ASRB_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            try { forward_step(s, false); }
            catch (...) { cudaStreamEndCapture(st, &g); if (g) cudaGraphDestroy(g); s->launches = before; throw; }
            ASRB_CUDA_CHECK(cudaStreamEndCapture(st, &g));
            ASRB_CUDA_CHECK(cudaGraphInstantiate(&s->step_graph, g, 0));
            cudaGraphDestroy(g);
            s->graph_mode = mode_key; s->graph_B = (int)(s->launches - before);   // kernels per replay
            s->launches = before;
        }
    };
    const int check_every = 16;
    bool all_done = false;
    for (int it = 0; it < steps && !all_done; ++it) {
        // the fused step covers contexts up to 1152 keys; beyond that (long generations) the per-phase path takes over
        if (use_mega(s, false)) forward_step(s, false);
        else { ensure_graph(); ASRB_CUDA_CHECK(cudaGraphLaunch(s->step_graph, st)); s->launches += s->graph_B; }
        if (beam) { launch_beam_step(beam_args(s), false, nullptr, st, &s->launches); s->beam_steps += 1; }   // select, reorder
        s->decode_steps += 1; s->greedy_done += 1;
        if ((it + 1) % check_every == 0 && it + 1 < steps) {
            ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_done, s->db.done, R * sizeof(int), cudaMemcpyDeviceToHost, st));
            ASRB_CUDA_CHECK(cudaStreamSynchronize(st));
            all_done = true;
            for (int b = 0; b < R; ++b) all_done = all_done && s->h_done[b];
        }
    }
    if (beam) beam_finalize(s);     // result rows 0..B-1: the best hypothesis of each utterance
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_nout, s->db.n_out, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_ids, s->db.ids_out, (size_t)B * s->max_new * sizeof(int), cudaMemcpyDeviceToHost, st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b) {
        int n = std::min(s->h_nout[b], max_new_tokens);
        lens_out[b] = n;
        for (int i = 0; i < n; ++i) ids_out[(size_t)b * max_new_tokens + i] = s->h_ids[(size_t)b * s->max_new + i];
    }
}

// the stage clock of a call, ev[0] .. ev[5]: the mel (ev[1] after its H2D copy) and the encoder here, then the
// caller's two stages, closed by stage_times
static void timed_mel_encode(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* view_off) {
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[0], s->st));
    s->timing = true;
    try { mel_impl(s, samples, n_samples, batch, view_off, nullptr); } catch (...) { s->timing = false; throw; }
    s->timing = false;
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[2], s->st));
    session_encode(s, nullptr);
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[3], s->st));
}
// ev[5] recorded and waited for: last_ms[i] = ev[i] .. ev[i + 1], last_ms[5] the whole call
static void stage_times(Session* s) {
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[5], s->st));
    ASRB_CUDA_CHECK(cudaEventSynchronize(s->ev[5]));
    for (int i = 0; i < 5; ++i) ASRB_CUDA_CHECK(cudaEventElapsedTime(&s->last_ms[i], s->ev[i], s->ev[i + 1]));
    ASRB_CUDA_CHECK(cudaEventElapsedTime(&s->last_ms[5], s->ev[0], s->ev[5]));
}

static void transcribe_impl(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* view_off,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                            int32_t* ids_out, int32_t* lens_out) {
    ASRB_REQUIRE(ids_out && lens_out, ASRB_ERR_INVALID, "null output");
    if (samples == nullptr && view_off == nullptr) batch = (int)s->ingested_n.size();      // asrb_transcribe_ingested
    check_sampling_options(s, batch);
    check_context(s, batch);
    ASRB_REQUIRE(max_new_tokens >= 1 && max_new_tokens <= s->max_new, ASRB_ERR_INVALID, "max_new_tokens exceeds session capacity");
    s->launches = 0; s->decode_steps = 0;
    timed_mel_encode(s, samples, n_samples, batch, view_off);
    session_prefill(s, lang_ids, n_lang_ids, nullptr, nullptr);
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[4], s->st));
    session_generate(s, max_new_tokens, ids_out, lens_out);
    stage_times(s);
}
void session_transcribe_ids(Session* s, const float* const* samples, const int64_t* n_samples, int batch,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                            int32_t* ids_out, int32_t* lens_out) {
    transcribe_impl(s, samples, n_samples, batch, nullptr, lang_ids, n_lang_ids, max_new_tokens, ids_out, lens_out);
}

// n views [start, end) of the long-audio files as one batch (asrb_transcribe_segments, asrb_align_segments): their
// offsets in the long-audio buffer and lengths, every argument checked first
static void segment_views(const Session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                          std::vector<int64_t>& off, std::vector<int64_t>& len, const char* who) {
    const std::string w(who);
    ASRB_REQUIRE(!s->long_n.empty(), ASRB_ERR_STATE, w + ": nothing ingested with asrb_ingest_long");
    ASRB_REQUIRE(n >= 1 && n <= s->max_batch, ASRB_ERR_INVALID, w + ": n must be in [1, max_batch]");
    off.assign((size_t)n, 0); len.assign((size_t)n, 0);
    for (int i = 0; i < n; ++i) {
        const int f = file[i];
        ASRB_REQUIRE(f >= 0 && f < (int)s->long_n.size(), ASRB_ERR_INVALID, w + ": file index out of range");
        ASRB_REQUIRE(start[i] >= 0 && start[i] < end[i] && end[i] <= s->long_n[f], ASRB_ERR_INVALID,
                     w + ": need 0 <= start < end <= the file's samples");
        len[i] = end[i] - start[i];
        ASRB_REQUIRE(len[i] >= 201 && len[i] <= s->max_samples, ASRB_ERR_INVALID, w + ": a view must hold 201 .. max_samples samples");
        off[i] = s->long_off[f] + start[i];
    }
}

void session_transcribe_segments(Session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                                 const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens,
                                 int32_t* ids_out, int32_t* lens_out) {
    std::vector<int64_t> off, len;
    segment_views(s, n, file, start, end, off, len, "transcribe_segments");
    transcribe_impl(s, nullptr, len.data(), n, off.data(), lang_ids, n_lang_ids, max_new_tokens, ids_out, lens_out);
}

// -------------------------------------------------------------------------------------------------
// teacher-forced scoring (asrb_score_ids, DESIGN.md 4.8): one prefill over every candidate, flat candidates sharing
// their utterance's prompt through the K/V fan-out, then the score head over the rows that predict the given ids
// -------------------------------------------------------------------------------------------------
// device buffers taken all or none: a failed cudaMalloc frees the ones already taken and throws, and nothing of the
// session has changed; commit() hands them to the session
struct AllocAll {
    std::vector<void*> got, got_host;
    ~AllocAll() { for (void* p : got) cudaFree(p); for (void* p : got_host) cudaFreeHost(p); }
    template <typename T> T* take(size_t n, bool pinned = false) {     // pinned: host memory
        void* p = nullptr;
        if (pinned) ASRB_CUDA_CHECK(cudaMallocHost(&p, std::max<size_t>(n, 1) * sizeof(T)));
        else ASRB_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
        (pinned ? got_host : got).push_back(p);
        return static_cast<T*>(p);
    }
    void commit(Session* s) {
        s->owned.insert(s->owned.end(), got.begin(), got.end()); got.clear();
        s->owned_host.insert(s->owned_host.end(), got_host.begin(), got_host.end()); got_host.clear();
    }
};

// a scoring call's prefill of `rows` rows, `score_rows` head rows and a plan of `plan_ints` ints: every buffer is grown
// to fit first, then the old ones are released, so a failed allocation leaves the session as it was
static void ensure_score_bufs(Session* s, size_t rows, int score_rows, size_t plan_ints) {
    const Model& m = *s->m; const Dims& d = m.d; const asrb_dims& c = d.c;
    Session::ScoreBufs& b = s->sc;
    const bool act = rows > s->act_rows, head = score_rows > b.rows_cap, plan = plan_ints > b.int_cap;
    if (!act && !head && !plan) return;
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));      // the old buffers may still be read
    AllocAll a;
    float *hid = nullptr, *dqkv = nullptr, *qrot = nullptr; bf16 *dh = nullptr, *dattn = nullptr, *dact = nullptr;
    if (act) {
        hid = a.take<float>(rows * c.hidden_size); dqkv = a.take<float>(rows * d.qkv_dim); qrot = a.take<float>(rows * d.q_dim);
        dh = a.take<bf16>(3 * rows * c.hidden_size); dattn = a.take<bf16>(3 * rows * d.q_dim);
        dact = a.take<bf16>(3 * rows * c.intermediate_size);
    }
    const size_t R = std::max(score_rows, b.rows_cap);
    float *gathered = nullptr, *lp = nullptr, *tk_lp = nullptr; bf16* planes = nullptr; ScorePart* part = nullptr; int* tk_ids = nullptr;
    if (head) {
        gathered = a.take<float>(R * c.hidden_size); planes = a.take<bf16>(3 * R * c.hidden_size);
        part = a.take<ScorePart>(R * score_slices(m)); lp = a.take<float>(R);
        tk_ids = a.take<int>(R * TK_MAX); tk_lp = a.take<float>(R * TK_MAX);
    }
    int *d_int = nullptr, *h_int = nullptr;
    if (plan) { d_int = a.take<int>(plan_ints); h_int = a.take<int>(plan_ints, true); }
    // every allocation succeeded: swap in, release the old buffers
    a.commit(s);
    if (act) {
        for (void* p : {(void*)s->hid, (void*)s->dqkv, (void*)s->qrot, (void*)s->dh, (void*)s->dattn, (void*)s->dact}) release_owned(s, p);
        s->hid = hid; s->dqkv = dqkv; s->qrot = qrot; s->dh = dh; s->dattn = dattn; s->dact = dact;
        s->dh_ps = rows * c.hidden_size; s->dattn_ps = rows * d.q_dim; s->dact_ps = rows * c.intermediate_size;
        s->act_rows = rows;
    }
    if (head) {
        for (void* p : {(void*)b.gathered, (void*)b.planes, (void*)b.part, (void*)b.lp, (void*)b.tk_ids, (void*)b.tk_lp}) release_owned(s, p);
        b.gathered = gathered; b.planes = planes; b.part = part; b.lp = lp; b.tk_ids = tk_ids; b.tk_lp = tk_lp;
        b.rows_cap = (int)R;
    }
    if (plan) {
        release_owned(s, b.d_int); release_owned(s, b.h_int);
        b.d_int = d_int; b.h_int = h_int; b.int_cap = plan_ints;
    }
}

// the plan of a teacher-forced prefill (asrb_score_ids, asrb_align_ids): slot q = candidate q; the first candidate of an
// utterance leads (its prompt and its ids but the last), the others (followers) compute their ids but the last from
// position S_b on, their prompt K/V fanned out.  Grows the buffers (the score head's only with `head`).  Behind the plan,
// for each id in candidate order (candidate q's from coff[q] on): the row predicting it (src), then the ids (tgt)
static PrefillPlan plan_teacher_forced(Session* s, int B, const int64_t* const* lang_ids, const std::vector<int>& nl,
                                       const int32_t* n_cand, const int64_t* const* cand_ids, const int32_t* cand_len, int N,
                                       bool head, std::vector<int>& coff) {
    s->S.assign(B, 0);
    std::vector<PrefillSeq> seq((size_t)N);
    coff.assign(N + 1, 0);
    size_t totS = 0;
    for (int b = 0, q = 0; b < B; ++b)
        for (int j = 0; j < n_cand[b]; ++j, ++q) {
            PrefillSeq& x = seq[q];
            build_prompt(s, b, lang_ids, nl[b], x.pid, x.parow);
            s->S[b] = (int)x.pid.size();
            if (j > 0) { x.lead = q - j; x.from = s->S[b]; }
            for (int i = 0; i + 1 < cand_len[q]; ++i) { x.pid.push_back((int)cand_ids[q][i]); x.parow.push_back(-1); }
            totS += x.pid.size() - x.from;
            coff[q + 1] = coff[q] + cand_len[q];
        }
    const int R = coff[N];
    ensure_score_bufs(s, totS, head ? R : 0, 4 * totS + 7 * (size_t)N + 2 * (size_t)R);
    return plan_prefill(s, seq, s->sc.h_int, s->sc.d_int, s->sc.int_cap, 2 * R, [&](int* src, const PrefillPlan& p) {
        for (int b = 0, q = 0; b < B; ++b)
            for (int j = 0; j < n_cand[b]; ++j, ++q)
                for (int i = 0; i < cand_len[q]; ++i) {
                    const int o = i == 0 ? q - j : q;     // id i is predicted at position S_b + i - 1: the leader's for id 0
                    src[coff[q] + i] = p.srow0[o] + s->S[b] + i - 1 - seq[o].from;
                    src[R + coff[q] + i] = (int)cand_ids[q][i];
                }
    });
}

void session_score_ids(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* const* lang_ids,
                       const int32_t* n_lang_ids, const int32_t* n_cand, const int64_t* const* cand_ids, const int32_t* cand_len,
                       int max_new_tokens, float* logprob_out, int32_t* top_ids_out, float* top_lp_out) {
    ASRB_REQUIRE(logprob_out && n_cand && cand_ids && cand_len, ASRB_ERR_INVALID, "score: null argument");
    if (samples == nullptr) {
        batch = (int)s->ingested_n.size();          // asrb_score_ingested
        ASRB_REQUIRE(batch >= 1, ASRB_ERR_STATE, "score_ingested: no ingested audio");
    }
    Model& m = *s->m; const asrb_dims& c = m.d.c;
    // ---- every argument checked before any work ----
    ASRB_REQUIRE(batch >= 1 && batch <= s->max_batch, ASRB_ERR_INVALID, "score: batch exceeds session capacity");
    ASRB_REQUIRE(max_new_tokens >= 1 && max_new_tokens <= s->max_new, ASRB_ERR_INVALID, "max_new_tokens exceeds session capacity");
    check_context(s, batch);
    check_score_head(m);
    int64_t n_total = 0;
    std::vector<int> nl((size_t)batch);
    for (int b = 0; b < batch; ++b) {
        ASRB_REQUIRE(n_cand[b] >= 1, ASRB_ERR_INVALID, "score: every utterance needs at least one candidate");
        n_total += n_cand[b];
        nl[b] = lang_count(s, lang_ids, n_lang_ids, b);
    }
    ASRB_REQUIRE(n_total <= s->max_batch, ASRB_ERR_INVALID,
                 "score: " + std::to_string(n_total) + " candidates exceed the session's max_batch (one KV slot each)");
    const int N = (int)n_total;
    for (int q = 0; q < N; ++q) {
        ASRB_REQUIRE(cand_len[q] >= 1 && cand_len[q] <= max_new_tokens, ASRB_ERR_INVALID, "score: candidate length outside [1, max_new_tokens]");
        ASRB_REQUIRE(cand_ids[q], ASRB_ERR_INVALID, "score: null candidate");
        for (int i = 0; i < cand_len[q]; ++i)
            ASRB_REQUIRE(cand_ids[q][i] >= 0 && cand_ids[q][i] < c.vocab_size, ASRB_ERR_INVALID, "score: candidate id out of vocabulary");
    }
    const int k = s->top_k;
    const bool topk = k >= 1 && top_ids_out && top_lp_out;
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    cudaStream_t st = s->st;
    s->launches = 0; s->decode_steps = 0;
    s->nbest_valid = false; s->lp_valid = false; s->tk_valid = 0;
    timed_mel_encode(s, samples, n_samples, batch, nullptr);
    s->stage = 2;                                     // the KV slots are overwritten: no run to continue after this call
    std::vector<int> coff;
    const PrefillPlan pf = plan_teacher_forced(s, batch, lang_ids, nl, n_cand, cand_ids, cand_len, N, true, coff);
    const int R = coff[N];
    Session::ScoreBufs& sb = s->sc;
    prefill_layers(s, pf, s->audio);
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[4], st));
    launch_score_head(m, s->hid, pf.d_tail, pf.d_tail + R, R, sb.gathered, sb.planes, (size_t)sb.rows_cap * c.hidden_size,
                      s->nplanes, sb.part, topk, sb.lp, sb.tk_ids, sb.tk_lp, st, &s->launches);
    stage_times(s);
    std::vector<float> lp((size_t)R), tlp(topk ? (size_t)R * TK_MAX : 0);
    std::vector<int> tid(tlp.size());
    ASRB_CUDA_CHECK(cudaMemcpyAsync(lp.data(), sb.lp, lp.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (topk) {
        ASRB_CUDA_CHECK(cudaMemcpyAsync(tid.data(), sb.tk_ids, tid.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
        ASRB_CUDA_CHECK(cudaMemcpyAsync(tlp.data(), sb.tk_lp, tlp.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    ASRB_CUDA_CHECK(cudaStreamSynchronize(st));
    const float nan = std::numeric_limits<float>::quiet_NaN();
    for (int q = 0; q < N; ++q)
        for (int i = 0; i < max_new_tokens; ++i) {
            const bool in = i < cand_len[q];
            const size_t o = (size_t)q * max_new_tokens + i, r = (size_t)coff[q] + i;
            logprob_out[o] = in ? lp[r] : nan;
            if (topk)
                for (int j = 0; j < k; ++j) {
                    top_ids_out[o * k + j] = in ? tid[r * TK_MAX + j] : -1;
                    top_lp_out[o * k + j] = in ? tlp[r * TK_MAX + j] : nan;
                }
        }
}

// -------------------------------------------------------------------------------------------------
// word-timing alignment (asrb_align_ids, DESIGN.md 4.10): a teacher-forced prefill of one candidate per utterance up to
// the last listed layer, the audio-key probabilities of the listed heads folded into M as each layer passes, then DTW
// -------------------------------------------------------------------------------------------------
struct AlignHook : LayerHook {
    Session* s = nullptr;
    std::vector<int> first, count;      // per layer: its heads in the sorted list (count 0: not listed)
    int last = -1, n_heads = 0, B = 0, maxN = 0, maxT = 0, maxNT = 0;
    const int *d_heads = nullptr, *d_qrow0 = nullptr, *d_N = nullptr, *d_T = nullptr, *d_a0 = nullptr, *d_slot = nullptr;
    const long long* d_moff = nullptr;
    size_t plane = 0;
    void run(int l) override {
        if (count[l] == 0) return;
        const asrb_dims& c = s->m->d.c;
        AlignProbArgs pa{};
        pa.q = s->qrot; pa.ldq = s->m->d.q_dim;
        pa.k = s->kcache + (size_t)l * s->cache_layer_stride; pa.seg_stride = s->cache_seq_stride;
        pa.head_stride = (size_t)s->max_ctx * c.head_dim; pa.hd = c.head_dim; pa.group = c.num_attention_heads / c.num_key_value_heads;
        pa.qrow0 = d_qrow0; pa.N = d_N; pa.T = d_T; pa.a0 = d_a0; pa.slot = d_slot; pa.moff = d_moff;
        pa.heads = d_heads + first[l]; pa.nheads = count[l]; pa.P = s->al.P; pa.plane = plane;
        launch_align_probs(pa, B, maxN, s->st);
        AlignFoldArgs fa{};
        fa.N = d_N; fa.T = d_T; fa.moff = d_moff; fa.P = s->al.P; fa.plane = plane; fa.nheads = count[l]; fa.M = s->al.M;
        fa.count = l == last ? n_heads : 0;
        launch_align_fold(fa, B, maxT, maxNT, s->st);
        s->launches += 3;
    }
};

// the alignment scratch of a call: every buffer grown to fit first, then the old ones released (all or none)
static void ensure_align_bufs(Session* s, size_t p_floats, size_t m_floats, size_t trace_words, size_t start_ints) {
    Session::AlignBufs& b = s->al;
    const bool grow = p_floats > b.p_cap || m_floats > b.m_cap || trace_words > b.trace_cap || start_ints > b.start_cap;
    if (!grow) return;
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    AllocAll a;
    const size_t pc = std::max(p_floats, b.p_cap), mc = std::max(m_floats, b.m_cap);
    const size_t tc = std::max(trace_words, b.trace_cap), sc = std::max(start_ints, b.start_cap);
    float* P = a.take<float>(pc); float* M = a.take<float>(mc);
    uint32_t* trace = a.take<uint32_t>(tc); int* start = a.take<int>(sc);
    a.commit(s);
    for (void* p : {(void*)b.P, (void*)b.M, (void*)b.trace, (void*)b.start}) if (p) release_owned(s, p);
    b.P = P; b.M = M; b.trace = trace; b.start = start;
    b.p_cap = pc; b.m_cap = mc; b.trace_cap = tc; b.start_cap = sc;
}

// view_off: as transcribe_impl (asrb_align_segments); samples == view_off == nullptr: the ingested utterances
static void align_impl(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* view_off,
                       const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                       const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids,
                       int32_t* start_out, int32_t* end_out) {
    ASRB_REQUIRE(ids && n_ids && text_from && start_out && end_out, ASRB_ERR_INVALID, "align: null argument");
    const bool ingested = samples == nullptr && view_off == nullptr;
    if (ingested) {
        batch = (int)s->ingested_n.size();
        ASRB_REQUIRE(batch >= 1, ASRB_ERR_STATE, "align_ingested: no ingested audio");
    }
    Model& m = *s->m; const asrb_dims& c = m.d.c;
    // ---- every argument checked before any work ----
    ASRB_REQUIRE(batch >= 1 && batch <= s->max_batch, ASRB_ERR_INVALID, "align: batch outside [1, max_batch]");
    ASRB_REQUIRE(max_ids >= 1, ASRB_ERR_INVALID, "align: max_ids must be >= 1");
    check_context(s, batch);
    int maxn = 0;
    std::vector<int> nl((size_t)batch);
    for (int b = 0; b < batch; ++b) {
        if (!ingested && !view_off) {
            ASRB_REQUIRE(samples[b] && n_samples[b] > 0 && n_samples[b] <= s->max_samples, ASRB_ERR_INVALID, "n_samples out of session capacity");
            ASRB_REQUIRE(((n_samples[b] + 159) / 160) * 160 > 200, ASRB_ERR_INVALID, "utterance too short for reflect padding (needs > 200 samples)");
        }
        nl[b] = lang_count(s, lang_ids, n_lang_ids, b);
        const int n = n_ids[b];
        ASRB_REQUIRE(n >= 1 && n <= max_ids && n <= s->max_new, ASRB_ERR_INVALID,
                     "align: n_ids outside [1, min(max_ids, the session's max_new_tokens)]");
        ASRB_REQUIRE(ids[b], ASRB_ERR_INVALID, "align: null id row");
        for (int i = 0; i < n; ++i) ASRB_REQUIRE(ids[b][i] >= 0 && ids[b][i] < c.vocab_size, ASRB_ERR_INVALID, "align: id out of vocabulary");
        ASRB_REQUIRE(text_from[b] >= 0 && text_from[b] <= n - 1, ASRB_ERR_INVALID, "align: text_from outside [0, n_ids - 1]");
        maxn = std::max(maxn, n);
    }
    ASRB_REQUIRE(n_heads >= 0 && (n_heads == 0 || heads), ASRB_ERR_INVALID, "align: bad head list");
    std::vector<std::pair<int, int>> hs;
    if (n_heads == 0) {
        for (int l = c.num_hidden_layers / 2; l < c.num_hidden_layers; ++l)
            for (int h = 0; h < c.num_attention_heads; ++h) hs.push_back({l, h});
    } else {
        for (int k = 0; k < n_heads; ++k) {
            const int l = heads[2 * k], h = heads[2 * k + 1];
            ASRB_REQUIRE(l >= 0 && l < c.num_hidden_layers && h >= 0 && h < c.num_attention_heads, ASRB_ERR_INVALID,
                         "align: head outside the model");
            hs.push_back({l, h});
        }
        std::sort(hs.begin(), hs.end());
        ASRB_REQUIRE(std::adjacent_find(hs.begin(), hs.end()) == hs.end(), ASRB_ERR_INVALID, "align: duplicate head");
    }
    ASRB_REQUIRE(align_dtw_smem(maxn, 0, false) <= m.ctx->smem_optin, ASRB_ERR_INVALID, "align: too many ids for the DTW kernel");
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    cudaStream_t st = s->st;
    s->launches = 0; s->decode_steps = 0;
    s->nbest_valid = false; s->lp_valid = false; s->tk_valid = 0;
    s->al.N.clear(); s->al.T.clear(); s->al.moff.clear();
    timed_mel_encode(s, samples, n_samples, batch, view_off);
    s->stage = 2;                                     // the KV slots are overwritten: no run to continue after this call
    const int B = batch;
    // ---- plan: one candidate per utterance (slot b), no score head ----
    const std::vector<int32_t> ones((size_t)B, 1);
    std::vector<int> coff;
    const PrefillPlan pf = plan_teacher_forced(s, B, lang_ids, nl, ones.data(), ids, n_ids, B, false, coff);
    std::vector<int> N(B), T(B), pi(7 * (size_t)B + hs.size());
    std::vector<long long> moff(B), toff(B);
    int* qrow0 = pi.data(); int* pN = qrow0 + B; int* pT = pN + B; int* a0 = pT + B; int* slot = a0 + B; int* soff = slot + B;
    int* in_smem = soff + B; int* hl = in_smem + B;
    long long sumNT = 0, words = 0; int sumN = 0, maxN = 0, maxT = 0, maxNT = 0; size_t smem = 0;
    for (int b = 0; b < B; ++b) {
        N[b] = n_ids[b] - text_from[b]; T[b] = s->T[b];
        qrow0[b] = pf.srow0[b] + s->S[b] - 1 + text_from[b]; pN[b] = N[b]; pT[b] = T[b];
        a0[b] = audio_start((int)context_of(s, b).size()); slot[b] = b; soff[b] = sumN;
        moff[b] = sumNT; sumNT += (long long)N[b] * T[b]; sumN += N[b];
        in_smem[b] = align_dtw_smem(N[b], T[b], true) <= m.ctx->smem_optin;
        smem = std::max(smem, align_dtw_smem(N[b], T[b], in_smem[b] != 0));
        toff[b] = words; if (!in_smem[b]) words += ((long long)N[b] * T[b] + 15) / 16;
        maxN = std::max(maxN, N[b]); maxT = std::max(maxT, T[b]); maxNT = std::max(maxNT, N[b] * T[b]);
    }
    AlignHook hook;
    hook.s = s; hook.first.assign(c.num_hidden_layers, 0); hook.count.assign(c.num_hidden_layers, 0);
    int most = 0;
    for (size_t k = 0; k < hs.size(); ++k) {
        hl[k] = hs[k].second;
        if (hook.count[hs[k].first]++ == 0) hook.first[hs[k].first] = (int)k;
        most = std::max(most, hook.count[hs[k].first]);
    }
    hook.last = hs.back().first; hook.n_heads = (int)hs.size();
    ensure_align_bufs(s, (size_t)most * sumNT, (size_t)sumNT, (size_t)words, (size_t)sumN + pi.size() + 4 * (size_t)B + 2);
    // the per-utterance plan rides behind the start tokens: [sumN starts | ints | long longs (8-byte aligned)]
    Session::AlignBufs& ab = s->al;
    int* d_pi = ab.start + sumN;
    long long* d_pl = reinterpret_cast<long long*>(ab.start + ((sumN + pi.size() + 1) & ~(size_t)1));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(d_pi, pi.data(), pi.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(d_pl, moff.data(), B * sizeof(long long), cudaMemcpyHostToDevice, st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(d_pl + B, toff.data(), B * sizeof(long long), cudaMemcpyHostToDevice, st));
    ASRB_CUDA_CHECK(cudaMemsetAsync(ab.M, 0, (size_t)sumNT * sizeof(float), st));
    if (words) ASRB_CUDA_CHECK(cudaMemsetAsync(ab.trace, 0, (size_t)words * sizeof(uint32_t), st));
    hook.B = B; hook.maxN = maxN; hook.maxT = maxT; hook.maxNT = maxNT; hook.plane = (size_t)sumNT;
    hook.d_qrow0 = d_pi + (qrow0 - pi.data()); hook.d_N = d_pi + (pN - pi.data()); hook.d_T = d_pi + (pT - pi.data());
    hook.d_a0 = d_pi + (a0 - pi.data()); hook.d_slot = d_pi + (slot - pi.data()); hook.d_heads = d_pi + (hl - pi.data());
    hook.d_moff = d_pl;
    prefill_layers(s, pf, s->audio, hook.last + 1, &hook);
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[4], st));
    AlignDtwArgs da{};
    da.N = hook.d_N; da.T = hook.d_T; da.moff = d_pl; da.M = ab.M; da.smem_trace = d_pi + (in_smem - pi.data());
    da.trace = ab.trace; da.toff = d_pl + B; da.start = ab.start; da.soff = d_pi + (soff - pi.data());
    launch_align_dtw(da, B, smem, st);
    s->launches += 1;
    stage_times(s);
    std::vector<int> tok((size_t)sumN);
    ASRB_CUDA_CHECK(cudaMemcpyAsync(tok.data(), ab.start, (size_t)sumN * sizeof(int), cudaMemcpyDeviceToHost, st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(st));
    ab.N = N; ab.T = T; ab.moff = moff;
    // ---- frames: audio token t of chunk k starts at frame k * chunk_frames + 8 t ----
    const int cf = m.d.chunk_frames;
    for (int b = 0; b < B; ++b) {
        std::vector<int> frame;
        for (int k = 0; k < s->C[b]; ++k) {
            const int valid = chunk_tokens((int)std::min<int64_t>(cf, s->F[b] - (int64_t)k * cf));
            for (int t = 0; t < valid; ++t) frame.push_back(k * cf + 8 * t);
        }
        int32_t* so = start_out + (size_t)b * max_ids; int32_t* eo = end_out + (size_t)b * max_ids;
        for (int x = 0; x < max_ids; ++x) { so[x] = -1; eo[x] = -1; }
        const int f = text_from[b];
        for (int i = 0; i < N[b]; ++i) so[f + i] = frame[tok[soff[b] + i]];
        for (int i = 0; i < N[b]; ++i) eo[f + i] = i + 1 < N[b] ? so[f + i + 1] : (int32_t)s->F[b];
    }
}

void session_align_ids(Session* s, const float* const* samples, const int64_t* n_samples, int batch, const int64_t* const* lang_ids,
                       const int32_t* n_lang_ids, const int64_t* const* ids, const int32_t* n_ids, const int32_t* text_from,
                       const int32_t* heads, int n_heads, int max_ids, int32_t* start_out, int32_t* end_out) {
    align_impl(s, samples, n_samples, batch, nullptr, lang_ids, n_lang_ids, ids, n_ids, text_from, heads, n_heads, max_ids,
               start_out, end_out);
}

void session_align_segments(Session* s, int n, const int32_t* file, const int64_t* start, const int64_t* end,
                            const int64_t* const* lang_ids, const int32_t* n_lang_ids, const int64_t* const* ids,
                            const int32_t* n_ids, const int32_t* text_from, const int32_t* heads, int n_heads, int max_ids,
                            int32_t* start_out, int32_t* end_out) {
    std::vector<int64_t> off, len;
    segment_views(s, n, file, start, end, off, len, "align_segments");
    align_impl(s, nullptr, len.data(), n, off.data(), lang_ids, n_lang_ids, ids, n_ids, text_from, heads, n_heads, max_ids,
               start_out, end_out);
}

void session_last_align_dims(Session* s, int b, int32_t* n_rows, int32_t* n_tokens) {
    ASRB_REQUIRE(b >= 0 && b < (int)s->al.N.size(), ASRB_ERR_STATE, "last_align_dims: no alignment for this index");
    if (n_rows) *n_rows = s->al.N[b];
    if (n_tokens) *n_tokens = s->al.T[b];
}

void session_align_matrix_read(Session* s, int b, float* out) {
    ASRB_REQUIRE(b >= 0 && b < (int)s->al.N.size(), ASRB_ERR_STATE, "align_matrix_read: no alignment for this index");
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    ASRB_CUDA_CHECK(cudaMemcpy(out, s->al.M + s->al.moff[b], (size_t)s->al.N[b] * s->al.T[b] * sizeof(float), cudaMemcpyDeviceToHost));
}

// -------------------------------------------------------------------------------------------------
// streaming (asrb_stream_*, DESIGN.md 4.9): stream b in KV slot b; per push the mel of its new frames, the encoder over
// the windows whose clamped mel may have changed, and the prefill from the first position those change
// -------------------------------------------------------------------------------------------------
static int stream_win_frames(const Session* s) {     // frames of one encoder window (the whole stream without windows)
    const Dims& d = s->m->d;
    return d.chunks_per_window > 0 ? d.chunk_frames * d.chunks_per_window : s->maxF;
}

static void stream_clear(Session* s, int b) {
    Session::Stream& x = s->streams[b];
    x = Session::Stream();
    x.ctx = context_of(s, b);                        // latched when the stream starts
    x.win_phi.assign(s->str_maxW, 0.f); x.win_final.assign(s->str_maxW, 0);
    float* row = s->h_str_stats + (size_t)b * s->str_stats_ld;
    row[0] = -INFINITY; row[1] = -INFINITY;
    for (int w = 0; w < s->str_maxW; ++w) row[2 + w] = INFINITY;
    ASRB_CUDA_CHECK(cudaMemcpy(s->str_stats + (size_t)b * s->str_stats_ld, row, s->str_stats_ld * sizeof(float), cudaMemcpyHostToDevice));
}

void session_stream_open(Session* s, int n_streams, int rollback, int unfixed) {
    ASRB_REQUIRE(n_streams >= 1 && n_streams <= s->max_batch, ASRB_ERR_INVALID, "stream_open: n_streams must be in [1, max_batch]");
    ASRB_REQUIRE(rollback >= 0 && unfixed >= 0, ASRB_ERR_INVALID, "stream_open: rollback_ids and unfixed_pushes must be >= 0");
    check_context(s, n_streams);
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    s->streams_open = false;
    if (!s->str_samples) {
        const Dims& d = s->m->d; const size_t Bm = s->max_batch;
        const int cpw = d.chunks_per_window;
        s->str_maxW = cpw > 0 ? (s->maxC + cpw - 1) / cpw : 1;
        s->str_stats_ld = 2 + s->str_maxW;
        s->str_int_cap = 8 * Bm + 4 * Bm * s->str_maxW + 16;
        AllocAll a;
        float* smp = a.take<float>(Bm * s->max_npad);
        float* raw = a.take<float>(Bm * d.c.num_mel_bins * s->maxF);
        float* tok = a.take<float>(Bm * s->maxT * d.c.output_dim);
        float* stats = a.take<float>(Bm * s->str_stats_ld);
        int* pi = a.take<int>(s->str_int_cap);
        float* hs = a.take<float>(Bm * s->str_stats_ld, true);
        int* hi = a.take<int>(s->str_int_cap, true);
        a.commit(s);
        s->str_samples = smp; s->str_raw = raw; s->str_tok = tok; s->str_stats = stats; s->str_int = pi;
        s->h_str_stats = hs; s->h_str_int = hi;
    }
    s->str_rollback = rollback; s->str_unfixed = unfixed;
    s->streams.assign(n_streams, Session::Stream());
    for (int b = 0; b < n_streams; ++b) stream_clear(s, b);
    for (auto& v : s->str_counts) v = 0;
    s->streams_open = true;
}

void session_stream_reset(Session* s, int b) {
    ASRB_REQUIRE(s->streams_open, ASRB_ERR_STATE, "stream_reset: no open streams");
    ASRB_REQUIRE(b >= 0 && b < (int)s->streams.size(), ASRB_ERR_INVALID, "stream_reset: no such stream");
    check_context(s, (int)s->streams.size());
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    stream_clear(s, b);
}

void session_stream_push(Session* s, int nst, const float* const* samples, const int64_t* n_samples, const int32_t* is_final,
                         const int64_t* const* lang_ids, const int32_t* n_lang_ids, int max_new_tokens, int max_ids,
                         int32_t* hyp_out, int32_t* hyp_len_out, int32_t* fixed_len_out) {
    ASRB_REQUIRE(s->streams_open, ASRB_ERR_STATE, "stream_push: no open streams (a non-stream call ends them)");
    ASRB_REQUIRE(nst == (int)s->streams.size(), ASRB_ERR_INVALID, "stream_push: n_streams differs from asrb_stream_open's");
    ASRB_REQUIRE(n_samples && hyp_out && hyp_len_out && fixed_len_out, ASRB_ERR_INVALID, "stream_push: null argument");
    ASRB_REQUIRE(s->beam_k == 1, ASRB_ERR_INVALID, "stream_push: beam_size > 1 is not available on streams (streams own their slots)");
    check_sampling_options(s, nst);
    ASRB_REQUIRE(max_new_tokens >= 1 && max_new_tokens <= s->max_new, ASRB_ERR_INVALID, "max_new_tokens exceeds session capacity");
    Model& m = *s->m; const Dims& d = m.d; const asrb_dims& c = d.c;
    const int cf = d.chunk_frames, cpw = d.chunks_per_window, od = c.output_dim;
    const int Wf = stream_win_frames(s), Bm = s->max_batch;
    // ---- every argument checked before any work ----
    std::vector<char> act((size_t)nst, 0), fin((size_t)nst, 0);
    std::vector<int> nl((size_t)nst, 0);
    int n_act = 0;
    for (int b = 0; b < nst; ++b) {
        const Session::Stream& x = s->streams[b];
        const int64_t nb = n_samples[b];
        fin[b] = is_final && is_final[b];
        act[b] = nb > 0 || fin[b];
        ASRB_REQUIRE(nb >= 0 && (nb == 0 || (samples && samples[b])), ASRB_ERR_INVALID, "stream_push: bad samples");
        ASRB_REQUIRE((int)x.hyp.size() <= max_ids, ASRB_ERR_INVALID, "stream_push: max_ids is below a stream's hypothesis");
        if (!act[b]) continue;
        ++n_act;
        ASRB_REQUIRE(!x.closed, ASRB_ERR_STATE, "stream_push: stream " + std::to_string(b) + " is closed (asrb_stream_reset reopens it)");
        ASRB_REQUIRE(x.n + nb <= s->max_samples, ASRB_ERR_INVALID, "stream_push: samples past the session's max_samples");
        ASRB_REQUIRE(((x.n + nb + 159) / 160) * 160 > 200, ASRB_ERR_INVALID, "stream_push: a stream needs > 160 samples before its first push");
        nl[b] = lang_count(s, lang_ids, n_lang_ids, b, (int)x.p.size(),
                           "stream_push: language ids + forced prefix exceed the session's max_lang_ids");
        ASRB_REQUIRE((int)x.p.size() + max_new_tokens <= max_ids, ASRB_ERR_INVALID, "stream_push: max_ids < forced prefix + max_new_tokens");
    }
    ASRB_CUDA_CHECK(cudaSetDevice(m.ctx->device));
    cudaStream_t st = s->st;
    for (auto& v : s->str_counts) v = 0;
    auto write_out = [&]() {
        for (int b = 0; b < nst; ++b) {
            const Session::Stream& x = s->streams[b];
            for (size_t i = 0; i < x.hyp.size(); ++i) hyp_out[(size_t)b * max_ids + i] = x.hyp[i];
            hyp_len_out[b] = (int32_t)x.hyp.size(); fixed_len_out[b] = x.fixed;
        }
    };
    if (n_act == 0) { write_out(); return; }
    ASRB_CUDA_CHECK(cudaStreamSynchronize(st));     // the pinned plan buffers below may still feed an earlier copy
    s->launches = 0; s->decode_steps = 0; s->stream_run = false; s->nbest_valid = false;
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[0], st));
    // ---- samples, then the mel of frames [Ffin, F) and the fold of the frames that became final ----
    std::vector<int> F((size_t)nst, 0), Ffin((size_t)nst, 0);
    int4* fold = reinterpret_cast<int4*>(s->h_str_int);
    int* ffirst = s->h_str_int + 4 * Bm;
    int64_t* h = s->h_i64;
    int max_new_frames = 0;
    for (int b = 0; b < nst; ++b) {
        Session::Stream& x = s->streams[b];
        const int64_t n = x.n + n_samples[b], np = ((n + 159) / 160) * 160;
        if (n_samples[b] > 0)
            ASRB_CUDA_CHECK(cudaMemcpyAsync(s->str_samples + (size_t)b * s->max_npad + x.n, samples[b], n_samples[b] * sizeof(float),
                                            cudaMemcpyHostToDevice, st));
        F[b] = act[b] ? (int)(np / 160) : 0;
        // frame f reads samples [160 f - 200, 160 f + 200): final once 160 f + 200 <= n, whatever arrives later
        Ffin[b] = !act[b] ? 0 : fin[b] ? F[b] : (int)std::min<int64_t>(F[b], n >= 200 ? (n - 200) / 160 + 1 : 0);
        h[b] = (int64_t)b * s->max_npad; h[Bm + b] = act[b] ? n : 0; h[2 * Bm + b] = act[b] ? np : 0; h[3 * Bm + b] = (int64_t)b * s->maxF;
        ffirst[b] = act[b] ? x.Ffin : 0;
        fold[b] = make_int4(x.Ffin, Ffin[b], F[b], act[b]);
        if (act[b]) { x.n = n; max_new_frames = std::max(max_new_frames, F[b] - x.Ffin); }
    }
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_i64, h, 4 * Bm * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->str_int, s->h_str_int, 5 * Bm * sizeof(int), cudaMemcpyHostToDevice, st));
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[1], st));
    launch_mel_stream(m, s->str_samples, s->d_i64, s->d_i64 + Bm, s->d_i64 + 2 * Bm, s->d_i64 + 3 * Bm, s->str_int + 4 * Bm, nst,
                      max_new_frames, s->maxF, s->str_raw, reinterpret_cast<const int4*>(s->str_int), Wf, s->str_stats,
                      s->str_stats_ld, st);
    s->launches += max_new_frames > 0 ? 2 : 1;
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_str_stats, s->str_stats, (size_t)nst * s->str_stats_ld * sizeof(float), cudaMemcpyDeviceToHost, st));
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[2], st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(st));
    // ---- the reuse rule: which windows are encoded again, and from which prompt position the decoder recomputes ----
    struct Utt { int slot, w, f0, frames, tok0; float phi; };
    std::vector<Utt> utts;
    std::vector<int> P((size_t)nst, 0), T((size_t)nst, 0);
    for (int b = 0; b < nst; ++b) {
        if (!act[b]) continue;
        Session::Stream& x = s->streams[b];
        const float* row = s->h_str_stats + (size_t)b * s->str_stats_ld;
        const float phi = fmaxf(row[0], row[1]) - 8.0f;       // = mel_finalize_kernel's floor of the offline mel of x[0..n)
        const int C = (F[b] + cf - 1) / cf, W = cpw > 0 ? (C + cpw - 1) / cpw : 1;
        int first_re = W, tok = 0, tok_re = -1;   // tok_re: first token of the first re-encoded window
        for (int w = 0; w < W; ++w) {
            const int f0 = w * Wf, f1 = std::min(F[b], (w + 1) * Wf);
            int wt = 0;
            for (int k = f0 / cf; k * cf < f1; ++k) wt += chunk_tokens(std::min(cf, F[b] - k * cf));
            const bool finished = f1 <= Ffin[b];
            const bool was_final = x.win_final[w];
            const bool floor_ok = phi == x.win_phi[w] || row[2 + w] >= fmaxf(phi, x.win_phi[w]);
            if (finished && was_final && floor_ok) s->str_counts[1] += 1;
            else {
                if (finished && was_final) s->str_counts[2] += 1;
                utts.push_back({b, w, f0, f1 - f0, tok, phi});
                x.win_phi[w] = phi; x.win_final[w] = finished;
                first_re = std::min(first_re, w);
            }
            if (w == first_re && tok_re < 0) tok_re = tok;
            tok += wt;
        }
        T[b] = tok;
        x.phi = phi; x.Ffin = Ffin[b]; x.T = tok;
        // P_b: head, context and the pads of the windows before the first re-encoded one (0 before the first prefill)
        P[b] = std::min(audio_start((int)x.ctx.size()) + (tok_re < 0 ? tok : tok_re), x.kv_valid);
    }
    s->str_counts[0] = (int64_t)utts.size();
    // ---- encoder: the re-encoded windows as pseudo-utterances of at most one window each, in waves of max_batch ----
    int4* stage = reinterpret_cast<int4*>(s->h_str_int + 8 * Bm);
    for (size_t u = 0; u < utts.size(); ++u) {
        int phi_bits; memcpy(&phi_bits, &utts[u].phi, sizeof(phi_bits));
        stage[u] = make_int4(utts[u].slot, utts[u].f0, utts[u].frames, phi_bits);
    }
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->str_int + 8 * Bm, stage, utts.size() * sizeof(int4), cudaMemcpyHostToDevice, st));
    for (size_t w0 = 0; w0 < utts.size(); w0 += Bm) {
        const int nu = (int)std::min<size_t>(Bm, utts.size() - w0);
        if (w0 > 0) ASRB_CUDA_CHECK(cudaStreamSynchronize(st));      // the pinned plans of the previous wave
        s->B = nu;
        s->F.assign(nu, 0); s->foff.assign(nu, 0);
        int64_t fo = 0;
        for (int u = 0; u < nu; ++u) {
            s->F[u] = utts[w0 + u].frames; s->foff[u] = fo; fo += s->F[u];
            h[3 * Bm + u] = s->foff[u]; h[4 * Bm + u] = s->F[u];
        }
        ASRB_CUDA_CHECK(cudaMemcpyAsync(s->d_i64, h, 5 * Bm * sizeof(int64_t), cudaMemcpyHostToDevice, st));
        launch_mel_stream_stage(m, s->str_raw, reinterpret_cast<const int4*>(s->str_int + 8 * Bm) + w0, s->d_i64 + 3 * Bm, nu,
                                s->maxF, s->d_mel, st);
        s->launches += 1;
        s->stage = 1;
        session_encode(s, nullptr);
        for (int u = 0; u < nu; ++u) {
            const Utt& q = utts[w0 + u];
            ASRB_CUDA_CHECK(cudaMemcpyAsync(s->str_tok + ((size_t)q.slot * s->maxT + q.tok0) * od, s->audio + (size_t)s->toff[u] * od,
                                            (size_t)s->T[u] * od * sizeof(float), cudaMemcpyDeviceToDevice, st));
        }
    }
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[3], st));
    // ---- prefill: stream b's rows from position P_b on, attending to the K/V its slot keeps below P_b ----
    const int B = nst;
    s->B = B; s->run_k = 1; s->run_alpha = -1.0; s->nslots = B;
    s->S.assign(B, 0); s->maxlenS = 0;
    std::vector<PrefillSeq> seq((size_t)B);
    int64_t kept = 0;
    for (int b = 0; b < B; ++b) {
        const Session::Stream& x = s->streams[b];
        seq[b].lead = b;                                          // its slot keeps positions [0, from)
        s->maxlenS = std::max(s->maxlenS, x.kv_valid + 1);       // an idle row's decode position (below)
        if (!act[b]) continue;
        build_prompt(x.ctx, T[b], b * s->maxT, nl[b] > 0 ? lang_ids[b] : nullptr, nl[b], x.p, seq[b].pid, seq[b].parow);
        seq[b].from = P[b]; kept += P[b];
        s->S[b] = (int)seq[b].pid.size(); s->maxlenS = std::max(s->maxlenS, s->S[b]);
    }
    // idle: no rows, done.  The batched decode step still writes a done row's K/V at its position: kv_valid, the first
    // position the stream's next prefill recomputes
    const PrefillPlan pf = plan_prefill(s, seq, s->h_int + s->enc_int_cap, s->d_int + s->enc_int_cap, s->int_cap - s->enc_int_cap,
                                        3 * B, [&](int* t, const PrefillPlan& p) {   // lastrow | pos0 | done0
        for (int b = 0; b < B; ++b) {
            t[b] = act[b] ? p.srow0[b] + s->S[b] - P[b] - 1 : 0;
            t[B + b] = act[b] ? s->S[b] - 1 : s->streams[b].kv_valid;
            t[2 * B + b] = !act[b];
        }
    });
    s->str_counts[3] = pf.totS; s->str_counts[4] = kept;
    begin_run(s, B, pf.d_tail);
    prefill_layers(s, pf, s->str_tok);
    first_token(s, B, false, nullptr);
    s->stage = 3;
    ASRB_CUDA_CHECK(cudaEventRecord(s->ev[4], st));
    // ---- decode: the offline batch's paths; idle streams are done from the start ----
    std::vector<int32_t> g((size_t)B * max_new_tokens), glen((size_t)B);
    session_generate(s, max_new_tokens, g.data(), glen.data());
    stage_times(s);
    s->stream_run = true;
    // ---- hypotheses and the next forced prefixes ----
    for (int b = 0; b < B; ++b) {
        if (!act[b]) continue;
        Session::Stream& x = s->streams[b];
        x.kv_valid = audio_start((int)x.ctx.size()) + T[b];
        std::vector<int> hyp = x.p;
        hyp.insert(hyp.end(), g.begin() + (size_t)b * max_new_tokens, g.begin() + (size_t)b * max_new_tokens + glen[b]);
        if (fin[b]) { x.p = hyp; x.closed = true; }
        else if (x.k + 1 >= s->str_unfixed) x.p.assign(hyp.begin(), hyp.begin() + std::max(0, (int)hyp.size() - s->str_rollback));
        else x.p.clear();
        x.fixed = (int)x.p.size(); x.hyp = std::move(hyp); x.k += 1;
    }
    write_out();
}

// the stream's mel after its last push: bitwise asrb_mel of its samples ([n_mels][F])
void session_stream_mel_read(Session* s, int b, float* out) {
    ASRB_REQUIRE(s->streams_open && b >= 0 && b < (int)s->streams.size() && s->streams[b].n > 0, ASRB_ERR_STATE,
                 "stream_mel_read: no pushed audio on this stream");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    const Session::Stream& x = s->streams[b];
    const int nm = s->m->d.c.num_mel_bins, F = (int)((x.n + 159) / 160);
    ASRB_CUDA_CHECK(cudaMemcpy2D(out, F * sizeof(float), s->str_raw + (size_t)b * nm * s->maxF, s->maxF * sizeof(float),
                                 F * sizeof(float), nm, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < (size_t)nm * F; ++i) out[i] = (std::max(out[i], x.phi) + 4.0f) / 4.0f;   // mel_finalize_kernel
}

void session_stream_encode_read(Session* s, int b, float* out) {
    ASRB_REQUIRE(s->streams_open && b >= 0 && b < (int)s->streams.size() && s->streams[b].n > 0, ASRB_ERR_STATE,
                 "stream_encode_read: no pushed audio on this stream");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    const int od = s->m->d.c.output_dim;
    ASRB_CUDA_CHECK(cudaMemcpy(out, s->str_tok + (size_t)b * s->maxT * od, (size_t)s->streams[b].T * od * sizeof(float),
                               cudaMemcpyDeviceToHost));
}

// [0] windows encoded  [1] windows reused  [2] windows re-encoded because the floor moved  [3] prompt rows computed
// [4] prompt rows kept from earlier pushes; over the streams of the last push
void session_last_stream_stats(Session* s, int64_t* out, int n) {
    for (int i = 0; i < n && i < 5; ++i) out[i] = s->str_counts[i];
}

void session_last_timings(Session* s, float* ms6, int64_t* kernels, int64_t* steps) {
    if (ms6) for (int i = 0; i < 6; ++i) ms6[i] = s->last_ms[i];
    if (kernels) *kernels = s->launches;
    if (steps) *steps = s->decode_steps;
}

void session_device_ids(Session* s, const int32_t** ids, const int32_t** lens, int* stride, int* batch) {
    ASRB_REQUIRE(s->stage >= 3, ASRB_ERR_STATE, "device_ids: nothing generated yet");
    *ids = s->db.ids_out; *lens = s->db.n_out; *stride = s->max_new; *batch = s->B;
}

// log-probabilities of the last run (prefill + generate / decode steps): [batch][max_new_tokens], NaN at and beyond the
// sequence's length; eos_out[b] = that of the EOS token that ended sequence b, NaN if it did not end on EOS
void session_last_logprobs(Session* s, int max_new_tokens, float* out, float* eos_out) {
    ASRB_REQUIRE(s->stage >= 3 && s->lp_valid, ASRB_ERR_STATE,
                 "last_logprobs: the last run did not record log-probabilities (set option logprobs=1 before the prefill)");
    ASRB_REQUIRE(max_new_tokens >= 1, ASRB_ERR_INVALID, "max_new_tokens must be >= 1");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    const int B = s->B;
    std::vector<float> lp((size_t)B * s->max_new), eos((size_t)B);
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_nout, s->db.n_out, B * sizeof(int), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(lp.data(), s->db.lp_out, lp.size() * sizeof(float), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(eos.data(), s->db.eos_lp, eos.size() * sizeof(float), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    const float nan = std::numeric_limits<float>::quiet_NaN();
    for (int b = 0; b < B; ++b) {
        const int n = std::min(s->h_nout[b], max_new_tokens);
        for (int i = 0; i < max_new_tokens; ++i) out[(size_t)b * max_new_tokens + i] = i < n ? lp[(size_t)b * s->max_new + i] : nan;
        if (eos_out) eos_out[b] = eos[b];
    }
}

// top-k alternatives of the last run: [batch][max_new_tokens][k] ids and log-probabilities, best first, -1 / NaN at and
// beyond the sequence's length; eos rows [batch][k] those of the step that selected the EOS ending sequence b
void session_last_top_logprobs(Session* s, int max_new_tokens, int k, int32_t* ids_out, float* lp_out, int32_t* eos_ids_out,
                               float* eos_lp_out) {
    ASRB_REQUIRE(s->stage >= 3 && s->tk_valid > 0, ASRB_ERR_STATE,
                 "last_top_logprobs: the last run did not record alternatives (set option top_logprobs before the prefill)");
    ASRB_REQUIRE(max_new_tokens >= 1, ASRB_ERR_INVALID, "max_new_tokens must be >= 1");
    ASRB_REQUIRE(k >= 1 && k <= s->tk_valid, ASRB_ERR_INVALID, "k must be in [1, top_logprobs of the last run]");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    const int B = s->B;
    std::vector<int32_t> ids((size_t)B * s->max_new * TK_MAX), eids((size_t)B * TK_MAX);
    std::vector<float> lp(ids.size()), elp(eids.size());
    ASRB_CUDA_CHECK(cudaMemcpyAsync(s->h_nout, s->db.n_out, B * sizeof(int), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(ids.data(), s->db.tk_ids, ids.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(lp.data(), s->db.tk_lp, lp.size() * sizeof(float), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(eids.data(), s->db.tk_eos_ids, eids.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaMemcpyAsync(elp.data(), s->db.tk_eos_lp, elp.size() * sizeof(float), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    const float nan = std::numeric_limits<float>::quiet_NaN();
    for (int b = 0; b < B; ++b) {
        const int n = std::min(s->h_nout[b], max_new_tokens);
        for (int i = 0; i < max_new_tokens; ++i)
            for (int j = 0; j < k; ++j) {
                const size_t o = ((size_t)b * max_new_tokens + i) * k + j, src = ((size_t)b * s->max_new + i) * TK_MAX + j;
                ids_out[o] = i < n ? ids[src] : -1;
                lp_out[o] = i < n ? lp[src] : nan;
            }
        for (int j = 0; j < k; ++j) {
            if (eos_ids_out) eos_ids_out[(size_t)b * k + j] = eids[(size_t)b * TK_MAX + j];
            if (eos_lp_out) eos_lp_out[(size_t)b * k + j] = elp[(size_t)b * TK_MAX + j];
        }
    }
}

void session_stats(Session* s, int64_t* out, int n) {
    unsigned long long hq[4] = {0, 0, 0, 0};
    if (n > 5 && s->mega.hq_stats) {
        ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
        ASRB_CUDA_CHECK(cudaMemcpyAsync(hq, s->mega.hq_stats, sizeof(hq), cudaMemcpyDeviceToHost, s->st));
        ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    }
    const int64_t v[8] = {s->n_batch_steps, s->n_mega_steps, s->n_phase_steps, g_gemm_simt_fallbacks.load(), g_gemm_tc_launches.load(),
                          (int64_t)hq[1], (int64_t)hq[2], (int64_t)hq[3]};
    for (int i = 0; i < n && i < 8; ++i) out[i] = v[i];
}

// ranked hypotheses of the last beam run: ids [batch][k][max_new_tokens] (-1 beyond the length), lens / sums / scores /
// EOS ids (-1: stopped by the cap) [batch][k]
void session_last_nbest(Session* s, int max_new_tokens, int k, int32_t* ids_out, int32_t* lens_out, float* sum_out,
                        float* score_out, int32_t* eos_out) {
    ASRB_REQUIRE(s->stage >= 3 && s->nbest_valid, ASRB_ERR_STATE, "last_nbest: the last run was not a beam run");
    ASRB_REQUIRE(max_new_tokens >= 1, ASRB_ERR_INVALID, "max_new_tokens must be >= 1");
    ASRB_REQUIRE(k >= 1 && k <= s->run_k, ASRB_ERR_INVALID, "k must be in [1, beam_size of the last run]");
    ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
    const int B = s->B, K = s->run_k;
    std::vector<int32_t> ids((size_t)B * K * s->max_new);
    ASRB_CUDA_CHECK(cudaMemcpyAsync(ids.data(), s->beam.nb_ids, ids.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s->st));
    ASRB_CUDA_CHECK(cudaStreamSynchronize(s->st));
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < k; ++j) {
            const size_t o = (size_t)b * K + j, d = (size_t)b * k + j;
            const int n = std::min(s->nb_n[o], max_new_tokens);
            if (ids_out)
                for (int i = 0; i < max_new_tokens; ++i) ids_out[d * max_new_tokens + i] = i < n ? ids[o * s->max_new + i] : -1;
            if (lens_out) lens_out[d] = n;
            if (sum_out) sum_out[d] = s->nb_sum[o];
            if (score_out) score_out[d] = (float)s->nb_score[o];
            if (eos_out) eos_out[d] = s->nb_eos[o];
        }
}

// [0] beam steps  [1] slots reassigned  [2] KV bytes copied by the expansion  [3] KV bytes copied by reorders
void session_last_beam_stats(Session* s, int64_t* out, int n) {
    ASRB_REQUIRE(s->nbest_valid, ASRB_ERR_STATE, "last_beam_stats: the last run was not a beam run");
    const int64_t v[4] = {s->beam_steps, s->beam_reassigned, s->beam_expand_bytes, s->beam_reorder_bytes};
    for (int i = 0; i < n && i < 4; ++i) out[i] = v[i];
}

// options "logprobs" / "top_logprobs" / "beam_size" -> kernel variants; buffers are allocated when first needed, so a
// session that never records keeps its allocations unchanged.  Beam search reads the TOPK records.
static void apply_record_options(Session* s) {
    DecodeBufs& b = s->db;
    b.logprobs = s->opt_logprobs || s->top_k > 0 || s->beam_k > 1;   // the candidates' values need the selected token's log-probability
    b.topk = s->top_k > 0 || s->beam_k > 1;
    if (b.logprobs && !b.lp_out) {
        ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
        b.part_sum = salloc<float>(s, (size_t)s->max_batch * b.n_part);
        b.lp_out = salloc<float>(s, (size_t)s->max_batch * s->max_new);
        b.eos_lp = salloc<float>(s, s->max_batch);
    }
    if (b.topk && !b.tk_ids) {
        ASRB_CUDA_CHECK(cudaSetDevice(s->m->ctx->device));
        b.tk_part_val = salloc<float>(s, (size_t)s->max_batch * b.n_part * TK_MAX);
        b.tk_part_idx = salloc<int>(s, (size_t)s->max_batch * b.n_part * TK_MAX);
        b.tk_ids = salloc<int>(s, (size_t)s->max_batch * s->max_new * TK_MAX);
        b.tk_lp = salloc<float>(s, (size_t)s->max_batch * s->max_new * TK_MAX);
        b.tk_eos_ids = salloc<int>(s, (size_t)s->max_batch * TK_MAX);
        b.tk_eos_lp = salloc<float>(s, (size_t)s->max_batch * TK_MAX);
    }
    ensure_sample_bufs(s);                           // logprobs switched on during a sampled run
}

// option values: a decimal temperature, 0 or a finite value in [1e-6, 100]; a decimal unsigned 64-bit seed.  The whole
// string must be consumed, with no sign or leading space.
static double parse_temperature(const std::string& v) {
    ASRB_REQUIRE(!v.empty() && (isdigit((unsigned char)v[0]) || v[0] == '.') &&
                 v.find_first_not_of("0123456789.eE+-") == std::string::npos,
                 ASRB_ERR_INVALID, "temperature must be a decimal number");   // no sign, space, hex, inf or nan
    errno = 0;
    char* end = nullptr;
    const double t = strtod(v.c_str(), &end);
    ASRB_REQUIRE(end && *end == '\0' && errno == 0 && std::isfinite(t), ASRB_ERR_INVALID, "temperature must be a decimal number");
    ASRB_REQUIRE(t == 0.0 || (t >= 1e-6 && t <= 100.0), ASRB_ERR_INVALID, "temperature must be 0 or in [1e-6, 100]");
    return t;
}
static double parse_length_penalty(const std::string& v) {     // "none" is handled by the caller
    ASRB_REQUIRE(!v.empty() && (isdigit((unsigned char)v[0]) || v[0] == '.') &&
                 v.find_first_not_of("0123456789.eE+-") == std::string::npos,
                 ASRB_ERR_INVALID, "length_penalty must be none or a decimal number");
    errno = 0;
    char* end = nullptr;
    const double a = strtod(v.c_str(), &end);
    ASRB_REQUIRE(end && *end == '\0' && errno == 0 && std::isfinite(a) && a >= 0.0 && a <= 10.0, ASRB_ERR_INVALID,
                 "length_penalty must be none or a decimal in [0, 10]");
    return a;
}
// repetition controls: N a decimal integer in 0..16; the penalty a decimal in [1, 10], parsed in double
static int parse_ngram(const std::string& v) {
    ASRB_REQUIRE(!v.empty() && v.size() <= 2 && v.find_first_not_of("0123456789") == std::string::npos, ASRB_ERR_INVALID,
                 "no_repeat_ngram_size must be 0..16");
    const int n = atoi(v.c_str());
    ASRB_REQUIRE(n >= 0 && n <= 16, ASRB_ERR_INVALID, "no_repeat_ngram_size must be 0..16");
    return n;
}
static double parse_rep_penalty(const std::string& v) {
    ASRB_REQUIRE(!v.empty() && (isdigit((unsigned char)v[0]) || v[0] == '.') &&
                 v.find_first_not_of("0123456789.eE+-") == std::string::npos,
                 ASRB_ERR_INVALID, "repetition_penalty must be a decimal number");   // no sign, space, hex, inf or nan
    errno = 0;
    char* end = nullptr;
    const double t = strtod(v.c_str(), &end);
    ASRB_REQUIRE(end && *end == '\0' && errno == 0 && std::isfinite(t) && t >= 1.0 && t <= 10.0, ASRB_ERR_INVALID,
                 "repetition_penalty must be a decimal in [1, 10]");
    return t;
}
static uint64_t parse_seed(const std::string& v) {
    ASRB_REQUIRE(!v.empty() && isdigit((unsigned char)v[0]), ASRB_ERR_INVALID, "seed must be a decimal unsigned 64-bit integer");
    errno = 0;
    char* end = nullptr;
    const unsigned long long x = strtoull(v.c_str(), &end, 10);
    ASRB_REQUIRE(end && *end == '\0' && errno == 0, ASRB_ERR_INVALID, "seed must be a decimal unsigned 64-bit integer");
    return (uint64_t)x;
}

void session_set_option(Session* s, const char* key, const char* value) {
    std::string k(key ? key : ""), v(value ? value : "");
    if (s->step_graph) { cudaGraphExecDestroy(s->step_graph); s->step_graph = nullptr; s->graph_mode = -1; }   // captured with the old options
    if (k == "gemm") {
        if (v == "tc") s->gemm_impl = GEMM_TC; else if (v == "simt") s->gemm_impl = GEMM_SIMT;
        else throw Error(ASRB_ERR_INVALID, "gemm must be tc|simt");
    } else if (k == "decode") {
        if (v == "mega") s->decode_mode = 1; else if (v == "phases") s->decode_mode = 0;
        else throw Error(ASRB_ERR_INVALID, "decode must be mega|phases");
    } else if (k == "batch_step") {
        s->batch_step = (v == "1");
    } else if (k == "planes") {
        int p = atoi(v.c_str());
        ASRB_REQUIRE(p >= 1 && p <= 3, ASRB_ERR_INVALID, "planes must be 1..3");
        s->nplanes = p;
    } else if (k == "resident") {
        s->resident = (v == "1");
    } else if (k == "logprobs") {
        ASRB_REQUIRE(v == "1" || v == "0", ASRB_ERR_INVALID, "logprobs must be 1|0");
        s->opt_logprobs = (v == "1");
        apply_record_options(s);
    } else if (k == "top_logprobs") {
        ASRB_REQUIRE(v.size() == 1 && v[0] >= '0' && v[0] < '0' + 1 + TK_MAX, ASRB_ERR_INVALID, "top_logprobs must be 0..8");
        s->top_k = v[0] - '0';
        apply_record_options(s);
    } else if (k == "temperature") {
        s->temperature = parse_temperature(v);
    } else if (k == "seed") {
        s->seed = parse_seed(v);
    } else if (k == "beam_size") {
        ASRB_REQUIRE(v.size() == 1 && v[0] >= '1' && v[0] <= '0' + BEAM_MAX, ASRB_ERR_INVALID, "beam_size must be 1..6");
        s->beam_k = v[0] - '0';
        apply_record_options(s);
    } else if (k == "length_penalty") {
        s->length_penalty = v == "none" ? -1.0 : parse_length_penalty(v);
    } else if (k == "no_repeat_ngram_size") {
        s->ngram = parse_ngram(v);
    } else if (k == "repetition_penalty") {
        s->rep_penalty = parse_rep_penalty(v);
    } else throw Error(ASRB_ERR_INVALID, "unknown option: " + k);
}

}  // namespace asrb
