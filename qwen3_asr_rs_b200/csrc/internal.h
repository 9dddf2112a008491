// internal.h -- host-side structures and kernel launch prototypes (not part of the ABI).
#pragma once
#include <atomic>
#include <map>
#include <string>
#include <vector>
#include "../../include/asr_b200.h"
#include "common.cuh"

namespace asrb {

// ---------------------------------------------------------------------------------------
// dims: asrb_dims + derived geometry (reference: src/config.rs, src/audio_encoder.rs:79-134)
// ---------------------------------------------------------------------------------------
struct Dims {
    asrb_dims c;
    int enc_hd;             // d_model / heads
    int chunk_frames;       // 2 * n_window                       (audio_encoder.rs:83)
    int chunks_per_window;  // n_window_infer / chunk_frames      (audio_encoder.rs:179)
    int conv_h[4];          // freq extent  128 -> 64 -> 32 -> 16
    int conv_w[4];          // time extent  100 -> 50 -> 25 -> 13
    int tok_per_chunk;      // conv_w[3]
    int cpad;               // downsample_hidden_size rounded up to 64 (TMA / wgmma K-block)
    int feat;               // dsh * conv_h[3]  (conv_out in-features, 7680)
    int q_dim, kv_dim, qkv_dim;
    void derive();
};
void validate_dims(const asrb_dims& d);   // c_api.cu: throws ASRB_ERR_INVALID
inline int conv_out_len(int l) { return (l - 1) / 2 + 1; }   // audio_encoder.rs:263-266

struct Ctx {
    int device = 0;
    int sm_count = 132;
    size_t smem_optin = 0;
};

struct EncLayerW {
    float *ln1_w, *ln1_b, *ln2_w, *ln2_b;
    bf16 *wqkv, *wo, *fc1, *fc2;
    float *bqkv, *bo, *b1, *b2;
};
struct DecLayerW {
    float *ln_in, *ln_post, *qnorm, *knorm;
    bf16 *wqkv, *wo, *wgu, *wdown;   // wgu rows interleaved: 2j = gate_j, 2j+1 = up_j
};

struct RawTensor {
    void* dev = nullptr;       // bf16 for matrices, f32 for vectors
    bool is_bf16 = false;
    std::vector<int64_t> shape;
    size_t numel = 0;
};

struct Model {
    Ctx* ctx = nullptr;
    Dims d;
    bool finalized = false;
    bool lossy_weights = false;          // an F32/F16 matrix was not bf16-representable (only with ASRB_ALLOW_LOSSY_WEIGHTS=1)
    int lossy_count = 0;
    std::map<std::string, RawTensor> raw;
    std::vector<void*> owned;            // packed buffers created at finalize

    // mel constants (src/mel.rs:115-187 + periodic Hann + DFT twiddles)
    float *mel_fb = nullptr, *dft_cos = nullptr, *dft_sin = nullptr, *hann = nullptr, *dft_tw = nullptr;
    int* mel_krange = nullptr;           // [num_mels][2] non-zero bin range of each filter
    // encoder
    float *conv1_w = nullptr, *conv1_b = nullptr, *conv2_b = nullptr, *conv3_b = nullptr, *conv_out_b = nullptr;
    bf16 *conv2_w = nullptr, *conv3_w = nullptr, *conv_out_w = nullptr;   // conv: [dsh][9][cpad]
    float* pos_emb = nullptr;            // [tok_per_chunk][d_model]
    std::vector<EncLayerW> enc;
    float *lnpost_w = nullptr, *lnpost_b = nullptr, *proj1_b = nullptr, *proj2_b = nullptr;
    bf16 *proj1 = nullptr, *proj2 = nullptr;
    // decoder
    bf16 *embed = nullptr, *lm_head = nullptr;
    std::vector<DecLayerW> dec;
    float* final_norm = nullptr;
    DecLayerW* d_dec_layers = nullptr;   // device copy of `dec` for the fused decode step; its ln_in / ln_post point at
                                         // copies stored in the step's bank-conflict-free activation layout (decode_mega.cu)
    float* final_norm_sw = nullptr;      // final norm weight in the same layout
    // batch-aware fused step (decode_batch.cu): weight matrices with the 16-byte chunks of every row XOR-swizzled by
    // (row & 7) -- bank-conflict-free ldmatrix on bulk-copied rows -- and plain norm vectors; null for unsupported dims
    DecLayerW* d_dec_layers_b = nullptr;
    bf16* lm_head_b = nullptr;
    // greedy fused single-sequence step (decode_mega.cu consume_head_q): int8 copy of the lm_head and per row {scale s_r,
    // bound constant C_r}; null for dims without that instantiation
    int8_t* lm_head_q = nullptr;
    float2* lm_head_sc = nullptr;
    float *rope_cos = nullptr, *rope_sin = nullptr;   // [rope_max_pos][head_dim/2]
    int rope_max_pos = 0;

    ~Model();
};

// ---------------------------------------------------------------------------------------
// GEMM plumbing shared by the SIMT and tensor-core (wgmma) implementations
//   D[m][n] = sum_k A(m,k) * W[n][k]      W: bf16 [N][K] row-major (HF layout, layers.rs:74-80)
// ---------------------------------------------------------------------------------------
enum { A_PLAIN = 0, A_CONV = 1 };
struct GemmA {
    int mode = A_PLAIN;
    const bf16* a = nullptr;     // split3 planes
    size_t plane_stride = 0;     // elements between planes
    int nplanes = 3;
    int M = 0, K = 0, lda = 0;
    // A_CONV: implicit 3x3 / stride 2 / pad 1 conv over the parity-split channels-last layout
    //   in[(((chunk*2+ph)*2+pw)*Hh + hh)*Wh + wh][cpad],  m = (chunk, oh, ow),  k = (tap, cin)
    int OH = 0, OW = 0, Hh = 0, Wh = 0, cpad = 0;
};
enum { EPI_PLAIN = 0, EPI_SWIGLU = 1, EPI_CONV_PARITY = 2, EPI_CONV_FEAT = 3, EPI_CONVOUT = 4 };
struct GemmEpi {
    int mode = EPI_PLAIN;
    const float* bias = nullptr;      // [N]
    int act = 0;                      // 1 = exact-erf GELU
    const float* residual = nullptr;  // fp32 [M][ldr]
    int ldr = 0;
    float* out_f32 = nullptr;
    int ldo = 0;
    bf16* out_s3 = nullptr;
    size_t s3_plane_stride = 0;
    int lds = 0;
    // conv epilogues
    int OH = 0, OW = 0, Hh2 = 0, Wh2 = 0, cpad = 0;
    // EPI_CONVOUT
    const int* row_map = nullptr;     // [M] -> token row or -1
    const float* pos = nullptr;       // [pos_period][N]
    int pos_period = 1;
    // optional fp32 workspace for split-K (EPI_PLAIN GEMMs with too few tiles to fill the GPU): >= SPLITK_WS_FLOATS floats
    float* splitk_ws = nullptr;
    int64_t* extra_launches = nullptr;   // incremented by the number of kernels launched beyond the one GEMM kernel
};
static constexpr size_t SPLITK_WS_FLOATS = (size_t)4 * 64 * 128 * 128;   // 4 splits x 64 tiles of 128 x 128
enum { GEMM_SIMT = 0, GEMM_TC = 1 };
extern std::atomic<int64_t> g_gemm_simt_fallbacks, g_gemm_tc_launches;   // gemm_simt.cu: tensor core requested but SIMT ran / tensor-core launches
void launch_gemm(const GemmA& A, const bf16* W, int N, const GemmEpi& E, int impl, cudaStream_t st);
// wgmma implementation (gemm_tc.cu); returns false when the shape is unsupported
bool launch_gemm_tc(const GemmA& A, const bf16* W, int N, const GemmEpi& E, cudaStream_t st);
// What launch_gemm_tc launches for a shape on a GPU of `sms` SMs (host only, no device call): tc = false when the
// wgmma kernel cannot take the shape or epilogue (launch_gemm then runs the SIMT GEMM); otherwise the k-split factor,
// the output tiles and the persistent grid (work items = tiles_m * tiles_n * splits, dealt round-robin over the grid)
struct GemmPlan { bool tc = false; int splits = 1, tiles_m = 0, tiles_n = 0, grid = 0, box_h = 0; };
GemmPlan plan_gemm_tc(const GemmA& A, int N, const GemmEpi& E, int sms);
void launch_gemm_simt(const GemmA& A, const bf16* W, int N, const GemmEpi& E, cudaStream_t st);

// ---------------------------------------------------------------------------------------
// kernels (each .cu exposes launchers; all asynchronous on `st`)
// ---------------------------------------------------------------------------------------
// mel.cu
void launch_mel(const Model& m, const float* samples, const int64_t* d_soff, const int64_t* d_n,
                const int64_t* d_npad, const int64_t* d_foff, int batch, int max_frames,
                float* mel_out, int* d_maxkey, cudaStream_t st);
// streaming (DESIGN.md 4.9): frames [ffirst[b], F_b) of stream b into its raw log-mel rows (raw + b * n_mels * ldo), then
// the fold of the frames that became final (d_fold[b] = {f_old, f_new, F, active}) into stats row b
void launch_mel_stream(const Model& m, const float* samples, const int64_t* d_soff, const int64_t* d_n, const int64_t* d_npad,
                       const int64_t* d_foff, const int* d_ffirst, int n_streams, int max_new_frames, int ldo, float* raw,
                       const int4* d_fold, int win_frames, float* stats, int stats_ld, cudaStream_t st);
// the re-encoded windows as clamped, scaled pseudo-utterances (d_plan[u] = {slot, first frame, frames, phi bits})
void launch_mel_stream_stage(const Model& m, const float* raw, const int4* d_plan, const int64_t* d_foff, int n_utt, int ldo,
                             float* mel_out, cudaStream_t st);
// segment.cu: window energies and cut points of the long-audio files (DESIGN.md section 4.6)
void launch_segment(const float* d_long, const int64_t* d_plan, int n_files, int64_t total_blocks, int64_t max_seg,
                    int64_t search, double* d_blk, int64_t* d_cuts, int64_t* d_ncuts, int sm_count, cudaStream_t st);
// elementwise.cu
void launch_conv1(const Model& m, const float* mel, const int* d_chunk_clip, const int* d_chunk_f0,
                  const int64_t* d_foff, const int64_t* d_frames, int n_chunks,
                  bf16* out_s3, size_t plane_stride, cudaStream_t st);
void launch_layernorm_s3(const float* x, const float* w, const float* b, int rows, int dim, float eps,
                         bf16* out_s3, size_t plane_stride, cudaStream_t st);
void launch_rmsnorm_s3(const float* x, const float* w, int rows, int dim, float eps,
                       bf16* out_s3, size_t plane_stride, cudaStream_t st);
void launch_embed_inject(const bf16* embed, int hidden, const int* d_ids, const int* d_audio_row,
                         const float* audio, int rows, float* out, cudaStream_t st);
// prefill K/V fan-out of shared context prefixes (DESIGN.md 4.5), device arrays indexed by sequence
struct FanOut {
    const int* n;       // [nseq] follower slots of a leader (0: not a leader)
    const int* off;     // [nseq] index of its first follower slot in `slots`
    const int* P;       // [nseq] shared prefix length of a leader's group: positions 0..P-1 are fanned out
    const int* slots;   // follower slots, grouped by leader
};
void launch_qk_norm_rope(const float* qkv, int rows, const int* d_row_seq, const int* d_row_pos,
                         const float* qnorm, const float* knorm, float eps,
                         const float* rope_cos, const float* rope_sin,
                         int nq, int nkv, int hd, float* q_out, float* kcache, float* vcache,
                         size_t cache_seq_stride, int max_ctx, cudaStream_t st, const FanOut* fan = nullptr);
// attention.cu
struct AttnParams {
    const float* q; int ldq;            // q row r, head h at q + r*ldq + h*hd
    const float* k; const float* v;     // key j of segment s, kv-head g at k + s*seg_stride + g*head_stride + j*ldk
    size_t seg_stride, head_stride; int ldk;
    const int* seg_q0;                  // [nseg] first q row of segment (also index base of keys when keys_in_rows)
    const int* seg_len;                 // [nseg]
    int keys_in_rows;                   // 1: key j lives at row (seg_q0+j) of the k/v buffers (encoder qkv buffer)
    int nseg, nheads, group;            // q head h uses kv head h / group
    int causal; int max_len;
    bf16* out_s3; size_t plane_stride; int ldo;
    const int* seg_pos0;                // [nseg] or null (causal cache keys only): query row i of segment s is at position
                                        // seg_pos0[s] + i and attends to keys 0..seg_pos0[s] + i of its slot (DESIGN.md 4.5)
};
void launch_attention(const AttnParams& p, int hd, cudaStream_t st);
// decode.cu  (per-phase kernels, any batch <= 8) -- see decode_mega.cu for the fused step
struct DecodeBufs {
    float* x;        // [B][H] residual stream
    float* qkv;      // [B][qkv_dim]
    float* attn;     // [B][q_dim]
    float* act;      // [B][I]
    float* logits;   // [B][V] or null
    float* part_val; int* part_idx; int n_part;   // argmax partials [B][n_part]
    int* pos;        // [B] position of the token being processed (= ctx length before append)
    int* done;       // [B]
    int* next_id;    // [B]
    int* ids_out;    // [B][max_new]
    int* n_out;      // [B]
    int max_new;
    // per-token log-probabilities (session option "logprobs"): buffers allocated when the option is first enabled
    bool logprobs;   // launch the LOGPROB kernel variants
    float* part_sum; // [B][n_part] sum of exp(logit - part_val) per argmax partial
    float* lp_out;   // [B][max_new] log-probability of each appended token
    float* eos_lp;   // [B] log-probability of the EOS token that ended the sequence (NaN until then)
    // top-k alternatives (session option "top_logprobs" >= 1, which also sets `logprobs`): allocated when first enabled;
    // the kernels always keep TK_MAX candidates per step, best first (-1 / NaN until written)
    bool topk;          // launch the TOPK kernel variants
    float* tk_part_val; // [B][n_part][TK_MAX] per-CTA candidate logits
    int* tk_part_idx;   // [B][n_part][TK_MAX] their ids
    int* tk_ids;        // [B][max_new][TK_MAX] candidates of the step that selected each appended token
    float* tk_lp;       // [B][max_new][TK_MAX] their log-probabilities
    int* tk_eos_ids;    // [B][TK_MAX] candidates of the step that selected the EOS token ending the sequence
    float* tk_eos_lp;   // [B][TK_MAX]
    // seeded temperature sampling (session options "temperature" / "seed", latched at the prefill): the kernels select
    // the argmax of the Gumbel keys (common.cuh) instead of the logits
    bool sample;              // launch the SAMPLE kernel variants
    const SampleParams* smp;  // device: 1 / temperature and the seed of the current run
    float* part_max;          // [B][n_part] sampling with logprobs: raw maximum logit per argmax partial (part_val holds keys)
    float* part_sel;          // [B][n_part] raw logit of each partial's best-key row (allocated when first needed)
    // repetition controls (session options "no_repeat_ngram_size" / "repetition_penalty", latched at the prefill): the
    // REP kernel variants fold the processed logits.  The fused steps build their bit arrays themselves; before a
    // per-phase step launch_rep_mask builds each sequence's over the whole vocabulary
    bool rep;                     // the REP kernel variants
    const RepParams* rep_params;  // device: the penalty and N of the current run
    uint32_t* rep_mask;           // per-phase: [B][2][rep_words] bits; fused steps: [G][sequences][2][rep_cta_words]
    int rep_words;                // (vocab + 31) / 32
};
void launch_rep_mask(const DecodeBufs& b, int R, cudaStream_t st, int64_t* launches);
// words of one repetition bit array covering a fused step CTA's lm_head rows (a contiguous range of at most
// ceil(vocab / G) rows, which may start mid-word)
inline int rep_cta_words(const asrb_dims& c, int G) { return ((c.vocab_size + G - 1) / G + 31) / 32 + 1; }
void launch_decode_step_phases(const Model& m, const DecodeBufs& b, int B, float* kcache, float* vcache,
                               size_t cache_layer_stride, size_t cache_seq_stride, int max_ctx,
                               bool write_logits, cudaStream_t st, int64_t* launches);
// shared memory the per-phase decode attention needs for a session of max_ctx positions: the queries of one GQA group,
// one fp32 score per (query head, key), and its static reduction scratch.  Checked at session creation.
size_t dec_attn_smem_bytes(const Model& m, int max_ctx);
// final-norm + lm_head + argmax on arbitrary rows of a residual stream (prefill last rows);
// also performs the greedy bookkeeping of src/inference.rs:161-170 (EOS check, append, embed)
struct MegaBufs { unsigned* bar = nullptr; float* part = nullptr; long long* dbg = nullptr; size_t part_bytes = 0; unsigned* steps_issued = nullptr;
                  uint32_t* sx = nullptr; size_t sx_bytes = 0; int* sx_nb = nullptr;   // sx: decode_batch.cu's self-validating words   // per-session state of the fused step
                  uint32_t* sx_seq = nullptr;   // decode_mega.cu's self-validating words (outside `part`: never wiped to 0)
                  unsigned long long* hq_stats = nullptr; };   // [4] int8 lm_head counters of the greedy single-sequence step
size_t decode_mega_part_floats(const Model& m);
bool decode_mega_dims(const asrb_dims& c);   // (hidden, q_dim, intermediate) the single-sequence fused step is compiled for
size_t decode_mega_sx_bytes(const Model& m);
size_t decode_batch_part_floats(const Model& m);
size_t decode_batch_sx_bytes(const Model& m);   // decode_batch.cu: NB sequences per fused launch
bool decode_batch_supported(const Model& m, int B, int ctx);
int decode_mega_dbg_slots();
void launch_greedy(const Model& m, const DecodeBufs& b, int B, cudaStream_t st, int64_t* launches);
void launch_lmhead_argmax(const Model& m, const float* x_rows, const int* d_row_idx, int B,
                          const DecodeBufs& b, bool write_logits, cudaStream_t st, int64_t* launches);

// score.cu -- teacher-forced scoring head (asrb_score_ids, DESIGN.md 4.8)
constexpr int SCORE_SLICES = 64;    // column slices per row: the partial workspace is rows x SCORE_SLICES, whatever the vocab
struct ScorePart {                  // one (row, column slice): max logit, sum of exp(l - max), target logit (-inf: not here)
    float m, s, t;
    float tv[TK_MAX]; int ti[TK_MAX];   // TOPK: the slice's best (logit, id), best first
};
struct ScoreHeadPlan { int tiles_m = 0, tiles_n = 0, nslices = 0, grid = 0; };
// the head's work items (M tile, column slice) and persistent grid on `sms` SMs; grid_cap > 0 caps the grid further
ScoreHeadPlan plan_score_head(int rows, int V, int sms, int grid_cap);
int score_slices(const Model& m);
void check_score_head(const Model& m);   // throws ASRB_ERR_INVALID for a shape the wgmma head cannot take
// rows r of hid[d_src[r]] -> final norm -> lm_head; lp_out[r] = log p(d_target[r]), with topk the 8 best of each row.
// The first form takes the head's weights and dims explicitly (the probes); the second is the model's, on all its SMs
void launch_score_head(const bf16* lm_head, const float* final_norm, int H, int V, float eps, int sms, int grid_cap,
                       const float* hid, const int* d_src, const int* d_target, int rows, float* gathered, bf16* planes,
                       size_t plane_stride, int nplanes, ScorePart* part, bool topk, float* lp_out, int* tk_ids,
                       float* tk_lp, cudaStream_t st, int64_t* launches);
void launch_score_head(const Model& m, const float* hid, const int* d_src, const int* d_target, int rows, float* gathered,
                       bf16* planes, size_t plane_stride, int nplanes, ScorePart* part, bool topk, float* lp_out,
                       int* tk_ids, float* tk_lp, cudaStream_t st, int64_t* launches);

// align.cu -- word-timing alignment (asrb_align_ids, DESIGN.md 4.10); per-utterance device arrays indexed by b
struct AlignProbArgs {
    const float* q; int ldq;                   // post-RoPE q rows (s->qrot)
    const float* k; size_t seg_stride, head_stride; int hd, group;   // the layer's K cache
    const int *qrow0, *N, *T, *a0, *slot;      // first aligned row, rows, audio keys, first audio position, KV slot
    const long long* moff;                     // offset of utterance b's [N][T] block in a plane
    const int* heads; int nheads;              // query heads of the layer (device), in list order
    float* P; size_t plane;                    // [nheads][plane] probabilities
};
struct AlignFoldArgs {
    const int *N, *T; const long long* moff;
    float* P; size_t plane; int nheads;        // z-scores in place
    float* M;                                  // [sum N T] running head sum (the last listed layer: the mean)
    int count;                                 // > 0 on the last listed layer: divide by it
};
struct AlignDtwArgs {
    const int *N, *T; const long long* moff;
    const float* M;
    const int* smem_trace;                     // 1: trace in shared memory, else at trace + toff[b]
    uint32_t* trace; const long long* toff;
    int* start; const int* soff;               // start[soff[b] + i]: least column of the path in row i
};
constexpr size_t ALIGN_PROBS_SMEM_MAX = 64 * 1024;
size_t align_probs_smem(int hd);   // dynamic shared memory of align_probs_kernel; refused above ALIGN_PROBS_SMEM_MAX
void launch_align_probs(const AlignProbArgs& a, int B, int maxN, cudaStream_t st);
void launch_align_fold(const AlignFoldArgs& a, int B, int maxT, int maxNT, cudaStream_t st);
size_t align_dtw_smem(int N, int T, bool trace_in_smem);
void launch_align_dtw(const AlignDtwArgs& a, int B, size_t smem, cudaStream_t st);

// beam.cu -- beam search over the TOPK records (session option "beam_size"); the spec is in include/asr_b200.h
constexpr int BEAM_MAX = 6;
struct BeamUtt {                   // device state of one utterance's search
    int t;                         // records consumed = ids in every alive beam
    int done;                      // K finished hypotheses
    int S;                         // prompt length
    int nfin;                      // finished hypotheses so far, in admission order:
    int fin_depth[BEAM_MAX];       //   last id's depth in the history (-1: no id), = n - 1
    int fin_slot[BEAM_MAX];        //   its slot at that depth
    int fin_eos[BEAM_MAX];         //   the EOS id
    float fin_eos_lp[BEAM_MAX], fin_sum[BEAM_MAX];
    int slot_of_rank[BEAM_MAX];    // alive beams, best first
    float sum_of_rank[BEAM_MAX];
    int cp[BEAM_MAX][BEAM_MAX];    // by beam index: depth of the deepest common node of two beams (-1: the prompt only)
    long long reassigned, reorder_bytes, expand_bytes;
};
struct BeamArgs {
    int B, K, max_new, hidden, ldh;          // utterances, beams, id capacity, hidden size, history row stride (max_batch)
    long long bytes_per_pos;                 // K and V bytes of one cache position over all layers and kv heads
    BeamUtt* u;
    const int* tk_ids; const float* tk_lp; const int* tk_eos_ids; const float* tk_eos_lp;
    int *done, *pos, *next_id, *n_out, *ids_out;
    float* x; const bf16* embed;
    int *hist_tok, *hist_par; float* hist_lp;   // [max_new][max_batch]: id, parent slot (-1: the prompt), log p
    int *cp_src, *cp_p0, *cp_n;                 // [max_batch] KV copy plan of the step, by destination slot
    int* nb_ids; float* nb_lp;                  // [B][K][max_new] ranked hypotheses
    float *lp_out, *eos_lp;
    float *kcache, *vcache; int layers, nkv, head_dim, max_ctx; size_t layer_stride, seq_stride;
};
void launch_beam_step(const BeamArgs& a, bool first, const int* pos0, cudaStream_t st, int64_t* launches);
void launch_beam_finalize(const BeamArgs& a, const int* hyp, const float* best_eos_lp, cudaStream_t st, int64_t* launches);

}  // namespace asrb
