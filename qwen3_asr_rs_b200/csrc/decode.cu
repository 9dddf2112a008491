// decode.cu -- one greedy decode iteration (inference.rs:160-200) as per-phase kernels, any batch
// (processed in sub-batches of 8 sequences).
//
// This is the general-batch path and the on-device reference of the fused single-kernel step
// (decode_mega.cu).  All phases are HBM-bandwidth kernels: each weight byte is read exactly once
// per step with 128-bit coalesced loads, bf16 -> fp32 up-cast is exact, accumulation is fp32, so
// results track the fp32 oracle to summation-order noise.  Phases per layer (layers.rs:442-463):
//   qkv   : RMSNorm (layers.rs:48-54) fused into the [q|k|v] GEMV                (layers.rs:297-299)
//   attn  : per-head QK-RMSNorm + RoPE + KV append + softmax(q.K/sqrt(d)).V, GQA by indexing
//   oproj : GEMV + residual                                                      (layers.rs:338-339,454)
//   gateup: RMSNorm fused into the interleaved gate/up GEMV + SiLU*mul           (layers.rs:396-399)
//   down  : GEMV + residual                                                      (layers.rs:400,460)
// then final RMSNorm + tied lm_head GEMV + argmax partials (text_decoder.rs:111-112) and the greedy
// bookkeeping kernel (argmax, EOS check, append, embed next token; inference.rs:161-170) -- the
// 151936 logits are only written in parity mode and no host sync happens per token.
#include <algorithm>
#include <type_traits>
#include "internal.h"

namespace asrb {

static constexpr int DG_THREADS = 256, DG_WARPS = 8;
// DE_ARGMAX_LSE: DE_ARGMAX + per-CTA sum of exp(logit - max) (part_sum), the partial record of the token log-probability
// DE_ARGMAX_GUMBEL: argmax of the sampling keys fmaf(logit, inv_t, g) instead of the logits (common.cuh); part_val holds
// the CTA's best key.  DE_ARGMAX_GUMBEL_LSE: + the raw (max, sum) record (part_max, part_sum) and the raw logit of the
// best-key row (part_sel)
enum { DE_STORE = 0, DE_RESID = 1, DE_SWIGLU = 2, DE_ARGMAX = 3, DE_ARGMAX_LSE = 4, DE_ARGMAX_GUMBEL = 5, DE_ARGMAX_GUMBEL_LSE = 6 };

struct GemvParams {
    const bf16* W; int N, K;
    const float* x; int ldx; const int* row_idx;   // input rows: x + row_idx[b]*ldx (row_idx may be null)
    const float* norm_w; float eps;                 // PRE_NORM
    float* out; int ldo;                            // STORE / RESID (in place on out) / SWIGLU
    float* logits; int ldl;                         // ARGMAX: optional full logits
    float* part_val; int* part_idx;                 // ARGMAX: [B][gridDim.x]
    int B;
    float* part_sum;                                // ARGMAX_LSE: [B][gridDim.x]
};
// ARGMAX_GUMBEL*: a second kernel argument (the `sample` pack), so the parameter block of the other epilogues stays as it is
struct GemvSample {
    const SampleParams* smp;                        // the run's 1 / temperature and seed
    const int* n_out; int row0;                     // each sequence's step n (= ids generated so far), global row of sequence 0
    float* part_max; float* part_sel;               // ARGMAX_GUMBEL_LSE: [B][gridDim.x]
};

// ARGMAX epilogues with the repetition controls: one more kernel argument, after the `sample` pack when there is one
struct GemvRep {
    const uint32_t* mask; int words;                // [B][2][words] each sequence's bit arrays (common.cuh), built before the step
    const RepParams* rep;                           // the run's penalty
};

// the extra argument of type T
template <typename T, typename S0, typename... S> __device__ __forceinline__ const T& gemv_arg(const S0& s0, const S&... s) {
    if constexpr (std::is_same_v<T, S0>) return s0;
    else return gemv_arg<T>(s...);
}

template <int MAXB, bool PRE_NORM, int EPI, typename... Extra>
__global__ void __launch_bounds__(DG_THREADS) dec_gemv_kernel(GemvParams p, Extra... extra) {
    extern __shared__ float xs[];          // [MAXB][K]
    __shared__ float red[32];
    __shared__ float bestv[DG_WARPS][MAXB];
    __shared__ int besti[DG_WARPS][MAXB];
    constexpr bool SMP = EPI == DE_ARGMAX_GUMBEL || EPI == DE_ARGMAX_GUMBEL_LSE, SLSE = EPI == DE_ARGMAX_GUMBEL_LSE;
    constexpr bool ARGMAX = EPI == DE_ARGMAX || EPI == DE_ARGMAX_LSE || SMP, LSE = EPI == DE_ARGMAX_LSE;
    constexpr bool REP = (std::is_same_v<GemvRep, Extra> || ...);
    const int K = p.K, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int b = 0; b < MAXB; ++b) {
        if (b < p.B) {
            const float* xr = p.x + (size_t)(p.row_idx ? p.row_idx[b] : b) * p.ldx;
            if (PRE_NORM) {
                float s = 0.f;
                for (int i = tid; i < K; i += DG_THREADS) s = fmaf(xr[i], xr[i], s);
                const float r = 1.0f / sqrtf(block_sum(s, red) / K + p.eps);
                for (int i = tid; i < K; i += DG_THREADS) xs[b * K + i] = (xr[i] * r) * p.norm_w[i];
            } else {
                for (int i = tid; i < K; i += DG_THREADS) xs[b * K + i] = xr[i];
            }
        } else {
            for (int i = tid; i < K; i += DG_THREADS) xs[b * K + i] = 0.f;
        }
    }
    __syncthreads();
    constexpr int RSTEP = (EPI == DE_SWIGLU) ? 2 : 1;     // SWIGLU: a warp owns the (gate_j, up_j) pair
    const int units = p.N / RSTEP;
    const int per_cta = (units + gridDim.x - 1) / gridDim.x;
    const int u0 = blockIdx.x * per_cta, u1 = min(units, u0 + per_cta);
    float bv[MAXB]; int bi[MAXB];
    float bs[(LSE || SLSE) ? MAXB : 1];           // LSE: sum of exp(logit - bv[b]) over this warp's rows (SLSE: - bm[b])
    float bm[SLSE ? MAXB : 1], bsel[SLSE ? MAXB : 1];   // SLSE: raw maximum logit, raw logit of the best-key row
#pragma unroll
    for (int b = 0; b < MAXB; ++b) { bv[b] = -INFINITY; bi[b] = 0x7fffffff; if constexpr (LSE) bs[b] = 0.f; }
    Draw dr[SMP ? MAXB : 1];                      // SMP: each sequence's draw (global row row0 + b, step n_out[b])
    if constexpr (SMP) {
#pragma unroll
        for (int b = 0; b < MAXB; ++b) {
            const GemvSample& ps = gemv_arg<GemvSample>(extra...);
            dr[b] = make_draw(ps.smp, b < p.B ? __ldg(ps.n_out + b) : 0, ps.row0 + b);
            if constexpr (SLSE) { bs[b] = 0.f; bm[b] = -INFINITY; bsel[b] = 0.f; }
        }
    }
    for (int u = u0 + warp; u < u1; u += DG_WARPS) {
        float acc[RSTEP][MAXB];
#pragma unroll
        for (int r = 0; r < RSTEP; ++r)
#pragma unroll
            for (int b = 0; b < MAXB; ++b) acc[r][b] = 0.f;
#pragma unroll
        for (int r = 0; r < RSTEP; ++r) {
            const uint4* wrow = reinterpret_cast<const uint4*>(p.W + (size_t)(u * RSTEP + r) * K);
            for (int c = lane; c < K / 8; c += 32) {
                uint4 wv = __ldg(wrow + c);
                float w0 = bf16_lo(wv.x), w1 = bf16_hi(wv.x), w2 = bf16_lo(wv.y), w3 = bf16_hi(wv.y);
                float w4 = bf16_lo(wv.z), w5 = bf16_hi(wv.z), w6 = bf16_lo(wv.w), w7 = bf16_hi(wv.w);
#pragma unroll
                for (int b = 0; b < MAXB; ++b) {
                    const float4 xa = *reinterpret_cast<const float4*>(&xs[b * K + c * 8]);
                    const float4 xb = *reinterpret_cast<const float4*>(&xs[b * K + c * 8 + 4]);
                    float a = acc[r][b];
                    a = fmaf(w0, xa.x, a); a = fmaf(w1, xa.y, a); a = fmaf(w2, xa.z, a); a = fmaf(w3, xa.w, a);
                    a = fmaf(w4, xb.x, a); a = fmaf(w5, xb.y, a); a = fmaf(w6, xb.z, a); a = fmaf(w7, xb.w, a);
                    acc[r][b] = a;
                }
            }
        }
#pragma unroll
        for (int r = 0; r < RSTEP; ++r)
#pragma unroll
            for (int b = 0; b < MAXB; ++b) acc[r][b] = warp_sum(acc[r][b]);
        if (lane == 0) {
#pragma unroll
            for (int b = 0; b < MAXB; ++b) {
                if (b >= p.B) break;
                if (EPI == DE_STORE) p.out[(size_t)b * p.ldo + u] = acc[0][b];
                if (EPI == DE_RESID) p.out[(size_t)b * p.ldo + u] += acc[0][b];
                if (EPI == DE_SWIGLU) p.out[(size_t)b * p.ldo + u] = silu(acc[0][b]) * acc[RSTEP - 1][b];
                if (ARGMAX) {
                    bool keep = true;                // REP: the processed logit replaces the raw one everywhere
                    if constexpr (REP) {
                        const GemvRep& pr = gemv_arg<GemvRep>(extra...);
                        const uint32_t* h = pr.mask + (size_t)b * 2 * pr.words;
                        keep = rep_logit(RepBits{h, h + pr.words, 0, __ldg(&pr.rep->theta)}, u, acc[0][b]);
                    }
                    if (p.logits) p.logits[(size_t)b * p.ldl + u] = acc[0][b];
                    if (!keep) continue;             // banned: -inf in the logits, no part in any fold
                    if constexpr (SMP) {
                        float unused = 0.f;
                        if constexpr (SLSE) sample_fold<true>(dr[b], acc[0][b], u, bv[b], bi[b], bs[b], bm[b], bsel[b]);
                        else sample_fold<false>(dr[b], acc[0][b], u, bv[b], bi[b], unused, unused, unused);
                    }
                    else if constexpr (LSE) lse_fold(acc[0][b], u, bv[b], bi[b], bs[b]);
                    else if (acc[0][b] > bv[b]) { bv[b] = acc[0][b]; bi[b] = u; }   // rows ascend per warp: first max wins
                }
            }
        }
    }
    if (EPI == DE_ARGMAX || EPI == DE_ARGMAX_GUMBEL) {      // GUMBEL: the same merge over the keys
        if (lane == 0)
            for (int b = 0; b < MAXB; ++b) { bestv[warp][b] = bv[b]; besti[warp][b] = bi[b]; }
        __syncthreads();
        if (tid < p.B) {
            float v = -INFINITY; int idx = 0x7fffffff;
            for (int w = 0; w < DG_WARPS; ++w)
                if (bestv[w][tid] > v || (bestv[w][tid] == v && besti[w][tid] < idx)) { v = bestv[w][tid]; idx = besti[w][tid]; }
            p.part_val[(size_t)tid * gridDim.x + blockIdx.x] = v;
            p.part_idx[(size_t)tid * gridDim.x + blockIdx.x] = idx;
        }
    }
    if constexpr (LSE) {
        __shared__ float bests[DG_WARPS][MAXB];
        if (lane == 0)
            for (int b = 0; b < MAXB; ++b) { bestv[warp][b] = bv[b]; besti[warp][b] = bi[b]; bests[warp][b] = bs[b]; }
        __syncthreads();
        if (tid < p.B) {
            float v = -INFINITY; int idx = 0x7fffffff;
            for (int w = 0; w < DG_WARPS; ++w)
                if (bestv[w][tid] > v || (bestv[w][tid] == v && besti[w][tid] < idx)) { v = bestv[w][tid]; idx = besti[w][tid]; }
            float sum = 0.f;                     // the warps' sums rescaled to the CTA maximum, in warp order
            for (int w = 0; w < DG_WARPS; ++w) sum += lse_rescale(bests[w][tid], bestv[w][tid], v);
            p.part_val[(size_t)tid * gridDim.x + blockIdx.x] = v;
            p.part_idx[(size_t)tid * gridDim.x + blockIdx.x] = idx;
            p.part_sum[(size_t)tid * gridDim.x + blockIdx.x] = sum;
        }
    }
    if constexpr (SLSE) {
        __shared__ float bests[DG_WARPS][MAXB], bestm[DG_WARPS][MAXB], bestsel[DG_WARPS][MAXB];
        if (lane == 0)
            for (int b = 0; b < MAXB; ++b) {
                bestv[warp][b] = bv[b]; besti[warp][b] = bi[b]; bests[warp][b] = bs[b]; bestm[warp][b] = bm[b]; bestsel[warp][b] = bsel[b];
            }
        __syncthreads();
        if (tid < p.B) {
            float v = -INFINITY; int idx = 0x7fffffff, ws = 0; float M = -INFINITY;
            for (int w = 0; w < DG_WARPS; ++w) {
                if (bestv[w][tid] > v || (bestv[w][tid] == v && besti[w][tid] < idx)) { v = bestv[w][tid]; idx = besti[w][tid]; ws = w; }
                M = fmaxf(M, bestm[w][tid]);
            }
            float sum = 0.f;                     // the warps' raw sums rescaled to the CTA's raw maximum, in warp order
            for (int w = 0; w < DG_WARPS; ++w) sum += lse_rescale(bests[w][tid], bestm[w][tid], M);
            const size_t o = (size_t)tid * gridDim.x + blockIdx.x;
            const GemvSample& ps = gemv_arg<GemvSample>(extra...);
            p.part_val[o] = v; p.part_idx[o] = idx; p.part_sum[o] = sum; ps.part_max[o] = M; ps.part_sel[o] = bestsel[ws][tid];
        }
    }
}

template <int MB, bool PRE_NORM, int EPI, typename... Extra>
static void launch_gemv_kernel(const GemvParams& p, int grid, size_t smem, cudaStream_t st, const Extra&... extra) {
    auto kern = dec_gemv_kernel<MB, PRE_NORM, EPI, Extra...>;
    if (smem > 48 * 1024) ASRB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, DG_THREADS, smem, st>>>(p, extra...);
}

template <bool PRE_NORM, int EPI>
static void run_gemv(const GemvParams& p, int grid, cudaStream_t st, const GemvSample* ps = nullptr, const GemvRep* pr = nullptr) {
    size_t smem_of[4] = {(size_t)1 * p.K * 4, (size_t)2 * p.K * 4, (size_t)4 * p.K * 4, (size_t)8 * p.K * 4};
    ASRB_REQUIRE(p.K % 256 == 0, ASRB_ERR_INVALID, "decode GEMV needs K % 256 == 0");
    ASRB_REQUIRE(p.B >= 1 && p.B <= 8, ASRB_ERR_INVALID, "per-phase decode supports batch 1..8");
#define ASRB_GEMV_CASE(MB, IDX)                                                                              \
    {                                                                                                        \
        if constexpr (EPI == DE_ARGMAX || EPI == DE_ARGMAX_LSE || EPI == DE_ARGMAX_GUMBEL || EPI == DE_ARGMAX_GUMBEL_LSE) \
            if (pr) {                                                                                        \
                if constexpr (EPI == DE_ARGMAX_GUMBEL || EPI == DE_ARGMAX_GUMBEL_LSE)                        \
                    launch_gemv_kernel<MB, PRE_NORM, EPI>(p, grid, smem_of[IDX], st, *ps, *pr);              \
                else launch_gemv_kernel<MB, PRE_NORM, EPI>(p, grid, smem_of[IDX], st, *pr);                  \
                ASRB_CUDA_CHECK(cudaGetLastError());                                                         \
                return;                                                                                      \
            }                                                                                                \
        if constexpr (EPI == DE_ARGMAX_GUMBEL || EPI == DE_ARGMAX_GUMBEL_LSE) {                       \
            auto kern = dec_gemv_kernel<MB, PRE_NORM, EPI, GemvSample>;                                      \
            if (smem_of[IDX] > 48 * 1024)                                                                    \
                ASRB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_of[IDX])); \
            kern<<<grid, DG_THREADS, smem_of[IDX], st>>>(p, *ps);                                            \
        } else {                                                                                             \
            auto kern = dec_gemv_kernel<MB, PRE_NORM, EPI>;                                                  \
            if (smem_of[IDX] > 48 * 1024)                                                                    \
                ASRB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_of[IDX])); \
            kern<<<grid, DG_THREADS, smem_of[IDX], st>>>(p);                                                 \
        }                                                                                                    \
    }
    if (p.B == 1) ASRB_GEMV_CASE(1, 0)
    else if (p.B == 2) ASRB_GEMV_CASE(2, 1)
    else if (p.B <= 4) ASRB_GEMV_CASE(4, 2)
    else ASRB_GEMV_CASE(8, 3)
#undef ASRB_GEMV_CASE
    ASRB_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// decode attention: grid (nkv, B), 128 threads (= head_dim).  Applies per-head RMSNorm + RoPE to the
// new q (group heads) and k, appends k,v at index pos, then softmax(q.K^T / sqrt(d)) V over 0..pos.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) dec_attn_kernel(const float* __restrict__ qkv, int qkv_dim,
                                                       const int* __restrict__ pos_arr, const int* __restrict__ done,
                                                       const float* __restrict__ qnorm, const float* __restrict__ knorm,
                                                       float eps, const float* __restrict__ rope_cos,
                                                       const float* __restrict__ rope_sin, int nq, int nkv, int group,
                                                       float* __restrict__ kcache, float* __restrict__ vcache,
                                                       size_t cache_seq_stride, int max_ctx,
                                                       float* __restrict__ attn_out) {
    constexpr int HD = 128;
    extern __shared__ float sm[];
    float* qs = sm;                       // [group][HD]
    float* sc = qs + group * HD;          // [group][max_ctx]
    __shared__ float tmp[HD];
    __shared__ float red[32];
    const int g = blockIdx.x, b = blockIdx.y, d = threadIdx.x, lane = d & 31, warp = d >> 5;
    if (done[b]) return;
    const int pos = pos_arr[b];
    const float* row = qkv + (size_t)b * qkv_dim;
    const int half = HD / 2;
    const float c = rope_cos[(size_t)pos * half + (d % half)], s = rope_sin[(size_t)pos * half + (d % half)];
    float* kc = kcache + (size_t)b * cache_seq_stride + (size_t)g * max_ctx * HD;
    float* vc = vcache + (size_t)b * cache_seq_stride + (size_t)g * max_ctx * HD;
    {   // new K
        float x = row[(size_t)(nq + g) * HD + d];
        float var = block_sum(x * x, red) / HD;
        float y = (x * (1.0f / sqrtf(var + eps))) * knorm[d];
        tmp[d] = y;
        __syncthreads();
        float rot = d < half ? -tmp[d + half] : tmp[d - half];
        kc[(size_t)pos * HD + d] = y * c + rot * s;
        vc[(size_t)pos * HD + d] = row[(size_t)(nq + nkv + g) * HD + d];
        __syncthreads();
    }
    for (int hq = 0; hq < group; ++hq) {
        float x = row[(size_t)(g * group + hq) * HD + d];
        float var = block_sum(x * x, red) / HD;
        float y = (x * (1.0f / sqrtf(var + eps))) * qnorm[d];
        tmp[d] = y;
        __syncthreads();
        float rot = d < half ? -tmp[d + half] : tmp[d - half];
        qs[hq * HD + d] = y * c + rot * s;
        __syncthreads();
    }
    const int nkeys = pos + 1;
    const float div = sqrtf((float)HD);
    for (int j = warp; j < nkeys; j += 4) {
        const float4 kv = *reinterpret_cast<const float4*>(kc + (size_t)j * HD + lane * 4);
        for (int hq = 0; hq < group; ++hq) {
            const float4 qv = *reinterpret_cast<const float4*>(qs + hq * HD + lane * 4);
            float dot = kv.x * qv.x + kv.y * qv.y + kv.z * qv.z + kv.w * qv.w;
            dot = warp_sum(dot);
            if (lane == 0) sc[hq * max_ctx + j] = dot / div;
        }
    }
    __syncthreads();
    for (int hq = 0; hq < group; ++hq) {
        float mx = -INFINITY;
        for (int j = d; j < nkeys; j += HD) mx = fmaxf(mx, sc[hq * max_ctx + j]);
        mx = block_max(mx, red);
        float sum = 0.f;
        for (int j = d; j < nkeys; j += HD) { float e = expf(sc[hq * max_ctx + j] - mx); sc[hq * max_ctx + j] = e; sum += e; }
        sum = block_sum(sum, red);
        __syncthreads();
        float acc = 0.f;
        for (int j = 0; j < nkeys; ++j) acc = fmaf(sc[hq * max_ctx + j], vc[(size_t)j * HD + d], acc);
        attn_out[(size_t)b * nq * HD + (size_t)(g * group + hq) * HD + d] = acc / sum;
    }
}

// ---------------------------------------------------------------------------------------------
// greedy bookkeeping (inference.rs:161-170): finish the argmax, EOS check, append, embed.
// LOGPROB: also merge the (max, sum of exponentials) records and store the selected token's log-probability in
// lp_out (appended token) or eos_lp (EOS).
// TOPK (with LOGPROB): also select the TK_MAX best (logit, id) pairs of the step's logits [B][vocab] (written by the
// lm_head GEMV) and store them in tk_ids / tk_lp [B][max_new][TK_MAX] or the EOS rows tk_eos_ids / tk_eos_lp [B][TK_MAX].
// SAMPLE (with LOGPROB; without it the plain kernel merges the keys): part_val holds keys, the raw records are
// (part_max, part_sum) and part_sel the raw logit of each record's best-key row; the value recorded is (l_sel - M) - log S.
// grid = B blocks.
// ---------------------------------------------------------------------------------------------
template <bool LOGPROB, bool TOPK = false, bool SAMPLE = false>
__global__ void greedy_kernel(const float* __restrict__ part_val, const int* __restrict__ part_idx, int n_part,
                              int* __restrict__ done, int* __restrict__ pos, int* __restrict__ next_id,
                              int* __restrict__ ids_out, int* __restrict__ n_out, int max_new,
                              const bf16* __restrict__ embed, int hidden, float* __restrict__ x,
                              const float* __restrict__ part_sum, float* __restrict__ lp_out, float* __restrict__ eos_lp,
                              const float* __restrict__ logits, int vocab, int* __restrict__ tk_ids, float* __restrict__ tk_lp,
                              int* __restrict__ tk_eos_ids, float* __restrict__ tk_eos_lp,
                              const float* __restrict__ part_max, const float* __restrict__ part_sel) {
    static_assert(!TOPK || LOGPROB, "the candidates' log-probabilities need the sum of exponentials");
    static_assert(!SAMPLE || (LOGPROB && !TOPK), "SAMPLE: the logprob variant only, never with the candidates");
    __shared__ float sv[32];
    __shared__ int si[32];
    __shared__ int tok_s;
    int* srec = nullptr; float* smax = nullptr;    // SAMPLE: per warp, the best key's record and the raw maximum
    if constexpr (SAMPLE) { __shared__ int srec_[32]; __shared__ float smax_[32]; srec = srec_; smax = smax_; }
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (done[b]) { if (tid == 0) next_id[b] = -1; return; }
    float v = -INFINITY; int idx = 0x7fffffff;
    int rec = 0; float mloc = -INFINITY;          // SAMPLE: the best key's record, the raw maximum of the records
    for (int i = tid; i < n_part; i += blockDim.x) {
        float pv = part_val[(size_t)b * n_part + i]; int pi = part_idx[(size_t)b * n_part + i];
        if (pv > v || (pv == v && pi < idx)) { v = pv; idx = pi; if constexpr (SAMPLE) rec = i; }
        if constexpr (SAMPLE) mloc = fmaxf(mloc, part_max[(size_t)b * n_part + i]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, v, o); int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        int orec = 0;
        if constexpr (SAMPLE) orec = __shfl_xor_sync(0xffffffffu, rec, o);
        if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; if constexpr (SAMPLE) rec = orec; }
    }
    if constexpr (SAMPLE) mloc = warp_max(mloc);
    if (lane == 0) { sv[warp] = v; si[warp] = idx; if constexpr (SAMPLE) { srec[warp] = rec; smax[warp] = mloc; } }
    __syncthreads();
    float lp = 0.f, M = 0.f;
    if constexpr (LOGPROB) {
        // S = sum_c s_c exp(m_c - M) over the n_part records, M = the maximum logit: each thread its records in index
        // order, then a fixed tree over lanes and warps; logprob = -log S
        __shared__ float ss[32];
        const int nw = (blockDim.x + 31) / 32;
        const float* rmax = SAMPLE ? part_max : part_val;      // SAMPLE: part_val holds keys
        M = SAMPLE ? smax[0] : sv[0];
        for (int w = 1; w < nw; ++w) M = fmaxf(M, SAMPLE ? smax[w] : sv[w]);
        float sum = 0.f;
        for (int i = tid; i < n_part; i += blockDim.x) sum += lse_rescale(part_sum[(size_t)b * n_part + i], rmax[(size_t)b * n_part + i], M);
        sum = warp_sum(sum);
        if (lane == 0) ss[warp] = sum;
        __syncthreads();
        if (tid == 0) {
            float S = 0.f;
            for (int w = 0; w < nw; ++w) S += ss[w];
            lp = -logf(S);
        }
    }
    TopK tk;
    if constexpr (TOPK) {
        // each thread its rows (ascending), a butterfly per warp, then thread 0 merges the warps' lists
        __shared__ float tkv[32 * TK_MAX];
        __shared__ int tki[32 * TK_MAX];
        tk_init(tk);
        const float* lg = logits + (size_t)b * vocab;
        for (int i = tid; i < vocab; i += blockDim.x) tk_insert(tk, lg[i], i);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tk_merge_xor(tk, o);
        if (lane == 0) tk_store(tk, tkv + warp * TK_MAX, tki + warp * TK_MAX);
        __syncthreads();
        if (tid == 0) {
            const int nw = (blockDim.x + 31) / 32;
            for (int w = 1; w < nw; ++w) tk_merge_from(tk, tkv + w * TK_MAX, tki + w * TK_MAX, false);
        }
    }
    if (tid == 0) {
        int nw = (blockDim.x + 31) / 32;
        for (int w = 1; w < nw; ++w)
            if (sv[w] > v || (sv[w] == v && si[w] < idx)) { v = sv[w]; idx = si[w]; if constexpr (SAMPLE) rec = srec[w]; }
        int tok = idx;
        if constexpr (SAMPLE) lp = (part_sel[(size_t)b * n_part + rec] - M) + lp;   // (l_sel - M) - log S
        if constexpr (LOGPROB) {
            if (tok == 151643 || tok == 151645) eos_lp[b] = lp;
            else if (n_out[b] < max_new) lp_out[(size_t)b * max_new + n_out[b]] = lp;
        }
        if constexpr (TOPK) {
            if (tok == 151643 || tok == 151645) tk_write(tk, lp, tk_eos_ids + (size_t)b * TK_MAX, tk_eos_lp + (size_t)b * TK_MAX);
            else if (n_out[b] < max_new) {
                const size_t o = ((size_t)b * max_new + n_out[b]) * TK_MAX;
                tk_write(tk, lp, tk_ids + o, tk_lp + o);
            }
        }
        if (tok == 151643 || tok == 151645 || n_out[b] >= max_new) {   // EOS ids, inference.rs:154
            done[b] = 1; next_id[b] = -1; tok = -1;
        } else {
            ids_out[(size_t)b * max_new + n_out[b]] = tok;
            n_out[b] += 1;
            pos[b] += 1;
            next_id[b] = tok;
        }
        tok_s = tok;
    }
    __syncthreads();
    const int tok = tok_s;
    if (tok < 0) return;
    const bf16* e = embed + (size_t)tok * hidden;                         // text_decoder.rs:90-92
    for (int i = tid; i < hidden; i += blockDim.x) x[(size_t)b * hidden + i] = __bfloat162float(e[i]);
}

void launch_greedy(const Model& m, const DecodeBufs& b, int B, cudaStream_t st, int64_t* launches) {
    if (b.sample && b.logprobs)     // sampling without logprobs: the plain kernel below merges the keys
        greedy_kernel<true, false, true><<<B, 256, 0, st>>>(b.part_val, b.part_idx, b.n_part, b.done, b.pos, b.next_id, b.ids_out, b.n_out,
                                                            b.max_new, m.embed, m.d.c.hidden_size, b.x, b.part_sum, b.lp_out, b.eos_lp,
                                                            nullptr, 0, nullptr, nullptr, nullptr, nullptr, b.part_max, b.part_sel);
    else if (b.topk && !b.sample)     // the lm_head wrote the logits (launch_lmhead_argmax): one CTA per sequence selects the candidates
        greedy_kernel<true, true><<<B, 256, 0, st>>>(b.part_val, b.part_idx, b.n_part, b.done, b.pos, b.next_id, b.ids_out, b.n_out,
                                                     b.max_new, m.embed, m.d.c.hidden_size, b.x, b.part_sum, b.lp_out, b.eos_lp,
                                                     b.logits, m.d.c.vocab_size, b.tk_ids, b.tk_lp, b.tk_eos_ids, b.tk_eos_lp,
                                                     nullptr, nullptr);
    else if (b.logprobs && !b.sample)
        greedy_kernel<true><<<B, 256, 0, st>>>(b.part_val, b.part_idx, b.n_part, b.done, b.pos, b.next_id, b.ids_out, b.n_out,
                                               b.max_new, m.embed, m.d.c.hidden_size, b.x, b.part_sum, b.lp_out, b.eos_lp,
                                               nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    else
        greedy_kernel<false><<<B, 256, 0, st>>>(b.part_val, b.part_idx, b.n_part, b.done, b.pos, b.next_id, b.ids_out, b.n_out,
                                                b.max_new, m.embed, m.d.c.hidden_size, b.x, nullptr, nullptr, nullptr,
                                                nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    ASRB_CUDA_CHECK(cudaGetLastError());
    if (launches) *launches += 1;
}

// repetition controls, per-phase path: one CTA per sequence builds its bit arrays over the whole vocabulary from its
// generated ids (common.cuh), before the step
__global__ void __launch_bounds__(256) rep_mask_kernel(const int* __restrict__ ids_out, const int* __restrict__ n_out, int max_new,
                                                       const RepParams* __restrict__ rep, uint32_t* __restrict__ mask, int words, int vocab) {
    const int b = blockIdx.x;
    uint32_t* h = mask + (size_t)b * 2 * words;
    for (int i = threadIdx.x; i < 2 * words; i += blockDim.x) h[i] = 0u;
    __syncthreads();
    rep_mark(ids_out + (size_t)b * max_new, min(n_out[b], max_new), __ldg(&rep->ngram), 0, vocab, h, h + words, threadIdx.x, blockDim.x);
}

void launch_rep_mask(const DecodeBufs& b, int R, cudaStream_t st, int64_t* launches) {
    rep_mask_kernel<<<R, 256, 0, st>>>(b.ids_out, b.n_out, b.max_new, b.rep_params, b.rep_mask, b.rep_words, 32 * b.rep_words);
    ASRB_CUDA_CHECK(cudaGetLastError());
    if (launches) *launches += 1;
}

static DecodeBufs offset_bufs(const DecodeBufs& b, int b0, const Model& m) {
    const asrb_dims& c = m.d.c;
    DecodeBufs o = b;
    o.x = b.x + (size_t)b0 * c.hidden_size; o.qkv = b.qkv + (size_t)b0 * m.d.qkv_dim; o.attn = b.attn + (size_t)b0 * m.d.q_dim;
    o.act = b.act + (size_t)b0 * c.intermediate_size; o.logits = b.logits ? b.logits + (size_t)b0 * c.vocab_size : nullptr;
    o.part_val = b.part_val + (size_t)b0 * b.n_part; o.part_idx = b.part_idx + (size_t)b0 * b.n_part;
    o.part_sum = b.part_sum ? b.part_sum + (size_t)b0 * b.n_part : nullptr;
    o.part_max = b.part_max ? b.part_max + (size_t)b0 * b.n_part : nullptr;
    o.part_sel = b.part_sel ? b.part_sel + (size_t)b0 * b.n_part : nullptr;
    o.pos = b.pos + b0; o.done = b.done + b0; o.next_id = b.next_id + b0; o.ids_out = b.ids_out + (size_t)b0 * b.max_new; o.n_out = b.n_out + b0;
    return o;
}

void launch_lmhead_argmax(const Model& m, const float* x_rows, const int* d_row_idx, int B, const DecodeBufs& b,
                          bool write_logits, cudaStream_t st, int64_t* launches) {
    const asrb_dims& c = m.d.c;
    for (int b0 = 0; b0 < B; b0 += 8) {              // GEMV kernels hold up to 8 activation vectors in shared memory
        const int nb = std::min(8, B - b0);
        const DecodeBufs ob = offset_bufs(b, b0, m);
        GemvParams p{};
        p.W = m.lm_head; p.N = c.vocab_size; p.K = c.hidden_size;
        p.x = d_row_idx ? x_rows : x_rows + (size_t)b0 * c.hidden_size; p.ldx = c.hidden_size; p.row_idx = d_row_idx ? d_row_idx + b0 : nullptr;
        p.norm_w = m.final_norm; p.eps = (float)c.rms_norm_eps;
        p.logits = (write_logits || (b.topk && !b.sample)) ? ob.logits : nullptr; p.ldl = c.vocab_size;   // TOPK: greedy_kernel reads them
        p.part_val = ob.part_val; p.part_idx = ob.part_idx; p.B = nb;
        GemvRep pr{b.rep_mask + (size_t)b0 * 2 * b.rep_words, b.rep_words, b.rep_params};
        const GemvRep* prp = b.rep ? &pr : nullptr;  // the repetition controls: the processed logits everywhere below
        if (b.sample) {                              // the draw's row is global: b0 + the sequence's index in the launch
            GemvSample ps{};
            ps.smp = b.smp; ps.n_out = ob.n_out; ps.row0 = b0;
            if (b.logprobs) {
                p.part_sum = ob.part_sum; ps.part_max = ob.part_max; ps.part_sel = ob.part_sel;
                run_gemv<true, DE_ARGMAX_GUMBEL_LSE>(p, b.n_part, st, &ps, prp);
            }
            else run_gemv<true, DE_ARGMAX_GUMBEL>(p, b.n_part, st, &ps, prp);
        }
        else if (b.logprobs) { p.part_sum = ob.part_sum; run_gemv<true, DE_ARGMAX_LSE>(p, b.n_part, st, nullptr, prp); }
        else run_gemv<true, DE_ARGMAX>(p, b.n_part, st, nullptr, prp);
        if (launches) *launches += 1;
    }
}

static constexpr size_t DEC_ATTN_STATIC_SMEM = (128 + 32) * sizeof(float);   // tmp + red of dec_attn_kernel
size_t dec_attn_smem_bytes(const Model& m, int max_ctx) {
    const size_t group = m.d.c.num_attention_heads / m.d.c.num_key_value_heads;
    return group * (128 + (size_t)max_ctx) * sizeof(float) + DEC_ATTN_STATIC_SMEM;
}

void launch_decode_step_phases(const Model& m, const DecodeBufs& ball, int Ball, float* kcache_all, float* vcache_all,
                               size_t cache_layer_stride, size_t cache_seq_stride, int max_ctx, bool write_logits,
                               cudaStream_t st, int64_t* launches) {
    const asrb_dims& c = m.d.c;
    const Dims& d = m.d;
    ASRB_REQUIRE(c.head_dim == 128, ASRB_ERR_INVALID, "decode attention needs head_dim 128");
    const int sms = m.ctx->sm_count;
    const int group = c.num_attention_heads / c.num_key_value_heads;
    const size_t attn_smem = dec_attn_smem_bytes(m, max_ctx) - DEC_ATTN_STATIC_SMEM;
    if (attn_smem > 48 * 1024)     // per device attribute: set on every launch (a process may drive several GPUs)
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(dec_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_smem));
    for (int b0 = 0; b0 < Ball; b0 += 8) {           // sub-batches of 8 sequences (weights are re-streamed per sub-batch)
      const int B = std::min(8, Ball - b0);
      const DecodeBufs b = offset_bufs(ball, b0, m);
      float* kcache = kcache_all + (size_t)b0 * cache_seq_stride;
      float* vcache = vcache_all + (size_t)b0 * cache_seq_stride;
      for (int l = 0; l < c.num_hidden_layers; ++l) {
        const DecLayerW& w = m.dec[l];
        GemvParams p{};
        p.B = B; p.eps = (float)c.rms_norm_eps;
        // qkv
        p.W = w.wqkv; p.N = d.qkv_dim; p.K = c.hidden_size; p.x = b.x; p.ldx = c.hidden_size; p.row_idx = nullptr;
        p.norm_w = w.ln_in; p.out = b.qkv; p.ldo = d.qkv_dim;
        run_gemv<true, DE_STORE>(p, min(sms * 2, (p.N + 7) / 8), st);
        // attention
        dim3 ag(c.num_key_value_heads, B);
        dec_attn_kernel<<<ag, 128, attn_smem, st>>>(b.qkv, d.qkv_dim, b.pos, b.done, w.qnorm, w.knorm,
                                                    (float)c.rms_norm_eps, m.rope_cos, m.rope_sin,
                                                    c.num_attention_heads, c.num_key_value_heads, group,
                                                    kcache + (size_t)l * cache_layer_stride,
                                                    vcache + (size_t)l * cache_layer_stride, cache_seq_stride,
                                                    max_ctx, b.attn);
        ASRB_CUDA_CHECK(cudaGetLastError());
        // o_proj + residual
        p.W = w.wo; p.N = c.hidden_size; p.K = d.q_dim; p.x = b.attn; p.ldx = d.q_dim; p.norm_w = nullptr;
        p.out = b.x; p.ldo = c.hidden_size;
        run_gemv<false, DE_RESID>(p, min(sms * 2, (p.N + 7) / 8), st);
        // gate/up + SiLU*mul
        p.W = w.wgu; p.N = 2 * c.intermediate_size; p.K = c.hidden_size; p.x = b.x; p.ldx = c.hidden_size;
        p.norm_w = w.ln_post; p.out = b.act; p.ldo = c.intermediate_size;
        run_gemv<true, DE_SWIGLU>(p, min(sms * 2, (c.intermediate_size + 7) / 8), st);
        // down + residual
        p.W = w.wdown; p.N = c.hidden_size; p.K = c.intermediate_size; p.x = b.act; p.ldx = c.intermediate_size;
        p.norm_w = nullptr; p.out = b.x; p.ldo = c.hidden_size;
        run_gemv<false, DE_RESID>(p, min(sms * 2, (p.N + 7) / 8), st);
        if (launches) *launches += 5;
      }
    }
    launch_lmhead_argmax(m, ball.x, nullptr, Ball, ball, write_logits, st, launches);
}

}  // namespace asrb
