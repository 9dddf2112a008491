// score.cu -- teacher-forced scoring head (asrb_score_ids, DESIGN.md 4.8): log p(target | row) and the top-8 of every
// gathered decoder row, without materialising the [rows][vocab] logits.
//
//   gather + final RMSNorm -> split3 planes -> wgmma GEMM against lm_head with a folding epilogue -> per-row merge
//
// The GEMM is gemm_tc.cu's (TMA ring of 3 stages, warpgroup 0 the producer, warpgroups 1-2 the wgmma consumers, CH
// k-blocks per tensor-core accumulation -- 1 here, 4 there -- three planes), but its work item is (M tile, column
// slice): a CTA walks the contiguous N tiles of one slice for one M tile and folds each finished 128 x 128 logit tile
// into per-row running state held in registers.  Lane l of a consumer warp owns row l & 15 of the warp's 16 rows and 16 of every 32
// columns; the two lanes of a row merge at the end of the slice and write one partial (max m, sum of exp(l - m), the
// target's logit when it lies in the slice, and with TOPK the slice's 8 best (logit, id)).  At most SCORE_SLICES
// slices per row, so the workspace is rows x 64 partials whatever the vocabulary.  Columns >= vocab (the zero-filled
// TMA rows of a ragged last tile) are skipped, so any vocabulary size works.
#include <cuda.h>
#include <algorithm>
#include "internal.h"
#include "wgmma.cuh"

namespace asrb {
namespace score {

using namespace tc;
static constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3;
static constexpr int TILE_A_BYTES = BM * BK * 2;
static constexpr int TILE_B_BYTES = BN * BK * 2;
static constexpr int STAGE_BYTES = 3 * TILE_A_BYTES + TILE_B_BYTES;
static constexpr int NTHREADS = 384;
static constexpr int CONS_WARPS = 8;
static constexpr int SLAB_LD = 40;
// one k-block (3 planes x 4 k16 steps) per tensor-core accumulation, then a round-to-nearest add into the fp32 sums.
// The tensor core truncates its running sum at every k16 step; gemm_tc.cu's 4-block chunks (48 truncations) put a
// peaked row's log-probabilities (every product of the winning logit one sign) at up to 12 x the fp32 error
static constexpr int CH = 1;

template <bool TOPK>
__global__ void __launch_bounds__(NTHREADS, 1)
score_head_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, int M, int V, int K,
                  int nplanes, int tiles_m, int tiles_n, int nslices, const int* __restrict__ target,
                  ScorePart* __restrict__ part) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    float* epi_slab = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + 256);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_kb = K / BK;
    const int n_items = tiles_m * nslices;
    // item = slice * tiles_m + m tile: CTAs running together read the same lm_head tiles (L2 hits across M tiles)
    auto slice_range = [&](int slice, int& t0, int& t1) {
        t0 = (int)((long long)slice * tiles_n / nslices); t1 = (int)((long long)(slice + 1) * tiles_n / nslices);
    };

    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // warpgroup 0 hands registers to the consumers (40 + 2 x 232 per thread fits the 64 K register file): the TOPK
        // fold keeps a per-lane top-8 list beside the two 64-register accumulator sets
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (warp != 0 || lane != 0) return;
        // ================= TMA producer =================
        const uint32_t stage_tx = (uint32_t)nplanes * TILE_A_BYTES + (uint32_t)TILE_B_BYTES;
        uint32_t kg = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int mt = item % tiles_m, slice = item / tiles_m;
            int t0, t1; slice_range(slice, t0, t1);
            for (int nt = t0; nt < t1; ++nt)
                for (int kb = 0; kb < num_kb; ++kb, ++kg) {
                    const int s = kg % STAGES; const uint32_t par = (kg / STAGES) & 1;
                    mbar_wait(&empty[s], par ^ 1);
                    uint8_t* st = smem + s * STAGE_BYTES;
                    mbar_expect_tx(&full[s], stage_tx);
                    for (int p = 0; p < nplanes; ++p) tma_load_3d(st + p * TILE_A_BYTES, &mapA, kb * BK, mt * BM, p, &full[s]);
                    tma_load_2d(st + 3 * TILE_A_BYTES, &mapB, kb * BK, nt * BN, &full[s]);
                }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
        // ================= wgmma consumers + folding epilogue =================
        const int half = (warp >> 2) - 1, q = warp & 3;
        const int cw = warp - 4;
        float* slab = epi_slab + cw * (16 * SLAB_LD);
        const int lr = lane & 15, lh = lane >> 4;         // folding: row lr of the warp's 16, columns 16 lh .. 16 lh + 15
        float acc[64], sum[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] = 0.f;
        uint32_t kg = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int mt = item % tiles_m, slice = item / tiles_m;
            int t0, t1; slice_range(slice, t0, t1);
            const int row = mt * BM + half * 64 + q * 16 + lr;
            const int tgt = row < M ? __ldg(target + row) : -1;
            float mx = -INFINITY, se = 0.f, tl = -INFINITY;
            TopK tk;
            if constexpr (TOPK) tk_init(tk);
            for (int nt = t0; nt < t1; ++nt) {
#pragma unroll
                for (int j = 0; j < 64; ++j) sum[j] = 0.f;
                consume_k_blocks<STAGES, STAGE_BYTES, TILE_A_BYTES, BK, CH>(smem, full, empty, half, lane, num_kb, nplanes, kg, acc, sum);
                // fold the tile 32 columns at a time through the warp's shared-memory slab
#pragma unroll
                for (int g = 0; g < BN / 32; ++g) {
                    stage_slab<SLAB_LD>(slab, sum, g, lane);
                    const int n = nt * BN + g * 32 + 16 * lh;
                    const int nv = min(16, V - n);          // columns of the vocabulary (the last tile may be ragged)
                    const float* sr = slab + lr * SLAB_LD + 16 * lh;
                    float gm = -INFINITY;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float4 x = *reinterpret_cast<const float4*>(sr + 4 * i);
                        if (4 * i < nv) gm = fmaxf(gm, x.x);
                        if (4 * i + 1 < nv) gm = fmaxf(gm, x.y);
                        if (4 * i + 2 < nv) gm = fmaxf(gm, x.z);
                        if (4 * i + 3 < nv) gm = fmaxf(gm, x.w);
                    }
                    if (gm > mx) { se = lse_rescale(se, mx, gm); mx = gm; }
#pragma unroll
                    for (int i = 0; i < 16; ++i)
                        if (i < nv) {
                            const float x = sr[i];
                            se += expf(x - mx);
                            if (n + i == tgt) tl = x;
                            if constexpr (TOPK) tk_insert(tk, x, n + i);
                        }
                    __syncwarp();                           // the slab is rewritten by the next group
                }
            }
            // the two lanes of a row: one partial per (row, slice)
            const float om = __shfl_xor_sync(0xffffffffu, mx, 16), os = __shfl_xor_sync(0xffffffffu, se, 16);
            const float ot = __shfl_xor_sync(0xffffffffu, tl, 16);
            se = lse_merge(mx, se, om, os); mx = fmaxf(mx, om); tl = fmaxf(tl, ot);
            if constexpr (TOPK) tk_merge_xor(tk, 16);
            if (lh == 0 && row < M) {
                ScorePart* o = part + (size_t)row * nslices + slice;
                o->m = mx; o->s = se; o->t = tl;
                if constexpr (TOPK) tk_store(tk, o->tv, o->ti);
            }
        }
    }
}

// one warp per row: the slices in a fixed order per lane, then a fixed butterfly.  log p = (l - M) - log S with M the
// row's maximum logit, as the greedy kernels' records
template <bool TOPK>
__global__ void __launch_bounds__(32) score_merge_kernel(const ScorePart* __restrict__ part, int nslices,
                                                         float* __restrict__ lp_out, int* __restrict__ tk_ids,
                                                         float* __restrict__ tk_lp) {
    const int row = blockIdx.x, lane = threadIdx.x;
    const ScorePart* p = part + (size_t)row * nslices;
    float M = -INFINITY, tl = -INFINITY;
    for (int j = lane; j < nslices; j += 32) { M = fmaxf(M, p[j].m); tl = fmaxf(tl, p[j].t); }
    M = warp_max(M); tl = warp_max(tl);
    float S = 0.f;
    for (int j = lane; j < nslices; j += 32) S += lse_rescale(p[j].s, p[j].m, M);
    S = warp_sum(S);
    const float lse = logf(S);
    TopK tk;
    if constexpr (TOPK) {
        tk_init(tk);
        for (int j = lane; j < nslices; j += 32) tk_merge_from(tk, p[j].tv, p[j].ti, false);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tk_merge_xor(tk, o);
    }
    if (lane == 0) {
        lp_out[row] = (tl - M) - lse;
        if constexpr (TOPK) {
#pragma unroll
            for (int j = 0; j < TK_MAX; ++j) { tk_ids[(size_t)row * TK_MAX + j] = tk.i[j]; tk_lp[(size_t)row * TK_MAX + j] = (tk.v[j] - M) - lse; }
        }
    }
}

__global__ void gather_rows_kernel(const float* __restrict__ x, const int* __restrict__ src, int H, float* __restrict__ out) {
    const float* a = x + (size_t)src[blockIdx.x] * H;
    float* b = out + (size_t)blockIdx.x * H;
    for (int i = threadIdx.x * 4; i < H; i += blockDim.x * 4) *reinterpret_cast<float4*>(b + i) = *reinterpret_cast<const float4*>(a + i);
}

static size_t smem_bytes() { return (size_t)STAGES * STAGE_BYTES + 1024 + 256 + CONS_WARPS * 16 * SLAB_LD * 4; }

}  // namespace score

void check_score_head(const Model& m) {
    const asrb_dims& c = m.d.c;
    ASRB_REQUIRE(c.hidden_size % score::BK == 0, ASRB_ERR_INVALID,
                 "score: the wgmma score head needs hidden_size % 64 == 0, got " + std::to_string(c.hidden_size));
}

ScoreHeadPlan plan_score_head(int rows, int V, int sms, int grid_cap) {
    using namespace score;
    ScoreHeadPlan p;
    p.tiles_m = (rows + BM - 1) / BM; p.tiles_n = (V + BN - 1) / BN;
    p.nslices = std::min(SCORE_SLICES, p.tiles_n);
    p.grid = std::min(p.tiles_m * p.nslices, sms);
    if (grid_cap > 0) p.grid = std::min(p.grid, grid_cap);
    return p;
}

int score_slices(const Model& m) { return plan_score_head(1, m.d.c.vocab_size, 1, 0).nslices; }

void launch_score_head(const bf16* lm_head, const float* final_norm, int H, int V, float eps, int sms, int grid_cap,
                       const float* hid, const int* d_src, const int* d_target, int rows, float* gathered, bf16* planes,
                       size_t plane_stride, int nplanes, ScorePart* part, bool topk, float* lp_out, int* tk_ids,
                       float* tk_lp, cudaStream_t st, int64_t* launches) {
    using namespace score;
    ASRB_REQUIRE(H > 0 && H % BK == 0 && V >= 1 && sms >= 1 && grid_cap >= 0, ASRB_ERR_INVALID, "score: bad head dims");
    ASRB_REQUIRE(rows >= 1 && nplanes >= 1 && nplanes <= 3, ASRB_ERR_INVALID, "score: bad head shape");
    gather_rows_kernel<<<rows, 128, 0, st>>>(hid, d_src, H, gathered);
    ASRB_CUDA_CHECK(cudaGetLastError());
    launch_rmsnorm_s3(gathered, final_norm, rows, H, eps, planes, plane_stride, st);
    cuuint64_t ad[3] = {(cuuint64_t)H, (cuuint64_t)rows, 3};
    cuuint64_t as[2] = {(cuuint64_t)H * 2, (cuuint64_t)plane_stride * 2};
    cuuint32_t ab[3] = {(cuuint32_t)BK, (cuuint32_t)BM, 1};
    const CUtensorMap mapA = tc_cached_map(planes, 3, ad, as, ab);
    cuuint64_t bd[2] = {(cuuint64_t)H, (cuuint64_t)V};
    cuuint64_t bs[1] = {(cuuint64_t)H * 2};
    cuuint32_t bb[2] = {(cuuint32_t)BK, (cuuint32_t)BN};
    const CUtensorMap mapB = tc_cached_map(lm_head, 2, bd, bs, bb);
    const ScoreHeadPlan p = plan_score_head(rows, V, sms, grid_cap);
    const int tiles_m = p.tiles_m, tiles_n = p.tiles_n, nslices = p.nslices, grid = p.grid;
    const size_t smem = smem_bytes();
    if (topk) {
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(score_head_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        score_head_kernel<true><<<grid, NTHREADS, smem, st>>>(mapA, mapB, rows, V, H, nplanes, tiles_m, tiles_n, nslices, d_target, part);
        ASRB_CUDA_CHECK(cudaGetLastError());
        score_merge_kernel<true><<<rows, 32, 0, st>>>(part, nslices, lp_out, tk_ids, tk_lp);
    } else {
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(score_head_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        score_head_kernel<false><<<grid, NTHREADS, smem, st>>>(mapA, mapB, rows, V, H, nplanes, tiles_m, tiles_n, nslices, d_target, part);
        ASRB_CUDA_CHECK(cudaGetLastError());
        score_merge_kernel<false><<<rows, 32, 0, st>>>(part, nslices, lp_out, nullptr, nullptr);
    }
    ASRB_CUDA_CHECK(cudaGetLastError());
    if (launches) *launches += 4;
}

void launch_score_head(const Model& m, const float* hid, const int* d_src, const int* d_target, int rows, float* gathered,
                       bf16* planes, size_t plane_stride, int nplanes, ScorePart* part, bool topk, float* lp_out,
                       int* tk_ids, float* tk_lp, cudaStream_t st, int64_t* launches) {
    check_score_head(m);
    const asrb_dims& c = m.d.c;
    launch_score_head(m.lm_head, m.final_norm, c.hidden_size, c.vocab_size, (float)c.rms_norm_eps, m.ctx->sm_count, 0, hid,
                      d_src, d_target, rows, gathered, planes, plane_stride, nplanes, part, topk, lp_out, tk_ids, tk_lp, st,
                      launches);
}

}  // namespace asrb
