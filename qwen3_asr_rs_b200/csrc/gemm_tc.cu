// gemm_tc.cu -- wgmma tensor-core GEMM for the encoder / prefill contractions (sm_90a).
//
//   D[m][n] = sum_p sum_k A_p(m,k) * W[n][k]        p = bf16 split planes of the fp32 activation
//
// Replaces every Linear::forward (layers.rs:74-80) with M > 1 and conv2d2/conv2d3 (audio_encoder.rs:
// 128-129) as implicit GEMM.  Hopper structure: one 128x128 output tile per CTA at a time, operands
// staged by TMA (cp.async.bulk.tensor, 128B swizzle) into a 3-stage shared-memory ring guarded by
// mbarriers; warpgroup 0 is the TMA producer, warpgroups 1 and 2 each own 64 rows of the tile and
// issue wgmma.mma_async (m64n128k16, bf16 x bf16 -> fp32 registers) straight from the swizzled
// shared-memory tiles, then apply the fused epilogues of epilogue.cuh.
//
// Precision: weights are exact bf16; each fp32 activation is stored as 3 bf16 planes
// (hi + mid + lo == x to 1 ulp, common.cuh).  bf16 x bf16 products are exact in fp32 and the
// accumulator is fp32, so the result matches an fp32 GEMM to accumulation-order noise -- that is
// what keeps greedy token ids identical to the fp32 oracle.  planes = 1 gives the plain bf16 GEMM.
//
// The conv A-operand is never materialised (no im2col): the activation lives in a parity-split
// channels-last layout so that each of the 9 filter taps is a plain (unit-stride) TMA box of a
// 5-D tensor map; out-of-bounds coordinates (the conv padding) are zero-filled by TMA.
#include <cuda.h>
#include <algorithm>
#include <cstring>
#include <map>
#include <tuple>
#include "internal.h"
#include "epilogue.cuh"
#include "wgmma.cuh"

namespace asrb {
namespace tc {

static constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3;
static constexpr int TILE_A_BYTES = BM * BK * 2;      // 16 KB per plane
static constexpr int TILE_B_BYTES = BN * BK * 2;      // 16 KB
static constexpr int STAGE_BYTES = 3 * TILE_A_BYTES + TILE_B_BYTES;   // 64 KB
static constexpr int NTHREADS = 384;                  // warpgroup 0: TMA producer; warpgroups 1-2: wgmma + epilogue
static constexpr int CONS_WARPS = 8;                  // consumer warps; warp w of a consumer warpgroup owns 16 tile rows
static constexpr int SLAB_LD = 40;                    // floats per staged epilogue row (32 + 8: conflict-free float2 writes / float4 reads)
static constexpr int CH = 4;                          // k-blocks (of 64) accumulated inside the tensor core per chunk

struct ConvGeom { int OH, OW, box_h, tiles_per_chunk, kblk_per_tap, a_box_bytes; };

// A_MODE 0: plain [planes][M][K];  1: conv taps over the parity layout
//
// Accumulation: a tensor core that adds products into its fp32 accumulator without round-to-nearest biases long-K sums
// (an accumulator that rounds toward zero gave an order of magnitude larger logit errors on the 0.6B model than an fp32
// FMA GEMM).  So the tensor core only accumulates CH k-blocks (K = 256) at a time into the wgmma registers; each
// finished chunk is added into a second set of fp32 registers (round-to-nearest).
template <int A_MODE, int EPI_MODE>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
               int M, int N, int K, int nplanes, int tiles_m, int tiles_n, int splits, ConvGeom cg, GemmEpi E) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    float* epi_slab = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + 256);   // CONS_WARPS x [16][SLAB_LD]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // Persistent CTAs: work item = (m tile, n tile, k split), dealt round-robin (item = blockIdx.x + i * gridDim.x; n
    // fastest so that concurrently running CTAs share the A tile in L2).  The producer keeps a GLOBAL stage counter
    // across items, so the TMA loads of the next tile are issued while the consumers run the previous tile's epilogue.
    // split-K: `splits` items share one output tile, each contracts num_kb k-blocks starting at kb0 and writes its
    // partial tile to row block z of a [splits][M][N] fp32 workspace (plain epilogue, see launch_gemm_tc)
    const int num_kb = K / BK / splits;
    const int n_items = tiles_m * tiles_n * splits;

    if (threadIdx.x == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
    }
    __syncthreads();

    // item -> tile coordinates
    auto item_coords = [&](int item, int& n0, int& m0, int& chunk, int& oh0, int& z) {
        const int nt = item % tiles_n; int rest = item / tiles_n;
        const int mt = rest % tiles_m; z = rest / tiles_m;
        n0 = nt * BN; m0 = mt * BM; chunk = 0; oh0 = 0;
        if (A_MODE == 1) { chunk = mt / cg.tiles_per_chunk; oh0 = (mt % cg.tiles_per_chunk) * cg.box_h; }
    };

    if (warp == 0 && lane == 0) {
        // ================= TMA producer =================
        // TMA always delivers (and counts) the full box, zero-filling out-of-bounds elements; the conv box
        // has OW*box_h (<= 128) rows, the remaining rows of the MMA tile are never read back.
        const uint32_t a_bytes = (A_MODE == 0) ? (uint32_t)TILE_A_BYTES : (uint32_t)cg.a_box_bytes;
        const uint32_t stage_tx = (uint32_t)nplanes * a_bytes + (uint32_t)TILE_B_BYTES;
        uint32_t kg = 0;                                   // global k-block counter (ring position)
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            int n0, m0, chunk, oh0, z;
            item_coords(item, n0, m0, chunk, oh0, z);
            const int kb0 = z * num_kb;
            for (int kb = 0; kb < num_kb; ++kb, ++kg) {
                const int s = kg % STAGES; const uint32_t par = (kg / STAGES) & 1;
                mbar_wait(&empty[s], par ^ 1);
                uint8_t* st = smem + s * STAGE_BYTES;
                mbar_expect_tx(&full[s], stage_tx);
                if (A_MODE == 0) {
                    for (int p = 0; p < nplanes; ++p) tma_load_3d(st + p * TILE_A_BYTES, &mapA, (kb0 + kb) * BK, m0, p, &full[s]);
                } else {
                    const int tap = kb / cg.kblk_per_tap, cb = kb % cg.kblk_per_tap;
                    const int kh = tap / 3, kw = tap % 3;
                    const int ph = (kh == 1) ? 0 : 1, pw = (kw == 1) ? 0 : 1;
                    const int h = oh0 + (kh == 0 ? -1 : 0), w = (kw == 0 ? -1 : 0);
                    for (int p = 0; p < nplanes; ++p)
                        tma_load_5d(st + p * TILE_A_BYTES, &mapA, cb * BK, w, h, (chunk * 2 + ph) * 2 + pw, p, &full[s]);
                }
                tma_load_2d(st + 3 * TILE_A_BYTES, &mapB, (kb0 + kb) * BK, n0, &full[s]);
            }
        }
    } else if (warp >= 4) {
        // ================= wgmma consumers + epilogue =================
        // Warpgroup h (0 / 1) computes tile rows [64h, 64h + 64); in the wgmma accumulator layout warp q of the
        // warpgroup holds rows 16q + lane / 4 and 16q + lane / 4 + 8, columns 8j + 2 (lane % 4) + {0, 1}, j < 16.
        const int half = (warp >> 2) - 1, q = warp & 3;
        const int cw = warp - 4;                       // consumer warp index: its epilogue slab
        float acc[64], sum[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] = 0.f;
        uint32_t kg = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            int n0, m0, chunk, oh0, z;
            item_coords(item, n0, m0, chunk, oh0, z);
#pragma unroll
            for (int j = 0; j < 64; ++j) sum[j] = 0.f;
            consume_k_blocks<STAGES, STAGE_BYTES, TILE_A_BYTES, BK, CH>(smem, full, empty, half, lane, num_kb, nplanes, kg, acc, sum);
            // Store through a per-warp shared-memory transpose, 32 columns at a time.  Each lane holds column PAIRS of two
            // rows; staged as [16][SLAB_LD] floats, lane l re-reads columns 4 (l & 7).. of rows 4 i + (l >> 3): a warp store
            // instruction covers 4 rows x 128 contiguous bytes.
            float* slab = epi_slab + cw * (16 * SLAB_LD);
            const int lr = lane >> 3, lc = (lane & 7) * 4;
#pragma unroll
            for (int g = 0; g < BN / 32; ++g) {
                stage_slab<SLAB_LD>(slab, sum, g, lane);
                const int n = n0 + g * 32 + lc;
                const bool ncol = n < N;
                const float4 bias4 = ncol ? epi_bias4<EPI_MODE>(E, n) : make_float4(0.f, 0.f, 0.f, 0.f);
                float4 v[4]; long long mr[4]; EpiIn in[4];            // 4 rows per lane: every global load first, then the stores
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int rr = half * 64 + q * 16 + 4 * i + lr;   // row inside the tile
                    v[i] = *reinterpret_cast<const float4*>(slab + (4 * i + lr) * SLAB_LD + lc);
                    long long m = -1;
                    if (A_MODE == 0) { if (m0 + rr < M) m = m0 + rr + (long long)z * M; }
                    else {
                        const int oh = oh0 + rr / cg.OW, ow = rr % cg.OW;
                        if (rr < cg.box_h * cg.OW && oh < cg.OH) m = ((long long)chunk * cg.OH + oh) * cg.OW + ow;
                    }
                    mr[i] = (m >= 0 && ncol) ? m : -1;
                    if (mr[i] >= 0) in[i] = epi_fetch4<EPI_MODE>(E, N, (int)mr[i], n);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (mr[i] >= 0) epi_store4<EPI_MODE>(E, N, (int)mr[i], n, v[i], bias4, in[i]);
                __syncwarp();
            }
        }
    }
}

// split-K second pass: sum the partial tiles in a fixed order, then the GEMM's own epilogue (bias / GELU / residual / split3)
template <int MODE>
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, int S, int M, int N, GemmEpi E) {
    const int n8 = N / 8;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= M * n8) return;
    const int m = idx / n8, n = (idx - m * n8) * 8;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
    for (int sp = 0; sp < S; ++sp) {
        const float* src = ws + ((size_t)sp * M + m) * N + n;
        const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
        v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
    }
    epi_store8<MODE>(E, N, m, n, v);
}

// ---- host: tensor maps ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        ASRB_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
        ASRB_REQUIRE(p != nullptr && qr == cudaDriverEntryPointSuccess, ASRB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
        fn = (EncodeTiledFn)p;
    }
    return fn;
}
static CUtensorMap make_map(const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box) {
    CUtensorMap m;
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = get_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw Error(ASRB_ERR_CUDA, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
    return m;
}

// Tensor maps depend only on (base, shape, strides, box): encode once per distinct operand instead of on every launch
// (a clip issues ~400 GEMMs over a few dozen distinct operands).  Thread-local: sessions on different host threads.
struct MapKey {
    const void* base; int rank; cuuint64_t d[5]; cuuint64_t s[4]; cuuint32_t b[5];
    bool operator<(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) < 0; }
};
static const CUtensorMap& cached_map(const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box) {
    static thread_local std::map<MapKey, CUtensorMap> cache;
    MapKey k;
    memset(&k, 0, sizeof(k));
    k.base = base; k.rank = rank;
    for (int i = 0; i < rank; ++i) { k.d[i] = dims[i]; k.b[i] = box[i]; }
    for (int i = 0; i + 1 < rank; ++i) k.s[i] = strides_bytes[i];
    auto it = cache.find(k);
    if (it == cache.end()) {
        if (cache.size() > 4096) cache.clear();
        it = cache.emplace(k, make_map(base, rank, dims, strides_bytes, box)).first;
    }
    return it->second;
}

static int sm_count() {
    int dev = 0, n = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}
static size_t smem_bytes() { return (size_t)STAGES * STAGE_BYTES + 1024 + 256 + CONS_WARPS * 16 * SLAB_LD * 4; }   // stages + alignment slack + barriers + epilogue slabs

}  // namespace tc

const CUtensorMap& tc_cached_map(const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                                 const cuuint32_t* box) {
    return tc::cached_map(base, rank, dims, strides_bytes, box);
}

GemmPlan plan_gemm_tc(const GemmA& A, int N, const GemmEpi& E, int sms) {
    using namespace tc;
    GemmPlan p;
    if (A.K % BK != 0 || A.M <= 0 || N <= 0 || N % 8 != 0) return p;
    if (A.nplanes < 1 || A.nplanes > 3) return p;
    if (A.mode == A_PLAIN) {
        if (A.plane_stride % 8 != 0 && A.nplanes > 1) return p;
        if (E.mode != EPI_PLAIN && E.mode != EPI_SWIGLU && E.mode != EPI_CONVOUT) return p;
        p.tiles_n = (N + BN - 1) / BN; p.tiles_m = (A.M + BM - 1) / BM;
        // Split-K for plain GEMMs that cannot fill the GPU (e.g. prefill o_proj / down_proj: 32 tiles, K = 2048 / 3072;
        // encoder fc2: 28 tiles, K = 3584): such a CTA is bound by its own TMA load rate (64 KB of operands per k-block),
        // so 2-4 CTAs per tile finish 2-4x sooner; a second pass sums the partial tiles (fixed order) and applies the
        // epilogue.  Deterministic; costs one extra fp32 round trip of the tile through L2.
        const int tiles = p.tiles_n * p.tiles_m, kblocks = A.K / BK;
        if ((E.mode == EPI_PLAIN || E.mode == EPI_CONVOUT) && E.splitk_ws && tiles <= 64 && (size_t)4 * A.M * N <= SPLITK_WS_FLOATS) {
            for (int sp = 4; sp >= 2; --sp)
                if (kblocks % sp == 0 && kblocks / sp >= 6 && tiles * sp <= sms + sms / 12) { p.splits = sp; break; }   // at most ~1.1 waves
        }
    } else {
        if (A.cpad % BK != 0 || A.OW > BM || A.OW <= 0 || A.OH <= 0) return p;
        if (E.mode != EPI_CONV_PARITY && E.mode != EPI_CONV_FEAT) return p;
        p.box_h = std::min(A.OH, BM / A.OW);
        p.tiles_n = (N + BN - 1) / BN;
        p.tiles_m = (A.M / (A.OH * A.OW)) * ((A.OH + p.box_h - 1) / p.box_h);
    }
    p.grid = std::min(p.tiles_m * p.tiles_n * p.splits, sms);
    p.tc = p.grid > 0;
    return p;
}

bool launch_gemm_tc(const GemmA& A, const bf16* W, int N, const GemmEpi& Ein, cudaStream_t st) {
    using namespace tc;
    const GemmEpi& E = Ein;
    // ASRB_GEMM_TIME=1: CUDA-event time of every launch (synchronises per launch; measurement runs only)
    static const bool time_all = getenv("ASRB_GEMM_TIME") != nullptr;
    struct Timer {
        bool on; cudaEvent_t e0, e1; int M, N, K, mode; cudaStream_t st;
        Timer(bool o, int M_, int N_, int K_, int mode_, cudaStream_t s) : on(o), M(M_), N(N_), K(K_), mode(mode_), st(s) {
            if (on) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
        }
        ~Timer() {
            if (!on) return;
            cudaEventRecord(e1, st); cudaEventSynchronize(e1);
            float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1);
            fprintf(stderr, "[gemm_tc time] M=%d N=%d K=%d epi=%d %.1f us\n", M, N, K, mode, ms * 1000.f);
            cudaEventDestroy(e0); cudaEventDestroy(e1);
        }
    } timer(time_all, A.M, N, A.K, E.mode, st);
    const GemmPlan pl = plan_gemm_tc(A, N, E, sm_count());
    if (!pl.tc) return false;
    if ((reinterpret_cast<uintptr_t>(A.a) & 15) || (reinterpret_cast<uintptr_t>(W) & 15)) return false;
    // B: [N][K] row-major bf16
    cuuint64_t bd[2] = {(cuuint64_t)A.K, (cuuint64_t)N};
    cuuint64_t bs[1] = {(cuuint64_t)A.K * 2};
    cuuint32_t bb[2] = {(cuuint32_t)BK, (cuuint32_t)BN};
    const CUtensorMap mapB = cached_map(W, 2, bd, bs, bb);
    ConvGeom cg{};
    const size_t smem = smem_bytes();
    const int tiles_m = pl.tiles_m, tiles_n = pl.tiles_n;
    if (A.mode == A_PLAIN) {
        cuuint64_t ad[3] = {(cuuint64_t)A.K, (cuuint64_t)A.M, (cuuint64_t)3};
        cuuint64_t as[2] = {(cuuint64_t)A.lda * 2, (cuuint64_t)A.plane_stride * 2};
        cuuint32_t ab[3] = {(cuuint32_t)BK, (cuuint32_t)BM, 1};
        const CUtensorMap mapA = cached_map(A.a, 3, ad, as, ab);
        if (pl.splits > 1) {
            GemmEpi P;                               // partial tiles: plain fp32 rows [split][M][N]
            P.out_f32 = E.splitk_ws; P.ldo = N;
            // (the attribute is per device: set on every launch, a process may hold contexts on several GPUs)
            ASRB_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<0, EPI_PLAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            gemm_tc_kernel<0, EPI_PLAIN><<<pl.grid, NTHREADS, smem, st>>>(mapA, mapB, A.M, N, A.K, A.nplanes, tiles_m, tiles_n, pl.splits, cg, P);
            const int work = A.M * (N / 8);
            if (E.mode == EPI_PLAIN) splitk_reduce_kernel<EPI_PLAIN><<<(work + 255) / 256, 256, 0, st>>>(E.splitk_ws, pl.splits, A.M, N, E);
            else splitk_reduce_kernel<EPI_CONVOUT><<<(work + 255) / 256, 256, 0, st>>>(E.splitk_ws, pl.splits, A.M, N, E);
            ASRB_CUDA_CHECK(cudaGetLastError());
            if (E.extra_launches) *E.extra_launches += 1;
            return true;
        }
#define ASRB_TC_LAUNCH(AM, EM)                                                                                         \
    {                                                                                                                  \
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<AM, EM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        gemm_tc_kernel<AM, EM><<<pl.grid, NTHREADS, smem, st>>>(mapA, mapB, A.M, N, A.K, A.nplanes, tiles_m, tiles_n, 1, cg, E); \
    }
        if (E.mode == EPI_PLAIN) ASRB_TC_LAUNCH(0, EPI_PLAIN)
        else if (E.mode == EPI_SWIGLU) ASRB_TC_LAUNCH(0, EPI_SWIGLU)
        else ASRB_TC_LAUNCH(0, EPI_CONVOUT)
    } else {
        const int chunks = A.M / (A.OH * A.OW);
        cg.OH = A.OH; cg.OW = A.OW; cg.box_h = pl.box_h;
        cg.tiles_per_chunk = (A.OH + cg.box_h - 1) / cg.box_h; cg.kblk_per_tap = A.cpad / BK;
        cg.a_box_bytes = A.OW * cg.box_h * BK * 2;
        // [plane][chunk*4 + ph*2 + pw][Hh][Wh][cpad]
        cuuint64_t ad[5] = {(cuuint64_t)A.cpad, (cuuint64_t)A.Wh, (cuuint64_t)A.Hh, (cuuint64_t)chunks * 4, 3};
        cuuint64_t as[4] = {(cuuint64_t)A.cpad * 2, (cuuint64_t)A.Wh * A.cpad * 2, (cuuint64_t)A.Hh * A.Wh * A.cpad * 2,
                            (cuuint64_t)A.plane_stride * 2};
        cuuint32_t ab[5] = {(cuuint32_t)BK, (cuuint32_t)A.OW, (cuuint32_t)cg.box_h, 1, 1};
        const CUtensorMap mapA = cached_map(A.a, 5, ad, as, ab);
        if (E.mode == EPI_CONV_PARITY) ASRB_TC_LAUNCH(1, EPI_CONV_PARITY)
        else ASRB_TC_LAUNCH(1, EPI_CONV_FEAT)
#undef ASRB_TC_LAUNCH
    }
    ASRB_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace asrb
