// segment.cu -- cut points of long recordings at low-energy windows (DESIGN.md section 4.6).
//
// Input: the 16 kHz mono f32 files that asrb_ingest_long wrote into the session's long-audio buffer.  Window energy
// e[j] = sum x[i]^2 over i in [160 j, 160 j + 1600) (100 ms every 10 ms), in fp64.  Cut rule, per file of N samples:
// c_0 = 0; while N - c_k > max_seg, c_{k+1} = the window centre p = 160 j + 800 with the least e[j] among
// c_k + max_seg - search <= p <= min(c_k + max_seg, N - 16000), ties to the largest p.  Segments [c_k, c_{k+1}) and
// [c_K, N): each at most max_seg samples, the last at least 1 s.
//
// Two kernels, both deterministic (no atomics, fixed summation orders):
//   segment_energy_kernel  one warp per 160-sample block: lane l squares samples l, l+32, .., l+128 in that order, then
//                          an xor butterfly; blk[m] = the block's sum of squares.  Grid-stride over every file's blocks.
//   segment_cut_kernel     one CTA per file; the cuts are sequential, each one block-parallel: thread t scans candidates
//                          j0 + t, j0 + t + T, .. with e[j] = blk[j] + .. + blk[j + 9] added left to right, then a
//                          (energy, -j) minimum over the CTA.  That order is total, so the reduction order is irrelevant.
// Every candidate window lies inside the file (p <= N - 16000), so only full blocks are read.
#include <cmath>
#include "internal.h"

namespace asrb {

static constexpr int SEG_HOP = 160, SEG_WIN_BLOCKS = 10, SEG_THREADS = 256;

__global__ void __launch_bounds__(SEG_THREADS)
segment_energy_kernel(const float* __restrict__ x, const int64_t* __restrict__ off, const int64_t* __restrict__ boff,
                      int n_files, double* __restrict__ blk) {
    const int lane = threadIdx.x & 31;
    const int64_t total = boff[n_files];
    const int64_t warps = (int64_t)gridDim.x * (SEG_THREADS / 32);
    int f = 0;
    for (int64_t g = (int64_t)blockIdx.x * (SEG_THREADS / 32) + (threadIdx.x >> 5); g < total; g += warps) {
        while (g >= boff[f + 1]) ++f;                        // g only grows: files are visited in order
        const float* p = x + off[f] + (g - boff[f]) * SEG_HOP;
        double v = 0.0;
#pragma unroll
        for (int i = 0; i < SEG_HOP / 32; ++i) { const double s = (double)p[lane + 32 * i]; v = fma(s, s, v); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) blk[g] = v;
    }
}

// (e, j) is better than (be, bj): less energy, or the same energy at a later window.  NaN counts as +inf.
__device__ __forceinline__ bool seg_better(double e, int64_t j, double be, int64_t bj) {
    return e < be || (e == be && j > bj);
}

__global__ void __launch_bounds__(SEG_THREADS)
segment_cut_kernel(const double* __restrict__ blk, const int64_t* __restrict__ boff, const int64_t* __restrict__ n,
                   const int64_t* __restrict__ coff, int64_t max_seg, int64_t search, int64_t* __restrict__ cuts,
                   int64_t* __restrict__ ncuts) {
    __shared__ double red_e[SEG_THREADS / 32];
    __shared__ int64_t red_j[SEG_THREADS / 32];
    const int f = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t N = n[f];
    const double* b = blk + boff[f];
    int64_t* out = cuts + coff[f];
    int64_t c = 0, k = 0;
    while (N - c > max_seg) {
        const int64_t lo = c + max_seg - search, hi = min(c + max_seg, N - 16000);
        const int64_t j0 = (lo - SEG_HOP * SEG_WIN_BLOCKS / 2) / SEG_HOP, j1 = (hi - SEG_HOP * SEG_WIN_BLOCKS / 2) / SEG_HOP;
        double be = INFINITY; int64_t bj = -1;
        for (int64_t j = j0 + threadIdx.x; j <= j1; j += SEG_THREADS) {
            double e = 0.0;
#pragma unroll
            for (int i = 0; i < SEG_WIN_BLOCKS; ++i) e += b[j + i];
            if (isnan(e)) e = INFINITY;
            if (seg_better(e, j, be, bj)) { be = e; bj = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double oe = __shfl_xor_sync(0xffffffffu, be, o);
            const int64_t oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (seg_better(oe, oj, be, bj)) { be = oe; bj = oj; }
        }
        if (lane == 0) { red_e[warp] = be; red_j[warp] = bj; }
        __syncthreads();
        be = red_e[0]; bj = red_j[0];
        for (int w = 1; w < SEG_THREADS / 32; ++w)
            if (seg_better(red_e[w], red_j[w], be, bj)) { be = red_e[w]; bj = red_j[w]; }
        __syncthreads();                                     // everyone has read red_* before the next cut writes them
        c = bj * SEG_HOP + SEG_HOP * SEG_WIN_BLOCKS / 2;     // j0 <= bj <= j1: every candidate beats (inf, -1)
        if (threadIdx.x == 0) out[k] = c;
        ++k;
    }
    if (threadIdx.x == 0) ncuts[f] = k;
}

// d_plan: off[F] | n[F] | boff[F + 1] (prefix of floor(n / 160) blocks) | coff[F] (prefix of cut capacities)
void launch_segment(const float* d_long, const int64_t* d_plan, int n_files, int64_t total_blocks, int64_t max_seg,
                    int64_t search, double* d_blk, int64_t* d_cuts, int64_t* d_ncuts, int sm_count, cudaStream_t st) {
    const int64_t *off = d_plan, *n = off + n_files, *boff = n + n_files, *coff = boff + n_files + 1;
    if (total_blocks > 0) {
        const int64_t want = (total_blocks + SEG_THREADS / 32 - 1) / (SEG_THREADS / 32);
        const int grid = (int)std::min<int64_t>(want, (int64_t)sm_count * 8);
        segment_energy_kernel<<<grid, SEG_THREADS, 0, st>>>(d_long, off, boff, n_files, d_blk);
    }
    segment_cut_kernel<<<n_files, SEG_THREADS, 0, st>>>(d_blk, boff, n, coff, max_seg, search, d_cuts, d_ncuts);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

}  // namespace asrb
