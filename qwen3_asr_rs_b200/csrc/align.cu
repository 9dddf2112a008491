// align.cu -- word-timing alignment from the decoder's audio attention (asrb_align_ids, DESIGN.md 4.10).
//
//   align_probs_kernel   softmax over the utterance's audio keys of each aligned row, one listed head of one layer
//   align_zscore_kernel  per (head, column) mean / population std over the rows, z-scores in place (std = 0: z = 0;
//                        a column of equal values has std exactly 0)
//   align_median_kernel  per element: width-7 median along the columns (mirror padding) of every listed head of the
//                        layer, added into M in list order; the last listed layer divides by the head count
//   align_dtw_kernel     one CTA per utterance: DTW on -M over anti-diagonals, 2-bit trace, backtrace on the device
#include <cmath>
#include "internal.h"

namespace asrb {

namespace {

constexpr int PROB_ROWS = 16;     // aligned rows per CTA of align_probs_kernel
constexpr int PROB_KEYS = 32;     // audio keys per shared-memory tile
constexpr int PROB_THREADS = 128;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// grid (row tiles, heads of the layer, utterances).  Scores: an fmaf chain over d, then a divide by sqrt(hd), as in
// attn_f32_kernel; then per row max, sum of expf(s - max) and e / sum, each reduced in a fixed order.
__global__ void __launch_bounds__(PROB_THREADS) align_probs_kernel(AlignProbArgs a) {
    extern __shared__ float sm[];
    const int b = blockIdx.z, hl = blockIdx.y, hd = a.hd;
    const int N = a.N[b], T = a.T[b];
    const int i0 = blockIdx.x * PROB_ROWS;
    if (i0 >= N || T <= 0) return;
    const int nr = min(PROB_ROWS, N - i0);
    const int h = a.heads[hl], g = h / a.group;
    float* qs = sm;                                  // [PROB_ROWS][hd]
    float* ks = sm + PROB_ROWS * hd;                 // [PROB_KEYS][hd + 1]
    const float* q = a.q + (size_t)(a.qrow0[b] + i0) * a.ldq + (size_t)h * hd;
    for (int e = threadIdx.x; e < nr * hd; e += blockDim.x) qs[e] = q[(size_t)(e / hd) * a.ldq + e % hd];
    const float* kb = a.k + (size_t)a.slot[b] * a.seg_stride + (size_t)g * a.head_stride + (size_t)a.a0[b] * hd;
    float* P = a.P + (size_t)hl * a.plane + a.moff[b] + (size_t)i0 * T;
    const float div = sqrtf((float)hd);
    for (int j0 = 0; j0 < T; j0 += PROB_KEYS) {
        const int nk = min(PROB_KEYS, T - j0);
        __syncthreads();
        for (int e = threadIdx.x; e < nk * hd; e += blockDim.x) ks[(e / hd) * (hd + 1) + e % hd] = kb[(size_t)(j0 + e / hd) * hd + e % hd];
        __syncthreads();
        for (int p = threadIdx.x; p < nr * PROB_KEYS; p += blockDim.x) {
            const int r = p / PROB_KEYS, jj = p % PROB_KEYS;
            if (jj >= nk) continue;
            const float* qr = qs + r * hd;
            const float* kr = ks + jj * (hd + 1);
            float acc = 0.f;
            for (int d = 0; d < hd; ++d) acc = fmaf(qr[d], kr[d], acc);
            P[(size_t)r * T + j0 + jj] = acc / div;
        }
    }
    __syncthreads();                                 // the raw scores of the tile's rows are visible to the whole CTA
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int r = warp; r < nr; r += nw) {
        float* row = P + (size_t)r * T;
        float mx = -INFINITY;
        for (int j = lane; j < T; j += 32) mx = fmaxf(mx, row[j]);
        mx = warp_max(mx);
        float sum = 0.f;
        for (int j = lane; j < T; j += 32) sum += expf(row[j] - mx);
        sum = warp_sum(sum);
        for (int j = lane; j < T; j += 32) row[j] = expf(row[j] - mx) / sum;
    }
}

// grid (column tiles, heads of the layer, utterances): thread = column j of one head's [N][T] plane
__global__ void align_zscore_kernel(AlignFoldArgs a) {
    const int b = blockIdx.z, hl = blockIdx.y;
    const int N = a.N[b], T = a.T[b];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= T) return;
    float* P = a.P + (size_t)hl * a.plane + a.moff[b] + j;
    // the mean as P[0] + mean(P - P[0]): a column of equal values has mean == P[0] exactly, so std = 0 and z = 0 (a
    // plain fp32 sum of N equal values rounds, which left such columns at z = +-1)
    const float p0 = P[0];
    float sum = 0.f;
    for (int i = 0; i < N; ++i) sum += P[(size_t)i * T] - p0;
    const float mean = p0 + sum / (float)N;
    float var = 0.f;
    for (int i = 0; i < N; ++i) { const float d = P[(size_t)i * T] - mean; var = fmaf(d, d, var); }
    const float sd = sqrtf(var / (float)N);
    for (int i = 0; i < N; ++i) {
        float* p = P + (size_t)i * T;
        *p = sd > 0.f ? (*p - mean) / sd : 0.f;
    }
}

__device__ __forceinline__ void cswap(float& x, float& y) { const float lo = fminf(x, y), hi = fmaxf(x, y); x = lo; y = hi; }
__device__ __forceinline__ int mirror(int j, int T) { return j < 0 ? -j : (j >= T ? 2 * (T - 1) - j : j); }

// grid (element tiles, utterances): thread = element (i, j) of utterance b's M; the layer's heads in list order
__global__ void align_median_kernel(AlignFoldArgs a) {
    const int b = blockIdx.y;
    const int N = a.N[b], T = a.T[b];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N * T) return;
    const int i = e / T, j = e % T;
    float acc = a.M[a.moff[b] + e];
    for (int hl = 0; hl < a.nheads; ++hl) {
        const float* z = a.P + (size_t)hl * a.plane + a.moff[b] + (size_t)i * T;
        float med;
        if (T <= 3) med = z[j];
        else {
            float v[7];
#pragma unroll
            for (int t = 0; t < 7; ++t) v[t] = z[mirror(j + t - 3, T)];
            // sorting network for 7 inputs (16 compare-exchanges); the median is v[3]
            cswap(v[0], v[6]); cswap(v[2], v[3]); cswap(v[4], v[5]);
            cswap(v[0], v[2]); cswap(v[1], v[4]); cswap(v[3], v[6]);
            cswap(v[0], v[1]); cswap(v[2], v[5]); cswap(v[3], v[4]);
            cswap(v[1], v[2]); cswap(v[4], v[6]);
            cswap(v[2], v[3]); cswap(v[4], v[5]);
            cswap(v[1], v[2]); cswap(v[3], v[4]); cswap(v[5], v[6]);
            med = v[3];
        }
        acc += med;
    }
    if (a.count > 0) acc = acc / (float)a.count;
    a.M[a.moff[b] + e] = acc;
}

constexpr int DTW_THREADS = 256;

// one CTA per utterance.  Cost C[i][j] (0 <= i <= N, 0 <= j <= T) over anti-diagonals d = i + j, the last three in
// shared memory indexed by i; trace 2 bits per cell (i, j >= 1) at bit 2 * ((i - 1) * T + j - 1), in shared memory when
// a.smem_trace, else in the utterance's global words (zeroed by the host).  Then the backtrace from (N, T) by one thread:
// start[i] = least column of the path in row i.
__global__ void __launch_bounds__(DTW_THREADS) align_dtw_kernel(AlignDtwArgs a) {
    extern __shared__ float sm[];
    const int b = blockIdx.x;
    const int N = a.N[b], T = a.T[b];
    const float* M = a.M + a.moff[b];
    float* diag = sm;                                              // [3][N + 1]
    uint32_t* trace = a.smem_trace[b] ? reinterpret_cast<uint32_t*>(sm + 3 * (N + 1)) : a.trace + a.toff[b];
    const size_t words = ((size_t)N * T + 15) / 16;
    if (a.smem_trace[b]) for (size_t w = threadIdx.x; w < words; w += blockDim.x) trace[w] = 0u;
    if (threadIdx.x == 0) { diag[0] = 0.f; diag[(N + 1) + 0] = INFINITY; diag[(N + 1) + 1] = INFINITY; }
    __syncthreads();
    for (int d = 2; d <= N + T; ++d) {
        float* cur = diag + (d % 3) * (N + 1);
        const float* p1 = diag + ((d + 2) % 3) * (N + 1);         // diagonal d - 1
        const float* p2 = diag + ((d + 1) % 3) * (N + 1);         // diagonal d - 2
        const int ilo = max(0, d - T), ihi = min(N, d);
        for (int i = ilo + threadIdx.x; i <= ihi; i += blockDim.x) {
            const int j = d - i;
            if (i == 0 || j == 0) { cur[i] = INFINITY; continue; }
            const float c0 = p2[i - 1], c1 = p1[i - 1], c2 = p1[i];
            float c; uint32_t t;
            if (c0 < c1 && c0 < c2) { c = c0; t = 0u; }
            else if (c1 < c0 && c1 < c2) { c = c1; t = 1u; }
            else { c = c2; t = 2u; }
            cur[i] = -M[(size_t)(i - 1) * T + (j - 1)] + c;
            if (t) {
                const size_t cell = (size_t)(i - 1) * T + (j - 1);
                atomicOr(trace + cell / 16, t << (2 * (cell % 16)));
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int* start = a.start + a.soff[b];
        int i = N, j = T;
        while (i > 0 && j > 0) {
            start[i - 1] = j - 1;
            const size_t cell = (size_t)(i - 1) * T + (j - 1);
            const uint32_t t = (trace[cell / 16] >> (2 * (cell % 16))) & 3u;
            if (t == 0u) { --i; --j; } else if (t == 1u) --i; else --j;
        }
        // the border is never entered before (0, 0) (C is +inf on it): i == j == 0 here
    }
}

}  // namespace

size_t align_probs_smem(int hd) { return (size_t)(PROB_ROWS * hd + PROB_KEYS * (hd + 1)) * sizeof(float); }

void launch_align_probs(const AlignProbArgs& a, int B, int maxN, cudaStream_t st) {
    const size_t smem = align_probs_smem(a.hd);
    ASRB_REQUIRE(smem <= ALIGN_PROBS_SMEM_MAX, ASRB_ERR_INVALID, "align: head_dim too large for the probability kernel");
    ASRB_CUDA_CHECK(cudaFuncSetAttribute(align_probs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((maxN + PROB_ROWS - 1) / PROB_ROWS, a.nheads, B);
    align_probs_kernel<<<grid, PROB_THREADS, smem, st>>>(a);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

void launch_align_fold(const AlignFoldArgs& a, int B, int maxT, int maxNT, cudaStream_t st) {
    align_zscore_kernel<<<dim3((maxT + 127) / 128, a.nheads, B), 128, 0, st>>>(a);
    ASRB_CUDA_CHECK(cudaGetLastError());
    align_median_kernel<<<dim3((maxNT + 255) / 256, B), 256, 0, st>>>(a);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

size_t align_dtw_smem(int N, int T, bool trace_in_smem) {
    return 3 * (size_t)(N + 1) * sizeof(float) + (trace_in_smem ? (((size_t)N * T + 15) / 16) * sizeof(uint32_t) : 0);
}

void launch_align_dtw(const AlignDtwArgs& a, int B, size_t smem, cudaStream_t st) {
    ASRB_CUDA_CHECK(cudaFuncSetAttribute(align_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    align_dtw_kernel<<<B, DTW_THREADS, smem, st>>>(a);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

}  // namespace asrb
