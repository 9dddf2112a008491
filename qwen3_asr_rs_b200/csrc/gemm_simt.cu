// gemm_simt.cu -- fp32 CUDA-core GEMM with the shared A-loaders / epilogues.
// Role: (1) on-device reference for the wgmma GEMM (same inputs, same epilogues),
// (2) the path for shapes the tensor-core kernel does not cover.  64x64x16 tiles, 256 threads,
// 4x4 register blocking, fp32 accumulate of exact bf16*bf16 products.
//
// Accumulation: as in the wgmma GEMM (gemm_tc.cu), the products of each K = 256 chunk are summed in one set of fp32
// registers and each finished chunk is added into a second set.  One running sum over all of K grows its rounding error
// with K: at K = 7680 (conv_out) it measured 10x the error of a blocked fp32 GEMM on an H100; with chunks, under 1x.
#include "internal.h"
#include "epilogue.cuh"

namespace asrb {

static constexpr int BM = 64, BN = 64, BK = 16, CHUNK_K = 256;

__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmA A, const bf16* __restrict__ W, int N, GemmEpi E) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Ws[BK][BN + 4];
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;   // 16 x 16 threads, each 4(m) x 4(n)
    float acc[4][4], sum[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = sum[i][j] = 0.f;
    for (int k0 = 0; k0 < A.K; k0 += BK) {
        // load tiles: 64x16 elements each, 256 threads x 4
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int idx = tid + i * 256;
            int r = idx >> 4, kk = idx & 15;
            int m = m0 + r, k = k0 + kk;
            As[kk][r] = (m < A.M && k < A.K) ? load_a(A, m, k) : 0.f;
            int n = n0 + r;
            Ws[kk][r] = (n < N && k < A.K) ? __bfloat162float(W[(size_t)n * A.K + k]) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[4], w[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) w[j] = Ws[kk][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
        __syncthreads();
        if ((k0 + BK) % CHUNK_K == 0 || k0 + BK >= A.K) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) { sum[i][j] += acc[i][j]; acc[i][j] = 0.f; }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int m = m0 + ty * 4 + i;
        if (m >= A.M) continue;
#pragma unroll
        for (int j = 0; j < 4; j += 2) {
            int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            epi_store2(E, N, m, n, sum[i][j], sum[i][j + 1], n + 1 < N);
        }
    }
}

void launch_gemm_simt(const GemmA& A, const bf16* W, int N, const GemmEpi& E, cudaStream_t st) {
    dim3 grid((N + BN - 1) / BN, (A.M + BM - 1) / BM);
    if (A.M <= 0 || N <= 0) return;
    gemm_simt_kernel<<<grid, 256, 0, st>>>(A, W, N, E);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

std::atomic<int64_t> g_gemm_simt_fallbacks{0}, g_gemm_tc_launches{0};

void launch_gemm(const GemmA& A, const bf16* W, int N, const GemmEpi& E, int impl, cudaStream_t st) {
    if (impl == GEMM_TC) {
        if (launch_gemm_tc(A, W, N, E, st)) { g_gemm_tc_launches += 1; return; }
        g_gemm_simt_fallbacks += 1;        // counted, never silent: asrb_session_stats()[3] (bench.py requires 0)
    }
    launch_gemm_simt(A, W, N, E, st);
}

}  // namespace asrb
