// attention_tc.cu -- flash-style attention on the tensor cores with 3xTF32 error compensation.
//
// Same contract as attention.cu (encoder windows, layers.rs:152-172 + audio_encoder.rs:172-260;
// prefill causal GQA, layers.rs:284-342 + text_decoder.rs:121-131) but the two contractions
// S = Q.K^T and O = P.V run as mma.sync.m16n8k8 TF32 MMAs.  Both operands are fp32 activations, so
// each is split x = hi + lo (hi = tf32(x), lo = tf32(x - hi)) and every product is formed as
// lo*hi + hi*lo + hi*hi with fp32 accumulation: ~2^-21 relative per product, i.e. fp32-grade.
// (The dense wgmma path is kept for weight GEMMs; these are small batched matmuls -- 64x64x128
// per tile -- whose operands change every tile, which is what warp-level MMA is for.)
// CTA = 4 warps x 16 query rows = 64 queries of one head of one segment; K/V tiles of 64 keys are
// staged in padded shared memory (bank-conflict-free fragment loads), online softmax in fp32,
// P goes through a per-warp shared tile to be re-read in A-fragment layout.
#include "internal.h"

namespace asrb {

namespace atc {

static constexpr int QT = 64, KT = 64, THREADS = 128;

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    float r = x - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int HD>
__global__ void __launch_bounds__(THREADS, 1) attn_tc_kernel(AttnParams p) {
    constexpr int QS = HD + 4, VS = HD + 8, PS = KT + 4;
    extern __shared__ float sm[];
    float* Qs = sm;                      // [QT][QS]
    float* Ks = Qs + QT * QS;            // [KT][QS]
    float* Vs = Ks + KT * QS;            // [KT][VS]
    float* Ps = Vs + KT * VS;            // [4][16][PS]
    const int seg = blockIdx.z, h = blockIdx.y;
    const int q0 = p.seg_q0[seg], len = p.seg_len[seg];
    const int qt0 = blockIdx.x * QT;
    if (qt0 >= len) return;
    const int gkv = h / p.group;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const float* kbase; const float* vbase;
    if (p.keys_in_rows) {
        kbase = p.k + (size_t)q0 * p.ldk + (size_t)gkv * p.head_stride;
        vbase = p.v + (size_t)q0 * p.ldk + (size_t)gkv * p.head_stride;
    } else {
        kbase = p.k + (size_t)seg * p.seg_stride + (size_t)gkv * p.head_stride;
        vbase = p.v + (size_t)seg * p.seg_stride + (size_t)gkv * p.head_stride;
    }
    // Q tile (rows beyond len are zero)
    for (int idx = tid; idx < QT * (HD / 4); idx += THREADS) {
        const int r = idx / (HD / 4), c4 = idx - r * (HD / 4);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (qt0 + r < len) v = *reinterpret_cast<const float4*>(p.q + (size_t)(q0 + qt0 + r) * p.ldq + (size_t)h * HD + c4 * 4);
        *reinterpret_cast<float4*>(Qs + r * QS + c4 * 4) = v;
    }
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const int row0 = qt0 + warp * 16 + g;            // this thread's query rows: row0 and row0 + 8
    const int kend = p.causal ? min(len, qt0 + QT) : len;
    const float inv_div = sqrtf((float)HD);
    float* Pw = Ps + warp * 16 * PS;

    for (int kt0 = 0; kt0 < kend; kt0 += KT) {
        __syncthreads();
        for (int idx = tid; idx < KT * (HD / 4); idx += THREADS) {
            const int r = idx / (HD / 4), c4 = idx - r * (HD / 4);
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (kt0 + r < kend) {
                kv = *reinterpret_cast<const float4*>(kbase + (size_t)(kt0 + r) * p.ldk + c4 * 4);
                vv = *reinterpret_cast<const float4*>(vbase + (size_t)(kt0 + r) * p.ldk + c4 * 4);
            }
            *reinterpret_cast<float4*>(Ks + r * QS + c4 * 4) = kv;
            *reinterpret_cast<float4*>(Vs + r * VS + c4 * 4) = vv;
        }
        __syncthreads();
        // ---- S = Q K^T (16 x 64 per warp) ----
        float s[KT / 8][4];
#pragma unroll
        for (int i = 0; i < KT / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll 2
        for (int ks = 0; ks < HD / 8; ++ks) {
            uint32_t ah[4], al[4];
            const float* qa = Qs + (warp * 16 + g) * QS + ks * 8 + t;
            split_tf32(qa[0], ah[0], al[0]);
            split_tf32(qa[8 * QS], ah[1], al[1]);
            split_tf32(qa[4], ah[2], al[2]);
            split_tf32(qa[8 * QS + 4], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < KT / 8; ++nt) {
                uint32_t bh[2], bl[2];
                const float* kb = Ks + (nt * 8 + g) * QS + ks * 8 + t;
                split_tf32(kb[0], bh[0], bl[0]);
                split_tf32(kb[4], bh[1], bl[1]);
                mma_tf32(s[nt], al, bh);
                mma_tf32(s[nt], ah, bl);
                mma_tf32(s[nt], ah, bh);
            }
        }
        // ---- scale, mask, online softmax (rows row0, row0+8; cols nt*8 + 2t, +1) ----
        float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < KT / 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = row0 + (e >> 1) * 8, j = kt0 + nt * 8 + 2 * t + (e & 1);
                const bool valid = (r < len) && (j < len) && (!p.causal || j <= r);
                const float v = valid ? s[nt][e] / inv_div : -INFINITY;
                s[nt][e] = v;
                tmax[e >> 1] = fmaxf(tmax[e >> 1], v);
            }
        }
        float corr[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            tmax[rr] = fmaxf(tmax[rr], __shfl_xor_sync(0xffffffffu, tmax[rr], 1));
            tmax[rr] = fmaxf(tmax[rr], __shfl_xor_sync(0xffffffffu, tmax[rr], 2));
            const float m_new = fmaxf(m_run[rr], tmax[rr]);
            corr[rr] = (m_new == -INFINITY) ? 1.f : expf(m_run[rr] - m_new);
            m_run[rr] = m_new;
        }
        float psum[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < KT / 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int rr = e >> 1;
                const float pv = (m_run[rr] == -INFINITY) ? 0.f : expf(s[nt][e] - m_run[rr]);
                psum[rr] += pv;
                Pw[(g + rr * 8) * PS + nt * 8 + 2 * t + (e & 1)] = pv;
            }
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            psum[rr] += __shfl_xor_sync(0xffffffffu, psum[rr], 1);
            psum[rr] += __shfl_xor_sync(0xffffffffu, psum[rr], 2);
            l_run[rr] = l_run[rr] * corr[rr] + psum[rr];
        }
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) { o[i][0] *= corr[0]; o[i][1] *= corr[0]; o[i][2] *= corr[1]; o[i][3] *= corr[1]; }
        __syncwarp();
        // ---- O += P V (16 x HD per warp) ----
#pragma unroll 2
        for (int ks = 0; ks < KT / 8; ++ks) {
            uint32_t ah[4], al[4];
            const float* pa = Pw + g * PS + ks * 8 + t;
            split_tf32(pa[0], ah[0], al[0]);
            split_tf32(pa[8 * PS], ah[1], al[1]);
            split_tf32(pa[4], ah[2], al[2]);
            split_tf32(pa[8 * PS + 4], ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < HD / 8; ++nt) {
                uint32_t bh[2], bl[2];
                const float* vb = Vs + (ks * 8 + t) * VS + nt * 8 + g;
                split_tf32(vb[0], bh[0], bl[0]);
                split_tf32(vb[4 * VS], bh[1], bl[1]);
                mma_tf32(o[nt], al, bh);
                mma_tf32(o[nt], ah, bl);
                mma_tf32(o[nt], ah, bh);
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int r = row0 + rr * 8;
        if (r >= len) continue;
        const float inv = 1.0f / l_run[rr];
        const size_t base = (size_t)(q0 + r) * p.ldo + (size_t)h * HD;
#pragma unroll
        for (int nt = 0; nt < HD / 8; ++nt) {
            store_split3(p.out_s3, p.plane_stride, base + nt * 8 + 2 * t, o[nt][rr * 2] * inv);
            store_split3(p.out_s3, p.plane_stride, base + nt * 8 + 2 * t + 1, o[nt][rr * 2 + 1] * inv);
        }
    }
}

template <int HD> static size_t smem_bytes() {
    return (size_t)(QT * (HD + 4) + KT * (HD + 4) + KT * (HD + 8) + 4 * 16 * (KT + 4)) * sizeof(float);
}

}  // namespace atc

bool launch_attention_tc(const AttnParams& p, int hd, cudaStream_t st) {
    using namespace atc;
    if (p.nseg <= 0 || p.max_len <= 0) return true;
    if ((p.ldq % 4) || (p.ldk % 4) || (p.head_stride % 4) || (p.seg_stride % 4)) return false;
    if (p.seg_pos0) return false;                // no query position offset here: the simple kernel takes it
    dim3 grid((p.max_len + QT - 1) / QT, p.nheads, p.nseg);
    if (hd == 64) {
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<64>()));   // per device: set on every launch
        attn_tc_kernel<64><<<grid, THREADS, smem_bytes<64>(), st>>>(p);
    } else if (hd == 128) {
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<128>()));   // per device: set on every launch
        attn_tc_kernel<128><<<grid, THREADS, smem_bytes<128>(), st>>>(p);
    } else return false;
    ASRB_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace asrb
