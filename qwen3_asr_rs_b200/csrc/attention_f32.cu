// attention_f32.cu -- register-tiled fp32 flash attention on the CUDA cores (default path).
//
// Same contract as attention.cu (encoder windows, layers.rs:152-172 + audio_encoder.rs:172-260; prefill causal GQA,
// layers.rs:284-342 + text_decoder.rs:121-131).  Both contractions are plain fp32 FMAs, i.e. the arithmetic of the
// reference's tch-CPU matmuls, organised like an SGEMM:
//   CTA = 128 threads = 32 queries of one head of one segment, keys in tiles of 64.
//   S = Q K^T : Q and K tiles are stored TRANSPOSED in shared memory ([d][row]) so that each thread reads its 4 query
//               rows and 4 key columns of one d as two LDS.128 and issues 16 FMAs (4 x 4 register micro-tile).
//   softmax   : online (running max / sum per query row, fp32), rows are reduced over the 16 lanes that share them.
//   O += P V  : P goes through a small shared tile (row-major, read back as broadcasts), V stays row-major; a thread
//               owns 4 rows x HD/16 columns of O.
// 88 KB of shared memory at head_dim 128: two CTAs per SM overlap one CTA's tile loads with the other's FMAs.
// Why not the tensor cores: the operands are fp32 activations that change every tile; the 3xTF32 mma.sync variant
// (attention_tc.cu, kept for comparison: ASRB_ATTN=tc) triples the MMAs and adds the operand splits on the CUDA cores,
// and a wgmma formulation needs both operands split into bf16 planes in shared memory per tile.  The 0.8 GFLOP of a
// prefill layer is ~12 us of fp32 FMA time on the 132 SMs of an H100 (data-sheet rate).
#include "internal.h"

namespace asrb {

namespace af32 {

static constexpr int QT = 32, KT = 64, THREADS = 128, PS = KT + 4;

// OFF: causal segments with a query position offset (p.seg_pos0): query row r is at position pos0 + r and sees keys
// 0..pos0 + r.  A tile's key count still grows with its index, so the tile pairing below stays balanced.
template <int HD, bool OFF>
__global__ void __launch_bounds__(THREADS, 2) attn_f32_kernel(AttnParams p) {
    constexpr int NG = HD / 64;                 // column groups of 64 owned 4 columns at a time by the 16 tx lanes
    extern __shared__ __align__(16) float sm[];
    float* Qt = sm;                             // [HD][QT]   Q tile, transposed
    float* Kt = Qt + HD * QT;                   // [HD][KT]   K tile, transposed
    float* Vs = Kt + HD * KT;                   // [KT][HD]
    float* Ps = Vs + KT * HD;                   // [QT][PS]
    const int seg = blockIdx.z, h = blockIdx.y;
    const int q0 = p.seg_q0[seg], len = p.seg_len[seg];
    const int pos0 = OFF ? p.seg_pos0[seg] : 0;
    const int nqt = (len + QT - 1) / QT;
    const int gkv = h / p.group;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const float* kbase; const float* vbase;
    if (p.keys_in_rows) {
        kbase = p.k + (size_t)q0 * p.ldk + (size_t)gkv * p.head_stride;
        vbase = p.v + (size_t)q0 * p.ldk + (size_t)gkv * p.head_stride;
    } else {
        kbase = p.k + (size_t)seg * p.seg_stride + (size_t)gkv * p.head_stride;
        vbase = p.v + (size_t)seg * p.seg_stride + (size_t)gkv * p.head_stride;
    }
    // Causal segments: a query tile needs keys up to its own end only, so tile x costs ~(x + 1) key tiles.  One CTA takes
    // tiles x and nqt-1-x back to back: every CTA then has the same amount of work (the long tiles alone made the kernel
    // twice as long as its average SM was busy).  Non-causal segments: one tile per CTA.
    const int npass = p.causal ? 2 : 1;
    for (int pass = 0; pass < npass; ++pass) {
    const int qtile = pass == 0 ? (int)blockIdx.x : nqt - 1 - (int)blockIdx.x;
    // causal: CTA x owns tiles x (x < ceil(nqt / 2)) and nqt-1-x (when that is a different, later tile)
    if (qtile >= nqt || qtile < 0 || (p.causal && pass == 0 && 2 * qtile >= nqt) || (pass == 1 && qtile <= (int)blockIdx.x)) continue;
    const int qt0 = qtile * QT;
    __syncthreads();                            // previous pass done with Qt / Ps
    // Q tile, transposed on the way in (lanes run along the rows: conflict-free scalar stores); rows >= len are zero
    {
        constexpr int NQ = QT * (HD / 4) / THREADS;          // 8 (head_dim 128) or 4 (64): one batch
        float4 qr[NQ];
#pragma unroll
        for (int u = 0; u < NQ; ++u) {
            const int idx = tid + u * THREADS, r = idx % QT, c4 = idx / QT;
            qr[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (qt0 + r < len) qr[u] = *reinterpret_cast<const float4*>(p.q + (size_t)(q0 + qt0 + r) * p.ldq + (size_t)h * HD + c4 * 4);
        }
#pragma unroll
        for (int u = 0; u < NQ; ++u) {
            const int idx = tid + u * THREADS, r = idx % QT, c4 = idx / QT;
            Qt[(c4 * 4 + 0) * QT + r] = qr[u].x; Qt[(c4 * 4 + 1) * QT + r] = qr[u].y;
            Qt[(c4 * 4 + 2) * QT + r] = qr[u].z; Qt[(c4 * 4 + 3) * QT + r] = qr[u].w;
        }
    }
    float o[4][NG][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int gq = 0; gq < NG; ++gq) { o[i][gq][0] = o[i][gq][1] = o[i][gq][2] = o[i][gq][3] = 0.f; }
    float m_run[4], l_run[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { m_run[i] = -INFINITY; l_run[i] = 0.f; }
    const int kend = p.causal ? pos0 + min(len, qt0 + QT) : len;
    const float div = sqrtf((float)HD);

    for (int kt0 = 0; kt0 < kend; kt0 += KT) {
        __syncthreads();
        // K tile (transposed) and V tile (row-major); keys >= kend are zero.  Loads are issued in batches of 8 per
        // thread before any of them is used: a rolled loop would pay one L2 round trip per 16 bytes.
        constexpr int NLD = KT * (HD / 4) / THREADS, LB = 8;
        static_assert(NLD % LB == 0, "tile load batches");
#pragma unroll
        for (int b0 = 0; b0 < NLD; b0 += LB) {
            float4 kr[LB];
#pragma unroll
            for (int u = 0; u < LB; ++u) {
                const int idx = tid + (b0 + u) * THREADS, r = idx % KT, c4 = idx / KT;
                kr[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (kt0 + r < kend) kr[u] = *reinterpret_cast<const float4*>(kbase + (size_t)(kt0 + r) * p.ldk + c4 * 4);
            }
#pragma unroll
            for (int u = 0; u < LB; ++u) {
                const int idx = tid + (b0 + u) * THREADS, r = idx % KT, c4 = idx / KT;
                Kt[(c4 * 4 + 0) * KT + r] = kr[u].x; Kt[(c4 * 4 + 1) * KT + r] = kr[u].y;
                Kt[(c4 * 4 + 2) * KT + r] = kr[u].z; Kt[(c4 * 4 + 3) * KT + r] = kr[u].w;
            }
        }
#pragma unroll
        for (int b0 = 0; b0 < NLD; b0 += LB) {
            float4 vr[LB];
#pragma unroll
            for (int u = 0; u < LB; ++u) {
                const int idx = tid + (b0 + u) * THREADS, r = idx / (HD / 4), c4 = idx - r * (HD / 4);
                vr[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (kt0 + r < kend) vr[u] = *reinterpret_cast<const float4*>(vbase + (size_t)(kt0 + r) * p.ldk + c4 * 4);
            }
#pragma unroll
            for (int u = 0; u < LB; ++u) {
                const int idx = tid + (b0 + u) * THREADS, r = idx / (HD / 4), c4 = idx - r * (HD / 4);
                *reinterpret_cast<float4*>(Vs + r * HD + c4 * 4) = vr[u];
            }
        }
        __syncthreads();
        // ---- S = Q K^T: rows ty*4 + i, columns tx*4 + j ----
        float s[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll 8
        for (int d = 0; d < HD; ++d) {
            const float4 a = *reinterpret_cast<const float4*>(Qt + d * QT + ty * 4);
            const float4 b = *reinterpret_cast<const float4*>(Kt + d * KT + tx * 4);
            s[0][0] = fmaf(a.x, b.x, s[0][0]); s[0][1] = fmaf(a.x, b.y, s[0][1]); s[0][2] = fmaf(a.x, b.z, s[0][2]); s[0][3] = fmaf(a.x, b.w, s[0][3]);
            s[1][0] = fmaf(a.y, b.x, s[1][0]); s[1][1] = fmaf(a.y, b.y, s[1][1]); s[1][2] = fmaf(a.y, b.z, s[1][2]); s[1][3] = fmaf(a.y, b.w, s[1][3]);
            s[2][0] = fmaf(a.z, b.x, s[2][0]); s[2][1] = fmaf(a.z, b.y, s[2][1]); s[2][2] = fmaf(a.z, b.z, s[2][2]); s[2][3] = fmaf(a.z, b.w, s[2][3]);
            s[3][0] = fmaf(a.w, b.x, s[3][0]); s[3][1] = fmaf(a.w, b.y, s[3][1]); s[3][2] = fmaf(a.w, b.z, s[3][2]); s[3][3] = fmaf(a.w, b.w, s[3][3]);
        }
        // ---- scale (divide, layers.rs:161-162,327-328), mask, online softmax ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = qt0 + ty * 4 + i;
            float tmax = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = kt0 + tx * 4 + j;
                const bool valid = (r < len) && (col < pos0 + len) && (!p.causal || col <= pos0 + r);
                const float v = valid ? s[i][j] / div : -INFINITY;
                s[i][j] = v;
                tmax = fmaxf(tmax, v);
            }
#pragma unroll
            for (int off = 1; off < 16; off <<= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, off));
            const float m_new = fmaxf(m_run[i], tmax);
            const float corr = (m_new == -INFINITY) ? 1.f : expf(m_run[i] - m_new);
            m_run[i] = m_new;
            float psum = 0.f;
            float4 pv;
            pv.x = (m_new == -INFINITY) ? 0.f : expf(s[i][0] - m_new);
            pv.y = (m_new == -INFINITY) ? 0.f : expf(s[i][1] - m_new);
            pv.z = (m_new == -INFINITY) ? 0.f : expf(s[i][2] - m_new);
            pv.w = (m_new == -INFINITY) ? 0.f : expf(s[i][3] - m_new);
            psum = (pv.x + pv.y) + (pv.z + pv.w);
#pragma unroll
            for (int off = 1; off < 16; off <<= 1) psum += __shfl_xor_sync(0xffffffffu, psum, off);
            l_run[i] = l_run[i] * corr + psum;
#pragma unroll
            for (int gq = 0; gq < NG; ++gq) { o[i][gq][0] *= corr; o[i][gq][1] *= corr; o[i][gq][2] *= corr; o[i][gq][3] *= corr; }
            *reinterpret_cast<float4*>(Ps + (ty * 4 + i) * PS + tx * 4) = pv;
        }
        __syncwarp();                               // a P row is written and read by the same warp (two ty values per warp)
        // ---- O += P V: rows ty*4 + i, columns gq*64 + tx*4 + e ----
#pragma unroll 4
        for (int j = 0; j < KT; ++j) {
            float a[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = Ps[(ty * 4 + i) * PS + j];
#pragma unroll
            for (int gq = 0; gq < NG; ++gq) {
                const float4 b = *reinterpret_cast<const float4*>(Vs + j * HD + gq * 64 + tx * 4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    o[i][gq][0] = fmaf(a[i], b.x, o[i][gq][0]); o[i][gq][1] = fmaf(a[i], b.y, o[i][gq][1]);
                    o[i][gq][2] = fmaf(a[i], b.z, o[i][gq][2]); o[i][gq][3] = fmaf(a[i], b.w, o[i][gq][3]);
                }
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = qt0 + ty * 4 + i;
        if (r >= len) continue;
        const float inv = 1.0f / l_run[i];
        const size_t base = (size_t)(q0 + r) * p.ldo + (size_t)h * HD;
#pragma unroll
        for (int gq = 0; gq < NG; ++gq)
#pragma unroll
            for (int e = 0; e < 4; ++e) store_split3(p.out_s3, p.plane_stride, base + gq * 64 + tx * 4 + e, o[i][gq][e] * inv);
    }
    }   // pass
}

template <int HD> static size_t smem_bytes() { return (size_t)(HD * QT + HD * KT + KT * HD + QT * PS) * sizeof(float); }

}  // namespace af32

bool launch_attention_f32(const AttnParams& p, int hd, cudaStream_t st) {
    using namespace af32;
    if (p.nseg <= 0 || p.max_len <= 0) return true;
    if ((p.ldq % 4) || (p.ldk % 4) || (p.head_stride % 4) || (p.seg_stride % 4)) return false;
    const int nqt_max = (p.max_len + QT - 1) / QT;
    dim3 grid(p.causal ? (nqt_max + 1) / 2 : nqt_max, p.nheads, p.nseg);
    auto run = [&](auto kern, size_t smem) {
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // per device: set on every launch
        kern<<<grid, THREADS, smem, st>>>(p);
    };
    const bool off = p.seg_pos0 != nullptr;
    if (off && !p.causal) return false;
    if (hd == 64) run(off ? attn_f32_kernel<64, true> : attn_f32_kernel<64, false>, smem_bytes<64>());
    else if (hd == 128) run(off ? attn_f32_kernel<128, true> : attn_f32_kernel<128, false>, smem_bytes<128>());
    else return false;
    ASRB_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace asrb
