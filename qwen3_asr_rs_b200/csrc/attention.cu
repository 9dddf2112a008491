// attention.cu -- fp32 flash-style attention over independent segments.
//
// Encoder (layers.rs:152-172 + the block-diagonal mask of audio_encoder.rs:172-260): each window of
// <= 104 tokens is a segment; the T x T additive mask is never materialised, windows simply do
// not see each other.  Prefill (layers.rs:284-342): each utterance is a causal segment, K/V come
// from the static KV cache, GQA handled by indexing (q head h reads kv head h / group; no
// repeat_kv copy, layers.rs:350-358), the causal mask (text_decoder.rs:121-131) is implicit.
// Scores are (q.k) / sqrt(hd) -- divide, as layers.rs:161-162,327-328 -- softmax in fp32.
// CTA = 16 queries x 1 head, 128 threads; K/V streamed through shared memory in 64-key tiles with
// an online softmax.  Output emitted as split3 planes for the out/o projection GEMM.
#include "internal.h"

namespace asrb {

static constexpr int QT = 16, KT = 64, ATT_THREADS = 128;

// OFF: causal segments with a query position offset (p.seg_pos0): query row q is at position pos0 + q and sees keys
// 0..pos0 + q of its slot
template <int HD, bool OFF>
__global__ void __launch_bounds__(ATT_THREADS) attn_kernel(AttnParams p) {
    extern __shared__ float sm[];
    float* Qs = sm;                          // [QT][HD+1]
    float* Ks = Qs + QT * (HD + 1);          // [KT][HD+1]
    float* Vs = Ks + KT * (HD + 1);          // [KT][HD]
    float* Ps = Vs + KT * HD;                // [QT][KT]
    const int seg = blockIdx.z, h = blockIdx.y;
    const int q0 = p.seg_q0[seg], len = p.seg_len[seg];
    const int pos0 = OFF ? p.seg_pos0[seg] : 0;
    const int qt0 = blockIdx.x * QT;
    if (qt0 >= len) return;
    const int g = h / p.group;
    const int tid = threadIdx.x, qi = tid >> 3, sub = tid & 7;
    const float inv_div = sqrtf((float)HD);

    for (int idx = tid; idx < QT * HD; idx += ATT_THREADS) {
        int r = idx / HD, d = idx - r * HD;
        int q = qt0 + r;
        Qs[r * (HD + 1) + d] = (q < len) ? p.q[(size_t)(q0 + q) * p.ldq + (size_t)h * HD + d] : 0.f;
    }
    const float* kbase;
    const float* vbase;
    size_t kld;
    if (p.keys_in_rows) {
        kbase = p.k + (size_t)q0 * p.ldk + (size_t)g * p.head_stride;
        vbase = p.v + (size_t)q0 * p.ldk + (size_t)g * p.head_stride;
    } else {
        kbase = p.k + (size_t)seg * p.seg_stride + (size_t)g * p.head_stride;
        vbase = p.v + (size_t)seg * p.seg_stride + (size_t)g * p.head_stride;
    }
    kld = p.ldk;

    float m_run = -INFINITY, l_run = 0.f;
    float acc[HD / 8];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) acc[i] = 0.f;
    const int my_q = qt0 + qi;
    const int kend = p.causal ? pos0 + min(len, qt0 + QT) : len;

    for (int kt0 = 0; kt0 < kend; kt0 += KT) {
        __syncthreads();
        for (int idx = tid; idx < KT * HD; idx += ATT_THREADS) {
            int r = idx / HD, d = idx - r * HD;
            int j = kt0 + r;
            float kv = 0.f, vv = 0.f;
            if (j < kend) { kv = kbase[(size_t)j * kld + d]; vv = vbase[(size_t)j * kld + d]; }
            Ks[r * (HD + 1) + d] = kv;
            Vs[r * HD + d] = vv;
        }
        __syncthreads();
        float s[8];
        float tmax = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            int kj = sub + 8 * jj;
            float dot = 0.f;
#pragma unroll 8
            for (int d = 0; d < HD; ++d) dot = fmaf(Qs[qi * (HD + 1) + d], Ks[kj * (HD + 1) + d], dot);
            int kidx = kt0 + kj;
            bool valid = (my_q < len) && (kidx < pos0 + len) && (!p.causal || kidx <= pos0 + my_q);
            s[jj] = valid ? dot / inv_div : -INFINITY;
            tmax = fmaxf(tmax, s[jj]);
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
        const float m_new = fmaxf(m_run, tmax);
        float corr = 1.f, psum = 0.f;
        if (m_new == -INFINITY) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) Ps[qi * KT + sub + 8 * jj] = 0.f;
        } else {
            corr = expf(m_run - m_new);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                float pv = expf(s[jj] - m_new);      // exp(-inf) = 0 for masked keys
                Ps[qi * KT + sub + 8 * jj] = pv;
                psum += pv;
            }
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) psum += __shfl_xor_sync(0xffffffffu, psum, o);
        l_run = l_run * corr + psum;
        m_run = m_new;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) acc[i] *= corr;
        __syncwarp();
        const int nk = min(KT, kend - kt0);
        for (int j = 0; j < nk; ++j) {
            float pv = Ps[qi * KT + j];
#pragma unroll
            for (int i = 0; i < HD / 8; ++i) acc[i] = fmaf(pv, Vs[j * HD + i * 8 + sub], acc[i]);
        }
    }
    if (my_q < len) {
        const float inv = 1.0f / l_run;
        size_t row = (size_t)(q0 + my_q) * p.ldo + (size_t)h * HD;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) store_split3(p.out_s3, p.plane_stride, row + i * 8 + sub, acc[i] * inv);
    }
}

bool launch_attention_tc(const AttnParams& p, int hd, cudaStream_t st);    // attention_tc.cu  (3xTF32 mma.sync; ASRB_ATTN=tc)
bool launch_attention_f32(const AttnParams& p, int hd, cudaStream_t st);   // attention_f32.cu (register-tiled fp32; default)

void launch_attention(const AttnParams& p, int hd, cudaStream_t st) {
    if (p.nseg <= 0 || p.max_len <= 0) return;
    // 0 = register-tiled fp32 (default), 1 = 3xTF32 tensor-core variant, 2 = the simple kernel below
    static const int which = [] { const char* e = getenv("ASRB_ATTN"); return !e ? 0 : std::string(e) == "tc" ? 1 : std::string(e) == "simt" ? 2 : 0; }();
    if (which == 0 && launch_attention_f32(p, hd, st)) return;
    if (which == 1 && launch_attention_tc(p, hd, st)) return;     // declines a query position offset
    ASRB_REQUIRE(!p.seg_pos0 || p.causal, ASRB_ERR_INVALID, "attention: a query position offset needs a causal segment");
    dim3 grid((p.max_len + QT - 1) / QT, p.nheads, p.nseg);
    auto run = [&](auto kern, size_t smem) {
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // per device: set on every launch
        kern<<<grid, ATT_THREADS, smem, st>>>(p);
    };
    const bool off = p.seg_pos0 != nullptr;
    if (hd == 64) {
        run(off ? attn_kernel<64, true> : attn_kernel<64, false>, (QT * 65 + KT * 65 + KT * 64 + QT * KT) * sizeof(float));
    } else if (hd == 128) {
        run(off ? attn_kernel<128, true> : attn_kernel<128, false>, (QT * 129 + KT * 129 + KT * 128 + QT * KT) * sizeof(float));
    } else {
        throw Error(ASRB_ERR_INVALID, "attention head_dim must be 64 or 128");
    }
    ASRB_CUDA_CHECK(cudaGetLastError());
}

}  // namespace asrb
