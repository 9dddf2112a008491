// elementwise.cu -- bandwidth kernels: conv2d1+GELU, LayerNorm, RMSNorm, embedding gather with
// audio injection, per-head QK-RMSNorm + RoPE + KV-cache write.  All emit GEMM A-operands as
// split3 bf16 planes (common.cuh) so the tensor-core GEMMs that follow need no conversion pass.
#include "internal.h"

namespace asrb {

// ---------------------------------------------------------------------------------------------
// conv2d1 (Cin = 1, 3x3, stride 2, pad 1) + bias + exact-erf GELU.
// Reference: chunking/zero-pad of the tail chunk (audio_encoder.rs:83-124), conv2d1.forward().gelu()
// (audio_encoder.rs:127, layers.rs:109-118).  9 MACs per output: a bandwidth kernel.  One CTA = one
// (chunk, output row); three mel rows staged in shared memory; thread = output channel; output
// written channels-last into the parity-split layout conv2's implicit GEMM (TMA) consumes.
// ---------------------------------------------------------------------------------------------
__global__ void conv1_gelu_kernel(const float* __restrict__ mel, const int* __restrict__ chunk_clip,
                                  const int* __restrict__ chunk_f0, const int64_t* __restrict__ foff,
                                  const int64_t* __restrict__ frames, int n_mels, int W, int OH, int OW,
                                  const float* __restrict__ w, const float* __restrict__ bias, int dsh,
                                  int cpad, bf16* __restrict__ out, size_t plane_stride) {
    extern __shared__ float rows[];                 // [3][W + 2]
    const int chunk = blockIdx.y, oh = blockIdx.x;
    const int clip = chunk_clip[chunk], f0 = chunk_f0[chunk];
    const int F = (int)frames[clip];
    const float* mp = mel + (size_t)n_mels * foff[clip];
    for (int idx = threadIdx.x; idx < 3 * (W + 2); idx += blockDim.x) {
        int kh = idx / (W + 2), wi = idx - kh * (W + 2);
        int h = 2 * oh + kh - 1, wcol = wi - 1;      // input coords; -1 / W are the conv padding
        float v = 0.f;
        if (h >= 0 && h < n_mels && wcol >= 0 && wcol < W && f0 + wcol < F) v = mp[(size_t)h * F + f0 + wcol];
        rows[idx] = v;
    }
    __syncthreads();
    const int c = threadIdx.x;
    if (c >= dsh) return;
    float wk[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) wk[i] = w[c * 9 + i];
    const float bc = bias ? bias[c] : 0.f;
    const int Hh = OH / 2 + (OH & 1), Wh = (OW + 1) / 2;     // next conv's half extents (= its OH, OW)
    for (int ow = 0; ow < OW; ++ow) {
        float acc = bc;
#pragma unroll
        for (int kh = 0; kh < 3; ++kh)
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) acc = fmaf(wk[kh * 3 + kw], rows[kh * (W + 2) + 2 * ow + kw], acc);
        float v = gelu_erf(acc);
        size_t pos = ((((size_t)chunk * 2 + (oh & 1)) * 2 + (ow & 1)) * Hh + (oh >> 1)) * Wh + (ow >> 1);
        store_split3(out, plane_stride, pos * cpad + c, v);
    }
}

void launch_conv1(const Model& m, const float* mel, const int* d_chunk_clip, const int* d_chunk_f0,
                  const int64_t* d_foff, const int64_t* d_frames, int n_chunks, bf16* out_s3,
                  size_t plane_stride, cudaStream_t st) {
    const Dims& d = m.d;
    int W = d.conv_w[0], OH = d.conv_h[1], OW = d.conv_w[1];
    dim3 grid(OH, n_chunks);
    int threads = ((d.c.downsample_hidden_size + 31) / 32) * 32;
    size_t smem = 3 * (W + 2) * sizeof(float);
    conv1_gelu_kernel<<<grid, threads, smem, st>>>(mel, d_chunk_clip, d_chunk_f0, d_foff, d_frames,
                                                   d.c.num_mel_bins, W, OH, OW, m.conv1_w, m.conv1_b,
                                                   d.c.downsample_hidden_size, d.cpad, out_s3, plane_stride);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (layers.rs:25-28, eps 1e-5) / RMSNorm (layers.rs:48-54) -> split3 planes
// ---------------------------------------------------------------------------------------------
__global__ void layernorm_s3_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                    const float* __restrict__ b, int dim, float eps, bf16* __restrict__ out,
                                    size_t plane_stride) {
    __shared__ float red[32];
    const size_t row = blockIdx.x;
    const float* xr = x + row * dim;
    float s = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) s += xr[i];
    const float mean = block_sum(s, red) / dim;
    float v = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) { float dlt = xr[i] - mean; v = fmaf(dlt, dlt, v); }
    const float var = block_sum(v, red) / dim;
    const float rstd = 1.0f / sqrtf(var + eps);
    for (int i = threadIdx.x; i < dim; i += blockDim.x)
        store_split3(out, plane_stride, row * dim + i, (xr[i] - mean) * rstd * w[i] + b[i]);
}
__global__ void rmsnorm_s3_kernel(const float* __restrict__ x, const float* __restrict__ w, int dim, float eps,
                                  bf16* __restrict__ out, size_t plane_stride) {
    __shared__ float red[32];
    const size_t row = blockIdx.x;
    const float* xr = x + row * dim;
    float s = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) s = fmaf(xr[i], xr[i], s);
    const float var = block_sum(s, red) / dim;
    const float r = 1.0f / sqrtf(var + eps);               // sqrt().reciprocal()  (tensor.rs:323-326)
    for (int i = threadIdx.x; i < dim; i += blockDim.x)
        store_split3(out, plane_stride, row * dim + i, (xr[i] * r) * w[i]);
}
void launch_layernorm_s3(const float* x, const float* w, const float* b, int rows, int dim, float eps,
                         bf16* out_s3, size_t plane_stride, cudaStream_t st) {
    if (rows <= 0) return;
    layernorm_s3_kernel<<<rows, 128, 0, st>>>(x, w, b, dim, eps, out_s3, plane_stride);
    ASRB_CUDA_CHECK(cudaGetLastError());
}
void launch_rmsnorm_s3(const float* x, const float* w, int rows, int dim, float eps, bf16* out_s3,
                       size_t plane_stride, cudaStream_t st) {
    if (rows <= 0) return;
    rmsnorm_s3_kernel<<<rows, 128, 0, st>>>(x, w, dim, eps, out_s3, plane_stride);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// Embedding gather + audio injection in one pass.  Replaces Tensor::embedding
// (text_decoder.rs:90-92) followed by T slice_scatter calls (inference.rs:110-124).
// ---------------------------------------------------------------------------------------------
__global__ void embed_inject_kernel(const bf16* __restrict__ embed, int hidden, const int* __restrict__ ids,
                                    const int* __restrict__ audio_row, const float* __restrict__ audio,
                                    float* __restrict__ out) {
    const size_t row = blockIdx.x;
    const int ar = audio_row[row];
    float* o = out + row * hidden;
    if (ar >= 0) {
        const float* a = audio + (size_t)ar * hidden;
        for (int i = threadIdx.x; i < hidden; i += blockDim.x) o[i] = a[i];
    } else {
        const bf16* e = embed + (size_t)ids[row] * hidden;
        for (int i = threadIdx.x; i < hidden; i += blockDim.x) o[i] = __bfloat162float(e[i]);
    }
}
void launch_embed_inject(const bf16* embed, int hidden, const int* d_ids, const int* d_audio_row,
                         const float* audio, int rows, float* out, cudaStream_t st) {
    if (rows <= 0) return;
    embed_inject_kernel<<<rows, 256, 0, st>>>(embed, hidden, d_ids, d_audio_row, audio, out);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------
// Prefill: per-head RMSNorm on q,k (layers.rs:303-304) -> NeoX rotate-half RoPE (layers.rs:307-308,
// 361-375; the three MRoPE streams are equal, inference.rs:259-266, so it is plain RoPE) -> K,V
// written straight into the static KV cache (replaces the growing Tensor::cat of layers.rs:311-317).
// FAN: a leader row at position pos < fan.P[seq] also writes its K,V into every follower slot of its shared context
// (DESIGN.md 4.5), so a follower holds the prefix before this layer's attention reads it.
// grid (rows, nq + 2*nkv); block = head_dim threads.
// ---------------------------------------------------------------------------------------------
template <bool FAN>
__global__ void qk_norm_rope_kernel(const float* __restrict__ qkv, const int* __restrict__ row_seq,
                                    const int* __restrict__ row_pos, const float* __restrict__ qnorm,
                                    const float* __restrict__ knorm, float eps,
                                    const float* __restrict__ rope_cos, const float* __restrict__ rope_sin,
                                    int nq, int nkv, int hd, float* __restrict__ q_out,
                                    float* __restrict__ kcache, float* __restrict__ vcache,
                                    size_t cache_seq_stride, int max_ctx, FanOut fan) {
    extern __shared__ float sh[];     // [hd] + 32
    float* ys = sh;
    float* red = sh + hd;
    const size_t row = blockIdx.x;
    const int head = blockIdx.y, d = threadIdx.x;
    const int qkv_dim = (nq + 2 * nkv) * hd;
    const float x = qkv[row * qkv_dim + (size_t)head * hd + d];
    const int seq = row_seq[row], pos = row_pos[row];
    const int nfan = FAN && pos < fan.P[seq] ? fan.n[seq] : 0;
    const int* fslots = FAN ? fan.slots + fan.off[seq] : nullptr;
    if (head >= nq + nkv) {           // V: plain copy into the cache
        const size_t o = ((size_t)(head - nq - nkv) * max_ctx + pos) * hd + d;
        vcache[seq * cache_seq_stride + o] = x;
        for (int j = 0; j < nfan; ++j) vcache[(size_t)fslots[j] * cache_seq_stride + o] = x;
        return;
    }
    const float* nw = head < nq ? qnorm : knorm;
    const float var = block_sum(x * x, red) / hd;
    const float y = (x * (1.0f / sqrtf(var + eps))) * nw[d];
    ys[d] = y;
    __syncthreads();
    const int half = hd / 2;
    const float rot = d < half ? -ys[d + half] : ys[d - half];
    const float c = rope_cos[(size_t)pos * half + (d % half)], s = rope_sin[(size_t)pos * half + (d % half)];
    const float o = y * c + rot * s;
    if (head < nq) q_out[row * ((size_t)nq * hd) + (size_t)head * hd + d] = o;
    else {
        const size_t ko = ((size_t)(head - nq) * max_ctx + pos) * hd + d;
        kcache[seq * cache_seq_stride + ko] = o;
        for (int j = 0; j < nfan; ++j) kcache[(size_t)fslots[j] * cache_seq_stride + ko] = o;
    }
}
void launch_qk_norm_rope(const float* qkv, int rows, const int* d_row_seq, const int* d_row_pos,
                         const float* qnorm, const float* knorm, float eps, const float* rope_cos,
                         const float* rope_sin, int nq, int nkv, int hd, float* q_out, float* kcache,
                         float* vcache, size_t cache_seq_stride, int max_ctx, cudaStream_t st, const FanOut* fan) {
    if (rows <= 0) return;
    dim3 grid(rows, nq + 2 * nkv);
    const size_t smem = (hd + 32) * sizeof(float);
    if (fan) qk_norm_rope_kernel<true><<<grid, hd, smem, st>>>(qkv, d_row_seq, d_row_pos, qnorm, knorm, eps, rope_cos, rope_sin,
                                                               nq, nkv, hd, q_out, kcache, vcache, cache_seq_stride, max_ctx, *fan);
    else qk_norm_rope_kernel<false><<<grid, hd, smem, st>>>(qkv, d_row_seq, d_row_pos, qnorm, knorm, eps, rope_cos, rope_sin,
                                                            nq, nkv, hd, q_out, kcache, vcache, cache_seq_stride, max_ctx, FanOut{});
    ASRB_CUDA_CHECK(cudaGetLastError());
}

}  // namespace asrb
