// mel.cu -- 16 kHz f32 samples -> 128-bin Whisper log-mel, fused.
//
// Replaces WhisperFeatureExtractor::extract (/root/reference/src/mel.rs:49-96): zero-pad to a
// multiple of hop (:51-53), reflect pad n_fft/2 (:63-65), periodic-Hann STFT 400/160 without
// centering (:68-76), |.|^2 (:80), drop the last frame (:83-84), filterbank matmul (:87),
// log10(clamp 1e-10) (:90), global max - 8 clamp (:91-92), (x+4)/4 (:93).
//
// One CTA = 16 frames.  The 400-point real DFT uses the even / odd symmetry of the twiddles about n = 200:
//   re[k] = x[0] + (-1)^k x[200] + sum_{n=1..199} (x[n] + x[400-n]) cos(2 pi k n / 400)
//   im[k] =                         sum_{n=1..199} (x[n] - x[400-n]) sin(2 pi k n / 400)
// i.e. half the FMAs of the direct form.  The pair sums / differences of the 16 windowed frames are staged in shared
// memory as [n][16 frames] (every thread reads them with broadcast LDS.128), the {cos, sin} table (400 entries, 3.2 KB)
// lives in shared memory too and thread k walks it with r += k (mod 400) -- the [400][208] table the first version
// streamed from L2 cost 125 MB of L2 traffic per 30 s clip, 60x the kernel's HBM bytes.  Power spectrum kept in shared
// memory (the [201, F+1] STFT magnitude is never written to HBM), triangular filters applied over their non-zero
// support only, log10 and the per-utterance running max (atomicMax on an order-preserving int key).  A second
// elementwise kernel applies the max-8 clamp and affine.
// Bound: fp32 FMA (241 MFMA per 30 s clip); HBM traffic 1.92 MB in + 1.54 MB out per clip.
#include "internal.h"

namespace asrb {

static constexpr int NFFT = 400, HOP = 160, NBIN = 201, KP = 208, FT = 16, MEL_THREADS = 224;

// STREAM: utterance b's frames [ffirst[b], F) only, rows of ldo floats, no running max (the streams' raw log-mel store,
// folded by mel_stream_fold_kernel).  A frame's arithmetic does not depend on the 16-frame block it falls in, so a frame
// computed here is bitwise the offline one.  The offline instantiation passes neither and compiles to the same SASS.
template <bool STREAM>
__global__ void __launch_bounds__(MEL_THREADS)
mel_power_kernel(const float* __restrict__ samples, const int64_t* __restrict__ soff,
                 const int64_t* __restrict__ n_true, const int64_t* __restrict__ n_pad,
                 const int64_t* __restrict__ foff, const float* __restrict__ hann,
                 const float2* __restrict__ tw,
                 const float* __restrict__ fb, const int* __restrict__ krange, int n_mels,
                 float* __restrict__ mel_out, int* __restrict__ maxkey,
                 const int* __restrict__ ffirst = nullptr, int ldo = 0) {
    constexpr int NH = NFFT / 2;                           // 200
    __shared__ __align__(16) float buf[(2 * NH + 1) * FT];
    float (*xe)[FT] = reinterpret_cast<float (*)[FT]>(buf);                   // xe[n] = x[n] + x[400-n] (n = 1..199); xe[0] = x[0]; xe[200] = x[200]
    float (*xo)[FT] = reinterpret_cast<float (*)[FT]>(buf + (NH + 1) * FT);   // xo[n] = x[n] - x[400-n]
    __shared__ float2 tws[NFFT];
    __shared__ float red[32];
    float (*pw)[KP] = reinterpret_cast<float (*)[KP]>(buf);                   // power spectrum [FT][KP] reuses the buffer after the DFT
    static_assert(FT * KP <= (2 * NH + 1) * FT, "pw must fit in the pair buffer");
    const int b = blockIdx.y;
    const int64_t npad = n_pad[b], ntrue = n_true[b];
    const int F = (int)(npad / HOP);
    const int f0 = (STREAM ? ffirst[b] : 0) + blockIdx.x * FT;
    if (f0 >= F) return;
    const float* x = samples + soff[b];
    for (int i = threadIdx.x; i < NFFT; i += MEL_THREADS) tws[i] = tw[i];
    auto sample = [&](int f, int n) {                          // windowed sample n of frame f (0 beyond the utterance)
        if (f >= F) return 0.f;
        int64_t j = (int64_t)f * HOP + n - NFFT / 2;          // index into the hop-padded waveform
        if (j < 0) j = -j;                                    // reflection_pad1d (mel.rs:63-65)
        if (j >= npad) j = 2 * (npad - 1) - j;
        return ((j < ntrue) ? x[j] : 0.f) * hann[n];          // zero padding of mel.rs:51-53, periodic Hann
    };
    for (int idx = threadIdx.x; idx < FT * (NH + 1); idx += MEL_THREADS) {
        const int fi = idx / (NH + 1), n = idx - fi * (NH + 1);
        const float a = sample(f0 + fi, n);
        if (n == 0 || n == NH) xe[n][fi] = a;
        else {
            const float c = sample(f0 + fi, NFFT - n);
            xe[n][fi] = a + c; xo[n][fi] = a - c;
        }
    }
    __syncthreads();
    const int k = threadIdx.x;
    float re[FT], im[FT];
    if (k < NBIN) {
        const float sgn = (k & 1) ? -1.f : 1.f;
#pragma unroll
        for (int i = 0; i < FT; ++i) { re[i] = xe[0][i] + sgn * xe[NH][i]; im[i] = 0.f; }
        int r = 0;
#pragma unroll 2
        for (int n = 1; n < NH; ++n) {
            r += k; if (r >= NFFT) r -= NFFT;
            const float2 t = tws[r];
#pragma unroll
            for (int i4 = 0; i4 < FT; i4 += 4) {
                const float4 e = *reinterpret_cast<const float4*>(&xe[n][i4]);
                const float4 o = *reinterpret_cast<const float4*>(&xo[n][i4]);
                re[i4] = fmaf(e.x, t.x, re[i4]); re[i4 + 1] = fmaf(e.y, t.x, re[i4 + 1]); re[i4 + 2] = fmaf(e.z, t.x, re[i4 + 2]); re[i4 + 3] = fmaf(e.w, t.x, re[i4 + 3]);
                im[i4] = fmaf(o.x, t.y, im[i4]); im[i4 + 1] = fmaf(o.y, t.y, im[i4 + 1]); im[i4 + 2] = fmaf(o.z, t.y, im[i4 + 2]); im[i4 + 3] = fmaf(o.w, t.y, im[i4 + 3]);
            }
        }
    }
    __syncthreads();                                          // every thread is done reading xe / xo: pw may overwrite them
    if (k < NBIN) {
#pragma unroll
        for (int i = 0; i < FT; ++i) pw[i][k] = re[i] * re[i] + im[i] * im[i];   // abs().square()
    }
    __syncthreads();
    float lmax = -INFINITY;
    float* out = mel_out + (size_t)n_mels * foff[b];
    for (int idx = threadIdx.x; idx < n_mels * FT; idx += MEL_THREADS) {
        int m = idx / FT, fi = idx - m * FT;
        int f = f0 + fi;
        int k0 = krange[2 * m], k1 = krange[2 * m + 1];
        float acc = 0.f;
        for (int kk = k0; kk < k1; ++kk) acc = fmaf(fb[m * NBIN + kk], pw[fi][kk], acc);
        float v = log10f(fmaxf(acc, 1e-10f));                     // clamp_min(1e-10).log10()
        if (f < F) {
            out[(size_t)m * (STREAM ? ldo : F) + f] = v;
            lmax = fmaxf(lmax, v);
        }
    }
    if constexpr (!STREAM) {
        lmax = block_max(lmax, red);
        if (threadIdx.x == 0) atomicMax(&maxkey[b], float_to_ordered(lmax));
    }
}

__global__ void mel_finalize_kernel(float* __restrict__ mel, const int64_t* __restrict__ foff,
                                    const int64_t* __restrict__ n_pad, int n_mels,
                                    const int* __restrict__ maxkey) {
    const int b = blockIdx.y;
    const int64_t total = (int64_t)n_mels * (n_pad[b] / HOP);
    float* p = mel + (size_t)n_mels * foff[b];
    const float floor_v = ordered_to_float(maxkey[b]) - 8.0f;     // maximum(max - 8)  (mel.rs:91-92)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        float v = fmaxf(p[i], floor_v);
        p[i] = (v + 4.0f) / 4.0f;                                 // mel.rs:93
    }
}

__global__ void mel_init_max_kernel(int* maxkey, int batch) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < batch) maxkey[i] = float_to_ordered(-INFINITY);
}

void launch_mel(const Model& m, const float* samples, const int64_t* d_soff, const int64_t* d_n,
                const int64_t* d_npad, const int64_t* d_foff, int batch, int max_frames,
                float* mel_out, int* d_maxkey, cudaStream_t st) {
    mel_init_max_kernel<<<(batch + 127) / 128, 128, 0, st>>>(d_maxkey, batch);
    dim3 grid((max_frames + FT - 1) / FT, batch);
    mel_power_kernel<false><<<grid, MEL_THREADS, 0, st>>>(samples, d_soff, d_n, d_npad, d_foff, m.hann,
                                                   reinterpret_cast<const float2*>(m.dft_tw), m.mel_fb, m.mel_krange,
                                                   m.d.c.num_mel_bins, mel_out, d_maxkey);
    dim3 g2(132, batch);                                          // one CTA per H100 SM per clip
    mel_finalize_kernel<<<g2, 256, 0, st>>>(mel_out, d_foff, d_npad, m.d.c.num_mel_bins, d_maxkey);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

// ---- streaming (DESIGN.md 4.9) ----
// one CTA per stream: frames [f_old, f_new) became final this push -- fold them into the stream's final maximum and into
// the minima of their encoder windows (win_frames frames each); the maximum over the provisional frames [f_new, F) is
// written beside them.  stats row b: [0] final max  [1] provisional max (-inf: none)  [2 + w] minimum of window w.
// max / min are exact in any order, so the values do not depend on the reduction order.
__global__ void mel_stream_fold_kernel(const float* __restrict__ raw, const int4* __restrict__ plan, int n_mels, int ldo,
                                       int win_frames, float* __restrict__ stats, int stats_ld) {
    __shared__ float red[32];
    const int b = blockIdx.x;
    const int4 q = plan[b];                                     // {f_old, f_new, F, active}
    if (!q.w) return;
    const float* r = raw + (size_t)b * n_mels * ldo;
    float* out = stats + (size_t)b * stats_ld;
    auto range_max = [&](int f0, int f1, float sign) {          // max of sign * v over frames [f0, f1) of every mel row
        float v = -INFINITY;
        const int nf = f1 - f0;
        for (int i = threadIdx.x; i < n_mels * nf; i += blockDim.x) {
            const int m = i / nf, f = f0 + (i - m * nf);
            v = fmaxf(v, sign * r[(size_t)m * ldo + f]);
        }
        return block_max(v, red);
    };
    if (q.y > q.x) {
        const float fm = range_max(q.x, q.y, 1.f);
        if (threadIdx.x == 0) out[0] = fmaxf(out[0], fm);
        for (int w = q.x / win_frames; w * win_frames < q.y; ++w) {
            const float mn = -range_max(max(q.x, w * win_frames), min(q.y, (w + 1) * win_frames), -1.f);
            if (threadIdx.x == 0) out[2 + w] = fminf(out[2 + w], mn);
        }
    }
    const float tm = q.z > q.y ? range_max(q.y, q.z, 1.f) : -INFINITY;
    if (threadIdx.x == 0) out[1] = tm;
}

// the re-encoded windows of a push as pseudo-utterances for the encoder: utterance u = frames [fs, fs + Fu) of stream
// slot's raw log-mel, clamped at the stream's floor phi and scaled as mel_finalize_kernel does, written [n_mels][Fu] at
// frame offset foff[u] of mel_out.  plan row u: {slot, fs, Fu, float bits of phi}
__global__ void mel_stream_stage_kernel(const float* __restrict__ raw, const int4* __restrict__ plan,
                                        const int64_t* __restrict__ foff, int n_mels, int ldo, float* __restrict__ mel_out) {
    const int u = blockIdx.y;
    const int4 q = plan[u];
    const float floor_v = __int_as_float(q.w);
    const float* r = raw + (size_t)q.x * n_mels * ldo + q.y;
    float* p = mel_out + (size_t)n_mels * foff[u];
    const int64_t total = (int64_t)n_mels * q.z;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / q.z), f = (int)(i - (int64_t)m * q.z);
        const float v = fmaxf(r[(size_t)m * ldo + f], floor_v);
        p[i] = (v + 4.0f) / 4.0f;
    }
}

void launch_mel_stream(const Model& m, const float* samples, const int64_t* d_soff, const int64_t* d_n, const int64_t* d_npad,
                       const int64_t* d_foff, const int* d_ffirst, int n_streams, int max_new_frames, int ldo, float* raw,
                       const int4* d_fold, int win_frames, float* stats, int stats_ld, cudaStream_t st) {
    if (max_new_frames > 0) {
        dim3 grid((max_new_frames + FT - 1) / FT, n_streams);
        mel_power_kernel<true><<<grid, MEL_THREADS, 0, st>>>(samples, d_soff, d_n, d_npad, d_foff, m.hann,
                                                             reinterpret_cast<const float2*>(m.dft_tw), m.mel_fb, m.mel_krange,
                                                             m.d.c.num_mel_bins, raw, nullptr, d_ffirst, ldo);
    }
    mel_stream_fold_kernel<<<n_streams, 256, 0, st>>>(raw, d_fold, m.d.c.num_mel_bins, ldo, win_frames, stats, stats_ld);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

void launch_mel_stream_stage(const Model& m, const float* raw, const int4* d_plan, const int64_t* d_foff, int n_utt, int ldo,
                             float* mel_out, cudaStream_t st) {
    dim3 grid(32, n_utt);
    mel_stream_stage_kernel<<<grid, 256, 0, st>>>(raw, d_plan, d_foff, m.d.c.num_mel_bins, ldo, mel_out);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

}  // namespace asrb
