// model.cu -- weight intake, one-time repack to kernel layouts, host-built constant tables.
//
// Reference behaviour restated: tensors are looked up by HF name (audio_encoder.rs:37-55,
// layers.rs:135-150,185-227,262-281,388-439, text_decoder.rs:54-79); bf16/f16 are widened to f32
// by the reference (weights.rs:74-89) -- here matrices stay bf16 on the device (lossless for bf16
// checkpoints) and vectors (norm weights, biases, the 9-tap conv2d1 filter) become f32.
// Host tables are computed in f64 then narrowed exactly as the reference does: mel filterbank
// (mel.rs:115-187), sinusoidal positions (audio_encoder.rs:283-301), RoPE cos/sin
// (layers.rs:471-522; three equal MRoPE streams == plain RoPE, inference.rs:259-266).
#include <cmath>
#include <cstring>
#include "internal.h"

namespace asrb {

void Dims::derive() {
    enc_hd = c.d_model / c.encoder_attention_heads;
    chunk_frames = 2 * c.n_window;
    chunks_per_window = c.n_window_infer / chunk_frames;
    conv_h[0] = c.num_mel_bins;
    conv_w[0] = chunk_frames;
    for (int i = 1; i < 4; ++i) { conv_h[i] = conv_out_len(conv_h[i - 1]); conv_w[i] = conv_out_len(conv_w[i - 1]); }
    tok_per_chunk = conv_w[3];
    cpad = ((c.downsample_hidden_size + 63) / 64) * 64;
    feat = c.downsample_hidden_size * conv_h[3];
    q_dim = c.num_attention_heads * c.head_dim;
    kv_dim = c.num_key_value_heads * c.head_dim;
    qkv_dim = q_dim + 2 * kv_dim;
}

Model::~Model() {
    for (auto& kv : raw) if (kv.second.dev) cudaFree(kv.second.dev);
    for (void* p : owned) cudaFree(p);
}

static inline uint16_t f32_to_bf16_rne(float f, bool* inexact) {
    uint32_t u; memcpy(&u, &f, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return (uint16_t)(u >> 16);     // inf / nan
    uint32_t r = u + 0x7fffu + ((u >> 16) & 1u);
    if (u & 0xffffu) *inexact = true;
    return (uint16_t)(r >> 16);
}
static inline float f16_to_f32(uint16_t h) {                               // weights.rs:156-181
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1f, man = h & 0x3ffu, u;
    if (exp == 0) {
        if (man == 0) u = sign;
        else { int e = -1; do { man <<= 1; ++e; } while (!(man & 0x400u)); u = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13); }
    } else if (exp == 31) u = sign | 0x7f800000u | (man << 13);
    else u = sign | ((exp + 112) << 23) | (man << 13);
    float f; memcpy(&f, &u, 4); return f;
}

static bool is_matrix_name(const std::string& name, int ndim) {
    if (ndim < 2) return false;
    if (name.find("conv2d1.weight") != std::string::npos) return false;    // [dsh,1,3,3]: 9 taps, f32
    return true;
}

// Matrices are stored as bf16 (exact for the released bf16 checkpoints, which the reference widens to f32,
// weights.rs:74-89).  An F32 / F16 matrix that is NOT bf16-representable would silently change logits and ids, so it is
// an error unless ASRB_ALLOW_LOSSY_WEIGHTS=1, in which case it is rounded (RNE) and counted (asrb_model_lossy_tensors).
static void note_lossy(Model* m, const std::string& name) {
    const char* e = getenv("ASRB_ALLOW_LOSSY_WEIGHTS");
    if (!(e && e[0] == '1'))
        throw Error(ASRB_ERR_INVALID, "tensor " + name + " is not bf16-representable: this library keeps matrices in bf16 (exact for bf16 "
                                      "checkpoints); set ASRB_ALLOW_LOSSY_WEIGHTS=1 to round it (results then differ from the f32 reference)");
    m->lossy_weights = true; m->lossy_count += 1;
}

void model_set_tensor(Model* m, const char* name_c, int dtype, const int64_t* shape, int ndim, const void* host) {
    ASRB_REQUIRE(!m->finalized, ASRB_ERR_STATE, "model already finalized");
    ASRB_REQUIRE(name_c && host && ndim >= 1 && ndim <= 4, ASRB_ERR_INVALID, "set_tensor: bad arguments");
    std::string name(name_c);
    size_t numel = 1;
    for (int i = 0; i < ndim; ++i) { ASRB_REQUIRE(shape[i] > 0, ASRB_ERR_INVALID, "set_tensor: bad shape"); numel *= (size_t)shape[i]; }
    RawTensor t;
    t.shape.assign(shape, shape + ndim);
    t.numel = numel;
    t.is_bf16 = is_matrix_name(name, ndim);
    auto it = m->raw.find(name);
    if (it != m->raw.end()) { cudaFree(it->second.dev); m->raw.erase(it); }
    if (t.is_bf16) {
        std::vector<uint16_t> tmp;
        const void* src = host;
        if (dtype == ASRB_DT_F32) {
            tmp.resize(numel); bool inexact = false; const float* f = (const float*)host;
            for (size_t i = 0; i < numel; ++i) tmp[i] = f32_to_bf16_rne(f[i], &inexact);
            if (inexact) note_lossy(m, name);
            src = tmp.data();
        } else if (dtype == ASRB_DT_F16) {
            tmp.resize(numel); bool inexact = false; const uint16_t* h = (const uint16_t*)host;
            for (size_t i = 0; i < numel; ++i) tmp[i] = f32_to_bf16_rne(f16_to_f32(h[i]), &inexact);
            if (inexact) note_lossy(m, name);
            src = tmp.data();
        } else ASRB_REQUIRE(dtype == ASRB_DT_BF16, ASRB_ERR_INVALID, "set_tensor: unsupported dtype");
        ASRB_CUDA_CHECK(cudaMalloc(&t.dev, numel * 2));
        ASRB_CUDA_CHECK(cudaMemcpy(t.dev, src, numel * 2, cudaMemcpyHostToDevice));
    } else {
        std::vector<float> tmp;
        const void* src = host;
        if (dtype == ASRB_DT_BF16) {
            tmp.resize(numel); const uint16_t* h = (const uint16_t*)host;
            for (size_t i = 0; i < numel; ++i) { uint32_t u = (uint32_t)h[i] << 16; memcpy(&tmp[i], &u, 4); }
            src = tmp.data();
        } else if (dtype == ASRB_DT_F16) {
            tmp.resize(numel); const uint16_t* h = (const uint16_t*)host;
            for (size_t i = 0; i < numel; ++i) tmp[i] = f16_to_f32(h[i]);
            src = tmp.data();
        } else ASRB_REQUIRE(dtype == ASRB_DT_F32, ASRB_ERR_INVALID, "set_tensor: unsupported dtype");
        ASRB_CUDA_CHECK(cudaMalloc(&t.dev, numel * 4));
        ASRB_CUDA_CHECK(cudaMemcpy(t.dev, src, numel * 4, cudaMemcpyHostToDevice));
    }
    m->raw[name] = t;
}

// ---- finalize helpers -------------------------------------------------------------------------
static const RawTensor& need(Model* m, const std::string& name, std::initializer_list<int64_t> shape, bool bf) {
    auto it = m->raw.find(name);
    if (it == m->raw.end()) throw Error(ASRB_ERR_INVALID, "missing tensor: " + name);
    const RawTensor& t = it->second;
    std::vector<int64_t> want(shape);
    if (t.shape != want) {
        std::string s = "tensor " + name + " has shape [";
        for (auto v : t.shape) s += std::to_string(v) + ",";
        s += "] expected [";
        for (auto v : want) s += std::to_string(v) + ",";
        throw Error(ASRB_ERR_INVALID, s + "]");
    }
    ASRB_REQUIRE(t.is_bf16 == bf, ASRB_ERR_INVALID, "tensor " + name + " has the wrong storage class");
    return t;
}
template <typename T> static T* take(Model* m, const std::string& name, std::initializer_list<int64_t> shape, bool bf) {
    return (T*)need(m, name, shape, bf).dev;
}
static float* opt_f32(Model* m, const std::string& name, std::initializer_list<int64_t> shape) {
    if (m->raw.find(name) == m->raw.end()) return nullptr;                  // get_weight_opt, weights.rs:199-212
    return take<float>(m, name, shape, false);
}
template <typename T> static T* dev_alloc(Model* m, size_t n) {
    T* p = nullptr;
    ASRB_CUDA_CHECK(cudaMalloc(&p, n * sizeof(T)));
    m->owned.push_back(p);
    return p;
}

// Copy of a bf16 [N][K] matrix with the 16-byte chunks of row r stored at chunk index (c & ~7) | ((c ^ r) & 7): rows that
// are bulk-copied into shared memory at a 2 KB pitch then feed ldmatrix without bank conflicts (decode_batch.cu)
__global__ void swizzle_rows_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, size_t n_rows, int chunks) {
    const size_t total = n_rows * (size_t)chunks;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / chunks; const int cc = (int)(i - r * chunks);
        out[r * chunks + ((cc & ~7) | ((cc ^ (int)(r & 7)) & 7))] = in[i];
    }
}
static bf16* swizzled_rows_copy(Model* m, const bf16* src, size_t n_rows, int K) {
    ASRB_REQUIRE(K % 64 == 0, ASRB_ERR_INVALID, "swizzled copy needs K % 64 == 0");
    bf16* dst = nullptr;
    ASRB_CUDA_CHECK(cudaMalloc(&dst, n_rows * (size_t)K * 2));
    m->owned.push_back(dst);
    swizzle_rows_kernel<<<1184, 256>>>(reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), n_rows, K / 8);
    ASRB_CUDA_CHECK(cudaGetLastError());
    return dst;
}

// int8 copy of the lm_head for the greedy single-sequence fused step (decode_mega.cu consume_head_q; derivation in
// DESIGN.md section 4.1), one warp per row: s_r = absmax / 127 (fp32), q_r = round(w_r / s_r), and in fp64
//   C_r = |w_r - s_r q_r|_2 + gamma_n |w_r|_2 + gamma_(n+1) s_r |q_r|_2,   n = K / 64 + 6,  gamma_k = k u / (1 - k u),
// enlarged by a relative 1e-9 (the fp64 sums' own rounding) and rounded up to fp32.  |x|_2 C_r bounds the distance between
// the kernel's fp32 logit of the bf16 row and its fp32 approximation s_r * sum_i q_ri x_i.
__global__ void quantize_head_kernel(const bf16* __restrict__ w, int8_t* __restrict__ q, float2* __restrict__ sc, int V, int K,
                                     double gn, double gn1) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= V) return;
    const bf16* wr = w + (size_t)row * K;
    float amax = 0.f;
    for (int k = lane; k < K; k += 32) amax = fmaxf(amax, fabsf(__bfloat162float(wr[k])));
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float s = amax / 127.f;
    double r2 = 0.0, w2 = 0.0, q2 = 0.0;
    for (int k = lane; k < K; k += 32) {
        const float v = __bfloat162float(wr[k]);
        const float qf = s > 0.f ? fminf(fmaxf(rintf(v / s), -127.f), 127.f) : 0.f;
        q[(size_t)row * K + k] = (int8_t)qf;
        const double d = (double)v - (double)s * (double)qf;
        r2 += d * d; w2 += (double)v * (double)v; q2 += (double)qf * (double)qf;
    }
    for (int o = 16; o > 0; o >>= 1) {
        r2 += __shfl_xor_sync(0xffffffffu, r2, o); w2 += __shfl_xor_sync(0xffffffffu, w2, o); q2 += __shfl_xor_sync(0xffffffffu, q2, o);
    }
    if (lane == 0) {
        const double C = (sqrt(r2) + gn * sqrt(w2) + gn1 * (double)s * sqrt(q2)) * (1.0 + 1e-9);
        sc[row] = make_float2(s, __double2float_ru(C));
    }
}

// Copy of an fp32 vector in the activation layout of the fused decode step (decode_mega.cu, xs_swz): 16-byte group k
// is stored at k ^ ((k >> 3) & 1), which makes the per-lane 32-byte register loads of the GEMV bank-conflict free.
static float* swizzled_copy(Model* m, const float* dev_src, int n) {
    std::vector<float> h((size_t)n), o((size_t)n);
    ASRB_CUDA_CHECK(cudaMemcpy(h.data(), dev_src, (size_t)n * 4, cudaMemcpyDeviceToHost));
    for (int e = 0; e < n; ++e) { const int k = e >> 2; o[(size_t)((k ^ ((k >> 3) & 1)) << 2) + (e & 3)] = h[e]; }
    float* d = dev_alloc<float>(m, (size_t)n);
    ASRB_CUDA_CHECK(cudaMemcpy(d, o.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    return d;
}
template <typename T> static T* dev_upload(Model* m, const std::vector<T>& h) {
    T* p = dev_alloc<T>(m, h.size());
    ASRB_CUDA_CHECK(cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    return p;
}
static void drop_raw(Model* m, const std::string& name) {
    auto it = m->raw.find(name);
    if (it != m->raw.end()) { cudaFree(it->second.dev); m->raw.erase(it); }
}

__global__ void repack_conv_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int co, int ci, int cpad) {
    // src [co][ci][3][3] -> dst [co][tap = kh*3+kw][cpad], zero for cin >= ci
    size_t total = (size_t)co * 9 * cpad;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        int cin = (int)(i % cpad); size_t r = i / cpad; int tap = (int)(r % 9); int o = (int)(r / 9);
        dst[i] = cin < ci ? src[((size_t)o * ci + cin) * 9 + tap] : __float2bfloat16(0.f);
    }
}

// conv_out.weight [dm][c*OH + oh] -> [dm][oh*dsh + c]: the conv3 epilogue then writes 8 consecutive channels of one
// (chunk, ow, oh) as one 16-byte store per plane instead of 2-byte stores 2*OH bytes apart (the contraction over the
// 7680 features is the same sum in a different order)
__global__ void permute_convout_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, size_t rows, int dsh, int OH) {
    const size_t feat = (size_t)dsh * OH, total = rows * feat;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / feat; const int k = (int)(i - r * feat); const int oh = k / dsh, c = k - oh * dsh;
        dst[i] = src[r * feat + (size_t)c * OH + oh];
    }
}

static void build_mel_tables(Model* m) {
    // mel.rs:115-187, f64 -> f32 with the reference's f32 multiply by enorm
    const int num_mels = m->d.c.num_mel_bins, n_fft = 400, n_freqs = 201;
    const double sr = 16000.0, f_sp = 200.0 / 3.0, min_log_hz = 1000.0;
    const double min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
    auto hz_to_mel = [&](double f) { return f < min_log_hz ? f / f_sp : min_log_mel + std::log(f / min_log_hz) / logstep; };
    auto mel_to_hz = [&](double mm) { return mm < min_log_mel ? f_sp * mm : min_log_hz * std::exp(logstep * (mm - min_log_mel)); };
    const double mel_min = hz_to_mel(0.0), mel_max = hz_to_mel(sr / 2.0);
    std::vector<double> ff(num_mels + 2), af(n_freqs), fd(num_mels + 1);
    for (int i = 0; i < num_mels + 2; ++i) ff[i] = mel_to_hz(mel_min + (mel_max - mel_min) * i / (double)(num_mels + 1));
    for (int j = 0; j < n_freqs; ++j) af[j] = j * sr / n_fft;
    for (int i = 0; i <= num_mels; ++i) fd[i] = ff[i + 1] - ff[i];
    std::vector<float> fb((size_t)num_mels * n_freqs);
    for (int j = 0; j < n_freqs; ++j)
        for (int i = 0; i < num_mels; ++i) {
            double down = (af[j] - ff[i]) / fd[i], up = (ff[i + 2] - af[j]) / fd[i + 1];
            fb[(size_t)i * n_freqs + j] = (float)std::max(std::min(down, up), 0.0);
        }
    std::vector<int> kr(2 * num_mels);
    for (int i = 0; i < num_mels; ++i) {
        float enorm = (float)(2.0 / (ff[i + 2] - ff[i]));
        int k0 = n_freqs, k1 = 0;
        for (int j = 0; j < n_freqs; ++j) {
            fb[(size_t)i * n_freqs + j] *= enorm;
            if (fb[(size_t)i * n_freqs + j] != 0.f) { k0 = std::min(k0, j); k1 = std::max(k1, j + 1); }
        }
        if (k0 >= k1) { k0 = 0; k1 = 0; }
        kr[2 * i] = k0; kr[2 * i + 1] = k1;
    }
    m->mel_fb = dev_upload(m, fb);
    m->mel_krange = dev_upload(m, kr);
    const int KP = 208;
    std::vector<float> dc((size_t)n_fft * KP, 0.f), ds((size_t)n_fft * KP, 0.f), hw(n_fft);
    const double two_pi = 6.283185307179586476925286766559;
    for (int n = 0; n < n_fft; ++n) {
        hw[n] = (float)(0.5 * (1.0 - std::cos(two_pi * n / n_fft)));        // periodic Hann (tensor.rs:215-219)
        for (int k = 0; k < n_freqs; ++k) {
            int r = (int)(((long long)n * k) % n_fft);
            dc[(size_t)n * KP + k] = (float)std::cos(two_pi * r / n_fft);
            ds[(size_t)n * KP + k] = (float)std::sin(two_pi * r / n_fft);
        }
    }
    m->dft_cos = dev_upload(m, dc); m->dft_sin = dev_upload(m, ds); m->hann = dev_upload(m, hw);
    // 1-D twiddle table {cos, sin}(2 pi r / 400), r = 0..399 (mel.cu keeps it in shared memory and walks it with r += k mod 400)
    std::vector<float> tw((size_t)2 * n_fft);
    for (int r = 0; r < n_fft; ++r) { tw[2 * r] = (float)std::cos(two_pi * r / n_fft); tw[2 * r + 1] = (float)std::sin(two_pi * r / n_fft); }
    m->dft_tw = dev_upload(m, tw);
}

static void build_pos_tables(Model* m) {
    const Dims& d = m->d;
    {   // audio_encoder.rs:283-301, rows 0..tok_per_chunk-1 (the only rows forward() ever reads, :137)
        const int dim = d.c.d_model, half = dim / 2;
        const double inc = std::log(10000.0) / (double)(half - 1);
        std::vector<float> pe((size_t)d.tok_per_chunk * dim);
        for (int pos = 0; pos < d.tok_per_chunk; ++pos)
            for (int i = 0; i < half; ++i) {
                double ang = pos * std::exp(-(double)i * inc);
                pe[(size_t)pos * dim + i] = (float)std::sin(ang);
                pe[(size_t)pos * dim + half + i] = (float)std::cos(ang);
            }
        m->pos_emb = dev_upload(m, pe);
    }
    {   // layers.rs:471-522
        const int hd = d.c.head_dim, half = hd / 2;
        m->rope_max_pos = 32768;
        std::vector<float> rc((size_t)m->rope_max_pos * half), rs((size_t)m->rope_max_pos * half);
        std::vector<double> inv(half);
        for (int j = 0; j < half; ++j) inv[j] = 1.0 / std::pow(d.c.rope_theta, 2.0 * j / (double)hd);
        for (int p = 0; p < m->rope_max_pos; ++p)
            for (int j = 0; j < half; ++j) {
                double ang = (double)p * inv[j];
                rc[(size_t)p * half + j] = (float)std::cos(ang);
                rs[(size_t)p * half + j] = (float)std::sin(ang);
            }
        m->rope_cos = dev_upload(m, rc); m->rope_sin = dev_upload(m, rs);
    }
}

void model_finalize(Model* m) {
    ASRB_REQUIRE(!m->finalized, ASRB_ERR_STATE, "model already finalized");
    const asrb_dims& c = m->d.c;
    const Dims& d = m->d;
    ASRB_REQUIRE(c.d_model % c.encoder_attention_heads == 0 && (d.enc_hd == 64 || d.enc_hd == 128), ASRB_ERR_INVALID,
                 "encoder head_dim must be 64 or 128");
    ASRB_REQUIRE(c.head_dim == 128, ASRB_ERR_INVALID, "decoder head_dim must be 128");
    ASRB_REQUIRE(c.num_attention_heads % c.num_key_value_heads == 0, ASRB_ERR_INVALID, "GQA group must be integral");
    ASRB_REQUIRE(c.hidden_size % 256 == 0 && c.intermediate_size % 256 == 0 && d.q_dim % 256 == 0, ASRB_ERR_INVALID,
                 "decoder dims must be multiples of 256");
    ASRB_REQUIRE(c.d_model % 64 == 0 && c.encoder_ffn_dim % 64 == 0 && d.feat % 64 == 0, ASRB_ERR_INVALID,
                 "encoder dims must be multiples of 64");
    ASRB_REQUIRE(c.output_dim == c.hidden_size, ASRB_ERR_INVALID, "audio output_dim must equal text hidden_size");
    const int64_t dsh = c.downsample_hidden_size, dm = c.d_model, ffn = c.encoder_ffn_dim;
    const std::string a = "thinker.audio_tower";
    m->conv1_w = take<float>(m, a + ".conv2d1.weight", {dsh, 1, 3, 3}, false);
    m->conv1_b = opt_f32(m, a + ".conv2d1.bias", {dsh});
    for (int ci = 2; ci <= 3; ++ci) {
        std::string nm = a + ".conv2d" + std::to_string(ci);
        const bf16* src = take<bf16>(m, nm + ".weight", {dsh, dsh, 3, 3}, true);
        bf16* dst = dev_alloc<bf16>(m, (size_t)dsh * 9 * d.cpad);
        repack_conv_kernel<<<256, 256>>>(src, dst, (int)dsh, (int)dsh, d.cpad);
        ASRB_CUDA_CHECK(cudaGetLastError());
        ASRB_CUDA_CHECK(cudaDeviceSynchronize());
        drop_raw(m, nm + ".weight");
        float* b = opt_f32(m, nm + ".bias", {dsh});
        if (!b) { std::vector<float> z(dsh, 0.f); b = dev_upload(m, z); }
        if (ci == 2) { m->conv2_w = dst; m->conv2_b = b; } else { m->conv3_w = dst; m->conv3_b = b; }
    }
    {
        const bf16* src = take<bf16>(m, a + ".conv_out.weight", {dm, (int64_t)d.feat}, true);
        bf16* dst = dev_alloc<bf16>(m, (size_t)dm * d.feat);
        permute_convout_kernel<<<1184, 256>>>(src, dst, (size_t)dm, (int)dsh, d.conv_h[3]);
        ASRB_CUDA_CHECK(cudaGetLastError());
        ASRB_CUDA_CHECK(cudaDeviceSynchronize());
        drop_raw(m, a + ".conv_out.weight");
        m->conv_out_w = dst;
    }
    m->conv_out_b = opt_f32(m, a + ".conv_out.bias", {dm});
    m->enc.resize(c.encoder_layers);
    for (int i = 0; i < c.encoder_layers; ++i) {
        std::string p = a + ".layers." + std::to_string(i);
        EncLayerW& w = m->enc[i];
        w.ln1_w = take<float>(m, p + ".self_attn_layer_norm.weight", {dm}, false);
        w.ln1_b = take<float>(m, p + ".self_attn_layer_norm.bias", {dm}, false);
        w.ln2_w = take<float>(m, p + ".final_layer_norm.weight", {dm}, false);
        w.ln2_b = take<float>(m, p + ".final_layer_norm.bias", {dm}, false);
        w.wqkv = dev_alloc<bf16>(m, (size_t)3 * dm * dm);
        w.bqkv = dev_alloc<float>(m, (size_t)3 * dm);
        const char* names[3] = {"q_proj", "k_proj", "v_proj"};
        for (int j = 0; j < 3; ++j) {
            std::string q = p + ".self_attn." + names[j];
            ASRB_CUDA_CHECK(cudaMemcpy(w.wqkv + (size_t)j * dm * dm, take<bf16>(m, q + ".weight", {dm, dm}, true),
                                       (size_t)dm * dm * 2, cudaMemcpyDeviceToDevice));
            float* bj = opt_f32(m, q + ".bias", {dm});
            if (bj) ASRB_CUDA_CHECK(cudaMemcpy(w.bqkv + (size_t)j * dm, bj, dm * 4, cudaMemcpyDeviceToDevice));
            else ASRB_CUDA_CHECK(cudaMemset(w.bqkv + (size_t)j * dm, 0, dm * 4));
            drop_raw(m, q + ".weight");
        }
        w.wo = take<bf16>(m, p + ".self_attn.out_proj.weight", {dm, dm}, true);
        w.bo = opt_f32(m, p + ".self_attn.out_proj.bias", {dm});
        w.fc1 = take<bf16>(m, p + ".fc1.weight", {ffn, dm}, true);
        w.b1 = opt_f32(m, p + ".fc1.bias", {ffn});
        w.fc2 = take<bf16>(m, p + ".fc2.weight", {dm, ffn}, true);
        w.b2 = opt_f32(m, p + ".fc2.bias", {dm});
    }
    m->lnpost_w = take<float>(m, a + ".ln_post.weight", {dm}, false);
    m->lnpost_b = take<float>(m, a + ".ln_post.bias", {dm}, false);
    m->proj1 = take<bf16>(m, a + ".proj1.weight", {dm, dm}, true);
    m->proj1_b = opt_f32(m, a + ".proj1.bias", {dm});
    m->proj2 = take<bf16>(m, a + ".proj2.weight", {(int64_t)c.output_dim, dm}, true);
    m->proj2_b = opt_f32(m, a + ".proj2.bias", {(int64_t)c.output_dim});

    const std::string t = "thinker.model";
    const int64_t H = c.hidden_size, I = c.intermediate_size, hd = c.head_dim, V = c.vocab_size;
    const int64_t qd = d.q_dim, kvd = d.kv_dim;
    m->embed = take<bf16>(m, t + ".embed_tokens.weight", {V, H}, true);
    m->lm_head = c.tie_word_embeddings ? m->embed : take<bf16>(m, "thinker.lm_head.weight", {V, H}, true);
    m->final_norm = take<float>(m, t + ".norm.weight", {H}, false);
    m->dec.resize(c.num_hidden_layers);
    for (int i = 0; i < c.num_hidden_layers; ++i) {
        std::string p = t + ".layers." + std::to_string(i);
        DecLayerW& w = m->dec[i];
        w.ln_in = take<float>(m, p + ".input_layernorm.weight", {H}, false);
        w.ln_post = take<float>(m, p + ".post_attention_layernorm.weight", {H}, false);
        w.qnorm = take<float>(m, p + ".self_attn.q_norm.weight", {hd}, false);
        w.knorm = take<float>(m, p + ".self_attn.k_norm.weight", {hd}, false);
        w.wqkv = dev_alloc<bf16>(m, (size_t)d.qkv_dim * H);
        ASRB_CUDA_CHECK(cudaMemcpy(w.wqkv, take<bf16>(m, p + ".self_attn.q_proj.weight", {qd, H}, true), (size_t)qd * H * 2, cudaMemcpyDeviceToDevice));
        ASRB_CUDA_CHECK(cudaMemcpy(w.wqkv + (size_t)qd * H, take<bf16>(m, p + ".self_attn.k_proj.weight", {kvd, H}, true), (size_t)kvd * H * 2, cudaMemcpyDeviceToDevice));
        ASRB_CUDA_CHECK(cudaMemcpy(w.wqkv + (size_t)(qd + kvd) * H, take<bf16>(m, p + ".self_attn.v_proj.weight", {kvd, H}, true), (size_t)kvd * H * 2, cudaMemcpyDeviceToDevice));
        drop_raw(m, p + ".self_attn.q_proj.weight"); drop_raw(m, p + ".self_attn.k_proj.weight"); drop_raw(m, p + ".self_attn.v_proj.weight");
        w.wo = take<bf16>(m, p + ".self_attn.o_proj.weight", {H, qd}, true);
        w.wgu = dev_alloc<bf16>(m, (size_t)2 * I * H);          // interleave rows: 2j = gate_j, 2j+1 = up_j
        ASRB_CUDA_CHECK(cudaMemcpy2D(w.wgu, (size_t)2 * H * 2, take<bf16>(m, p + ".mlp.gate_proj.weight", {I, H}, true), (size_t)H * 2, (size_t)H * 2, I, cudaMemcpyDeviceToDevice));
        ASRB_CUDA_CHECK(cudaMemcpy2D(w.wgu + H, (size_t)2 * H * 2, take<bf16>(m, p + ".mlp.up_proj.weight", {I, H}, true), (size_t)H * 2, (size_t)H * 2, I, cudaMemcpyDeviceToDevice));
        drop_raw(m, p + ".mlp.gate_proj.weight"); drop_raw(m, p + ".mlp.up_proj.weight");
        w.wdown = take<bf16>(m, p + ".mlp.down_proj.weight", {H, I}, true);
    }
    {   // pointer table of the fused decode step: norm weights in its swizzled activation layout
        std::vector<DecLayerW> tab = m->dec;
        for (DecLayerW& w : tab) { w.ln_in = swizzled_copy(m, w.ln_in, (int)H); w.ln_post = swizzled_copy(m, w.ln_post, (int)H); }
        m->final_norm_sw = swizzled_copy(m, m->final_norm, (int)H);
        m->d_dec_layers = dev_alloc<DecLayerW>(m, tab.size());
        ASRB_CUDA_CHECK(cudaMemcpy(m->d_dec_layers, tab.data(), tab.size() * sizeof(DecLayerW), cudaMemcpyHostToDevice));
    }
    // chunk-swizzled weight copies for the batch-aware fused step (dims it is instantiated for: 0.6B and the test config)
    if (c.head_dim == 128 && c.num_attention_heads == 2 * c.num_key_value_heads &&
        ((H == 1024 && qd == 2048 && I == 3072) || (H == 256 && qd == 512 && I == 512))) {
        std::vector<DecLayerW> tab = m->dec;
        for (DecLayerW& w : tab) {
            w.wqkv = swizzled_rows_copy(m, w.wqkv, (size_t)d.qkv_dim, (int)H);
            w.wo = swizzled_rows_copy(m, w.wo, (size_t)H, (int)qd);
            w.wgu = swizzled_rows_copy(m, w.wgu, (size_t)2 * I, (int)H);
            w.wdown = swizzled_rows_copy(m, w.wdown, (size_t)H, (int)I);
        }
        m->lm_head_b = swizzled_rows_copy(m, m->lm_head, (size_t)V, (int)H);
        m->d_dec_layers_b = dev_alloc<DecLayerW>(m, tab.size());
        ASRB_CUDA_CHECK(cudaMemcpy(m->d_dec_layers_b, tab.data(), tab.size() * sizeof(DecLayerW), cudaMemcpyHostToDevice));
    }
    if (decode_mega_dims(c)) {                                  // int8 lm_head copy for the single-sequence fused step
        const int n = (int)H / 64 + 6;                       // roundings on a term's path in row_dot4 / row_dot (and row_dot4_q)
        const double u = std::ldexp(1.0, -24);
        auto gamma = [&](int k) { return k * u / (1.0 - k * u); };
        m->lm_head_q = dev_alloc<int8_t>(m, (size_t)V * H);
        m->lm_head_sc = dev_alloc<float2>(m, (size_t)V);
        quantize_head_kernel<<<(unsigned)((V + 7) / 8), 256>>>(m->lm_head, m->lm_head_q, m->lm_head_sc, (int)V, (int)H, gamma(n), gamma(n + 1));
        ASRB_CUDA_CHECK(cudaGetLastError());
    }
    build_mel_tables(m);
    build_pos_tables(m);
    ASRB_CUDA_CHECK(cudaDeviceSynchronize());
    m->finalized = true;
}

}  // namespace asrb
