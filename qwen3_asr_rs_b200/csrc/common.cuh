// common.cuh -- shared device helpers for the sm_90a kernels of the Qwen3-ASR hot path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdexcept>
#include <string>

namespace asrb {

struct Error : public std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define ASRB_CUDA_CHECK(expr)                                                              \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess)                                                             \
            throw ::asrb::Error(2, std::string(#expr) + " failed: " + cudaGetErrorString(_e) + \
                                       " (" __FILE__ ":" + std::to_string(__LINE__) + ")"); \
    } while (0)

#define ASRB_REQUIRE(cond, code, msg)                                          \
    do {                                                                       \
        if (!(cond)) throw ::asrb::Error((code), std::string(msg));            \
    } while (0)

typedef __nv_bfloat16 bf16;

// ---- bf16 <-> fp32 (bit-exact up-cast, as src/weights.rs:134-142) --------------------
__device__ __forceinline__ float bf16_bits_to_f32(uint32_t bits16) { return __uint_as_float(bits16 << 16); }
__device__ __forceinline__ float bf16_lo(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t packed) { return __uint_as_float(packed & 0xffff0000u); }

// ---- exact 3-way bf16 split of an fp32 activation: x == hi + mid + lo (to 1 ulp) -----
// GEMM A-operands are stored as three bf16 planes so bf16 wgmma MMAs with exact
// bf16 weights reproduce fp32 products (bf16*bf16 is exact in fp32; fp32 accumulate).
struct Split3 { bf16 hi, mid, lo; };
__device__ __forceinline__ Split3 split3(float x) {
    Split3 s;
    s.hi = __float2bfloat16_rn(x);
    float r = x - __bfloat162float(s.hi);
    s.mid = __float2bfloat16_rn(r);
    r = r - __bfloat162float(s.mid);
    s.lo = __float2bfloat16_rn(r);
    return s;
}
__device__ __forceinline__ void store_split3(bf16* base, size_t plane_stride, size_t idx, float x) {
    Split3 s = split3(x);
    base[idx] = s.hi;
    base[plane_stride + idx] = s.mid;
    base[2 * plane_stride + idx] = s.lo;
}
__device__ __forceinline__ float load_split3(const bf16* base, size_t plane_stride, size_t idx, int nplanes) {
    float v = __bfloat162float(base[idx]);
    if (nplanes > 1) v += __bfloat162float(base[plane_stride + idx]);
    if (nplanes > 2) v += __bfloat162float(base[2 * plane_stride + idx]);
    return v;
}

// ---- math matching the ATen CPU ops the reference's tch arm dispatches to --------------
__device__ __forceinline__ float gelu_erf(float x) {            // gelu("none"), src/tensor.rs:350
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }   // src/tensor.rs:354

// ---- warp / block reductions -----------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// blockDim.x multiple of 32, <= 1024; scratch >= 32 floats; result broadcast to all threads
__device__ __forceinline__ float block_sum(float v, float* scratch) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) scratch[w] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : 0.f;
    r = warp_sum(r);
    return r;
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) scratch[w] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : -INFINITY;
    r = warp_max(r);
    return r;
}

// ---- log-sum-exp partial records (max m, s = sum_j exp(l_j - m)) beside the greedy argmax ----------------
// s rescaled from max m to max M >= m; an empty record (m = -inf, s = 0) stays 0, and m == M skips the exp
__device__ __forceinline__ float lse_rescale(float s, float m, float M) { return m == M ? s : s * expf(m - M); }
// fold logit v of `row` into a running (argmax, sum): strict > keeps the first maximum, as the plain argmax does
__device__ __forceinline__ void lse_fold(float v, int row, float& best_v, int& best_i, float& best_s) {
    if (v > best_v) { best_s = lse_rescale(best_s, best_v, v) + 1.f; best_v = v; best_i = row; }
    else best_s += expf(v - best_v);
}
// merge two records (m, s), (om, os) into (max, rescaled sum); symmetric, so both lanes of a shuffle agree bitwise
__device__ __forceinline__ float lse_merge(float m, float s, float om, float os) {
    const float M = fmaxf(m, om);
    return lse_rescale(s, m, M) + lse_rescale(os, om, M);
}

// ---- top-k candidate lists beside the greedy argmax -----------------------------------------------------
// TK_MAX (logit, id) pairs kept sorted best first under the argmax's total order: logit descending, then id ascending.
// Ids are distinct across the rows folded anywhere, so the top TK_MAX of any union is one set whatever the merge order.
// Empty entries are (-inf, 0x7fffffff).  All indices are compile-time: the lists stay in registers.
constexpr int TK_MAX = 8;
struct TopK { float v[TK_MAX]; int i[TK_MAX]; };
__device__ __forceinline__ bool tk_before(float a, int ai, float b, int bi) { return a > b || (a == b && ai < bi); }
__device__ __forceinline__ void tk_init(TopK& t) {
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j) { t.v[j] = -INFINITY; t.i[j] = 0x7fffffff; }
}
// fold logit v of `row`: one compare unless it beats the tail, then it bubbles into place and the tail drops out
__device__ __forceinline__ void tk_insert(TopK& t, float v, int row) {
    if (!tk_before(v, row, t.v[TK_MAX - 1], t.i[TK_MAX - 1])) return;
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j)
        if (tk_before(v, row, t.v[j], t.i[j])) { const float tv = t.v[j]; const int ti = t.i[j]; t.v[j] = v; t.i[j] = row; v = tv; row = ti; }
}
// t <- top TK_MAX of t and u (both sorted): the better of t[j] and u[TK_MAX-1-j] is a bitonic sequence holding the top
// TK_MAX of the union, which three half-cleaner stages sort
__device__ __forceinline__ void tk_merge(TopK& t, const TopK& u) {
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j)
        if (!tk_before(t.v[j], t.i[j], u.v[TK_MAX - 1 - j], u.i[TK_MAX - 1 - j])) { t.v[j] = u.v[TK_MAX - 1 - j]; t.i[j] = u.i[TK_MAX - 1 - j]; }
#pragma unroll
    for (int d = TK_MAX / 2; d > 0; d >>= 1)
#pragma unroll
        for (int j = 0; j < TK_MAX; ++j)
            if ((j & d) == 0 && tk_before(t.v[j + d], t.i[j + d], t.v[j], t.i[j])) {
                const float tv = t.v[j]; const int ti = t.i[j];
                t.v[j] = t.v[j + d]; t.i[j] = t.i[j + d]; t.v[j + d] = tv; t.i[j + d] = ti;
            }
}
// merge with the list of lane ^ o (both lanes end with the same list)
__device__ __forceinline__ void tk_merge_xor(TopK& t, int o) {
    TopK u;
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j) { u.v[j] = __shfl_xor_sync(0xffffffffu, t.v[j], o); u.i[j] = __shfl_xor_sync(0xffffffffu, t.i[j], o); }
    tk_merge(t, u);
}
__device__ __forceinline__ void tk_store(const TopK& t, float* v, int* i) {
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j) { v[j] = t.v[j]; i[j] = t.i[j]; }
}
// merge a list published by another thread of this CTA (shared memory) or, with L2 loads, by another CTA
__device__ __forceinline__ void tk_merge_from(TopK& t, const float* v, const int* i, bool l2) {
    TopK u;
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j) { u.v[j] = l2 ? __ldcg(v + j) : v[j]; u.i[j] = l2 ? __ldcg(i + j) : i[j]; }
    tk_merge(t, u);
}
// the step's record: entry j = (l_j - l_0) + lp where l_0 is the maximum logit and lp = -log S the selected token's
// log-probability; entry 0 is lp itself, bitwise
__device__ __forceinline__ void tk_write(const TopK& t, float lp, int* ids, float* lps) {
#pragma unroll
    for (int j = 0; j < TK_MAX; ++j) { ids[j] = t.i[j]; lps[j] = j == 0 ? lp : (t.v[j] - t.v[0]) + lp; }
}

// ---- seeded temperature sampling by the Gumbel-max trick ------------------------------------------------
// For sequence row r (0-based in the call's batch), step n (ids already generated for that sequence when the step
// selects; 0 for the token selected after the prefill, the EOS-selecting step included) and token id v:
//   x0    = word 0 of Philox4x32-10 (Random123 constants), key (seed & 0xffffffff, seed >> 32), counter (v, n, r, 0)
//   u     = (float)((x0 >> 8) | 1) * 2^-24               exact, in [2^-24, 1 - 2^-24]: never 0 or 1
//   g_v   = -logf(-logf(u))                              full-precision logf, g in about [-2.8, 16.6]
//   key_v = fmaf(l_v, inv_t, g_v)                        inv_t = (float)(1.0 / T), computed on the host in double
// and the selected id is the argmax of key_v under (key descending, id ascending), the greedy argmax's own order.  The
// draw is a pure function of (seed, r, n, v): every decode path selects the same ids, whatever its merge order.
// With LOGPROB the kernels also keep the raw (max, sum of exponentials) record of the logits and the raw logit of the
// best-key row, so the recorded value is the model's own (temperature-1) log-probability (l_sel - M) - log S.
struct SampleParams {       // device-resident, written at the prefill: a captured graph reads the values of its run
    float inv_t;            // 1 / temperature
    uint32_t k0, k1;        // seed & 0xffffffff, seed >> 32
};
__host__ __device__ __forceinline__ uint32_t philox4x32_10_x0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        if (i > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        c0 = n0; c1 = (uint32_t)p1; c2 = n2; c3 = (uint32_t)p0;
    }
    return c0;
}
// one sequence's draw context: the run's parameters and the (step, row) of the counter
struct Draw {
    float inv_t; uint32_t k0, k1, n, r;
};
__device__ __forceinline__ Draw make_draw(const SampleParams* sp, int n, int r) {
    Draw d; d.inv_t = __ldg(&sp->inv_t); d.k0 = __ldg(&sp->k0); d.k1 = __ldg(&sp->k1); d.n = (uint32_t)n; d.r = (uint32_t)r;
    return d;
}
__device__ __forceinline__ float gumbel_noise(uint32_t x0) {
    const float u = (float)((x0 >> 8) | 1u) * 0x1p-24f;
    return -logf(-logf(u));
}
__device__ __forceinline__ float sample_key(const Draw& d, float l, int v) {
    return fmaf(l, d.inv_t, gumbel_noise(philox4x32_10_x0((uint32_t)v, d.n, d.r, 0u, d.k0, d.k1)));
}
// fold logit l of `row` (rows ascend per thread: strict > keeps the first maximum): (best_v, best_i) = argmax of the
// keys; LOGPROB: (m, best_s) = raw (max, sum of exp(l - m)) record, sel = raw logit of the best-key row
template <bool LOGPROB>
__device__ __forceinline__ void sample_fold(const Draw& d, float l, int row, float& best_v, int& best_i, float& best_s, float& m,
                                            float& sel) {
    const float k = sample_key(d, l, row);
    if (k > best_v) { best_v = k; best_i = row; if constexpr (LOGPROB) sel = l; }
    if constexpr (LOGPROB) {
        if (l > m) { best_s = lse_rescale(best_s, m, l) + 1.f; m = l; }
        else best_s += expf(l - m);
    }
}
// merge with the records of lane ^ o (both lanes end with the same records)
template <bool LOGPROB>
__device__ __forceinline__ void sample_merge_xor(int o, float& best_v, int& best_i, float& best_s, float& m, float& sel) {
    const float ov = __shfl_xor_sync(0xffffffffu, best_v, o); const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    float osel = 0.f;
    if constexpr (LOGPROB) {
        osel = __shfl_xor_sync(0xffffffffu, sel, o);
        const float om = __shfl_xor_sync(0xffffffffu, m, o);
        best_s = lse_merge(m, best_s, om, __shfl_xor_sync(0xffffffffu, best_s, o));
        m = fmaxf(m, om);
    }
    if (ov > best_v || (ov == best_v && oi < best_i)) { best_v = ov; best_i = oi; if constexpr (LOGPROB) sel = osel; }
}

// ---- repetition controls: no-repeat n-gram bans and a repetition penalty --------------------------------
// For sequence b at step n the history is ids[0 .. n), the ids this run generated for it (ids_out; never the prompt,
// context, audio or forced-language ids, never EOS).  Before any use of the step's logits, logit l_v becomes
//   penalty  v in the history:  l_v < 0 ? l_v * theta : l_v / theta       (IEEE fp32 multiply / round-to-nearest divide)
//   ban      N >= 1 and some i in [0, n - N] with ids[i .. i+N-2] == ids[n-N+1 .. n-1], v = ids[i+N-1]:  -inf
// Each sequence's rule is a pair of bit arrays over a range of ids, "in history" and "banned", built from its ids_out row
// (rep_mark) and tested once per lm_head row at the fold (rep_logit).  The fused steps build them per CTA for the CTA's
// own lm_head rows while layer 0's weights stream in; the per-phase path builds them over the whole vocabulary in
// rep_mask_kernel.  A banned row takes part in no fold: its exp is 0, it is never the argmax, never a sampling draw and
// never a candidate (the vocabulary always keeps more than TK_MAX finite logits).
struct RepParams {          // device-resident, written at the prefill: a captured graph reads the values of its run
    float theta;            // penalty, 1 = off
    int ngram;              // N, 0 = off
};
// one sequence's bit arrays: bit (v & 31) of word (v >> 5) - w0 of hist / ban, for ids v of the range they cover
struct RepBits {
    const uint32_t* hist; const uint32_t* ban; int w0; float theta;
};
// set the bits of ids in [lo, hi) (w0 = lo >> 5) for history ids[0 .. n); thread t of nt; the arrays are zeroed and the
// caller's threads synchronised before, and again before the bits are read
__device__ __forceinline__ void rep_mark(const int* __restrict__ ids, int n, int N, int lo, int hi, uint32_t* hist,
                                         uint32_t* ban, int t, int nt) {
    const int w0 = lo >> 5;
    for (int i = t; i < n; i += nt) {
        const int v = __ldcg(ids + i);
        if (v >= lo && v < hi) atomicOr(hist + ((v >> 5) - w0), 1u << (v & 31));
        if (N >= 1 && i <= n - N) {            // the N-gram starting at i continues the current (N-1)-suffix
            bool match = true;
            for (int j = 0; j < N - 1 && match; ++j) match = __ldcg(ids + i + j) == __ldcg(ids + n - N + 1 + j);
            if (match) {
                const int u = __ldcg(ids + i + N - 1);
                if (u >= lo && u < hi) atomicOr(ban + ((u >> 5) - w0), 1u << (u & 31));
            }
        }
    }
}
// l <- the processed logit of row v; false: v is banned (l' = -inf) and takes part in no fold
__device__ __forceinline__ bool rep_logit(const RepBits& r, int v, float& l) {
    const int w = (v >> 5) - r.w0;
    const uint32_t bit = 1u << (v & 31);
    if (r.ban[w] & bit) { l = -INFINITY; return false; }
    if (r.hist[w] & bit) l = l < 0.f ? l * r.theta : l / r.theta;
    return true;
}
// the fold sites' form: REP = false compiles to nothing
template <bool REP>
__device__ __forceinline__ bool rep_keep(const RepBits* r, int v, float& l) {
    if constexpr (REP) return rep_logit(*r, v, l);
    else return true;
}

// order-preserving float <-> int key (for atomicMax on floats of either sign)
__device__ __host__ __forceinline__ int float_to_ordered(float f) {
#ifdef __CUDA_ARCH__
    int i = __float_as_int(f);
#else
    int i; memcpy(&i, &f, 4);
#endif
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int k) {
    int i = k >= 0 ? k : k ^ 0x7fffffff;
    return __int_as_float(i);
}

}  // namespace asrb
