// decode_mega.cu -- one greedy decode iteration (inference.rs:160-200) as ONE persistent kernel.
//
// Why: at batch 1 a decoder forward is 1.19 GB of weights read once (HBM-bound, ~360 us at the
// H100 data sheet's 3.35 TB/s) but has ~141 dependent phases (28 layers x {qkv, attention, o_proj, gate/up,
// down} + lm_head).  As separate kernels each phase pays launch latency and a cold weight stream;
// with device-wide barriers each phase pays an atomic + spin + re-read.
// Here one CTA per SM stays resident for the whole step:
//   * a producer warp streams this CTA's slice of EVERY weight matrix and the K/V rows of earlier
//     positions, in consumption order, into a shared-memory ring with cp.async.bulk (TMA bulk copy) +
//     mbarrier transaction counts.  None of these addresses depend on activations, so the producer
//     runs AHEAD across phase boundaries: HBM stays busy while consumers wait for activations.
//   * 8 consumer warps do the fp32 GEMV from shared memory (activation vector held in registers,
//     bf16 -> fp32 up-cast is exact, fp32 FMA accumulate).
//   * activations are exchanged between CTAs WITHOUT barriers, and data and "ready" flag arrive in the
//     same L2 round trip (the low-latency protocol of collective libraries, on-chip).  The vectors every
//     CTA reads in full (x after o_proj and after down_proj, attention output, SwiGLU activations) travel
//     as self-validating 4-byte words (the fp32 value itself, 0xFFFFFFFF = not written yet), published
//     with one fire-and-forget `red.and` and polled as 16-byte quads; two sets of per-layer regions
//     alternate between launches (mega_common.cuh).  The few-reader q/k/v rows and attention partials
//     travel in 8-byte {value, tag} words (tag = launch epoch/layer/phase), published with one 64-bit
//     `red.max` (performed at L2 immediately; the tag grows monotonically so max acts as an exchange)
//     and polled until the tags match.
//   * attention (QK-RMSNorm + RoPE + KV append + softmax.V) is split over kv-heads x 64-key tiles;
//     the tile-0 CTA of each kv-head merges the partials and publishes the head outputs.
//   * the last CTA to finish the lm_head performs the greedy bookkeeping (argmax, EOS, append,
//     embedding of the next token), so there is no host sync and no extra launch per token.
// Reference semantics per phase: see decode.cu.  The kernel advances ONE sequence; a batch is B back-to-back launches
// (decode.cu remains the path for logits output, other model dimensions and contexts beyond 1152 keys).
#include <cfloat>
#include <climits>
#include "mega_common.cuh"

namespace asrb {

namespace mega {

struct Params {
    const DecLayerW* layers;     // device array [L]
    const bf16* lm_head;
    const bf16* embed;
    const float* final_norm;
    const float* rope_cos; const float* rope_sin;
    float eps;
    int L, H, QD, KVD, I, V, nq, nkv, group;
    // plain state (kernel-boundary visibility)
    float* x;                    // [H] embedding of the pending token (in) / of the next token (out)
    float* kcache; float* vcache; size_t cache_layer_stride; int max_ctx;
    int nsplit;
    float* part_val; int* part_idx;     // [gridDim.x]
    int* pos; int* done; int* next_id; int* ids_out; int* n_out; int max_new;
    unsigned* bar;               // [0] finish ticket, [1] launch epoch (starts at 1; 0 marks never-written words),
                                 // [3] executed launches of this kernel (selects the set of self-validating words)
    uint2* qkv_ll; uint2* part_ll;      // tagged exchange buffers ({value, tag} words)
    uint32_t* sx;                // self-validating words [2 sets][L][x_o H | x_d H | attn QD | act I]
    long long* dbg;              // optional timeline [2][DBG_SLOTS] of clock64 (CTA 0 and CTA G-1), else null
    // LOGPROB instantiations only (appended: the offsets above stay those of the default instantiations)
    float* part_sum;             // [gridDim.x] sum of exp(logit - part_val) over the CTA's lm_head rows
    float* lp_out;               // [max_new] log-probability of each appended token
    float* eos_lp;               // log-probability of the EOS token that ends the sequence
    // TOPK instantiations only (appended as well)
    float* tk_part_val; int* tk_part_idx;   // [gridDim.x][TK_MAX] the CTA's best (logit, id) candidates
    int* tk_ids; float* tk_lp;              // [max_new][TK_MAX] candidates of each appended token's step, best first
    int* tk_eos_ids; float* tk_eos_lp;      // [TK_MAX] those of the step that selects EOS
    // SAMPLE instantiations only (appended as well)
    const SampleParams* smp;     // 1 / temperature and seed of the run
    int row;                     // the sequence's row in the call's batch (the draw's counter)
    float* part_max; float* part_sel;       // LOGPROB: [gridDim.x] raw maximum logit, raw logit of the best-key row
    // REP instantiations only (appended as well)
    uint32_t* rep_bits;          // [gridDim.x][2][rep_words] each CTA's history / banned bits of its lm_head rows
    int rep_words;
    const RepParams* rep;        // the run's penalty and N
    // default (greedy) instantiations only (appended as well): the lm_head streams from its int8 copy
    const int8_t* lm_head_q;     // [V][H]
    const float2* lm_head_sc;    // [V] {scale s_r, bound constant C_r} (model.cu quantize_head_kernel)
    unsigned long long* hq_stats;   // [0] rows recomputed in this step, [1] in all steps, [2] most in one step, [3] fallbacks
};

static_assert(KV_KEYS * HD * 4 == SLOT_BYTES, "K / V tiles travel through the weight ring: one tile per slot");

// GEMV row mapping: a row of K bf16 weights is contracted by one warp; lane `lane` holds the activations of elements
// (c * 32 + lane) * 8 .. +8 for every 256-element chunk c in registers.
template <int K>
__device__ __forceinline__ void load_xr(const float* xs, float (&xr)[K / 32], int lane) {
    const int sw = ((lane >> 2) & 1) * 4;          // xs_swz for this lane's two 16-byte groups: swapped when bit 3 of k is set
#pragma unroll
    for (int c = 0; c < K / 256; ++c) {
        const float4 a = *reinterpret_cast<const float4*>(xs + (c * 32 + lane) * 8 + sw);
        const float4 b = *reinterpret_cast<const float4*>(xs + (c * 32 + lane) * 8 + 4 - sw);
        xr[c * 8 + 0] = a.x; xr[c * 8 + 1] = a.y; xr[c * 8 + 2] = a.z; xr[c * 8 + 3] = a.w;
        xr[c * 8 + 4] = b.x; xr[c * 8 + 5] = b.y; xr[c * 8 + 6] = b.z; xr[c * 8 + 7] = b.w;
    }
}
// same, with the RMSNorm applied on the fly: xr = (x * r) * w  (rounding order of layers.rs:48-54)
template <int K>
__device__ __forceinline__ void load_xr_norm(const float* xs, const float* wn, float r, float (&xr)[K / 32], int lane) {
    const int sw = ((lane >> 2) & 1) * 4;          // both vectors are stored in the xs_swz layout
#pragma unroll
    for (int c = 0; c < K / 256; ++c) {
        const int o = (c * 32 + lane) * 8;
        const float4 a = *reinterpret_cast<const float4*>(xs + o + sw), b = *reinterpret_cast<const float4*>(xs + o + 4 - sw);
        const float4 wa = *reinterpret_cast<const float4*>(wn + o + sw), wb = *reinterpret_cast<const float4*>(wn + o + 4 - sw);
        xr[c * 8 + 0] = (a.x * r) * wa.x; xr[c * 8 + 1] = (a.y * r) * wa.y; xr[c * 8 + 2] = (a.z * r) * wa.z; xr[c * 8 + 3] = (a.w * r) * wa.w;
        xr[c * 8 + 4] = (b.x * r) * wb.x; xr[c * 8 + 5] = (b.y * r) * wb.y; xr[c * 8 + 6] = (b.z * r) * wb.z; xr[c * 8 + 7] = (b.w * r) * wb.w;
    }
}

template <int K>
__device__ __forceinline__ float row_dot(const uint4* wrow, const float (&xr)[K / 32], int lane) {
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int c = 0; c < K / 256; ++c) {
        const uint4 w = wrow[c * 32 + lane];
        a0 = fmaf(bf16_lo(w.x), xr[c * 8 + 0], a0); a1 = fmaf(bf16_hi(w.x), xr[c * 8 + 1], a1);
        a0 = fmaf(bf16_lo(w.y), xr[c * 8 + 2], a0); a1 = fmaf(bf16_hi(w.y), xr[c * 8 + 3], a1);
        a0 = fmaf(bf16_lo(w.z), xr[c * 8 + 4], a0); a1 = fmaf(bf16_hi(w.z), xr[c * 8 + 5], a1);
        a0 = fmaf(bf16_lo(w.w), xr[c * 8 + 6], a0); a1 = fmaf(bf16_hi(w.w), xr[c * 8 + 7], a1);
    }
    return warp_sum(a0 + a1);
}
// two rows at once (independent FMA chains, one shared reduction): the result of row 0 ends up in lanes 0-15 and
// that of row 1 in lanes 16-31
template <int K>
__device__ __forceinline__ float row_dot2(const uint4* w0, const uint4* w1, const float (&xr)[K / 32], int lane) {
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
#pragma unroll
    for (int c = 0; c < K / 256; ++c) {
        const uint4 w = w0[c * 32 + lane], v = w1[c * 32 + lane];
        a0 = fmaf(bf16_lo(w.x), xr[c * 8 + 0], a0); a1 = fmaf(bf16_hi(w.x), xr[c * 8 + 1], a1);
        b0 = fmaf(bf16_lo(v.x), xr[c * 8 + 0], b0); b1 = fmaf(bf16_hi(v.x), xr[c * 8 + 1], b1);
        a0 = fmaf(bf16_lo(w.y), xr[c * 8 + 2], a0); a1 = fmaf(bf16_hi(w.y), xr[c * 8 + 3], a1);
        b0 = fmaf(bf16_lo(v.y), xr[c * 8 + 2], b0); b1 = fmaf(bf16_hi(v.y), xr[c * 8 + 3], b1);
        a0 = fmaf(bf16_lo(w.z), xr[c * 8 + 4], a0); a1 = fmaf(bf16_hi(w.z), xr[c * 8 + 5], a1);
        b0 = fmaf(bf16_lo(v.z), xr[c * 8 + 4], b0); b1 = fmaf(bf16_hi(v.z), xr[c * 8 + 5], b1);
        a0 = fmaf(bf16_lo(w.w), xr[c * 8 + 6], a0); a1 = fmaf(bf16_hi(w.w), xr[c * 8 + 7], a1);
        b0 = fmaf(bf16_lo(v.w), xr[c * 8 + 6], b0); b1 = fmaf(bf16_hi(v.w), xr[c * 8 + 7], b1);
    }
    const float ra = a0 + a1, rb = b0 + b1;
    const bool hi = lane & 16;
    float keep = (hi ? rb : ra) + __shfl_xor_sync(0xffffffffu, hi ? ra : rb, 16);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) keep += __shfl_xor_sync(0xffffffffu, keep, o);
    return keep;
}

// same contraction with the activation vector read from shared memory (long K: keeps registers free)
template <int K>
__device__ __forceinline__ float row_dot_smem(const uint4* wrow, const float* xs, int lane) {
    float a0 = 0.f, a1 = 0.f;
    const int sw = ((lane >> 2) & 1) * 4;
#pragma unroll 4
    for (int c = 0; c < K / 256; ++c) {
        const uint4 w = wrow[c * 32 + lane];
        const float4 xa = *reinterpret_cast<const float4*>(xs + (c * 32 + lane) * 8 + sw);
        const float4 xb = *reinterpret_cast<const float4*>(xs + (c * 32 + lane) * 8 + 4 - sw);
        a0 = fmaf(bf16_lo(w.x), xa.x, a0); a1 = fmaf(bf16_hi(w.x), xa.y, a1);
        a0 = fmaf(bf16_lo(w.y), xa.z, a0); a1 = fmaf(bf16_hi(w.y), xa.w, a1);
        a0 = fmaf(bf16_lo(w.z), xb.x, a0); a1 = fmaf(bf16_hi(w.z), xb.y, a1);
        a0 = fmaf(bf16_lo(w.w), xb.z, a0); a1 = fmaf(bf16_hi(w.w), xb.w, a1);
    }
    return warp_sum(a0 + a1);
}


// four rows at once (K <= 1024, activations in registers): 8 independent FMA chains and ONE 6-shuffle transposed
// reduction for the four rows instead of two 5-shuffle reductions of row pairs.  The sum of row j ends up in all 8 lanes
// with (lane >> 3) == j.
template <int K>
__device__ __forceinline__ float row_dot4(const uint4* w0, const uint4* w1, const uint4* w2, const uint4* w3,
                                          const float (&xr)[K / 32], int lane) {
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f, c0 = 0.f, c1 = 0.f, d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int c = 0; c < K / 256; ++c) {
        const uint4 wa = w0[c * 32 + lane], wb = w1[c * 32 + lane], wc = w2[c * 32 + lane], wd = w3[c * 32 + lane];
#define ROW4_STEP(F, X0, X1)                                                                                          \
        a0 = fmaf(bf16_lo(wa.F), X0, a0); a1 = fmaf(bf16_hi(wa.F), X1, a1);                                           \
        b0 = fmaf(bf16_lo(wb.F), X0, b0); b1 = fmaf(bf16_hi(wb.F), X1, b1);                                           \
        c0 = fmaf(bf16_lo(wc.F), X0, c0); c1 = fmaf(bf16_hi(wc.F), X1, c1);                                           \
        d0 = fmaf(bf16_lo(wd.F), X0, d0); d1 = fmaf(bf16_hi(wd.F), X1, d1);
        ROW4_STEP(x, xr[c * 8 + 0], xr[c * 8 + 1])
        ROW4_STEP(y, xr[c * 8 + 2], xr[c * 8 + 3])
        ROW4_STEP(z, xr[c * 8 + 4], xr[c * 8 + 5])
        ROW4_STEP(w, xr[c * 8 + 6], xr[c * 8 + 7])
#undef ROW4_STEP
    }
    const float ra = a0 + a1, rb = b0 + b1, rc = c0 + c1, rd = d0 + d1;
    const bool h16 = lane & 16, h8 = lane & 8;
    float k0 = (h16 ? rc : ra) + __shfl_xor_sync(0xffffffffu, h16 ? ra : rc, 16);      // rows {0,1} stay low, {2,3} high
    float k1 = (h16 ? rd : rb) + __shfl_xor_sync(0xffffffffu, h16 ? rb : rd, 16);
    float keep = (h8 ? k1 : k0) + __shfl_xor_sync(0xffffffffu, h8 ? k0 : k1, 8);
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) keep += __shfl_xor_sync(0xffffffffu, keep, o);
    return keep;
}

// 4 int8 weights (one word, element 0 in the low byte) -> 4 exact floats: byte b + 128 becomes the low mantissa byte of
// 2^23, and 2^23 + 128 is subtracted (one PRMT and one FADD per element instead of a quarter-rate I2F)
__device__ __forceinline__ void i8x4_f32(uint32_t w, float (&f)[4]) {
    const uint32_t u = w ^ 0x80808080u;
    f[0] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7540)) - 8388736.f;
    f[1] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7541)) - 8388736.f;
    f[2] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7542)) - 8388736.f;
    f[3] = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7543)) - 8388736.f;
}
// sum_i q_i x_i of four int8 rows (8 bytes per lane and 256-element chunk, the elements of row_dot4's lane mapping), with
// row_dot4's structure: two FMA chains of K / 64 terms per lane and row, one add, a 5-level butterfly.  The total of row j
// ends up in the lanes with (lane >> 3) == j.
template <int K>
__device__ __forceinline__ float row_dot4_q(const uint2* w0, const uint2* w1, const uint2* w2, const uint2* w3,
                                            const float (&xr)[K / 32], int lane) {
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f, c0 = 0.f, c1 = 0.f, d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int c = 0; c < K / 256; ++c) {
        const uint2 wa = w0[c * 32 + lane], wb = w1[c * 32 + lane], wc = w2[c * 32 + lane], wd = w3[c * 32 + lane];
        float fa[4], fb[4], fc[4], fd[4];
#define ROWQ_STEP(F, O)                                                                                               \
        i8x4_f32(wa.F, fa); i8x4_f32(wb.F, fb); i8x4_f32(wc.F, fc); i8x4_f32(wd.F, fd);                               \
        a0 = fmaf(fa[0], xr[c * 8 + O], a0); a1 = fmaf(fa[1], xr[c * 8 + O + 1], a1);                                 \
        b0 = fmaf(fb[0], xr[c * 8 + O], b0); b1 = fmaf(fb[1], xr[c * 8 + O + 1], b1);                                 \
        c0 = fmaf(fc[0], xr[c * 8 + O], c0); c1 = fmaf(fc[1], xr[c * 8 + O + 1], c1);                                 \
        d0 = fmaf(fd[0], xr[c * 8 + O], d0); d1 = fmaf(fd[1], xr[c * 8 + O + 1], d1);                                 \
        a0 = fmaf(fa[2], xr[c * 8 + O + 2], a0); a1 = fmaf(fa[3], xr[c * 8 + O + 3], a1);                             \
        b0 = fmaf(fb[2], xr[c * 8 + O + 2], b0); b1 = fmaf(fb[3], xr[c * 8 + O + 3], b1);                             \
        c0 = fmaf(fc[2], xr[c * 8 + O + 2], c0); c1 = fmaf(fc[3], xr[c * 8 + O + 3], c1);                             \
        d0 = fmaf(fd[2], xr[c * 8 + O + 2], d0); d1 = fmaf(fd[3], xr[c * 8 + O + 3], d1);
        ROWQ_STEP(x, 0)
        ROWQ_STEP(y, 4)
#undef ROWQ_STEP
    }
    const float ra = a0 + a1, rb = b0 + b1, rc = c0 + c1, rd = d0 + d1;
    const bool h16 = lane & 16, h8 = lane & 8;
    float k0 = (h16 ? rc : ra) + __shfl_xor_sync(0xffffffffu, h16 ? ra : rc, 16);
    float k1 = (h16 ? rd : rb) + __shfl_xor_sync(0xffffffffu, h16 ? rb : rd, 16);
    float keep = (h8 ? k1 : k0) + __shfl_xor_sync(0xffffffffu, h8 ? k0 : k1, 8);
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) keep += __shfl_xor_sync(0xffffffffu, keep, o);
    return keep;
}
// order-preserving int image of a float (-0 and +0 map to the same value): lets a CTA keep its running threshold with
// one shared-memory atomicMax
__device__ __forceinline__ int f32_ord(float f) { const int i = __float_as_int(f); return i >= 0 ? i : -(i & 0x7fffffff); }

static constexpr int HQ_CAP = 256;                      // candidate rows one CTA lists per step (xs region)

// Greedy lm_head of the default instantiation (DESIGN.md section 4.1, "lm_head from its int8 copy").  The producer
// streams the CTA's rows of the int8 copy (SLOT_BYTES / K rows per slot).  Row r yields a_r = s_r * sum_i q_ri x_i and
// B_r = |x|_2 C_r, rounded outwards, with the logit f_r the bf16 row gives under row_dot4 / row_dot in [a_r - B_r, a_r + B_r].
// The CTA keeps T = max_r (a_r - B_r) and lists the rows with a_r + B_r >= T (the threshold only grows, so a row left out
// when it was seen stays out).  Every row whose f_r equals the CTA's maximum is listed; the listed rows whose upper bound
// reaches the final T are recomputed from their bf16 rows with row_dot -- row_dot4's arithmetic, so f_r is bit for bit
// that of the bf16 form -- and folded by (value, lower id).  A list longer than HQ_CAP, or a non-finite bound, recomputes
// every row of the slice instead.  best_v / best_i end up the same in every lane of a warp.  xs holds the candidate list
// after the register load; its header st: [0] T as f32_ord, [1] rows listed, [2] non-finite bound seen, [3] rows recomputed.
template <int K>
__device__ __forceinline__ void consume_head_q(const Slice& s, const Ring& ring, uint32_t& q, float* xs, const float2* hsc,
                                               float& best_v, int& best_i, const float* norm_w, float norm_r) {
    static_assert(SLOT_BYTES / K == 16 || (SLOT_BYTES / K) % 32 == 0, "a turn is 32 rows: one slot, or a pair of 16-row slots");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NU = K / 8;                      // 8-byte groups per int8 row
    float xr[K / 32];
    load_xr_norm<K>(xs, norm_w, norm_r, xr, lane);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < K / 32; ++i) ss = fmaf(xr[i], xr[i], ss);
    // |x|_2 rounded up: the relative 2^-12 covers the rounding of the squares' sum, the square root and the product below
    ss = warp_sum(ss);
    const float nx = __fmul_ru(sqrtf(ss), 1.f + 0x1p-12f);
    int* const st = reinterpret_cast<int*>(xs);
    int2* const cl = reinterpret_cast<int2*>(xs + 4);              // [HQ_CAP] (row, f32_ord of its upper bound)
    cons_sync();                                   // every warp holds its copy: xs becomes the candidate list
    // below |x|_2^2 = 2^-60 the squares may have underflowed and |x|_2 no longer bounds anything: recompute in full
    if (threadIdx.x == 0) { st[0] = INT_MIN; st[1] = 0; st[2] = !(ss >= 0x1p-60f); st[3] = 0; }
    cons_sync();
    // a lane's t-th row is s.r0 + 32 t + 4 warp + (lane >> 3) (every turn but the last is 32 rows); the 8 lanes of a row
    // group fetch {s_r, C_r} of 8 turns ahead, one turn each, so the loads have 8 turns to arrive
    const int j = lane >> 3;
    auto fetch = [&](int t) { return __ldg(hsc + min(s.r0 + 32 * t + 4 * warp + j, s.r1 - 1)); };
    float2 win = fetch(lane & 7), nxt = fetch(8 + (lane & 7));
    int t = 0;
    for (int r = s.r0; r < s.r1;) {
        const int rowsA = min(s.rpc, s.r1 - r);
        const uint32_t slotA = q % ring.nslot;
        mbar_wait(&ring.full[slotA], (q / ring.nslot) & 1);
        const bool pair = s.rpc < 32 && r + rowsA < s.r1;
        const int rowsB = pair ? min(s.rpc, s.r1 - r - rowsA) : 0;
        const uint32_t slotB = (q + 1) % ring.nslot;
        if (pair) mbar_wait(&ring.full[slotB], ((q + 1) / ring.nslot) & 1);
        const uint2* baseA = reinterpret_cast<const uint2*>(ring.slots + (size_t)slotA * SLOT_BYTES);
        const uint2* baseB = reinterpret_cast<const uint2*>(ring.slots + (size_t)slotB * SLOT_BYTES);
        const int R = rowsA + rowsB;
        for (int i0 = 4 * warp; i0 < R; i0 += 4 * NCONS_WARPS, ++t) {
            const int nv = min(4, R - i0);
            const uint2* rp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int ri = i0 + (i < nv ? i : 0);
                rp[i] = ri < rowsA ? baseA + (size_t)ri * NU : baseB + (size_t)(ri - rowsA) * NU;
            }
            const float g = row_dot4_q<K>(rp[0], rp[1], rp[2], rp[3], xr, lane);
            const int src = (lane & 24) | (t & 7);
            const float sr = __shfl_sync(0xffffffffu, win.x, src), cr = __shfl_sync(0xffffffffu, win.y, src);
            if ((t & 7) == 7) { win = nxt; nxt = fetch(t + 9 + (lane & 7)); }
            const float a = g * sr;
            const float b = __fadd_ru(__fmul_ru(nx, cr), 0x1p-100f);   // + a floor for results flushed to zero
            const float lo = __fsub_rd(a, b), hi = __fadd_ru(a, b);
            const bool mine = (lane & 7) == 0 && j < nv;
            const bool finite = fabsf(lo) <= FLT_MAX && fabsf(hi) <= FLT_MAX;
            if (mine && !finite) st[2] = 1;
            int tw = mine && finite ? f32_ord(lo) : INT_MIN;
            tw = max(tw, __shfl_xor_sync(0xffffffffu, tw, 8));
            tw = max(tw, __shfl_xor_sync(0xffffffffu, tw, 16));
            int T = 0;
            if (lane == 0) T = max(atomicMax(st, tw), tw);
            T = __shfl_sync(0xffffffffu, T, 0);
            if (mine && finite && f32_ord(hi) >= T) {
                const int k = atomicAdd(st + 1, 1);
                if (k < HQ_CAP) cl[k] = make_int2(r + i0 + j, f32_ord(hi));
            }
        }
        __syncwarp();
        if (lane == 0) { mbar_arrive(&ring.empty[slotA]); if (pair) mbar_arrive(&ring.empty[slotB]); }
        r += R; q += pair ? 2 : 1;
    }
    cons_sync();
    const int T = st[0], n = st[1];
    const bool full = n > HQ_CAP || st[2] != 0;
    const int cnt = full ? s.r1 - s.r0 : n;
    int done = 0;
    for (int k = warp; k < cnt; k += NCONS_WARPS) {
        int row = s.r0 + k;
        if (!full) { const int2 e = cl[k]; if (e.y < T) continue; row = e.x; }
        const float v = row_dot<K>(reinterpret_cast<const uint4*>(s.W + (size_t)row * K), xr, lane);
        if (v > best_v || (v == best_v && row < best_i)) { best_v = v; best_i = row; }
        ++done;
    }
    if (lane == 0) atomicAdd(st + 3, done);
}

// transposed warp reduction of 8 per-lane partials: returns, in every lane, the warp total of value index (lane >> 2)
__device__ __forceinline__ float warp_reduce8(const float (&a)[8], int lane) {
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
    float k[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) k[i] = (h16 ? a[4 + i] : a[i]) + __shfl_xor_sync(0xffffffffu, h16 ? a[i] : a[4 + i], 16);
    float m0 = (h8 ? k[2] : k[0]) + __shfl_xor_sync(0xffffffffu, h8 ? k[0] : k[2], 8);
    float m1 = (h8 ? k[3] : k[1]) + __shfl_xor_sync(0xffffffffu, h8 ? k[1] : k[3], 8);
    float v = (h4 ? m1 : m0) + __shfl_xor_sync(0xffffffffu, h4 ? m0 : m1, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

enum { ME_STORE = 0, ME_SWIGLU = 1, ME_ARGMAX = 2 };

// Residual GEMVs (o_proj, down_proj: a handful of rows per CTA, long K): all 8 warps split K of EVERY row instead of one
// warp per row.  A thread owns the 16-byte weight groups tid, tid + 256, ... of each row (its 8 activations per group come
// straight from xs), keeps one partial per row (8 independent FMA chains), the warp reduces its 8 partials with one
// transposed reduction (9 shuffles), the 8 warp partials of a row are summed in a fixed order by one thread, which applies
// the residual and publishes to `out`.  Rows are taken 8 at a time; a group spans two ring slots when a slot holds fewer
// than 8.
// (The one-warp-per-row form left 1 of 8 warps idle and paid the load -> unpack -> FMA -> 5-shuffle latency chain once per
// row with nothing to overlap it.  Feeding each thread's activations straight from the exchange words into registers,
// without the copy into xs and its barrier, measured 4.5 % slower per step on the H100: see DESIGN.md section 4.1.)
template <int K>
__device__ __forceinline__ void consume_ksplit(const Slice& s, const Ring& ring, uint32_t& q, const float* xs, uint32_t* out,
                                               float* xres, float* part) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NU = K / 8;                                  // 16-byte groups per row
    constexpr int J = (NU + NCONS - 1) / NCONS;
    uint32_t grp = 0;
    for (int r = s.r0; r < s.r1;) {
        const int rowsA = min(s.rpc, s.r1 - r);
        const uint32_t slotA = q % ring.nslot;
        mbar_wait(&ring.full[slotA], (q / ring.nslot) & 1);
        const bool pair = s.rpc < 8 && r + rowsA < s.r1;
        const int rowsB = pair ? min(s.rpc, s.r1 - r - rowsA) : 0;
        const uint32_t slotB = (q + 1) % ring.nslot;
        if (pair) mbar_wait(&ring.full[slotB], ((q + 1) / ring.nslot) & 1);
        const uint4* baseA = reinterpret_cast<const uint4*>(ring.slots + (size_t)slotA * SLOT_BYTES);
        const uint4* baseB = reinterpret_cast<const uint4*>(ring.slots + (size_t)slotB * SLOT_BYTES);
        const int R = rowsA + rowsB;
        for (int g0 = 0; g0 < R; g0 += 8, ++grp) {
            const int ng = min(8, R - g0);
            const uint4* rp[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int ri = g0 + (i < ng ? i : 0);              // rows past the group re-read row 0 (result unused)
                rp[i] = ri < rowsA ? baseA + (size_t)ri * NU : baseB + (size_t)(ri - rowsA) * NU;
            }
            float acc[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
            for (int j = 0; j < J; ++j) {
                const int idx = tid + j * NCONS;
                if (idx < NU) {
                    const int sw = ((idx >> 2) & 1) * 4;            // xs_swz of the two 16-byte activation groups
                    const float4 xa = *reinterpret_cast<const float4*>(xs + idx * 8 + sw);
                    const float4 xb = *reinterpret_cast<const float4*>(xs + idx * 8 + 4 - sw);
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const uint4 w = rp[i][idx];
                        float t = acc[i];
                        t = fmaf(bf16_lo(w.x), xa.x, t); t = fmaf(bf16_hi(w.x), xa.y, t);
                        t = fmaf(bf16_lo(w.y), xa.z, t); t = fmaf(bf16_hi(w.y), xa.w, t);
                        t = fmaf(bf16_lo(w.z), xb.x, t); t = fmaf(bf16_hi(w.z), xb.y, t);
                        t = fmaf(bf16_lo(w.w), xb.z, t); t = fmaf(bf16_hi(w.w), xb.w, t);
                        acc[i] = t;
                    }
                }
            }
            const float v = warp_reduce8(acc, lane);
            if (g0 + 8 >= R) {                                      // last group of these slots: every weight has been consumed
                __syncwarp();
                if (lane == 0) { mbar_arrive(&ring.empty[slotA]); if (pair) mbar_arrive(&ring.empty[slotB]); }
            }
            float* pb = part + (grp & 1) * 64;
            if ((lane & 3) == 0) pb[warp * 8 + (lane >> 2)] = v;
            cons_sync();                                            // (also: every read of xs by this group is done)
            if (tid < ng) {
                float t = pb[tid];
#pragma unroll
                for (int w8 = 1; w8 < NCONS_WARPS; ++w8) t += pb[w8 * 8 + tid];
                const int row = r + g0 + tid;
                const float nv = xres[row - s.r0] + t; xres[row - s.r0] = nv;
                sx_store(out + row, nv);
            }
        }
        r += R; q += pair ? 2 : 1;
    }
}

// K <= 1024 GEMVs (qkv, gate/up, lm_head of the 0.6B dims): four rows per warp and turn, two ring slots (32 rows) per turn.
template <int K, int EPI, bool LOGPROB, bool TOPK, bool SAMPLE, bool REP>
__device__ __forceinline__ void consume_quad(const Slice& s, const Ring& ring, uint32_t& q, const float* xs, uint2* out,
                                             uint32_t tag, uint32_t* sxo, float& best_v, int& best_i, float& best_s,
                                             const float* norm_w, float norm_r, long long* fine, TopK* tk,
                                             const Draw* dr, float* smx, float* ssel, const RepBits* rb) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int fi = 0;
#define CF() do { if (fine && threadIdx.x == 0 && fi < 24) fine[fi++] = clock64(); } while (0)
    CF();
    constexpr int NU = K / 8;
    float xr[K / 32];
    if (norm_w) load_xr_norm<K>(xs, norm_w, norm_r, xr, lane);
    else load_xr<K>(xs, xr, lane);
    cons_sync();                                   // every warp holds its copy: xs may be overwritten from here on
    CF();
    const int j = lane >> 3;                       // row of the quad whose total this lane holds after row_dot4
    for (int r = s.r0; r < s.r1;) {
        const int rowsA = min(s.rpc, s.r1 - r);
        const uint32_t slotA = q % ring.nslot;
        mbar_wait(&ring.full[slotA], (q / ring.nslot) & 1);
        const bool pair = s.rpc < 32 && r + rowsA < s.r1;
        const int rowsB = pair ? min(s.rpc, s.r1 - r - rowsA) : 0;
        const uint32_t slotB = (q + 1) % ring.nslot;
        if (pair) mbar_wait(&ring.full[slotB], ((q + 1) / ring.nslot) & 1);
        CF();
        const uint4* baseA = reinterpret_cast<const uint4*>(ring.slots + (size_t)slotA * SLOT_BYTES);
        const uint4* baseB = reinterpret_cast<const uint4*>(ring.slots + (size_t)slotB * SLOT_BYTES);
        const int R = rowsA + rowsB;
        for (int i0 = 4 * warp; i0 < R; i0 += 4 * NCONS_WARPS) {
            const int nv = min(4, R - i0);
            const uint4* rp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int ri = i0 + (i < nv ? i : 0);
                rp[i] = ri < rowsA ? baseA + (size_t)ri * NU : baseB + (size_t)(ri - rowsA) * NU;
            }
            float v = row_dot4<K>(rp[0], rp[1], rp[2], rp[3], xr, lane);
            const int row = r + i0 + j;
            if (EPI == ME_SWIGLU) {                // rows (gate, up, gate, up): lanes 0 / 16 hold a gate, lanes 8 / 24 its up row
                const float up = __shfl_xor_sync(0xffffffffu, v, 8);
                if ((lane & 15) == 0 && j < nv) sx_store(sxo + (row >> 1), silu(v) * up);
            } else if (EPI == ME_STORE) {
                if ((lane & 7) == 0 && j < nv) ll_store(out + row, v, tag);
            } else if constexpr (SAMPLE) {         // ME_ARGMAX over the sampling keys (+ the raw record with LOGPROB)
                if ((lane & 7) == 0 && j < nv && rep_keep<REP>(rb, row, v))
                    sample_fold<LOGPROB>(*dr, v, row, best_v, best_i, best_s, *smx, *ssel);
            } else if constexpr (LOGPROB) {        // ME_ARGMAX + running sum of exponentials (the lanes that keep best_v)
                if ((lane & 7) == 0 && j < nv && rep_keep<REP>(rb, row, v)) {
                    lse_fold(v, row, best_v, best_i, best_s);
                    if constexpr (TOPK) tk_insert(*tk, v, row);           // TOPK: + the lane's best TK_MAX rows
                }
            } else {                               // ME_ARGMAX: rows arrive in increasing order per lane, strict > keeps the first maximum
                if ((lane & 7) == 0 && j < nv && rep_keep<REP>(rb, row, v) && v > best_v) { best_v = v; best_i = row; }
            }
        }
        CF();
        __syncwarp();
        if (lane == 0) { mbar_arrive(&ring.empty[slotA]); if (pair) mbar_arrive(&ring.empty[slotB]); }
        r += R; q += pair ? 2 : 1;
    }
    CF();
#undef CF
}

// consumer: process all chunks of a slice.  `xs` holds the (already normalised) activation vector.
// Results are published as tagged words to `out` (ME_STORE), as self-validating words to `sxo` (ME_SWIGLU), or folded
// into the running argmax (ME_ARGMAX; with LOGPROB also into the running sum of exponentials `best_s`, with TOPK also
// into the sorted candidate list `*tk`; with SAMPLE the argmax is over the sampling keys of the draw `*dr`, and LOGPROB
// keeps the raw (max `*smx`, sum `best_s`) record and the raw logit `*ssel` of the best-key row; with REP every logit is
// first replaced by its processed value under the bit arrays `*rb`, common.cuh).
template <int K, int EPI, bool LOGPROB = false, bool TOPK = false, bool SAMPLE = false, bool REP = false>
__device__ __forceinline__ void consume(const Slice& s, const Ring& ring, uint32_t& q, const float* xs, uint2* out,
                                        uint32_t tag, uint32_t* sxo, float& best_v, int& best_i, float& best_s,
                                        const float* norm_w = nullptr, float norm_r = 1.f, long long* fine = nullptr,
                                        TopK* tk = nullptr, const Draw* dr = nullptr, float* smx = nullptr, float* ssel = nullptr,
                                        const RepBits* rb = nullptr) {
    if constexpr (K <= 1024) {
        consume_quad<K, EPI, LOGPROB, TOPK, SAMPLE, REP>(s, ring, q, xs, out, tag, sxo, best_v, best_i, best_s, norm_w, norm_r, fine, tk,
                                                         dr, smx, ssel, rb);
        return;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int fi = 0;
#define CF() do { if (fine && threadIdx.x == 0 && fi < 24) fine[fi++] = clock64(); } while (0)
    CF();
    constexpr int RSTEP = (EPI == ME_SWIGLU) ? 2 : 1;
    constexpr bool XREG = K <= 2048;               // long-K slices (down_proj, 7 rows per CTA) read x from smem instead
    constexpr bool DUAL = XREG && K <= 1024;       // two rows per warp and turn: a 16-row slot is one pass of the 8 warps
    constexpr int KX = XREG ? K : 256;             // dummy instantiation size when x stays in smem
    constexpr int UPW = (DUAL && EPI != ME_SWIGLU) ? 2 : 1;       // units (rows or pairs) a warp takes per turn
    const int sub = lane >> 4;
    float xr[XREG ? K / 32 : 1];
    if (XREG) {
        if (norm_w) load_xr_norm<KX>(xs, norm_w, norm_r, reinterpret_cast<float (&)[KX / 32]>(xr), lane);
        else load_xr<KX>(xs, reinterpret_cast<float (&)[KX / 32]>(xr), lane);
        cons_sync();                               // every warp holds its copy: xs may be overwritten from here on
    }
    CF();
    int unit = 0;                                  // unit index within this CTA's slice (kept a multiple of UPW per slot)
    for (int r = s.r0; r < s.r1; r += s.rpc, ++q) {
        const int rows = min(s.rpc, s.r1 - r);
        const uint32_t slot = q % ring.nslot, par = (q / ring.nslot) & 1;
        mbar_wait(&ring.full[slot], par);
        CF();
        const uint4* base = reinterpret_cast<const uint4*>(ring.slots + (size_t)slot * SLOT_BYTES);
        const int units_here = rows / RSTEP;
        // units are dealt round-robin to warps across the whole slice (UPW consecutive units per warp and turn)
        const int first = (warp - ((unit / UPW) % NCONS_WARPS) + NCONS_WARPS) % NCONS_WARPS;
        for (int ub = first * UPW; ub < units_here; ub += NCONS_WARPS * UPW) {
            if (EPI == ME_SWIGLU) {
                const int row = r + ub * 2;        // gate row; up row = row + 1
                float v0, v1;
                if (DUAL) {
                    const float v = row_dot2<KX>(base + (size_t)(ub * 2) * (K / 8), base + (size_t)(ub * 2 + 1) * (K / 8),
                                                 reinterpret_cast<const float (&)[KX / 32]>(xr), lane);
                    v0 = v; v1 = __shfl_xor_sync(0xffffffffu, v, 16);      // valid on the lower half (lane 0 publishes)
                } else if (XREG) {
                    v0 = row_dot<KX>(base + (size_t)(ub * 2) * (K / 8), reinterpret_cast<const float (&)[KX / 32]>(xr), lane);
                    v1 = row_dot<KX>(base + (size_t)(ub * 2 + 1) * (K / 8), reinterpret_cast<const float (&)[KX / 32]>(xr), lane);
                } else {
                    v0 = row_dot_smem<K>(base + (size_t)(ub * 2) * (K / 8), xs, lane);
                    v1 = row_dot_smem<K>(base + (size_t)(ub * 2 + 1) * (K / 8), xs, lane);
                }
                if (lane == 0) sx_store(sxo + (row >> 1), silu(v0) * v1);
            } else {
                bool act; int row; float v0;
                if (DUAL) {
                    const bool two = ub + 1 < units_here;                 // the slot's last turn may hold a single row
                    v0 = row_dot2<KX>(base + (size_t)ub * (K / 8), base + (size_t)(two ? ub + 1 : ub) * (K / 8),
                                      reinterpret_cast<const float (&)[KX / 32]>(xr), lane);
                    act = ((lane & 15) == 0) && (sub == 0 || two);
                    row = r + ub + sub;
                } else {
                    if (XREG) v0 = row_dot<KX>(base + (size_t)ub * (K / 8), reinterpret_cast<const float (&)[KX / 32]>(xr), lane);
                    else v0 = row_dot_smem<K>(base + (size_t)ub * (K / 8), xs, lane);
                    act = lane == 0; row = r + ub;
                }
                if (EPI == ME_STORE) {
                    if (act) ll_store(out + row, v0, tag);
                } else if constexpr (SAMPLE) {
                    if (act && rep_keep<REP>(rb, row, v0)) sample_fold<LOGPROB>(*dr, v0, row, best_v, best_i, best_s, *smx, *ssel);
                } else if constexpr (LOGPROB) {
                    if (act && rep_keep<REP>(rb, row, v0)) {
                        lse_fold(v0, row, best_v, best_i, best_s);
                        if constexpr (TOPK) tk_insert(*tk, v0, row);
                    }
                } else {
                    if (act && rep_keep<REP>(rb, row, v0) && v0 > best_v) { best_v = v0; best_i = row; }
                }
            }
        }
        unit += (units_here + UPW - 1) / UPW * UPW;
        CF();
        __syncwarp();
        if (lane == 0) mbar_arrive(&ring.empty[slot]);
    }
    CF();
#undef CF
    if (!XREG) cons_sync();                        // xs was read in place: nobody may overwrite it before this point
}

// all consumer threads: gather the N self-validating words at `src` into xs (xs_swz layout) and return this thread's sum of
// squares of elements 2i, 2i + 1 for i = tid, tid + NCONS, ... in that order (the partial sums norm_scale reduces).
// Warp w polls exactly the quads that hold its threads' pairs -- quads 16 w + (0..15) + NCONS / 2 * u, lane taking
// u = 2 k + (lane >> 4) -- so the squares are read back from xs after a __syncwarp, without a CTA barrier.
template <int N>
__device__ __forceinline__ float sx_gather(const uint32_t* src, float* xs) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NQ = N / 4;
    constexpr int KQ = (NQ + NCONS - 1) / NCONS;              // quads per thread
    int qi[KQ];
    uint4 v[KQ];
#pragma unroll
    for (int k = 0; k < KQ; ++k) {
        qi[k] = 16 * warp + (lane & 15) + (NCONS / 2) * (2 * k + (lane >> 4));
        v[k] = make_uint4(SX_EMPTY, SX_EMPTY, SX_EMPTY, SX_EMPTY);
    }
    bool ok;
    do {                                                       // only the quads still missing are re-read
        ok = true;
#pragma unroll
        for (int k = 0; k < KQ; ++k)
            if (qi[k] < NQ && !sx_ready(v[k])) v[k] = sx_load4(src + 4 * qi[k]);
#pragma unroll
        for (int k = 0; k < KQ; ++k)
            if (qi[k] < NQ) ok = ok && sx_ready(v[k]);
    } while (!ok);
#pragma unroll
    for (int k = 0; k < KQ; ++k)
        if (qi[k] < NQ) *reinterpret_cast<uint4*>(xs + xs_swz(4 * qi[k])) = v[k];
    __syncwarp();
    float ss = 0.f;
#pragma unroll
    for (int i = tid; i < N / 2; i += NCONS) {
        const float2 x = *reinterpret_cast<const float2*>(xs + xs_swz(2 * i));
        ss = fmaf(x.x, x.x, ss); ss = fmaf(x.y, x.y, ss);
    }
    return ss;
}

// all consumer threads: copy the N self-validating words at `src` into xs (xs_swz layout), the input of o_proj / down_proj.
// A thread spins on one quad at a time: a single load in flight per thread while the words are not yet published keeps
// the polling traffic of 132 CTAs low (measured faster than re-polling all of a thread's missing quads per round).
template <int N>
__device__ __forceinline__ void sx_copy(const uint32_t* src, float* xs) {
    for (int j = threadIdx.x; j < N / 4; j += NCONS) {
        uint4 v;
        do { v = sx_load4(src + 4 * j); } while (!sx_ready(v));
        *reinterpret_cast<uint4*>(xs + xs_swz(4 * j)) = v;
    }
}

// RMSNorm scale of the vector sitting in xs from the per-thread partial sums of squares; the scaling itself is
// fused into the register load of the GEMV (load_xr_norm).  Ends with a barrier: xs is complete for every warp.
__device__ __forceinline__ float norm_scale(float ss, int n, float eps, float* red) {
    const int tid = threadIdx.x;
    ss = warp_sum(ss);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    cons_sync();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < NCONS_WARPS; ++i) tot += red[i];
    return 1.0f / sqrtf(tot / n + eps);
}

// per-head RMSNorm + RoPE of one 128-vector by one warp (lane holds d = lane, +32, +64, +96);
// input = tagged words
__device__ __forceinline__ void head_norm_rope(const uint2* __restrict__ src, uint32_t tag, const float* __restrict__ nw,
                                               float eps, const float* __restrict__ cs, const float* __restrict__ sn,
                                               float* dst, int lane) {
    float v[4];
    ll_poll4(src + lane, 32, tag, v);
    float ss = warp_sum(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
    const float r = 1.0f / sqrtf(ss / 128.f + eps);
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = (v[i] * r) * nw[lane + 32 * i];
    // pairs (d, d+64): (lane, lane+64) and (lane+32, lane+96)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int d = lane + 32 * i;
        const float c = cs[d], s = sn[d];
        const float a = v[i], b = v[i + 2];
        dst[d] = a * c - b * s;
        dst[d + 64] = b * c + a * s;
    }
}

#define MEGA_FINE(k)                                                                                    \
    do {                                                                                               \
        if (dbg_row && tid == 0 && l == 5) dbg_row[400 + (k)] = clock64();                              \
    } while (0)
// every CTA: wall-clock (globaltimer, ns) of three events of layer 5 -> row 0, slots [512 + 3 * cta ...)
#define MEGA_GT(k)                                                                                     \
    do {                                                                                               \
        if (p.dbg && tid == 0 && l == 5) {                                                             \
            unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));               \
            p.dbg[512 + 3 * blockIdx.x + (k)] = (long long)t_;                                         \
        }                                                                                              \
    } while (0)
#define MEGA_MARK()                                                                                    \
    do {                                                                                               \
        if (dbg_row && tid == 0 && dbg_i < DBG_SLOTS) dbg_row[dbg_i++] = clock64();                    \
    } while (0)

// LOGPROB: the lm_head also keeps (max, sum of exponentials) per lane, and the last CTA records the log-probability of
// the selected token (p.lp_out / p.eos_lp)
// TOPK (with LOGPROB): each folding lane also keeps its best TK_MAX (logit, id) pairs; they are merged across lanes,
// warps and CTAs, and the last CTA records the step's candidates (p.tk_ids / p.tk_lp, or the EOS row)
// SAMPLE: the lm_head folds the sampling keys of draw (p.row, n = *p.n_out) instead of the logits (common.cuh); with
// LOGPROB the lanes, warps and CTAs also carry the raw (max, sum) record and the raw logit of the best-key row
// REP: every lm_head logit is replaced by its processed value (repetition controls, common.cuh) before any fold
template <int H, int QD, int I, int NS, bool LOGPROB, bool TOPK = false, bool SAMPLE = false, bool REP = false>
__global__ void __launch_bounds__(NTHREADS, 1) decode_step_kernel(const Params p) {
    constexpr int XS_FLOATS = (I > XS_MIN ? I : XS_MIN) + 64;
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int PARAM_FLOATS = 2 * H + 2 * HD;      // per-layer small vectors: ln_in[H], ln_post[H], q_norm[128], k_norm[128]
    Ring ring;
    ring.slots = smem;
    ring.nslot = NS;
    float* xs = reinterpret_cast<float*>(smem + (size_t)NS * SLOT_BYTES);
    float* xres = xs + XS_FLOATS;                                      // [XRES_MAX] residual rows owned by this CTA
    float* pbuf = xres + XRES_MAX;                                     // [2][PARAM_FLOATS] per-layer small vectors (double buffer)
    float* ropes = pbuf + 2 * PARAM_FLOATS;                            // [128] cos | sin of this step's position
    DecLayerW* ltab = reinterpret_cast<DecLayerW*>(ropes + 128);       // [MAX_LAYERS]
    uint64_t* bars = reinterpret_cast<uint64_t*>(ltab + MAX_LAYERS);
    ring.full = bars; ring.empty = bars + NSLOT_MAX;
    uint64_t* p_full = bars + 2 * NSLOT_MAX; uint64_t* p_empty = p_full + 2;   // [2] each
    float* red = reinterpret_cast<float*>(bars + 2 * NSLOT_MAX + 4);      // [64]
    int* ired = reinterpret_cast<int*>(red + 64);                      // [64]
    float* part = reinterpret_cast<float*>(ired + 64);                 // [2][8 warps][8 rows] K-split partials (consume_ksplit)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool is_producer = warp == NCONS_WARPS;
    constexpr bool HEADQ = !LOGPROB && !TOPK && !SAMPLE && !REP;   // greedy: the lm_head streams from its int8 copy

    if (__ldcg(p.done) != 0) return;            // sequence finished: nothing to do this step

    if (tid == 0) {
        for (int i = 0; i < NS; ++i) { mbar_init(&ring.full[i], 1); mbar_init(&ring.empty[i], NCONS_WARPS); }
        for (int i = 0; i < 2; ++i) { mbar_init(&p_full[i], 1); mbar_init(&p_empty[i], NCONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // Small read-only tables go to shared memory: with 1.2 GB streaming through L2 every step they are never
    // L2-resident, and a dependent DRAM round trip (~1-2 us) per use is what the phases cannot afford.
    const int pos = __ldcg(p.pos);
    {
        const uint2* src = reinterpret_cast<const uint2*>(p.layers);
        uint2* dst = reinterpret_cast<uint2*>(ltab);
        for (int i = tid; i < p.L * (int)(sizeof(DecLayerW) / 8); i += NTHREADS) dst[i] = src[i];
        if (tid < 64) ropes[tid] = p.rope_cos[(size_t)pos * 64 + tid];
        else if (tid < 128) ropes[tid] = p.rope_sin[(size_t)pos * 64 + tid - 64];
    }
    __syncthreads();

    // attention work item of this CTA: (kv head att_g, keys [att_j0, att_j0 + KV_KEYS)); keys < pos are
    // already in the cache (n_old of them fall in this split), key `pos` is produced in this step.
    const bool att_cta = (int)blockIdx.x < p.nkv * p.nsplit;
    const int att_g = blockIdx.x / p.nsplit, att_sp = blockIdx.x % p.nsplit, att_j0 = att_sp * KV_KEYS;
    const int n_old = att_cta ? max(0, min(pos - att_j0, KV_KEYS)) : 0;
    const bool merger = att_cta && att_sp == 0;     // merges the attention partials of kv head att_g and publishes its outputs
    // residual rows owned by this CTA (same row partition for o_proj and down_proj), and its gate/up units
    const Slice xsl = make_slice(nullptr, H, QD, 1), sl_gu = make_slice(nullptr, 2 * I, H, 2);

    // self-validating words of this launch: set = parity of bar[3], the count of executed launches of THIS kernel (the
    // launch epoch bar[1] also advances on batched steps, which would break the strict alternation the re-arm relies on)
    constexpr size_t SXL = 2 * H + QD + I;          // words per (set, layer): x_o | x_d | attn | act
    const unsigned sstep = __ldcg(p.bar + 3);
    uint32_t* const sx_cur = p.sx + (size_t)(sstep & 1u) * p.L * SXL;
    // Re-arm of layer l of the other set (consumer threads): exactly the words this CTA publishes, from the slices and head
    // mapping its publishing code uses -- its residual rows of x_o and x_d (consume_ksplit over sl_o / sl_dn, the rows of
    // xsl), the act rows of its gate/up units, and as merging CTA the group x 128 attention outputs of its kv head.  Every
    // word of a set is published in every executed step (pos >= 1, so split 0 of every kv head always merges), so the
    // re-arms of all CTAs cover the whole set.
    auto rearm = [&](int l) __attribute__((always_inline)) {
        uint32_t* const base = p.sx + (size_t)((sstep & 1u) ^ 1u) * p.L * SXL + (size_t)l * SXL;
        const int xrows = xsl.r1 - xsl.r0, a0 = sl_gu.r0 / 2, arows = sl_gu.r1 / 2 - a0;
        const int nattn = merger ? p.group * HD : 0;
        for (int i = tid; i < xrows; i += NCONS) { base[xsl.r0 + i] = SX_EMPTY; base[H + xsl.r0 + i] = SX_EMPTY; }
        for (int i = tid; i < nattn; i += NCONS) base[2 * H + att_g * p.group * HD + i] = SX_EMPTY;
        for (int i = tid; i < arows; i += NCONS) base[2 * H + QD + a0 + i] = SX_EMPTY;
    };
    uint32_t q = 0;
    if (is_producer) {
        // ONE stream in consumption order through ONE ring: per layer the [q|k|v] rows, this CTA's K tile and V tile of
        // the earlier positions (one slot each, when its split holds any), the o_proj, gate/up and down_proj rows; then the
        // lm_head.  The copies carry an L2 evict_first hint: every line is read once per step.  (Prefetching further ahead
        // into L2 measured slower on the H100 at any distance: see DESIGN.md section 4.1.)
        if (lane == 0) {
            const uint64_t pol = l2_evict_first_policy();
            auto issue = [&](const void* src, uint32_t bytes) __attribute__((always_inline)) {
                const uint32_t slot = q % NS, par = (q / NS) & 1;
                mbar_wait(&ring.empty[slot], par ^ 1);
                mbar_expect_tx(&ring.full[slot], bytes);
                bulk_g2s_hint(ring.slots + (size_t)slot * SLOT_BYTES, src, bytes, &ring.full[slot], pol);
                ++q;
            };
            auto issue_slice = [&](const Slice& s) __attribute__((always_inline)) {
                for (int r = s.r0; r < s.r1; r += s.rpc) issue(s.W + (size_t)r * s.K, (uint32_t)min(s.rpc, s.r1 - r) * s.K * 2);
            };
            const size_t kv_row = ((size_t)att_g * p.max_ctx + att_j0) * HD;
            for (int l = 0; l <= p.L; ++l) {
                {   // small per-layer vectors -> pbuf[l & 1] (layer L = final norm only)
                    float* pb = pbuf + (l & 1) * PARAM_FLOATS;
                    mbar_wait(&p_empty[l & 1], ((l >> 1) & 1) ^ 1);
                    if (l < p.L) {
                        const DecLayerW w = ltab[l];
                        mbar_expect_tx(&p_full[l & 1], (uint32_t)(2 * H + 2 * HD) * 4);
                        bulk_g2s(pb, w.ln_in, H * 4, &p_full[l & 1]);
                        bulk_g2s(pb + H, w.ln_post, H * 4, &p_full[l & 1]);
                        bulk_g2s(pb + 2 * H, w.qnorm, HD * 4, &p_full[l & 1]);
                        bulk_g2s(pb + 2 * H + HD, w.knorm, HD * 4, &p_full[l & 1]);
                    } else {
                        mbar_expect_tx(&p_full[l & 1], (uint32_t)H * 4);
                        bulk_g2s(pb, p.final_norm, H * 4, &p_full[l & 1]);
                        break;
                    }
                }
                const DecLayerW w = ltab[l];
                issue_slice(make_slice(w.wqkv, QD + 2 * p.KVD, H, 1));
                if (n_old > 0) {
                    const size_t off = (size_t)l * p.cache_layer_stride + kv_row;
                    issue(p.kcache + off, (uint32_t)n_old * HD * 4);
                    issue(p.vcache + off, (uint32_t)n_old * HD * 4);
                }
                issue_slice(make_slice(w.wo, H, QD, 1));
                issue_slice(make_slice(w.wgu, 2 * I, H, 2));
                issue_slice(make_slice(w.wdown, H, I, 1));
            }
            if constexpr (HEADQ) {
                const Slice sl = make_slice(nullptr, p.V, H, 1);
                constexpr int RQ = SLOT_BYTES / H;
                for (int r = sl.r0; r < sl.r1; r += RQ) issue(p.lm_head_q + (size_t)r * H, (uint32_t)min(RQ, sl.r1 - r) * H);
            } else {
                issue_slice(make_slice(p.lm_head, p.V, H, 1));
            }
        }
        return;
    }

    // ------------------------------ consumers ------------------------------
    long long* dbg_row = nullptr; int dbg_i = 0;
    if (p.dbg && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) dbg_row = p.dbg + (blockIdx.x == 0 ? 0 : DBG_SLOTS);
    MEGA_MARK();
    const int half = HD / 2;
    const float* cs = ropes;
    const float* sn = ropes + half;
    const unsigned G = gridDim.x;
    RepBits rb{};                                     // REP: this CTA's bits of its lm_head rows, built while layer 0's
    if constexpr (REP) {                              // weights stream in (n_out changes only after every CTA's ticket)
        const Slice sl = make_slice(nullptr, p.V, H, 1);
        uint32_t* hist = p.rep_bits + (size_t)blockIdx.x * 2 * p.rep_words;
        for (int i = tid; i < 2 * p.rep_words; i += NCONS) hist[i] = 0u;
        cons_sync();
        rep_mark(p.ids_out, min(__ldcg(p.n_out), p.max_new), __ldg(&p.rep->ngram), sl.r0, sl.r1, hist, hist + p.rep_words, tid, NCONS);
        rb = RepBits{hist, hist + p.rep_words, sl.r0 >> 5, __ldg(&p.rep->theta)};
    }
    float best_v = -INFINITY; int best_i = 0x7fffffff;
    float best_s = 0.f;                               // LOGPROB: sum of exp(logit - best_v) over the rows this lane folded
    static_assert(!TOPK || LOGPROB, "the candidates' log-probabilities need the sum of exponentials");
    TopK tk;                                          // TOPK: this lane's best rows
    if constexpr (TOPK) tk_init(tk);
    // tag = launch epoch (unique per executed step, survives new utterances that revisit the same positions)
    const unsigned epoch = __ldcg(p.bar + 1);
    const uint32_t tag_base = (epoch & 0xffffffu) << 8;
    // slice geometry does not depend on the layer: computed once, only the weight pointer changes
    Slice sl_qkv = make_slice(nullptr, QD + 2 * p.KVD, H, 1), sl_o = make_slice(nullptr, H, QD, 1), sl_dn = make_slice(nullptr, H, I, 1);
    for (int i = tid; i < xsl.r1 - xsl.r0; i += NCONS) xres[i] = __ldcg(p.x + xsl.r0 + i);
    for (int l = 0; l < p.L; ++l) rearm(l);

    for (int l = 0; l < p.L; ++l) {
        const DecLayerW w = ltab[l];
        const uint32_t tl = tag_base | ((uint32_t)l << 3);
        const float* pb = pbuf + (l & 1) * PARAM_FLOATS;               // ln_in | ln_post | q_norm | k_norm of this layer
        uint32_t* const sx_xo = sx_cur + (size_t)l * SXL;
        uint32_t* const sx_xd = sx_xo + H;
        uint32_t* const sx_attn = sx_xo + 2 * H;
        uint32_t* const sx_act = sx_xo + 2 * H + QD;
        mbar_wait(&p_full[l & 1], (l >> 1) & 1);
        // ---- phase 1: RMSNorm + [q|k|v] GEMV ----
        float nr;
        {
            float ss = 0.f;
            if (l == 0) { for (int i = tid; i < H; i += NCONS) { const float v = __ldcg(p.x + i); xs[xs_swz(i)] = v; ss = fmaf(v, v, ss); } }
            else { MEGA_FINE(0); MEGA_FINE(1); ss = sx_gather<H>(sx_xd - SXL, xs); MEGA_FINE(2); }     // x_d of layer l - 1
            nr = norm_scale(ss, H, p.eps, red);
            MEGA_FINE(3);
        }
        consume<H, ME_STORE>(sl_qkv, ring, q, xs, p.qkv_ll, tl | PH_QKV, nullptr, best_v, best_i, best_s, pb, nr);
        MEGA_FINE(4);
        MEGA_GT(0);
        MEGA_MARK();
        // ---- phase 2: attention partials, work item = (kv head, 64-key split) ----
        {
            // Splits only hold keys that were cached before this step (n_old of them, prefetched by the producer, so a
            // split depends on nothing but q); the key/value of the current token is folded in as one more partial by the
            // merging CTA (split 0 of the kv head), which also appends it to the cache.
            const int nloc = n_old;
            const int nact = min(p.nsplit, (pos + KV_KEYS - 1) / KV_KEYS);      // splits holding at least one cached key
            if (nloc > 0) {                                                     // pos >= 1: split 0 always has cached keys
                const int g = att_g;
                float* qs = xs;                       // [group][128]
                float* kn = qs + p.group * HD;        // [128]
                float* vn = kn + HD;                  // [128]
                float* sc = vn + HD;                  // [group][KV_KEYS]
                float* ml = sc + p.group * KV_KEYS;   // [group][2] (max, sum)   (generic path) / score of the new key per head
                float* osum = ml + 8;                 // [warps][2][128] per-warp partial outputs (group == 2 path)
                float* wml = osum + NCONS_WARPS * 2 * HD;   // [warps][2][2] per-warp (max, sum)
                float* snew = wml + NCONS_WARPS * 4;  // [group] score of the current token's key per head (merging CTA)
                // the producer streams this split's K tile and V tile right after the [q|k|v] rows
                const uint32_t ksl = q % ring.nslot, vsl = (q + 1) % ring.nslot;
                const float* Ks = reinterpret_cast<const float*>(ring.slots + (size_t)ksl * SLOT_BYTES);
                const float* Vs = reinterpret_cast<const float*>(ring.slots + (size_t)vsl * SLOT_BYTES);
                MEGA_FINE(24);
                cons_sync();                          // xs (phase-1 activations) no longer needed by any warp; q/k/v words are
                                                      // polled directly below (few readers per word)
                if (warp < p.group) head_norm_rope(p.qkv_ll + (size_t)(g * p.group + warp) * HD, tl | PH_QKV, pb + 2 * H, p.eps, cs, sn, qs + warp * HD, lane);
                else if (warp == p.group && merger) head_norm_rope(p.qkv_ll + QD + (size_t)g * HD, tl | PH_QKV, pb + 2 * H + HD, p.eps, cs, sn, kn, lane);
                else if (warp == p.group + 1 && merger) {
                    float vv[4];
                    ll_poll4(p.qkv_ll + QD + p.KVD + (size_t)g * HD + lane, 32, tl | PH_QKV, vv);
#pragma unroll
                    for (int i = 0; i < 4; ++i) vn[lane + 32 * i] = vv[i];
                }
                MEGA_FINE(25);
                mbar_wait(&ring.full[ksl], (q / ring.nslot) & 1);
                mbar_wait(&ring.full[vsl], ((q + 1) / ring.nslot) & 1);
                cons_sync();
                MEGA_FINE(26);
                if (merger) {
                    if (tid < HD) {                   // KV append (replaces Tensor::cat, layers.rs:311-317)
                        float* kc = p.kcache + (size_t)l * p.cache_layer_stride + ((size_t)g * p.max_ctx + pos) * HD;
                        float* vc = p.vcache + (size_t)l * p.cache_layer_stride + ((size_t)g * p.max_ctx + pos) * HD;
                        kc[tid] = kn[tid]; vc[tid] = vn[tid];
                    }
                    if (warp >= NCONS_WARPS - p.group) {   // score of the new key for head hq (last `group` warps)
                        const int hq = warp - (NCONS_WARPS - p.group);
                        const float4 a = *reinterpret_cast<const float4*>(qs + hq * HD + lane * 4);
                        const float4 b = *reinterpret_cast<const float4*>(kn + lane * 4);
                        const float sn_ = warp_sum(fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w))));
                        if (lane == 0) snew[hq] = sn_ / sqrtf((float)HD);
                    }
                }
                MEGA_FINE(27);
                if (p.group == 2) {
                    // 2 query heads per kv head: warp w owns keys w, w+8, ... of the split and computes a complete local softmax
                    // partial (max, sum, unnormalised output) for them; the 8 warp partials are merged through shared memory
                    // exactly like the per-split partials are merged later.  One barrier, no score array.
                    //  scores: every lane multiplies its 4 dims of the K row (one conflict-free LDS.128) with both q vectors held
                    //  in registers; the 16 partial sums per lane (8 keys x 2 heads) are reduced across the warp with a
                    //  transposing butterfly (16 shuffles instead of 80); lane 2 * (2 * kk + h) (and its odd twin) ends up
                    //  with the score of key kk, head h
                    const float4 q0 = *reinterpret_cast<const float4*>(qs + lane * 4);
                    const float4 q1 = *reinterpret_cast<const float4*>(qs + HD + lane * 4);
                    float pv[16];
#pragma unroll
                    for (int kk = 0; kk < 8; ++kk) {
                        const int j = warp + 8 * kk;
                        // branch-free: rows past the split's last key are read (stale data) and masked below
                        const float4 kv = *reinterpret_cast<const float4*>(Ks + j * HD + lane * 4);
                        pv[2 * kk] = fmaf(kv.x, q0.x, fmaf(kv.y, q0.y, fmaf(kv.z, q0.z, kv.w * q0.w)));
                        pv[2 * kk + 1] = fmaf(kv.x, q1.x, fmaf(kv.y, q1.y, fmaf(kv.z, q1.z, kv.w * q1.w)));
                    }
#pragma unroll
                    for (int o = 16, n = 16; n > 1; o >>= 1, n >>= 1) {
                        const bool up = lane & o;
#pragma unroll
                        for (int i = 0; i < n / 2; ++i) {
                            const float send = up ? pv[i] : pv[i + n / 2];
                            const float keep = up ? pv[i + n / 2] : pv[i];
                            pv[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                        }
                    }
                    pv[0] += __shfl_xor_sync(0xffffffffu, pv[0], 1);
                    const bool mine = warp + 8 * (lane >> 2) < nloc;               // this lane's key exists
                    const float sv = mine ? pv[0] / sqrtf((float)HD) : -INFINITY;
                    float mw = sv;                                                   // max over this warp's keys, per head (lane bit 1)
                    mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, 4));
                    mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, 8));
                    mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, 16));
                    const float ev = mine ? expf(sv - mw) : 0.f;
                    float lw = ev;
                    lw += __shfl_xor_sync(0xffffffffu, lw, 4);
                    lw += __shfl_xor_sync(0xffffffffu, lw, 8);
                    lw += __shfl_xor_sync(0xffffffffu, lw, 16);
                    // o_w[h][d] = sum_kk e[kk][h] * V[j][d]: 4 dims per lane (one LDS.128 of V per key), both heads
                    float4 o0 = make_float4(0.f, 0.f, 0.f, 0.f), o1 = o0;
#pragma unroll
                    for (int kk = 0; kk < 8; ++kk) {
                        const int j = warp + 8 * kk;
                        const float4 vv = *reinterpret_cast<const float4*>(Vs + j * HD + lane * 4);
                        const float e0 = __shfl_sync(0xffffffffu, ev, 4 * kk), e1 = __shfl_sync(0xffffffffu, ev, 4 * kk + 2);
                        if (j < nloc) {       // (a stale V row may hold non-finite garbage: 0 * inf must not reach the sum)
                            o0.x = fmaf(e0, vv.x, o0.x); o0.y = fmaf(e0, vv.y, o0.y); o0.z = fmaf(e0, vv.z, o0.z); o0.w = fmaf(e0, vv.w, o0.w);
                            o1.x = fmaf(e1, vv.x, o1.x); o1.y = fmaf(e1, vv.y, o1.y); o1.z = fmaf(e1, vv.z, o1.z); o1.w = fmaf(e1, vv.w, o1.w);
                        }
                    }
                    *reinterpret_cast<float4*>(osum + (warp * 2 + 0) * HD + lane * 4) = o0;
                    *reinterpret_cast<float4*>(osum + (warp * 2 + 1) * HD + lane * 4) = o1;
                    if (lane == 0 || lane == 2) { wml[(warp * 2 + (lane >> 1)) * 2] = mw; wml[(warp * 2 + (lane >> 1)) * 2 + 1] = lw; }
                    cons_sync();
                    MEGA_FINE(28);
                    {
                        const int hq = tid / HD, d = tid - hq * HD;      // NCONS == 2 * HD
                        float M = -INFINITY;
#pragma unroll
                        for (int w8 = 0; w8 < NCONS_WARPS; ++w8) M = fmaxf(M, wml[(w8 * 2 + hq) * 2]);
                        float acc = 0.f, Ls = 0.f;
#pragma unroll
                        for (int w8 = 0; w8 < NCONS_WARPS; ++w8) {
                            const float f = expf(wml[(w8 * 2 + hq) * 2] - M);           // exp(-inf) = 0: warps without keys
                            acc = fmaf(f, osum[(w8 * 2 + hq) * HD + d], acc);
                            Ls = fmaf(f, wml[(w8 * 2 + hq) * 2 + 1], Ls);
                        }
                        uint2* rec = p.part_ll + ((size_t)blockIdx.x * 2 + hq) * PSTRIDE;
                        ll_store(rec + d, acc, tl | PH_PART);
                        if (d < 2) ll_store(rec + HD + d, d == 0 ? M : Ls, tl | PH_PART);
                    }
                    MEGA_FINE(29);
                } else {
                    // generic group size: one thread per (head, key); the d loop is rotated by the key index so that the
                    // 32 lanes of a warp hit 32 different banks of the row-major K tile
                    for (int idx = tid; idx < p.group * KV_KEYS; idx += NCONS) {
                        const int hq = idx / KV_KEYS, j = idx - hq * KV_KEYS;
                        if (j < nloc) {
                            const float* kr = Ks + j * HD; const float* qr = qs + hq * HD;
                            float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
                            for (int dd = 0; dd < HD; dd += 2) {
                                const int d0 = (dd + j) & (HD - 1), d1 = (dd + 1 + j) & (HD - 1);
                                a0 = fmaf(kr[d0], qr[d0], a0); a1 = fmaf(kr[d1], qr[d1], a1);
                            }
                            sc[hq * KV_KEYS + j] = (a0 + a1) / sqrtf((float)HD);
                        }
                    }
                    cons_sync();
                    if (warp < p.group) {                 // softmax partial of head `warp` over this split
                        float mx = -INFINITY;
                        for (int j = lane; j < nloc; j += 32) mx = fmaxf(mx, sc[warp * KV_KEYS + j]);
                        mx = warp_max(mx);
                        float sum = 0.f;
                        for (int j = lane; j < nloc; j += 32) {
                            float e = expf(sc[warp * KV_KEYS + j] - mx);
                            sc[warp * KV_KEYS + j] = e; sum += e;
                        }
                        sum = warp_sum(sum);
                        if (lane == 0) { ml[warp * 2] = mx; ml[warp * 2 + 1] = sum; }
                    }
                    cons_sync();
                    for (int idx = tid; idx < p.group * HD; idx += NCONS) {
                        const int hq = idx / HD, d = idx - hq * HD;
                        float acc = 0.f;
                        for (int j = 0; j < nloc; ++j) acc = fmaf(sc[hq * KV_KEYS + j], Vs[j * HD + d], acc);
                        uint2* rec = p.part_ll + ((size_t)blockIdx.x * p.group + hq) * PSTRIDE;
                        ll_store(rec + d, acc, tl | PH_PART);
                        if (d < 2) ll_store(rec + HD + d, ml[hq * 2 + d], tl | PH_PART);
                    }
                }
                {                                     // hand the K / V slots back to the producer
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) { mbar_arrive(&ring.empty[ksl]); mbar_arrive(&ring.empty[vsl]); }
                    q += 2;
                }
                MEGA_FINE(30);
                MEGA_GT(1);
                // split 0 of every kv head merges the partials of all active splits and publishes the head outputs
                if (merger) {
                    for (int idx = tid; idx < p.group * HD; idx += NCONS) {
                        const int hq = idx / HD, d = idx - hq * HD;          // hq is uniform per warp (HD = 4 warps)
                        // lane s of every warp fetches (max, sum) of split s (nact <= MAX_SPLITS <= 32 lanes); all loads of a
                        // round are issued before any tag is examined (one round trip when ready)
                        const uint32_t tg = tl | PH_PART;
                        constexpr int RB = 9;                                // partial outputs fetched per round (registers)
                        uint2 mv, lv, ov[RB];
                        bool ok;
                        auto load_round = [&](int u0) {
#pragma unroll
                            for (int u = 0; u < RB; ++u) {
                                if (u0 + u < nact) {
                                    const uint2* rec = p.part_ll + ((size_t)(g * p.nsplit + u0 + u) * p.group + hq) * PSTRIDE;
                                    asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(ov[u].x), "=r"(ov[u].y) : "l"(rec + d) : "memory");
                                }
                            }
                        };
                        auto round_ok = [&](int u0) {
                            bool k = true;
#pragma unroll
                            for (int u = 0; u < RB; ++u) if (u0 + u < nact) k = k && (ov[u].y == tg);
                            return k;
                        };
                        do {        // first round: (max, sum) of every split + the first RB partial outputs, one round trip
                            mv.y = tg; lv.y = tg; mv.x = 0u; lv.x = 0u;
                            if (lane < nact) {
                                const uint2* rec = p.part_ll + ((size_t)(g * p.nsplit + lane) * p.group + hq) * PSTRIDE;
                                asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(mv.x), "=r"(mv.y) : "l"(rec + HD) : "memory");
                                asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(lv.x), "=r"(lv.y) : "l"(rec + HD + 1) : "memory");
                            }
                            load_round(0);
                            ok = __all_sync(0xffffffffu, (mv.y == tg) && (lv.y == tg) && round_ok(0));
                        } while (!ok);
                        MEGA_FINE(35);
                        // softmax merge, one partial per lane: lanes < nact hold a split, lane nact the current token's key
                        // (max = its score, sum = 1, output = its value row)
                        const float m_l = lane < nact ? __uint_as_float(mv.x) : (lane == nact ? snew[hq] : -INFINITY);
                        const float l_l = lane < nact ? __uint_as_float(lv.x) : (lane == nact ? 1.f : 0.f);
                        const float M = warp_max(m_l);
                        const float f = expf(m_l - M);                       // exp(-inf) = 0 on idle lanes
                        const float Lsum = warp_sum(f * l_l);
                        float O = __shfl_sync(0xffffffffu, f, nact) * vn[d];
                        for (int u0 = 0; u0 < nact; u0 += RB) {              // contexts beyond 9 splits: one more round trip each
                            if (u0 > 0) { do { load_round(u0); ok = __all_sync(0xffffffffu, round_ok(u0)); } while (!ok); }
#pragma unroll
                            for (int u = 0; u < RB; ++u)
                                if (u0 + u < nact) O = fmaf(__shfl_sync(0xffffffffu, f, u0 + u), __uint_as_float(ov[u].x), O);
                        }
                        sx_store(sx_attn + (size_t)(g * p.group + hq) * HD + d, O / Lsum);
                    }
                }
                MEGA_FINE(31);
                cons_sync();                          // attention scratch (aliases xs) is free again
            }
        }
        MEGA_MARK();
        // ---- phase 3: o_proj GEMV + residual ----
        MEGA_FINE(32);
        sx_copy<QD>(sx_attn, xs);
        MEGA_FINE(33);
        MEGA_GT(2);
        cons_sync();
        consume_ksplit<QD>(sl_o, ring, q, xs, sx_xo, xres, part);
        MEGA_FINE(34);
        MEGA_MARK();
        // ---- phase 4: RMSNorm + gate/up GEMV + SiLU*mul ----
        cons_sync();
        {
            MEGA_FINE(8); MEGA_FINE(9);
            const float ss = sx_gather<H>(sx_xo, xs); MEGA_FINE(10);
            nr = norm_scale(ss, H, p.eps, red); MEGA_FINE(11);
        }
        consume<H, ME_SWIGLU>(sl_gu, ring, q, xs, nullptr, 0u, sx_act, best_v, best_i, best_s, pb + H, nr, (dbg_row && l == 5) ? dbg_row + 440 : nullptr);
        MEGA_FINE(12);
        MEGA_FINE(13);
        MEGA_MARK();
        // ---- phase 5: down GEMV + residual ----
        MEGA_FINE(16); MEGA_FINE(17);
        sx_copy<I>(sx_act, xs); MEGA_FINE(18);
        cons_sync();
        consume_ksplit<I>(sl_dn, ring, q, xs, sx_xd, xres, part);
        MEGA_FINE(19);
        MEGA_FINE(20);
        MEGA_MARK();
        cons_sync();
        if (lane == 0) mbar_arrive(&p_empty[l & 1]);                   // this layer's parameter buffer may be refilled
    }
    // ---- final RMSNorm + tied lm_head GEMV + argmax ----
    float nrf;
    {
        const float ss = sx_gather<H>(sx_cur + (size_t)(p.L - 1) * SXL + H, xs);     // x_d of the last layer
        mbar_wait(&p_full[p.L & 1], (p.L >> 1) & 1);
        nrf = norm_scale(ss, H, p.eps, red);
    }
    static_assert(!(SAMPLE && TOPK), "sampling is never combined with the candidate lists");
    static_assert(4 * NCONS_WARPS <= 62, "per-warp records must fit red / ired");
    constexpr bool SLP = SAMPLE && LOGPROB;
    Draw dr{};
    float smx = -INFINITY, ssel = 0.f;                 // SLP: this lane's raw maximum logit, raw logit of its best-key row
    if constexpr (SAMPLE) dr = make_draw(p.smp, __ldcg(p.n_out), p.row);   // n_out changes only after every CTA's ticket
    if constexpr (HEADQ) {
        Slice sl = make_slice(p.lm_head, p.V, H, 1);
        sl.rpc = SLOT_BYTES / H;                       // rows per slot of the int8 copy
        consume_head_q<H>(sl, ring, q, xs, p.lm_head_sc, best_v, best_i, pbuf + (p.L & 1) * PARAM_FLOATS, nrf);
    } else {
        consume<H, ME_ARGMAX, LOGPROB, TOPK, SAMPLE, REP>(make_slice(p.lm_head, p.V, H, 1), ring, q, xs, nullptr, 0u, nullptr, best_v,
                                                          best_i, best_s, pbuf + (p.L & 1) * PARAM_FLOATS, nrf, nullptr, &tk, &dr, &smx,
                                                          &ssel, &rb);
    }
    MEGA_MARK();
    // candidates live in lanes 0, 8, 16, 24 of every warp (the four rows of a turn; lanes 0 / 16 in the two-row form):
    // merge them, lane 0 publishes the warp's best
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
        if constexpr (SAMPLE) {
            sample_merge_xor<LOGPROB>(o, best_v, best_i, best_s, smx, ssel);
        } else {
            const float ov = __shfl_xor_sync(0xffffffffu, best_v, o); const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
            if constexpr (LOGPROB) best_s = lse_merge(best_v, best_s, ov, __shfl_xor_sync(0xffffffffu, best_s, o));
            if (ov > best_v || (ov == best_v && oi < best_i)) { best_v = ov; best_i = oi; }
            if constexpr (TOPK) tk_merge_xor(tk, o);
        }
    }
    cons_sync();
    // TOPK: the warps' lists go to xs ([NCONS_WARPS][TK_MAX] values, then ids), free once the lm_head has read it
    float* tkv = xs; int* tki = reinterpret_cast<int*>(xs + NCONS_WARPS * TK_MAX);
    if (lane == 0) { red[warp] = best_v; ired[warp] = best_i; if constexpr (LOGPROB) red[NCONS_WARPS + warp] = best_s; }
    if constexpr (SLP) if (lane == 0) { red[2 * NCONS_WARPS + warp] = smx; red[3 * NCONS_WARPS + warp] = ssel; }
    if constexpr (TOPK) if (lane == 0) tk_store(tk, tkv + warp * TK_MAX, tki + warp * TK_MAX);
    cons_sync();
    int& is_last = ired[63];
    if (tid == 0) {
        float v = -INFINITY; int idx = 0x7fffffff; int ws = 0;
        for (int wq = 0; wq < NCONS_WARPS; ++wq)
            if (red[wq] > v || (red[wq] == v && ired[wq] < idx)) { v = red[wq]; idx = ired[wq]; if constexpr (SLP) ws = wq; }
        p.part_val[blockIdx.x] = v; p.part_idx[blockIdx.x] = idx;
        if constexpr (SLP) {                 // the warps' raw sums rescaled to the CTA's raw maximum, in warp order
            float M = -INFINITY;
            for (int wq = 0; wq < NCONS_WARPS; ++wq) M = fmaxf(M, red[2 * NCONS_WARPS + wq]);
            float sum = 0.f;
            for (int wq = 0; wq < NCONS_WARPS; ++wq) sum += lse_rescale(red[NCONS_WARPS + wq], red[2 * NCONS_WARPS + wq], M);
            p.part_sum[blockIdx.x] = sum; p.part_max[blockIdx.x] = M; p.part_sel[blockIdx.x] = red[3 * NCONS_WARPS + ws];
        }
        else if constexpr (LOGPROB) {        // the warps' sums rescaled to the CTA maximum, in warp order
            float sum = 0.f;
            for (int wq = 0; wq < NCONS_WARPS; ++wq) sum += lse_rescale(red[NCONS_WARPS + wq], red[wq], v);
            p.part_sum[blockIdx.x] = sum;
        }
        if constexpr (TOPK) {                // the CTA's TK_MAX best of its warps' lists
            for (int wq = 1; wq < NCONS_WARPS; ++wq) tk_merge_from(tk, tkv + wq * TK_MAX, tki + wq * TK_MAX, false);
            tk_store(tk, p.tk_part_val + (size_t)blockIdx.x * TK_MAX, p.tk_part_idx + (size_t)blockIdx.x * TK_MAX);
        }
        if constexpr (HEADQ) {               // candidate list header of consume_head_q (still in xs)
            const int* st = reinterpret_cast<const int*>(xs);
            atomicAdd(p.hq_stats, (unsigned long long)st[3]);
            if (st[1] > HQ_CAP || st[2] != 0) atomicAdd(p.hq_stats + 3, 1ull);
        }
        __threadfence();
        unsigned t = atomicAdd(p.bar, 1u);
        is_last = (t == G - 1);
    }
    cons_sync();
    if (!is_last) return;
    // ---- greedy bookkeeping by the last CTA (inference.rs:161-170) ----
    __threadfence();
    {
        float v = -INFINITY; int idx = 0x7fffffff;
        int rec = 0; float mloc = -INFINITY;         // SLP: the best key's record, the raw maximum of the records
        for (int i = tid; i < (int)G; i += NCONS) {
            float pv = __ldcg(p.part_val + i); int pi = __ldcg(p.part_idx + i);
            if (pv > v || (pv == v && pi < idx)) { v = pv; idx = pi; if constexpr (SLP) rec = i; }
            if constexpr (SLP) mloc = fmaxf(mloc, __ldcg(p.part_max + i));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ov = __shfl_xor_sync(0xffffffffu, v, o); int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            int orec = 0;
            if constexpr (SLP) orec = __shfl_xor_sync(0xffffffffu, rec, o);
            if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; if constexpr (SLP) rec = orec; }
        }
        if constexpr (SLP) mloc = warp_max(mloc);
        if (lane == 0) { red[warp] = v; ired[warp] = idx; }
        if constexpr (SLP) if (lane == 0) { ired[NCONS_WARPS + warp] = rec; red[2 * NCONS_WARPS + warp] = mloc; }
        cons_sync();
        float lp = 0.f, M = 0.f;
        if constexpr (LOGPROB) {
            // S = sum_c s_c exp(m_c - M) over the G records, M = the step's maximum logit (= that of the selected token
            // when not sampling): each thread its records in index order, then the warps in a fixed tree; logprob = -log S
            const float* rmax = SLP ? p.part_max : p.part_val;
            M = red[SLP ? 2 * NCONS_WARPS : 0];
            for (int wq = 1; wq < NCONS_WARPS; ++wq) M = fmaxf(M, red[(SLP ? 2 * NCONS_WARPS : 0) + wq]);
            float sum = 0.f;
            for (int i = tid; i < (int)G; i += NCONS) sum += lse_rescale(__ldcg(p.part_sum + i), __ldcg(rmax + i), M);
            sum = warp_sum(sum);
            if (lane == 0) red[NCONS_WARPS + warp] = sum;
            cons_sync();
            if (tid == 0) {
                float S = 0.f;
                for (int wq = 0; wq < NCONS_WARPS; ++wq) S += red[NCONS_WARPS + wq];
                lp = -logf(S);
            }
        }
        if constexpr (TOPK) {
            // the step's TK_MAX best of the G CTA lists: each thread merges its CTAs', then a butterfly per warp and
            // thread 0 the warps' lists (the exact top of one set: the order of the merges does not matter)
            tk_init(tk);
            for (int i = tid; i < (int)G; i += NCONS) tk_merge_from(tk, p.tk_part_val + (size_t)i * TK_MAX, p.tk_part_idx + (size_t)i * TK_MAX, true);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) tk_merge_xor(tk, o);
            if (lane == 0) tk_store(tk, tkv + warp * TK_MAX, tki + warp * TK_MAX);
            cons_sync();
            if (tid == 0)
                for (int wq = 1; wq < NCONS_WARPS; ++wq) tk_merge_from(tk, tkv + wq * TK_MAX, tki + wq * TK_MAX, false);
        }
        int& tok_s = ired[62];
        if (tid == 0) {
            for (int wq = 1; wq < NCONS_WARPS; ++wq)
                if (red[wq] > v || (red[wq] == v && ired[wq] < idx)) { v = red[wq]; idx = ired[wq]; if constexpr (SLP) rec = ired[NCONS_WARPS + wq]; }
            int tok = idx;
            if constexpr (SLP) lp = (__ldcg(p.part_sel + rec) - M) + lp;      // (l_sel - M) - log S
            const int n = *p.n_out;
            if constexpr (LOGPROB) {
                if (tok == 151643 || tok == 151645) *p.eos_lp = lp;
                else if (n < p.max_new) p.lp_out[n] = lp;
            }
            if constexpr (TOPK) {
                if (tok == 151643 || tok == 151645) tk_write(tk, lp, p.tk_eos_ids, p.tk_eos_lp);
                else if (n < p.max_new) tk_write(tk, lp, p.tk_ids + (size_t)n * TK_MAX, p.tk_lp + (size_t)n * TK_MAX);
            }
            if (tok == 151643 || tok == 151645 || n >= p.max_new) { *p.done = 1; *p.next_id = -1; tok = -1; }
            else { p.ids_out[n] = tok; *p.n_out = n + 1; *p.pos = pos + 1; *p.next_id = tok; }
            tok_s = tok;
            if constexpr (HEADQ) {               // every CTA has added its recomputed rows before its ticket
                const unsigned long long nr = __ldcg(p.hq_stats);
                p.hq_stats[0] = 0; p.hq_stats[1] = __ldcg(p.hq_stats + 1) + nr;
                if (nr > __ldcg(p.hq_stats + 2)) p.hq_stats[2] = nr;
            }
            p.bar[0] = 0;                        // every CTA has taken its ticket: reset for the next launch
            p.bar[1] = p.bar[1] + 1;             // new epoch: words published by this step can never match again
            p.bar[3] = p.bar[3] + 1;             // executed launches of this kernel: the next one uses the other set
        }
        cons_sync();
        const int tok = tok_s;
        if (tok >= 0) {
            const bf16* e = p.embed + (size_t)tok * H;
            for (int i = tid; i < H; i += NCONS) p.x[i] = __bfloat162float(e[i]);
        }
    }
}

}  // namespace mega

// host side ---------------------------------------------------------------------------------------
static long long* g_last_dbg = nullptr;   // debug only (ASRB_MEGA_DEBUG): timeline buffer of the last launch

static int mega_xs_floats(int I) { return std::max(I, mega::XS_MIN) + 64; }
static size_t mega_smem_bytes(int H, int I, int nslot) {
    return (size_t)nslot * mega::SLOT_BYTES +
           (mega_xs_floats(I) + mega::XRES_MAX + 2 * (2 * H + 2 * mega::HD) + 128) * 4 + mega::MAX_LAYERS * sizeof(DecLayerW) +
           (2 * mega::NSLOT_MAX + 4) * 8 + 64 * 4 + 64 * 4 + 128 * 4 + 64;
}
// instantiations: (hidden, q_dim, intermediate) -> ring depth
static int mega_nslot(const asrb_dims& c) { return c.hidden_size > 1024 ? 5 : 6; }

template <int H, int QD, int I> static bool dims_match(const asrb_dims& c) {
    return c.hidden_size == H && c.num_attention_heads * c.head_dim == QD && c.intermediate_size == I;
}

// `ctx` = number of keys the step may attend to (position + 1 upper bound), NOT the cache capacity
bool decode_mega_supported(const Model& m, int B, int ctx) {
    const int max_ctx = ctx;
    const asrb_dims& c = m.d.c;
    if (B < 1 || c.head_dim != 128) return false;      // batch > 1: one fused launch per sequence, back to back
    const int group = c.num_attention_heads / c.num_key_value_heads;
    if (group + 2 > mega::NCONS_WARPS) return false;
    if ((size_t)(group * 128 + 256 + group * mega::KV_KEYS + 8 + mega::NCONS_WARPS * 2 * 128 + mega::NCONS_WARPS * 4 + 8) > (size_t)mega_xs_floats(c.intermediate_size)) return false;
    if (m.ctx->smem_optin < mega_smem_bytes(c.hidden_size, c.intermediate_size, mega_nslot(c))) return false;
    if ((c.hidden_size + m.ctx->sm_count - 1) / m.ctx->sm_count + 1 > mega::XRES_MAX) return false;
    if (c.num_hidden_layers > 32) return false;                  // 5-bit layer field
    if ((max_ctx + mega::KV_KEYS - 1) / mega::KV_KEYS > mega::MAX_SPLITS) return false;                           // merge loop bound (SB)
    if (((max_ctx + mega::KV_KEYS - 1) / mega::KV_KEYS) * c.num_key_value_heads > m.ctx->sm_count) return false;   // one CTA per (kv head, 64-key split)
    return decode_mega_dims(c);
}
bool decode_mega_dims(const asrb_dims& c) {
    return dims_match<1024, 2048, 3072>(c) || dims_match<2048, 2048, 6144>(c) || dims_match<256, 512, 512>(c);
}

// floats of session scratch the fused step needs: tagged exchange buffers (2 floats per value)
size_t decode_mega_part_floats(const Model& m) {
    const asrb_dims& c = m.d.c;
    const int group = c.num_attention_heads / c.num_key_value_heads;
    const size_t words = (size_t)m.d.qkv_dim + (size_t)m.ctx->sm_count * group * mega::PSTRIDE + 64;
    return 2 * words + 64;
}
// bytes of the self-validating exchange words: [2 sets][L][x_o H | x_d H | attn QD | act I] uint32
size_t decode_mega_sx_bytes(const Model& m) {
    const asrb_dims& c = m.d.c;
    return 2 * (size_t)c.num_hidden_layers * (2 * (size_t)c.hidden_size + m.d.q_dim + c.intermediate_size) * sizeof(uint32_t);
}

// the instantiation for the model's dims and the run's options: sampling (with or without the log-probability record)
// is never combined with the candidate lists
template <bool LP, bool TK, bool SM, bool RP>
static const void* step_fn_dims(const asrb_dims& c) {
    if (dims_match<1024, 2048, 3072>(c)) return (const void*)mega::decode_step_kernel<1024, 2048, 3072, 6, LP, TK, SM, RP>;   // Qwen3-ASR-0.6B
    if (dims_match<2048, 2048, 6144>(c)) return (const void*)mega::decode_step_kernel<2048, 2048, 6144, 5, LP, TK, SM, RP>;   // Qwen3-ASR-1.7B
    return (const void*)mega::decode_step_kernel<256, 512, 512, 6, LP, TK, SM, RP>;                                           // test config
}
template <bool RP>
static const void* step_fn(const DecodeBufs& b, const asrb_dims& c) {
    if (b.sample) return b.logprobs ? step_fn_dims<true, false, true, RP>(c) : step_fn_dims<false, false, true, RP>(c);
    if (b.topk) return step_fn_dims<true, true, false, RP>(c);
    if (b.logprobs) return step_fn_dims<true, false, false, RP>(c);
    return step_fn_dims<false, false, false, RP>(c);
}

void launch_decode_step_mega(const Model& m, const DecodeBufs& b, int B, float* kcache, float* vcache,
                             size_t cache_layer_stride, size_t cache_seq_stride, int max_ctx, int ctx_now, const MegaBufs& mb,
                             cudaStream_t st, int64_t* launches) {
    ASRB_REQUIRE(decode_mega_supported(m, B, ctx_now), ASRB_ERR_STATE, "fused decode step not supported for this model/batch/context");
    ASRB_REQUIRE(m.d_dec_layers && mb.bar && mb.part && mb.sx_seq, ASRB_ERR_STATE, "fused decode step buffers missing");
    const bool greedy = !b.logprobs && !b.topk && !b.sample && !b.rep;      // the instantiation that reads the int8 copy
    ASRB_REQUIRE(!greedy || (m.lm_head_q && m.lm_head_sc && mb.hq_stats), ASRB_ERR_STATE, "fused decode step: int8 lm_head copy missing");
    const asrb_dims& c = m.d.c;
    const int G = m.ctx->sm_count;
    const int group = c.num_attention_heads / c.num_key_value_heads;
    // split count is fixed per session (buffer layout); splits beyond the current context are simply empty
    const int nsplit = std::min(mega::MAX_SPLITS, std::min(G / c.num_key_value_heads, (max_ctx + mega::KV_KEYS - 1) / mega::KV_KEYS));
    const size_t smem = mega_smem_bytes(c.hidden_size, c.intermediate_size, mega_nslot(c));
    const void* fn = b.rep ? step_fn<true>(b, c) : step_fn<false>(b, c);
    ASRB_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // The kernel handles one sequence.  A batch runs as B launches on the stream (weights are re-streamed per sequence:
    // 2.0 k tokens/s at any batch size, still ~1.8x the per-phase path at batch 8); a sequence that has finished
    // returns at once.  Exchange buffers are shared: launches are serialised by the stream, the tagged words carry the
    // epoch and the self-validating words switch sets with every executed launch.
    for (int sb = 0; sb < B; ++sb) {
        mega::Params p{};
        p.layers = m.d_dec_layers; p.lm_head = m.lm_head; p.embed = m.embed; p.final_norm = m.final_norm_sw;
        p.rope_cos = m.rope_cos; p.rope_sin = m.rope_sin; p.eps = (float)c.rms_norm_eps;
        p.L = c.num_hidden_layers; p.H = c.hidden_size; p.QD = m.d.q_dim; p.KVD = m.d.kv_dim; p.I = c.intermediate_size;
        p.V = c.vocab_size; p.nq = c.num_attention_heads; p.nkv = c.num_key_value_heads; p.group = group;
        p.x = b.x + (size_t)sb * c.hidden_size;
        p.kcache = kcache + (size_t)sb * cache_seq_stride; p.vcache = vcache + (size_t)sb * cache_seq_stride;
        p.cache_layer_stride = cache_layer_stride; p.max_ctx = max_ctx; p.nsplit = nsplit;
        p.part_val = b.part_val; p.part_idx = b.part_idx;
        p.pos = b.pos + sb; p.done = b.done + sb; p.next_id = b.next_id + sb;
        p.ids_out = b.ids_out + (size_t)sb * b.max_new; p.n_out = b.n_out + sb; p.max_new = b.max_new;
        p.bar = mb.bar;
        uint2* w = reinterpret_cast<uint2*>(mb.part);            // 16-byte aligned sub-buffers (even word counts)
        p.qkv_ll = w; w += m.d.qkv_dim;
        p.part_ll = w;
        p.sx = mb.sx_seq;
        p.dbg = mb.dbg;
        g_last_dbg = mb.dbg;
        if (b.logprobs) { p.part_sum = b.part_sum; p.lp_out = b.lp_out + (size_t)sb * b.max_new; p.eos_lp = b.eos_lp + sb; }
        if (b.topk) {
            p.tk_part_val = b.tk_part_val; p.tk_part_idx = b.tk_part_idx;
            p.tk_ids = b.tk_ids + (size_t)sb * b.max_new * TK_MAX; p.tk_lp = b.tk_lp + (size_t)sb * b.max_new * TK_MAX;
            p.tk_eos_ids = b.tk_eos_ids + (size_t)sb * TK_MAX; p.tk_eos_lp = b.tk_eos_lp + (size_t)sb * TK_MAX;
        }
        if (b.sample) {                      // per-sequence launches: the draw's row is the sequence's index in the batch
            p.smp = b.smp; p.row = sb;
            if (b.logprobs) { p.part_max = b.part_max; p.part_sel = b.part_sel; }
        }
        if (b.rep) { p.rep_bits = b.rep_mask; p.rep_words = rep_cta_words(c, G); p.rep = b.rep_params; }
        p.lm_head_q = m.lm_head_q; p.lm_head_sc = m.lm_head_sc; p.hq_stats = mb.hq_stats;
        // tags must stay monotonic for red.max publication: long before the 24-bit epoch wraps, wipe the tagged exchange
        // buffers (the self-validating words live elsewhere and are left alone: to them 0 would be a published 0.0)
        if (mb.steps_issued && ++*mb.steps_issued >= 0xFFFF00u) {
            ASRB_CUDA_CHECK(cudaMemsetAsync(mb.part, 0, mb.part_bytes, st));
            const unsigned one = 1;
            ASRB_CUDA_CHECK(cudaMemcpyAsync(mb.bar + 1, &one, sizeof(one), cudaMemcpyHostToDevice, st));
            *mb.steps_issued = 1;
        }
        void* args[] = {(void*)&p};
        ASRB_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(G), dim3(mega::NTHREADS), args, smem, st));
        if (launches) *launches += 1;
    }
}

// debug: copy the clock64 timeline of the most recent fused step (CTA 0 then CTA G-1), returns slots per CTA
int decode_mega_debug_timeline(long long* out, int cap) {
    if (!g_last_dbg || cap < 2 * mega::DBG_SLOTS) return 0;
    cudaDeviceSynchronize();
    cudaMemcpy(out, g_last_dbg, 2 * mega::DBG_SLOTS * sizeof(long long), cudaMemcpyDeviceToHost);
    return mega::DBG_SLOTS;
}
int decode_mega_dbg_slots() { return 4 * mega::DBG_SLOTS; }   // [0, 2048): two CTA timelines; [2048, 4096): per-CTA wall-clock table (decode_batch.cu)

}  // namespace asrb
