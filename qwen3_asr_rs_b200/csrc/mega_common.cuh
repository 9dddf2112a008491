// mega_common.cuh -- device helpers shared by the fused decode steps (decode_mega.cu: one sequence per launch,
// decode_batch.cu: NB sequences per launch): mbarrier / bulk-copy PTX, the tagged and the self-validating exchange
// words, the weight ring.
#pragma once
#include "internal.h"

namespace asrb {
namespace mega {

static constexpr int NCONS_WARPS = 8;
static constexpr int NCONS = NCONS_WARPS * 32;          // 256 consumer threads
static constexpr int NTHREADS = NCONS + 32;             // + 1 producer warp
static constexpr int SLOT_BYTES = 32 * 1024;           // 16 rows of K = 1024: one row per half-warp and pass
static constexpr int NSLOT_MAX = 6;                     // weight ring: 6 x 32 KB per SM (5 for the 1.7B dims: larger vectors)
static constexpr int KV_KEYS = 64;                      // keys per attention split (the K and V tiles are one ring slot each)
static constexpr int XS_MIN = 3072;                     // activation vector / attention scratch: max(I, XS_MIN) + 64 floats
static constexpr int XRES_MAX = 64;
static constexpr int MAX_LAYERS = 32;                   // layer table staged in shared memory                     // residual rows owned by one CTA (H / gridDim.x, rounded up)
static constexpr int HD = 128;
static constexpr int PSTRIDE = HD + 2;                  // partial record: o[128], m, l
static constexpr int DBG_SLOTS = 1024;
static constexpr int MAX_SPLITS = 18;                   // 64-key attention splits per kv head (also bounded by SMs / kv heads: 16 for the 0.6B dims on 132 SMs)

// phases of the tagged words (3 bits of the tag)
enum { PH_QKV = 1, PH_PART = 2 };

// ---- PTX helpers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// L2 policy for data read exactly once per step: its lines are the first to go when L2 needs room
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void cons_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NCONS) : "memory"); }

// ---- tagged exchange ({fp32 value, tag} in one 64-bit word) ------------------------------------
// Publication is a fire-and-forget 64-bit `red.max`: the tag sits in the upper 32 bits and grows monotonically for
// every word (epoch, then layer, then phase), so the new word is always the maximum, i.e. the reduction acts as an
// exchange.  Reductions are performed at L2 as soon as they are issued and return nothing: plain/volatile stores
// can linger in the SM before they become visible, a release fence per publication is expensive, and `atom.exch`
// (which returns the old value) serialises each warp's publications on the atomic round trip.
__device__ __forceinline__ void ll_store(uint2* p, float v, uint32_t tag) {
    const unsigned long long val = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
    asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" ::"l"(p), "l"(val) : "memory");
}
__device__ __forceinline__ float ll_poll1(const uint2* p, uint32_t tag) {
    uint2 v;
    do {
        asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    } while (v.y != tag);
    return __uint_as_float(v.x);
}
// four words at p, p+stride, ... : all loads are issued before any tag is examined (one round trip when ready)
__device__ __forceinline__ void ll_poll4(const uint2* p, int stride, uint32_t tag, float (&out)[4]) {
    uint2 v[4];
    bool ok;
    do {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v[i].x), "=r"(v[i].y) : "l"(p + (size_t)i * stride) : "memory");
        ok = (v[0].y == tag) && (v[1].y == tag) && (v[2].y == tag) && (v[3].y == tag);
    } while (!ok);
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = __uint_as_float(v[i].x);
}
// ---- self-validating 4-byte exchange words (the all-to-all vectors: x after o_proj / down_proj, attention output,
// SwiGLU activations).  A word is the fp32 value itself; 0xFFFFFFFF (a NaN pattern no result is ever published with)
// means "not written yet".  Publication = one fire-and-forget red.and (performed at L2 at once, like red.max of the
// tagged words); a gather polls 16-byte quads until none of the 4 words is the sentinel -- half the L2 traffic of
// {value, tag} words, and that traffic (one CTA per SM x every vector) is what bounds the all-gathers.
// Every (layer, vector) has its own region, and there are two such sets: step s uses set s & 1 and, at its start,
// re-arms (stores the sentinel into) the words THIS CTA wrote into the other set during step s - 1.  The kernel
// boundary orders that re-arm before any publication of step s + 1 into it, so a poll can only ever see the sentinel or
// the current step's value.  Each kernel counts its own executed steps for the set parity.
static constexpr uint32_t SX_EMPTY = 0xFFFFFFFFu;
__device__ __forceinline__ void sx_store(uint32_t* p, float v) {
    uint32_t b = __float_as_uint(v);
    if (b == SX_EMPTY) b = 0x7FFFFFFFu;                   // (another NaN)
    asm volatile("red.relaxed.gpu.global.and.b32 [%0], %1;" ::"l"(p), "r"(b) : "memory");
}
__device__ __forceinline__ uint4 sx_load4(const uint32_t* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ bool sx_ready(const uint4& v) {
    return v.x != SX_EMPTY && v.y != SX_EMPTY && v.z != SX_EMPTY && v.w != SX_EMPTY;
}

// Activation vectors in shared memory are stored with 16-byte group k at k ^ ((k >> 3) & 1).  The GEMV register loads
// read, per lane, the two groups of 8 consecutive elements (32-byte lane stride): unswizzled, lanes i and i+4 of every
// quarter warp hit the same banks (2-way conflict on every LDS.128).
__device__ __forceinline__ int xs_swz(int e) { const int k = e >> 2; return ((k ^ ((k >> 3) & 1)) << 2) | (e & 3); }

struct Ring {
    uint8_t* slots; uint64_t* full; uint64_t* empty;
    uint32_t nslot;         // ring depth (compile-time constant of the instantiation, propagated through inlining)
};

// one weight phase as seen by a CTA: rows [r0, r1) of W[N][K]
struct Slice { const bf16* W; int K, r0, r1, rpc; };
__device__ __forceinline__ Slice make_slice(const bf16* W, int N, int K, int rstep) {
    Slice s; s.W = W; s.K = K;
    const unsigned units = (unsigned)(N / rstep);      // units * gridDim.x < 2^32 for every matrix of the model
    const int u0 = (int)((blockIdx.x * units) / gridDim.x), u1 = (int)(((blockIdx.x + 1) * units) / gridDim.x);
    s.r0 = u0 * rstep; s.r1 = u1 * rstep;
    s.rpc = SLOT_BYTES / (K * 2);
    s.rpc &= ~1;                        // keep (gate, up) pairs together
    return s;
}

}  // namespace mega
}  // namespace asrb
