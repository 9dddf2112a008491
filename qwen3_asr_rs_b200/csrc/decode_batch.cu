// decode_batch.cu -- one greedy decode iteration (inference.rs:160-200) for NB INDEPENDENT sequences as ONE
// persistent kernel: every weight byte is streamed from HBM once per step and contracted against the activation
// vectors of all NB sequences (the reference runs the same loop body once per utterance, src/inference.rs:89).
//
// Same machinery as the single-sequence step (decode_mega.cu): one CTA per SM, a producer warp that streams this
// CTA's row slice of every weight matrix through a shared-memory ring with cp.async.bulk + mbarrier, 8 consumer
// warps, {value, tag} words published with fire-and-forget red.max and polled by the consumers (no grid barriers).
// What changes with a batch:
//   * the GEMVs become skinny GEMMs [16 weight rows] x [NB sequences] on the tensor cores: fp32 CUDA-core FMAs cost
//     rows x K x NB / 128 cycles per SM at best (128 fp32 FMA lanes per SM), of the order of the HBM time of the
//     whole step at NB = 8.  Activations are written into shared memory as THREE bf16
//     planes (hi + mid + lo == x to 1 ulp, common.cuh: bf16 x bf16 products are exact in fp32), weights are bf16
//     already, so mma.sync.m16n8k16 with fp32 accumulation reproduces the fp32 GEMV to accumulation-order noise.  A
//     16-row tile is contracted by all 8 warps (each takes 1/8 of K: at most 384 products per accumulator, which also
//     keeps the tensor core's truncating accumulation below the noise floor), partial tiles are summed through
//     shared memory in a fixed order.  The tile shape follows the CTA's row slice (7 .. 42 rows per matrix), which is
//     why this is the warp-level MMA and not a 64-row wgmma tile.
//     Weight rows are read from a copy whose 16-byte chunks are XOR-swizzled by (row & 7) (model.cu), so that the
//     bulk-copied rows (2 KB pitch) are bank-conflict free for ldmatrix.
//   * o_proj / down_proj (7 rows per CTA, K = 2048 / 3072) keep their rows resident in the ring and walk K in
//     chunks of H (the capacity of the activation planes).
//   * attention work items are (sequence, kv head, KVK-key split of the CACHED keys), dealt round-robin to the
//     CTAs; K and V tiles travel through a two-slot shared-memory stage that the producer refills while the
//     consumers compute; one CTA per (sequence, kv head) merges the partials, folds in the current token's own
//     key/value and appends it to the cache (replaces Tensor::cat, layers.rs:311-317).
//   * greedy bookkeeping (argmax, EOS, append, next embedding; inference.rs:161-170) for every sequence by the
//     last CTA to finish the lm_head.
// Arithmetic per (row, sequence) is the fp32 FMA chain of decode_mega.cu (same lane -> element mapping, same
// reduction tree for the K = H phases), so a batch reproduces the single-sequence results.
#include <algorithm>
#include "mega_common.cuh"

namespace asrb {

namespace megab {
using namespace mega;

static constexpr int MAXSPLIT = 32;       // partial records per (sequence, kv head): lanes of the merging warps
static constexpr int MAXROWS = 8;         // residual rows owned by one CTA (H / gridDim.x rounded up)
static constexpr int ATT_SCRATCH = 4 * HD + NCONS_WARPS * 2 * HD + NCONS_WARPS * 4 + 8 + 8 + 2 * HD;   // q[2][128] k v, per-warp partials, merge q

struct Params {
    const DecLayerW* layers;     // device array [L]: weight matrices = the chunk-swizzled copies (model.cu), norm vectors plain
    const bf16* lm_head;
    const bf16* embed;
    const float* final_norm;
    const float* rope_cos; const float* rope_sin;
    float eps;
    int L, H, QD, KVD, I, V, nkv;
    int nb;                      // active sequences of this launch (<= NB)
    float* x;                    // [nb][H] embedding of the pending tokens (in) / of the next tokens (out)
    float* kcache; float* vcache; size_t cache_layer_stride, cache_seq_stride; int max_ctx;
    float* part_val; int* part_idx; int n_part;     // [nb][n_part] argmax partials (first gridDim.x used)
    int* pos; int* done; int* next_id; int* ids_out; int* n_out; int max_new;
    unsigned* bar;               // [0] finish ticket, [1] launch epoch, [2] batched steps executed
    uint2* qkv_ll; uint2* part_ll;      // tagged {value, tag} words (few readers per word)
    uint32_t* sx;                        // self-validating 4-byte words [2 sets][L][XO | XD | ATTN | ACT][NB][rows]
    long long* dbg;              // optional timeline [2][DBG_SLOTS] of clock64 (CTA 0 and CTA G-1), else null
    int flags;                   // bit 0: L2 prefetch of the next layer's K/V tiles
    // LOGPROB instantiations only (appended: the offsets above stay those of the default instantiations)
    float* part_sum;             // [nb][n_part] sum of exp(logit - part_val) over the CTA's lm_head rows
    float* lp_out;               // [nb][max_new] log-probability of each appended token
    float* eos_lp;               // [nb] log-probability of the EOS token that ends the sequence
    // TOPK instantiations only (appended as well)
    float* tk_part_val; int* tk_part_idx;   // [nb][n_part][TK_MAX] each CTA's best (logit, id) candidates per sequence
    int* tk_ids; float* tk_lp;              // [nb][max_new][TK_MAX] candidates of each appended token's step, best first
    int* tk_eos_ids; float* tk_eos_lp;      // [nb][TK_MAX] those of the step that selects EOS
    // SAMPLE instantiations only (appended as well)
    const SampleParams* smp;     // 1 / temperature and seed of the run
    int row0;                    // row of sequence 0 of this launch in the call's batch (the draw's counter)
    float* part_max; float* part_sel;       // LOGPROB: [nb][n_part] raw maximum logit, raw logit of the best-key row
    // REP instantiations only (appended as well)
    uint32_t* rep_bits;                     // [gridDim.x][NB][2][rep_words] each CTA's history / banned bits of its lm_head rows
    int rep_words;
    const RepParams* rep;                   // the run's penalty and N
};

__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}

// ---- warp-level tensor-core pieces ---------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// 16-byte chunk c of a row whose chunks are XOR-swizzled by `key` (low 3 bits) inside every 128-byte group
__device__ __forceinline__ int swz16(int c, int key) { return (c & ~7) | ((c ^ key) & 7); }

// One 16-row weight tile x NB sequences over NKS k-steps (16 elements each).
// (template NKS = k-steps)
//   arow  : shared-memory address of THIS LANE's A row (row lane & 15 of the tile), first byte of the row
//   akey  : swizzle key of that row (global row index & 7);  ac0: first 16-byte chunk of the k-range inside the row
//   xp    : shared-memory address of activation plane 0, sequence 0;  planes PSTR bytes apart, sequences H * 2 bytes apart,
//           chunks swizzled by (sequence & 7);  xc0: first chunk of the k-range inside the activation row
// acc[nt] = the m16n8 accumulator fragment of sequences 8 nt .. 8 nt + 7
template <int H, int NT, int PSTR, int NKS>
__device__ __forceinline__ void mma_tile(uint32_t arow, int akey, int ac0, uint32_t xp, int xc0, int lane, float (&acc)[NT][4]) {
    const int ahalf = lane >> 4;                         // A: lanes 16-31 address the k 8..15 halves
    const int bpl = lane >> 4, bhalf = (lane >> 3) & 1, bseq = lane & 7;   // B x4: planes 0 / 1 by half-warp
    float acc1[NT][4], acc2[NT][4];                      // one chain per activation plane (the MMAs of a chain are dependent)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int k = 0; k < 4; ++k) { acc1[nt][k] = 0.f; acc2[nt][k] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < NKS; ++ks) {
        uint32_t a0, a1, a2, a3;
        ldsm_x4(arow + (uint32_t)swz16(ac0 + 2 * ks + ahalf, akey) * 16u, a0, a1, a2, a3);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int sq = nt * 8 + bseq;
            const uint32_t xrow = xp + (uint32_t)sq * (H * 2) + (uint32_t)swz16(xc0 + 2 * ks + bhalf, sq & 7) * 16u;
            uint32_t b00, b01, b10, b11, b20, b21;
            ldsm_x4(xrow + (uint32_t)bpl * PSTR, b00, b01, b10, b11);
            ldsm_x2(xrow + 2u * PSTR, b20, b21);         // (lanes 16-31 pass valid addresses that are ignored)
            mma16816(acc[nt], a0, a1, a2, a3, b00, b01);
            mma16816(acc1[nt], a0, a1, a2, a3, b10, b11);
            mma16816(acc2[nt], a0, a1, a2, a3, b20, b21);
        }
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[nt][k] += acc1[nt][k] + acc2[nt][k];
}

// (the all-to-all vectors travel as self-validating 4-byte words: SX_EMPTY, sx_store, sx_load4 in mega_common.cuh;
//  the multiplier of their traffic here is NB sequences)

// per-head RMSNorm + RoPE of one 128-vector by one warp (lane holds d = lane, +32, +64, +96); input = tagged words
__device__ __forceinline__ void head_norm_rope_b(const uint2* __restrict__ src, uint32_t tag, const float* __restrict__ nw,
                                                 float eps, const float* __restrict__ cs, const float* __restrict__ sn,
                                                 float* dst, int lane) {
    float v[4];
    ll_poll4(src + lane, 32, tag, v);
    const float ss = warp_sum(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
    const float r = 1.0f / sqrtf(ss / 128.f + eps);
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = (v[i] * r) * __ldg(nw + lane + 32 * i);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int d = lane + 32 * i;
        const float c = cs[d], s = sn[d];
        const float a = v[i], b = v[i + 2];
        dst[d] = a * c - b * s;
        dst[d + 64] = b * c + a * s;
    }
}

enum { BE_STORE = 0, BE_SWIGLU = 1, BE_ARGMAX = 2 };

// LOGPROB: the lm_head also keeps (max, sum of exponentials) per (tile row, sequence), and the last CTA records the
// log-probability of each selected token (p.lp_out / p.eos_lp)
// TOPK (with LOGPROB): each (tile row, sequence) thread also keeps its best TK_MAX (logit, id) pairs; they are merged
// per sequence across tile rows and CTAs, and the last CTA records each step's candidates (p.tk_ids / p.tk_lp, or the
// EOS rows)
// SAMPLE: each (tile row, sequence) thread folds the sampling keys of draw (p.row0 + sequence, n = p.n_out[sequence])
// instead of the logits (common.cuh); with LOGPROB the tile-row, CTA and last-CTA merges also carry the raw (max, sum)
// record and the raw logit of the best-key row
// REP: each (tile row, sequence) thread first replaces the logit by its processed value under its sequence's bit arrays
// (repetition controls, common.cuh), built for the CTA's lm_head rows while layer 0's weights stream in
template <int H, int QD, int I, int NB, int NS, int KVK, bool LOGPROB, bool TOPK = false, bool SAMPLE = false, bool REP = false>
__global__ void __launch_bounds__(NTHREADS, 1) decode_batch_kernel(const Params p) {   // 9 warps are allocated as 12 (granularity 4): 168 registers
    static_assert(NB % 8 == 0 && NB <= 16, "NB must be 8 or 16");
    static_assert(H % 256 == 0 && QD % H == 0 && I % H == 0, "chunking needs QD, I multiples of H, H multiple of 256");
    constexpr int NT = NB / 8;                  // m16n8 accumulator tiles per 16-row weight tile
    constexpr int PSTR = NB * H * 2;            // bytes between the bf16 activation planes
    constexpr int KSW = (H / 16) / NCONS_WARPS; // k-steps (of 16) each warp contracts per H-long chunk
    static_assert(KSW >= 1, "H too small for an 8-way K split");
    constexpr int KPW = KVK / NCONS_WARPS;      // keys per warp in an attention tile
    constexpr int NV = 2 * KPW;                 // scores per lane before the butterfly (keys x 2 heads)
    constexpr int KV_TILE = KVK * HD * 4;
    constexpr int GROUP = 2;                    // q heads per kv head (checked on the host)
    constexpr int XS_FLOATS = (3 * PSTR / 4 > ATT_SCRATCH) ? 3 * PSTR / 4 : ATT_SCRATCH;   // activation planes; attention scratch aliases them
    static_assert(!TOPK || LOGPROB, "the candidates' log-probabilities need the sum of exponentials");
    static_assert(16 * NB * (1 + 2 * TK_MAX) <= XS_FLOATS, "lm_head merge records must fit the activation planes");
    static_assert(!(SAMPLE && TOPK), "sampling is never combined with the candidate lists");
    constexpr bool SLP = SAMPLE && LOGPROB;
    extern __shared__ __align__(128) uint8_t smem[];
    Ring ring;
    ring.slots = smem; ring.nslot = NS;
    static_assert(KV_TILE == SLOT_BYTES, "K / V tiles travel through the weight ring: one tile per slot");
    float* xs = reinterpret_cast<float*>(smem + (size_t)NS * SLOT_BYTES);   // bf16 planes [3][NB][H] (chunks swizzled by sequence)
    float4* pbuf = reinterpret_cast<float4*>(xs + XS_FLOATS);           // [2][8 warps][NT][32 lanes] partial accumulator fragments
    float* xres = reinterpret_cast<float*>(pbuf + 2 * NCONS_WARPS * NT * 32);   // [NB][MAXROWS]
    float* ropes = xres + NB * MAXROWS;                                 // [NB][128]  cos | sin of each sequence's position
    float* redk = ropes + NB * 128;                                     // [8 warps][32] K-split partials / scratch
    float* ssred = redk + NCONS_WARPS * 32;                             // [8 warps][NB] sums of squares
    float* rs = ssred + NCONS_WARPS * NB;                               // [NB] RMSNorm scales
    float* bestv = rs + NB;                                             // [16 rows][NB]
    int* besti = reinterpret_cast<int*>(bestv + 16 * NB);               // [16 rows][NB]
    int* seqi = besti + 16 * NB;                               // pos[NB] | nact[NB] | off[NB + 1] | misc[4]
    DecLayerW* ltab = reinterpret_cast<DecLayerW*>(seqi + 3 * NB + 8);  // [MAX_LAYERS]
    uint64_t* bars = reinterpret_cast<uint64_t*>(ltab + MAX_LAYERS);
    ring.full = bars; ring.empty = bars + 8;                          // up to 8 slots
    int* pos_s = seqi; int* nact_s = seqi + NB; int* off_s = seqi + 2 * NB; int* misc = seqi + 3 * NB + 1;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool is_producer = warp == NCONS_WARPS;
    const int nb = p.nb;
    const unsigned G = gridDim.x;

    {   // every sequence finished: nothing to do this step
        bool all = true;
        for (int b = 0; b < nb; ++b) all = all && (__ldcg(p.done + b) != 0);
        if (all) return;
    }
    if (tid == 0) {
        for (int i = 0; i < NS; ++i) { mbar_init(&ring.full[i], 1); mbar_init(&ring.empty[i], NCONS_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        int o = 0;
        for (int b = 0; b < NB; ++b) {
            const int ps = b < nb ? __ldcg(p.pos + b) : 0;
            pos_s[b] = ps; nact_s[b] = (ps + KVK - 1) / KVK; off_s[b] = o; o += nact_s[b];
        }
        off_s[NB] = o;
    }
    {
        const uint2* src = reinterpret_cast<const uint2*>(p.layers);
        uint2* dst = reinterpret_cast<uint2*>(ltab);
        for (int i = tid; i < p.L * (int)(sizeof(DecLayerW) / 8); i += NTHREADS) dst[i] = src[i];
        for (int i = tid; i < nb * 128; i += NTHREADS) {
            const int b = i >> 7, d = i & 127;
            const int ps = __ldcg(p.pos + b);
            ropes[i] = d < 64 ? p.rope_cos[(size_t)ps * 64 + d] : p.rope_sin[(size_t)ps * 64 + d - 64];
        }
    }
    __syncthreads();
    const int T = off_s[NB] * p.nkv;            // attention work items of this step: (sequence, kv head, split)
    // item t -> (b, g, sp): sequence-major, then kv head, then split
    auto item_decode = [&](int t, int& b, int& g, int& sp) __attribute__((always_inline)) {
        b = 0;
#pragma unroll
        for (int i = 1; i < NB; ++i) if (t >= off_s[i] * p.nkv) b = i;
        const int r = t - off_s[b] * p.nkv, na = nact_s[b];
        g = r / na; sp = r - g * na;
    };

    // contiguous item range of this CTA and the owner of an item
    // (the top nb * nkv CTAs also merge one (sequence, kv head) each -- about two tiles' worth of latency -- so they take
    //  half a share of the items: range_start is piecewise linear in the CTA index)
    const int n_merge = min(nb * p.nkv, (int)G);
    const int c_merge = (int)G - n_merge;                             // first merging CTA
    const int W2 = 2 * c_merge + n_merge;                             // total capacity in half shares (cw * T < 2^21: 32-bit math)
    auto range_start = [&](int c) __attribute__((always_inline)) { const int cw = c <= c_merge ? 2 * c : 2 * c_merge + (c - c_merge); return (int)(((unsigned)cw * (unsigned)T) / (unsigned)W2); };
    auto item_owner = [&](int t) __attribute__((always_inline)) {                                    // largest c with range_start(c) <= t
        int lo = 0, hi = (int)G - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (range_start(mid) <= t) lo = mid; else hi = mid - 1; }
        return lo;
    };
    const int it0 = range_start((int)blockIdx.x), it1 = range_start((int)blockIdx.x + 1);

    if (is_producer) {
        // ONE stream in consumption order through ONE ring: [q|k|v] rows, this CTA's K / V tiles (K then V per item), o_proj,
        // gate/up, down_proj rows of every layer, then the lm_head.  Nothing in it depends on activations, so it runs
        // ahead across phase boundaries as far as the ring allows; during the attention phase the whole ring is in
        // flight for K / V (the phase is bound by bytes in flight per SM x latency), otherwise it holds upcoming weights.
        if (lane == 0) {
            uint32_t q = 0;
            auto issue = [&](const void* src, uint32_t bytes) __attribute__((always_inline)) {
                const uint32_t slot = q % NS, par = (q / NS) & 1;
                mbar_wait(&ring.empty[slot], par ^ 1);
                mbar_expect_tx(&ring.full[slot], bytes);
                bulk_g2s(ring.slots + (size_t)slot * SLOT_BYTES, src, bytes, &ring.full[slot]);
                ++q;
            };
            auto issue_slice = [&](const Slice& s) __attribute__((always_inline)) {
                for (int r = s.r0; r < s.r1; r += s.rpc) issue(s.W + (size_t)r * s.K, (uint32_t)min(s.rpc, s.r1 - r) * s.K * 2);
            };
            for (int l = 0; l < p.L; ++l) {
                const DecLayerW w = ltab[l];
                issue_slice(make_slice(w.wqkv, QD + 2 * p.KVD, H, 1));
                for (int t = it0; t < it1; ++t) {
                    int kb, kg, ksp;
                    item_decode(t, kb, kg, ksp);
                    const int nloc = min(KVK, pos_s[kb] - ksp * KVK);
                    const size_t off = (size_t)l * p.cache_layer_stride + (size_t)kb * p.cache_seq_stride +
                                       ((size_t)kg * p.max_ctx + (size_t)ksp * KVK) * HD;
                    issue(p.kcache + off, (uint32_t)nloc * HD * 4);
                    issue(p.vcache + off, (uint32_t)nloc * HD * 4);
                }
                issue_slice(make_slice(w.wo, H, QD, 1));
                issue_slice(make_slice(w.wgu, 2 * I, H, 2));
                issue_slice(make_slice(w.wdown, H, I, 1));
            }
            issue_slice(make_slice(p.lm_head, p.V, H, 1));
        }
        return;
    }

    // ------------------------------ consumers ------------------------------
    long long* dbg_row = nullptr; int dbg_i = 0;
    if (p.dbg && (blockIdx.x == 0 || blockIdx.x == G - 1)) dbg_row = p.dbg + (blockIdx.x == 0 ? 0 : DBG_SLOTS);
#define MARK() do { if (dbg_row && tid == 0 && dbg_i < DBG_SLOTS) dbg_row[dbg_i++] = clock64(); } while (0)
    int fine_l = -1, fine_i = 0;   // detail marks of layer 5 -> slots 600...
// every CTA: wall clock (globaltimer, ns) of event k of layer 5 -> slots [2048 + 8 * cta + k)
#define GT(k) do { if (p.dbg && tid == 0 && fine_l == 5) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); p.dbg[2 * DBG_SLOTS + 8 * blockIdx.x + (k)] = (long long)t_; } } while (0)
#define FINE() do { if (dbg_row && tid == 0 && fine_l == 5 && fine_i < 200) dbg_row[600 + fine_i++] = clock64(); } while (0)
    MARK();
    uint32_t q = 0;
    const unsigned epoch = __ldcg(p.bar + 1);
    const uint32_t tag_base = (epoch & 0xffffffu) << 8;
    const Slice xsl = make_slice(nullptr, H, QD, 1);                  // residual rows owned by this CTA
    const int xrows = xsl.r1 - xsl.r0;
    for (int i = tid; i < nb * xrows; i += NCONS) {
        const int b = i / xrows, r = i - b * xrows;
        xres[b * MAXROWS + r] = __ldcg(p.x + (size_t)b * H + xsl.r0 + r);
    }
    float best_v = -INFINITY; int best_i = 0x7fffffff;      // lm_head: running argmax of (tile row tid / NB, sequence tid % NB)
    float best_s = 0.f;                                      // LOGPROB: its sum of exp(logit - best_v)
    TopK tk;                                                 // TOPK: its best rows
    if constexpr (TOPK) tk_init(tk);
    Draw dr{};                                               // SAMPLE: the draw of its sequence (n_out changes only after
    float smx = -INFINITY, ssel = 0.f;                       // every CTA's ticket); SLP: raw maximum, raw logit of the best key
    if constexpr (SAMPLE) if (tid < 16 * NB && tid % NB < nb) dr = make_draw(p.smp, __ldcg(p.n_out + tid % NB), p.row0 + tid % NB);
    RepBits rb{};                                            // REP: the bit arrays of its sequence (n_out changes only after
    if constexpr (REP) {                                     // every CTA's ticket)
        const Slice sl = make_slice(nullptr, p.V, H, 1);
        uint32_t* rbits = p.rep_bits + (size_t)blockIdx.x * NB * 2 * p.rep_words;   // this CTA's [NB][2][rep_words]
        const int W = p.rep_words, N = __ldg(&p.rep->ngram);
        for (int i = tid; i < NB * 2 * W; i += NCONS) rbits[i] = 0u;
        cons_sync();
        for (int b = 0; b < nb; ++b)
            rep_mark(p.ids_out + (size_t)b * p.max_new, min(__ldcg(p.n_out + b), p.max_new), N, sl.r0, sl.r1, rbits + b * 2 * W,
                     rbits + b * 2 * W + W, tid, NCONS);
        const uint32_t* h = rbits + (tid % NB) * 2 * W;
        rb = RepBits{h, h + W, sl.r0 >> 5, __ldg(&p.rep->theta)};
    }
    // merging CTA: which (sequence, kv head), and which record slots will be written for it -- slot u holds a record iff a
    // run starts at split u, i.e. u == 0 or item base + u opens its owner's range.  Positions do not change within the
    // step, so this is computed once, not per layer (the owner search is a dozen integer divisions per slot).
    const int mid = (int)G - 1 - (int)blockIdx.x;
    const bool merger = mid < nb * p.nkv;
    const int mb_ = merger ? mid / p.nkv : 0, mg_ = merger ? mid - mb_ * p.nkv : 0;
    unsigned merge_mask = 0;
    if (merger) {
        const int base_t = off_s[mb_] * p.nkv + mg_ * nact_s[mb_];
        for (int u = 0; u < nact_s[mb_]; ++u)
            if (u == 0 || range_start(item_owner(base_t + u)) == base_t + u) merge_mask |= 1u << u;
    }
    // exchange regions of this step (set = epoch parity) and re-arm of the other set (words this CTA wrote last step)
    constexpr size_t SX_LAYER = (size_t)NB * (2 * H + QD + I);            // words per (set, layer): XO | XD | ATTN | ACT, each [seq][row]
    // (set = parity of the BATCHED-step counter bar[2]: the launch epoch bar[1] is shared with the single-sequence kernel,
    //  whose launches in between would break the strict alternation the re-arm relies on)
    const unsigned bstep = __ldcg(p.bar + 2);
    uint32_t* const sx_cur = p.sx + (size_t)(bstep & 1u) * p.L * SX_LAYER;
    {
        uint32_t* const other = p.sx + (size_t)((bstep & 1u) ^ 1u) * p.L * SX_LAYER;
        const Slice sa = make_slice(nullptr, I, H, 1);                    // act rows of this CTA = gate/up units
        const Slice sq = make_slice(nullptr, QD, H, 1);                   // (attention outputs are re-armed by row range too)
        for (int l = 0; l < p.L; ++l) {
            uint32_t* base = other + (size_t)l * SX_LAYER;
            for (int i = tid; i < NB * xrows; i += NCONS) {
                const int b = i / xrows, r = i - b * xrows;
                base[(size_t)b * H + xsl.r0 + r] = SX_EMPTY;                              // XO
                base[(size_t)NB * H + (size_t)b * H + xsl.r0 + r] = SX_EMPTY;             // XD
            }
            const int ar = sa.r1 - sa.r0;
            for (int i = tid; i < NB * ar; i += NCONS) {
                const int b = i / ar, r = i - b * ar;
                base[(size_t)NB * (2 * H + QD) + (size_t)b * I + sa.r0 + r] = SX_EMPTY;   // ACT
            }
            const int qr = sq.r1 - sq.r0;
            for (int i = tid; i < NB * qr; i += NCONS) {
                const int b = i / qr, r = i - b * qr;
                base[(size_t)NB * 2 * H + (size_t)b * QD + sq.r0 + r] = SX_EMPTY;         // ATTN
            }
        }
    }

    // ---- gather of one H-long chunk of every active sequence into the activation planes, optional RMSNorm ----
    // src: self-validating words, sequence b at src + b * src_stride.  Values stay in registers between the poll and
    // the plane stores; NORM: x <- (x * r_b) * w  (rounding order of layers.rs:48-54), then the exact 3-way bf16 split.
    const uint32_t xp_addr = smem_u32(xs);
    // exact 3-way bf16 split by TRUNCATION: hi = top 16 bits of x, mid = top 16 bits of (x - hi), lo = x - hi - mid.  Both
    // subtractions are exact and lo has <= 8 significant bits, so hi + mid + lo == x exactly; logic + FADD only (the
    // round-to-nearest split of common.cuh needs three F2F conversions per value, which issue at quarter rate).
    auto store_planes = [&](int b, int j, float4 f) __attribute__((always_inline)) {       // quad j (elements 4 j .. 4 j + 3) of sequence b
        const float xv[4] = {f.x, f.y, f.z, f.w};
        uint32_t hb[4], mb[4], lb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            hb[i] = __float_as_uint(xv[i]) & 0xffff0000u;
            const float r1 = xv[i] - __uint_as_float(hb[i]);
            mb[i] = __float_as_uint(r1) & 0xffff0000u;
            lb[i] = __float_as_uint(r1 - __uint_as_float(mb[i]));
        }
        uint8_t* dst = reinterpret_cast<uint8_t*>(xs) + (size_t)b * (H * 2) + swz16(j >> 1, b & 7) * 16 + (j & 1) * 8;
        *reinterpret_cast<uint2*>(dst) = make_uint2(__byte_perm(hb[0], hb[1], 0x7632), __byte_perm(hb[2], hb[3], 0x7632));
        *reinterpret_cast<uint2*>(dst + PSTR) = make_uint2(__byte_perm(mb[0], mb[1], 0x7632), __byte_perm(mb[2], mb[3], 0x7632));
        *reinterpret_cast<uint2*>(dst + 2 * PSTR) = make_uint2(__byte_perm(lb[0], lb[1], 0x7632), __byte_perm(lb[2], lb[3], 0x7632));
    };
    constexpr int PP = (H / 4 + NCONS - 1) / NCONS;     // 16-byte quads per thread and sequence
    static_assert(NB * PP <= 16, "gather keeps NB * PP quads per thread in registers");
    // gather pieces: g_load issues this thread's 16-byte loads of one H-long chunk of every sequence (idle slots re-read the
    // last active sequence / quad 0, so everything stays in registers), g_valid checks the self-validating words
    auto g_load = [&](uint4 (&v)[NB][PP], const uint32_t* src, size_t src_stride) __attribute__((always_inline)) {
#pragma unroll
        for (int b = 0; b < NB; ++b)
#pragma unroll
            for (int i = 0; i < PP; ++i) {
                const int j = tid + i * NCONS;
                const int bb = min(b, nb - 1), jj = (PP * NCONS > H / 4 && j >= H / 4) ? 0 : j;
                v[b][i] = sx_load4(src + (size_t)bb * src_stride + 4 * jj);
            }
    };
    auto g_valid = [&](const uint4 (&v)[NB][PP]) __attribute__((always_inline)) {
        bool ok = true;
#pragma unroll
        for (int b = 0; b < NB; ++b)
#pragma unroll
            for (int i = 0; i < PP; ++i)
                ok = ok && (v[b][i].x != SX_EMPTY) && (v[b][i].y != SX_EMPTY) && (v[b][i].z != SX_EMPTY) && (v[b][i].w != SX_EMPTY);
        return ok;
    };
    // values -> (optional RMSNorm: x <- (x * r_b) * w, rounding order of layers.rs:48-54) -> bf16 planes; ends with a barrier
    auto g_store = [&](const uint4 (&v)[NB][PP], const float* normw) __attribute__((always_inline)) {
        float4 wv[PP];
        if (normw) {
#pragma unroll
            for (int i = 0; i < PP; ++i) {
                const int j = tid + i * NCONS;
                wv[i] = (j < H / 4) ? __ldg(reinterpret_cast<const float4*>(normw + 4 * j)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                float t = 0.f;
#pragma unroll
                for (int i = 0; i < PP; ++i) {
                    const int j = tid + i * NCONS;
                    if (j < H / 4) {
                        const float x0 = __uint_as_float(v[b][i].x), x1 = __uint_as_float(v[b][i].y), x2 = __uint_as_float(v[b][i].z), x3 = __uint_as_float(v[b][i].w);
                        t = fmaf(x0, x0, t); t = fmaf(x1, x1, t); t = fmaf(x2, x2, t); t = fmaf(x3, x3, t);
                    }
                }
                t = warp_sum(t);
                if (lane == 0) ssred[warp * NB + b] = t;
            }
            cons_sync();
            if (tid < nb) {
                float tot = 0.f;
#pragma unroll
                for (int w8 = 0; w8 < NCONS_WARPS; ++w8) tot += ssred[w8 * NB + tid];
                rs[tid] = 1.0f / sqrtf(tot / H + p.eps);
            }
            cons_sync();
        }
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            if (b < nb) {
                const float r = normw ? rs[b] : 1.f;
#pragma unroll
                for (int i = 0; i < PP; ++i) {
                    const int j = tid + i * NCONS;
                    if (j < H / 4) {
                        float4 f = make_float4(__uint_as_float(v[b][i].x), __uint_as_float(v[b][i].y), __uint_as_float(v[b][i].z), __uint_as_float(v[b][i].w));
                        if (normw) f = make_float4((f.x * r) * wv[i].x, (f.y * r) * wv[i].y, (f.z * r) * wv[i].z, (f.w * r) * wv[i].w);
                        store_planes(b, j, f);
                    }
                }
            }
        }
        FINE();
        cons_sync();
    };
    // from_sx: poll self-validating words; else plain fp32 rows (layer 0: embeddings written by the previous step / prefill)
    auto gather = [&](const uint32_t* src, size_t src_stride, const float* normw, bool from_sx) __attribute__((always_inline)) {
        uint4 v[NB][PP];
        do { g_load(v, src, src_stride); } while (from_sx && !g_valid(v));
        FINE();
        g_store(v, normw);
    };

    // sum of the 8 warps' partial accumulator fragments (fixed order) for element (tile row tid / NB, sequence tid % NB)
    auto tile_sum = [&](int par) __attribute__((always_inline)) {
        const int row = tid / NB, sq = tid - row * NB;
        const int nt = sq >> 3, col = sq & 7;
        const int ln = (row & 7) * 4 + (col >> 1), reg = (row >> 3) * 2 + (col & 1);
        const float* pb = reinterpret_cast<const float*>(pbuf + (size_t)par * NCONS_WARPS * NT * 32) + ((size_t)nt * 32 + ln) * 4 + reg;
        float t = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < NCONS_WARPS; ++w8) t += pb[(size_t)w8 * NT * 32 * 4];
        return t;
    };
    int ppar = 0;      // partial-buffer parity (double buffer: a tile's sums are read while the next tile's partials are written)

    // ---- K = H phases: rows stream through the ring; every 16-row tile is contracted by all 8 warps (K split 8 ways) ----
    // BE_STORE publishes tagged words into `out` (q/k/v: read by the few attention CTAs of each head), BE_SWIGLU publishes
    // self-validating words into `sxo` (activations: gathered by every CTA), BE_ARGMAX keeps the running argmax
    auto rows_phase = [&](const Slice& s, int epi, uint2* out, size_t out_stride, uint32_t tag, uint32_t* sxo) __attribute__((always_inline)) {
        for (int r = s.r0; r < s.r1; r += s.rpc, ++q) {
            const int rows = min(s.rpc, s.r1 - r);
            const uint32_t slot = q % NS, par = (q / NS) & 1;
            mbar_wait(&ring.full[slot], par);
            const uint32_t sbase = smem_u32(ring.slots + (size_t)slot * SLOT_BYTES);
            for (int t0 = 0; t0 < rows; t0 += 16) {
                const int ri = min(t0 + (lane & 15), rows - 1);          // rows past the slot's last row alias it (never published)
                float acc[NT][4];
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int k = 0; k < 4; ++k) acc[nt][k] = 0.f;
                mma_tile<H, NT, PSTR, KSW>(sbase + (uint32_t)ri * (H * 2), (r + ri) & 7, warp * KSW * 2, xp_addr, warp * KSW * 2, lane, acc);
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
                    pbuf[((size_t)ppar * NCONS_WARPS + warp) * NT * 32 + nt * 32 + lane] = make_float4(acc[nt][0], acc[nt][1], acc[nt][2], acc[nt][3]);
                if (t0 + 16 >= rows) {                                   // last tile of the slot: this warp is done with its weights
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ring.empty[slot]);
                }
                cons_sync();
                if (tid < 16 * NB) {
                    float v = tile_sum(ppar);
                    const int rr = t0 + tid / NB, sq = tid % NB, row = r + rr;
                    const bool valid = rr < rows && sq < nb;
                    if (epi == BE_STORE) {
                        if (valid) ll_store(out + (size_t)sq * out_stride + row, v, tag);
                    } else if (epi == BE_SWIGLU) {
                        const float up = __shfl_down_sync(0xffffffffu, v, NB);     // rows 2j (gate) and 2j + 1 (up): NB threads apart
                        if (valid && !(rr & 1)) sx_store(sxo + (size_t)sq * I + (row >> 1), silu(v) * up);
                    } else if constexpr (SAMPLE) {
                        if (valid && rep_keep<REP>(&rb, row, v))
                            sample_fold<LOGPROB>(dr, v, row, best_v, best_i, best_s, smx, ssel);   // rows ascend per thread
                    } else if constexpr (LOGPROB) {
                        if (valid && rep_keep<REP>(&rb, row, v)) {
                            lse_fold(v, row, best_v, best_i, best_s);     // rows ascend per thread: ties keep the first
                            if constexpr (TOPK) tk_insert(tk, v, row);
                        }
                    } else {
                        if (valid && rep_keep<REP>(&rb, row, v) && (v > best_v || (v == best_v && row < best_i))) { best_v = v; best_i = row; }
                    }
                }
                ppar ^= 1;
            }
        }
    };

    // ---- K = NCH * H phases with <= 8 resident rows (o_proj, down_proj): the activation planes hold one H-long chunk at
    //      a time, every chunk is contracted by all 8 warps into the same accumulators; result: residual add +
    //      publication into `sxo` (layers.rs:454,460) ----
    auto resident_phase = [&](const Slice& s, int NCH, const uint32_t* src, size_t src_stride, uint32_t* sxo) __attribute__((always_inline)) {
        const int rows = s.r1 - s.r0;
        const int nslots = (rows + s.rpc - 1) / s.rpc;
        const int ri = min(lane & 15, rows - 1);                          // rows past the slice alias the last row (never published)
        const uint32_t arow = smem_u32(ring.slots + (size_t)((q + ri / s.rpc) % NS) * SLOT_BYTES) + (uint32_t)(ri % s.rpc) * (uint32_t)(s.K * 2);
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[nt][k] = 0.f;
        // chunk pipeline: the loads of chunk c + 1 are in flight while chunk c is split into planes and contracted
        uint4 cur[NB][PP];
        g_load(cur, src, src_stride);
        for (int ch = 0; ch < NCH; ++ch) {
            while (!g_valid(cur)) g_load(cur, src + (size_t)ch * H, src_stride);
            FINE();
            g_store(cur, nullptr);
            uint4 nxt[NB][PP];
            const int chn = min(ch + 1, NCH - 1);                     // (the last iteration re-reads its own chunk: unconditional, registers only)
            g_load(nxt, src + (size_t)chn * H, src_stride);           // in flight during the MMAs
            if (ch == 0)
                for (int i = 0; i < nslots; ++i) mbar_wait(&ring.full[(q + i) % NS], ((q + i) / NS) & 1);
            FINE();
            mma_tile<H, NT, PSTR, KSW>(arow, (s.r0 + ri) & 7, ch * (H / 8) + warp * KSW * 2, xp_addr, warp * KSW * 2, lane, acc);
            FINE();
            cons_sync();                                                  // the planes may be overwritten by the next chunk
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int i = 0; i < PP; ++i) cur[b][i] = nxt[b][i];
        }
        __syncwarp();
        if (lane == 0) for (int i = 0; i < nslots; ++i) mbar_arrive(&ring.empty[(q + i) % NS]);
        q += nslots;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
            pbuf[((size_t)ppar * NCONS_WARPS + warp) * NT * 32 + nt * 32 + lane] = make_float4(acc[nt][0], acc[nt][1], acc[nt][2], acc[nt][3]);
        cons_sync();
        if (tid < 16 * NB) {
            const float tot = tile_sum(ppar);
            const int rr = tid / NB, sq = tid % NB;
            if (rr < rows && sq < nb) {
                const float nv = xres[sq * MAXROWS + rr] + tot;
                xres[sq * MAXROWS + rr] = nv;
                sx_store(sxo + (size_t)sq * H + s.r0 + rr, nv);
            }
        }
        ppar ^= 1;
    };

    for (int l = 0; l < p.L; ++l) {
        const DecLayerW w = ltab[l];
        fine_l = l;
        const uint32_t tl = tag_base | ((uint32_t)l << 3);
        uint32_t* const sxl = sx_cur + (size_t)l * SX_LAYER;                       // this layer's XO | XD | ATTN | ACT words
        uint32_t* const sx_xo = sxl; uint32_t* const sx_xd = sxl + (size_t)NB * H;
        uint32_t* const sx_attn = sxl + (size_t)NB * 2 * H; uint32_t* const sx_act = sxl + (size_t)NB * (2 * H + QD);
        // ---- phase 1: RMSNorm + [q|k|v] GEMV ----
        if (l == 0) gather(reinterpret_cast<const uint32_t*>(p.x), H, w.ln_in, false);
        else gather(sxl - SX_LAYER + (size_t)NB * H, H, w.ln_in, true);            // XD of the previous layer
        MARK();
        GT(0);
        rows_phase(make_slice(w.wqkv, QD + 2 * p.KVD, H, 1), BE_STORE, p.qkv_ll, (size_t)(QD + 2 * p.KVD), tl | PH_QKV, nullptr);
        cons_sync();                                  // xs is free: attention scratch aliases it
        MARK();
        GT(1);
        // ---- phase 2: attention partials of this CTA's work items ----
        // Items are sorted (sequence, kv head, split) and dealt in CONTIGUOUS ranges: a CTA's range consists of a few
        // "runs" of consecutive splits of one (sequence, kv head).  Within a run every warp keeps an online-softmax
        // state (max, sum, 4 output dims per lane, both q heads) in registers over the tiles -- no CTA barrier per
        // tile -- and the 8 warp states are merged through shared memory once per run: one partial record per
        // (CTA, run), stored at the slot of the run's first split.  A run starts at split 0 and wherever a CTA's range
        // starts, so the merging CTA can enumerate the slots that will be written.
        {
            float* qs = xs;                           // [2][128]
            float* kn = qs + GROUP * HD;              // [128]
            float* vn = kn + HD;                      // [128]
            float* osum = vn + HD;                    // [warps][2][128]
            float* wml = osum + NCONS_WARPS * GROUP * HD;   // [warps][2][2]
            float* snew = wml + NCONS_WARPS * 4;      // [2]
            constexpr int SH = (NV == 16) ? 1 : (NV == 8 ? 2 : 3);
            // merging CTA: the current token's q / k / v of its (sequence, kv head) are ready as soon as the [q|k|v] phase is
            // (long before the partial records), so RMSNorm + RoPE, the cache append and the new key's scores happen NOW,
            // off the tail of the phase
            float* mq = snew + 8;                     // [2][128] q heads of the merge (the item runs reuse qs)
            if (merger) {
                const float* cs = ropes + mb_ * 128; const float* sn = cs + 64;
                const uint2* qkvb = p.qkv_ll + (size_t)mb_ * (QD + 2 * p.KVD);
                if (warp < GROUP) head_norm_rope_b(qkvb + (size_t)(mg_ * GROUP + warp) * HD, tl | PH_QKV, w.qnorm, p.eps, cs, sn, mq + warp * HD, lane);
                else if (warp == GROUP) head_norm_rope_b(qkvb + QD + (size_t)mg_ * HD, tl | PH_QKV, w.knorm, p.eps, cs, sn, kn, lane);
                else if (warp == GROUP + 1) {
                    float vv[4];
                    ll_poll4(qkvb + QD + p.KVD + (size_t)mg_ * HD + lane, 32, tl | PH_QKV, vv);
#pragma unroll
                    for (int i = 0; i < 4; ++i) vn[lane + 32 * i] = vv[i];
                }
                cons_sync();
                if (tid < HD) {                       // KV append (replaces Tensor::cat, layers.rs:311-317)
                    const size_t off = (size_t)l * p.cache_layer_stride + (size_t)mb_ * p.cache_seq_stride + ((size_t)mg_ * p.max_ctx + pos_s[mb_]) * HD;
                    p.kcache[off + tid] = kn[tid]; p.vcache[off + tid] = vn[tid];
                }
                if (warp >= NCONS_WARPS - GROUP) {    // score of the new key for head hq
                    const int hq = warp - (NCONS_WARPS - GROUP);
                    const float4 a = *reinterpret_cast<const float4*>(mq + hq * HD + lane * 4);
                    const float4 c4 = *reinterpret_cast<const float4*>(kn + lane * 4);
                    const float s_ = warp_sum(fmaf(a.x, c4.x, fmaf(a.y, c4.y, fmaf(a.z, c4.z, a.w * c4.w))));
                    if (lane == 0) snew[hq] = s_ / sqrtf((float)HD);
                }
                // (the barrier before the first run / the merge orders these writes)
            }
            int t = it0;
            while (t < it1) {
                int b, g, sp;
                item_decode(t, b, g, sp);
                const int nrun = min(nact_s[b] - sp, it1 - t);
                const float* cs = ropes + b * 128; const float* sn = cs + 64;
                if (warp < GROUP)
                    head_norm_rope_b(p.qkv_ll + (size_t)b * (QD + 2 * p.KVD) + (size_t)(g * GROUP + warp) * HD, tl | PH_QKV,
                                     w.qnorm, p.eps, cs, sn, qs + warp * HD, lane);
                cons_sync();
                const float4 q0 = *reinterpret_cast<const float4*>(qs + lane * 4);
                const float4 q1 = *reinterpret_cast<const float4*>(qs + HD + lane * 4);
                float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;       // running (max, sum) of head 0 / 1
                float4 o0 = make_float4(0.f, 0.f, 0.f, 0.f), o1 = o0;
                for (int it = 0; it < nrun; ++it) {
                    const int nloc = min(KVK, pos_s[b] - (sp + it) * KVK);
                    const uint32_t ksl = q % NS, vsl = (q + 1) % NS;
                    const float* Ks = reinterpret_cast<const float*>(ring.slots + (size_t)ksl * SLOT_BYTES);
                    const float* Vs = reinterpret_cast<const float*>(ring.slots + (size_t)vsl * SLOT_BYTES);
                    mbar_wait(&ring.full[ksl], (q / NS) & 1);
                    float pv[NV];
#pragma unroll
                    for (int kk = 0; kk < KPW; ++kk) {
                        const int j = warp + 8 * kk;      // rows past the split's last key hold stale data and are masked below
                        const float4 kv = *reinterpret_cast<const float4*>(Ks + j * HD + lane * 4);
                        pv[2 * kk] = fmaf(kv.x, q0.x, fmaf(kv.y, q0.y, fmaf(kv.z, q0.z, kv.w * q0.w)));
                        pv[2 * kk + 1] = fmaf(kv.x, q1.x, fmaf(kv.y, q1.y, fmaf(kv.z, q1.z, kv.w * q1.w)));
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ring.empty[ksl]);  // K tile consumed by this warp
                    // transposing butterfly: lane L ends with score index L >> SH (index = 2 * key + head)
#pragma unroll
                    for (int o = 16, n = NV; n > 1; o >>= 1, n >>= 1) {
                        const bool up = lane & o;
#pragma unroll
                        for (int i = 0; i < n / 2; ++i) {
                            const float send = up ? pv[i] : pv[i + n / 2];
                            const float keep = up ? pv[i + n / 2] : pv[i];
                            pv[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                        }
                    }
#pragma unroll
                    for (int o = (1 << SH) >> 1; o > 0; o >>= 1) pv[0] += __shfl_xor_sync(0xffffffffu, pv[0], o);
                    const int sidx = lane >> SH;                                   // 2 * kk + head
                    const bool mine = warp + 8 * (sidx >> 1) < nloc;
                    const float sv = mine ? pv[0] / sqrtf((float)HD) : -INFINITY;
                    float mw = sv;                                                 // max over this warp's keys of the tile, per head
#pragma unroll
                    for (int o = 2 << SH; o < 32; o <<= 1) mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, o));
                    const float mwo = __shfl_xor_sync(0xffffffffu, mw, 1 << SH);  // the other head's
                    const bool h1 = sidx & 1;
                    const float n0 = fmaxf(m0, h1 ? mwo : mw), n1 = fmaxf(m1, h1 ? mw : mwo);     // new running maxima
                    const float c0 = (m0 == -INFINITY) ? 0.f : expf(m0 - n0), c1 = (m1 == -INFINITY) ? 0.f : expf(m1 - n1);
                    const float ev = mine ? expf(sv - (h1 ? n1 : n0)) : 0.f;
                    float lw = ev;
#pragma unroll
                    for (int o = 2 << SH; o < 32; o <<= 1) lw += __shfl_xor_sync(0xffffffffu, lw, o);
                    const float lwo = __shfl_xor_sync(0xffffffffu, lw, 1 << SH);
                    l0 = fmaf(l0, c0, h1 ? lwo : lw); l1 = fmaf(l1, c1, h1 ? lw : lwo);
                    m0 = n0; m1 = n1;
                    o0.x *= c0; o0.y *= c0; o0.z *= c0; o0.w *= c0; o1.x *= c1; o1.y *= c1; o1.z *= c1; o1.w *= c1;
                    mbar_wait(&ring.full[vsl], ((q + 1) / NS) & 1);
#pragma unroll
                    for (int kk = 0; kk < KPW; ++kk) {
                        const int j = warp + 8 * kk;
                        const float4 vv = *reinterpret_cast<const float4*>(Vs + j * HD + lane * 4);
                        const float e0 = __shfl_sync(0xffffffffu, ev, (2 * kk) << SH), e1 = __shfl_sync(0xffffffffu, ev, (2 * kk + 1) << SH);
                        if (j < nloc) {       // (a stale V row may hold non-finite garbage: 0 * inf must not reach the sum)
                            o0.x = fmaf(e0, vv.x, o0.x); o0.y = fmaf(e0, vv.y, o0.y); o0.z = fmaf(e0, vv.z, o0.z); o0.w = fmaf(e0, vv.w, o0.w);
                            o1.x = fmaf(e1, vv.x, o1.x); o1.y = fmaf(e1, vv.y, o1.y); o1.z = fmaf(e1, vv.z, o1.z); o1.w = fmaf(e1, vv.w, o1.w);
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ring.empty[vsl]);  // V tile consumed by this warp
                    q += 2;
                }
                *reinterpret_cast<float4*>(osum + (warp * 2 + 0) * HD + lane * 4) = o0;
                *reinterpret_cast<float4*>(osum + (warp * 2 + 1) * HD + lane * 4) = o1;
                if (lane == 0) { wml[(warp * 2 + 0) * 2] = m0; wml[(warp * 2 + 0) * 2 + 1] = l0; wml[(warp * 2 + 1) * 2] = m1; wml[(warp * 2 + 1) * 2 + 1] = l1; }
                cons_sync();
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
                    // record slot = split index of the run's first tile
                    uint2* rec = p.part_ll + ((((size_t)b * p.nkv + g) * MAXSPLIT + sp) * GROUP + hq) * PSTRIDE;
                    ll_store(rec + d, acc, tl | PH_PART);
                    if (d < 2) ll_store(rec + HD + d, d == 0 ? M : Ls, tl | PH_PART);
                }
                cons_sync();                          // scratch may be overwritten by the next run
                t += nrun;
            }
            MARK();
            GT(2);
            // ---- merge of one (sequence, kv head): all its partial records + the current token's key / value ----
            if (merger) {
                const int b = mb_, g = mg_;
                const int nact = nact_s[b];                                                        // record slots of (b, g)
                const unsigned startmask = merge_mask;
                cons_sync();                          // kn / vn / snew of the early preparation are visible to every warp
                {
                    const int hq = tid / HD, d = tid - hq * HD;          // hq is uniform per warp (HD = 4 warps)
                    const uint32_t tg = tl | PH_PART;
                    constexpr int RB = 8;                                // partial outputs fetched per round (registers)
                    uint2 mv, lv, ov[RB];
                    bool ok;
                    const uint2* recb = p.part_ll + (((size_t)b * p.nkv + g) * MAXSPLIT * GROUP + hq) * PSTRIDE;
                    auto load_round = [&](int u0) {
#pragma unroll
                        for (int u = 0; u < RB; ++u)
                            if (u0 + u < nact && ((startmask >> (u0 + u)) & 1u)) {
                                const uint2* rec = recb + (size_t)(u0 + u) * GROUP * PSTRIDE;
                                asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(ov[u].x), "=r"(ov[u].y) : "l"(rec + d) : "memory");
                            }
                    };
                    auto round_ok = [&](int u0) {
                        bool k = true;
#pragma unroll
                        for (int u = 0; u < RB; ++u) if (u0 + u < nact && ((startmask >> (u0 + u)) & 1u)) k = k && (ov[u].y == tg);
                        return k;
                    };
                    const bool has_rec = lane < nact && ((startmask >> lane) & 1u);
                    do {        // first round: (max, sum) of every record (one per lane) + the first RB partial outputs
                        mv.y = tg; lv.y = tg; mv.x = 0u; lv.x = 0u;
                        if (has_rec) {
                            const uint2* rec = recb + (size_t)lane * GROUP * PSTRIDE;
                            asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(mv.x), "=r"(mv.y) : "l"(rec + HD) : "memory");
                            asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(lv.x), "=r"(lv.y) : "l"(rec + HD + 1) : "memory");
                        }
                        load_round(0);
                        ok = __all_sync(0xffffffffu, (mv.y == tg) && (lv.y == tg) && round_ok(0));
                    } while (!ok);
                    // softmax merge, one record per lane; the current token's key is one more partial (max = its score,
                    // sum = 1, output = its value row)
                    const float m_l = has_rec ? __uint_as_float(mv.x) : -INFINITY;
                    const float l_l = has_rec ? __uint_as_float(lv.x) : 0.f;
                    const float sn_ = snew[hq];
                    const float M = fmaxf(warp_max(m_l), sn_);
                    const float f = expf(m_l - M);                       // exp(-inf) = 0 on idle lanes
                    const float fn = expf(sn_ - M);
                    const float Lsum = warp_sum(f * l_l) + fn;
                    float O = fn * vn[d];
                    for (int u0 = 0; u0 < nact; u0 += RB) {
                        if (u0 > 0) { do { load_round(u0); ok = __all_sync(0xffffffffu, round_ok(u0)); } while (!ok); }
#pragma unroll
                        for (int u = 0; u < RB; ++u)
                            if (u0 + u < nact && ((startmask >> (u0 + u)) & 1u)) O = fmaf(__shfl_sync(0xffffffffu, f, u0 + u), __uint_as_float(ov[u].x), O);
                    }
                    sx_store(sx_attn + (size_t)b * QD + (size_t)(g * GROUP + hq) * HD + d, O / Lsum);
                }
                cons_sync();                          // attention scratch (aliases xs) is free again
            }
        }
        MARK();
        GT(3);
        // ---- phase 3: o_proj GEMV + residual ----
        resident_phase(make_slice(w.wo, H, QD, 1), QD / H, sx_attn, QD, sx_xo);
        MARK();
        GT(4);
        // ---- phase 4: RMSNorm + gate/up GEMV + SiLU*mul ----
        gather(sx_xo, H, w.ln_post, true);
        MARK();
        rows_phase(make_slice(w.wgu, 2 * I, H, 2), BE_SWIGLU, nullptr, 0, 0u, sx_act);
        cons_sync();
        MARK();
        GT(5);
        // ---- phase 5: down GEMV + residual ----
        resident_phase(make_slice(w.wdown, H, I, 1), I / H, sx_act, I, sx_xd);
        MARK();
    }
    // ---- final RMSNorm + tied lm_head GEMV + argmax ----
    gather(sx_cur + (size_t)(p.L - 1) * SX_LAYER + (size_t)NB * H, H, p.final_norm, true);
    MARK();
    rows_phase(make_slice(p.lm_head, p.V, H, 1), BE_ARGMAX, nullptr, 0, 0u, nullptr);
    MARK();
    // every thread tid < 16 NB holds the best row of (tile row tid / NB, sequence tid % NB): merge the 16 tile rows per sequence
    cons_sync();
    // LOGPROB: the sums go to the activation planes, which nothing reads once the lm_head tiles are contracted
    float* bests = xs;                                       // [16 rows][NB]
    float* tkv = xs + 16 * NB;                               // TOPK: [16 rows][NB][TK_MAX] candidate values, then ids
    int* tki = reinterpret_cast<int*>(tkv + 16 * NB * TK_MAX);
    float* smxs = xs + 16 * NB;                              // SLP: [16 rows][NB] raw maxima, then raw logits of the best keys
    float* ssels = smxs + 16 * NB;
    if (tid < 16 * NB) { bestv[tid] = best_v; besti[tid] = best_i; if constexpr (LOGPROB) bests[tid] = best_s; }
    if constexpr (SLP) if (tid < 16 * NB) { smxs[tid] = smx; ssels[tid] = ssel; }
    if constexpr (TOPK) if (tid < 16 * NB) tk_store(tk, tkv + tid * TK_MAX, tki + tid * TK_MAX);
    cons_sync();
    int& is_last = misc[0];
    if (tid < nb) {
        float v = -INFINITY; int idx = 0x7fffffff; int ws = 0;
        for (int wq = 0; wq < 16; ++wq) {
            const float cv = bestv[wq * NB + tid]; const int ci = besti[wq * NB + tid];
            if (cv > v || (cv == v && ci < idx)) { v = cv; idx = ci; if constexpr (SLP) ws = wq; }
        }
        p.part_val[(size_t)tid * p.n_part + blockIdx.x] = v; p.part_idx[(size_t)tid * p.n_part + blockIdx.x] = idx;
        if constexpr (SLP) {                                 // the 16 tile rows' raw sums rescaled to the CTA's raw maximum
            float M = -INFINITY;
            for (int wq = 0; wq < 16; ++wq) M = fmaxf(M, smxs[wq * NB + tid]);
            float sum = 0.f;
            for (int wq = 0; wq < 16; ++wq) sum += lse_rescale(bests[wq * NB + tid], smxs[wq * NB + tid], M);
            const size_t o = (size_t)tid * p.n_part + blockIdx.x;
            p.part_sum[o] = sum; p.part_max[o] = M; p.part_sel[o] = ssels[ws * NB + tid];
        }
        else if constexpr (LOGPROB) {                             // the 16 tile rows' sums rescaled to the CTA maximum, in row order
            float sum = 0.f;
            for (int wq = 0; wq < 16; ++wq) sum += lse_rescale(bests[wq * NB + tid], bestv[wq * NB + tid], v);
            p.part_sum[(size_t)tid * p.n_part + blockIdx.x] = sum;
        }
        if constexpr (TOPK) {                                // the CTA's TK_MAX best of the sequence's 16 tile rows
            tk_init(tk);
            for (int wq = 0; wq < 16; ++wq) tk_merge_from(tk, tkv + (wq * NB + tid) * TK_MAX, tki + (wq * NB + tid) * TK_MAX, false);
            const size_t o = ((size_t)tid * p.n_part + blockIdx.x) * TK_MAX;
            tk_store(tk, p.tk_part_val + o, p.tk_part_idx + o);
        }
        __threadfence();
    }
    cons_sync();
    if (tid == 0) {
        __threadfence();
        const unsigned t = atomicAdd(p.bar, 1u);
        is_last = (t == G - 1);
    }
    cons_sync();
    if (!is_last) return;
    // ---- greedy bookkeeping by the last CTA (inference.rs:161-170), one warp per sequence ----
    __threadfence();
    for (int b = warp; b < nb; b += NCONS_WARPS) {
        if (__ldcg(p.done + b) != 0) { if (lane == 0) p.next_id[b] = -1; continue; }
        float v = -INFINITY; int idx = 0x7fffffff;
        int rec = 0; float M = -INFINITY;                    // SLP: the best key's record, the raw maximum of the records
        for (int i = lane; i < (int)G; i += 32) {
            const float pv = __ldcg(p.part_val + (size_t)b * p.n_part + i); const int pi = __ldcg(p.part_idx + (size_t)b * p.n_part + i);
            if (pv > v || (pv == v && pi < idx)) { v = pv; idx = pi; if constexpr (SLP) rec = i; }
            if constexpr (SLP) M = fmaxf(M, __ldcg(p.part_max + (size_t)b * p.n_part + i));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, v, o); const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            int orec = 0;
            if constexpr (SLP) orec = __shfl_xor_sync(0xffffffffu, rec, o);
            if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; if constexpr (SLP) rec = orec; }
        }
        if constexpr (SLP) M = warp_max(M);
        int tok = idx;
        const int n = p.n_out[b];
        if constexpr (LOGPROB) {
            // S = sum_c s_c exp(m_c - M) over the G records (M = v, the maximum: every lane holds it after the butterfly;
            // SLP: the raw maximum), each lane its records in index order, then a fixed butterfly; logprob = -log S
            // (SLP: (l_sel - M) - log S)
            float sum = 0.f;
            for (int i = lane; i < (int)G; i += 32) {
                if constexpr (SLP) sum += lse_rescale(__ldcg(p.part_sum + (size_t)b * p.n_part + i), __ldcg(p.part_max + (size_t)b * p.n_part + i), M);
                else sum += lse_rescale(__ldcg(p.part_sum + (size_t)b * p.n_part + i), __ldcg(p.part_val + (size_t)b * p.n_part + i), v);
            }
            float lp = -logf(warp_sum(sum));
            if constexpr (SLP) lp = (__ldcg(p.part_sel + (size_t)b * p.n_part + rec) - M) + lp;
            if (lane == 0) {
                if (tok == 151643 || tok == 151645) p.eos_lp[b] = lp;
                else if (n < p.max_new) p.lp_out[(size_t)b * p.max_new + n] = lp;
            }
            if constexpr (TOPK) {
                // the TK_MAX best of the G CTA lists: each lane merges its CTAs', then a butterfly (every lane ends
                // with the same list, the exact top of one set whatever the order)
                tk_init(tk);
                for (int i = lane; i < (int)G; i += 32) {
                    const size_t o = ((size_t)b * p.n_part + i) * TK_MAX;
                    tk_merge_from(tk, p.tk_part_val + o, p.tk_part_idx + o, true);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) tk_merge_xor(tk, o);
                if (lane == 0) {
                    if (tok == 151643 || tok == 151645) tk_write(tk, lp, p.tk_eos_ids + (size_t)b * TK_MAX, p.tk_eos_lp + (size_t)b * TK_MAX);
                    else if (n < p.max_new) {
                        const size_t o = ((size_t)b * p.max_new + n) * TK_MAX;
                        tk_write(tk, lp, p.tk_ids + o, p.tk_lp + o);
                    }
                }
            }
        }
        if (tok == 151643 || tok == 151645 || n >= p.max_new) {
            if (lane == 0) { p.done[b] = 1; p.next_id[b] = -1; }
            tok = -1;
        } else if (lane == 0) {
            p.ids_out[(size_t)b * p.max_new + n] = tok; p.n_out[b] = n + 1; p.pos[b] = pos_s[b] + 1; p.next_id[b] = tok;
        }
        if (tok >= 0) {
            const bf16* e = p.embed + (size_t)tok * H;
            for (int i = lane; i < H; i += 32) p.x[(size_t)b * H + i] = __bfloat162float(e[i]);
        }
    }
    cons_sync();
    if (tid == 0) {
        p.bar[0] = 0;                        // every CTA has taken its ticket: reset for the next launch
        p.bar[1] = p.bar[1] + 1;             // new epoch: words published by this step can never match again
        p.bar[2] = p.bar[2] + 1;             // batched steps executed: selects the exchange set of the next one
    }
}

}  // namespace megab

// host side ---------------------------------------------------------------------------------------
static long long* g_last_dbg_batch = nullptr;   // debug only (ASRB_MEGA_DEBUG): timeline buffer of the last batched launch
int decode_batch_debug_timeline(long long* out, int cap) {
    if (!g_last_dbg_batch || cap < 4 * mega::DBG_SLOTS) return 0;
    cudaDeviceSynchronize();
    cudaMemcpy(out, g_last_dbg_batch, 4 * mega::DBG_SLOTS * sizeof(long long), cudaMemcpyDeviceToHost);
    return mega::DBG_SLOTS;
}

template <int H, int QD, int I> static bool bdims_match(const asrb_dims& c) {
    return c.hidden_size == H && c.num_attention_heads * c.head_dim == QD && c.intermediate_size == I;
}
struct BatchCfg { int NB, NS, KVK; };
static BatchCfg batch_cfg(int B) { return B <= 8 ? BatchCfg{8, 5, 64} : BatchCfg{16, 3, 64}; }

static size_t batch_smem_bytes(int H, const BatchCfg& k) {
    return (size_t)k.NS * mega::SLOT_BYTES +
           (std::max<size_t>((size_t)3 * k.NB * H / 2, megab::ATT_SCRATCH) + k.NB * megab::MAXROWS + k.NB * 128 + mega::NCONS_WARPS * 32 + mega::NCONS_WARPS * k.NB + k.NB +
            2 * 16 * k.NB + 3 * k.NB + 8) * 4 + (size_t)2 * mega::NCONS_WARPS * (k.NB / 8) * 32 * 16 +
           mega::MAX_LAYERS * sizeof(DecLayerW) + 16 * 8 + 128;
}

// `ctx` = upper bound of (position + 1) over the batch for this step
bool decode_batch_supported(const Model& m, int B, int ctx) {
    const asrb_dims& c = m.d.c;
    if (B < 2 || c.head_dim != 128) return false;
    if (c.num_attention_heads != 2 * c.num_key_value_heads) return false;
    if (!(bdims_match<1024, 2048, 3072>(c) || bdims_match<256, 512, 512>(c))) return false;
    if (!m.d_dec_layers_b) return false;
    if (c.num_hidden_layers > 32) return false;
    const int G = m.ctx->sm_count;
    if ((c.hidden_size + G - 1) / G > megab::MAXROWS) return false;
    const BatchCfg k = batch_cfg(std::min(B, 16));
    if (k.NB * c.num_key_value_heads > G) return false;                    // one merging CTA per (sequence, kv head)
    if ((ctx + k.KVK - 1) / k.KVK > megab::MAXSPLIT) return false;
    if (m.ctx->smem_optin < batch_smem_bytes(c.hidden_size, k)) return false;
    return true;
}

// floats of session scratch the batched step needs (tagged exchange buffers, 2 floats per word)
size_t decode_batch_part_floats(const Model& m) {
    const asrb_dims& c = m.d.c;
    const size_t NBm = 16;
    const size_t words = NBm * (size_t)m.d.qkv_dim + NBm * c.num_key_value_heads * megab::MAXSPLIT * 2 * mega::PSTRIDE + 64;
    return 2 * words + 64;
}
// bytes of the self-validating exchange words: 2 sets x layers x 16 sequences x (x after o_proj, x after down_proj, attention
// output, activations)
size_t decode_batch_sx_bytes(const Model& m) {
    const asrb_dims& c = m.d.c;
    return (size_t)2 * c.num_hidden_layers * 16 * ((size_t)2 * c.hidden_size + m.d.q_dim + c.intermediate_size) * 4;
}

// the instantiation for the model's dims, NB and the run's options: sampling (with or without the log-probability
// record) is never combined with the candidate lists
template <bool LP, bool TK, bool SM, bool RP>
static const void* batch_fn_dims(const asrb_dims& c, int NB) {
    if (bdims_match<1024, 2048, 3072>(c))
        return NB == 8 ? (const void*)megab::decode_batch_kernel<1024, 2048, 3072, 8, 5, 64, LP, TK, SM, RP>
                       : (const void*)megab::decode_batch_kernel<1024, 2048, 3072, 16, 3, 64, LP, TK, SM, RP>;
    return NB == 8 ? (const void*)megab::decode_batch_kernel<256, 512, 512, 8, 5, 64, LP, TK, SM, RP>
                   : (const void*)megab::decode_batch_kernel<256, 512, 512, 16, 3, 64, LP, TK, SM, RP>;
}
template <bool RP>
static const void* batch_fn(const DecodeBufs& b, const asrb_dims& c, int NB) {
    if (b.sample) return b.logprobs ? batch_fn_dims<true, false, true, RP>(c, NB) : batch_fn_dims<false, false, true, RP>(c, NB);
    if (b.topk) return batch_fn_dims<true, true, false, RP>(c, NB);
    if (b.logprobs) return batch_fn_dims<true, false, false, RP>(c, NB);
    return batch_fn_dims<false, false, false, RP>(c, NB);
}

void launch_decode_step_batch(const Model& m, const DecodeBufs& b, int B, float* kcache, float* vcache,
                              size_t cache_layer_stride, size_t cache_seq_stride, int max_ctx, int ctx_now, const MegaBufs& mb,
                              cudaStream_t st, int64_t* launches) {
    ASRB_REQUIRE(decode_batch_supported(m, B, ctx_now), ASRB_ERR_STATE, "batched fused decode step not supported for this model/batch/context");
    ASRB_REQUIRE(m.d_dec_layers_b && m.lm_head_b && mb.bar && mb.part && mb.sx, ASRB_ERR_STATE, "fused decode step buffers missing");
    const asrb_dims& c = m.d.c;
    const int G = m.ctx->sm_count;
    for (int b0 = 0; b0 < B; b0 += 16) {             // passes of up to 16 sequences (weights are streamed once per pass)
        const int nb = std::min(16, B - b0);
        const BatchCfg k = batch_cfg(nb);
        const size_t smem = batch_smem_bytes(c.hidden_size, k);
        const void* fn = b.rep ? batch_fn<true>(b, c, k.NB) : batch_fn<false>(b, c, k.NB);
        ASRB_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        megab::Params p{};
        p.layers = m.d_dec_layers_b; p.lm_head = m.lm_head_b; p.embed = m.embed; p.final_norm = m.final_norm;
        p.rope_cos = m.rope_cos; p.rope_sin = m.rope_sin; p.eps = (float)c.rms_norm_eps;
        p.L = c.num_hidden_layers; p.H = c.hidden_size; p.QD = m.d.q_dim; p.KVD = m.d.kv_dim; p.I = c.intermediate_size;
        p.V = c.vocab_size; p.nkv = c.num_key_value_heads; p.nb = nb;
        p.x = b.x + (size_t)b0 * c.hidden_size;
        p.kcache = kcache + (size_t)b0 * cache_seq_stride; p.vcache = vcache + (size_t)b0 * cache_seq_stride;
        p.cache_layer_stride = cache_layer_stride; p.cache_seq_stride = cache_seq_stride; p.max_ctx = max_ctx;
        p.part_val = b.part_val + (size_t)b0 * b.n_part; p.part_idx = b.part_idx + (size_t)b0 * b.n_part; p.n_part = b.n_part;
        p.pos = b.pos + b0; p.done = b.done + b0; p.next_id = b.next_id + b0;
        p.ids_out = b.ids_out + (size_t)b0 * b.max_new; p.n_out = b.n_out + b0; p.max_new = b.max_new;
        p.bar = mb.bar;
        uint2* w = reinterpret_cast<uint2*>(mb.part);            // 16-byte aligned sub-buffers (even word counts)
        p.qkv_ll = w; w += (size_t)16 * m.d.qkv_dim;
        p.part_ll = w;
        p.sx = mb.sx;
        if (mb.sx_nb && *mb.sx_nb != k.NB) {        // region layout depends on NB: re-arm everything when the instantiation changes
            ASRB_CUDA_CHECK(cudaMemsetAsync(mb.sx, 0xFF, mb.sx_bytes, st));
            *mb.sx_nb = k.NB;
        }
        p.dbg = mb.dbg;
        g_last_dbg_batch = mb.dbg;
        if (b.logprobs) {
            p.part_sum = b.part_sum + (size_t)b0 * b.n_part; p.lp_out = b.lp_out + (size_t)b0 * b.max_new; p.eos_lp = b.eos_lp + b0;
        }
        if (b.topk) {
            p.tk_part_val = b.tk_part_val + (size_t)b0 * b.n_part * TK_MAX; p.tk_part_idx = b.tk_part_idx + (size_t)b0 * b.n_part * TK_MAX;
            p.tk_ids = b.tk_ids + (size_t)b0 * b.max_new * TK_MAX; p.tk_lp = b.tk_lp + (size_t)b0 * b.max_new * TK_MAX;
            p.tk_eos_ids = b.tk_eos_ids + (size_t)b0 * TK_MAX; p.tk_eos_lp = b.tk_eos_lp + (size_t)b0 * TK_MAX;
        }
        if (b.sample) {                              // passes of 16: the draw's row is global
            p.smp = b.smp; p.row0 = b0;
            if (b.logprobs) { p.part_max = b.part_max + (size_t)b0 * b.n_part; p.part_sel = b.part_sel + (size_t)b0 * b.n_part; }
        }
        if (b.rep) { p.rep_bits = b.rep_mask; p.rep_words = rep_cta_words(c, G); p.rep = b.rep_params; }
        { static const int fl = getenv("ASRB_BATCH_FLAGS") ? atoi(getenv("ASRB_BATCH_FLAGS")) : 0; p.flags = fl; }   // bit 0 (K/V L2 prefetch): measured slower, off
        if (mb.steps_issued && ++*mb.steps_issued >= 0xFFFF00u) {   // tags must stay monotonic: wipe long before the epoch wraps
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

}  // namespace asrb
