// beam.cu -- beam search around the decode kernels' TOPK records (session option "beam_size" = K in 2..BEAM_MAX).
//
// Utterance b owns K slots: beam j lives in slot j*B + b (beam 0 is slot b, which holds the prefill).  Every decode path
// already writes, per slot and step, the exact TK_MAX best (id, log p) of the step into tk_ids / tk_lp (tk_eos_* when
// the top candidate is EOS).  Around that:
//   beam_step_kernel<true>   after the prefill: the token-0 walk on the single record, and the prompt expansion plan
//   beam_step_kernel<false>  after every decode step: the walk over the K beams' records and the slot assignment
//   beam_kv_copy_kernel      the KV copies those plans describe (positions after the last common ancestor only; the
//                            ids_out entries of the same positions are copied by beam_step_kernel<false>)
//   beam_finalize_kernel     backtracks the ranked hypotheses through the per-step history
// The walk (one thread; at most BEAM_MAX * (BEAM_MAX + 2) = 48 candidates):
//   candidates  the first K + 2 entries of each alive beam's record (at most two are EOS), sum = sum_parent + lp (fp32)
//   order       sum descending, parent rank ascending, position in the record ascending
//   walk        EOS -> newly finished, else the next alive beam; stop at K alive; then admit the newly finished in walk
//               order while the utterance has fewer than K finished hypotheses (K finished: the utterance is done)
//   slots       a parent's best-ranked child keeps the parent's slot; the other children take, in rank order, the slots
//               of childless beams in ascending slot order.  Sources (parents with children) and destinations
//               (childless slots) are disjoint, so the copies need no scratch and no ordering.
#include <algorithm>
#include "internal.h"

namespace asrb {

static constexpr int BEAM_THREADS = 64;     // >= BEAM_MAX * (BEAM_MAX + 2) candidates
static_assert(BEAM_MAX + 2 <= TK_MAX, "a beam's candidates come from its step's TK_MAX record");
static_assert(BEAM_MAX * (BEAM_MAX + 2) <= BEAM_THREADS, "one thread per candidate");

__device__ __forceinline__ bool is_eos(int id) { return id == 151643 || id == 151645; }

template <bool FIRST>
__global__ void __launch_bounds__(BEAM_THREADS) beam_step_kernel(BeamArgs a, const int* __restrict__ pos0) {
    __shared__ int c_id[BEAM_THREADS], c_par[BEAM_THREADS], order[BEAM_THREADS];
    __shared__ float c_lp[BEAM_THREADS], c_sum[BEAM_THREADS];
    __shared__ int new_slot[BEAM_MAX], new_tok[BEAM_MAX], s_live;
    const int b = blockIdx.x, tid = threadIdx.x, K = a.K, B = a.B, C = K + 2;
    BeamUtt& u = a.u[b];
    if constexpr (FIRST) {
        if (tid == 0) {
            u.t = 0; u.done = 0; u.nfin = 0; u.S = pos0[b] + 1; u.reassigned = 0; u.reorder_bytes = 0; u.expand_bytes = 0;
            // every slot of the utterance gets a valid position and count before anything else: a batched decode step
            // reads (and appends K/V at) the position of a done row whenever another row of its pass is alive, so a
            // slot of an utterance finished at token 0 must not keep one from an earlier run or from fresh memory
            for (int j = 0; j < K; ++j) { a.pos[j * B + b] = u.S; a.n_out[j * B + b] = 0; }
        }
        __syncthreads();
    }
    if (u.done) {                                  // finished at an earlier step: nothing to copy for its slots
        if (tid < K) a.cp_n[tid * B + b] = 0;
        return;
    }
    const int t = u.t;
    const int nparent = FIRST ? 1 : K, ncand = nparent * C;
    if (tid < ncand) {                             // candidate i = (parent rank i / C, record position i % C)
        const int r = tid / C, j = tid % C;
        const int slot = FIRST ? b : u.slot_of_rank[r];
        const bool eos_top = a.done[slot] != 0;    // the decode step saw EOS on top: the record is in the EOS rows
        const size_t o = eos_top ? (size_t)slot * TK_MAX + j : ((size_t)slot * a.max_new + t) * TK_MAX + j;
        const int id = eos_top ? a.tk_eos_ids[o] : a.tk_ids[o];
        const float lp = eos_top ? a.tk_eos_lp[o] : a.tk_lp[o];
        c_id[tid] = id; c_lp[tid] = lp; c_par[tid] = slot;
        c_sum[tid] = (FIRST ? 0.f : u.sum_of_rank[r]) + lp;
    }
    __syncthreads();
    if (tid < ncand) {                             // rank under the strict total order (sum desc, candidate index asc)
        const float s = c_sum[tid];
        int rank = 0;
        for (int i = 0; i < ncand; ++i) rank += (c_sum[i] > s || (c_sum[i] == s && i < tid)) ? 1 : 0;
        order[rank] = tid;
    }
    __syncthreads();
    if (tid == 0) {
        // the walk passes up to two EOS candidates per beam; only the first K - nfin of them can be admitted
        int alive[BEAM_MAX], nalive = 0, fresh[BEAM_MAX], nfresh = 0;
        const int room = K - u.nfin;
        for (int q = 0; q < ncand && nalive < K; ++q) {
            const int c = order[q];
            if (is_eos(c_id[c])) { if (nfresh < room) fresh[nfresh++] = c; }
            else alive[nalive++] = c;
        }
        for (int q = 0; q < nfresh; ++q) {                  // admission order = index in the finished list
            const int c = fresh[q], f = u.nfin++;
            u.fin_depth[f] = t - 1; u.fin_slot[f] = FIRST ? -1 : c_par[c];
            u.fin_eos[f] = c_id[c]; u.fin_eos_lp[f] = c_lp[c]; u.fin_sum[f] = c_sum[c];
        }
        if (u.nfin >= K) {                         // K finished hypotheses: the utterance is done
            u.done = 1;
            for (int j = 0; j < K; ++j) { const int s = j * B + b; a.done[s] = 1; a.next_id[s] = -1; a.cp_n[s] = 0; }
            s_live = 0;
        } else {
            // beam index of each new beam's parent; FIRST: every child's parent is beam 0
            int pj[BEAM_MAX], dst[BEAM_MAX];
            bool has_child[BEAM_MAX], claimed[BEAM_MAX];
            for (int j = 0; j < K; ++j) { has_child[j] = false; claimed[j] = false; }
            for (int r = 0; r < K; ++r) { pj[r] = FIRST ? 0 : (c_par[alive[r]] - b) / B; has_child[pj[r]] = true; }
            for (int r = 0; r < K; ++r) {
                dst[r] = -1;
                if (!claimed[pj[r]]) { dst[r] = pj[r]; claimed[pj[r]] = true; }
            }
            int next_free = 0;
            for (int r = 0; r < K; ++r) {
                if (dst[r] >= 0) continue;
                while (has_child[next_free]) ++next_free;
                dst[r] = next_free++;
            }
            int cp_old[BEAM_MAX][BEAM_MAX];
            for (int i = 0; i < K; ++i) for (int j = 0; j < K; ++j) cp_old[i][j] = u.cp[i][j];
            long long moved = 0, bytes = 0;
            for (int r = 0; r < K; ++r) {
                const int c = alive[r], j = dst[r], s = j * B + b, ps = pj[r] * B + b;
                int n = 0, p0 = 0;
                if (j != pj[r]) {
                    if (FIRST) { p0 = 0; n = u.S; }                 // the prompt, positions 0 .. S-1
                    else {                                         // positions after the last common ancestor
                        const int common = cp_old[j][pj[r]];
                        p0 = u.S + common + 1; n = t - 1 - common;
                        ++moved;
                    }
                }
                a.cp_src[s] = ps; a.cp_p0[s] = p0; a.cp_n[s] = n;
                bytes += (long long)n * (long long)a.bytes_per_pos;
                const size_t h = (size_t)t * a.ldh + s;
                a.hist_tok[h] = c_id[c]; a.hist_par[h] = FIRST ? -1 : ps; a.hist_lp[h] = c_lp[c];
                a.done[s] = 0; a.next_id[s] = c_id[c]; a.n_out[s] = t + 1; a.pos[s] = u.S + t;
                a.ids_out[(size_t)s * a.max_new + t] = c_id[c];
                u.slot_of_rank[r] = s; u.sum_of_rank[r] = c_sum[c];
                new_slot[r] = s; new_tok[r] = c_id[c];
            }
            for (int x = 0; x < K; ++x)            // children of one parent share the parent's node at depth t - 1
                for (int y = 0; y < K; ++y) {
                    int v = t;
                    if (x != y) v = pj[x] == pj[y] ? t - 1 : cp_old[pj[x]][pj[y]];
                    u.cp[dst[x]][dst[y]] = v;
                }
            if (FIRST) u.expand_bytes = bytes;
            else { u.reassigned += moved; u.reorder_bytes += bytes; }
            u.t = t + 1;
            s_live = 1;
        }
    }
    __syncthreads();
    if (!s_live) {
        if constexpr (FIRST)                       // done at token 0: a defined residual stream for the done slots
            for (int j = 0; j < K; ++j)
                for (int i = tid; i < a.hidden; i += BEAM_THREADS) a.x[(size_t)(j * B + b) * a.hidden + i] = 0.f;
        return;
    }
    if constexpr (!FIRST)                          // a reassigned slot takes its new lineage's ids with its K/V: the same
        for (int r = 0; r < K; ++r) {              // positions, ids[common + 1 .. t - 1] (the repetition controls' history)
            const int s = new_slot[r], n = a.cp_n[s], i0 = a.cp_p0[s] - u.S;
            const int* src = a.ids_out + (size_t)a.cp_src[s] * a.max_new + i0;
            int* dst = a.ids_out + (size_t)s * a.max_new + i0;
            for (int i = tid; i < n; i += BEAM_THREADS) dst[i] = src[i];
        }
    for (int r = 0; r < K; ++r) {                  // the next token's embedding (text_decoder.rs:90-92)
        const bf16* e = a.embed + (size_t)new_tok[r] * a.hidden;
        float* xr = a.x + (size_t)new_slot[r] * a.hidden;
        for (int i = tid; i < a.hidden; i += BEAM_THREADS) xr[i] = __bfloat162float(e[i]);
    }
}

// grid (slots, layers * kv heads): slot s receives positions [p0, p0 + n) of every (layer, kv head) from slot src,
// K and V, 16 bytes per load
__global__ void __launch_bounds__(256) beam_kv_copy_kernel(float* __restrict__ kcache, float* __restrict__ vcache,
                                                           const int* __restrict__ cp_src, const int* __restrict__ cp_p0,
                                                           const int* __restrict__ cp_n, int nkv, int hd, int max_ctx,
                                                           size_t layer_stride, size_t seq_stride) {
    const int s = blockIdx.x, n = cp_n[s];
    if (n <= 0) return;
    const int l = blockIdx.y / nkv, g = blockIdx.y % nkv;
    const size_t head = (size_t)l * layer_stride + (size_t)g * max_ctx * hd + (size_t)cp_p0[s] * hd;
    const size_t dst = head + (size_t)s * seq_stride, src = head + (size_t)cp_src[s] * seq_stride;
    const float4* ks = reinterpret_cast<const float4*>(kcache + src);
    const float4* vs = reinterpret_cast<const float4*>(vcache + src);
    float4* kd = reinterpret_cast<float4*>(kcache + dst);
    float4* vd = reinterpret_cast<float4*>(vcache + dst);
    const int count = n * hd / 4;
    for (int i = threadIdx.x; i < count; i += blockDim.x) { kd[i] = ks[i]; vd[i] = vs[i]; }
}

// grid B, one thread per hypothesis: hypothesis k of utterance b (ranked on the host) ends at node (depth, slot) of the
// history; its ids / log-probabilities go to nb_ids / nb_lp [b][k][max_new], and rank 0 also to the result rows b of
// ids_out / lp_out (NaN beyond its length) / n_out / eos_lp
__global__ void beam_finalize_kernel(BeamArgs a, const int* __restrict__ hyp /* [B][K][2] depth, slot */,
                                     const float* __restrict__ best_eos_lp /* [B] */) {
    const int b = blockIdx.x, k = threadIdx.x, K = a.K;
    if (k >= K) return;
    const int depth = hyp[((size_t)b * K + k) * 2], slot = hyp[((size_t)b * K + k) * 2 + 1];
    int* ids = a.nb_ids + ((size_t)b * K + k) * a.max_new;
    float* lps = a.nb_lp + ((size_t)b * K + k) * a.max_new;
    int s = slot;
    for (int d = depth; d >= 0; --d) {
        const size_t h = (size_t)d * a.ldh + s;
        ids[d] = a.hist_tok[h]; lps[d] = a.hist_lp[h]; s = a.hist_par[h];
    }
    if (k != 0) return;
    const float nan = __int_as_float(0x7fffffff);
    for (int d = 0; d < a.max_new; ++d) {
        if (d <= depth) a.ids_out[(size_t)b * a.max_new + d] = ids[d];
        if (a.lp_out) a.lp_out[(size_t)b * a.max_new + d] = d <= depth ? lps[d] : nan;
    }
    a.n_out[b] = depth + 1;
    if (a.eos_lp) a.eos_lp[b] = best_eos_lp[b];
}

void launch_beam_step(const BeamArgs& a, bool first, const int* pos0, cudaStream_t st, int64_t* launches) {
    if (first) beam_step_kernel<true><<<a.B, BEAM_THREADS, 0, st>>>(a, pos0);
    else beam_step_kernel<false><<<a.B, BEAM_THREADS, 0, st>>>(a, nullptr);
    ASRB_CUDA_CHECK(cudaGetLastError());
    const dim3 grid(a.B * a.K, a.layers * a.nkv);
    beam_kv_copy_kernel<<<grid, 256, 0, st>>>(a.kcache, a.vcache, a.cp_src, a.cp_p0, a.cp_n, a.nkv, a.head_dim, a.max_ctx,
                                              a.layer_stride, a.seq_stride);
    ASRB_CUDA_CHECK(cudaGetLastError());
    if (launches) *launches += 2;
}

void launch_beam_finalize(const BeamArgs& a, const int* hyp, const float* best_eos_lp, cudaStream_t st, int64_t* launches) {
    beam_finalize_kernel<<<a.B, 32, 0, st>>>(a, hyp, best_eos_lp);
    ASRB_CUDA_CHECK(cudaGetLastError());
    if (launches) *launches += 1;
}

}  // namespace asrb
