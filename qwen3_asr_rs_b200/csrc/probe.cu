// probe.cu -- kernel-level entry points for tests (csrc/probe.h): the library's split3, norm, GEMM and attention
// launchers run on host arrays, so that each kernel can be compared with a float64 reference of the same operation at
// shapes chosen for it.  Nothing here is on the inference path.
#include <algorithm>
#include <functional>
#include <vector>
#include "internal.h"
#include "probe.h"

namespace asrb {
int run_guarded(const std::function<void()>& f);                           // c_api.cu
bool launch_attention_f32(const AttnParams& p, int hd, cudaStream_t st);   // attention_f32.cu (the default kernel)

namespace {

// device buffers and a stream of the probe's own, released on every exit
struct Scope {
    cudaStream_t st = nullptr;
    std::vector<void*> bufs;
    Scope() { ASRB_CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)); }
    ~Scope() {
        if (st) cudaStreamSynchronize(st);
        for (void* p : bufs) cudaFree(p);
        if (st) cudaStreamDestroy(st);
    }
    template <typename T> T* alloc(size_t n, int fill_byte = 0) {
        void* p = nullptr;
        ASRB_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
        bufs.push_back(p);
        ASRB_CUDA_CHECK(cudaMemsetAsync(p, fill_byte, std::max<size_t>(n, 1) * sizeof(T), st));
        return static_cast<T*>(p);
    }
    template <typename T> T* upload(const T* h, size_t n) {
        T* d = alloc<T>(n);
        if (h && n) ASRB_CUDA_CHECK(cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, st));
        return d;
    }
    template <typename T> void download(T* h, const T* d, size_t n) {
        if (n) ASRB_CUDA_CHECK(cudaMemcpyAsync(h, d, n * sizeof(T), cudaMemcpyDeviceToHost, st));
    }
    void sync() { ASRB_CUDA_CHECK(cudaStreamSynchronize(st)); ASRB_CUDA_CHECK(cudaGetLastError()); }
};

__global__ void split3_kernel(const float* __restrict__ x, size_t n, bf16* __restrict__ out, size_t plane_stride) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        store_split3(out, plane_stride, i, x[i]);
}
void split3_planes(Scope& s, const float* d_x, size_t n, bf16* d_out, size_t plane_stride) {
    if (n == 0) return;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
    split3_kernel<<<blocks, 256, 0, s.st>>>(d_x, n, d_out, plane_stride);
    ASRB_CUDA_CHECK(cudaGetLastError());
}

int device_sms() {
    int dev = 0, n = 0;
    ASRB_CUDA_CHECK(cudaGetDevice(&dev));
    ASRB_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    return n;
}

void write_plan(const GemmPlan& p, int* out) {
    const int items = p.tiles_m * p.tiles_n * p.splits;
    out[0] = p.tc ? 1 : 0; out[1] = p.splits; out[2] = p.tiles_m; out[3] = p.tiles_n; out[4] = p.grid;
    out[5] = p.grid > 0 ? (items + p.grid - 1) / p.grid : 0; out[6] = 0; out[7] = p.box_h;
}

GemmA plan_operand(int M, int K, int a_mode, int OH, int OW, int cpad, size_t plane_stride) {
    GemmA A; A.mode = a_mode; A.M = M; A.K = K; A.lda = K; A.nplanes = 3; A.plane_stride = plane_stride;
    A.OH = OH; A.OW = OW; A.Hh = OH; A.Wh = OW; A.cpad = cpad;
    return A;
}
size_t round8(size_t n) { return (n + 7) / 8 * 8; }

void write_score_plan(const ScoreHeadPlan& p, int* out) {
    const int items = p.tiles_m * p.nslices;
    int lo = p.tiles_n, hi = 0;
    for (int s = 0; s < p.nslices; ++s) {   // slice s covers tiles [s * tiles_n / nslices, (s + 1) * tiles_n / nslices)
        const int w = (int)((long long)(s + 1) * p.tiles_n / p.nslices - (long long)s * p.tiles_n / p.nslices);
        lo = std::min(lo, w); hi = std::max(hi, w);
    }
    out[0] = p.tiles_m; out[1] = p.tiles_n; out[2] = p.nslices; out[3] = p.grid;
    out[4] = (items + p.grid - 1) / p.grid; out[5] = lo; out[6] = hi;
}

void check_score_dims(int rows, int V, int H, int grid_cap) {
    ASRB_REQUIRE(rows >= 1 && V >= 1 && H > 0 && H % 64 == 0 && grid_cap >= 0, ASRB_ERR_INVALID,
                 "asrbt_score: rows >= 1, V >= 1, H % 64 == 0 and grid_cap >= 0");
}

}  // namespace
}  // namespace asrb

using namespace asrb;

extern "C" {

int asrbt_split3(const float* x, int64_t n, uint16_t* planes_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(x && planes_out && n >= 0, ASRB_ERR_INVALID, "asrbt_split3: bad arguments");
        Scope s;
        float* d_x = s.upload(x, (size_t)n);
        bf16* d_p = s.alloc<bf16>(3 * (size_t)n);
        split3_planes(s, d_x, (size_t)n, d_p, (size_t)n);
        s.download(planes_out, reinterpret_cast<const uint16_t*>(d_p), 3 * (size_t)n);
        s.sync();
    });
}

int asrbt_norm_s3(int kind, const float* x, const float* w, const float* b, int rows, int dim, float eps, uint16_t* planes_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(x && w && planes_out && rows > 0 && dim > 0 && (kind == 1 || b), ASRB_ERR_INVALID, "asrbt_norm_s3: bad arguments");
        ASRB_REQUIRE(kind == 0 || kind == 1, ASRB_ERR_INVALID, "asrbt_norm_s3: kind is 0 (LayerNorm) or 1 (RMSNorm)");
        Scope s;
        const size_t n = (size_t)rows * dim;
        const float* d_x = s.upload(x, n);
        const float* d_w = s.upload(w, (size_t)dim);
        bf16* d_p = s.alloc<bf16>(3 * n);
        if (kind == 0) launch_layernorm_s3(d_x, d_w, s.upload(b, (size_t)dim), rows, dim, eps, d_p, n, s.st);
        else launch_rmsnorm_s3(d_x, d_w, rows, dim, eps, d_p, n, s.st);
        s.download(planes_out, reinterpret_cast<const uint16_t*>(d_p), 3 * n);
        s.sync();
    });
}

int asrbt_gemm_plan(int M, int N, int K, int a_mode, int epi, int sms, int use_splitk, int OH, int OW, int cpad, int* plan_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(plan_out && sms > 0, ASRB_ERR_INVALID, "asrbt_gemm_plan: bad arguments");
        GemmEpi E; E.mode = epi;
        E.splitk_ws = use_splitk ? reinterpret_cast<float*>(16) : nullptr;   // only its presence is read
        write_plan(plan_gemm_tc(plan_operand(M, K, a_mode, OH, OW, cpad, round8((size_t)M * K)), N, E, sms), plan_out);
    });
}

int asrbt_gemm(const asrbt_gemm_args* a, int* plan_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(a && plan_out && a->x && a->w && a->M > 0 && a->N > 0 && a->K > 0, ASRB_ERR_INVALID, "asrbt_gemm: bad arguments");
        ASRB_REQUIRE(a->out_f32 || a->out_planes, ASRB_ERR_INVALID, "asrbt_gemm: no output");
        ASRB_REQUIRE(a->nplanes >= 1 && a->nplanes <= 3, ASRB_ERR_INVALID, "asrbt_gemm: nplanes is 1..3");
        Scope s;
        // ---- A operand: split3 planes, plain rows or the conv parity layout ----
        GemmA A; A.mode = a->a_mode; A.M = a->M; A.K = a->K; A.lda = a->K; A.nplanes = a->nplanes;
        size_t n_act;
        std::vector<float> lay;
        const float* host_act = a->x;
        if (a->a_mode == A_PLAIN) {
            n_act = (size_t)a->M * a->K;
        } else {
            ASRB_REQUIRE(a->OH > 0 && a->OW > 0 && a->Hh > 0 && a->Wh > 0 && a->cpad > 0 && a->K == 9 * a->cpad &&
                             a->M % (a->OH * a->OW) == 0, ASRB_ERR_INVALID, "asrbt_gemm: bad conv geometry");
            A.OH = a->OH; A.OW = a->OW; A.Hh = a->Hh; A.Wh = a->Wh; A.cpad = a->cpad;
            const int chunks = a->M / (a->OH * a->OW), H = 2 * a->Hh, W = 2 * a->Wh;
            n_act = (size_t)chunks * 4 * a->Hh * a->Wh * a->cpad;
            lay.assign(n_act, 0.f);
            for (int ch = 0; ch < chunks; ++ch)
                for (int h = 0; h < H; ++h)
                    for (int w = 0; w < W; ++w) {
                        const size_t dst = ((((size_t)ch * 2 + (h & 1)) * 2 + (w & 1)) * a->Hh + (h >> 1)) * a->Wh + (w >> 1);
                        const float* src = a->x + (((size_t)ch * H + h) * W + w) * a->cpad;
                        std::copy(src, src + a->cpad, lay.begin() + dst * a->cpad);
                    }
            host_act = lay.data();
        }
        A.plane_stride = round8(n_act);
        const float* d_x = s.upload(host_act, n_act);
        bf16* d_a = s.alloc<bf16>(3 * A.plane_stride);
        split3_planes(s, d_x, n_act, d_a, A.plane_stride);
        A.a = d_a;
        const bf16* d_w = reinterpret_cast<const bf16*>(s.upload(a->w, (size_t)a->N * a->K));
        // ---- epilogue ----
        GemmEpi E; E.mode = a->epi; E.act = a->gelu;
        if (a->bias) E.bias = s.upload(a->bias, (size_t)a->N);
        float* d_out = nullptr;
        const size_t n_out = a->out_f32 ? (size_t)a->out_f32_rows * a->ldo : 0;
        if (a->out_f32) {
            d_out = s.alloc<float>(n_out, 0xff);                          // NaN: an element never written reads non-finite
            if (a->residual) {                                            // in place, x += proj(...), as the session does
                ASRB_REQUIRE(a->out_f32_rows == a->M, ASRB_ERR_INVALID, "asrbt_gemm: residual rows");
                ASRB_CUDA_CHECK(cudaMemcpyAsync(d_out, a->residual, n_out * sizeof(float), cudaMemcpyHostToDevice, s.st));
                E.residual = d_out; E.ldr = a->ldo;
            }
            E.out_f32 = d_out; E.ldo = a->ldo;
        }
        bf16* d_planes = nullptr;
        if (a->out_planes) {
            d_planes = s.alloc<bf16>(3 * (size_t)a->out_plane_elems);     // zero: the parity layout's unwritten padding
            E.out_s3 = d_planes; E.s3_plane_stride = (size_t)a->out_plane_elems; E.lds = a->lds;
        }
        E.OH = a->OH; E.OW = a->OW; E.Hh2 = a->Hh2; E.Wh2 = a->Wh2; E.cpad = a->cpad2;
        if (a->row_map) E.row_map = s.upload(a->row_map, (size_t)a->M);
        if (a->pos) { E.pos = s.upload(a->pos, (size_t)a->pos_period * a->N); E.pos_period = a->pos_period; }
        if (a->use_splitk) E.splitk_ws = s.alloc<float>(SPLITK_WS_FLOATS);
        int64_t extra = 0;
        E.extra_launches = &extra;
        // ---- run ----
        const int64_t fb0 = g_gemm_simt_fallbacks.load();
        launch_gemm(A, d_w, a->N, E, a->impl == 1 ? GEMM_TC : GEMM_SIMT, s.st);
        s.sync();
        const int64_t fb = g_gemm_simt_fallbacks.load() - fb0;
        if (a->impl == 1 && fb == 0) {
            const GemmPlan p = plan_gemm_tc(A, a->N, E, device_sms());
            ASRB_REQUIRE(extra == (p.splits > 1 ? 1 : 0), ASRB_ERR_STATE, "asrbt_gemm: launches differ from the plan");
            write_plan(p, plan_out);
        } else {
            GemmPlan p; p.tiles_m = (a->M + 63) / 64; p.tiles_n = (a->N + 63) / 64; p.grid = p.tiles_m * p.tiles_n;
            write_plan(p, plan_out);                                      // SIMT: one 64 x 64 tile per CTA
        }
        plan_out[6] = (int)fb;
        if (a->out_f32) s.download(a->out_f32, d_out, n_out);
        if (a->out_planes) s.download(a->out_planes, reinterpret_cast<const uint16_t*>(d_planes), 3 * (size_t)a->out_plane_elems);
        s.sync();
    });
}

int asrbt_attention(const asrbt_attn_args* a) {
    return run_guarded([&] {
        ASRB_REQUIRE(a && a->buf && a->seg_q0 && a->seg_len && a->out_planes && a->nseg > 0, ASRB_ERR_INVALID,
                     "asrbt_attention: bad arguments");
        Scope s;
        const float* d_buf = s.upload(a->buf, (size_t)a->buf_elems);
        AttnParams p{};
        p.q = d_buf + a->q_off; p.ldq = a->ldq;
        p.k = d_buf + a->k_off; p.v = d_buf + a->v_off; p.ldk = a->ldk;
        p.seg_stride = (size_t)a->seg_stride; p.head_stride = (size_t)a->head_stride;
        p.seg_q0 = s.upload(a->seg_q0, (size_t)a->nseg); p.seg_len = s.upload(a->seg_len, (size_t)a->nseg);
        p.seg_pos0 = a->seg_pos0 ? s.upload(a->seg_pos0, (size_t)a->nseg) : nullptr;
        p.keys_in_rows = a->keys_in_rows; p.nseg = a->nseg; p.nheads = a->nheads; p.group = a->group;
        p.causal = a->causal; p.max_len = a->max_len;
        const size_t n_out = (size_t)a->out_rows * a->ldo;
        bf16* d_planes = s.alloc<bf16>(3 * n_out, 0xff);                  // NaN: a row never written reads non-finite
        p.out_s3 = d_planes; p.plane_stride = n_out; p.ldo = a->ldo;
        ASRB_REQUIRE(launch_attention_f32(p, a->hd, s.st), ASRB_ERR_INVALID, "asrbt_attention: the fp32 attention kernel declined the shape");
        s.download(a->out_planes, reinterpret_cast<const uint16_t*>(d_planes), 3 * n_out);
        s.sync();
    });
}

int asrbt_dtw(const float* M, int N, int T, int32_t* start_tok_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(M && start_tok_out && N >= 1 && T >= 1, ASRB_ERR_INVALID, "asrbt_dtw: bad arguments");
        int dev = 0;
        ASRB_CUDA_CHECK(cudaGetDevice(&dev));
        int optin = 0;
        ASRB_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        const bool in_smem = align_dtw_smem(N, T, true) <= (size_t)optin;
        const size_t smem = align_dtw_smem(N, T, in_smem);
        ASRB_REQUIRE(smem <= (size_t)optin, ASRB_ERR_INVALID, "asrbt_dtw: N too large for the DTW kernel");
        Scope s;
        const int h_int[4] = {N, T, in_smem ? 1 : 0, 0};
        const long long h_ll[2] = {0, 0};
        const int* d_int = s.upload(h_int, 4);
        const long long* d_ll = s.upload(h_ll, 2);
        AlignDtwArgs a{};
        a.N = d_int; a.T = d_int + 1; a.smem_trace = d_int + 2; a.soff = d_int + 3; a.moff = d_ll; a.toff = d_ll + 1;
        a.M = s.upload(M, (size_t)N * T);
        a.trace = s.alloc<uint32_t>(in_smem ? 1 : ((size_t)N * T + 15) / 16);
        int* d_start = s.alloc<int>((size_t)N, 0xff);
        a.start = d_start;
        launch_align_dtw(a, 1, smem, s.st);
        s.download(start_tok_out, d_start, (size_t)N);
        s.sync();
    });
}

int asrbt_score_plan(int rows, int V, int H, int sms, int grid_cap, int* plan_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(plan_out && sms > 0, ASRB_ERR_INVALID, "asrbt_score_plan: bad arguments");
        check_score_dims(rows, V, H, grid_cap);
        write_score_plan(plan_score_head(rows, V, sms, grid_cap), plan_out);
    });
}

int asrbt_score_head(const asrbt_score_args* a, int* plan_out) {
    return run_guarded([&] {
        ASRB_REQUIRE(a && plan_out && a->hid && a->norm_w && a->lm_head && a->target && a->lp_out, ASRB_ERR_INVALID,
                     "asrbt_score_head: bad arguments");
        check_score_dims(a->rows, a->V, a->H, a->grid_cap);
        ASRB_REQUIRE(a->nplanes >= 1 && a->nplanes <= 3 && (a->topk == 0 || a->topk == 1), ASRB_ERR_INVALID,
                     "asrbt_score_head: nplanes is 1..3, topk 0 or 1");
        ASRB_REQUIRE(!a->topk || (a->tk_ids_out && a->tk_lp_out), ASRB_ERR_INVALID, "asrbt_score_head: no top-k output");
        ASRB_REQUIRE(a->src ? a->n_hid >= 1 : a->n_hid == a->rows, ASRB_ERR_INVALID, "asrbt_score_head: bad n_hid");
        std::vector<int> src(a->rows);
        for (int r = 0; r < a->rows; ++r) {
            src[r] = a->src ? a->src[r] : r;
            ASRB_REQUIRE(src[r] >= 0 && src[r] < a->n_hid, ASRB_ERR_INVALID, "asrbt_score_head: src out of range");
            ASRB_REQUIRE(a->target[r] >= 0 && a->target[r] < a->V, ASRB_ERR_INVALID, "asrbt_score_head: target out of range");
        }
        Scope s;
        const int rows = a->rows, H = a->H, V = a->V;
        const float* d_hid = s.upload(a->hid, (size_t)a->n_hid * H);
        const int* d_src = s.upload(src.data(), (size_t)rows);
        const int* d_tgt = s.upload(a->target, (size_t)rows);
        const float* d_w = s.upload(a->norm_w, (size_t)H);
        const bf16* d_head = reinterpret_cast<const bf16*>(s.upload(a->lm_head, (size_t)V * H));
        const size_t plane_stride = round8((size_t)rows * H);
        float* d_gathered = s.alloc<float>((size_t)rows * H);
        bf16* d_planes = s.alloc<bf16>(3 * plane_stride);
        const ScoreHeadPlan p = plan_score_head(rows, V, device_sms(), a->grid_cap);
        ScorePart* d_part = s.alloc<ScorePart>((size_t)rows * p.nslices, 0xff);   // NaN: a partial never written
        float* d_lp = s.alloc<float>((size_t)rows, 0xff);
        int* d_tki = a->topk ? s.alloc<int>((size_t)rows * TK_MAX, 0xff) : nullptr;
        float* d_tkl = a->topk ? s.alloc<float>((size_t)rows * TK_MAX, 0xff) : nullptr;
        launch_score_head(d_head, d_w, H, V, a->eps, device_sms(), a->grid_cap, d_hid, d_src, d_tgt, rows, d_gathered,
                          d_planes, plane_stride, a->nplanes, d_part, a->topk != 0, d_lp, d_tki, d_tkl, s.st, nullptr);
        write_score_plan(p, plan_out);
        s.download(a->lp_out, d_lp, (size_t)rows);
        if (a->topk) {
            s.download(a->tk_ids_out, d_tki, (size_t)rows * TK_MAX);
            s.download(a->tk_lp_out, d_tkl, (size_t)rows * TK_MAX);
        }
        s.sync();
    });
}

int asrbt_align(const asrbt_align_args* a) {
    return run_guarded([&] {
        ASRB_REQUIRE(a && a->heads && a->qrow0 && a->N && a->T && a->a0 && a->slot && a->q && a->k && a->P_out &&
                         a->Z_out && a->M_out, ASRB_ERR_INVALID, "asrbt_align: bad arguments");
        ASRB_REQUIRE(a->B >= 1 && a->hd >= 1 && a->group >= 1 && a->nheads >= 1 && a->count >= 0 && a->ldq >= 1 &&
                         a->q_rows >= 1 && a->k_elems >= 1 && a->seg_stride >= 0 && a->head_stride >= 0,
                     ASRB_ERR_INVALID, "asrbt_align: bad dims");
        ASRB_REQUIRE(align_probs_smem(a->hd) <= ALIGN_PROBS_SMEM_MAX, ASRB_ERR_INVALID, "asrbt_align: head_dim too large");
        int maxG = 0;
        for (int i = 0; i < a->nheads; ++i) {
            ASRB_REQUIRE(a->heads[i] >= 0 && (int64_t)(a->heads[i] + 1) * a->hd <= a->ldq, ASRB_ERR_INVALID,
                         "asrbt_align: head outside the q row");
            maxG = std::max(maxG, a->heads[i] / a->group);
        }
        std::vector<long long> moff(a->B);
        long long total = 0;
        int maxN = 0, maxT = 0, maxNT = 0;
        for (int b = 0; b < a->B; ++b) {
            const int N = a->N[b], T = a->T[b];
            ASRB_REQUIRE(N >= 1 && T >= 1 && (int64_t)N * T <= INT32_MAX && a->qrow0[b] >= 0 && a->a0[b] >= 0 && a->slot[b] >= 0,
                         ASRB_ERR_INVALID, "asrbt_align: bad utterance");
            ASRB_REQUIRE((int64_t)a->qrow0[b] + N <= a->q_rows, ASRB_ERR_INVALID, "asrbt_align: q rows out of range");
            ASRB_REQUIRE(a->slot[b] * a->seg_stride + (int64_t)maxG * a->head_stride + ((int64_t)a->a0[b] + T) * a->hd <= a->k_elems,
                         ASRB_ERR_INVALID, "asrbt_align: keys out of range");
            moff[b] = total; total += (long long)N * T;
            maxN = std::max(maxN, N); maxT = std::max(maxT, T); maxNT = std::max(maxNT, N * T);
        }
        Scope s;
        const size_t plane = (size_t)total, nP = (size_t)a->nheads * plane;
        std::vector<int> ints;
        for (const int* v : {a->qrow0, a->N, a->T, a->a0, a->slot}) ints.insert(ints.end(), v, v + a->B);
        ints.insert(ints.end(), a->heads, a->heads + a->nheads);
        const int* d_int = s.upload(ints.data(), ints.size());
        const long long* d_moff = s.upload(moff.data(), moff.size());
        AlignProbArgs pa{};
        pa.q = s.upload(a->q, (size_t)a->q_rows * a->ldq); pa.ldq = a->ldq;
        pa.k = s.upload(a->k, (size_t)a->k_elems); pa.seg_stride = (size_t)a->seg_stride; pa.head_stride = (size_t)a->head_stride;
        pa.hd = a->hd; pa.group = a->group;
        pa.qrow0 = d_int; pa.N = d_int + a->B; pa.T = d_int + 2 * a->B; pa.a0 = d_int + 3 * a->B; pa.slot = d_int + 4 * a->B;
        pa.moff = d_moff; pa.heads = d_int + 5 * a->B; pa.nheads = a->nheads;
        pa.P = s.alloc<float>(nP, 0xff); pa.plane = plane;                  // NaN: an element never written
        float* d_M = a->M_in ? s.upload(a->M_in, plane) : s.alloc<float>(plane);
        launch_align_probs(pa, a->B, maxN, s.st);
        s.download(a->P_out, pa.P, nP);
        AlignFoldArgs fa{};
        fa.N = pa.N; fa.T = pa.T; fa.moff = d_moff; fa.P = pa.P; fa.plane = plane; fa.nheads = a->nheads; fa.M = d_M;
        fa.count = a->count;
        launch_align_fold(fa, a->B, maxT, maxNT, s.st);
        s.download(a->Z_out, pa.P, nP);
        s.download(a->M_out, d_M, plane);
        s.sync();
    });
}

}  // extern "C"
