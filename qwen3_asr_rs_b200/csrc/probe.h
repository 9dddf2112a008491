/* probe.h -- kernel-level entry points for tests (not part of the ABI in include/asr_b200.h).
 *
 * Each probe runs one of the library's own launchers on host arrays: it allocates its device buffers, runs on a
 * stream of its own, synchronises, copies the results back and frees everything.  Status and message follow the
 * library's convention (ASRB_OK / ASRB_ERR_*, asrb_last_error()).  bf16 values cross as raw uint16 bits; split3
 * outputs are three planes of n values each, hi first.  asrbt_gemm_plan and asrbt_score_plan need no GPU.
 */
#ifndef ASR_B200_PROBE_H
#define ASR_B200_PROBE_H
#include <stdint.h>
#include "../../include/asr_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* GEMM path report: [0] 1 = the wgmma kernel ran, 0 = the SIMT kernel; [1] k-split factor; [2] tiles_m; [3] tiles_n;
 * [4] persistent grid; [5] most work items any CTA took (ceil(tiles * splits / grid)); [6] SIMT fall-backs this call
 * added (a tensor-core request the wgmma kernel declined); [7] conv box height (output rows per tile, A_CONV) */
#define ASRBT_PLAN_LEN 8

typedef struct {
    int impl;                  /* 0 = SIMT GEMM, 1 = tensor-core (wgmma) GEMM requested */
    int a_mode;                /* 0 = plain rows [M][K], 1 = 3x3 / stride 2 / pad 1 conv taps */
    int epi;                   /* 0 PLAIN, 1 SWIGLU, 2 CONV_PARITY, 3 CONV_FEAT, 4 CONVOUT */
    int M, N, K, nplanes;      /* nplanes 1..3 of the split3 activation reach the GEMM */
    /* activation: plain: x[M][K]; conv: x[chunks][2 Hh][2 Wh][cpad] channels-last (chunks = M / (OH * OW)), laid out
     * by the probe in the parity-split layout the kernels read; zero entries of x are the right / bottom padding */
    const float* x;
    int OH, OW, Hh, Wh, cpad;
    const uint16_t* w;         /* bf16 bits [N][K] */
    const float* bias;         /* [N] or null (required by the conv epilogues) */
    int gelu;                  /* EPI_PLAIN: exact-erf GELU after the bias */
    const float* residual;     /* EPI_PLAIN: [M][ldo] added in place (out_f32 starts as a copy of it), or null */
    const int* row_map;        /* EPI_CONVOUT: [M] -> output row or -1 */
    const float* pos;          /* EPI_CONVOUT: [pos_period][N] */
    int pos_period;
    int use_splitk;            /* 1: give the GEMM the split-K workspace, as the session does for PLAIN / CONVOUT */
    float* out_f32; int64_t out_f32_rows; int ldo;          /* fp32 output rows (null: none) */
    uint16_t* out_planes; int64_t out_plane_elems; int lds; /* split3 output, 3 x out_plane_elems (null: none) */
    int Hh2, Wh2, cpad2;       /* EPI_CONV_PARITY: the next conv's parity layout */
} asrbt_gemm_args;

typedef struct {
    int hd, nseg, nheads, group, causal, keys_in_rows, max_len;
    const int* seg_q0; const int* seg_len; const int* seg_pos0;   /* [nseg]; seg_pos0 null: no query offset */
    const float* buf; int64_t buf_elems;                          /* one fp32 buffer holding q, k and v */
    int64_t q_off, k_off, v_off;                                  /* element offsets of q, k and v in buf */
    int ldq, ldk; int64_t seg_stride, head_stride;                /* as AttnParams */
    uint16_t* out_planes; int64_t out_rows; int ldo;              /* split3 output, 3 x out_rows * ldo */
} asrbt_attn_args;

/* score head plan (csrc/score.cu): [0] tiles_m; [1] tiles_n (128-column lm_head tiles); [2] column slices; [3]
 * persistent grid; [4] most (M tile, slice) items any CTA takes; [5] / [6] narrowest / widest slice in tiles */
#define ASRBT_SCORE_PLAN_LEN 7

typedef struct {
    int rows, n_hid, H, V;     /* scored rows, pre-norm rows in hid, hidden size (% 64 == 0), vocabulary */
    const float* hid;          /* [n_hid][H] pre-norm rows */
    const int* src;            /* [rows] row r scores hid[src[r]]; null: identity (n_hid == rows) */
    const float* norm_w;       /* [H] final RMSNorm weight */
    float eps;
    const uint16_t* lm_head;   /* bf16 bits [V][H] */
    const int* target;         /* [rows] ids in [0, V) */
    int nplanes;               /* 1..3 split3 planes of the normed rows reach the GEMM (3 in production) */
    int topk;                  /* 1: also the 8 best of every row */
    int grid_cap;              /* 0: the launcher's grid; > 0: at most this many CTAs */
    float* lp_out;             /* [rows] log p(target) */
    int32_t* tk_ids_out;       /* [rows][8] with topk (else ignored) */
    float* tk_lp_out;          /* [rows][8] */
} asrbt_score_args;

typedef struct {
    int B, hd, group, nheads, count;   /* utterances; head_dim; query heads per kv head; listed heads; > 0: divide M */
    const int* heads;                  /* [nheads] query heads of the layer, list order */
    const int *qrow0, *N, *T, *a0, *slot;   /* [B] first q row, aligned rows, audio keys, first audio position, KV slot */
    const float* q; int64_t q_rows; int ldq;                  /* [q_rows][ldq] post-RoPE q rows, head h at h * hd */
    const float* k; int64_t k_elems, seg_stride, head_stride; /* one layer's K cache: slot, kv head, position, d */
    const float* M_in;                 /* [sum N T] incoming running sum (null: zeros) */
    float* P_out;                      /* [nheads][sum N T] probabilities, before the fold */
    float* Z_out;                      /* [nheads][sum N T] z-scores */
    float* M_out;                      /* [sum N T] the updated running sum (the mean when count > 0) */
} asrbt_align_args;

ASRB_API int asrbt_split3(const float* x, int64_t n, uint16_t* planes_out);
/* kind 0 = LayerNorm (w, b), 1 = RMSNorm (w; b ignored): x[rows][dim] -> split3 planes of rows * dim */
ASRB_API int asrbt_norm_s3(int kind, const float* x, const float* w, const float* b, int rows, int dim, float eps,
                           uint16_t* planes_out);
/* host only: the launch plan of launch_gemm_tc for a GPU of `sms` SMs; plan_out[ASRBT_PLAN_LEN] as above ([6] = 0) */
ASRB_API int asrbt_gemm_plan(int M, int N, int K, int a_mode, int epi, int sms, int use_splitk, int OH, int OW, int cpad,
                             int* plan_out);
ASRB_API int asrbt_gemm(const asrbt_gemm_args* a, int* plan_out);
ASRB_API int asrbt_attention(const asrbt_attn_args* a);
/* the alignment DTW kernel (DESIGN.md 4.10) on one caller matrix M [N][T]: start_tok_out[N] = the least column of the
 * path in each row.  The trace goes to shared memory when it fits, else to global memory, as in asrb_align_ids. */
ASRB_API int asrbt_dtw(const float* M, int N, int T, int32_t* start_tok_out);
/* host only: the score head's plan for `rows` rows of a V-word vocabulary on `sms` SMs; plan_out[ASRBT_SCORE_PLAN_LEN] */
ASRB_API int asrbt_score_plan(int rows, int V, int H, int sms, int grid_cap, int* plan_out);
/* the score head (gather, final RMSNorm to split3 planes, wgmma GEMM with the folding epilogue, per-row merge) on
 * caller weights; plan_out[ASRBT_SCORE_PLAN_LEN] = the plan that ran on this GPU */
ASRB_API int asrbt_score_head(const asrbt_score_args* a, int* plan_out);
/* one layer of the alignment fold (csrc/align.cu): probabilities of the listed heads, then z-scores and the width-7
 * median added into M; utterance b's [N][T] blocks at the prefix sums of N * T */
ASRB_API int asrbt_align(const asrbt_align_args* a);

#ifdef __cplusplus
}
#endif
#endif
