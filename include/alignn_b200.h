/*
 * alignn_b200.h -- C ABI of libalignn_b200.so: the H100 (sm_90a) edge-gated graph
 * convolution hot path of ALIGNN.
 *
 * Drop-in boundary.  The reference (usnistgov/alignn, 100 % Python) reaches its device
 * code through DGL's message-passing dispatch and ATen ops inside
 *     EdgeGatedGraphConv.forward      alignn/models/alignn.py:78-129
 *                                     (LayerNorm twin alignn/models/alignn_atomwise.py:157-208)
 * Each entry point below replaces a group of those call sites; the reference-side binding a
 * maintainer would add is the ctypes stub shown in INTEGRATION.md (and shipped as
 * alignn_b200/_lib.py).
 *
 * Conventions
 *   - Only POD crosses the boundary: device pointers, sizes, flags, a CUDA stream handle.
 *   - Ownership: the caller allocates every buffer (inputs, outputs, workspaces).  The library
 *     never allocates, frees, or retains a pointer past return.
 *   - Every call only ENQUEUES work on `stream` (no synchronisation, no host reads of device
 *     memory) and is re-entrant; one process per GPU.
 *   - Return value: 0 on success, a negative alignn_b200_status otherwise; nothing throws.
 *   - All feature matrices are fp32, row-major, contiguous, rows 16-byte aligned.
 *     All index arrays are int32.  `d` (features per row) must be one of 32, 64, 128, 256.
 *   - Results do not depend on launch geometry: no floating-point atomics anywhere.
 *
 * Node-projection layout.  `P` is the [Nn, 4d] output of the four node Linear layers, column
 * blocks in this order (chosen so that the per-edge source gather is one contiguous 2d chunk):
 *     P[:, 0:d]   = src_gate(x)     (alignn.py:98,  "e_src")
 *     P[:, d:2d]  = dst_update(x)   (alignn.py:104, "Bh")
 *     P[:, 2d:3d] = dst_gate(x)     (alignn.py:99,  "e_dst")
 *     P[:, 3d:4d] = src_update(x)   (alignn.py:110)
 * `GP` (its gradient) uses the same layout.
 *
 * Sorted-CSR edge index (int32): in_ptr[Nn+1] / in_eid[Ne] = edge ids stably sorted by
 * destination; out_ptr[Nn+1] / out_eid[Ne] = stably sorted by source.  in_eid may be NULL when
 * the edge list itself is destination-sorted (identity permutation).
 */
#ifndef ALIGNN_B200_H
#define ALIGNN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALIGNN_B200_VERSION 101

typedef enum {
  ALIGNN_OK = 0,
  ALIGNN_ERR_BAD_ARG = -1,        /* NULL where a pointer is required, negative size, bad flag */
  ALIGNN_ERR_UNSUPPORTED_D = -2,  /* d not in {32, 64, 128, 256} */
  ALIGNN_ERR_STRUCT_SIZE = -3,    /* args->struct_size != sizeof(args): header/binding mismatch */
  ALIGNN_ERR_CUDA = -4,           /* a CUDA runtime call failed; see alignn_b200_last_cuda_error */
  ALIGNN_ERR_WORKSPACE = -5       /* workspace too small */
} alignn_b200_status;

/* How the norm after the gate is applied (alignn.py:122-123). */
typedef enum {
  ALIGNN_NORM_LAYER = 0,   /* LayerNorm(d), eps; gamma/beta           (alignn_atomwise.py:151,155) */
  ALIGNN_NORM_AFFINE = 1,  /* per-channel scale/shift: BatchNorm1d in eval mode (alignn.py:72,76) */
  ALIGNN_NORM_STATS = 2    /* BatchNorm1d in train mode: emit pre-norm rows + per-channel partial
                              sums; finish with bn_finalize + bn_apply */
} alignn_b200_norm;

typedef void* alignn_stream_t; /* a cudaStream_t */

int alignn_b200_version(void);
const char* alignn_b200_strerror(int status);
int alignn_b200_last_cuda_error(void);      /* cudaError_t of the last failed runtime call */
uint64_t alignn_b200_launch_count(void);    /* kernels launched by this library so far */

/* Rows of per-block column partials the egc kernels write: grid size they will use. */
int alignn_b200_egc_partial_rows(int64_t Nn, int d);

/* ------------------------------------------------------------------------------------------
 * Forward of one EdgeGatedGraphConv, everything after the Linear layers
 * (replaces alignn.py:100-127: apply_edges(u_add_v), sigmoid, update_all(u_mul_e,sum),
 *  update_all(copy_e,sum), the division, both norms, SiLU and the residuals).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  size_t struct_size;
  int64_t Nn, Ne;
  int32_t d;
  int32_t norm_nodes, norm_edges; /* alignn_b200_norm */
  int32_t residual;               /* alignn.py:125 */
  int32_t gate_is_m;              /* != 0: G already holds m = e_src[src] + e_dst[dst] + edge_gate(y) (written with its
                                     batch statistics by alignn_b200_gemm_gather): no e_src / e_dst gathers, M is not
                                     written, no edge statistics; norm_edges must then be LAYER or AFFINE (or y_out NULL) */
  float gate_eps;                 /* 1e-6, alignn.py:109 */
  float ln_eps;                   /* LayerNorm eps */
  /* inputs */
  const float* x;       /* [Nn,d] node_feats */
  const float* y;       /* [Ne,d] edge_feats (residual input) */
  const float* G;       /* [Ne,d] edge_gate(y) = y W_eg^T + b_eg  (alignn.py:101) */
  const float* P;       /* [Nn,4d] node projections, layout above */
  const int32_t* src;   /* [Ne] */
  const int32_t* in_ptr;  /* [Nn+1] */
  const int32_t* in_eid;  /* [Ne] or NULL (identity) */
  /* norm parameters: LAYER -> (gamma, beta); AFFINE -> (scale, shift); STATS -> unused */
  const float* n_w; const float* n_b;   /* nodes  [d] */
  const float* e_w; const float* e_b;   /* edges  [d] */
  /* outputs */
  float* x_out;   /* [Nn,d]; may be NULL when norm_nodes == STATS */
  float* y_out;   /* [Ne,d]; NULL = edge output not needed (dead output / STATS) */
  float* M;       /* [Ne,d] pre-norm gate m (alignn.py:101); NULL in inference */
  float* XP;      /* [Nn,d] pre-norm node update x' (alignn.py:110); NULL in inference.  XP != NULL selects
                     training mode (M, S, H are then required; M may be NULL only when Ne == 0) */
  float* S;       /* [Nn,d] sum_sigma (alignn.py:108); NULL in inference */
  float* H;       /* [Nn,d] h = sum_sigma_h / (sum_sigma + eps) (alignn.py:109); NULL in inference */
  /* STATS mode: per-block partial column sums, [partial_rows, 4, d] = {sum m, sum m^2, sum x', sum x'^2} */
  float* partials;
  alignn_stream_t stream;
} alignn_b200_egc_fwd_args;

int alignn_b200_egc_forward(const alignn_b200_egc_fwd_args* args);

/* BatchNorm1d train mode, step 2: reduce partials -> batch mean / biased var (alignn.py:72,76,
 * torch BatchNorm1d semantics), emit scale = gamma*rstd, shift = beta - mean*scale, save mean and
 * rstd for backward, and update running_mean / running_var (momentum, unbiased var). */
int alignn_b200_bn_finalize(const float* partials, int partial_rows, int partial_stride /*floats between rows*/,
                            int which /*0: cols {0,1}; 1: cols {2,3} of the partial row*/,
                            int64_t count, int d, const float* gamma, const float* beta, float eps, float momentum,
                            float* running_mean, float* running_var /* may be NULL */,
                            float* scale, float* shift, float* mean, float* rstd, alignn_stream_t stream);

/* BatchNorm1d train mode, step 3: out = (residual ? res : 0) + silu(R*scale + shift), rows [n,d]. */
int alignn_b200_affine_silu_residual(const float* R, const float* res, const float* scale, const float* shift,
                                     float* out, int64_t n, int d, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Backward of the same stage.  Produces
 *   GM [Ne,d]  = dL/dm            (feeds  dL/dy += GM W_eg,  dL/dW_eg = GM^T y)
 *   GP [Nn,4d] = dL/dP            (feeds  dL/dx += GP Wcat,  dL/dWcat = GP^T x,  bias grads = colsum)
 *   norm parameter gradients as per-block partials.
 * The residual part of dL/dx, dL/dy (identity) is added by the caller.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  size_t struct_size;
  int64_t Nn, Ne;
  int32_t d;
  int32_t norm_nodes, norm_edges; /* LAYER, AFFINE (eval BN), STATS (train BN: needs bn_c1/bn_c2) */
  float gate_eps, ln_eps;
  /* saved from forward */
  const float* P; const float* M; const float* XP; const float* S; const float* H;
  const int32_t* src; const int32_t* dst;
  const int32_t* in_ptr; const int32_t* in_eid;
  const int32_t* out_ptr; const int32_t* out_eid;
  /* norm params: LAYER (gamma,beta); AFFINE/STATS (scale,shift) plus, for both, mean/rstd [d]
     (AFFINE/STATS only; used to form xhat for the gamma gradient) */
  const float* n_w; const float* n_b; const float* n_mean; const float* n_rstd;
  const float* e_w; const float* e_b; const float* e_mean; const float* e_rstd;
  /* STATS only: c1 = sum(gu)/count, c2 = sum(gu*xhat)/count per channel (from bn_backward_reduce) */
  const float* n_c1; const float* n_c2; const float* e_c1; const float* e_c2;
  /* incoming gradients */
  const float* gx_out;  /* [Nn,d] */
  const float* gy_out;  /* [Ne,d] or NULL (edge output unused) */
  /* outputs */
  float* GM; float* GP;
  float* GSh;           /* [Nn,d] workspace: dL/d(sum_sigma_h) */
  /* per-block partials of the destination-keyed pass, [partial_rows, 6, d] =
       {sum gu_e*xhat_e, sum gu_e, sum gu_n*xhat_n, sum gu_n, sum dL/dx', sum dL/d e_dst}
     (column sums of rows 0..3 are the norm weight/bias gradients; rows 4,5 are the bias gradients
      of src_update and of dst_gate == edge_gate == src_gate) */
  float* partials;
  /* per-block partials of the source-keyed pass, [partial_rows, 2, d] = {sum dL/d e_src, sum dL/d Bh} */
  float* partials_src;
  /* Line-graph descriptor, optional.  When this graph is L(g) of a parent graph g EXACTLY as the line-graph builders
     emit it (alignn_b200_line_graph_build_host / alignn_b200_line_graph_fill, then the CSR build: node i of L(g) is
     bond i of g; an edge (i -> j) for every pair with dst(i) == src(j), i != j; edges sorted by (j, position of i in
     the in-list of g), so in_eid is the identity and may be NULL), the parent's CSR (in_ptr, in_eid, out_ptr, out_eid
     of g, int32) and its node count may be given: one kernel then runs over the atoms of g and produces everything
     in one pass over the edge rows, bit-identical GM, GP and GSh; the per-block partial rows are grouped differently
     (same buffer shapes; rows no block owns are zeroed).  All NULL / 0: the destination- and source-keyed kernels. */
  const int32_t* parent_in_ptr; const int32_t* parent_in_eid;
  const int32_t* parent_out_ptr; const int32_t* parent_out_eid;
  int64_t parent_Nn;
  alignn_stream_t stream;
} alignn_b200_egc_bwd_args;

int alignn_b200_egc_backward(const alignn_b200_egc_bwd_args* args);

/* ------------------------------------------------------------------------------------------
 * Double backward of the same stage, LayerNorm only: the vector-Jacobian product of the first
 * backward, which `torch.autograd.grad(..., create_graph=True)` differentiates in force training
 * (alignn/models/alignn_atomwise.py:530-539).  The first backward maps (x, y, gx_out, gy_out) to
 *   gx = GP Wcat (+ gx_out),  gy = GM W_eg (+ gy_out);
 * given cotangents gx_bar, gy_bar of gx, gy, the caller first projects them through the same
 * weights (GPbar = gx_bar Wcat^T, GMbar = gy_bar W_eg^T) and this call produces
 *   Pbar [Nn,4d] = dL/dP (layout of P),  Mbar [Ne,d] = dL/dm,
 *   gx_out_bar, gy_out_bar (with the residual's gx_bar / gy_bar added when given),
 *   LayerNorm parameter cotangents and bias sums as per-block partials.
 * The caller finishes with x_bar = Pbar Wcat, y_bar = Mbar W_eg and the weight cotangents
 * Pbar^T x + GP^T gx_bar, Mbar^T y + GM^T gy_bar.  norm must be ALIGNN_NORM_LAYER (ALIGNN_ERR_BAD_ARG
 * otherwise; checked right after struct_size and d, before the graph sizes and pointers).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  size_t struct_size;
  int64_t Nn, Ne;
  int32_t d;
  int32_t norm;                   /* ALIGNN_NORM_LAYER (both norms of the conv) */
  float gate_eps, ln_eps;
  /* saved from forward */
  const float* P; const float* M; const float* XP; const float* S; const float* H;
  const int32_t* src; const int32_t* dst;
  const int32_t* in_ptr; const int32_t* in_eid;   /* in_eid NULL = identity */
  const int32_t* out_ptr; const int32_t* out_eid;
  const float* n_w; const float* n_b; const float* e_w; const float* e_b;   /* LayerNorm gamma, beta [d] */
  /* inputs of the first backward and its workspace */
  const float* gx_out;      /* [Nn,d] */
  const float* gy_out;      /* [Ne,d] or NULL (edge output unused) */
  const float* GSh;         /* [Nn,d] dL/d(sum_sigma_h) as alignn_b200_egc_backward wrote it */
  /* cotangents */
  const float* GPbar;       /* [Nn,4d] gx_bar Wcat^T */
  const float* GMbar;       /* [Ne,d] gy_bar W_eg^T, or NULL (zero) */
  const float* gx_bar_res;  /* [Nn,d] gx_bar, added to gx_out_bar (residual), or NULL */
  const float* gy_bar_res;  /* [Ne,d] gy_bar, added to gy_out_bar (residual), or NULL */
  /* outputs */
  float* Pbar;              /* [Nn,4d] */
  float* Mbar;              /* [Ne,d] */
  float* gx_out_bar;        /* [Nn,d] */
  float* gy_out_bar;        /* [Ne,d]; required when gy_out != NULL */
  float* Gamma;             /* [Ne,d] workspace: cotangent of GM */
  float* Shbar;             /* [Nn,d] workspace: dL/d(sum_sigma_h) of the forward */
  /* per-block partials, rows = alignn_b200_egc_partial_rows(Nn, d):
     destination pass [rows, 6, d] = {sum e_w_bar, sum e_b_bar, sum n_w_bar, sum n_b_bar, sum Pbar_D, sum Pbar_B};
     source pass      [rows, 2, d] = {sum Pbar_A, sum Pbar_C} */
  float* partials;
  float* partials_src;
  alignn_stream_t stream;
} alignn_b200_egc_bwd_vjp_args;

int alignn_b200_egc_backward_vjp(const alignn_b200_egc_bwd_vjp_args* args);

/* BatchNorm train-mode backward, pass 1: per-block partials of sum(gu) and sum(gu*xhat) over rows,
 * gu = g_out * silu'(R*scale+shift), xhat = (R-mean)*rstd.  partials: [rows_out, 2, d]. */
int alignn_b200_bn_backward_reduce(const float* R, const float* g_out, const float* scale, const float* shift,
                                   const float* mean, const float* rstd, int64_t n, int d,
                                   float* partials, int partial_rows, alignn_stream_t stream);

/* Linear -> BatchNorm1d(train) -> SiLU embedding layers (alignn.py:170-184) on rows [n,d]:
 *   rowstats_partials: per-block {sum, sum^2} partials ([rows, 2, d]; feed alignn_b200_bn_finalize with which = 0,
 *                      partial_stride = 2d), then alignn_b200_affine_silu_residual(res = NULL) applies norm + SiLU;
 *   bn_backward_apply: gR = scale * (gu - c1 - xhat*c2), gu = g_out * silu'(R*scale+shift)  (c1, c2 from
 *                      alignn_b200_bn_backward_reduce). */
int alignn_b200_rowstats_partials(const float* a, int64_t n, int d, float* partials, int partial_rows, alignn_stream_t stream);
int alignn_b200_bn_backward_apply(const float* R, const float* g_out, const float* scale, const float* shift,
                                  const float* mean, const float* rstd, const float* c1, const float* c2, int64_t n, int d,
                                  float* gR, alignn_stream_t stream);

/* Linear -> LayerNorm -> SiLU embedding layers of the LayerNorm model (alignn/models/alignn_atomwise.py:249-268) on the
 * rows h [n,d] the Linear produced:
 *   ln_silu_forward:  out[r] = silu(LayerNorm_eps(h[r]) * gamma + beta);  rowstat[r] = {mean, rstd}  ([n,2] floats)
 *   ln_silu_backward: gh = d loss / d h given g_out = d loss / d out; partials [partial_rows, 2, d] hold the per-block sums
 *                     for d gamma (index 0) and d beta (index 1): finish with alignn_b200_colsum.
 *                     partial_rows = alignn_b200_egc_partial_rows(n, d). */
int alignn_b200_ln_silu_forward(const float* h, const float* gamma, const float* beta, float eps, int64_t n, int d, float* out,
                                float* rowstat, alignn_stream_t stream);
int alignn_b200_ln_silu_backward(const float* h, const float* g_out, const float* rowstat, const float* gamma, const float* beta,
                                 int64_t n, int d, float* gh, float* partials, int partial_rows, alignn_stream_t stream);

/* One AdamW update (torch.optim.AdamW arithmetic, amsgrad off; the optimizer alignn/train.py:253-263 builds) over flat
 * 16-byte aligned fp32 buffers of n elements.  `step` is the DEVICE step counter (int64, starts at 0): the kernel uses
 * t = *step + 1 for the bias corrections and stores t back, so the same launch replays correctly inside a CUDA graph.
 * `ticket` is a zero-initialised device uint32 the kernel uses to find its last block (left at zero).  zero_grad != 0
 * clears `grad` after use. */
int alignn_b200_adamw_flat(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1,
                           float beta2, float eps, float weight_decay, int zero_grad, int64_t* step, uint32_t* ticket,
                           alignn_stream_t stream);

/* Per-block partial column sums of a tall contiguous [n, d] matrix (rows: alignn_b200_egc_partial_rows(n, d));
 * finish with alignn_b200_colsum.  Used for the bias gradients of the embedding Linears (alignn.py:201-222). */
int alignn_b200_colsum_partials(const float* a, int64_t n, int d, float* partials, int partial_rows, alignn_stream_t stream);

/* Deterministic column sum of a [rows, cols] fp32 matrix with row stride `stride` floats into
 * out[cols] (fp64 accumulation), optionally scaled by `alpha`. */
int alignn_b200_colsum(const float* a, int64_t rows, int cols, int64_t stride, float alpha, float* out,
                       alignn_stream_t stream);

/* Many column sums in one launch (same arithmetic as alignn_b200_colsum per problem): the bias and norm-parameter
 * gradients of all convs of a backward pass -- autograd's reductions of `alignn.py:98-127` over the per-block partial rows
 * alignn_b200_egc_backward leaves -- are off the critical path and are summed together at the end of backward.
 * `problems` is a HOST array (copied into the kernel parameters; capturable in a CUDA graph). */
typedef struct {
  const float* a; int64_t rows; int64_t stride;   /* [rows, >= cols] partial rows, row stride in floats */
  int cols; float alpha;
  float* out;                                     /* [cols] */
} alignn_b200_colsum_problem;
int alignn_b200_colsum_batch(const alignn_b200_colsum_problem* problems, int n, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Gather / segment-sum primitive alone (BASELINE.json config 5; DGL update_all(u_mul_e,sum) +
 * update_all(copy_e,sum), alignn.py:105-108):  Sh[v] = sum_{e->v} Bh[src e]*sigma[e],
 * S[v] = sum_{e->v} sigma[e].
 * ---------------------------------------------------------------------------------------- */
int alignn_b200_gather_segment_sum(const float* Bh, const float* sigma, const int32_t* src,
                                   const int32_t* in_ptr, const int32_t* in_eid, int64_t Nn, int64_t Ne, int d,
                                   float* Sh, float* S, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Linear layers on the Hopper tensor cores (wgmma, bf16x3 split operands, fp32 accumulate in
 * registers; results agree with an fp32 GEMM to ~1e-5 relative):
 *     C[M,N] = A[M,K] * W[N,K]^T (+ bias[N]) (+ R[M,N])
 * Replaces the nn.Linear call sites alignn.py:98,99,101,104,110 (forward) and their data-gradient
 * GEMMs.  W is first converted once per step to a bf16 hi/lo image (`gemm_prepare_table`;
 * `transpose != 0` takes W^T of a [K,N] array, which is what the data-gradient GEMMs need).
 * Constraints: K % 32 == 0, N % 32 == 0, lda/ldc/ldr % 4 == 0 and A, R, C 16-byte aligned (16-byte rows).
 * C must not overlap A, R or bias: the epilogue reads the addends while other rows of C are being written.
 * ---------------------------------------------------------------------------------------- */
size_t alignn_b200_gemm_weight_image_bytes(int N, int K);   /* 0 if the shape is unsupported */
/* Table-driven refresh of many operand images in one launch (+ one for the bias vectors).  Every entry converts one
 * source block W[rows, cols] (row stride ldw; transpose != 0: the block enters as its transpose) into the image of an
 * [N, K] operand at row offset n_off / column offset k_off (k_off % 8 == 0; blocks narrower than a multiple of 8 are
 * zero-padded).  Typical use: [src_gate; dst_update; dst_gate; src_update] stacked along N for the node projections,
 * the same four transposed and stacked along K for their data gradient (alignn.py:98,99,104,110).  The entry arrays live
 * in DEVICE memory (the caller builds them once; parameter storage is stable across optimizer steps).
 * max_units >= max over entries of image_rows * ceil(image_cols_of_block / 8). */
typedef struct {
  const float* W; int64_t ldw;
  int32_t rows, cols, transpose;
  int32_t n_off, k_off;
  int32_t N, K;
  void* image;
} alignn_b200_image_entry;
typedef struct { const float* a; const float* b; float* dst; int32_t n; } alignn_b200_bias_entry;   /* dst = a (+ b) */
int alignn_b200_gemm_prepare_table(const alignn_b200_image_entry* entries, int n_entries, int64_t max_units,
                                   const alignn_b200_bias_entry* bias_entries, int n_bias, alignn_stream_t stream);
int alignn_b200_gemm_nt(const float* A, int64_t lda, const void* w_image, int64_t M, int N, int K, const float* bias,
                        const float* R, int64_t ldr, float* C, int64_t ldc, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Linear layer with a gather-add epilogue and optional column statistics (csrc/gemm_tc.cu):
 *     C[r, 0:N] = A[r, 0:K] * W^T (+ bias) (+ add0[i0(r), 0:N]) (+ add1[i1(r), 0:N]),   i(r) = idx ? idx[r] : r
 *     stats[blk][0][c] / stats[blk][1][c] = per-CTA partial sums of C[:, c] and C[:, c]^2  (optional; needs N in
 *     {32, 64, 128, 256}; rows = alignn_b200_gemm_gather_stat_rows(M, N); feed alignn_b200_bn_finalize, which = 0)
 * The edge-gate use (alignn/models/alignn.py:98-101, 123): A = edge_feats, W = edge_gate.weight,
 * add0 = P + 0 (ld 4d, idx0 = src: e_src), add1 = P + 2d (ld 4d, idx1 = dst: e_dst, bias of edge_gate folded into the
 * dst_gate bias by the caller) gives m = e_src[src] + e_dst[dst] + edge_gate(y) and the batch statistics of
 * BatchNorm1d(m) in one pass over y -- apply_edges(u_add_v) and the Linear fused, no [Ne,d] temporary.
 * With add0 = R, idx0 = NULL it is the data-gradient GEMM with its residual; without addends a plain Linear.
 * A is streamed row by row (row stride lda floats, 16-byte aligned rows); W is an image from
 * alignn_b200_gemm_prepare_table.  Constraints: K % 32 == 0, N % 32 == 0, lda/ldc/ld0/ld1 % 4 == 0.
 * C must not overlap A, add0, add1, bias or stats: the epilogue reads the addends while other rows of C are being
 * written.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  size_t struct_size;
  int64_t M; int32_t N, K;
  const float* A; int64_t lda;
  const void* w_image;
  const float* bias;                                        /* [N] or NULL */
  const float* add0; int64_t ld0; const int32_t* idx0;      /* addend rows (NULL: none); idx NULL = identity */
  const float* add1; int64_t ld1; const int32_t* idx1;
  float* C; int64_t ldc;
  float* stats;                                             /* [stat_rows][2][N] or NULL */
  alignn_stream_t stream;
} alignn_b200_gemm_gather_args;

int alignn_b200_gemm_gather(const alignn_b200_gemm_gather_args* args);
int alignn_b200_gemm_gather_stat_rows(int64_t M, int N);

/* Weight gradients on the tensor cores (split-K over the batch rows, deterministic two-stage sum):
 *     out[g*DA + o, i] = sum_{r < K} A[r, g*DA + o] * B[r, i]        g < groups,  o < DA,  i < DB
 * i.e. dL/dW = GM^T y (groups = 1) and dL/dWcat = GP^T x (groups = 4) of SURVEY.md App. B, and the
 * rectangular weight gradients of the embedding MLPs (alignn.py:201-222).  Supported (DA, DB): DA == DB in
 * {32, 64, 128, 256}; (256,64), (256,96), (64,96), (64,32), (32,64), (32,96).
 * `workspace` holds the per-CTA partial tiles (size from alignn_b200_wgrad_workspace_bytes; 0 = unsupported). */
size_t alignn_b200_wgrad_workspace_bytes(int64_t K, int DA, int DB, int groups);
int alignn_b200_wgrad(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t K, int DA, int DB, int groups,
                      float* out, int64_t ld_out, void* workspace, size_t workspace_bytes, alignn_stream_t stream);

/* Many square weight gradients in ONE launch: out_p[o, i] = sum_{r < K_p} A_p[r, o] * B_p[r, i], o, i < D, for every
 * problem p < n (n <= 64).  The 4+4 stack's backward pass produces 24 such products per step (SURVEY.md App. B: GP^T x
 * per projection, GM^T y), none on its critical path; queued and launched together the small ones (K = atoms or bonds)
 * ride along at the memory rate instead of paying a launch prologue and a grid barrier each.  `problems` is a HOST array
 * (copied into the kernel parameters: capturable in a CUDA graph); A, B, out are device pointers, 16-byte aligned,
 * leading dimensions multiples of 4.  Deterministic (fixed-order split-K).  The fallback on a device that cannot
 * co-schedule one CTA per SM runs the problems one by one through alignn_b200_wgrad and needs that function's workspace. */
typedef struct {
  const float* A; int64_t lda;     /* [K, >= D] output-gradient rows                                   */
  const float* B; int64_t ldb;     /* [K, >= D] input rows                                             */
  int64_t K;
  float* out; int64_t ld_out;      /* [D, D] weight gradient, row o = output channel                   */
} alignn_b200_wgrad_problem;
size_t alignn_b200_wgrad_batch_workspace_bytes(const alignn_b200_wgrad_problem* problems, int n, int D);
int alignn_b200_wgrad_batch(const alignn_b200_wgrad_problem* problems, int n, int D, void* workspace, size_t workspace_bytes,
                            alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Host-side structure builders (plain CPU code, host pointers, no stream; usable without a GPU).
 * Replace the structure step DGL does on the CPU for the reference: `dgl.graph((u, v))` + CSR/CSC views
 * (alignn/graphs.py:544) and `g.line_graph(shared=True)` (alignn/graphs.py:588).  Integer-exact.
 *
 * csr_build_host: int64 (src, dst) -> int32 copies + stable sorted-CSR index (in_* by destination, out_* by
 *   source), whether the edge list is already destination-sorted, and the largest in-degree.
 * line_graph_count_host / line_graph_build_host: L(g) edges (i -> j) iff dst(i) == src(j), i != j, emitted
 *   destination-major (j ascending, then i ascending); `capacity` must equal the count; per-graph edge counts of
 *   L(g) are written to l_batch_num_edges[batch_size] from the per-graph bond counts of g.
 * ---------------------------------------------------------------------------------------- */
int alignn_b200_csr_build_host(const int64_t* src, const int64_t* dst, int64_t num_nodes, int64_t num_edges,
                               int32_t* src32, int32_t* dst32, int32_t* in_ptr, int32_t* in_eid, int32_t* out_ptr,
                               int32_t* out_eid, int32_t* dst_sorted, int32_t* max_in_degree);
int64_t alignn_b200_line_graph_count_host(const int32_t* src, const int32_t* in_ptr, const int32_t* in_eid,
                                          int64_t num_edges);
int alignn_b200_line_graph_build_host(const int32_t* src, const int32_t* in_ptr, const int32_t* in_eid,
                                      int64_t num_edges, const int64_t* batch_num_edges, int64_t batch_size,
                                      int64_t capacity, int64_t* lsrc, int64_t* ldst, int64_t* l_batch_num_edges);

/* Periodic radius graph on the host (alignn/graphs.py:267-364): bonds (u, image c of v) with
 * atol < |x_v + shifts[c] - x_u| <= cutoff in (u, c, v) order; r = displacement (fp32), image_index = c.
 * `shifts` [num_images,3] = cell offsets @ lattice (computed by the caller).  Two-pass: count, then build with
 * capacity == count. */
int64_t alignn_b200_radius_graph_count_host(const double* cart_coords, const double* shifts, int64_t num_atoms,
                                            int64_t num_images, double cutoff, double atol);
int alignn_b200_radius_graph_build_host(const double* cart_coords, const double* shifts, int64_t num_atoms,
                                        int64_t num_images, double cutoff, double atol, int64_t capacity, int64_t* u,
                                        int64_t* v, int64_t* image_index, float* r);

/* ------------------------------------------------------------------------------------------
 * Device-side structure builders and ALIGNN-FF reductions (csrc/graph_device.cu; the radius scan is in
 * csrc/crystal_graph_device.cu).  All pointers are DEVICE pointers;
 * the caller owns every buffer including the workspace; calls only enqueue on `stream`.  Integer results are
 * bit-identical to the host builders above; the two d=3 sums are deterministic (fixed order, no float atomics).
 * Replace, on the GPU: `dgl.graph((u, v))` + CSR/CSC views (alignn/graphs.py:544), `g.line_graph(shared=True)`
 * (alignn/graphs.py:588), the periodic radius graph (alignn/graphs.py:267-364), `update_all(copy_e, sum)` on g and on
 * dgl.reverse(g) (alignn/models/alignn_atomwise.py:547-563) and the per-crystal virial (:610-635).
 * ---------------------------------------------------------------------------------------- */
/* Sorted-CSR edge index on the device = alignn_b200_csr_build_host (`dgl.graph((u, v))`, alignn/graphs.py:544).
 * in_eid / out_eid: edge ids stably sorted by destination / source; flags[0] = 1 if dst is already non-decreasing,
 * flags[1] = largest in-degree. */
size_t alignn_b200_csr_build_workspace_bytes(int64_t num_nodes, int64_t num_edges);
int alignn_b200_csr_build(const int32_t* src, const int32_t* dst, int64_t num_nodes, int64_t num_edges, int32_t* in_ptr,
                          int32_t* in_eid, int32_t* out_ptr, int32_t* out_eid, int32_t* flags, void* workspace,
                          size_t workspace_bytes, alignn_stream_t stream);

/* Line graph on the device = alignn_b200_line_graph_{count,build}_host (`g.line_graph(shared=True)`,
 * alignn/graphs.py:588): offsets[j] = number of pairs (i -> j') with j' < j, offsets[E] = T (read it back to size
 * lsrc / ldst); the pairs are written destination-major with ascending sources, so `offsets` is L(g)'s in_ptr. */
size_t alignn_b200_line_graph_workspace_bytes(int64_t num_edges);
int alignn_b200_line_graph_offsets(const int32_t* src, const int32_t* dst, const int32_t* in_ptr, int64_t num_edges,
                                   int32_t* offsets, void* workspace, size_t workspace_bytes, alignn_stream_t stream);
int alignn_b200_line_graph_fill(const int32_t* src, const int32_t* dst, const int32_t* in_ptr, const int32_t* in_eid,
                                int64_t num_edges, const int32_t* offsets, int32_t* lsrc, int32_t* ldst, alignn_stream_t stream);

/* Periodic radius graph on the device = alignn_b200_radius_graph_{count,build}_host (alignn/graphs.py:267-364): bonds
 * u -> v for every image `c` of v with atol < |x_v + shifts[c] - x_u| <= cutoff, in (u, c, v) order, double precision
 * with the host builder's operation order (bit-identical bond list and displacement vectors).  offsets[u] = first bond
 * of atom u, offsets[N] = number of bonds (read it back to size the outputs); fill with empty outputs is an error only
 * if bonds exist.  The caller computes `shifts = cells @ lattice` and handles the cutoff-growth retry
 * (graphs.py:347-350) exactly as alignn_b200.neighbors.radius_graph does for the host scan. */
size_t alignn_b200_radius_graph_workspace_bytes(int64_t num_atoms);
int alignn_b200_radius_graph_offsets(const double* cart_coords, const double* shifts, int64_t num_atoms, int64_t num_images,
                                     double cutoff, double atol, int32_t* offsets, void* workspace, size_t workspace_bytes,
                                     alignn_stream_t stream);
int alignn_b200_radius_graph_fill(const double* cart_coords, const double* shifts, int64_t num_atoms, int64_t num_images,
                                  double cutoff, double atol, const int32_t* offsets, int32_t* u, int32_t* v,
                                  int32_t* image_index, float* r, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Crystal graphs for a batch of B structures on the device (csrc/crystal_graph_device.cu): the neighbour lists of
 * `Graph.atom_dgl_multigraph` (alignn/graphs.py:472-589) for both of its strategies.  Device pointers except
 * `lattices`, caller-owned buffers, enqueue-only on `stream`.  The caller builds, per crystal b, the image table
 * `cells` (integer cell offsets as doubles, meshgrid "ij" order) and `shifts = cells @ lattice_b`, concatenated over
 * the batch with shift_offsets[B+1]; atoms are concatenated with atom_offsets[B+1] and crystal_of_atom[N].
 * Rejected (ALIGNN_ERR_BAD_ARG, nothing enqueued): B < 1, N < 1, a NULL input, a lattice with zero or non-finite
 * determinant, max_neighbors < 1.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const double* cart_coords;      /* [N,3] Cartesian coordinates                                             */
  const double* shifts;           /* [I,3] per-crystal image shifts, concatenated                            */
  const double* cells;            /* [I,3] the matching cell offsets                                         */
  const double* lattices;         /* [B,3,3] lattice row vectors, HOST memory (checked, copied by the emit)  */
  const int64_t* atom_offsets;    /* [B+1]                                                                   */
  const int64_t* shift_offsets;   /* [B+1]                                                                   */
  const int32_t* crystal_of_atom; /* [N]                                                                     */
  const double* cutoffs;          /* [B] per-crystal cutoff                                                  */
  int64_t num_crystals;           /* B */
  int64_t num_atoms;              /* N */
  int64_t num_images;             /* I = shift_offsets[B] */
  int64_t max_images;             /* largest per-crystal image count */
  double atol;                    /* pairs with |d| <= atol are the atom itself */
} alignn_b200_crystal_batch;

/* Candidate scan (the radius scan above, batched): for every atom u of crystal b, every (image c, atom v of b) with
 * atol < |(shifts[c] + x_v) - x_u| <= cutoffs[b] in double precision.  offsets[N+1] = exclusive scan of the per-atom
 * counts (offsets[N] = total).  status[b] = the crystal's smallest per-atom count (strategy 1, k-NN: the crystal needs
 * a grown cutoff if it is below k, graphs.py:166-186) or 1 if the crystal's last atom has a bond (strategy 0, radius:
 * graphs.py:347-350).  Read status and offsets[N] back to decide the next round. */
size_t alignn_b200_crystal_scan_workspace_bytes(int64_t num_atoms);
int alignn_b200_crystal_scan_count(const alignn_b200_crystal_batch* batch, int strategy, int32_t* offsets, int32_t* status,
                                   void* workspace, size_t workspace_bytes, alignn_stream_t stream);
/* Radius strategy: the bonds in (u, c, v) order per atom, exactly `radius_graph` of each crystal concatenated with
 * atom ids offset: u, v [E] global ids, r [E,3] = fp32 displacement, images [E,3] = fp32 cell offsets. */
int alignn_b200_crystal_radius_fill(const alignn_b200_crystal_batch* batch, const int32_t* offsets, int32_t* u, int32_t* v,
                                    float* r, float* images, alignn_stream_t stream);

/* k-nearest strategy (`nearest_neighbor_edges` + `build_undirected_edgedata`, graphs.py:155-264, use_canonize=True),
 * three calls on one workspace sized for the candidate count C = offsets[N] of the final scan round.  The image tables
 * must be symmetric (cells[I-1-c] == -cells[c]).
 * select: per atom, candidates ordered by (dist, v, image); everything with dist <= the k-th distance is kept (exact
 *   double compare, graphs.py:202-214).  kept_offsets[N+1] = exclusive scan of the kept counts; read kept_offsets[N].
 * order:  each kept (u, v, c) -> (u, v, c) if v >= u else (v, u, -c); pairs in order of first encounter (atoms
 *   ascending, then (dist, v, image)), images ascending inside a pair, duplicates dropped (graphs.py:127-152,
 *   218-223, 240-244).  bond_offsets[B+1] int64 = first bond of each crystal; read it back to size the outputs.
 * emit:   every (a, b, image) -> rows (a, b, d) and (b, a, -d), d = fp32(((frac_b + image) - frac_a) @ lattice)
 *   in double (graphs.py:245-257); images [E,3] fp32 on both rows.  frac_coords [N,3] device. */
size_t alignn_b200_knn_graph_workspace_bytes(int64_t num_atoms, int64_t num_crystals, int64_t num_candidates);
int alignn_b200_knn_graph_select(const alignn_b200_crystal_batch* batch, const int32_t* offsets, int64_t num_candidates,
                                 int max_neighbors, int32_t* kept_offsets, void* workspace, size_t workspace_bytes,
                                 alignn_stream_t stream);
int alignn_b200_knn_graph_order(const alignn_b200_crystal_batch* batch, const int32_t* offsets, const int32_t* kept_offsets,
                                int64_t num_candidates, int64_t num_kept, int64_t* bond_offsets, void* workspace,
                                size_t workspace_bytes, alignn_stream_t stream);
int alignn_b200_knn_graph_emit(const alignn_b200_crystal_batch* batch, const double* frac_coords, int64_t num_candidates,
                               int64_t num_kept, int32_t* u, int32_t* v, float* r, float* images, void* workspace,
                               size_t workspace_bytes, alignn_stream_t stream);

/* forces[v] = sum over in-edges of pair_forces - (add_reverse ? sum over out-edges : 0)   (alignn_atomwise.py:547-563:
 * update_all(copy_e, sum) on g and on dgl.reverse(g)); pair_forces [E,3], forces [Nn,3].  in_eid NULL = identity. */
int alignn_b200_pair_force_scatter(const float* pair_forces, const int32_t* in_ptr, const int32_t* in_eid,
                                   const int32_t* out_ptr, const int32_t* out_eid, int64_t num_nodes, int add_reverse,
                                   float* forces, alignn_stream_t stream);

/* stress[b] = multiplier * -160.21766208 * (r_b^T pair_forces_b) / V[node_offsets[b]]   (alignn_atomwise.py:610-635);
 * edge_offsets / node_offsets [B+1] int64 prefix sums of batch_num_edges / batch_num_nodes; stress [B,3,3]. */
int alignn_b200_virial_stress(const float* r, const float* pair_forces, const int64_t* edge_offsets,
                              const int64_t* node_offsets, const float* V, int64_t batch_size, float multiplier,
                              float* stress, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * eALIGNN force-field steps (csrc/ff_device.cu).  Device pointers, caller-owned buffers, enqueue-only on `stream`.
 * ---------------------------------------------------------------------------------------- */
/* Bond cutoff filter = `lightweight_line_graph(g, "bondlength", gt inner_cutoff)` with the bond vectors of
 * `compute_pair_vector_and_distance` (alignn/models/utils.py:47-55, 129-222; called at ealignn_atomwise.py:309-318).
 * offsets: r[e] = (cart_coords[dst[e]] + images[e]) - cart_coords[src[e]] in fp32, one component at a time in that order
 *   (bit-identical to torch), r [E,3]; bond e is dropped iff |r[e]| > cutoff (a NaN length is kept, as torch.gt is false
 *   for NaN); offsets[E+1] = exclusive scan of the keep flags, offsets[E] = kept bonds.  |r| is computed in fp32 and may
 *   round differently from torch.norm: a bond within an ulp of the cutoff may be classified differently.
 * fill: the kept bonds in their original order -> src_out / dst_out / r_out [E',3] / images_out [E',3], and edge_ids
 *   [E'] int64 numbered as the reference does (utils.py:159-179, 206): the bond's index inside its crystal when
 *   batch_size > 1, its global index otherwise.  edge_offsets [batch_size+1] int64 = prefix of batch_num_edges.  Read
 *   offsets back at edge_offsets to get E' and the kept bonds per crystal. */
size_t alignn_b200_bond_cutoff_workspace_bytes(int64_t num_edges);
int alignn_b200_bond_cutoff_offsets(const float* cart_coords, const int32_t* src, const int32_t* dst, const float* images,
                                    int64_t num_edges, float cutoff, float* r, int32_t* offsets, void* workspace,
                                    size_t workspace_bytes, alignn_stream_t stream);
int alignn_b200_bond_cutoff_fill(const int32_t* src, const int32_t* dst, const float* r, const float* images,
                                 const int32_t* offsets, const int64_t* edge_offsets, int64_t batch_size, int64_t num_edges,
                                 int32_t* src_out, int32_t* dst_out, float* r_out, float* images_out, int64_t* edge_ids,
                                 alignn_stream_t stream);

/* Net-torque removal = `remove_net_torque` (alignn/models/utils.py:295-398, ealignn_atomwise.py:409-412), quirks kept:
 * com = mean of ALL positions of the batch, r_i = pos_i - com, tau = sum over the WHOLE batch of r_i x F_i; per crystal
 * b: M_b = sum r_i r_i^T - (sum |r_i|^2) I, mu_b = M_b^{-1} (-tau) (the same tau for every crystal);
 * out_i = F_i + r_i x mu_b.  pos / forces / out [N,3] fp32, node_offsets [B+1] int64.  Sums in double with fixed-order
 * block partials; each 3x3 system is solved in double by LU with partial pivoting, and by the pseudo-inverse
 * (symmetric eigendecomposition, eigenvalues below 3 eps max|lambda| dropped) when a pivot is exactly zero.  The
 * reference switches the WHOLE batch to the pseudo-inverse when any crystal is singular; choosing per crystal differs
 * from that by rounding only.  (That branch of the reference raises an IndexError on its 1-D right-hand side; this call
 * computes what it means.)  cross_dim0 = 1 (only valid with N == 3): torch.cross without `dim` crosses along dim 0
 * of the [3,3] tensors, i.e. the columns, and so does this call. */
size_t alignn_b200_remove_net_torque_workspace_bytes(int64_t batch_size);
int alignn_b200_remove_net_torque(const float* pos, const float* forces, const int64_t* node_offsets, int64_t batch_size,
                                  int64_t num_nodes, int cross_dim0, float* out, void* workspace, size_t workspace_bytes,
                                  alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Structure relaxation (csrc/fire_device.cu): one step of ASE 3.22.1's FIRE (`FIRE.step`, ase/optimize/fire.py) with
 * the convergence test and step limit of `Optimizer.converged` / `Dynamics.irun` (ase/optimize/optimize.py), for a
 * batch of crystals relaxed together -- what `ForceField.optimize_atoms(optimizer="FIRE", optimize_lattice=False)`
 * (alignn/ff/ff.py:373-417) runs one crystal at a time on the forces of `AlignnAtomwiseCalculator.calculate`
 * (alignn/ff/calculators.py:280-372).  Device pointers, caller-owned buffers, enqueue-only on `stream`.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  double maxstep;           /* cap on |dr| over the whole crystal (0.2)                    */
  double dtmax;             /* 1.0 */
  double finc, fdec;        /* 1.1, 0.5 */
  double astart, fa;        /* 0.1, 0.99 */
  double fmax;              /* converged when max_i |F_i|^2 < fmax^2 (strict)              */
  int32_t n_min;            /* Nmin = 5: dt grows only once Nsteps > n_min                 */
  int32_t max_steps;        /* steps >= 1: a crystal takes at most this many FIRE steps    */
  float force_multiplier;   /* F = fp32(grad * force_multiplier), the calculator's scaling */
} alignn_b200_fire_params;

/* One launch per relaxation step: one CTA per entry of active[num_active] (crystal ids, each listed once), for a model
 * batch holding those crystals' atoms in that order.  Per crystal c with status 0 (running):
 *   F = fp32(grad[batch_offsets[j] + i] * force_multiplier) for its atoms i, written to forces[atom_offsets[c] + i]
 *   (so forces hold the last evaluation); if max_i |F_i|^2 < fmax^2 the status becomes 1 (converged), else if c has
 *   taken max_steps steps it becomes 2 (step limit), else one FIRE step updates velocities, positions and the state.
 *   The j-th batch slice must be crystal c's atoms: batch_offsets[j+1] - batch_offsets[j] == atom_offsets[c+1] -
 *   atom_offsets[c], inside [0, grad_rows).  Otherwise nothing is read or written for c except its status, which
 *   becomes 3 (inconsistent input); read the status back to detect it.
 *   Sums are in double with a fixed-order block reduction; the per-element updates follow numpy's order exactly.
 * Crystals with a nonzero status, and ids outside [0, num_crystals), are not touched.
 *   grad [grad_rows, 3] fp32 (the model batch, atoms compacted); batch_offsets [num_active+1] int32;
 *   atom_offsets [num_crystals+1] int64; positions / velocities [N,3] double; forces [N,3] fp32;
 *   fstate [num_crystals,2] double = {dt, a}; istate [num_crystals,4] int32 = {Nsteps, first step pending (v is None),
 *   steps taken, status}.  Initial state: velocities 0, {dt, a} = {0.1, 0.1}, istate {0, 1, 0, 0}.
 * Rejected (ALIGNN_ERR_BAD_ARG, nothing enqueued): NULL params or a NULL array, num_active outside [0, num_crystals],
 * grad_rows < 0, maxstep or dtmax not > 0, fmax negative or not finite, a non-finite factor, n_min < 0, max_steps < 1. */
int alignn_b200_fire_step(const alignn_b200_fire_params* params, const int32_t* active, int64_t num_active,
                          const int64_t* atom_offsets, const int32_t* batch_offsets, int64_t num_crystals,
                          const float* grad, int64_t grad_rows, double* positions, double* velocities, float* forces,
                          double* fstate, int32_t* istate, alignn_stream_t stream);

/* Structure relaxation with the cell (csrc/fire_cell_device.cu): one FIRE step on ASE 3.22.1's `ExpCellFilter`
 * (ase/constraints.py; no mask, no hydrostatic strain, no constant volume, scalar_pressure 0, cell_factor 1) -- what
 * `ForceField.optimize_atoms(optimizer="FIRE", optimize_lattice=True)`, the reference's default, runs one crystal at a
 * time with the forces and Voigt stress of `AlignnAtomwiseCalculator.calculate`. */
typedef struct {
  alignn_b200_fire_params fire;
  float stress_wt;          /* the calculator's stress scaling: s = fp32(voigt(stress) * stress_wt / 160.21766208) */
} alignn_b200_fire_cell_params;

/* As alignn_b200_fire_step, on the filter's n + 3 rows: the atom rows f_i F and the cell rows (the symmetrised
 * -expm(Y)[0:3,3:6], Y = [[L, -W expm(-L)], [0, L]], W = -V full(s) F^-T, or W itself when the two are neither
 * np.isclose nor aligned with a cosine above 0.8).  Per running crystal c (j its index in active):
 *   stress [stress_rows = num_active, 3, 3] fp32: the model's stress of crystal active[j] in row j;
 *   stress_out [num_crystals, 6] fp32: the calculator's Voigt stress (xx yy zz yz xz xy, eV/A^3) of this evaluation;
 *   cell_forces [num_crystals, 3, 3] double: the filter's cell rows of this evaluation;
 *   filter state, [num_crystals, 3, 3] double each: cells0 (C0, the cell the relaxation started from), logdef (L),
 *   defgrad (F = expm(L)), cells (C = C0 F^T; rows are lattice vectors), cell_velocities (the cell rows' FIRE
 *   velocities).  Initial state: L = 0, F = I, C = C0, cell velocities 0.
 *   A step moves L += dr_cell, F = expm(L), C = C0 F^T and x_i = F_new (F^-1 x_i + dr_i); |dr| and the maxstep cap
 *   run over all n + 3 rows, and convergence is max over the n + 3 rows of |row|^2 < fmax^2.
 *   Status 4 (cell degenerate): |det C| is not finite and > 0 (nothing else is written), or expm(L) of the step is not
 *   finite (velocities and FIRE state are written, positions and the cell state are not); the crystal is frozen.
 * Rejected (ALIGNN_ERR_BAD_ARG, nothing enqueued): as alignn_b200_fire_step, and stress_rows != num_active or a
 * non-finite stress_wt. */
int alignn_b200_fire_cell_step(const alignn_b200_fire_cell_params* params, const int32_t* active, int64_t num_active,
                               const int64_t* atom_offsets, const int32_t* batch_offsets, int64_t num_crystals,
                               const float* grad, int64_t grad_rows, const float* stress, int64_t stress_rows,
                               double* positions, double* velocities, float* forces, double* cells0, double* logdef,
                               double* defgrad, double* cells, double* cell_velocities, double* cell_forces,
                               float* stress_out, double* fstate, int32_t* istate, alignn_stream_t stream);

/* Per-graph mean over node rows (dgl.nn.AvgPooling, alignn.py:325) and its backward. */
int alignn_b200_segment_mean(const float* x, const int32_t* graph_ptr /*[B+1]*/, int64_t B, int d, float* out,
                             alignn_stream_t stream);
int alignn_b200_segment_mean_backward(const float* g_out /*[B,d]*/, const int32_t* graph_ptr, int64_t B, int d,
                                      float* gx /*[N,d]*/, alignn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Development aids (A/B switches and tracing used by tools/; not needed by a caller of the path).
 * ---------------------------------------------------------------------------------------- */
void alignn_b200_debug_egc_flags(int flags);                /* bit 0: register-staged pass 2 instead of the ring */

#ifdef __cplusplus
}
#endif
#endif /* ALIGNN_B200_H */
