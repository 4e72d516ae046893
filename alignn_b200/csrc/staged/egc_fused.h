/* EXPERIMENTAL -- not part of libalignn_b200.so, not declared in include/alignn_b200.h.
 * Status: bit-identical to the shipped two-kernel forward (tests/test_staged.py) but not the shipped path.  On sm_90 the
 * accumulator tile lives in a per-CTA global scratch tile (acc_sm90.cuh), which costs L2 traffic the shipped path
 * does not pay.  The shipped forward is the two-pass composition of DESIGN.md.
 *
 * One-kernel forward of the edge side of EdgeGatedGraphConv (alignn/models/alignn.py:100-109,123,127):
 * the edge-gate Linear (`self.edge_gate(edge_feats)`, :101) runs on wgmma and the gate / segment-sum epilogue
 * consumes the accumulator tile, so G = edge_gate(y) is never written as a Linear output.
 * tools/build_staged.py builds this library into alignn_b200/csrc/staged/libalignn_b200_staged.so.
 */
#ifndef ALIGNN_B200_STAGED_EGC_FUSED_H
#define ALIGNN_B200_STAGED_EGC_FUSED_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALIGNN_FUSED_TILE_ROWS 128 /* in-edges (and destination nodes) per tile: the UMMA M */

/* Segment-aligned tiling of the destination-sorted edge list: tile i covers whole in-edge segments of the nodes
 * [v0, v0 + nseg) with rows <= 128 and nseg <= 128; descriptor = {v0, nseg, p0 = in_ptr[v0], rows}.
 * tiles == NULL: count only.  Returns the number of tiles, -1 on bad arguments, -2 if a node has more than 128
 * in-edges (the caller then keeps the two-kernel path). */
int64_t alignn_b200_segment_tiles_host(const int32_t* in_ptr, int64_t num_nodes, int32_t* tiles, int64_t capacity);

typedef struct {
  size_t struct_size;
  int64_t Nn, Ne;
  int32_t d;            /* 32, 64, 128 or 256; the gate Linear is d x d */
  int32_t norm_edges;   /* ALIGNN_NORM_STATS (train BatchNorm: M + column partials), ALIGNN_NORM_AFFINE (eval BatchNorm)
                           or ALIGNN_NORM_LAYER (LayerNorm) */
  int32_t residual;
  int32_t epilogue_groups; /* 1: four epilogue warps, 32-column chunks; 2: eight warps in two groups that alternate
                              16-column chunks (row phase of one overlaps the column phase of the other) */
  float gate_eps, ln_eps;
  const float* y;        /* [Ne,d] edge features = A operand of the gate GEMM */
  const void* w_image;   /* image of W_eg (alignn_b200_gemm_prepare_table, N=d, K=d) */
  const float* bias;     /* [d] edge_gate.bias */
  const float* P;        /* [Nn,4d] node projections [e_src | Bh | e_dst | src_update] */
  const int32_t* src; const int32_t* dst;
  const int32_t* in_ptr; const int32_t* in_eid;   /* in_eid NULL: edges already destination-sorted */
  const int32_t* tiles; int32_t num_tiles;
  const float* e_w; const float* e_b;             /* AFFINE: scale/shift; LAYER: gamma/beta */
  float* M;         /* [Ne,d] or NULL (inference) */
  float* y_out;     /* [Ne,d] or NULL; written for AFFINE / LAYER */
  float* XP;        /* [Nn,d] x' = src_update(x) + h  (always) */
  float* S; float* H; /* [Nn,d] or NULL (inference) */
  float* partials;  /* STATS: [min(num_tiles,132)][2][d] = column sums of m and m^2 */
  void* stream;
} alignn_b200_egc_fused_fwd_args;

int alignn_b200_egc_forward_fused(const alignn_b200_egc_fused_fwd_args* args);
int alignn_b200_egc_fused_partial_rows(int32_t num_tiles);

/* Node tail for LayerNorm models after the fused kernel: out = (res ? res : 0) + silu(LayerNorm(R) * gamma + beta),
 * rows [n,d] (alignn_atomwise.py:209-211 applied to x' = XP).  BatchNorm models use the shipped
 * rowstats_partials / bn_finalize / affine_silu_residual entry points on XP instead. */
int alignn_b200_ln_silu_residual(const float* R, const float* res, const float* gamma, const float* beta, float eps,
                                 float* out, int64_t n, int d, void* stream);
int alignn_b200_staged_last_cuda_error(void);

/* ---- backward, train-mode BatchNorm (ALIGNN_NORM_STATS) only -------------------------------------------------------
 * Node side (small, [Nn,d] rows): dL/dx' through the node BatchNorm + SiLU, and the two per-node factors the edge
 * side needs:  GPD = dL/dx' (goes to GP[:, 3d:4d]),  GSh = dL/dSh = dL/dx' / (S + eps),
 * GS = dL/dS = -dL/dx' * h / (S + eps);  partials [rows][d] = column sums of dL/dx' (bias gradient of src_update).
 * n_w / n_b = scale / shift of the batch statistics, n_c1 / n_c2 from alignn_b200_bn_backward_reduce. */
int alignn_b200_egc_backward_nodes(const float* XP, const float* gx_out, const float* S, const float* H, const float* n_w,
                                   const float* n_b, const float* n_mean, const float* n_rstd, const float* n_c1,
                                   const float* n_c2, float gate_eps, int64_t Nn, int d, float* GPD, int64_t ld_gpd,
                                   float* GSh, float* GS, float* partials, int partial_rows, void* stream);

/* Edge side in ONE tcgen05 kernel: the producer warps form  gm = dL/dm  per element from M, gy_out and the gathered
 * P[src, d:2d], GSh[dst], GS[dst] rows (BatchNorm + SiLU backward, gate backward), write GM and feed the bf16 hi/lo
 * split of the same values to the tensor cores;  gy = GM * W_eg (+ gy_out) leaves through the epilogue, which also
 * sums GM over every destination segment (GPB = GP[:, 2d:3d] = dL/d e_dst) -- i.e. egc_backward_dst_kernel's edge
 * loop and the data-gradient GEMM of alignn/models/alignn.py:101 in one pass over M and gy_out.
 * Same segment-aligned tiles as the forward kernel.  gy_out == NULL: dead edge output (no norm term, no residual). */
typedef struct {
  size_t struct_size;
  int64_t Nn, Ne;
  int32_t d;
  int32_t residual;
  const float* M; const float* gy_out;
  const float* P; const float* GSh; const float* GS;
  const void* w_image;   /* image of W_eg^T (alignn_b200_gemm_prepare_table, N=d, K=d, transpose=1) */
  const int32_t* src; const int32_t* dst; const int32_t* in_ptr; const int32_t* in_eid;
  const int32_t* tiles; int32_t num_tiles;
  const float* e_w; const float* e_b; const float* e_mean; const float* e_rstd; const float* e_c1; const float* e_c2;
  float* GM;             /* [Ne,d] */
  float* gy;             /* [Ne,d] or NULL */
  float* GPB; int64_t ld_gpb;   /* dL/d e_dst rows, e.g. GP + 2d with ld 4d */
  float* partials;       /* [min(num_tiles,132)][d] column sums of gm (= bias gradients of edge_gate and dst_gate) */
  void* stream;
} alignn_b200_egc_bwd_fused_args;

int alignn_b200_egc_backward_fused(const alignn_b200_egc_bwd_fused_args* args);

#ifdef __cplusplus
}
#endif
#endif
