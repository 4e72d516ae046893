// Quasi-Newton relaxation steps for a batch of crystals relaxed together: ASE 3.22.1's `LBFGS` and `BFGS`
// (ase/optimize/lbfgs.py, ase/optimize/bfgs.py) with the convergence test and step limit of `Optimizer.converged` /
// `Dynamics.irun`, on the atoms alone or on ASE's `ExpCellFilter` -- what `ForceField.optimize_atoms(optimizer="LBFGS"
// or "BFGS", optimize_lattice=...)` (alignn/ff/ff.py:385-412) runs one crystal at a time on the forces and Voigt
// stress of `AlignnAtomwiseCalculator.calculate`.  oracle/qn_oracle.py is the specification.
//
// Both optimizers work on the m rows of one crystal: its n atoms (r = x, f = fp32(grad * force_multiplier) widened),
// or under the filter n + 3 rows (atom rows r_i = F^-1 x_i, f_i F, cell rows L and the filter's cell forces G;
// filter_common.cuh).  A thread owns rows t, t + kBlock, ... of every per-row vector; sums are block reductions in
// double in a fixed order (a xor butterfly per warp, then the warps in order), with no floating-point atomics, so every
// result depends on the crystal's own data only: bitwise repeatable and independent of the batch around it.
//
//   lbfgs_step_kernel (one launch per step, one CTA per crystal): rows, decision, the (s, y, rho) pair of the last step
//     into a ring of `slots` pairs, the two-loop recursion with H0 = 1 / alpha, the longest-row cap, set_positions.
//   bfgs_rows_kernel, bfgs_hdr_kernel, bfgs_rank2_kernel (alignn_b200_bfgs_update): rows and decision per crystal,
//     then dg = H dr and H -= df df^T / a + dg dg^T / b with several CTAs per crystal, kTileRows rows of H each.
//   bfgs_vtf_kernel, bfgs_vw_kernel, bfgs_move_kernel (alignn_b200_bfgs_apply, after torch.linalg.eigh of H):
//     w = V^T f / |omega| and dr = V w with several CTAs per crystal, then the cap and set_positions per crystal.
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"
#include "filter_common.cuh"

namespace alignn {
namespace qn {

using filter::ExpmScratch;
using filter::expm_block;
using fire::div_rn;
using fire::nan_max;

constexpr int kBlock = 256, kWarps = kBlock / 32;
constexpr int kTileRows = 32;                                   // rows of H (or of V) per CTA in the dense kernels
enum { kRunning = 0, kConverged = 1, kExhausted = 2, kBadInput = 3, kCellDegenerate = 4, kBreakdown = 5 };
enum { kIter = 0, kPairs = 1, kTaken = 2, kStatus = 3 };       // LBFGS istate columns
enum { kHasPrev = 0, kPending = 1 };                            // BFGS istate columns 0, 1 (2, 3 as LBFGS)

// sum of v over the block, the same value on every thread; sh holds kWarps doubles
__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                              // sh is free: every thread has read its last use
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < kWarps; ++k) s += sh[k];
  return s;
}

// NaN-propagating max of v over the block, the same value on every thread
__device__ __forceinline__ double block_max(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = sh[0];
#pragma unroll
  for (int k = 1; k < kWarps; ++k) s = nan_max(s, sh[k]);
  return s;
}

__device__ __forceinline__ double sq3(const double* v) {       // (v_x^2 + v_y^2) + v_z^2
  return __dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2]));
}

// The filter state of one crystal in shared memory (read only when cells relax)
struct CellSmem {
  double C0[9], L[9], F[9], Fi[9], W[9], G[9], Ln[9], Fn[9], EmL[9];
  double Y[36], EY[36];
  ExpmScratch scratch;
  int bad;
};

// One crystal's rows: positions r and forces f of row i (< m) as the optimizer sees them
template <bool kCell>
struct Rows {
  const double* x;                                              // the crystal's Cartesian positions
  const float* fc;                                              // its fp32 forces of this evaluation
  const CellSmem* cs;
  int64_t n;
  __device__ __forceinline__ void r(int64_t i, double* o) const {
    if (!kCell) {
      o[0] = x[3 * i]; o[1] = x[3 * i + 1]; o[2] = x[3 * i + 2];
    } else if (i < n) {                                         // solve(F, X.T).T
      const double x0 = x[3 * i], x1 = x[3 * i + 1], x2 = x[3 * i + 2];
      const double* Fi = cs->Fi;
#pragma unroll
      for (int k = 0; k < 3; ++k) o[k] = Fi[3 * k] * x0 + Fi[3 * k + 1] * x1 + Fi[3 * k + 2] * x2;
    } else {                                                    // the carried log-deformation L
#pragma unroll
      for (int k = 0; k < 3; ++k) o[k] = cs->L[3 * (i - n) + k];
    }
  }
  __device__ __forceinline__ void f(int64_t i, double* o) const {
    if (!kCell) {
      o[0] = fc[3 * i]; o[1] = fc[3 * i + 1]; o[2] = fc[3 * i + 2];
    } else if (i < n) {                                         // f_i F
      const double f0 = fc[3 * i], f1 = fc[3 * i + 1], f2 = fc[3 * i + 2];
      const double* F = cs->F;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        o[k] = __dadd_rn(__dadd_rn(__dmul_rn(f0, F[k]), __dmul_rn(f1, F[3 + k])), __dmul_rn(f2, F[6 + k]));
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) o[k] = cs->G[3 * (i - n) + k];
    }
  }
};

// The part every step kernel shares: slice checks, the filter's cell forces, the fp32 forces of this evaluation and
// the convergence decision.  Returns false (on every thread) when the crystal does not step; then its status is set.
template <bool kCell>
__device__ __forceinline__ bool rows_and_decision(int64_t c, int64_t n, int64_t b0, const float* __restrict__ grad,
                                                  float force_multiplier, float stress_wt, double fmax,
                                                  int32_t max_steps, const float* __restrict__ stress,
                                                  double* x, float* forces,
                                                  const double* __restrict__ cells0, const double* __restrict__ logdef,
                                                  const double* __restrict__ defgrad, const double* __restrict__ cells,
                                                  double* __restrict__ cell_forces, float* __restrict__ stress_out,
                                                  int32_t* st, CellSmem& cs, double* red) {
  const int t = threadIdx.x;
  if (kCell) {
    if (t < 9) {
      cs.C0[t] = cells0[9 * c + t];
      cs.L[t] = logdef[9 * c + t];
      cs.F[t] = defgrad[9 * c + t];
    }
    __syncthreads();
    if (t == 0) filter::cell_stress(cells, stress, stress_wt, stress_out, st, kCellDegenerate, c, cs.F, cs.Fi, cs.W, cs.bad);
    __syncthreads();
    if (cs.bad) return false;                                   // status 4: nothing else is read or written
    filter::cell_rows(t, cs.L, cs.W, cs.G, cell_forces, c, cs.Ln, cs.EmL, cs.Y, cs.EY, cs.scratch);
  }
  const int64_t m = n + (kCell ? 3 : 0);
  const float* gr = grad + 3 * b0;
  double fm = 0.0;
  Rows<kCell> rows{x, forces, &cs, n};
  for (int64_t i = t; i < m; i += kBlock) {
    if (i < n) {
#pragma unroll
      for (int k = 0; k < 3; ++k) forces[3 * i + k] = __fmul_rn(gr[3 * i + k], force_multiplier);
    }
    double f[3];
    rows.f(i, f);                                               // reads back only this thread's own writes
    fm = nan_max(fm, sq3(f));
  }
  fm = block_max(fm, red);
  const bool conv = fm < fmax * fmax;                           // Optimizer.converged: strict
  const bool done = conv || st[kTaken] >= max_steps;            // Dynamics.irun: nsteps < max_steps
  __syncthreads();                                              // every thread has read st before thread 0 writes it
  if (done && t == 0) st[kStatus] = conv ? kConverged : kExhausted;
  return !done;
}

// set_positions(r + dr) for one crystal: dr is in `step` (its rows), r from `rows`; under the filter the new cell
// first (L + dr_cell, Fn = expm, status 4 if not finite), then x_i = Fn (r_i + dr_i).  Also r0 = r, f0 = f.  Returns
// false when the cell is degenerate (nothing written but the status).
template <bool kCell>
__device__ __forceinline__ bool move(int64_t c, int64_t n, const Rows<kCell>& rows, const double* step, double* x,
                                     double* __restrict__ r0, double* __restrict__ f0, double* __restrict__ logdef,
                                     double* __restrict__ defgrad, double* __restrict__ cells, int32_t* st, CellSmem& cs) {
  const int t = threadIdx.x;
  if (kCell) {
    if (t < 9) cs.Ln[t] = __dadd_rn(cs.L[t], step[3 * n + t]);  // the cell rows are rows n, n+1, n+2
    __syncthreads();
    expm_block(cs.Ln, 3, cs.Fn, cs.scratch);
    if (t == 0) {
      bool fin = true;
#pragma unroll
      for (int k = 0; k < 9; ++k) fin = fin && isfinite(cs.Fn[k]);
      cs.bad = !fin;
      if (!fin) st[kStatus] = kCellDegenerate;
    }
    __syncthreads();
    if (cs.bad) return false;
  }
  const int64_t m = n + (kCell ? 3 : 0);
  for (int64_t i = t; i < m; i += kBlock) {
    double r[3], f[3], p[3];
    rows.r(i, r);
    rows.f(i, f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      p[k] = __dadd_rn(r[k], step[3 * i + k]);
      r0[3 * i + k] = r[k];
      f0[3 * i + k] = f[k];
    }
    if (i < n) {
      if (kCell) {
        const double* Fn = cs.Fn;
#pragma unroll
        for (int k = 0; k < 3; ++k) x[3 * i + k] = Fn[3 * k] * p[0] + Fn[3 * k + 1] * p[1] + Fn[3 * k + 2] * p[2];
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) x[3 * i + k] = p[k];
      }
    }
  }
  if (kCell && t < 9) {
    const int r = t / 3, q = t % 3;
    logdef[9 * c + t] = cs.Ln[t];
    defgrad[9 * c + t] = cs.Fn[t];
    cells[9 * c + t] = cs.C0[3 * r] * cs.Fn[3 * q] + cs.C0[3 * r + 1] * cs.Fn[3 * q + 1] + cs.C0[3 * r + 2] * cs.Fn[3 * q + 2];
  }
  return true;
}

// determine_step: the longest row of step (in place); scale by maxstep / longest when longest >= maxstep, then by
// damping.  Returns false (every thread) when the step is not finite.
__device__ __forceinline__ bool cap_rows(double* step, int64_t m, double maxstep, double damping, double* red) {
  const int t = threadIdx.x;
  double lm = 0.0;
  for (int64_t i = t; i < m; i += kBlock) lm = nan_max(lm, sqrt(sq3(step + 3 * i)));
  const double longest = block_max(lm, red);
  if (!isfinite(longest)) return false;
  const bool cap = longest >= maxstep;
  const double sc = cap ? div_rn(maxstep, longest) : 1.0;
  for (int64_t i = t; i < m; i += kBlock) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double d = step[3 * i + k];
      if (cap) d = __dmul_rn(d, sc);
      step[3 * i + k] = __dmul_rn(d, damping);
    }
  }
  return true;
}

template <bool kCell>
__global__ void __launch_bounds__(kBlock)
lbfgs_step_kernel(const alignn_b200_lbfgs_params p, const int32_t* __restrict__ active, const int64_t* __restrict__ atom_off,
                  const int32_t* __restrict__ batch_off, int64_t B, const float* __restrict__ grad, int64_t grad_rows,
                  const float* __restrict__ stress, double* __restrict__ x, float* __restrict__ forces,
                  const double* __restrict__ cells0, double* __restrict__ logdef, double* __restrict__ defgrad,
                  double* __restrict__ cells, double* __restrict__ cell_forces, float* __restrict__ stress_out,
                  double* __restrict__ r0, double* __restrict__ f0, double* __restrict__ work, double* __restrict__ s_ring,
                  double* __restrict__ y_ring, double* __restrict__ hist, int32_t* __restrict__ istate) {
  __shared__ double red[kWarps];
  __shared__ CellSmem cs;
  const int64_t c = active[blockIdx.x];
  if (c < 0 || c >= B) return;
  int32_t* st = istate + 4 * c;
  if (st[kStatus] != kRunning) return;                          // frozen crystals are not touched
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  const int64_t b0 = batch_off[blockIdx.x], b1 = batch_off[blockIdx.x + 1];
  if (b0 < 0 || b1 > grad_rows || b1 - b0 != n) {               // the batch slice is not this crystal's atoms
    if (threadIdx.x == 0) st[kStatus] = kBadInput;
    return;
  }
  const int t = threadIdx.x;
  const int64_t ro = g0 + (kCell ? 3 * c : 0), m = n + (kCell ? 3 : 0), len = 3 * m;
  double* xc = x + 3 * g0;
  float* fc = forces + 3 * g0;
  if (!rows_and_decision<kCell>(c, n, b0, grad, p.force_multiplier, p.stress_wt, p.fmax, p.max_steps, stress, xc, fc,
                                cells0, logdef, defgrad, cells, cell_forces, stress_out, st, cs, red))
    return;
  const Rows<kCell> rows{xc, fc, &cs, n};
  double* r0c = r0 + 3 * ro;
  double* f0c = f0 + 3 * ro;
  double* q = work + 3 * ro;
  double* S = s_ring + 3 * p.slots * ro;                        // slot j of this crystal: S + j * len
  double* Yr = y_ring + 3 * p.slots * ro;
  double* rho = hist + 2 * (int64_t)p.slots * c;
  double* alph = rho + p.slots;
  const int32_t k = st[kIter];

  // ---- update: the pair of the last step, s = r - r0, y = f0 - f, rho = 1 / y.s
  if (k > 0) {
    double ys = 0.0;
    for (int64_t i = t; i < m; i += kBlock) {
      double r[3], f[3];
      rows.r(i, r);
      rows.f(i, f);
#pragma unroll
      for (int e = 0; e < 3; ++e) ys += __dadd_rn(f0c[3 * i + e], -f[e]) * __dadd_rn(r[e], -r0c[3 * i + e]);
    }
    ys = block_sum(ys, red);
    const double rh = __drcp_rn(ys);
    if (!(isfinite(ys) && ys != 0.0 && isfinite(rh))) {        // breakdown: nothing else is written
      if (t == 0) st[kStatus] = kBreakdown;
      return;
    }
    const int32_t slot = (k - 1) % p.slots;
    for (int64_t i = t; i < m; i += kBlock) {
      double r[3], f[3];
      rows.r(i, r);
      rows.f(i, f);
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        S[slot * len + 3 * i + e] = __dadd_rn(r[e], -r0c[3 * i + e]);
        Yr[slot * len + 3 * i + e] = __dadd_rn(f0c[3 * i + e], -f[e]);
      }
    }
    if (t == 0) rho[slot] = rh;
  }

  // ---- the two-loop recursion on q = -f, over the last min(memory, k) pairs
  const int32_t np = k < p.memory ? k : p.memory;
  for (int64_t i = t; i < m; i += kBlock) {
    double f[3];
    rows.f(i, f);
#pragma unroll
    for (int e = 0; e < 3; ++e) q[3 * i + e] = -f[e];
  }
  for (int32_t j = np - 1; j >= 0; --j) {
    const int32_t slot = (k - np + j) % p.slots;
    const double* s = S + slot * len;
    const double* y = Yr + slot * len;
    double d = 0.0;
    for (int64_t e = 3 * t; e < len; e += 3 * kBlock) d += (s[e] * q[e] + s[e + 1] * q[e + 1]) + s[e + 2] * q[e + 2];
    d = block_sum(d, red);                                      // its syncs also publish thread 0's rho write
    const double a = __dmul_rn(rho[slot], d);
    if (t == 0) alph[slot] = a;
    for (int64_t e = 3 * t; e < len; e += 3 * kBlock)
#pragma unroll
      for (int u = 0; u < 3; ++u) q[e + u] = __dadd_rn(q[e + u], -__dmul_rn(a, y[e + u]));
  }
  const double H0 = __drcp_rn(p.alpha);
  for (int64_t e = 3 * t; e < len; e += 3 * kBlock)
#pragma unroll
    for (int u = 0; u < 3; ++u) q[e + u] = __dmul_rn(H0, q[e + u]);   // z = H0 q
  for (int32_t j = 0; j < np; ++j) {
    const int32_t slot = (k - np + j) % p.slots;
    const double* s = S + slot * len;
    const double* y = Yr + slot * len;
    double d = 0.0;
    for (int64_t e = 3 * t; e < len; e += 3 * kBlock) d += (y[e] * q[e] + y[e + 1] * q[e + 1]) + y[e + 2] * q[e + 2];
    d = block_sum(d, red);
    const double bj = __dmul_rn(rho[slot], d);
    const double ab = __dadd_rn(alph[slot], -bj);
    for (int64_t e = 3 * t; e < len; e += 3 * kBlock)
#pragma unroll
      for (int u = 0; u < 3; ++u) q[e + u] = __dadd_rn(q[e + u], __dmul_rn(s[e + u], ab));
  }
  for (int64_t e = 3 * t; e < len; e += 3 * kBlock)
#pragma unroll
    for (int u = 0; u < 3; ++u) q[e + u] = -q[e + u];           // p = -z

  // ---- determine_step, set_positions(r + dr)
  if (!cap_rows(q, m, p.maxstep, p.damping, red)) {
    if (t == 0) st[kStatus] = kBreakdown;
    return;
  }
  __syncthreads();                                              // the cell rows of q are read by threads 0..8
  if (!move<kCell>(c, n, rows, q, xc, r0c, f0c, logdef, defgrad, cells, st, cs)) return;
  if (t == 0) {
    st[kIter] = k + 1;
    st[kPairs] = np;
    st[kTaken] += 1;
  }
}

// ---- BFGS ------------------------------------------------------------------------------------------------------------
// r, f: this evaluation's rows (written by bfgs_rows_kernel); work: [3][rows][3] = dg, w, dr.

template <bool kCell>
__global__ void __launch_bounds__(kBlock)
bfgs_rows_kernel(const alignn_b200_bfgs_params p, const int32_t* __restrict__ active, const int64_t* __restrict__ atom_off,
                 const int32_t* __restrict__ batch_off, int64_t B, int64_t max_dim, const float* __restrict__ grad,
                 int64_t grad_rows, const float* __restrict__ stress, double* __restrict__ x, float* __restrict__ forces,
                 const double* __restrict__ cells0, const double* __restrict__ logdef, const double* __restrict__ defgrad,
                 const double* __restrict__ cells, double* __restrict__ cell_forces, float* __restrict__ stress_out,
                 const int64_t* __restrict__ h_off, const double* __restrict__ r0, double* __restrict__ r,
                 double* __restrict__ f, int32_t* __restrict__ istate) {
  __shared__ double red[kWarps];
  __shared__ CellSmem cs;
  const int64_t c = active[blockIdx.x];
  if (c < 0 || c >= B) return;
  int32_t* st = istate + 4 * c;
  if (st[kStatus] != kRunning) return;
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  const int64_t b0 = batch_off[blockIdx.x], b1 = batch_off[blockIdx.x + 1];
  const int64_t m = n + (kCell ? 3 : 0), len = 3 * m;
  if (b0 < 0 || b1 > grad_rows || b1 - b0 != n || len > max_dim || h_off[c + 1] - h_off[c] != len * len) {
    if (threadIdx.x == 0) st[kStatus] = kBadInput;
    return;
  }
  const int t = threadIdx.x;
  const int64_t ro = g0 + (kCell ? 3 * c : 0);
  double* xc = x + 3 * g0;
  float* fc = forces + 3 * g0;
  if (!rows_and_decision<kCell>(c, n, b0, grad, p.force_multiplier, p.stress_wt, p.fmax, p.max_steps, stress, xc, fc,
                                cells0, logdef, defgrad, cells, cell_forces, stress_out, st, cs, red)) {
    if (t == 0) st[kPending] = 0;
    return;
  }
  const Rows<kCell> rows{xc, fc, &cs, n};
  const double* r0c = r0 + 3 * ro;
  double* rc = r + 3 * ro;
  double* fcur = f + 3 * ro;
  const bool prev = st[kHasPrev] != 0;                          // r0 and f0 hold the previous step's rows
  double dm = 0.0;
  for (int64_t i = t; i < m; i += kBlock) {
    double rr[3], ff[3];
    rows.r(i, rr);
    rows.f(i, ff);
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      rc[3 * i + e] = rr[e];
      fcur[3 * i + e] = ff[e];
      if (prev) dm = nan_max(dm, fabs(__dadd_rn(rr[e], -r0c[3 * i + e])));
    }
  }
  dm = block_max(dm, red);
  if (t == 0) {
    st[kPending] = prev && !(dm < 1e-7);                        // H is None, or the same configuration again: no update
    st[kHasPrev] = 1;
    st[kTaken] += 1;
  }
}

// per crystal of a dense launch (blockIdx.x over crystals, blockIdx.y over row tiles): its rows and H, or false
__device__ __forceinline__ bool dense_crystal(int64_t c, int64_t B, bool cell, const int64_t* atom_off,
                                              const int64_t* h_off, int64_t dim, const int32_t* st, int64_t& ro,
                                              int64_t& len) {
  if (c < 0 || c >= B || st[kStatus] != kRunning) return false;
  const int64_t g0 = atom_off[c], m = atom_off[c + 1] - g0 + (cell ? 3 : 0);
  ro = g0 + (cell ? 3 * c : 0);
  len = 3 * m;
  if (dim > 0 && len != dim) return false;                      // apply: not this group's size (bfgs_move reports it)
  return h_off == nullptr || h_off[c + 1] - h_off[c] == len * len;
}

// dg = H dr, dr = r - r0: one warp per row of H, kTileRows rows per CTA
__global__ void __launch_bounds__(kBlock)
bfgs_hdr_kernel(const int32_t* __restrict__ active, int64_t B, int32_t cell, const int64_t* __restrict__ atom_off,
                const int64_t* __restrict__ h_off, const double* __restrict__ H, const double* __restrict__ r0,
                const double* __restrict__ r, double* __restrict__ dg, const int32_t* __restrict__ istate) {
  const int64_t c = active[blockIdx.x];
  int64_t ro, len;
  if (c < 0 || c >= B) return;
  const int32_t* st = istate + 4 * c;
  if (!dense_crystal(c, B, cell != 0, atom_off, h_off, 0, st, ro, len) || !st[kPending]) return;
  const double* Hc = H + h_off[c];
  const double *r0c = r0 + 3 * ro, *rc = r + 3 * ro;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t i0 = (int64_t)blockIdx.y * kTileRows, i1 = (len - i0 < kTileRows) ? len : i0 + kTileRows;
  for (int64_t i = i0 + w; i < i1; i += kWarps) {
    double acc = 0.0;
    for (int64_t j = lane; j < len; j += 32) acc += Hc[i * len + j] * __dadd_rn(rc[j], -r0c[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) dg[3 * ro + i] = acc;
  }
}

// a = dr.df and b = dr.dg over the whole crystal (df = f - f0), the same on every thread of every CTA that computes it
__device__ __forceinline__ void bfgs_ab(int64_t len, const double* r0c, const double* rc, const double* f0c,
                                        const double* fcur, const double* dgc, double* red, double& a, double& b) {
  double sa = 0.0, sb = 0.0;
  for (int64_t j = threadIdx.x; j < len; j += kBlock) {
    const double d = __dadd_rn(rc[j], -r0c[j]);
    sa += d * __dadd_rn(fcur[j], -f0c[j]);
    sb += d * dgc[j];
  }
  a = block_sum(sa, red);
  b = block_sum(sb, red);
}

__device__ __forceinline__ bool ab_ok(double a, double b) {
  return isfinite(a) && a != 0.0 && isfinite(b) && b != 0.0;
}

// H -= outer(df, df) / a + outer(dg, dg) / b on kTileRows rows of H per CTA; a breakdown (a or b zero or not finite)
// leaves H as it is, and bfgs_move_kernel reports it
__global__ void __launch_bounds__(kBlock)
bfgs_rank2_kernel(const int32_t* __restrict__ active, int64_t B, int32_t cell, const int64_t* __restrict__ atom_off,
                  const int64_t* __restrict__ h_off, double* __restrict__ H, const double* __restrict__ r0,
                  const double* __restrict__ f0, const double* __restrict__ r, const double* __restrict__ f,
                  const double* __restrict__ dg, const int32_t* __restrict__ istate) {
  __shared__ double red[kWarps];
  const int64_t c = active[blockIdx.x];
  int64_t ro, len;
  if (c < 0 || c >= B) return;
  const int32_t* st = istate + 4 * c;
  if (!dense_crystal(c, B, cell != 0, atom_off, h_off, 0, st, ro, len) || !st[kPending]) return;
  const int64_t i0 = (int64_t)blockIdx.y * kTileRows;
  if (i0 >= len) return;
  const double *r0c = r0 + 3 * ro, *rc = r + 3 * ro, *f0c = f0 + 3 * ro, *fc = f + 3 * ro, *dgc = dg + 3 * ro;
  double a, b;
  bfgs_ab(len, r0c, rc, f0c, fc, dgc, red, a, b);
  if (!ab_ok(a, b)) return;
  double* Hc = H + h_off[c];
  const int64_t i1 = (len - i0 < kTileRows) ? len : i0 + kTileRows;
  for (int64_t i = i0; i < i1; ++i) {
    const double dfi = __dadd_rn(fc[i], -f0c[i]), dgi = dgc[i];
    for (int64_t j = threadIdx.x; j < len; j += kBlock) {
      const double u = div_rn(__dmul_rn(dfi, __dadd_rn(fc[j], -f0c[j])), a), v = div_rn(__dmul_rn(dgi, dgc[j]), b);
      Hc[i * len + j] = __dadd_rn(Hc[i * len + j], -__dadd_rn(u, v));
    }
  }
}

// w_j = (f V)_j / |omega_j| for kTileRows = 32 columns j per CTA: lane j, the 8 warps over rows i, summed in order
__global__ void __launch_bounds__(kBlock)
bfgs_vtf_kernel(const int32_t* __restrict__ group, int64_t B, int32_t cell, int64_t dim,
                const int64_t* __restrict__ atom_off, const double* __restrict__ omega, const double* __restrict__ V,
                const double* __restrict__ f, double* __restrict__ w, const int32_t* __restrict__ istate) {
  __shared__ double part[kWarps][32];
  const int64_t c = group[blockIdx.x];
  int64_t ro, len;
  if (c < 0 || c >= B) return;
  if (!dense_crystal(c, B, cell != 0, atom_off, nullptr, dim, istate + 4 * c, ro, len)) return;
  const double* Vg = V + (int64_t)blockIdx.x * dim * dim;
  const double* fc = f + 3 * ro;
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int64_t j = (int64_t)blockIdx.y * 32 + lane;
  double acc = 0.0;
  if (j < dim)
    for (int64_t i = wp; i < dim; i += kWarps) acc += fc[i] * Vg[i * dim + j];
  part[wp][lane] = acc;
  __syncthreads();
  if (wp == 0 && j < dim) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < kWarps; ++k) s += part[k][lane];
    w[3 * ro + j] = div_rn(s, fabs(omega[(int64_t)blockIdx.x * dim + j]));
  }
}

// dr = V w: one warp per row of V, kTileRows rows per CTA
__global__ void __launch_bounds__(kBlock)
bfgs_vw_kernel(const int32_t* __restrict__ group, int64_t B, int32_t cell, int64_t dim,
               const int64_t* __restrict__ atom_off, const double* __restrict__ V, const double* __restrict__ w,
               double* __restrict__ dr, const int32_t* __restrict__ istate) {
  const int64_t c = group[blockIdx.x];
  int64_t ro, len;
  if (c < 0 || c >= B) return;
  if (!dense_crystal(c, B, cell != 0, atom_off, nullptr, dim, istate + 4 * c, ro, len)) return;
  const double* Vg = V + (int64_t)blockIdx.x * dim * dim;
  const double* wc = w + 3 * ro;
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int64_t i0 = (int64_t)blockIdx.y * kTileRows, i1 = (dim - i0 < kTileRows) ? dim : i0 + kTileRows;
  for (int64_t i = i0 + wp; i < i1; i += kWarps) {
    double acc = 0.0;
    for (int64_t j = lane; j < dim; j += 32) acc += Vg[i * dim + j] * wc[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) dr[3 * ro + i] = acc;
  }
}

// per crystal of the group: the update's breakdown test (a and b again, bitwise as bfgs_rank2_kernel took them), the
// longest-row cap, set_positions(r + dr), r0 = r, f0 = f
template <bool kCell>
__global__ void __launch_bounds__(kBlock)
bfgs_move_kernel(const alignn_b200_bfgs_params p, const int32_t* __restrict__ group, int64_t B, int64_t dim,
                 const int64_t* __restrict__ atom_off, double* __restrict__ x, const double* __restrict__ cells0,
                 double* __restrict__ logdef, double* __restrict__ defgrad, double* __restrict__ cells,
                 double* __restrict__ r0, double* __restrict__ f0, const double* __restrict__ r,
                 const double* __restrict__ f, double* __restrict__ work, int64_t rows_total,
                 int32_t* __restrict__ istate) {
  __shared__ double red[kWarps];
  __shared__ CellSmem cs;
  const int64_t c = group[blockIdx.x];
  if (c < 0 || c >= B) return;
  int32_t* st = istate + 4 * c;
  if (st[kStatus] != kRunning) return;
  const int t = threadIdx.x;
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0, m = n + (kCell ? 3 : 0), len = 3 * m;
  if (len != dim) {
    if (t == 0) st[kStatus] = kBadInput;
    return;
  }
  const int64_t ro = g0 + (kCell ? 3 * c : 0);
  const double *rc = r + 3 * ro, *fc = f + 3 * ro;
  double* r0c = r0 + 3 * ro;
  double* f0c = f0 + 3 * ro;
  double* step = work + 2 * 3 * rows_total + 3 * ro;
  if (st[kPending]) {
    double a, b;
    bfgs_ab(len, r0c, rc, f0c, fc, work + 3 * ro, red, a, b);
    if (!ab_ok(a, b)) {
      if (t == 0) st[kStatus] = kBreakdown;
      return;
    }
  }
  if (!cap_rows(step, m, p.maxstep, 1.0, red)) {
    if (t == 0) st[kStatus] = kBreakdown;
    return;
  }
  if (kCell) {
    if (t < 9) {
      cs.C0[t] = cells0[9 * c + t];
      cs.L[t] = rc[3 * n + t];                                  // the rows r the step started from
    }
  }
  __syncthreads();
  if (kCell) {
    if (t < 9) cs.Ln[t] = __dadd_rn(cs.L[t], step[3 * n + t]);
    __syncthreads();
    expm_block(cs.Ln, 3, cs.Fn, cs.scratch);
    if (t == 0) {
      bool fin = true;
#pragma unroll
      for (int k = 0; k < 9; ++k) fin = fin && isfinite(cs.Fn[k]);
      cs.bad = !fin;
      if (!fin) st[kStatus] = kCellDegenerate;
    }
    __syncthreads();
    if (cs.bad) return;
  }
  double* xc = x + 3 * g0;
  for (int64_t i = t; i < m; i += kBlock) {
    double pp[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      pp[k] = __dadd_rn(rc[3 * i + k], step[3 * i + k]);
      r0c[3 * i + k] = rc[3 * i + k];
      f0c[3 * i + k] = fc[3 * i + k];
    }
    if (i < n) {
      if (kCell) {
        const double* Fn = cs.Fn;
#pragma unroll
        for (int k = 0; k < 3; ++k) xc[3 * i + k] = Fn[3 * k] * pp[0] + Fn[3 * k + 1] * pp[1] + Fn[3 * k + 2] * pp[2];
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) xc[3 * i + k] = pp[k];
      }
    }
  }
  if (kCell && t < 9) {
    const int rr = t / 3, q = t % 3;
    logdef[9 * c + t] = cs.Ln[t];
    defgrad[9 * c + t] = cs.Fn[t];
    cells[9 * c + t] = cs.C0[3 * rr] * cs.Fn[3 * q] + cs.C0[3 * rr + 1] * cs.Fn[3 * q + 1] + cs.C0[3 * rr + 2] * cs.Fn[3 * q + 2];
  }
}

}  // namespace qn
}  // namespace alignn

extern "C" {

int alignn_b200_lbfgs_step(const alignn_b200_lbfgs_params* params, const int32_t* active, int64_t num_active,
                           const int64_t* atom_offsets, const int32_t* batch_offsets, int64_t num_crystals,
                           const float* grad, int64_t grad_rows, const float* stress, int64_t stress_rows,
                           double* positions, float* forces, const double* cells0, double* logdef, double* defgrad,
                           double* cells, double* cell_forces, float* stress_out, double* r0, double* f0, double* work,
                           double* s_ring, double* y_ring, double* history, int32_t* istate, alignn_stream_t stream) {
  using namespace alignn::qn;
  if (!params || num_active < 0 || grad_rows < 0 || num_crystals < 1 || num_active > num_crystals || num_active > INT32_MAX)
    return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_lbfgs_params p = *params;
  const bool cell = p.cell != 0;
  if (!(p.maxstep > 0.0) || !isfinite(p.maxstep) || !(p.alpha > 0.0) || !isfinite(p.alpha) || !isfinite(p.damping) ||
      !(p.fmax >= 0.0) || !isfinite(p.fmax) || p.memory < 1 || p.max_steps < 1 ||
      p.slots < (p.memory < p.max_steps ? p.memory : p.max_steps) || !isfinite(p.force_multiplier) ||
      (p.cell != 0 && p.cell != 1) || (cell && (!isfinite(p.stress_wt) || stress_rows != num_active)))
    return ALIGNN_ERR_BAD_ARG;
  if (num_active == 0) return ALIGNN_OK;
  if (!active || !atom_offsets || !batch_offsets || !grad || !positions || !forces || !r0 || !f0 || !work || !s_ring ||
      !y_ring || !history || !istate)
    return ALIGNN_ERR_BAD_ARG;
  if (cell && (!stress || !cells0 || !logdef || !defgrad || !cells || !cell_forces || !stress_out)) return ALIGNN_ERR_BAD_ARG;
  auto k = cell ? lbfgs_step_kernel<true> : lbfgs_step_kernel<false>;
  k<<<(unsigned)num_active, kBlock, 0, (cudaStream_t)stream>>>(
      p, active, atom_offsets, batch_offsets, num_crystals, grad, grad_rows, stress, positions, forces, cells0, logdef,
      defgrad, cells, cell_forces, stress_out, r0, f0, work, s_ring, y_ring, history, istate);
  return alignn::check_launch();
}

static bool bfgs_params_ok(const alignn_b200_bfgs_params& p) {
  return p.maxstep > 0.0 && isfinite(p.maxstep) && p.alpha > 0.0 && isfinite(p.alpha) && p.fmax >= 0.0 &&
         isfinite(p.fmax) && p.max_steps >= 1 && isfinite(p.force_multiplier) && (p.cell == 0 || p.cell == 1) &&
         (p.cell == 0 || isfinite(p.stress_wt));
}

int alignn_b200_bfgs_update(const alignn_b200_bfgs_params* params, const int32_t* active, int64_t num_active,
                            const int64_t* atom_offsets, const int32_t* batch_offsets, int64_t num_crystals,
                            int64_t max_dim, const float* grad, int64_t grad_rows, const float* stress,
                            int64_t stress_rows, double* positions, float* forces, const double* cells0,
                            const double* logdef, const double* defgrad, const double* cells, double* cell_forces,
                            float* stress_out, const int64_t* h_offsets, double* H, double* r0, double* f0, double* r,
                            double* f, double* work, int32_t* istate, alignn_stream_t stream) {
  using namespace alignn::qn;
  if (!params || num_active < 0 || grad_rows < 0 || num_crystals < 1 || num_active > num_crystals ||
      num_active > INT32_MAX || max_dim < 3)
    return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_bfgs_params p = *params;
  const bool cell = p.cell != 0;
  if (!bfgs_params_ok(p) || (cell && stress_rows != num_active)) return ALIGNN_ERR_BAD_ARG;
  const int64_t tiles = (max_dim + kTileRows - 1) / kTileRows;
  if (tiles > 65535) return ALIGNN_ERR_BAD_ARG;
  if (num_active == 0) return ALIGNN_OK;
  if (!active || !atom_offsets || !batch_offsets || !grad || !positions || !forces || !h_offsets || !H || !r0 || !f0 ||
      !r || !f || !work || !istate)
    return ALIGNN_ERR_BAD_ARG;
  if (cell && (!stress || !cells0 || !logdef || !defgrad || !cells || !cell_forces || !stress_out)) return ALIGNN_ERR_BAD_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  auto k = cell ? bfgs_rows_kernel<true> : bfgs_rows_kernel<false>;
  k<<<(unsigned)num_active, kBlock, 0, s>>>(p, active, atom_offsets, batch_offsets, num_crystals, max_dim, grad, grad_rows,
                                            stress, positions, forces, cells0, logdef, defgrad, cells, cell_forces,
                                            stress_out, h_offsets, r0, r, f, istate);
  int rc = alignn::check_launch();
  if (rc != ALIGNN_OK) return rc;
  const dim3 grid((unsigned)num_active, (unsigned)tiles);
  bfgs_hdr_kernel<<<grid, kBlock, 0, s>>>(active, num_crystals, p.cell, atom_offsets, h_offsets, H, r0, r, work, istate);
  rc = alignn::check_launch();
  if (rc != ALIGNN_OK) return rc;
  bfgs_rank2_kernel<<<grid, kBlock, 0, s>>>(active, num_crystals, p.cell, atom_offsets, h_offsets, H, r0, f0, r, f, work,
                                            istate);
  return alignn::check_launch();
}

int alignn_b200_bfgs_apply(const alignn_b200_bfgs_params* params, const int32_t* group, int64_t group_size, int64_t dim,
                           const double* omega, const double* eigenvectors, const int64_t* atom_offsets,
                           int64_t num_crystals, int64_t num_rows, double* positions, const double* cells0,
                           double* logdef, double* defgrad, double* cells, double* r0, double* f0, const double* r,
                           const double* f, double* work, int32_t* istate, alignn_stream_t stream) {
  using namespace alignn::qn;
  if (!params || group_size < 0 || group_size > INT32_MAX || num_crystals < 1 || dim < 3 || num_rows < 1)
    return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_bfgs_params p = *params;
  const bool cell = p.cell != 0;
  if (!bfgs_params_ok(p)) return ALIGNN_ERR_BAD_ARG;
  const int64_t tiles = (dim + kTileRows - 1) / kTileRows;
  if (tiles > 65535) return ALIGNN_ERR_BAD_ARG;
  if (group_size == 0) return ALIGNN_OK;
  if (!group || !omega || !eigenvectors || !atom_offsets || !positions || !r0 || !f0 || !r || !f || !work || !istate)
    return ALIGNN_ERR_BAD_ARG;
  if (cell && (!cells0 || !logdef || !defgrad || !cells)) return ALIGNN_ERR_BAD_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t R3 = 3 * num_rows;
  const dim3 grid((unsigned)group_size, (unsigned)tiles);
  bfgs_vtf_kernel<<<grid, kBlock, 0, s>>>(group, num_crystals, p.cell, dim, atom_offsets, omega, eigenvectors, f,
                                          work + R3, istate);
  int rc = alignn::check_launch();
  if (rc != ALIGNN_OK) return rc;
  bfgs_vw_kernel<<<grid, kBlock, 0, s>>>(group, num_crystals, p.cell, dim, atom_offsets, eigenvectors, work + R3,
                                         work + 2 * R3, istate);
  rc = alignn::check_launch();
  if (rc != ALIGNN_OK) return rc;
  auto k = cell ? bfgs_move_kernel<true> : bfgs_move_kernel<false>;
  k<<<(unsigned)group_size, kBlock, 0, s>>>(p, group, num_crystals, dim, atom_offsets, positions, cells0, logdef, defgrad,
                                            cells, r0, f0, r, f, work, num_rows, istate);
  return alignn::check_launch();
}

}  // extern "C"
