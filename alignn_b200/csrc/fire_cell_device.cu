// One FIRE step on the atoms and the cell of a batch of crystals relaxed together: ASE 3.22.1's `ExpCellFilter`
// (ase/constraints.py) with FIRE run on it, as `ForceField.optimize_atoms(optimizer="FIRE", optimize_lattice=True)`
// (alignn/ff/ff.py:373-417, the reference's default) drives it with the forces and Voigt stress of
// `AlignnAtomwiseCalculator.calculate` (alignn/ff/calculators.py:280-372).  oracle/cell_filter_oracle.py is the
// specification; fire_device.cu is the same step with the cell held fixed.
//
// One CTA per running crystal, a fixed block size, and per crystal:
//   1. cell forces, in shared memory: the calculator's fp32 Voigt stress s (reported), V = |det C|, F^-1,
//      W = -V full(s) F^-T, expm(-L), the 6 x 6 expm(Y), Y = [[L, -W expm(-L)], [0, L]], G = -expm(Y)[0:3, 3:6]
//      symmetrised, and the filter's choice between G and W (np.isclose or a cosine above 0.8);
//   2. forces f = fp32(grad * force_multiplier) (reported) and the filter's atom rows f_i F; fixed-order block
//      reductions in double of F.v, F.F, v.v and the largest |row|^2 over the n + 3 rows, the cell rows added last;
//   3. thread 0: converged / out of steps / one FIRE update of (dt, a, Nsteps), exactly as fire_step_kernel;
//   4. velocities of the n + 3 rows, |dr|^2 over all of them, the whole-crystal maxstep cap;
//   5. the cell: L += dr_cell, Fn = expm(L), C = C0 Fn^T;
//   6. positions: x_i = Fn (F^-1 x_i + dr_i).
// The filter state carried per crystal is C0, L = log F, F and C.  ASE re-derives L = logm(solve(C0, C).T) every step;
// carrying it differs from that by rounding only.  Matrix exponentials: scaling and squaring of the degree-13 Pade
// approximant, |A / 2^s|_1 <= 5.37 (Higham 2005), on shared memory.  No floating-point atomics: every result depends on
// the crystal's own data and the fixed block size only, so it is bitwise repeatable and independent of the batch.
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"
#include "fire_common.cuh"

namespace alignn {
namespace fire_cell {

using fire::div_rn;
using fire::nan_max;

constexpr int kBlock = 256;
enum { kRunning = 0, kConverged = 1, kExhausted = 2, kBadInput = 3, kCellDegenerate = 4 };   // istate[c][3]
enum { kNsteps = 0, kFirst = 1, kTaken = 2, kStatus = 3 };      // istate columns
enum { kFrozen = 0, kFirstStep = 1, kMix = 2, kReset = 3 };     // what the velocity pass does

// shared scratch of one matrix exponential (n <= 6, row-major n x n)
struct ExpmScratch {
  double As[36], A2[36], A4[36], A6[36], X1[36], X2[36], X3[36];
  double scale;
  int s;
};

__device__ __forceinline__ double mm_entry(const double* A, const double* B, int n, int i, int j) {
  double acc = 0.0;
  for (int k = 0; k < n; ++k) acc += A[i * n + k] * B[k * n + j];
  return acc;
}

// out = expm(A) for an n x n matrix in shared memory (n <= 6); every thread of the block calls it.  A and out must not
// alias each other or the scratch.
__device__ void expm_block(const double* A, int n, double* out, ExpmScratch& w) {
  // Pade 13 coefficients b_0 .. b_13
  constexpr double b0 = 64764752532480000.0, b1 = 32382376266240000.0, b2 = 7771770303897600.0,
                   b3 = 1187353796428800.0, b4 = 129060195264000.0, b5 = 10559470521600.0, b6 = 670442572800.0,
                   b7 = 33522128640.0, b8 = 1323241920.0, b9 = 40840800.0, b10 = 960960.0, b11 = 16380.0, b12 = 182.0,
                   b13 = 1.0;
  constexpr double theta13 = 5.371920351148152;
  const int t = threadIdx.x, nn = n * n;
  const int i = t / n, j = t - (t / n) * n;
  const double eye = (i == j) ? 1.0 : 0.0;
  if (t == 0) {
    double norm = 0.0;                                          // 1-norm: the largest absolute column sum
    for (int c = 0; c < n; ++c) {
      double col = 0.0;
      for (int r = 0; r < n; ++r) col += fabs(A[r * n + c]);
      norm = nan_max(norm, col);
    }
    double sc = 1.0;
    int s = 0;
    while (norm > theta13 && s < 1000) {                        // halvings are exact; an infinite norm stops at 1000
      norm *= 0.5;
      sc *= 0.5;
      ++s;
    }
    w.scale = sc;
    w.s = s;
  }
  __syncthreads();
  if (t < nn) w.As[t] = A[t] * w.scale;
  __syncthreads();
  if (t < nn) w.A2[t] = mm_entry(w.As, w.As, n, i, j);
  __syncthreads();
  if (t < nn) w.A4[t] = mm_entry(w.A2, w.A2, n, i, j);
  __syncthreads();
  if (t < nn) {
    w.A6[t] = mm_entry(w.A4, w.A2, n, i, j);
  }
  __syncthreads();
  if (t < nn) {
    w.X1[t] = b13 * w.A6[t] + b11 * w.A4[t] + b9 * w.A2[t];
    w.X2[t] = b12 * w.A6[t] + b10 * w.A4[t] + b8 * w.A2[t];
  }
  __syncthreads();
  if (t < nn) {
    w.X3[t] = mm_entry(w.A6, w.X1, n, i, j) + b7 * w.A6[t] + b5 * w.A4[t] + b3 * w.A2[t] + b1 * eye;
    out[t] = mm_entry(w.A6, w.X2, n, i, j) + b6 * w.A6[t] + b4 * w.A4[t] + b2 * w.A2[t] + b0 * eye;   // V
  }
  __syncthreads();
  if (t < nn) w.X1[t] = mm_entry(w.As, w.X3, n, i, j);                                                    // U
  __syncthreads();
  if (t < nn) {
    const double u = w.X1[t], v = out[t];
    w.X2[t] = v - u;                                            // Q = V - U
    out[t] = v + u;                                             // P = V + U
  }
  __syncthreads();
  if (t == 0) {                                                 // Q X = P: Gaussian elimination, partial pivoting
    double* Q = w.X2;
    for (int k = 0; k < n; ++k) {
      int piv = k;
      for (int r = k + 1; r < n; ++r)
        if (fabs(Q[r * n + k]) > fabs(Q[piv * n + k])) piv = r;
      if (piv != k) {
        for (int c = 0; c < n; ++c) {
          const double q = Q[k * n + c]; Q[k * n + c] = Q[piv * n + c]; Q[piv * n + c] = q;
          const double p = out[k * n + c]; out[k * n + c] = out[piv * n + c]; out[piv * n + c] = p;
        }
      }
      for (int r = k + 1; r < n; ++r) {
        const double m = div_rn(Q[r * n + k], Q[k * n + k]);
        for (int c = k + 1; c < n; ++c) Q[r * n + c] -= m * Q[k * n + c];
        for (int c = 0; c < n; ++c) out[r * n + c] -= m * out[k * n + c];
      }
    }
    for (int k = n - 1; k >= 0; --k) {
      for (int c = 0; c < n; ++c) {
        double acc = out[k * n + c];
        for (int r = k + 1; r < n; ++r) acc -= Q[k * n + r] * out[r * n + c];
        out[k * n + c] = div_rn(acc, Q[k * n + k]);
      }
    }
  }
  __syncthreads();
  for (int q = 0; q < w.s; ++q) {                               // undo the scaling: s squarings
    if (t < nn) w.X1[t] = mm_entry(out, out, n, i, j);
    __syncthreads();
    if (t < nn) out[t] = w.X1[t];
    __syncthreads();
  }
}

// x / 160.21766208 in fp32, correctly rounded: the double quotient of two floats rounded to float is the correctly
// rounded float quotient (53 >= 2 * 24 + 2), and div_rn is the correctly rounded double quotient in this range
__device__ __forceinline__ float fdiv_rn(float x, float y) { return __double2float_rn(div_rn((double)x, (double)y)); }

__global__ void __launch_bounds__(kBlock)
fire_cell_step_kernel(const alignn_b200_fire_cell_params pc, const int32_t* __restrict__ active,
                      const int64_t* __restrict__ atom_off, const int32_t* __restrict__ batch_off, int64_t B,
                      const float* __restrict__ grad, int64_t grad_rows, const float* __restrict__ stress,
                      double* __restrict__ x, double* __restrict__ v, float* __restrict__ forces,
                      double* __restrict__ cells0, double* __restrict__ logdef, double* __restrict__ defgrad,
                      double* __restrict__ cells, double* __restrict__ cell_vel, double* __restrict__ cell_forces,
                      float* __restrict__ stress_out, double* __restrict__ fstate, int32_t* __restrict__ istate) {
  const alignn_b200_fire_params& p = pc.fire;
  __shared__ double red[kBlock][4];
  __shared__ double coef[5];                                    // dt, a (mixing), sqrt(F.F), sqrt(v.v), cap factor
  __shared__ double C0[9], L[9], F[9], Fi[9], W[9], G[9], Vc[9], Ln[9], Fn[9], EmL[9];
  __shared__ double Y[36], EY[36];
  __shared__ ExpmScratch scratch;
  __shared__ int mode, bad;
  const int64_t c = active[blockIdx.x];
  if (c < 0 || c >= B) return;
  int32_t* st = istate + 4 * c;
  if (st[kStatus] != kRunning) return;                          // frozen crystals are not touched
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  const int64_t b0 = batch_off[blockIdx.x], b1 = batch_off[blockIdx.x + 1];
  if (b0 < 0 || b1 > grad_rows || b1 - b0 != n) {               // the batch slice is not this crystal's atoms:
    if (threadIdx.x == 0) st[kStatus] = kBadInput;              // read nothing, report it
    return;
  }
  const float* gr = grad + 3 * b0;
  double* xc = x + 3 * g0;
  double* vc = v + 3 * g0;
  float* fc = forces + 3 * g0;
  const int t = threadIdx.x;

  // ---- 1. cell forces of this evaluation
  if (t < 9) {
    C0[t] = cells0[9 * c + t];
    L[t] = logdef[9 * c + t];
    F[t] = defgrad[9 * c + t];
    Vc[t] = cell_vel[9 * c + t];
  }
  __syncthreads();                                              // thread 0 reads the entries threads 1..8 stored
  if (t == 0) {
    const double* Cc = cells + 9 * c;
    const double V = fabs(Cc[0] * (Cc[4] * Cc[8] - Cc[5] * Cc[7]) - Cc[1] * (Cc[3] * Cc[8] - Cc[5] * Cc[6]) +
                          Cc[2] * (Cc[3] * Cc[7] - Cc[4] * Cc[6]));
    bad = !(isfinite(V) && V > 0.0);
    if (bad) {
      st[kStatus] = kCellDegenerate;
    } else {
      // full_3x3_to_voigt_6_stress (xx, yy, zz, yz, xz, xy) * stress_wt / 160.21766208, fp32 left to right
      const float* S = stress + 9 * blockIdx.x;
      float sv[6] = {S[0], S[4], S[8], __fmul_rn(__fadd_rn(S[5], S[7]), 0.5f), __fmul_rn(__fadd_rn(S[2], S[6]), 0.5f),
                     __fmul_rn(__fadd_rn(S[1], S[3]), 0.5f)};
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        sv[k] = fdiv_rn(__fmul_rn(sv[k], pc.stress_wt), 160.21766208f);
        stress_out[6 * c + k] = sv[k];
      }
      // F^-1 = adj(F) / det(F)
      const double* f = F;
      const double a00 = f[4] * f[8] - f[5] * f[7], a01 = f[2] * f[7] - f[1] * f[8], a02 = f[1] * f[5] - f[2] * f[4];
      const double a10 = f[5] * f[6] - f[3] * f[8], a11 = f[0] * f[8] - f[2] * f[6], a12 = f[2] * f[3] - f[0] * f[5];
      const double a20 = f[3] * f[7] - f[4] * f[6], a21 = f[1] * f[6] - f[0] * f[7], a22 = f[0] * f[4] - f[1] * f[3];
      const double det = f[0] * a00 + f[1] * a10 + f[2] * a20;
      Fi[0] = div_rn(a00, det); Fi[1] = div_rn(a01, det); Fi[2] = div_rn(a02, det);
      Fi[3] = div_rn(a10, det); Fi[4] = div_rn(a11, det); Fi[5] = div_rn(a12, det);
      Fi[6] = div_rn(a20, det); Fi[7] = div_rn(a21, det); Fi[8] = div_rn(a22, det);
      // W = -V full(s); W = solve(F, W.T).T = W F^-T
      const double s3[9] = {sv[0], sv[5], sv[4], sv[5], sv[1], sv[3], sv[4], sv[3], sv[2]};
      double w0[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) w0[k] = -V * s3[k];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int q = 0; q < 3; ++q)
          W[3 * r + q] = w0[3 * r] * Fi[3 * q] + w0[3 * r + 1] * Fi[3 * q + 1] + w0[3 * r + 2] * Fi[3 * q + 2];
    }
  }
  __syncthreads();
  if (bad) return;                                              // status 4: nothing else is read or written
  if (t < 9) Ln[t] = -L[t];
  __syncthreads();
  expm_block(Ln, 3, EmL, scratch);                              // expm(-L)
  if (t < 36) {
    const int r = t / 6, q = t % 6;
    double y = 0.0;
    if (r < 3 && q < 3) y = L[3 * r + q];
    else if (r >= 3 && q >= 3) y = L[3 * (r - 3) + q - 3];
    else if (r < 3) y = -(W[3 * r] * EmL[q - 3] + W[3 * r + 1] * EmL[3 + q - 3] + W[3 * r + 2] * EmL[6 + q - 3]);
    Y[t] = y;
  }
  __syncthreads();
  expm_block(Y, 6, EY, scratch);
  if (t == 0) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = 0; q < 3; ++q) G[3 * r + q] = -EY[6 * r + 3 + q];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int q = r + 1; q < 3; ++q) {
        const double ff = 0.5 * (G[3 * r + q] + G[3 * q + r]);
        G[3 * r + q] = ff;
        G[3 * q + r] = ff;
      }
    bool close = true;                                          // np.isclose(G, W): |G - W| <= 1e-8 + 1e-5 |W|
    double gw = 0.0, gg = 0.0, ww = 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const double a = G[k], b = W[k];
      close = close && ((a == b) || (fabs(a - b) <= 1e-8 + 1e-5 * fabs(b)));
      gw += a * b;
      gg += a * a;
      ww += b * b;
    }
    const bool exact = close || (gw / sqrt(gg * ww) > 0.8);     // a NaN cosine is not > 0.8
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (!exact) G[k] = W[k];
      cell_forces[9 * c + k] = G[k];
    }
  }
  __syncthreads();

  // ---- 2. forces, the filter's atom rows f_i F, and the sums FIRE and the convergence test need
  double fv = 0.0, ff = 0.0, vv = 0.0, fm = 0.0;
  for (int64_t i = t; i < n; i += kBlock) {
    float f[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      f[k] = __fmul_rn(gr[3 * i + k], p.force_multiplier);
      fc[3 * i + k] = f[k];
    }
    double f2 = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double fd = __dadd_rn(__dadd_rn(__dmul_rn(f[0], F[k]), __dmul_rn(f[1], F[3 + k])), __dmul_rn(f[2], F[6 + k]));
      const double vd = vc[3 * i + k];
      fv += fd * vd;
      ff += fd * fd;
      vv += vd * vd;
      f2 = __dadd_rn(f2, __dmul_rn(fd, fd));
    }
    fm = nan_max(fm, f2);
  }
  red[t][0] = fv; red[t][1] = ff; red[t][2] = vv; red[t][3] = fm;
  __syncthreads();
  for (int s = kBlock / 2; s > 0; s >>= 1) {
    if (t < s) {
      red[t][0] += red[t + s][0];
      red[t][1] += red[t + s][1];
      red[t][2] += red[t + s][2];
      red[t][3] = nan_max(red[t][3], red[t + s][3]);
    }
    __syncthreads();
  }

  // ---- 3. the decision and the scalar state (one thread); the cell rows join the sums first, in a fixed order
  if (t == 0) {
    double sfv = red[0][0], sff = red[0][1], svv = red[0][2], sfm = red[0][3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double f2 = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double fd = G[3 * r + k], vd = Vc[3 * r + k];
        sfv += fd * vd;
        sff += fd * fd;
        svv += vd * vd;
        f2 = __dadd_rn(f2, __dmul_rn(fd, fd));
      }
      sfm = nan_max(sfm, f2);
    }
    int m = kFrozen;
    if (sfm < p.fmax * p.fmax) {                                // Optimizer.converged on the filter: strict
      st[kStatus] = kConverged;
    } else if (st[kTaken] >= p.max_steps) {                     // Dynamics.irun: nsteps < max_steps
      st[kStatus] = kExhausted;
    } else {
      double* fs = fstate + 2 * c;
      double dt = fs[0], a = fs[1];
      coef[1] = a;                                              // the mix uses a before the a *= fa below
      if (st[kFirst]) {                                         // v is None: only v = 0
        st[kFirst] = 0;
        m = kFirstStep;
      } else if (sfv > 0.0) {                                   // vf > 0
        m = kMix;
        if (st[kNsteps] > p.n_min) {
          const double grown = __dmul_rn(dt, p.finc);
          dt = (p.dtmax < grown) ? p.dtmax : grown;             // Python min(dt * finc, dtmax)
          a = __dmul_rn(a, p.fa);
        }
        st[kNsteps] += 1;
      } else {
        m = kReset;
        a = p.astart;
        dt = __dmul_rn(dt, p.fdec);
        st[kNsteps] = 0;
      }
      st[kTaken] += 1;
      fs[0] = dt;
      fs[1] = a;
      coef[0] = dt;
      coef[2] = sqrt(sff);
      coef[3] = sqrt(svv);
    }
    mode = m;
  }
  __syncthreads();
  const int m = mode;
  if (m == kFrozen) return;
  const double dt = coef[0], am = coef[1], sf = coef[2], sv = coef[3];
  const double keep = __dadd_rn(1.0, -am);

  // ---- 4. velocities of the n + 3 rows, |dr|^2 over all of them
  double dr2 = 0.0;
  for (int64_t i = t; i < n; i += kBlock) {
    const double f0 = fc[3 * i], f1 = fc[3 * i + 1], f2 = fc[3 * i + 2];   // written by this thread above
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double fd = __dadd_rn(__dadd_rn(__dmul_rn(f0, F[k]), __dmul_rn(f1, F[3 + k])), __dmul_rn(f2, F[6 + k]));
      double vd = vc[3 * i + k];
      if (m == kFirstStep) vd = 0.0;
      else if (m == kMix) vd = __dadd_rn(__dmul_rn(keep, vd), __dmul_rn(div_rn(__dmul_rn(am, fd), sf), sv));
      else vd = __dmul_rn(vd, 0.0);                             // v[:] *= 0.0
      vd = __dadd_rn(vd, __dmul_rn(dt, fd));                    // v += dt * f
      vc[3 * i + k] = vd;
      const double dr = __dmul_rn(dt, vd);
      dr2 += dr * dr;
    }
  }
  if (t == 0) {                                                 // the cell rows, after this thread's atoms
    for (int k = 0; k < 9; ++k) {
      const double fd = G[k];
      double vd = Vc[k];
      if (m == kFirstStep) vd = 0.0;
      else if (m == kMix) vd = __dadd_rn(__dmul_rn(keep, vd), __dmul_rn(div_rn(__dmul_rn(am, fd), sf), sv));
      else vd = __dmul_rn(vd, 0.0);
      vd = __dadd_rn(vd, __dmul_rn(dt, fd));
      Vc[k] = vd;
      cell_vel[9 * c + k] = vd;
      const double dr = __dmul_rn(dt, vd);
      dr2 += dr * dr;
    }
  }
  __syncthreads();                                              // thread 0 is done reading red[0]
  red[t][0] = dr2;
  __syncthreads();
  for (int s = kBlock / 2; s > 0; s >>= 1) {
    if (t < s) red[t][0] += red[t + s][0];
    __syncthreads();
  }
  const double norm = sqrt(red[0][0]);
  const bool cap = norm > p.maxstep;

  // ---- 5. the cell: L += dr_cell, Fn = expm(L), C = C0 Fn^T
  if (t < 9) {
    double dr = __dmul_rn(dt, Vc[t]);
    if (cap) dr = div_rn(__dmul_rn(p.maxstep, dr), norm);       // maxstep * dr / normdr
    Ln[t] = __dadd_rn(L[t], dr);
  }
  __syncthreads();
  expm_block(Ln, 3, Fn, scratch);
  if (t == 0) {
    bool fin = true;
#pragma unroll
    for (int k = 0; k < 9; ++k) fin = fin && isfinite(Fn[k]);
    bad = !fin;
    if (bad) st[kStatus] = kCellDegenerate;
  }
  __syncthreads();
  if (bad) return;

  // ---- 6. positions x_i = Fn (F^-1 x_i + dr_i); the new filter state
  for (int64_t i = t; i < n; i += kBlock) {
    const double x0 = xc[3 * i], x1 = xc[3 * i + 1], x2 = xc[3 * i + 2];
    double r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double dr = __dmul_rn(dt, vc[3 * i + k]);
      if (cap) dr = div_rn(__dmul_rn(p.maxstep, dr), norm);
      r[k] = __dadd_rn(Fi[3 * k] * x0 + Fi[3 * k + 1] * x1 + Fi[3 * k + 2] * x2, dr);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) xc[3 * i + k] = Fn[3 * k] * r[0] + Fn[3 * k + 1] * r[1] + Fn[3 * k + 2] * r[2];
  }
  if (t < 9) {
    const int r = t / 3, q = t % 3;
    logdef[9 * c + t] = Ln[t];
    defgrad[9 * c + t] = Fn[t];
    cells[9 * c + t] = C0[3 * r] * Fn[3 * q] + C0[3 * r + 1] * Fn[3 * q + 1] + C0[3 * r + 2] * Fn[3 * q + 2];
  }
}

}  // namespace fire_cell
}  // namespace alignn

extern "C" {

int alignn_b200_fire_cell_step(const alignn_b200_fire_cell_params* params, const int32_t* active, int64_t num_active,
                               const int64_t* atom_offsets, const int32_t* batch_offsets, int64_t num_crystals,
                               const float* grad, int64_t grad_rows, const float* stress, int64_t stress_rows,
                               double* positions, double* velocities, float* forces, double* cells0, double* logdef,
                               double* defgrad, double* cells, double* cell_velocities, double* cell_forces,
                               float* stress_out, double* fstate, int32_t* istate, alignn_stream_t stream) {
  using namespace alignn::fire_cell;
  if (!params || num_active < 0 || grad_rows < 0 || num_crystals < 1 || num_active > num_crystals || num_active > INT32_MAX ||
      stress_rows != num_active)
    return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_fire_cell_params pc = *params;
  const alignn_b200_fire_params& p = pc.fire;
  if (!(p.maxstep > 0.0) || !(p.dtmax > 0.0) || !(p.fmax >= 0.0) || !isfinite(p.fmax) || !isfinite(p.finc) ||
      !isfinite(p.fdec) || !isfinite(p.astart) || !isfinite(p.fa) || p.n_min < 0 || p.max_steps < 1 ||
      !isfinite(p.force_multiplier) || !isfinite(pc.stress_wt))
    return ALIGNN_ERR_BAD_ARG;
  if (num_active == 0) return ALIGNN_OK;
  if (!active || !atom_offsets || !batch_offsets || !grad || !stress || !positions || !velocities || !forces || !cells0 ||
      !logdef || !defgrad || !cells || !cell_velocities || !cell_forces || !stress_out || !fstate || !istate)
    return ALIGNN_ERR_BAD_ARG;
  fire_cell_step_kernel<<<(unsigned)num_active, kBlock, 0, (cudaStream_t)stream>>>(
      pc, active, atom_offsets, batch_offsets, num_crystals, grad, grad_rows, stress, positions, velocities, forces, cells0,
      logdef, defgrad, cells, cell_velocities, cell_forces, stress_out, fstate, istate);
  return alignn::check_launch();
}

}  // extern "C"
