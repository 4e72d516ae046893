// ASE 3.22.1's `ExpCellFilter` on one CTA, shared by the filtered relaxation steps (fire_cell_device.cu and the
// quasi-Newton steps of qn_device.cu): the matrix exponential of a small matrix in shared memory and the filter's cell
// forces of one evaluation.  oracle/cell_filter_oracle.py is the specification.
#pragma once

#include <math.h>
#include <stdint.h>

#include "fire_common.cuh"

namespace alignn {
namespace filter {

using fire::div_rn;
using fire::nan_max;

constexpr int kStatusColumn = 3;                                // istate[c][3] of every relaxation step

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
// alias each other or the scratch.  Scaling and squaring of the degree-13 Pade approximant, |A / 2^s|_1 <= 5.37
// (Higham 2005).
static __device__ void expm_block(const double* A, int n, double* out, ExpmScratch& w) {
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

// The filter's cell rows of one evaluation (ExpCellFilter.get_forces), in two parts around the caller's
// `__syncthreads(); if (bad) return;`, after L and F = expm(L) are in shared memory and visible.  The quasi-Newton
// steps call these; fire_cell_step_kernel states the same lines inline, because calling them changes its register
// allocation and its SASS is kept as it was.
//
// cell_stress (thread 0 only): V = |det C| of cell c; if V is not finite and > 0, bad = 1 and st[3] = degenerate and
// nothing else is written; else bad = 0, the calculator's fp32 Voigt stress s of the model's stress in row blockIdx.x
// (written to stress_out[c]), F^-1 (Fi) and W = -V full(s) F^-T.
__device__ __forceinline__ void cell_stress(const double* cells, const float* stress, float stress_wt, float* stress_out,
                                            int32_t* st, int32_t degenerate, int64_t c, const double* F, double* Fi,
                                            double* W, int& bad) {
  const double* Cc = cells + 9 * c;
  const double V = fabs(Cc[0] * (Cc[4] * Cc[8] - Cc[5] * Cc[7]) - Cc[1] * (Cc[3] * Cc[8] - Cc[5] * Cc[6]) +
                        Cc[2] * (Cc[3] * Cc[7] - Cc[4] * Cc[6]));
  bad = !(isfinite(V) && V > 0.0);
  if (bad) {
    st[kStatusColumn] = degenerate;
  } else {
    float sv[6];
    fire::calculator_stress(stress + 9 * blockIdx.x, stress_wt, sv);
#pragma unroll
    for (int k = 0; k < 6; ++k) stress_out[6 * c + k] = sv[k];
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

// cell_rows (every thread of the block): expm(-L), the 6 x 6 expm(Y), Y = [[L, -W expm(-L)], [0, L]],
// G = -expm(Y)[0:3, 3:6] symmetrised, and the filter's choice between G and W (np.isclose or a cosine above 0.8),
// written to G and cell_forces[c].  Ln, EmL, Y and EY are scratch.
__device__ __forceinline__ void cell_rows(int t, const double* L, const double* W, double* G, double* cell_forces,
                                          int64_t c, double* Ln, double* EmL, double* Y, double* EY,
                                          ExpmScratch& scratch) {
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
}

}  // namespace filter
}  // namespace alignn
