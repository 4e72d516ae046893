// Batched equation-of-state fits: ASE 3.22.1's `EquationOfState(v, e, eos).fit()` (ase/eos.py) for the Murnaghan,
// Birch-Murnaghan and Vinet forms, what `ev_curve` (alignn/ff/ff.py:762-805) runs on one crystal's E(V) points.
// oracle/eos_oracle.py restates ASE's fit and gives the fully converged least-squares optimum the kernel is tested
// against.
//
// alignn_b200_eos_fit: one warp per row (volumes[r, :], energies[r, :], S points), kRowsPerBlock rows per CTA:
//   0. every volume finite and > 0 and every energy finite, else status 3 and NaN parameters;
//   1. seed: the least-squares parabola e = a + b V + c V^2 (ASE's first curve_fit, a linear problem), formed in
//      t = (V - mean V) / (half the volume range) with the energies centred, because the raw Vandermonde is badly
//      conditioned for volumes of 10-2000 A^3 spread over +-15 %; then vmin = -b / 2c and the seed is
//      (parabola(vmin), 2 c vmin, 4, vmin).  A non-finite seed (c = 0, all volumes equal) is status 2;
//   2. Levenberg-Marquardt from the seed on 0.5 sum r^2, r = E(V; p) - e, with the analytic Jacobian: the damped normal
//      equations (J^T J + lambda diag(D^2)) d = -J^T r, D^2 the running maximum of diag(J^T J) (MINPACK's scaling),
//      solved by a 4 x 4 Cholesky in registers; Nielsen's update of lambda.  A trial point whose sums are not all finite
//      (a residual, J^T J or J^T r) is rejected like an uphill step.  The fit stops when one iteration's step and its
//      cost change have both stalled at fp64 level -- |D d| <= kXtol |D p|, and the predicted and actual decreases
//      both <= kFtol of the cost -- or when the cost is exactly 0; after ALIGNN_B200_EOS_MAX_ITER iterations without
//      that it is status 2 with NaN parameters;
//   3. status 1 when V0 is not strictly inside (min V, max V): ASE only warns, so the parameters are written.
// Every lane holds the same parameters and takes the same branches: the per-point terms are summed lane by lane in
// point order and then by an xor-shuffle butterfly, whose every level adds the same two values on both partner lanes,
// so all lanes end with the same bits.  No atomics and nothing shared between rows: a row's result depends on its own
// data only, so it is bitwise repeatable and the same in any batch.
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace eos {

constexpr int kRowsPerBlock = 4;
constexpr int kBlock = 32 * kRowsPerBlock;
constexpr double kFtol = 1e-15;
constexpr double kXtol = 1e-15;
constexpr double kLambda0 = 1e-3;
enum { kOk = 0, kOutside = 1, kNoFit = 2, kBadInput = 3 };
constexpr int kSums = 15;                         // cost, J^T J (10, upper triangle by rows), J^T r (4)

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// E(V; p) and dE/dp for p = (E0, B0, BP, V0), ASE's formulas (ase/eos.py).  j[0] = dE/dE0 = 1 is implicit.
__device__ __forceinline__ double model(int form, double v, const double p[4], double j[4]) {
  const double E0 = p[0], B0 = p[1], BP = p[2], V0 = p[3];
  j[0] = 1.0;
  if (form == ALIGNN_B200_EOS_MURNAGHAN) {
    // E0 + B0 V / BP * ((V0/V)^BP / (BP - 1) + 1) - V0 B0 / (BP - 1)
    const double a = BP - 1.0, x = V0 / v, xb = pow(x, BP);
    const double g = (xb / a + 1.0) / BP;
    j[1] = v * g - V0 / a;
    j[2] = B0 * v * ((xb * log(x) / a - xb / (a * a)) / BP - g / BP) + V0 * B0 / (a * a);
    j[3] = B0 / a * (xb / x - 1.0);
    return E0 + B0 * v * g - V0 * B0 / a;
  }
  if (form == ALIGNN_B200_EOS_BIRCH_MURNAGHAN) {
    // eta = (V0/V)^(1/3); E0 + 9 B0 V0 / 16 (eta^2 - 1)^2 (6 + BP (eta^2 - 1) - 4 eta^2)
    const double eta = cbrt(V0 / v), e2 = eta * eta, u = e2 - 1.0, h = 6.0 + BP * u - 4.0 * e2, k = 9.0 / 16.0;
    j[1] = k * V0 * u * u * h;
    j[2] = k * B0 * V0 * u * u * u;
    j[3] = k * B0 * (u * u * h + (4.0 / 3.0) * e2 * u * h + u * u * (2.0 * BP - 8.0) * e2 / 3.0);
    return E0 + k * B0 * V0 * u * u * h;
  }
  // vinet: eta = (V/V0)^(1/3); E0 + 2 B0 V0 / (BP - 1)^2 (2 - (5 + 3 BP (eta - 1) - 3 eta) exp(-3 (BP - 1)(eta - 1) / 2))
  const double eta = cbrt(v / V0), w = eta - 1.0, a = BP - 1.0;
  const double q = 5.0 + 3.0 * BP * w - 3.0 * eta, ex = exp(-1.5 * a * w), Z = 2.0 - q * ex;
  j[1] = 2.0 * V0 / (a * a) * Z;
  j[2] = 2.0 * B0 * V0 * (-2.0 * Z / (a * a * a) - ex * w * (3.0 - 1.5 * q) / (a * a));
  j[3] = 2.0 * B0 / (a * a) * (Z + ex * eta * a * (1.0 - 0.5 * q));
  return E0 + 2.0 * B0 * V0 / (a * a) * Z;
}

// The row's sums at p, identical on every lane: s[0] = sum r^2, s[1..10] = J^T J (rows of the upper triangle),
// s[11..14] = J^T r.
__device__ __forceinline__ void sums(int form, const double* v, const double* e, int S, int lane, const double p[4],
                                     double s[kSums]) {
#pragma unroll
  for (int k = 0; k < kSums; ++k) s[k] = 0.0;
  for (int i = lane; i < S; i += 32) {
    double j[4];
    const double r = __dsub_rn(model(form, v[i], p, j), e[i]);
    s[0] = __fma_rn(r, r, s[0]);
    int k = 1;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
      for (int b = a; b < 4; ++b, ++k) s[k] = __fma_rn(j[a], j[b], s[k]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) s[11 + a] = __fma_rn(j[a], r, s[11 + a]);
  }
#pragma unroll
  for (int k = 0; k < kSums; ++k) s[k] = warp_sum(s[k]);
}

__device__ __forceinline__ bool all_finite(const double s[kSums]) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < kSums; ++k) ok &= isfinite(s[k]);
  return ok;
}

// Solves (A + lambda diag(D2)) d = -g by Cholesky, A the packed upper triangle s[1..10], g = s[11..14].  False when the
// damped matrix is not numerically positive definite.
__device__ __forceinline__ bool damped_step(const double s[kSums], const double D2[4], double lambda, double d[4]) {
  double L[4][4];
  int k = 1;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
#pragma unroll
    for (int b = a; b < 4; ++b, ++k) L[b][a] = s[k];        // lower triangle of the symmetric matrix
    L[a][a] = __fma_rn(lambda, D2[a], L[a][a]);
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    double dd = L[c][c];
#pragma unroll
    for (int m = 0; m < c; ++m) dd = __fma_rn(-L[c][m], L[c][m], dd);
    if (!(dd > 0.0) || !isfinite(dd)) return false;
    const double lc = sqrt(dd);
    L[c][c] = lc;
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      double x = L[r][c];
#pragma unroll
      for (int m = 0; m < c; ++m) x = __fma_rn(-L[r][m], L[c][m], x);
      L[r][c] = x / lc;
    }
  }
  double y[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    double x = -s[11 + r];
#pragma unroll
    for (int m = 0; m < r; ++m) x = __fma_rn(-L[r][m], y[m], x);
    y[r] = x / L[r][r];
  }
#pragma unroll
  for (int r = 3; r >= 0; --r) {
    double x = y[r];
#pragma unroll
    for (int m = r + 1; m < 4; ++m) x = __fma_rn(-L[m][r], d[m], x);
    d[r] = x / L[r][r];
  }
  bool ok = true;
#pragma unroll
  for (int r = 0; r < 4; ++r) ok &= isfinite(d[r]);
  return ok;
}

// Status and parameters of one row; every lane returns the same.
__device__ __forceinline__ int fit_row(int form, const double* v, const double* e, int S, int lane, double p[4]) {
  // ---- 0. input
  bool bad = false;
  double vlo = INFINITY, vhi = -INFINITY, vsum = 0.0, esum = 0.0;
  for (int i = lane; i < S; i += 32) {
    bad |= !(isfinite(v[i]) && v[i] > 0.0) || !isfinite(e[i]);
    vlo = fmin(vlo, v[i]);
    vhi = fmax(vhi, v[i]);
    vsum = __dadd_rn(vsum, v[i]);
    esum = __dadd_rn(esum, e[i]);
  }
  if (__any_sync(0xffffffffu, bad)) return kBadInput;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vlo = fmin(vlo, __shfl_xor_sync(0xffffffffu, vlo, o));
    vhi = fmax(vhi, __shfl_xor_sync(0xffffffffu, vhi, o));
  }
  const double vm = warp_sum(vsum) / S, em = warp_sum(esum) / S, h = 0.5 * (vhi - vlo);

  // ---- 1. the least-squares parabola in t = (V - vm) / h, energies centred: normal equations, 3 x 3 Cholesky
  double t1 = 0.0, t2 = 0.0, t3 = 0.0, t4 = 0.0, y0 = 0.0, y1 = 0.0, y2 = 0.0;
  for (int i = lane; i < S; i += 32) {
    const double t = (v[i] - vm) / h, tt = t * t, y = e[i] - em;
    t1 += t;
    t2 += tt;
    t3 += tt * t;
    t4 += tt * tt;
    y0 += y;
    y1 += t * y;
    y2 += tt * y;
  }
  t1 = warp_sum(t1); t2 = warp_sum(t2); t3 = warp_sum(t3); t4 = warp_sum(t4);
  y0 = warp_sum(y0); y1 = warp_sum(y1); y2 = warp_sum(y2);
  // [[S, t1, t2], [t1, t2, t3], [t2, t3, t4]] (alpha, beta, gamma) = (y0, y1, y2)
  const double l00 = sqrt((double)S), l10 = t1 / l00, l20 = t2 / l00;
  const double l11 = sqrt(t2 - l10 * l10), l21 = (t3 - l20 * l10) / l11;
  const double l22 = sqrt(t4 - l20 * l20 - l21 * l21);
  const double z0 = y0 / l00, z1 = (y1 - l10 * z0) / l11, z2 = (y2 - l20 * z0 - l21 * z1) / l22;
  const double gam = z2 / l22, bet = (z1 - l21 * gam) / l11, alp = (z0 - l10 * bet - l20 * gam) / l00;
  const double ts = -bet / (2.0 * gam);                        // the parabola's vertex in t
  const double vmin = vm + h * ts;
  p[0] = em + (alp + bet * ts + gam * ts * ts);
  p[1] = 2.0 * (gam / (h * h)) * vmin;                         // 2 c vmin, c = gamma / h^2
  p[2] = 4.0;
  p[3] = vmin;
  if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[3]))) return kNoFit;

  // ---- 2. Levenberg-Marquardt
  double s[kSums];
  sums(form, v, e, S, lane, p, s);
  if (!all_finite(s)) return kNoFit;
  double D2[4] = {0.0, 0.0, 0.0, 0.0};
  double lambda = kLambda0, nu = 2.0;
  bool done = s[0] == 0.0;
  for (int it = 0; it < ALIGNN_B200_EOS_MAX_ITER && !done; ++it) {
    D2[0] = fmax(D2[0], s[1]);
    D2[1] = fmax(D2[1], s[5]);
    D2[2] = fmax(D2[2], s[8]);
    D2[3] = fmax(D2[3], s[10]);
    double d[4];
    if (!damped_step(s, D2, lambda, d)) {
      lambda *= nu;
      nu *= 2.0;
      continue;
    }
    double q[4], sq[kSums];
#pragma unroll
    for (int a = 0; a < 4; ++a) q[a] = p[a] + d[a];
    sums(form, v, e, S, lane, q, sq);
    const double F = 0.5 * s[0], Fq = 0.5 * sq[0];
    double pred = 0.0, dn = 0.0, pn = 0.0;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      pred += d[a] * (lambda * D2[a] * d[a] - s[11 + a]);
      dn += D2[a] * d[a] * d[a];
      pn += D2[a] * p[a] * p[a];
    }
    pred *= 0.5;
    const bool finite = all_finite(sq);
    const bool stalled = finite && pred <= kFtol * F && fabs(F - Fq) <= kFtol * F && dn <= kXtol * kXtol * pn;
    if (finite && Fq < F) {
      const double rho = (F - Fq) / pred, c = 2.0 * rho - 1.0;
      lambda *= fmax(1.0 / 3.0, 1.0 - c * c * c);
      nu = 2.0;
#pragma unroll
      for (int a = 0; a < 4; ++a) p[a] = q[a];
#pragma unroll
      for (int k = 0; k < kSums; ++k) s[k] = sq[k];
    } else {
      lambda *= nu;
      nu *= 2.0;
    }
    done = stalled || s[0] == 0.0;
  }
  if (!done) return kNoFit;
  // ---- 3. ASE's warning
  return (vlo < p[3] && p[3] < vhi) ? kOk : kOutside;
}

__global__ void __launch_bounds__(kBlock)
eos_fit_kernel(const int form, const double* __restrict__ volumes, const double* __restrict__ energies,
               const int64_t rows, const int S, double* __restrict__ params, int32_t* __restrict__ status) {
  const int64_t r = (int64_t)blockIdx.x * kRowsPerBlock + (threadIdx.x >> 5);
  if (r >= rows) return;                                       // a whole warp leaves together
  const int lane = threadIdx.x & 31;
  double p[4];
  const int st = fit_row(form, volumes + r * S, energies + r * S, S, lane, p);
  if (lane == 0) {
    const bool keep = st == kOk || st == kOutside;
#pragma unroll
    for (int a = 0; a < 4; ++a) params[4 * r + a] = keep ? p[a] : __longlong_as_double(0x7ff8000000000000ll);
    status[r] = st;
  }
}

}  // namespace eos
}  // namespace alignn

extern "C" {

int alignn_b200_eos_fit(int32_t form, const double* volumes, const double* energies, int64_t rows, int32_t points,
                        double* params, int32_t* status, alignn_stream_t stream) {
  using namespace alignn::eos;
  if (form != ALIGNN_B200_EOS_MURNAGHAN && form != ALIGNN_B200_EOS_BIRCH_MURNAGHAN && form != ALIGNN_B200_EOS_VINET)
    return ALIGNN_ERR_BAD_ARG;
  if (rows < 0 || rows > (int64_t)INT32_MAX * kRowsPerBlock || points < 4 || points > ALIGNN_B200_EOS_MAX_POINTS)
    return ALIGNN_ERR_BAD_ARG;
  if (!volumes || !energies || !params || !status) return ALIGNN_ERR_BAD_ARG;
  if (rows == 0) return 0;
  const unsigned blocks = (unsigned)((rows + kRowsPerBlock - 1) / kRowsPerBlock);
  eos_fit_kernel<<<blocks, kBlock, 0, (cudaStream_t)stream>>>(form, volumes, energies, rows, points, params, status);
  return alignn::check_launch();
}

}  // extern "C"
