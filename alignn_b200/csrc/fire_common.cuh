// Scalar helpers shared by the FIRE step kernels (fire_device.cu, fire_cell_device.cu).
#pragma once

namespace alignn {
namespace fire {

// NaN-propagating max (numpy's max): once a NaN is seen it stays
__device__ __forceinline__ double nan_max(double m, double x) { return (x > m || x != x) ? x : m; }

// x / y rounded to nearest without the division's out-of-line slow path (which needs a stack frame): Markstein's
// correction of x * RN(1/y) with one fma is the correctly rounded quotient whenever no step overflows or underflows --
// forces, velocities and displacements are far inside that range.
__device__ __forceinline__ double div_rn(double x, double y) {
  const double r = __drcp_rn(y);
  const double q = __dmul_rn(x, r);
  return __fma_rn(__fma_rn(-y, q, x), r, q);
}

}  // namespace fire
}  // namespace alignn
