// Scalar helpers shared by the FIRE step kernels (fire_device.cu, fire_cell_device.cu) and, for the calculator's
// stress, the NPT step of md_device.cu.
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

// x / 160.21766208 in fp32, correctly rounded: the double quotient of two floats rounded to float is the correctly
// rounded float quotient (53 >= 2 * 24 + 2), and div_rn is the correctly rounded double quotient in this range
__device__ __forceinline__ float fdiv_rn(float x, float y) { return __double2float_rn(div_rn((double)x, (double)y)); }

// The calculator's Voigt stress (alignn/ff/calculators.py:328-346) of the model's fp32 [3,3] stress S:
// full_3x3_to_voigt_6_stress (xx, yy, zz, yz, xz, xy) * stress_wt / 160.21766208, fp32 left to right
__device__ __forceinline__ void calculator_stress(const float* S, float stress_wt, float sv[6]) {
  sv[0] = S[0];
  sv[1] = S[4];
  sv[2] = S[8];
  sv[3] = __fmul_rn(__fadd_rn(S[5], S[7]), 0.5f);
  sv[4] = __fmul_rn(__fadd_rn(S[2], S[6]), 0.5f);
  sv[5] = __fmul_rn(__fadd_rn(S[1], S[3]), 0.5f);
#pragma unroll
  for (int k = 0; k < 6; ++k) sv[k] = fdiv_rn(__fmul_rn(sv[k], stress_wt), 160.21766208f);
}

}  // namespace fire
}  // namespace alignn
