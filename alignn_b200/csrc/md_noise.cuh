// Counter-based noise for the stochastic MD thermostats (csrc/md_device.cu), fully specified here so that a trajectory
// is a function of its arguments: no curand state, no hidden global stream.  oracle/md_thermostat_oracle.py restates
// every line of this file in numpy.
//
// Generator: Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11), with the
// multipliers 0xD2511F53 / 0xCD9E8D57 and the Weyl key increments 0x9E3779B9 / 0xBB67AE85 of Random123 and of CUDA's
// curand_philox4x32_x.h.  Ten rounds; the key is bumped between rounds (nine bumps).  One call maps a 128-bit counter
// and a 64-bit key to four 32-bit words w0..w3.
//
// Layout of the stream:
//   key     = (seed & 0xFFFFFFFF, seed >> 32), the crystal's 64-bit seed;
//   counter = (atom, step, block, tag):
//             atom  the atom's index within its crystal, or kComAtom = 0xFFFFFFFF for a per-crystal draw;
//             step  the index s of the MD step, 0 for the step that follows evaluation 0 (so s = e for the first half
//                   launched at evaluation e);
//             block the Philox block within (atom, step), 0, 1, 2, ...;
//             tag   the thermostat: kTagLangevin = 2 or kTagAndersen = 3 (the ensemble codes of the entry point).
//   Uniform q of (atom, step) comes from block q / 2: q even takes (hi, lo) = (w0, w1), q odd takes (w2, w3).
//   k = (hi << 20) | (lo >> 12) is a 52-bit integer, u = (k + 0.5) * 2^-52: exact in double, strictly inside (0, 1),
//   a multiple of 2^-53 (so 1 - u is exact as well).
//   Standard normals 2j and 2j + 1 of (atom, step) are the Box-Muller pair of uniforms 2j, 2j + 1 (block j):
//   r = sqrt(-2 log u_2j), z_2j = r cos(2 pi u_2j+1), z_2j+1 = r sin(2 pi u_2j+1).
// Draws of one (atom, step):
//   Langevin  normals 0..5 (blocks 0..2): xi_x, xi_y, xi_z, eta_x, eta_y, eta_z;
//   Andersen  uniforms 0..8 (blocks 0..4): x_k = u_k and y_k = u_{3+k} of boltzmann_random for component k, and the
//             reassignment chance c_k = u_{6+k}; the centre-of-mass kick of the crystal uses uniforms 0..5 of kComAtom
//             the same way.
// sincospi / cospi take 2u exactly and need no stack frame (sincos would); log and sqrt are CUDA's double log and the
// correctly rounded __dsqrt_rn, so a draw agrees with numpy's transcendental functions to a few ulp, not bitwise.
#pragma once
#include <stdint.h>

namespace alignn {
namespace md {

constexpr uint32_t kComAtom = 0xFFFFFFFFu;
constexpr uint32_t kTagLangevin = 2, kTagAndersen = 3;

struct Words4 {
  uint32_t w[4];
};

__host__ __device__ __forceinline__ Words4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                         uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
    const uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
  }
  return Words4{{c0, c1, c2, c3}};
}

__host__ __device__ __forceinline__ Words4 noise_block(uint64_t seed, uint32_t atom, uint32_t step, uint32_t block,
                                                       uint32_t tag) {
  return philox4x32_10(atom, step, block, tag, (uint32_t)seed, (uint32_t)(seed >> 32));
}

// (k + 0.5) * 2^-52 with k = (hi << 20) | (lo >> 12): both operations are exact
__host__ __device__ __forceinline__ double unit_uniform(uint32_t hi, uint32_t lo) {
  const uint64_t k = ((uint64_t)hi << 20) | (uint64_t)(lo >> 12);
  return ((double)k + 0.5) * 0x1.0p-52;
}

// Box-Muller on one block's two uniforms
__device__ __forceinline__ void box_muller(double u1, double u2, double& z0, double& z1) {
  const double r = __dsqrt_rn(__dmul_rn(-2.0, log(u1)));
  double s, c;
  sincospi(__dmul_rn(2.0, u2), &s, &c);
  z0 = __dmul_rn(r, c);
  z1 = __dmul_rn(r, s);
}

// the uniforms u_{2b}, u_{2b+1} of block b
__device__ __forceinline__ void block_uniforms(uint64_t seed, uint32_t atom, uint32_t step, uint32_t block, uint32_t tag,
                                               double& ua, double& ub) {
  const Words4 w = noise_block(seed, atom, step, block, tag);
  ua = unit_uniform(w.w[0], w.w[1]);
  ub = unit_uniform(w.w[2], w.w[3]);
}

// ASE's Andersen.boltzmann_random on two uniforms: width * cos(2 pi x) * (-2 log(1 - y)) ** 0.5, in numpy's order
__device__ __forceinline__ double boltzmann_random(double width, double x, double y) {
  return __dmul_rn(__dmul_rn(width, cospi(__dmul_rn(2.0, x))), __dsqrt_rn(__dmul_rn(-2.0, log(__dsub_rn(1.0, y)))));
}

}  // namespace md
}  // namespace alignn
