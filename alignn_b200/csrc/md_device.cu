// One evaluation of molecular dynamics for a batch of crystals run in lockstep: ASE 3.22.1's `VelocityVerlet` and
// `NVTBerendsen` (fixcm=True) with the run loop of `MolecularDynamics.irun` (ase/md/verlet.py, ase/md/nvtberendsen.py,
// ase/md/md.py), as `ForceField.run_nve_velocity_verlet` / `run_nvt_berendsen` (alignn/ff/ff.py:419-443, 510-543) drive
// them with the forces of `AlignnAtomwiseCalculator.calculate`.  oracle/md_oracle.py is the specification.
//
// One launch per evaluation e (0..steps), one CTA per crystal, a fixed block size; per crystal:
//   1. forces F = fp32(grad * force_multiplier), written to the reported-forces array;
//   2. e >= 1: the second half-kick of the previous step, p = p + (0.5 dt) F;
//   3. a fixed-order block reduction in double of p . (p / m): ekin and T of evaluation e into the caller's log rows;
//   4. e == steps: done.  Otherwise the first half of step e + 1: for Berendsen the velocity scale s from this T
//      (thread 0) and p = s p; the half-kick p += (0.5 dt) F; for Berendsen a second reduction of sum_i p_i and
//      p = p - sum / n; the drift x = x + (dt p) / m.
// The per-element updates use explicitly rounded operations in numpy's evaluation order (no contraction into FMAs), and
// every division is IEEE's correctly rounded one, so T0 / T at rest is +inf as in numpy; the sums differ from numpy's
// only in their order.  No floating-point atomics: every result depends on the crystal's own atoms and the fixed block
// size only, so it is bitwise repeatable and independent of the batch around it.
//
// md_thermostat_kernel does the same for ASE 3.22.1's stochastic thermostats `Langevin` and `Andersen` (fixcm=True;
// ase/md/langevin.py, ase/md/andersen.py), which `ForceField.run_nvt_langevin` / `run_nvt_andersen`
// (alignn/ff/ff.py:444-508) run; oracle/md_thermostat_oracle.py is its specification.  Their noise is the
// counter-based stream of md_noise.cuh, keyed by each crystal's own seed.
//
// md_npt_step_kernel runs ASE 3.22.1's `NPTBerendsen` (fixcm=True; ase/md/nptberendsen.py), which
// `ForceField.run_npt_berendsen` (alignn/ff/ff.py:545-582) runs: the Berendsen thermostat above plus a barostat that
// rescales each crystal's cell and positions every step on the calculator's stress; oracle/md_npt_oracle.py is its
// specification.
//
// md_nose_hoover_kernel runs ASE 3.22.1's `NPT` (Nose-Hoover thermostat and Parrinello-Rahman barostat;
// ase/md/npt.py), which `ForceField.run_npt_nose_hoover` (alignn/ff/ff.py:584-617) runs: a central difference in
// fractional coordinates, one model evaluation per step; oracle/md_nose_hoover_oracle.py is its specification.
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"
#include "fire_common.cuh"
#include "md_noise.cuh"

namespace alignn {
namespace md {

constexpr int kBlock = 256;
enum { kOk = 0, kBadInput = 3, kCellDegenerate = 4, kOneAtom = 6 };
enum { kNVE = 0, kBerendsen = 1, kLangevin = 2, kAndersen = 3 };

// sum over the block of three per-thread partials, in a fixed order; every thread returns the totals
__device__ __forceinline__ void block_sum3(double (*red)[3], double a, double b, double c, double out[3]) {
  const int t = threadIdx.x;
  __syncthreads();                                              // earlier readers of red are done
  red[t][0] = a; red[t][1] = b; red[t][2] = c;
  __syncthreads();
  for (int s = kBlock / 2; s > 0; s >>= 1) {
    if (t < s) {
      red[t][0] = __dadd_rn(red[t][0], red[t + s][0]);
      red[t][1] = __dadd_rn(red[t][1], red[t + s][1]);
      red[t][2] = __dadd_rn(red[t][2], red[t + s][2]);
    }
    __syncthreads();
  }
  out[0] = red[0][0]; out[1] = red[0][1]; out[2] = red[0][2];
}

// NVTBerendsen.scale_velocities' factor sqrt(1 + (T0/T - 1) * (dt/taut)), clipped by two Python ifs (a NaN passes both)
__device__ __forceinline__ double berendsen_scale(double T0, double T, double dt, double taut) {
  const double tautscl = __ddiv_rn(dt, taut);
  double s = __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(__dadd_rn(__ddiv_rn(T0, T), -1.0), tautscl)));
  if (s > 1.1) s = 1.1;
  if (s < 0.9) s = 0.9;
  return s;
}

__global__ void __launch_bounds__(kBlock)
md_step_kernel(const alignn_b200_md_params p, const int64_t* __restrict__ atom_off, const float* __restrict__ grad,
               int64_t grad_rows, const double* __restrict__ masses, const double* __restrict__ target_T,
               double* __restrict__ x, double* __restrict__ mom, float* __restrict__ forces,
               double* __restrict__ ekin_out, double* __restrict__ temp_out, int32_t* __restrict__ status) {
  __shared__ double red[kBlock][3];
  __shared__ double scale;
  const int64_t c = blockIdx.x;
  if (status[c] != kOk) return;                                 // a crystal already reported is not touched
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  if (g0 < 0 || n < 1 || atom_off[c + 1] > grad_rows) {         // the slice is not inside the batch: read nothing
    if (threadIdx.x == 0) status[c] = kBadInput;
    return;
  }
  const float* gr = grad + 3 * g0;
  const double* mc = masses + g0;
  double* xc = x + 3 * g0;
  double* pc = mom + 3 * g0;
  float* fc = forces + 3 * g0;
  const int t = threadIdx.x;
  const double dt = p.dt;
  const double half_dt = __dmul_rn(0.5, dt);                    // 0.5 * self.dt, then times the forces
  const bool berendsen = p.ensemble == kBerendsen;

  // ---- 1-3. forces of this evaluation, the second half-kick, p . (p / m)
  double kin = 0.0;
  for (int64_t i = t; i < n; i += kBlock) {
    const double m = mc[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float f = __fmul_rn(gr[3 * i + k], p.force_multiplier);
      fc[3 * i + k] = f;
      double pd = pc[3 * i + k];
      if (p.evaluation >= 1) {
        pd = __dadd_rn(pd, __dmul_rn(half_dt, (double)f));
        pc[3 * i + k] = pd;
      }
      kin = __dadd_rn(kin, __dmul_rn(pd, __ddiv_rn(pd, m)));
    }
  }
  double tot[3];
  block_sum3(red, kin, 0.0, 0.0, tot);
  const double ekin = __dmul_rn(0.5, tot[0]);
  const double T = __ddiv_rn(__dmul_rn(2.0, ekin), __dmul_rn((double)(3 * n), p.kB));   // 2 ekin / (dof kB)
  if (t == 0) {
    ekin_out[c] = ekin;
    temp_out[c] = T;
  }
  if (p.evaluation == p.steps) return;                          // the last evaluation: no step follows

  // ---- 4. the first half of the next step
  if (berendsen) {
    if (t == 0) scale = berendsen_scale(target_T[c], T, dt, p.taut);   // NVTBerendsen.scale_velocities
    __syncthreads();
    const double s = scale;
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int64_t i = t; i < n; i += kBlock) {
      double q[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double fd = fc[3 * i + k];                        // written by this thread above
        q[k] = __dadd_rn(__dmul_rn(s, pc[3 * i + k]), __dmul_rn(half_dt, fd));
        pc[3 * i + k] = q[k];
      }
      sx = __dadd_rn(sx, q[0]);
      sy = __dadd_rn(sy, q[1]);
      sz = __dadd_rn(sz, q[2]);
    }
    block_sum3(red, sx, sy, sz, tot);
    const double nd = (double)n;
    const double mean[3] = {__ddiv_rn(tot[0], nd), __ddiv_rn(tot[1], nd), __ddiv_rn(tot[2], nd)};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double pd = __dsub_rn(pc[3 * i + k], mean[k]);   // p = p - psum
        pc[3 * i + k] = pd;
        xc[3 * i + k] = __dadd_rn(xc[3 * i + k], __ddiv_rn(__dmul_rn(dt, pd), m));
      }
    }
  } else {
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double pd = __dadd_rn(pc[3 * i + k], __dmul_rn(half_dt, (double)fc[3 * i + k]));
        pc[3 * i + k] = pd;
        xc[3 * i + k] = __dadd_rn(xc[3 * i + k], __ddiv_rn(__dmul_rn(dt, pd), m));
      }
    }
  }
}

// ASE 3.22.1's `Langevin` and `Andersen` (fixcm=True), one launch per evaluation e, one CTA per crystal; the noise of
// the step that follows evaluation e is md_noise.cuh's stream at step index e.  Per crystal:
//   1. forces F = fp32(grad * force_multiplier), written out;
//   2. e >= 1: the second half of the previous step on the velocities v and (Langevin) rnd_vel the first half left in
//      the workspaces: Langevin v += c1 F/m - c2 v + rnd_vel; Andersen v += 0.5 F/m dt, v -= (m.v)/M; then p = v m;
//   3. ekin and T of evaluation e from p, as md_step_kernel;
//   4. e < steps: the first half of step e + 1 (see the header), ending with x = x_new and the workspaces holding the
//      velocities recomputed from the positions (and rnd_vel).
// Divisions by 2 and 8 are multiplications by 0.5 and 0.125, the same correctly rounded result.  Each division by n or
// M and every sum is as in md_step_kernel: IEEE, fixed order, no atomics.
__global__ void __launch_bounds__(kBlock)
md_thermostat_kernel(const alignn_b200_md_thermostat_params p, const int64_t* __restrict__ atom_off,
                     const float* __restrict__ grad, int64_t grad_rows, const double* __restrict__ masses,
                     const double* __restrict__ target_T, const uint64_t* __restrict__ seeds, double* __restrict__ x,
                     double* __restrict__ mom, double* __restrict__ vel, double* __restrict__ rvel,
                     float* __restrict__ forces, double* __restrict__ ekin_out, double* __restrict__ temp_out,
                     int32_t* __restrict__ status) {
  __shared__ double red[kBlock][3];
  const int64_t c = blockIdx.x;
  if (status[c] != kOk) return;
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  if (g0 < 0 || n < 1 || atom_off[c + 1] > grad_rows) {
    if (threadIdx.x == 0) status[c] = kBadInput;
    return;
  }
  const bool langevin = p.ensemble == kLangevin;
  if (langevin && n == 1) {                                     // ASE divides by n - 1.0 = 0
    if (threadIdx.x == 0) status[c] = kOneAtom;
    return;
  }
  const float* gr = grad + 3 * g0;
  const double* mc = masses + g0;
  double* xc = x + 3 * g0;
  double* pc = mom + 3 * g0;
  double* vc = vel + 3 * g0;
  double* rc = rvel + 3 * g0;
  float* fc = forces + 3 * g0;
  const int t = threadIdx.x;
  const double dt = p.dt, fr = p.friction;
  const double kT = __dmul_rn(p.kB, target_T[c]);              // units.kB * temperature_K
  const uint64_t seed = seeds[c];
  const uint32_t step = (uint32_t)p.evaluation;
  // Langevin.updatevars' scalars: c1 = dt/2. - dt*dt*fr/8., c2 = dt*fr/2 - dt*dt*fr*fr/8.
  const double c1 = __dsub_rn(__dmul_rn(dt, 0.5), __dmul_rn(__dmul_rn(__dmul_rn(dt, dt), fr), 0.125));
  const double c2 = __dsub_rn(__dmul_rn(__dmul_rn(dt, fr), 0.5),
                              __dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(dt, dt), fr), fr), 0.125));
  double tot[3];
  double M = 0.0;                                               // Andersen: masses.sum()
  if (!langevin) {
    double s = 0.0;
    for (int64_t i = t; i < n; i += kBlock) s = __dadd_rn(s, mc[i]);
    block_sum3(red, s, 0.0, 0.0, tot);
    M = tot[0];
  }

  // ---- 1-3. forces, the second half of the previous step, p . (p / m)
  double kin = 0.0;
  if (p.evaluation == 0) {
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        fc[3 * i + k] = __fmul_rn(gr[3 * i + k], p.force_multiplier);
        const double pd = pc[3 * i + k];
        kin = __dadd_rn(kin, __dmul_rn(pd, __ddiv_rn(pd, m)));
      }
    }
  } else if (langevin) {
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float f = __fmul_rn(gr[3 * i + k], p.force_multiplier);
        fc[3 * i + k] = f;
        double v = vc[3 * i + k];
        v = __dadd_rn(v, __dadd_rn(__dsub_rn(__ddiv_rn(__dmul_rn(c1, (double)f), m), __dmul_rn(c2, v)), rc[3 * i + k]));
        const double pd = __dmul_rn(v, m);                      // set_momenta(v * masses)
        pc[3 * i + k] = pd;
        kin = __dadd_rn(kin, __dmul_rn(pd, __ddiv_rn(pd, m)));
      }
    }
  } else {
    double s[3] = {0.0, 0.0, 0.0};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float f = __fmul_rn(gr[3 * i + k], p.force_multiplier);
        fc[3 * i + k] = f;
        const double v = __dadd_rn(vc[3 * i + k], __dmul_rn(__ddiv_rn(__dmul_rn(0.5, (double)f), m), dt));
        vc[3 * i + k] = v;
        s[k] = __dadd_rn(s[k], __dmul_rn(m, v));
      }
    }
    block_sum3(red, s[0], s[1], s[2], tot);
    const double vcm[3] = {__ddiv_rn(tot[0], M), __ddiv_rn(tot[1], M), __ddiv_rn(tot[2], M)};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double pd = __dmul_rn(__dsub_rn(vc[3 * i + k], vcm[k]), m);
        pc[3 * i + k] = pd;
        kin = __dadd_rn(kin, __dmul_rn(pd, __ddiv_rn(pd, m)));
      }
    }
  }
  block_sum3(red, kin, 0.0, 0.0, tot);
  const double ekin = __dmul_rn(0.5, tot[0]);
  const double T = __ddiv_rn(__dmul_rn(2.0, ekin), __dmul_rn((double)(3 * n), p.kB));
  if (t == 0) {
    ekin_out[c] = ekin;
    temp_out[c] = T;
  }
  if (p.evaluation == p.steps) return;

  // ---- 4. the first half of the next step
  const double nd = (double)n;
  if (langevin) {
    // draws, rnd_pos = c5 eta and rnd_vel = c3 xi - c4 eta; rnd_pos waits in the velocity workspace for the sums
    double sp[3] = {0.0, 0.0, 0.0}, sv[3] = {0.0, 0.0, 0.0};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
      const double sigma = __dsqrt_rn(__ddiv_rn(__dmul_rn(__dmul_rn(2.0, kT), fr), m));
      const double c3 = __dsub_rn(__dmul_rn(__dmul_rn(p.sqrt_dt, sigma), 0.5),
                                  __dmul_rn(__dmul_rn(__dmul_rn(p.dt_1_5, fr), sigma), 0.125));
      const double c5 = __ddiv_rn(__dmul_rn(p.dt_1_5, sigma), p.two_sqrt3);
      const double c4 = __dmul_rn(__dmul_rn(fr, 0.5), c5);
      double z[6], u0, u1;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        block_uniforms(seed, (uint32_t)i, step, (uint32_t)j, kTagLangevin, u0, u1);
        box_muller(u0, u1, z[2 * j], z[2 * j + 1]);
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double rp = __dmul_rn(c5, z[3 + k]);
        const double rv = __dsub_rn(__dmul_rn(c3, z[k]), __dmul_rn(c4, z[3 + k]));
        vc[3 * i + k] = rp;
        rc[3 * i + k] = rv;
        sp[k] = __dadd_rn(sp[k], rp);
        sv[k] = __dadd_rn(sv[k], __dmul_rn(rv, m));
      }
    }
    double spt[3];
    block_sum3(red, sp[0], sp[1], sp[2], spt);
    block_sum3(red, sv[0], sv[1], sv[2], tot);
    const double factor = __dsqrt_rn(__ddiv_rn(nd, __dsub_rn(nd, 1.0)));
    const double mp[3] = {__ddiv_rn(spt[0], nd), __ddiv_rn(spt[1], nd), __ddiv_rn(spt[2], nd)};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
      const double mn = __dmul_rn(m, nd);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double rp = __dmul_rn(__dsub_rn(vc[3 * i + k], mp[k]), factor);
        const double rv = __dmul_rn(__dsub_rn(rc[3 * i + k], __ddiv_rn(tot[k], mn)), factor);
        const double f = fc[3 * i + k];
        double v = __ddiv_rn(pc[3 * i + k], m);                 // get_velocities()
        v = __dadd_rn(v, __dadd_rn(__dsub_rn(__ddiv_rn(__dmul_rn(c1, f), m), __dmul_rn(c2, v)), rv));
        const double x0 = xc[3 * i + k];
        const double xn = __dadd_rn(__dadd_rn(x0, __dmul_rn(dt, v)), rp);
        xc[3 * i + k] = xn;
        vc[3 * i + k] = __ddiv_rn(__dsub_rn(__dsub_rn(xn, x0), rp), dt);
        rc[3 * i + k] = rv;
      }
    }
  } else {
    // the centre-of-mass kick: every thread draws the crystal's three components itself
    const double wcom = __dsqrt_rn(__ddiv_rn(kT, M));
    double u[6];
#pragma unroll
    for (int j = 0; j < 3; ++j) block_uniforms(seed, kComAtom, step, (uint32_t)j, kTagAndersen, u[2 * j], u[2 * j + 1]);
    const double kick[3] = {boltzmann_random(wcom, u[0], u[3]), boltzmann_random(wcom, u[1], u[4]),
                            boltzmann_random(wcom, u[2], u[5])};
    double sx[3] = {0.0, 0.0, 0.0}, sv[3] = {0.0, 0.0, 0.0};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
      const double w = __dsqrt_rn(__ddiv_rn(kT, m));
      double a[10];
#pragma unroll
      for (int j = 0; j < 5; ++j) block_uniforms(seed, (uint32_t)i, step, (uint32_t)j, kTagAndersen, a[2 * j], a[2 * j + 1]);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        double v = __dadd_rn(__ddiv_rn(pc[3 * i + k], m), kick[k]);
        v = __dadd_rn(v, __dmul_rn(__ddiv_rn(__dmul_rn(0.5, (double)fc[3 * i + k]), m), dt));
        if (a[6 + k] <= p.andersen_prob) v = boltzmann_random(w, a[k], a[3 + k]);
        vc[3 * i + k] = v;
        sx[k] = __dadd_rn(sx[k], __dmul_rn(m, xc[3 * i + k]));
        sv[k] = __dadd_rn(sv[k], __dmul_rn(m, v));
      }
    }
    double sxt[3];
    block_sum3(red, sx[0], sx[1], sx[2], sxt);
    block_sum3(red, sv[0], sv[1], sv[2], tot);
    const double old_com[3] = {__ddiv_rn(sxt[0], M), __ddiv_rn(sxt[1], M), __ddiv_rn(sxt[2], M)};
    const double vcm[3] = {__ddiv_rn(tot[0], M), __ddiv_rn(tot[1], M), __ddiv_rn(tot[2], M)};
    // x_new = x + v dt waits in the velocity workspace for the sum of m x_new
    double sn[3] = {0.0, 0.0, 0.0};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double xn = __dadd_rn(xc[3 * i + k], __dmul_rn(__dsub_rn(vc[3 * i + k], vcm[k]), dt));
        vc[3 * i + k] = xn;
        sn[k] = __dadd_rn(sn[k], __dmul_rn(m, xn));
      }
    }
    block_sum3(red, sn[0], sn[1], sn[2], tot);
    const double shift[3] = {__dsub_rn(__ddiv_rn(tot[0], M), old_com[0]), __dsub_rn(__ddiv_rn(tot[1], M), old_com[1]),
                             __dsub_rn(__ddiv_rn(tot[2], M), old_com[2])};
    for (int64_t i = t; i < n; i += kBlock) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double x0 = xc[3 * i + k];
        const double xn = __dsub_rn(vc[3 * i + k], shift[k]);  // set_center_of_mass(old_com)
        xc[3 * i + k] = xn;
        vc[3 * i + k] = __ddiv_rn(__dsub_rn(xn, x0), dt);
      }
    }
  }
}

// p_a p_b / m per Voigt component (xx yy zz yz xz xy) added to g: the terms of Atoms.get_stress(include_ideal_gas=True)
__device__ __forceinline__ void add_ideal_gas_terms(const double q[3], double invm, double g[6]) {
  g[0] = __dadd_rn(g[0], __dmul_rn(__dmul_rn(q[0], q[0]), invm));
  g[1] = __dadd_rn(g[1], __dmul_rn(__dmul_rn(q[1], q[1]), invm));
  g[2] = __dadd_rn(g[2], __dmul_rn(__dmul_rn(q[2], q[2]), invm));
  g[3] = __dadd_rn(g[3], __dmul_rn(__dmul_rn(q[1], q[2]), invm));
  g[4] = __dadd_rn(g[4], __dmul_rn(__dmul_rn(q[0], q[2]), invm));
  g[5] = __dadd_rn(g[5], __dmul_rn(__dmul_rn(q[0], q[1]), invm));
}

// the ideal-gas-corrected stress, in place on the fp32 array as ASE does it (out_k = fp32(s_k - G_k * invvol)), and its
// pressure -trace / 3: the trace in fp32, the division in double (numpy 1.x's scalar promotion)
__device__ __forceinline__ double corrected_pressure(const float sv[6], const double G[6], double invvol, float out[6]) {
#pragma unroll
  for (int k = 0; k < 6; ++k) out[k] = __double2float_rn(__dsub_rn((double)sv[k], __dmul_rn(G[k], invvol)));
  const float trace = __fadd_rn(__fadd_rn(out[0], out[1]), out[2]);
  return __ddiv_rn(-(double)trace, 3.0);
}

// ASE 3.22.1's `NPTBerendsen` (fixcm=True), which `ForceField.run_npt_berendsen` (alignn/ff/ff.py:545-582) runs;
// oracle/md_npt_oracle.py is its specification.  A step needs two evaluations: evaluation A at the rescaled structure,
// whose forces only drive the half-kick, and the logged evaluation B.  So two launches per step, one CTA per crystal:
//   phase 0, after logged evaluation e, in three passes over the atoms so that nothing is written before the checks:
//     1. F = fp32(grad * force_multiplier); e >= 1: p_e = p + (0.5 dt) F (else p_e = p); sums of p_e . (p_e / m) and of
//        the ideal-gas terms p_a p_b / m; ekin, T and the logged pressure from the calculator's Voigt stress s;
//     2. e < steps: s_T from T (NVTBerendsen.scale_velocities) and the ideal-gas sums of s_T p_e, the barostat's
//        pressure P and mu = 1 - (dt/taup) c / 3 (P0 - P);
//     3. F, p = s_T p_e, x = mu x, C = mu C, and the log rows written.
//   phase 1, after evaluation A of step e + 1: p += (0.5 dt) F_A, p -= sum_i p_i / n, x += (dt p) / m -- the same
//   operations as md_step_kernel's Berendsen branch, so with mu = 1 (no barostat) the trajectory is its trajectory.
// The cell's volume V = |det C| (cofactor expansion) and mu must be finite and > 0: otherwise status 4 and nothing of
// the crystal is written in phase 0.  ASE would carry on; a run with a collapsed or inverted cell means nothing.
__global__ void __launch_bounds__(kBlock)
md_npt_step_kernel(const alignn_b200_md_npt_params p, const int64_t* __restrict__ atom_off,
                   const float* __restrict__ grad, int64_t grad_rows, const float* __restrict__ stress,
                   const double* __restrict__ masses, const double* __restrict__ target_T,
                   const double* __restrict__ target_P, const double* __restrict__ compress, double* __restrict__ cells,
                   double* __restrict__ x, double* __restrict__ mom, float* __restrict__ forces,
                   float* __restrict__ stress_out, double* __restrict__ ekin_out, double* __restrict__ temp_out,
                   double* __restrict__ press_out, int32_t* __restrict__ status) {
  __shared__ double red[kBlock][3];
  const int64_t c = blockIdx.x;
  if (status[c] != kOk) return;
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  if (g0 < 0 || n < 1 || atom_off[c + 1] > grad_rows) {
    if (threadIdx.x == 0) status[c] = kBadInput;
    return;
  }
  const float* gr = grad + 3 * g0;
  const double* mc = masses + g0;
  double* xc = x + 3 * g0;
  double* pc = mom + 3 * g0;
  const int t = threadIdx.x;
  const double dt = p.dt;
  const double half_dt = __dmul_rn(0.5, dt);
  double tot[3];

  if (p.phase == 1) {
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int64_t i = t; i < n; i += kBlock) {
      double q[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double fd = (double)__fmul_rn(gr[3 * i + k], p.force_multiplier);
        q[k] = __dadd_rn(pc[3 * i + k], __dmul_rn(half_dt, fd));
        pc[3 * i + k] = q[k];
      }
      sx = __dadd_rn(sx, q[0]);
      sy = __dadd_rn(sy, q[1]);
      sz = __dadd_rn(sz, q[2]);
    }
    block_sum3(red, sx, sy, sz, tot);
    const double nd = (double)n;
    const double mean[3] = {__ddiv_rn(tot[0], nd), __ddiv_rn(tot[1], nd), __ddiv_rn(tot[2], nd)};
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double pd = __dsub_rn(pc[3 * i + k], mean[k]);
        pc[3 * i + k] = pd;
        xc[3 * i + k] = __dadd_rn(xc[3 * i + k], __ddiv_rn(__dmul_rn(dt, pd), m));
      }
    }
    return;
  }

  // ---- phase 0.  The cell of this evaluation (every thread forms the same V)
  double C[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) C[k] = cells[9 * c + k];
  const double V = fabs(C[0] * (C[4] * C[8] - C[5] * C[7]) - C[1] * (C[3] * C[8] - C[5] * C[6]) +
                        C[2] * (C[3] * C[7] - C[4] * C[6]));
  if (!(isfinite(V) && V > 0.0)) {
    if (t == 0) status[c] = kCellDegenerate;
    return;
  }
  const double invvol = __ddiv_rn(1.0, V);
  const bool kick = p.evaluation >= 1;

  // ---- 1. p_e, its kinetic energy and ideal-gas sums
  double kin = 0.0, g[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t i = t; i < n; i += kBlock) {
    const double m = mc[i];
    double q[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double pd = pc[3 * i + k];
      if (kick) pd = __dadd_rn(pd, __dmul_rn(half_dt, (double)__fmul_rn(gr[3 * i + k], p.force_multiplier)));
      q[k] = pd;
      kin = __dadd_rn(kin, __dmul_rn(pd, __ddiv_rn(pd, m)));
    }
    add_ideal_gas_terms(q, __ddiv_rn(1.0, m), g);
  }
  double G[6], rest[3];
  block_sum3(red, kin, g[0], g[1], tot);
  block_sum3(red, g[2], g[3], g[4], G + 2);
  block_sum3(red, g[5], 0.0, 0.0, rest);
  G[0] = tot[1];
  G[1] = tot[2];
  G[5] = rest[0];
  const double ekin = __dmul_rn(0.5, tot[0]);
  const double T = __ddiv_rn(__dmul_rn(2.0, ekin), __dmul_rn((double)(3 * n), p.kB));
  float sv[6], sc[6];
  fire::calculator_stress(stress + 9 * c, p.stress_wt, sv);
  const double P_log = corrected_pressure(sv, G, invvol, sc);

  // ---- 2. the barostat on the scaled momenta
  const bool step = p.evaluation < p.steps;
  double s = 1.0, mu = 1.0;
  if (step) {
    s = berendsen_scale(target_T[c], T, dt, p.taut);
    double h[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int64_t i = t; i < n; i += kBlock) {
      double q[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        double pd = pc[3 * i + k];
        if (kick) pd = __dadd_rn(pd, __dmul_rn(half_dt, (double)__fmul_rn(gr[3 * i + k], p.force_multiplier)));
        q[k] = __dmul_rn(s, pd);
      }
      add_ideal_gas_terms(q, __ddiv_rn(1.0, mc[i]), h);
    }
    double H[6];
    block_sum3(red, h[0], h[1], h[2], H);
    block_sum3(red, h[3], h[4], h[5], H + 3);
    const double P = corrected_pressure(sv, H, invvol, sc);
    const double taupscl = __ddiv_rn(dt, p.taup);
    mu = __dsub_rn(1.0, __dmul_rn(__ddiv_rn(__dmul_rn(taupscl, compress[c]), 3.0), __dsub_rn(target_P[c], P)));
    if (!(isfinite(mu) && mu > 0.0)) {
      if (t == 0) status[c] = kCellDegenerate;
      return;
    }
  }

  // ---- 3. the writes
  float* fc = forces + 3 * g0;
  for (int64_t i = t; i < n; i += kBlock) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float f = __fmul_rn(gr[3 * i + k], p.force_multiplier);
      fc[3 * i + k] = f;
      double pd = pc[3 * i + k];
      if (kick) pd = __dadd_rn(pd, __dmul_rn(half_dt, (double)f));
      if (step) {
        pd = __dmul_rn(s, pd);                                  // NVTBerendsen.scale_velocities
        xc[3 * i + k] = __dmul_rn(mu, xc[3 * i + k]);           // set_cell(mu C, scale_atoms=True)
      }
      pc[3 * i + k] = pd;
    }
  }
  if (t == 0) {
    ekin_out[c] = ekin;
    temp_out[c] = T;
    press_out[c] = P_log;
#pragma unroll
    for (int k = 0; k < 6; ++k) stress_out[6 * c + k] = sv[k];
    if (step) {
#pragma unroll
      for (int k = 0; k < 9; ++k) cells[9 * c + k] = __dmul_rn(mu, C[k]);
    }
  }
}

// ---- ASE's NPT (Nose-Hoover / Parrinello-Rahman).  Row vectors times row-major 3 x 3 matrices, every product and sum
// rounded on its own in a fixed order (no contraction), so the result depends on the operands only.
__device__ __forceinline__ void vec_mat3(const double v[3], const double* M, double out[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k)
    out[k] = __dadd_rn(__dadd_rn(__dmul_rn(v[0], M[k]), __dmul_rn(v[1], M[3 + k])), __dmul_rn(v[2], M[6 + k]));
}

__device__ __forceinline__ void mat3_mul(const double* A, const double* B, double* out) {
#pragma unroll
  for (int i = 0; i < 3; ++i) vec_mat3(A + 3 * i, B, out + 3 * i);
}

__device__ __forceinline__ double det3(const double* A) {
  const double c0 = __dsub_rn(__dmul_rn(A[4], A[8]), __dmul_rn(A[5], A[7]));
  const double c1 = __dsub_rn(__dmul_rn(A[3], A[8]), __dmul_rn(A[5], A[6]));
  const double c2 = __dsub_rn(__dmul_rn(A[3], A[7]), __dmul_rn(A[4], A[6]));
  return __dadd_rn(__dsub_rn(__dmul_rn(A[0], c0), __dmul_rn(A[1], c1)), __dmul_rn(A[2], c2));
}

// A^-1 = adj(A) / det, det = det3(A) finite and nonzero
__device__ __forceinline__ void inv3(const double* A, double det, double* out) {
  const double adj[9] = {__dsub_rn(__dmul_rn(A[4], A[8]), __dmul_rn(A[5], A[7])),
                         __dsub_rn(__dmul_rn(A[2], A[7]), __dmul_rn(A[1], A[8])),
                         __dsub_rn(__dmul_rn(A[1], A[5]), __dmul_rn(A[2], A[4])),
                         __dsub_rn(__dmul_rn(A[5], A[6]), __dmul_rn(A[3], A[8])),
                         __dsub_rn(__dmul_rn(A[0], A[8]), __dmul_rn(A[2], A[6])),
                         __dsub_rn(__dmul_rn(A[2], A[3]), __dmul_rn(A[0], A[5])),
                         __dsub_rn(__dmul_rn(A[3], A[7]), __dmul_rn(A[4], A[6])),
                         __dsub_rn(__dmul_rn(A[1], A[6]), __dmul_rn(A[0], A[7])),
                         __dsub_rn(__dmul_rn(A[0], A[4]), __dmul_rn(A[1], A[3]))};
#pragma unroll
  for (int k = 0; k < 9; ++k) out[k] = __ddiv_rn(adj[k], det);
}

__device__ __forceinline__ bool finite_nonzero(double v) { return isfinite(v) && v != 0.0; }

// the state row of a crystal (ALIGNN_B200_MD_NH_STATE doubles): h_past, eta, eta_past (row-major 3 x 3), zeta, zeta_past
enum { kHPast = 0, kEta = 9, kEtaPast = 18, kZeta = 27, kZetaPast = 28 };
// the per-crystal matrices in shared memory
enum { kH = 0, kInvH = 9, kBetaM = 18, kInvBetaP = 27, kHs = 36, kHFut = 45, kMats = 54 };

// _calculate_q_future for one atom: alpha = (dt dt) ((F/m) h^-1); q_future = (2q + q_past (beta - I) + alpha)(beta + I)^-1
__device__ __forceinline__ void nh_q_future(const double* M, double dt2, const double f[3], double m, const double q[3],
                                            const double qp[3], double out[3]) {
  double fm[3], alpha[3], qb[3], s[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) fm[k] = __ddiv_rn(f[k], m);
  vec_mat3(fm, M + kInvH, alpha);
  vec_mat3(qp, M + kBetaM, qb);
#pragma unroll
  for (int k = 0; k < 3; ++k) s[k] = __dadd_rn(__dadd_rn(__dmul_rn(2.0, q[k]), qb[k]), __dmul_rn(dt2, alpha[k]));
  vec_mat3(s, M + kInvBetaP, out);
}

// p = ((q_future - q_past) (h / (2 dt))) m
__device__ __forceinline__ void nh_momenta(const double* M, const double qf[3], const double qp[3], double m,
                                           double p[3]) {
  const double d[3] = {__dsub_rn(qf[0], qp[0]), __dsub_rn(qf[1], qp[1]), __dsub_rn(qf[2], qp[2])};
  vec_mat3(d, M + kHs, p);
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = __dmul_rn(p[k], m);
}

// q_past = q - dt ((p/m) h^-1)
__device__ __forceinline__ void nh_q_past(const double* M, double dt, const double q[3], const double p[3], double m,
                                          double out[3]) {
  const double v[3] = {__ddiv_rn(p[0], m), __ddiv_rn(p[1], m), __ddiv_rn(p[2], m)};
  double w[3];
  vec_mat3(v, M + kInvH, w);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = __dsub_rn(q[k], __dmul_rn(dt, w[k]));
}

// ASE 3.22.1's `NPT` (ase/md/npt.py, mask None, frac_traceless 1), which `ForceField.run_npt_nose_hoover`
// (alignn/ff/ff.py:584-617) runs; oracle/md_nose_hoover_oracle.py is its specification.  One launch per evaluation e,
// one CTA per crystal.  Thread 0 forms the crystal's matrices (h, h^-1, beta - I, (beta + I)^-1, h / (2 dt) and, for
// e < steps, h_future) in shared memory and checks them before anything is written:
//   e == 0: p -= sum_i p_i / n (zero_center_of_mass_momentum); initialize(): q = r h^-1 - 0.5 and the two passes of
//           _calculate_q_past_and_future on the forces F of this evaluation -- pass 1 from p0, its mean kinetic energy
//           per atom (a block reduction), and below 1e-5 eV the first pass stands, else pass 2 from 2 p0 - p'.
//           The atoms keep p0; q_future goes to the second per-atom array.
//   e >= 1: the end of step e: that array holds q_past; q_future from F, then p = ((q_future - q_past)(h/(2dt))) m.
//   always: the forces, ekin, T, the calculator's stress and the ideal-gas pressure, as md_npt_step_kernel logs them.
//   e < steps: the start of step e + 1 on this evaluation's ideal-gas-corrected stress s and kinetic energy (for e = 0
//           the past values come from initialize(): h_past = h - dt h eta, eta_past = eta - U(-dt pfact det h (s - s_ext)),
//           zeta_past = zeta - dt tfact (ekin - desiredEkin)): h_future = h_past + 2dt h eta, eta_future = eta_past +
//           U(-2dt (pfact det h (s - s_ext))) (U(0) when pfact = 0: pfactor None, s unread), zeta_future = zeta_past +
//           2dt tfact (ekin - desiredEkin); the shift; q_past <-> q swapped between the two arrays; r = (q + 0.5) h_future.
// Status 3: the slice is outside grad, or (e == 0) h is not upper triangular.  Status 4: det h, det(beta + I) or, for
// e < steps, det h_future is not finite and nonzero.  Nothing of the crystal is written then, nor in later launches.
__global__ void __launch_bounds__(kBlock)
md_nose_hoover_kernel(const alignn_b200_md_nose_hoover_params p, const int64_t* __restrict__ atom_off,
                      const float* __restrict__ grad, int64_t grad_rows, const float* __restrict__ stress,
                      const double* __restrict__ masses, const double* __restrict__ tfact,
                      const double* __restrict__ pfact, const double* __restrict__ desired_ekin,
                      const double* __restrict__ ext_stress, double* __restrict__ cells, double* __restrict__ state,
                      double* __restrict__ x, double* __restrict__ mom, double* __restrict__ qa,
                      double* __restrict__ qb, float* __restrict__ forces, float* __restrict__ stress_out,
                      double* __restrict__ ekin_out, double* __restrict__ temp_out, double* __restrict__ press_out,
                      int32_t* __restrict__ status) {
  __shared__ double red[kBlock][3];
  __shared__ double M[kMats];
  __shared__ double sh_det;
  __shared__ int verdict;
  const int64_t c = blockIdx.x;
  if (status[c] != kOk) return;
  const int64_t g0 = atom_off[c], n = atom_off[c + 1] - g0;
  if (g0 < 0 || n < 1 || atom_off[c + 1] > grad_rows) {
    if (threadIdx.x == 0) status[c] = kBadInput;
    return;
  }
  const int t = threadIdx.x;
  const double dt = p.dt;
  const bool init = p.evaluation == 0, step = p.evaluation < p.steps;
  double* st = state + ALIGNN_B200_MD_NH_STATE * c;
  if (t == 0) {
    int v = kOk;
    double h[9], E[9], T1[9], beta[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) h[k] = cells[9 * c + k];
    if (init && !(h[3] == 0.0 && h[6] == 0.0 && h[7] == 0.0)) v = kBadInput;
    const double det = det3(h);
    if (v == kOk && !finite_nonzero(det)) v = kCellDegenerate;
    if (v == kOk) {
      inv3(h, det, M + kInvH);
      // beta = dt (h ((eta + (0.5 zeta) I) h^-1))
      const double hz = __dmul_rn(0.5, st[kZeta]);
#pragma unroll
      for (int k = 0; k < 9; ++k) E[k] = __dadd_rn(st[kEta + k], (k % 4 == 0) ? hz : 0.0);
      mat3_mul(E, M + kInvH, T1);
      mat3_mul(h, T1, beta);
      double bp[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double b = __dmul_rn(dt, beta[k]);
        M[kBetaM + k] = __dsub_rn(b, (k % 4 == 0) ? 1.0 : 0.0);
        bp[k] = __dadd_rn(b, (k % 4 == 0) ? 1.0 : 0.0);
      }
      const double detb = det3(bp);
      if (!finite_nonzero(detb)) v = kCellDegenerate;
      else inv3(bp, detb, M + kInvBetaP);
      const double two_dt = __dmul_rn(2.0, dt);
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        M[kH + k] = h[k];
        M[kHs + k] = __ddiv_rn(h[k], two_dt);
      }
      if (step) {                                               // h_future = h_past + 2dt (h eta)
        double he[9];
        mat3_mul(h, st + kEta, he);
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          const double hp = init ? __dsub_rn(h[k], __dmul_rn(dt, he[k])) : st[kHPast + k];
          M[kHFut + k] = __dadd_rn(hp, __dmul_rn(two_dt, he[k]));
        }
        if (!finite_nonzero(det3(M + kHFut))) v = kCellDegenerate;
      }
    }
    sh_det = det;
    verdict = v;
  }
  __syncthreads();
  if (verdict != kOk) {
    if (t == 0) status[c] = verdict;
    return;
  }
  const double det = sh_det;
  const double dt2 = __dmul_rn(dt, dt);
  const float* gr = grad + 3 * g0;
  const double* mc = masses + g0;
  double* xc = x + 3 * g0;
  double* pc = mom + 3 * g0;
  double* qac = qa + 3 * g0;
  double* qbc = qb + 3 * g0;
  float* fc = forces + 3 * g0;
  double tot[3];

  // ---- the momenta of this evaluation, their kinetic energy and ideal-gas sums
  double mean[3] = {0.0, 0.0, 0.0};
  if (init) {                                                   // zero_center_of_mass_momentum: p - p.sum(0) / n
    double s[3] = {0.0, 0.0, 0.0};
    for (int64_t i = t; i < n; i += kBlock) {
#pragma unroll
      for (int k = 0; k < 3; ++k) s[k] = __dadd_rn(s[k], pc[3 * i + k]);
    }
    block_sum3(red, s[0], s[1], s[2], tot);
    const double nd = (double)n;
#pragma unroll
    for (int k = 0; k < 3; ++k) mean[k] = __ddiv_rn(tot[k], nd);
  }
  double kin = 0.0, g[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, e1 = 0.0;
  for (int64_t i = t; i < n; i += kBlock) {
    const double m = mc[i];
    double f[3], pv[3], q[3], qp[3], qf[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float fv = __fmul_rn(gr[3 * i + k], p.force_multiplier);
      fc[3 * i + k] = fv;
      f[k] = fv;
    }
    if (init) {
      double r[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        pv[k] = __dsub_rn(pc[3 * i + k], mean[k]);
        pc[3 * i + k] = pv[k];
        r[k] = xc[3 * i + k];
      }
      vec_mat3(r, M + kInvH, q);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        q[k] = __dsub_rn(q[k], 0.5);
        qac[3 * i + k] = q[k];
      }
      double p1[3];                                             // the first pass
      nh_q_past(M, dt, q, pv, m, qp);
      nh_q_future(M, dt2, f, m, q, qp, qf);
      nh_momenta(M, qf, qp, m, p1);
      e1 = __dadd_rn(e1, __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(p1[0], p1[0]), __dmul_rn(p1[1], p1[1])),
                                             __dmul_rn(p1[2], p1[2])), m));
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        q[k] = qac[3 * i + k];
        qp[k] = qbc[3 * i + k];
      }
      nh_q_future(M, dt2, f, m, q, qp, qf);
      nh_momenta(M, qf, qp, m, pv);
#pragma unroll
      for (int k = 0; k < 3; ++k) pc[3 * i + k] = pv[k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      qbc[3 * i + k] = qf[k];
      kin = __dadd_rn(kin, __dmul_rn(pv[k], __ddiv_rn(pv[k], m)));
    }
    add_ideal_gas_terms(pv, __ddiv_rn(1.0, m), g);
  }
  double G[6], rest[3];
  block_sum3(red, kin, g[0], g[1], tot);
  block_sum3(red, g[2], g[3], g[4], G + 2);
  block_sum3(red, g[5], e1, 0.0, rest);
  G[0] = tot[1];
  G[1] = tot[2];
  G[5] = rest[0];

  // ---- initialize(): the second pass unless the first one's 0.5 sum(p'^2 / m) / n is below 1e-5 eV
  if (init && !(__ddiv_rn(__dmul_rn(0.5, rest[1]), (double)n) < 1e-5)) {
    for (int64_t i = t; i < n; i += kBlock) {
      const double m = mc[i];
      double f[3], p0[3], q[3], qp[3], qf[3], p1[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        f[k] = fc[3 * i + k];
        p0[k] = pc[3 * i + k];
        q[k] = qac[3 * i + k];
        qf[k] = qbc[3 * i + k];
      }
      nh_q_past(M, dt, q, p0, m, qp);                           // pass 1's q_past and p' again
      nh_momenta(M, qf, qp, m, p1);
#pragma unroll
      for (int k = 0; k < 3; ++k) p1[k] = __dadd_rn(__dsub_rn(p0[k], p1[k]), p0[k]);
      nh_q_past(M, dt, q, p1, m, qp);
      nh_q_future(M, dt2, f, m, q, qp, qf);
#pragma unroll
      for (int k = 0; k < 3; ++k) qbc[3 * i + k] = qf[k];
    }
  }

  // ---- the log rows
  const double ekin = __dmul_rn(0.5, tot[0]);
  const double T = __ddiv_rn(__dmul_rn(2.0, ekin), __dmul_rn((double)(3 * n), p.kB));
  float sv[6], sc[6];
  fire::calculator_stress(stress + 9 * c, p.stress_wt, sv);
  const double P_log = corrected_pressure(sv, G, __ddiv_rn(1.0, fabs(det)), sc);
  if (t == 0) {
    ekin_out[c] = ekin;
    temp_out[c] = T;
    press_out[c] = P_log;
#pragma unroll
    for (int k = 0; k < 6; ++k) stress_out[6 * c + k] = sv[k];
  }
  if (!step) return;

  // ---- the start of step e + 1: the shift of q, and r = (q + 0.5) h_future
  for (int64_t i = t; i < n; i += kBlock) {
    double q[3], r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      q[k] = qbc[3 * i + k];
      qbc[3 * i + k] = qac[3 * i + k];                          // q_past = q
      qac[3 * i + k] = q[k];                                    // q = q_future
      q[k] = __dadd_rn(q[k], 0.5);
    }
    vec_mat3(q, M + kHFut, r);
#pragma unroll
    for (int k = 0; k < 3; ++k) xc[3 * i + k] = r[k];
  }
  if (t == 0) {
    const double pf = pfact[c], tf = tfact[c];
    const double dE = __dsub_rn(ekin, desired_ekin[c]);
    double de[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, de0[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (pf != 0.0) {                                            // pfactor given: the stress is read
      const double a = __dmul_rn(pf, det), a0 = __dmul_rn(__dmul_rn(-dt, pf), det);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const double ds = __dsub_rn((double)sc[k], ext_stress[6 * c + k]);
        de[k] = __dmul_rn(__dmul_rn(-2.0, dt), __dmul_rn(a, ds));
        de0[k] = __dmul_rn(a0, ds);
      }
    }
    // U(v) = [[v0, v5, v4], [0, v1, v3], [0, 0, v2]] as (row-major index, Voigt index) pairs
    const int ui[6] = {0, 4, 8, 5, 2, 1};
    double eta[9], eta_past[9], zeta = st[kZeta], zeta_past;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      eta[k] = st[kEta + k];
      eta_past[k] = st[kEtaPast + k];
    }
    if (init) {                                                 // initialize()'s past values
#pragma unroll
      for (int k = 0; k < 9; ++k) eta_past[k] = eta[k];
#pragma unroll
      for (int j = 0; j < 6; ++j) eta_past[ui[j]] = __dsub_rn(eta[ui[j]], de0[j]);
      zeta_past = __dsub_rn(zeta, __dmul_rn(__dmul_rn(dt, tf), dE));
    } else {
      zeta_past = st[kZetaPast];
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) eta_past[ui[j]] = __dadd_rn(eta_past[ui[j]], de[j]);   // now eta_future
    const double zeta_future = __dadd_rn(zeta_past, __dmul_rn(__dmul_rn(__dmul_rn(2.0, dt), tf), dE));
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      st[kHPast + k] = M[kH + k];
      st[kEtaPast + k] = eta[k];
      st[kEta + k] = eta_past[k];
      cells[9 * c + k] = M[kHFut + k];
    }
    st[kZetaPast] = zeta;
    st[kZeta] = zeta_future;
  }
}

// the stream itself, for tests: item (a, j), a in [0, atoms), is block j of atom index atom0 + a (mod 2^32)
__global__ void __launch_bounds__(kBlock)
md_noise_kernel(uint64_t seed, uint32_t step, uint32_t tag, uint32_t atom0, int64_t items, int32_t blocks,
                uint32_t* __restrict__ words, double* __restrict__ uniforms, double* __restrict__ normals) {
  const int64_t q = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (q >= items) return;
  const uint32_t atom = atom0 + (uint32_t)(q / blocks), block = (uint32_t)(q % blocks);
  const Words4 w = noise_block(seed, atom, step, block, tag);
#pragma unroll
  for (int k = 0; k < 4; ++k) words[4 * q + k] = w.w[k];
  const double u0 = unit_uniform(w.w[0], w.w[1]), u1 = unit_uniform(w.w[2], w.w[3]);
  uniforms[2 * q] = u0;
  uniforms[2 * q + 1] = u1;
  box_muller(u0, u1, normals[2 * q], normals[2 * q + 1]);
}

}  // namespace md
}  // namespace alignn

extern "C" {

int alignn_b200_md_step(const alignn_b200_md_params* params, const int64_t* atom_offsets, int64_t num_crystals,
                        const float* grad, int64_t grad_rows, const double* masses, const double* target_temperature,
                        double* positions, double* momenta, float* forces, double* kinetic_energy, double* temperature,
                        int32_t* status, alignn_stream_t stream) {
  using namespace alignn::md;
  if (!params || num_crystals < 1 || num_crystals > INT32_MAX || grad_rows < 0) return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_md_params p = *params;
  if (p.steps < 1 || p.evaluation < 0 || p.evaluation > p.steps || !isfinite(p.dt) || !(p.dt > 0.0) ||
      !isfinite(p.kB) || !(p.kB > 0.0) || !isfinite(p.force_multiplier) || (p.ensemble != kNVE && p.ensemble != kBerendsen))
    return ALIGNN_ERR_BAD_ARG;
  if (p.ensemble == kBerendsen && (!target_temperature || !isfinite(p.taut) || !(p.taut >= p.dt)))
    return ALIGNN_ERR_BAD_ARG;
  if (!atom_offsets || !grad || !masses || !positions || !momenta || !forces || !kinetic_energy || !temperature || !status)
    return ALIGNN_ERR_BAD_ARG;
  md_step_kernel<<<(unsigned)num_crystals, kBlock, 0, (cudaStream_t)stream>>>(
      p, atom_offsets, grad, grad_rows, masses, target_temperature, positions, momenta, forces, kinetic_energy,
      temperature, status);
  return alignn::check_launch();
}

int alignn_b200_md_thermostat_step(const alignn_b200_md_thermostat_params* params, const int64_t* atom_offsets,
                                   int64_t num_crystals, const float* grad, int64_t grad_rows, const double* masses,
                                   const double* target_temperature, const uint64_t* seeds, double* positions,
                                   double* momenta, double* velocities, double* rnd_vel, float* forces,
                                   double* kinetic_energy, double* temperature, int32_t* status, alignn_stream_t stream) {
  using namespace alignn::md;
  if (!params || num_crystals < 1 || num_crystals > INT32_MAX || grad_rows < 0) return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_md_thermostat_params p = *params;
  const auto positive = [](double v) { return isfinite(v) && v > 0.0; };
  if (p.steps < 1 || p.evaluation < 0 || p.evaluation > p.steps || !positive(p.dt) || !positive(p.kB) ||
      !isfinite(p.force_multiplier) || !isfinite(p.friction) || !(p.friction >= 0.0) ||
      !(p.andersen_prob >= 0.0 && p.andersen_prob <= 1.0) || !positive(p.sqrt_dt) || !positive(p.dt_1_5) ||
      !positive(p.two_sqrt3) || (p.ensemble != kLangevin && p.ensemble != kAndersen))
    return ALIGNN_ERR_BAD_ARG;
  if (!atom_offsets || !grad || !masses || !target_temperature || !seeds || !positions || !momenta || !velocities ||
      !rnd_vel || !forces || !kinetic_energy || !temperature || !status)
    return ALIGNN_ERR_BAD_ARG;
  md_thermostat_kernel<<<(unsigned)num_crystals, kBlock, 0, (cudaStream_t)stream>>>(
      p, atom_offsets, grad, grad_rows, masses, target_temperature, seeds, positions, momenta, velocities, rnd_vel,
      forces, kinetic_energy, temperature, status);
  return alignn::check_launch();
}

int alignn_b200_md_npt_step(const alignn_b200_md_npt_params* params, const int64_t* atom_offsets, int64_t num_crystals,
                            const float* grad, int64_t grad_rows, const float* stress, const double* masses,
                            const double* target_temperature, const double* target_pressure,
                            const double* compressibility, double* cells, double* positions, double* momenta,
                            float* forces, float* stress_out, double* kinetic_energy, double* temperature,
                            double* pressure, int32_t* status, alignn_stream_t stream) {
  using namespace alignn::md;
  if (!params || num_crystals < 1 || num_crystals > INT32_MAX || grad_rows < 0) return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_md_npt_params p = *params;
  const auto positive = [](double v) { return isfinite(v) && v > 0.0; };
  if (p.steps < 1 || p.evaluation < 0 || p.evaluation > p.steps || (p.phase != 0 && p.phase != 1) ||
      (p.phase == 1 && p.evaluation == p.steps) || !positive(p.dt) || !positive(p.kB) || !positive(p.taut) ||
      !positive(p.taup) || !(p.taut >= p.dt) || !isfinite(p.force_multiplier) || !isfinite(p.stress_wt))
    return ALIGNN_ERR_BAD_ARG;
  if (!atom_offsets || !grad || !stress || !masses || !target_temperature || !target_pressure || !compressibility ||
      !cells || !positions || !momenta || !forces || !stress_out || !kinetic_energy || !temperature || !pressure || !status)
    return ALIGNN_ERR_BAD_ARG;
  md_npt_step_kernel<<<(unsigned)num_crystals, kBlock, 0, (cudaStream_t)stream>>>(
      p, atom_offsets, grad, grad_rows, stress, masses, target_temperature, target_pressure, compressibility, cells,
      positions, momenta, forces, stress_out, kinetic_energy, temperature, pressure, status);
  return alignn::check_launch();
}

int alignn_b200_md_nose_hoover_step(const alignn_b200_md_nose_hoover_params* params, const int64_t* atom_offsets,
                                    int64_t num_crystals, const float* grad, int64_t grad_rows, const float* stress,
                                    const double* masses, const double* tfact, const double* pfact,
                                    const double* desired_ekin, const double* external_stress, double* cells,
                                    double* state, double* positions, double* momenta, double* q, double* q_future,
                                    float* forces, float* stress_out, double* kinetic_energy, double* temperature,
                                    double* pressure, int32_t* status, alignn_stream_t stream) {
  using namespace alignn::md;
  if (!params || num_crystals < 1 || num_crystals > INT32_MAX || grad_rows < 0) return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_md_nose_hoover_params p = *params;
  const auto positive = [](double v) { return isfinite(v) && v > 0.0; };
  if (p.steps < 1 || p.evaluation < 0 || p.evaluation > p.steps || !positive(p.dt) || !positive(p.kB) ||
      !isfinite(p.force_multiplier) || !isfinite(p.stress_wt))
    return ALIGNN_ERR_BAD_ARG;
  if (!atom_offsets || !grad || !stress || !masses || !tfact || !pfact || !desired_ekin || !external_stress || !cells ||
      !state || !positions || !momenta || !q || !q_future || !forces || !stress_out || !kinetic_energy || !temperature ||
      !pressure || !status)
    return ALIGNN_ERR_BAD_ARG;
  md_nose_hoover_kernel<<<(unsigned)num_crystals, kBlock, 0, (cudaStream_t)stream>>>(
      p, atom_offsets, grad, grad_rows, stress, masses, tfact, pfact, desired_ekin, external_stress, cells, state,
      positions, momenta, q, q_future, forces, stress_out, kinetic_energy, temperature, pressure, status);
  return alignn::check_launch();
}

int alignn_b200_md_noise(uint64_t seed, int32_t step, int32_t tag, uint32_t atom0, int64_t atoms, int32_t blocks,
                         uint32_t* words, double* uniforms, double* normals, alignn_stream_t stream) {
  using namespace alignn::md;
  if (step < 0 || atoms < 0 || atoms > INT32_MAX || blocks < 1 || blocks > 64 || !words || !uniforms || !normals)
    return ALIGNN_ERR_BAD_ARG;
  const int64_t items = atoms * blocks;
  if (items == 0) return ALIGNN_OK;
  md_noise_kernel<<<(unsigned)((items + kBlock - 1) / kBlock), kBlock, 0, (cudaStream_t)stream>>>(
      seed, (uint32_t)step, (uint32_t)tag, atom0, items, blocks, words, uniforms, normals);
  return alignn::check_launch();
}

}  // extern "C"
