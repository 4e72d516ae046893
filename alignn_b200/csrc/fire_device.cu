// One FIRE step for a batch of crystals relaxed together: ASE 3.22.1's `FIRE.step` and the convergence test of
// `Optimizer.converged` / the loop of `Dynamics.irun` (ase/optimize/fire.py, ase/optimize/optimize.py), as
// `ForceField.optimize_atoms(optimizer="FIRE", optimize_lattice=False)` drives them (alignn/ff/ff.py:373-417) with the
// forces of `AlignnAtomwiseCalculator.calculate` (alignn/ff/calculators.py:280-372).
//
// One CTA per running crystal, a fixed block size, and per crystal:
//   1. forces F = fp32(grad * force_multiplier), written to the reported-forces array; fixed-order block reductions in
//      double of F.v, F.F, v.v and max_i |F_i|^2;
//   2. thread 0: converged (max |F_i|^2 < fmax^2), out of steps, or one FIRE update of (dt, a, Nsteps);
//   3. the velocity pass (mix or reset, v += dt F), a second reduction for |dr|^2 over the whole crystal, the position
//      pass (dr capped at maxstep).
// The per-element updates use explicitly rounded operations in numpy's evaluation order (no contraction into FMAs);
// the sums differ from numpy's only in their order.  No floating-point atomics: every result depends on the crystal's
// own atoms and the fixed block size only, so it is bitwise repeatable and independent of the batch around it.
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"
#include "fire_common.cuh"

namespace alignn {
namespace fire {

constexpr int kBlock = 256;
enum { kRunning = 0, kConverged = 1, kExhausted = 2, kBadInput = 3 };   // istate[c][3]
enum { kNsteps = 0, kFirst = 1, kTaken = 2, kStatus = 3 };      // istate columns
enum { kFrozen = 0, kFirstStep = 1, kMix = 2, kReset = 3 };     // what the velocity pass does

__global__ void __launch_bounds__(kBlock)
fire_step_kernel(const alignn_b200_fire_params p, const int32_t* __restrict__ active, const int64_t* __restrict__ atom_off,
                 const int32_t* __restrict__ batch_off, int64_t B, const float* __restrict__ grad, int64_t grad_rows,
                 double* __restrict__ x, double* __restrict__ v, float* __restrict__ forces,
                 double* __restrict__ fstate, int32_t* __restrict__ istate) {
  __shared__ double red[kBlock][4];
  __shared__ double coef[4];                                    // dt, a (mixing), sqrt(F.F), sqrt(v.v)
  __shared__ int mode;
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

  // ---- 1. forces of this evaluation and the sums FIRE and the convergence test need
  double fv = 0.0, ff = 0.0, vv = 0.0, fm = 0.0;
  for (int64_t i = t; i < n; i += kBlock) {
    double f2 = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float f = __fmul_rn(gr[3 * i + k], p.force_multiplier);
      fc[3 * i + k] = f;
      const double fd = f, vd = vc[3 * i + k];
      fv += fd * vd;
      ff += fd * fd;
      vv += vd * vd;
      f2 = __dadd_rn(f2, __dmul_rn(fd, fd));                    // (F_x^2 + F_y^2) + F_z^2
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

  // ---- 2. the decision and the scalar state (one thread)
  if (t == 0) {
    int m = kFrozen;
    if (red[0][3] < p.fmax * p.fmax) {                          // Optimizer.converged: strict
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
      } else if (red[0][0] > 0.0) {                             // vf > 0
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
      coef[2] = sqrt(red[0][1]);
      coef[3] = sqrt(red[0][2]);
    }
    mode = m;
  }
  __syncthreads();
  const int m = mode;
  if (m == kFrozen) return;
  const double dt = coef[0], am = coef[1], sf = coef[2], sv = coef[3];
  const double keep = __dadd_rn(1.0, -am);

  // ---- 3. velocities, |dr|^2 over the whole crystal, positions
  double dr2 = 0.0;
  for (int64_t i = t; i < n; i += kBlock) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double fd = fc[3 * i + k];                          // written by this thread above
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
  __syncthreads();                                              // thread 0 is done reading red[0]
  red[t][0] = dr2;
  __syncthreads();
  for (int s = kBlock / 2; s > 0; s >>= 1) {
    if (t < s) red[t][0] += red[t + s][0];
    __syncthreads();
  }
  const double norm = sqrt(red[0][0]);
  const bool cap = norm > p.maxstep;
  for (int64_t i = t; i < n; i += kBlock) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double dr = __dmul_rn(dt, vc[3 * i + k]);
      if (cap) dr = div_rn(__dmul_rn(p.maxstep, dr), norm);  // maxstep * dr / normdr
      xc[3 * i + k] = __dadd_rn(xc[3 * i + k], dr);
    }
  }
}

}  // namespace fire
}  // namespace alignn

extern "C" {

int alignn_b200_fire_step(const alignn_b200_fire_params* params, const int32_t* active, int64_t num_active,
                          const int64_t* atom_offsets, const int32_t* batch_offsets, int64_t num_crystals,
                          const float* grad, int64_t grad_rows, double* positions, double* velocities, float* forces, double* fstate,
                          int32_t* istate, alignn_stream_t stream) {
  using namespace alignn::fire;
  if (!params || num_active < 0 || grad_rows < 0 || num_crystals < 1 || num_active > num_crystals || num_active > INT32_MAX)
    return ALIGNN_ERR_BAD_ARG;
  const alignn_b200_fire_params p = *params;
  if (!(p.maxstep > 0.0) || !(p.dtmax > 0.0) || !(p.fmax >= 0.0) || !isfinite(p.fmax) || !isfinite(p.finc) ||
      !isfinite(p.fdec) || !isfinite(p.astart) || !isfinite(p.fa) || p.n_min < 0 || p.max_steps < 1 ||
      !isfinite(p.force_multiplier))
    return ALIGNN_ERR_BAD_ARG;
  if (num_active == 0) return ALIGNN_OK;
  if (!active || !atom_offsets || !batch_offsets || !grad || !positions || !velocities || !forces || !fstate || !istate)
    return ALIGNN_ERR_BAD_ARG;
  fire_step_kernel<<<(unsigned)num_active, kBlock, 0, (cudaStream_t)stream>>>(
      p, active, atom_offsets, batch_offsets, num_crystals, grad, grad_rows, positions, velocities, forces, fstate, istate);
  return alignn::check_launch();
}

}  // extern "C"
