// Finite-displacement phonons for a batch of crystals: ASE 3.22.1's `Phonons.read(acoustic=True)` (method='frederiksen',
// symmetrize=3) and the Fourier sum of `Phonons.band_structure` (ase/phonons.py), as `ase_phonon` (alignn/ff/ff.py:
// 1337-1430) drives them with the forces of `AlignnAtomwiseCalculator.calculate`.  oracle/phonon_oracle.py is the
// specification.
//
// alignn_b200_phonon_force_constants: one launch for the batch, one CTA per crystal, a fixed block size; per crystal:
//   0. every fp32 force product grad * force_multiplier must be finite, else status 5 and nothing is written;
//   1. C_N[cell, 3a+i, 3a'+j] = (f_minus - f_plus) / (2 delta) of displacement (a, i), row cell * n + a', component j;
//   2. the Frederiksen rows (cell 0, a' = a): one warp per (a, i) reduces each displaced set's force sum in a fixed
//      order and writes (f_minus[a] - sum_minus - (f_plus[a] - sum_plus)) / (2 delta);
//   3. three rounds of symmetrize (in place on partner pairs: cell R and cell -R transposed get the same
//      0.5 x + 0.5 y; for an even N the cells at N/2 along that axis are left out) and acoustic (each diagonal element
//      of cell 0 minus the sum over cells and a' of its row, subtracted in ASE's cell-major order);
//   4. D_N = C_N * (m_a^-1/2 m_a'^-1/2).
// C_N is its own working array (global memory: for n = 64 at (2,2,2) it is 2.4 MB).  Every step is elementwise with
// explicitly rounded operations in numpy's order, so only the Frederiksen sums differ from numpy's, in their order.
//
// alignn_b200_phonon_dynamical_matrix: one CTA per (crystal, q): the phase exp(-2 pi i q.R) of each cell once into
// shared memory (sincospi of -2 q.R: numpy rounds 2 pi q.R first, so the phases agree to rounding, not bitwise), then
// D(q)[r][s] = sum_R phase_R D_N[R][r][s] in the cell order of `lattice_vectors` for r <= s, written with its conjugate
// mirror (the upper triangle is what eigvalsh(UPLO='U') reads; the diagonal's imaginary part
// is written as 0).
// No floating-point atomics: every result depends on the crystal's own data and the fixed block sizes only, so it is
// bitwise repeatable and independent of the batch around it.
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace phonon {

constexpr int kBlock = 256;                       // force-constant kernel
constexpr int kDynBlock = 128;                    // dynamical-matrix kernel
constexpr int kWarps = kBlock / 32;
enum { kOk = 0, kBadInput = 3, kNonFinite = 5 };

struct Supercell {
  int32_t n0, n1, n2;
  int64_t cells;
};

__device__ __forceinline__ double load_force(const float* g, int64_t k, float mult) {
  return (double)__fmul_rn(g[k], mult);
}

__global__ void __launch_bounds__(kBlock)
force_constants_kernel(const Supercell sc, const double two_delta, const float mult, const int64_t* __restrict__ atom_off,
                       const int64_t* __restrict__ row_off, const float* __restrict__ grad, int64_t grad_rows,
                       const double* __restrict__ masses, const int64_t* __restrict__ fc_off, int64_t fc_elems,
                       double* __restrict__ C_all, double* __restrict__ D_all, int32_t* __restrict__ status) {
  const int64_t c = blockIdx.x;
  if (status[c] != kOk) return;                                 // a crystal already reported is not touched
  const int t = threadIdx.x;
  const int64_t n = atom_off[c + 1] - atom_off[c];
  const int64_t M = 3 * n, MM = M * M;
  const int64_t R = sc.cells * n;                               // rows of one supercell
  const int64_t r0 = row_off[c], f0 = fc_off[c];
  if (atom_off[c] < 0 || n < 1 || r0 < 0 || row_off[c + 1] - r0 != 6 * n * R || row_off[c + 1] > grad_rows ||
      f0 < 0 || fc_off[c + 1] - f0 != sc.cells * MM || fc_off[c + 1] > fc_elems) {
    if (t == 0) status[c] = kBadInput;                          // the slices are not inside the buffers: read nothing
    return;
  }
  const float* g = grad + 3 * r0;
  double* C = C_all + f0;
  double* D = D_all + f0;
  const double* m = masses + atom_off[c];

  // ---- 0. finite forces, or nothing is written
  int bad = 0;
  for (int64_t k = t; k < 18 * n * R; k += kBlock) bad |= !isfinite(__fmul_rn(g[k], mult));
  if (__syncthreads_or(bad)) {
    if (t == 0) status[c] = kNonFinite;
    return;
  }

  // ---- 1. central differences, the Frederiksen rows left to step 2
  for (int64_t e = t; e < sc.cells * MM; e += kBlock) {
    const int64_t cell = e / MM, rem = e - cell * MM;
    const int64_t r = rem / M, s = rem - r * M;
    const int64_t a = r / 3, i = r - 3 * a, a2 = s / 3, j = s - 3 * a2;
    if (cell == 0 && a2 == a) continue;
    const int64_t row = cell * n + a2;
    const double fm = load_force(g, 3 * ((6 * a + 2 * i) * R + row) + j, mult);
    const double fp = load_force(g, 3 * ((6 * a + 2 * i + 1) * R + row) + j, mult);
    C[e] = __ddiv_rn(__dsub_rn(fm, fp), two_delta);
  }

  // ---- 2. Frederiksen: f[a] -= f.sum(0) on both displaced sets of (a, i)
  const int lane = t & 31;
  for (int64_t p = t >> 5; p < M; p += kWarps) {
    const int64_t a = p / 3;
    double corr[2][3];
#pragma unroll
    for (int sg = 0; sg < 2; ++sg) {
      const float* gs = g + 3 * (2 * p + sg) * R;               // displaced set 6a + 2i + sg = 2p + sg
      double sx = 0.0, sy = 0.0, sz = 0.0;
      for (int64_t row = lane; row < R; row += 32) {
        sx = __dadd_rn(sx, load_force(gs, 3 * row + 0, mult));
        sy = __dadd_rn(sy, load_force(gs, 3 * row + 1, mult));
        sz = __dadd_rn(sz, load_force(gs, 3 * row + 2, mult));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {                        // butterfly: every lane ends with the same bits
        sx = __dadd_rn(sx, __shfl_xor_sync(0xffffffffu, sx, o));
        sy = __dadd_rn(sy, __shfl_xor_sync(0xffffffffu, sy, o));
        sz = __dadd_rn(sz, __shfl_xor_sync(0xffffffffu, sz, o));
      }
      corr[sg][0] = __dsub_rn(load_force(gs, 3 * a + 0, mult), sx);
      corr[sg][1] = __dsub_rn(load_force(gs, 3 * a + 1, mult), sy);
      corr[sg][2] = __dsub_rn(load_force(gs, 3 * a + 2, mult), sz);
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < 3; ++j) C[p * M + 3 * a + j] = __ddiv_rn(__dsub_rn(corr[0][j], corr[1][j]), two_delta);
    }
  }
  __syncthreads();

  // ---- 3. symmetrize + acoustic, three times
  const int h0 = (sc.n0 % 2 == 0) ? sc.n0 / 2 : -1;             // the cell left out along an even axis
  const int h1 = (sc.n1 % 2 == 0) ? sc.n1 / 2 : -1;
  const int h2 = (sc.n2 % 2 == 0) ? sc.n2 / 2 : -1;
  for (int round = 0; round < 3; ++round) {
    for (int64_t e = t; e < sc.cells * MM; e += kBlock) {
      const int64_t cell = e / MM, rem = e - cell * MM;
      const int64_t r = rem / M, s = rem - r * M;
      const int m2 = (int)(cell % sc.n2), m1 = (int)((cell / sc.n2) % sc.n1), m0 = (int)(cell / ((int64_t)sc.n1 * sc.n2));
      if (m0 == h0 || m1 == h1 || m2 == h2) continue;
      const int p0 = (sc.n0 - m0) % sc.n0, p1 = (sc.n1 - m1) % sc.n1, p2 = (sc.n2 - m2) % sc.n2;
      const int64_t pe = (((int64_t)p0 * sc.n1 + p1) * sc.n2 + p2) * MM + s * M + r;
      if (pe < e) continue;                                     // the pair is the other element's
      const double v = __dadd_rn(__dmul_rn(0.5, C[e]), __dmul_rn(0.5, C[pe]));
      C[e] = v;
      C[pe] = v;
    }
    __syncthreads();
    // a thread reads row 3a+i of every cell and writes only its own diagonal element of cell 0, which no other thread
    // reads: in place
    for (int64_t e = t; e < 9 * n; e += kBlock) {
      const int64_t a = e / 9, i = (e / 3) % 3, j = e % 3;
      const int64_t r = 3 * a + i;
      double v = C[r * M + 3 * a + j];
      for (int64_t cell = 0; cell < sc.cells; ++cell) {
        const double* row = C + cell * MM + r * M + j;
        for (int64_t a2 = 0; a2 < n; ++a2) v = __dsub_rn(v, row[3 * a2]);
      }
      C[r * M + 3 * a + j] = v;
    }
    __syncthreads();
  }

  // ---- 4. D_N = C_N * outer(m^-1/2, m^-1/2)
  for (int64_t e = t; e < sc.cells * MM; e += kBlock) {
    const int64_t rem = e % MM;
    const int64_t r = rem / M, s = rem - r * M;
    const double wr = __drcp_rn(__dsqrt_rn(m[r / 3])), ws = __drcp_rn(__dsqrt_rn(m[s / 3]));
    D[e] = __dmul_rn(C[e], __dmul_rn(wr, ws));
  }
}

__global__ void __launch_bounds__(kDynBlock)
dynamical_matrix_kernel(const Supercell sc, const int64_t M, const double* __restrict__ D_all,
                        const int64_t* __restrict__ fc_off, int64_t num_crystals, int64_t fc_elems,
                        const int32_t* __restrict__ crystals, const double* __restrict__ qpoints,
                        double* __restrict__ out, int32_t* __restrict__ status) {
  extern __shared__ double2 phase[];                            // [cells] (cos, sin) of -2 pi q.R
  const int64_t k = blockIdx.x;
  const int64_t c = crystals[k];
  if (c < 0 || c >= num_crystals || status[c] != kOk) return;
  const int t = threadIdx.x;
  const int64_t MM = M * M;
  const int64_t f0 = fc_off[c];
  if (f0 < 0 || fc_off[c + 1] - f0 != sc.cells * MM || fc_off[c + 1] > fc_elems) {
    if (t == 0) status[c] = kBadInput;                          // every CTA of c finds the same and writes the same
    return;
  }
  const double q0 = qpoints[3 * k], q1 = qpoints[3 * k + 1], q2 = qpoints[3 * k + 2];
  for (int64_t cell = t; cell < sc.cells; cell += kDynBlock) {
    const int m2 = (int)(cell % sc.n2), m1 = (int)((cell / sc.n2) % sc.n1), m0 = (int)(cell / ((int64_t)sc.n1 * sc.n2));
    // lattice_vectors: (m + N // 2) % N - N // 2
    const double R0 = (m0 + sc.n0 / 2) % sc.n0 - sc.n0 / 2;
    const double R1 = (m1 + sc.n1 / 2) % sc.n1 - sc.n1 / 2;
    const double R2 = (m2 + sc.n2 / 2) % sc.n2 - sc.n2 / 2;
    const double x = __dadd_rn(__dadd_rn(__dmul_rn(q0, R0), __dmul_rn(q1, R1)), __dmul_rn(q2, R2));
    double s, co;
    sincospi(__dmul_rn(-2.0, x), &s, &co);                      // exp(-2j * pi * x); sincos would need a stack frame
    phase[cell] = make_double2(co, s);
  }
  __syncthreads();
  const double* Dc = D_all + f0;
  double2* o = reinterpret_cast<double2*>(out) + k * MM;
  for (int64_t e = t; e < MM; e += kDynBlock) {
    const int64_t r = e / M, s = e - r * M;
    if (r > s) continue;
    double re = 0.0, im = 0.0;
    for (int64_t cell = 0; cell < sc.cells; ++cell) {
      const double d = Dc[cell * MM + e];
      const double2 ph = phase[cell];
      re = __dadd_rn(re, __dmul_rn(ph.x, d));
      im = __dadd_rn(im, __dmul_rn(ph.y, d));
    }
    if (r == s) {
      o[e] = make_double2(re, 0.0);
    } else {
      o[e] = make_double2(re, im);
      o[s * M + r] = make_double2(re, -im);
    }
  }
}

bool supercell_ok(const int32_t* supercell, Supercell* sc) {
  if (!supercell) return false;
  for (int i = 0; i < 3; ++i)
    if (supercell[i] < 1 || supercell[i] > ALIGNN_B200_PHONON_MAX_CELLS) return false;
  const int64_t cells = (int64_t)supercell[0] * supercell[1] * supercell[2];
  if (cells > ALIGNN_B200_PHONON_MAX_CELLS) return false;
  *sc = Supercell{supercell[0], supercell[1], supercell[2], cells};
  return true;
}

}  // namespace phonon
}  // namespace alignn

extern "C" {

int alignn_b200_phonon_force_constants(const int32_t* supercell, double delta, float force_multiplier,
                                       const int64_t* atom_offsets, int64_t num_crystals, const int64_t* row_offsets,
                                       const float* grad, int64_t grad_rows, const double* masses,
                                       const int64_t* fc_offsets, int64_t fc_elems, double* force_constants,
                                       double* dynamical_matrix, int32_t* status, alignn_stream_t stream) {
  using namespace alignn::phonon;
  Supercell sc;
  if (!supercell_ok(supercell, &sc) || !isfinite(delta) || !(delta > 0.0) || !isfinite(force_multiplier) ||
      num_crystals < 1 || num_crystals > INT32_MAX || grad_rows < 0 || fc_elems < 0)
    return ALIGNN_ERR_BAD_ARG;
  if (!atom_offsets || !row_offsets || !grad || !masses || !fc_offsets || !force_constants || !dynamical_matrix || !status)
    return ALIGNN_ERR_BAD_ARG;
  force_constants_kernel<<<(unsigned)num_crystals, kBlock, 0, (cudaStream_t)stream>>>(
      sc, 2.0 * delta, force_multiplier, atom_offsets, row_offsets, grad, grad_rows, masses, fc_offsets, fc_elems,
      force_constants, dynamical_matrix, status);
  return alignn::check_launch();
}

int alignn_b200_phonon_dynamical_matrix(const int32_t* supercell, int64_t modes, const double* dynamical_matrix,
                                        const int64_t* fc_offsets, int64_t num_crystals, int64_t fc_elems,
                                        const int32_t* crystals, const double* qpoints, int64_t num_q, double* out,
                                        int32_t* status, alignn_stream_t stream) {
  using namespace alignn::phonon;
  Supercell sc;
  if (!supercell_ok(supercell, &sc) || modes < 3 || modes % 3 != 0 || num_crystals < 1 || fc_elems < 0 || num_q < 0 ||
      num_q > INT32_MAX)
    return ALIGNN_ERR_BAD_ARG;
  if (!dynamical_matrix || !fc_offsets || !crystals || !qpoints || !out || !status) return ALIGNN_ERR_BAD_ARG;
  if (num_q == 0) return 0;
  dynamical_matrix_kernel<<<(unsigned)num_q, kDynBlock, sc.cells * sizeof(double2), (cudaStream_t)stream>>>(
      sc, modes, dynamical_matrix, fc_offsets, num_crystals, fc_elems, crystals, qpoints, out, status);
  return alignn::check_launch();
}

}  // extern "C"
