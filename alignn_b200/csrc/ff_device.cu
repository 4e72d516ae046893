// eALIGNN force-field steps that the reference runs as Python loops inside every forward:
//   * the bond cutoff filter behind `lightweight_line_graph` (alignn/models/utils.py:47-55, 129-222): recompute the bond
//     vectors from Cartesian coordinates and keep the bonds no longer than `inner_cutoff`, in their original order;
//   * the net-torque correction `remove_net_torque` (alignn/models/utils.py:295-398).
// Deterministic: an integer scan for the filter, fixed-order block partials in double for the torque sums, no float
// atomics.  CUB (CUDA toolkit) does the exclusive scan, as in csrc/graph_device.cu.
#include <cub/cub.cuh>
#include <float.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace ff {

constexpr int kBlock = 256;
constexpr int kMaxPartBlocks = 256;      // torque partials: the grid (and so the summation order) depends on N only
inline int blocks_for(int64_t n) { return (int)((n + kBlock - 1) / kBlock); }
inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }
inline int part_blocks(int64_t n) {
  const int b = blocks_for(n);
  return b < 1 ? 1 : (b > kMaxPartBlocks ? kMaxPartBlocks : b);
}

// ---- bond cutoff filter -------------------------------------------------------------------------------------------
// r = (cart[dst] + images) - cart[src], component by component in fp32 (compute_pair_vector_and_distance); the bond is
// dropped only if |r| > cutoff, so a NaN length is kept (torch.gt is false for NaN).
__global__ void cutoff_flag_kernel(const float* __restrict__ cart, const int32_t* __restrict__ src,
                                   const int32_t* __restrict__ dst, const float* __restrict__ images, int64_t E,
                                   float cutoff, float* __restrict__ r, int32_t* __restrict__ keep) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e > E) return;
  if (e == E) { keep[E] = 0; return; }
  const int64_t s = src[e], d = dst[e];
  float v[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = __fsub_rn(__fadd_rn(cart[3 * d + k], images[3 * e + k]), cart[3 * s + k]);
  r[3 * e] = v[0]; r[3 * e + 1] = v[1]; r[3 * e + 2] = v[2];
  const float len = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
  keep[e] = (len > cutoff) ? 0 : 1;
}

__global__ void cutoff_fill_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                   const float* __restrict__ r, const float* __restrict__ images,
                                   const int32_t* __restrict__ off, const int64_t* __restrict__ edge_off, int64_t B,
                                   int64_t E, int32_t* __restrict__ src_out, int32_t* __restrict__ dst_out,
                                   float* __restrict__ r_out, float* __restrict__ images_out,
                                   int64_t* __restrict__ edge_ids) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int32_t k = off[e];
  if (off[e + 1] == k) return;                                  // dropped
  src_out[k] = src[e];
  dst_out[k] = dst[e];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    r_out[3 * k + c] = r[3 * e + c];
    images_out[3 * k + c] = images[3 * e + c];
  }
  int64_t base = 0;
  if (B > 1) {                                                  // crystal-local ids when the batch holds several crystals
    int64_t lo = 0, hi = B;                                     // last b with edge_off[b] <= e
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) / 2;
      if (edge_off[mid] <= e) lo = mid; else hi = mid;
    }
    base = edge_off[lo];
  }
  edge_ids[k] = e - base;
}

// ---- net-torque removal ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// fixed-order tree over the block; red[kBlock][W]; thread 0 ends with the block sum in red[0]
template <int W>
__device__ void block_sum(double (*red)[W], const double* acc) {
#pragma unroll
  for (int k = 0; k < W; ++k) red[threadIdx.x][k] = acc[k];
  __syncthreads();
  for (int s = kBlock / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
#pragma unroll
      for (int k = 0; k < W; ++k) red[threadIdx.x][k] += red[threadIdx.x + s][k];
    __syncthreads();
  }
}

// sum of the G partials [G][3] in index order (every block that needs the total computes it the same way)
__device__ void sum_partials(const double* __restrict__ part, int G, double* out) {
  double a = 0.0, b = 0.0, c = 0.0;
  for (int i = 0; i < G; ++i) { a += part[3 * i]; b += part[3 * i + 1]; c += part[3 * i + 2]; }
  out[0] = a; out[1] = b; out[2] = c;
}

__global__ void __launch_bounds__(kBlock)
torque_com_kernel(const float* __restrict__ pos, int64_t N, double* __restrict__ part_pos) {
  __shared__ double red[kBlock][3];
  double acc[3] = {0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < N; i += (int64_t)gridDim.x * kBlock)
#pragma unroll
    for (int k = 0; k < 3; ++k) acc[k] += (double)pos[3 * i + k];
  block_sum<3>(red, acc);
  if (threadIdx.x < 3) part_pos[3 * blockIdx.x + threadIdx.x] = red[0][threadIdx.x];
}

// tau = sum_i r_i x F_i.  cross_dim0 (a batch of exactly 3 atoms): torch.cross without `dim` takes dim 0 of the [3,3]
// tensors, so the "vectors" are the columns -- tau[j] = sum of the components of (r[:,j] x F[:,j]).
__global__ void __launch_bounds__(kBlock)
torque_tau_kernel(const float* __restrict__ pos, const float* __restrict__ F, int64_t N, int cross_dim0,
                  const double* __restrict__ part_pos, double* __restrict__ part_tau) {
  __shared__ double red[kBlock][3];
  double com[3];
  sum_partials(part_pos, gridDim.x, com);
#pragma unroll
  for (int k = 0; k < 3; ++k) com[k] /= (double)N;
  double acc[3] = {0.0, 0.0, 0.0};
  if (cross_dim0) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      for (int j = 0; j < 3; ++j) {
        const double a[3] = {pos[j] - com[j], pos[3 + j] - com[j], pos[6 + j] - com[j]};
        const double b[3] = {F[j], F[3 + j], F[6 + j]};
        double c[3];
        cross3(a, b, c);
        acc[j] = (c[0] + c[1]) + c[2];
      }
    }
  } else {
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < N; i += (int64_t)gridDim.x * kBlock) {
      const double a[3] = {pos[3 * i] - com[0], pos[3 * i + 1] - com[1], pos[3 * i + 2] - com[2]};
      const double b[3] = {F[3 * i], F[3 * i + 1], F[3 * i + 2]};
      double c[3];
      cross3(a, b, c);
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[k] += c[k];
    }
  }
  block_sum<3>(red, acc);
  if (threadIdx.x < 3) part_tau[3 * blockIdx.x + threadIdx.x] = red[0][threadIdx.x];
}

// x = M^+ b for a symmetric 3x3 M: cyclic Jacobi eigendecomposition, eigenvalues with |l| <= 3 eps max|l| dropped
// (torch.linalg.pinv's default rtol = max(m, n) * eps).
__device__ void pinv_solve_sym3(const double M[3][3], const double* b, double* x) {
  double A[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { A[i][j] = M[i][j]; V[i][j] = (i == j) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 64; ++sweep) {
    const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
    if (off == 0.0) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (A[p][q] == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {                       // A <- A J
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {                       // A <- J^T A
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {                       // V <- V J
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  const double lmax = fmax(fabs(A[0][0]), fmax(fabs(A[1][1]), fabs(A[2][2])));
  const double cut = 3.0 * DBL_EPSILON * lmax;
  x[0] = x[1] = x[2] = 0.0;
  for (int k = 0; k < 3; ++k) {
    const double l = A[k][k];
    if (!(fabs(l) > cut)) continue;
    const double w = (V[0][k] * b[0] + V[1][k] * b[1] + V[2][k] * b[2]) / l;
    for (int i = 0; i < 3; ++i) x[i] += w * V[i][k];
  }
}

// LU with partial pivoting (LAPACK getrf's pivot choice); false if a pivot is exactly zero
__device__ bool lu_solve3(const double M[3][3], const double* b, double* x) {
  double A[3][3], y[3];
  for (int i = 0; i < 3; ++i) {
    y[i] = b[i];
    for (int j = 0; j < 3; ++j) A[i][j] = M[i][j];
  }
  for (int k = 0; k < 3; ++k) {
    int p = k;
    for (int i = k + 1; i < 3; ++i)
      if (fabs(A[i][k]) > fabs(A[p][k])) p = i;
    if (A[p][k] == 0.0) return false;
    if (p != k) {
      for (int j = 0; j < 3; ++j) { const double t = A[k][j]; A[k][j] = A[p][j]; A[p][j] = t; }
      const double t = y[k]; y[k] = y[p]; y[p] = t;
    }
    for (int i = k + 1; i < 3; ++i) {
      const double f = A[i][k] / A[k][k];
      for (int j = k; j < 3; ++j) A[i][j] -= f * A[k][j];
      y[i] -= f * y[k];
    }
  }
  for (int i = 2; i >= 0; --i) {
    double s = y[i];
    for (int j = i + 1; j < 3; ++j) s -= A[i][j] * x[j];
    x[i] = s / A[i][i];
  }
  return true;
}

// one block per crystal: S_b = sum r r^T, s_b = sum |r|^2, M_b = S_b - s_b I, mu_b = M_b^{-1} (-tau)
__global__ void __launch_bounds__(kBlock)
torque_solve_kernel(const float* __restrict__ pos, const int64_t* __restrict__ node_off, int64_t N,
                    const double* __restrict__ part_pos, const double* __restrict__ part_tau, int G,
                    double* __restrict__ mu) {
  __shared__ double red[kBlock][7];
  const int b = blockIdx.x;
  double com[3], tau[3];
  sum_partials(part_pos, G, com);
  sum_partials(part_tau, G, tau);
#pragma unroll
  for (int k = 0; k < 3; ++k) com[k] /= (double)N;
  double acc[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};      // xx yy zz xy xz yz |r|^2
  for (int64_t i = node_off[b] + threadIdx.x; i < node_off[b + 1]; i += kBlock) {
    const double x = pos[3 * i] - com[0], y = pos[3 * i + 1] - com[1], z = pos[3 * i + 2] - com[2];
    acc[0] += x * x; acc[1] += y * y; acc[2] += z * z;
    acc[3] += x * y; acc[4] += x * z; acc[5] += y * z;
    acc[6] += (x * x + y * y) + z * z;
  }
  block_sum<7>(red, acc);
  if (threadIdx.x != 0) return;
  const double* S = red[0];
  const double s = S[6];
  const double M[3][3] = {{S[0] - s, S[3], S[4]}, {S[3], S[1] - s, S[5]}, {S[4], S[5], S[2] - s}};
  const double rhs[3] = {-tau[0], -tau[1], -tau[2]};
  double x[3];
  if (!lu_solve3(M, rhs, x)) pinv_solve_sym3(M, rhs, x);
  mu[3 * b] = x[0]; mu[3 * b + 1] = x[1]; mu[3 * b + 2] = x[2];
}

// out_i = F_i + r_i x mu_(crystal of i)   (cross_dim0: column-wise, as in torque_tau_kernel)
__global__ void torque_apply_kernel(const float* __restrict__ pos, const float* __restrict__ F,
                                    const int64_t* __restrict__ node_off, int64_t B, int64_t N, int cross_dim0,
                                    const double* __restrict__ part_pos, int G, const double* __restrict__ mu,
                                    float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || (cross_dim0 && i > 0)) return;
  double com[3];
  sum_partials(part_pos, G, com);
#pragma unroll
  for (int k = 0; k < 3; ++k) com[k] /= (double)N;
  auto crystal_of = [&](int64_t a) {
    int64_t lo = 0, hi = B;                                     // last b with node_off[b] <= a
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) / 2;
      if (node_off[mid] <= a) lo = mid; else hi = mid;
    }
    return lo;
  };
  if (cross_dim0) {                                             // N == 3: one thread writes the whole [3,3]
    const double* m[3] = {mu + 3 * crystal_of(0), mu + 3 * crystal_of(1), mu + 3 * crystal_of(2)};
    for (int j = 0; j < 3; ++j) {
      const double a[3] = {pos[j] - com[j], pos[3 + j] - com[j], pos[6 + j] - com[j]};
      const double c_[3] = {m[0][j], m[1][j], m[2][j]};
      double c[3];
      cross3(a, c_, c);
      for (int row = 0; row < 3; ++row) out[3 * row + j] = (float)((double)F[3 * row + j] + c[row]);
    }
    return;
  }
  const double* m = mu + 3 * crystal_of(i);
  const double a[3] = {pos[3 * i] - com[0], pos[3 * i + 1] - com[1], pos[3 * i + 2] - com[2]};
  double c[3];
  cross3(a, m, c);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[3 * i + k] = (float)((double)F[3 * i + k] + c[k]);
}

struct TorqueWs {
  double *part_pos, *part_tau, *mu;
  size_t total;
};

inline TorqueWs torque_ws(void* base, int64_t B) {
  TorqueWs w{};
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  w.part_pos = reinterpret_cast<double*>(p + off); off += align256((size_t)kMaxPartBlocks * 3 * 8);
  w.part_tau = reinterpret_cast<double*>(p + off); off += align256((size_t)kMaxPartBlocks * 3 * 8);
  w.mu = reinterpret_cast<double*>(p + off); off += align256((size_t)(B > 0 ? B : 1) * 3 * 8);
  w.total = off;
  return w;
}

}  // namespace ff
}  // namespace alignn

extern "C" {

size_t alignn_b200_bond_cutoff_workspace_bytes(int64_t num_edges) {
  if (num_edges < 0 || num_edges >= ((int64_t)1 << 31) - 1) return 0;
  size_t scan_b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(num_edges + 1));
  return alignn::ff::align256((size_t)(num_edges + 1) * 4) + alignn::ff::align256(scan_b);
}

int alignn_b200_bond_cutoff_offsets(const float* cart_coords, const int32_t* src, const int32_t* dst, const float* images,
                                    int64_t num_edges, float cutoff, float* r, int32_t* offsets, void* workspace,
                                    size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::ff;
  if (num_edges < 0 || num_edges >= ((int64_t)1 << 31) - 1 || !offsets || !workspace) return ALIGNN_ERR_BAD_ARG;
  if (num_edges > 0 && (!cart_coords || !src || !dst || !images || !r)) return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < alignn_b200_bond_cutoff_workspace_bytes(num_edges)) return ALIGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* keep = reinterpret_cast<int32_t*>(workspace);
  void* cubws = reinterpret_cast<uint8_t*>(workspace) + align256((size_t)(num_edges + 1) * 4);
  size_t b = workspace_bytes - align256((size_t)(num_edges + 1) * 4);
  cutoff_flag_kernel<<<blocks_for(num_edges + 1), kBlock, 0, st>>>(cart_coords, src, dst, images, num_edges, cutoff, r, keep);
  cub::DeviceScan::ExclusiveSum(cubws, b, keep, offsets, (int)(num_edges + 1), st);   // offsets[E] = kept bonds
  return alignn::check_launch();
}

int alignn_b200_bond_cutoff_fill(const int32_t* src, const int32_t* dst, const float* r, const float* images,
                                 const int32_t* offsets, const int64_t* edge_offsets, int64_t batch_size, int64_t num_edges,
                                 int32_t* src_out, int32_t* dst_out, float* r_out, float* images_out, int64_t* edge_ids,
                                 alignn_stream_t stream) {
  using namespace alignn::ff;
  if (num_edges < 0 || batch_size < 1) return ALIGNN_ERR_BAD_ARG;
  if (num_edges == 0) return ALIGNN_OK;
  if (!src || !dst || !r || !images || !offsets || !edge_offsets) return ALIGNN_ERR_BAD_ARG;
  // empty outputs are allowed when nothing was kept; the kernel never writes them then
  cutoff_fill_kernel<<<blocks_for(num_edges), kBlock, 0, (cudaStream_t)stream>>>(
      src, dst, r, images, offsets, edge_offsets, batch_size, num_edges, src_out, dst_out, r_out, images_out, edge_ids);
  return alignn::check_launch();
}

size_t alignn_b200_remove_net_torque_workspace_bytes(int64_t batch_size) {
  if (batch_size < 0) return 0;
  return alignn::ff::torque_ws(nullptr, batch_size).total;
}

int alignn_b200_remove_net_torque(const float* pos, const float* forces, const int64_t* node_offsets, int64_t batch_size,
                                  int64_t num_nodes, int cross_dim0, float* out, void* workspace, size_t workspace_bytes,
                                  alignn_stream_t stream) {
  using namespace alignn::ff;
  if (batch_size < 1 || num_nodes < 0 || (cross_dim0 && num_nodes != 3)) return ALIGNN_ERR_BAD_ARG;
  if (num_nodes == 0) return ALIGNN_OK;
  if (!pos || !forces || !node_offsets || !out || !workspace) return ALIGNN_ERR_BAD_ARG;
  const TorqueWs w = torque_ws(workspace, batch_size);
  if (workspace_bytes < w.total) return ALIGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int G = part_blocks(num_nodes);
  torque_com_kernel<<<G, kBlock, 0, st>>>(pos, num_nodes, w.part_pos);
  torque_tau_kernel<<<G, kBlock, 0, st>>>(pos, forces, num_nodes, cross_dim0, w.part_pos, w.part_tau);
  torque_solve_kernel<<<(int)batch_size, kBlock, 0, st>>>(pos, node_offsets, num_nodes, w.part_pos, w.part_tau, G, w.mu);
  torque_apply_kernel<<<blocks_for(num_nodes), kBlock, 0, st>>>(pos, forces, node_offsets, batch_size, num_nodes, cross_dim0,
                                                                w.part_pos, G, w.mu, out);
  return alignn::check_launch();
}

}  // extern "C"
