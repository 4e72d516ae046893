// Device-side structure builders and the force / stress reductions of SURVEY.md section 8f -- the GPU twins of
// csrc/graph_host.cu (sorted-CSR index, line graph; bit-identical outputs; the periodic scans are in
// csrc/crystal_graph_device.cu) and
// the d=3 reductions of ALIGNN-FF (alignn/models/alignn_atomwise.py:547-563, 610-635).  Pure integer work except the two d=3 reductions; everything deterministic
// (stable radix sort, fixed-order sums, integer atomics only for counting).  CUB (ships with the CUDA toolkit) does
// the scans and the stable key-value sort; it is plumbing here, like cudart.
#include <cub/cub.cuh>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace device {

constexpr int kBlock = 256;
inline int blocks_for(int64_t n) { return (int)((n + kBlock - 1) / kBlock); }
inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// ---- sorted CSR -------------------------------------------------------------------------------
__global__ void iota_hist_kernel(const int32_t* __restrict__ key, int64_t E, int32_t* __restrict__ cnt, int32_t* __restrict__ iota) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  if (iota) iota[e] = (int32_t)e;
  atomicAdd(&cnt[key[e]], 1);           // integer counting: the result does not depend on the order
}

__global__ void sorted_flag_kernel(const int32_t* __restrict__ dst, int64_t E, int32_t* __restrict__ flag) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 1 && e < E && dst[e] < dst[e - 1]) atomicAnd(flag, 0);
}

struct CsrWs {
  int32_t* cnt;      // [Nn + 1]
  int32_t* iota;     // [E]
  int32_t* keys;     // [E] sorted keys (discarded)
  void* cub;
  size_t cub_bytes, total;
};

inline int key_bits(int64_t n) {
  int b = 1;
  while (((int64_t)1 << b) < n) ++b;
  return b;
}

CsrWs csr_ws(void* base, int64_t Nn, int64_t E) {
  CsrWs w{};
  size_t sort_b = 0, scan_b = 0, max_b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const int32_t*)nullptr, (int32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)E, 0, key_bits(Nn));
  cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(Nn + 1));
  cub::DeviceReduce::Max(nullptr, max_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(Nn + 1));
  w.cub_bytes = sort_b > scan_b ? sort_b : scan_b;
  if (max_b > w.cub_bytes) w.cub_bytes = max_b;
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  w.cnt = reinterpret_cast<int32_t*>(p + off); off += align256((size_t)(Nn + 1) * 4);
  w.iota = reinterpret_cast<int32_t*>(p + off); off += align256((size_t)E * 4);
  w.keys = reinterpret_cast<int32_t*>(p + off); off += align256((size_t)E * 4);
  w.cub = p + off; off += align256(w.cub_bytes);
  w.total = off;
  return w;
}

// one orientation: ptr[Nn+1], eid[E] = edge ids stably sorted by key; optionally the largest bucket
int csr_one(const int32_t* key, int64_t Nn, int64_t E, int32_t* ptr, int32_t* eid, int32_t* max_deg, const CsrWs& w,
            cudaStream_t st) {
  cudaMemsetAsync(w.cnt, 0, (size_t)(Nn + 1) * 4, st);
  if (E > 0) iota_hist_kernel<<<blocks_for(E), kBlock, 0, st>>>(key, E, w.cnt, w.iota);
  size_t b = w.cub_bytes;
  if (max_deg) cub::DeviceReduce::Max(w.cub, b, w.cnt, max_deg, (int)(Nn + 1), st);
  b = w.cub_bytes;
  cub::DeviceScan::ExclusiveSum(w.cub, b, w.cnt, ptr, (int)(Nn + 1), st);
  if (E > 0) {
    b = w.cub_bytes;
    cub::DeviceRadixSort::SortPairs(w.cub, b, key, w.keys, w.iota, eid, (int)E, 0, key_bits(Nn), st);   // LSD radix: stable
  }
  return alignn::check_launch();
}

// ---- line graph ---------------------------------------------------------------------------------
// pairs ending in bond j: every bond i that ends where j starts (dst(i) == src(j)), except j itself (a self-loop bond
// sits in the in-list of its own source)
__global__ void lg_count_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                const int32_t* __restrict__ in_ptr, int64_t E, int32_t* __restrict__ cnt) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j > E) return;
  if (j == E) { cnt[E] = 0; return; }
  const int32_t a = src[j];
  cnt[j] = in_ptr[a + 1] - in_ptr[a] - (dst[j] == a ? 1 : 0);
}

// one warp per bond j; sources ascending (the in-list is sorted by edge id), destination-major output
__global__ void lg_fill_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                               const int32_t* __restrict__ in_ptr, const int32_t* __restrict__ in_eid, int64_t E,
                               const int32_t* __restrict__ off, int32_t* __restrict__ lsrc, int32_t* __restrict__ ldst) {
  const int lane = threadIdx.x & 31;
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (j >= E) return;
  const int32_t a = src[j];
  const int32_t p0 = in_ptr[a], n = in_ptr[a + 1] - p0;
  const bool self = dst[j] == a;
  const int32_t o = off[j];
  for (int32_t q = lane; q < n; q += 32) {
    const int32_t i = in_eid[p0 + q];
    if (i == (int32_t)j) continue;
    const int32_t k = q - ((self && i > (int32_t)j) ? 1 : 0);     // entries after the self pair move up by one
    lsrc[o + k] = i;
    ldst[o + k] = (int32_t)j;
  }
}

// ---- forces and stress (alignn_atomwise.py:547-563, 610-635) -----------------------------------------
__global__ void pair_force_scatter_kernel(const float* __restrict__ pf, const int32_t* __restrict__ in_ptr,
                                          const int32_t* __restrict__ in_eid, const int32_t* __restrict__ out_ptr,
                                          const int32_t* __restrict__ out_eid, int64_t Nn, int add_reverse,
                                          float* __restrict__ forces) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= Nn) return;
  float fx = 0.f, fy = 0.f, fz = 0.f;
  for (int32_t p = in_ptr[v]; p < in_ptr[v + 1]; ++p) {           // copy_e/sum over in-edges, edge-id order
    const int64_t e = in_eid ? in_eid[p] : p;
    fx += pf[3 * e]; fy += pf[3 * e + 1]; fz += pf[3 * e + 2];
  }
  if (add_reverse) {
    float gx = 0.f, gy = 0.f, gz = 0.f;
    for (int32_t p = out_ptr[v]; p < out_ptr[v + 1]; ++p) {       // ... minus the same over out-edges
      const int64_t e = out_eid[p];
      gx += pf[3 * e]; gy += pf[3 * e + 1]; gz += pf[3 * e + 2];
    }
    fx -= gx; fy -= gy; fz -= gz;
  }
  forces[3 * v] = fx; forces[3 * v + 1] = fy; forces[3 * v + 2] = fz;
}

// one block per crystal: sum_e r_e (x) F_e over the crystal's edge range, fixed-order tree in shared memory
__global__ void __launch_bounds__(kBlock)
virial_stress_kernel(const float* __restrict__ r, const float* __restrict__ pf, const int64_t* __restrict__ edge_off,
                     const int64_t* __restrict__ node_off, const float* __restrict__ V, float factor,
                     float* __restrict__ out) {
  __shared__ float red[kBlock][9];
  const int b = blockIdx.x;
  float acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k] = 0.f;
  for (int64_t e = edge_off[b] + threadIdx.x; e < edge_off[b + 1]; e += kBlock) {
    const float rx = r[3 * e], ry = r[3 * e + 1], rz = r[3 * e + 2];
    const float fx = pf[3 * e], fy = pf[3 * e + 1], fz = pf[3 * e + 2];
    acc[0] += rx * fx; acc[1] += rx * fy; acc[2] += rx * fz;
    acc[3] += ry * fx; acc[4] += ry * fy; acc[5] += ry * fz;
    acc[6] += rz * fx; acc[7] += rz * fy; acc[8] += rz * fz;
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) red[threadIdx.x][k] = acc[k];
  __syncthreads();
  for (int s = kBlock / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
#pragma unroll
      for (int k = 0; k < 9; ++k) red[threadIdx.x][k] += red[threadIdx.x + s][k];
    __syncthreads();
  }
  if (threadIdx.x < 9) out[9 * b + threadIdx.x] = factor * red[0][threadIdx.x] / V[node_off[b]];   // first atom's volume
}

}  // namespace device
}  // namespace alignn

extern "C" {

size_t alignn_b200_csr_build_workspace_bytes(int64_t num_nodes, int64_t num_edges) {
  if (num_nodes < 0 || num_edges < 0 || num_nodes >= ((int64_t)1 << 31) - 1 || num_edges >= ((int64_t)1 << 31)) return 0;
  return alignn::device::csr_ws(nullptr, num_nodes, num_edges).total;
}

int alignn_b200_csr_build(const int32_t* src, const int32_t* dst, int64_t num_nodes, int64_t num_edges, int32_t* in_ptr,
                          int32_t* in_eid, int32_t* out_ptr, int32_t* out_eid, int32_t* flags, void* workspace,
                          size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::device;
  if (num_nodes < 0 || num_edges < 0 || num_nodes >= ((int64_t)1 << 31) - 1 || num_edges >= ((int64_t)1 << 31)) return ALIGNN_ERR_BAD_ARG;
  if (!in_ptr || !out_ptr || !flags || !workspace || (num_edges > 0 && (!src || !dst || !in_eid || !out_eid))) return ALIGNN_ERR_BAD_ARG;
  const CsrWs w = csr_ws(workspace, num_nodes, num_edges);
  if (workspace_bytes < w.total) return ALIGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t one = 1;
  cudaMemcpyAsync(flags, &one, 4, cudaMemcpyHostToDevice, st);      // flags[0] = dst_sorted (cleared by the check kernel)
  if (num_edges > 1) sorted_flag_kernel<<<blocks_for(num_edges), kBlock, 0, st>>>(dst, num_edges, flags);
  int rc = csr_one(dst, num_nodes, num_edges, in_ptr, in_eid, flags + 1, w, st);   // flags[1] = max in-degree
  if (rc != ALIGNN_OK) return rc;
  return csr_one(src, num_nodes, num_edges, out_ptr, out_eid, nullptr, w, st);
}

size_t alignn_b200_line_graph_workspace_bytes(int64_t num_edges) {
  if (num_edges < 0 || num_edges >= ((int64_t)1 << 31) - 1) return 0;
  size_t scan_b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(num_edges + 1));
  return alignn::device::align256((size_t)(num_edges + 1) * 4) + alignn::device::align256(scan_b);
}

int alignn_b200_line_graph_offsets(const int32_t* src, const int32_t* dst, const int32_t* in_ptr, int64_t num_edges,
                                   int32_t* offsets, void* workspace, size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::device;
  if (num_edges < 0 || num_edges >= ((int64_t)1 << 31) - 1 || !offsets || !workspace) return ALIGNN_ERR_BAD_ARG;
  if (num_edges > 0 && (!src || !dst || !in_ptr)) return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < alignn_b200_line_graph_workspace_bytes(num_edges)) return ALIGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* cnt = reinterpret_cast<int32_t*>(workspace);
  void* cubws = reinterpret_cast<uint8_t*>(workspace) + align256((size_t)(num_edges + 1) * 4);
  size_t b = workspace_bytes - align256((size_t)(num_edges + 1) * 4);
  lg_count_kernel<<<blocks_for(num_edges + 1), kBlock, 0, st>>>(src, dst, in_ptr, num_edges, cnt);
  cub::DeviceScan::ExclusiveSum(cubws, b, cnt, offsets, (int)(num_edges + 1), st);      // offsets[E] = T; also L(g)'s in_ptr
  return alignn::check_launch();
}

int alignn_b200_line_graph_fill(const int32_t* src, const int32_t* dst, const int32_t* in_ptr, const int32_t* in_eid,
                                int64_t num_edges, const int32_t* offsets, int32_t* lsrc, int32_t* ldst, alignn_stream_t stream) {
  using namespace alignn::device;
  if (num_edges < 0) return ALIGNN_ERR_BAD_ARG;
  if (num_edges == 0) return ALIGNN_OK;
  if (!src || !dst || !in_ptr || !in_eid || !offsets || !lsrc || !ldst) return ALIGNN_ERR_BAD_ARG;
  lg_fill_kernel<<<blocks_for(num_edges * 32), kBlock, 0, (cudaStream_t)stream>>>(src, dst, in_ptr, in_eid, num_edges, offsets,
                                                                                lsrc, ldst);
  return alignn::check_launch();
}

int alignn_b200_pair_force_scatter(const float* pair_forces, const int32_t* in_ptr, const int32_t* in_eid,
                                   const int32_t* out_ptr, const int32_t* out_eid, int64_t num_nodes, int add_reverse,
                                   float* forces, alignn_stream_t stream) {
  using namespace alignn::device;
  if (num_nodes < 0) return ALIGNN_ERR_BAD_ARG;
  if (num_nodes == 0) return ALIGNN_OK;
  if (!pair_forces || !in_ptr || !forces || (add_reverse && (!out_ptr || !out_eid))) return ALIGNN_ERR_BAD_ARG;
  pair_force_scatter_kernel<<<blocks_for(num_nodes), kBlock, 0, (cudaStream_t)stream>>>(pair_forces, in_ptr, in_eid, out_ptr,
                                                                                         out_eid, num_nodes, add_reverse, forces);
  return alignn::check_launch();
}

int alignn_b200_virial_stress(const float* r, const float* pair_forces, const int64_t* edge_offsets,
                              const int64_t* node_offsets, const float* V, int64_t batch_size, float multiplier,
                              float* stress, alignn_stream_t stream) {
  using namespace alignn::device;
  if (batch_size < 0) return ALIGNN_ERR_BAD_ARG;
  if (batch_size == 0) return ALIGNN_OK;
  if (!r || !pair_forces || !edge_offsets || !node_offsets || !V || !stress) return ALIGNN_ERR_BAD_ARG;
  virial_stress_kernel<<<(int)batch_size, kBlock, 0, (cudaStream_t)stream>>>(r, pair_forces, edge_offsets, node_offsets, V,
                                                                            -160.21766208f * multiplier, stress);
  return alignn::check_launch();
}

}  // extern "C"
