// Periodic crystal graphs built on the device for a whole batch of structures (SURVEY.md section 8f row 4): the
// neighbour scan shared by both strategies of `Graph.atom_dgl_multigraph` (alignn/graphs.py:472-589), and the k-nearest
// shell selection with undirected canonicalisation (`nearest_neighbor_edges` + `build_undirected_edgedata`,
// graphs.py:127-264, use_canonize=True).  The single-crystal radius entry points (alignn_b200_radius_graph_*) are a
// batch of one on the same scan kernel.
//
// Integer order comes from prefix sums and stable radix sorts; the only atomics are integer min / or on a per-crystal
// status word.  Distances are double precision with the host builder's operation order, so the device graphs are the
// host builders' graphs bit for bit.
#include <cub/cub.cuh>
#include <math.h>
#include <stdint.h>

#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace crystal {

constexpr int kBlock = 256;
inline int blocks_for(int64_t n) { return (int)((n + kBlock - 1) / kBlock); }
inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }
inline int key_bits(uint64_t n) {
  int b = 1;
  while (b < 64 && ((uint64_t)1 << b) < n) ++b;
  return b;
}

// The crystal-batch view the scan needs, by value.  `crystal == nullptr` is a batch of one: atoms [0, n), images
// [0, n_images), cutoff `cutoff1`.
struct ScanView {
  const double* X;
  const double* shifts;
  const double* cells;
  const int64_t* atom_off;
  const int64_t* shift_off;
  const int32_t* crystal;
  const double* cutoffs;
  int64_t n, n_images;
  double cutoff1, atol;
};

struct Range {
  int32_t b;
  int64_t a0, a1, s0, s1;
  double cutoff;
};

__device__ __forceinline__ Range range_of(const ScanView& s, int64_t u) {
  if (!s.crystal) return Range{0, 0, s.n, 0, s.n_images, s.cutoff1};
  const int32_t b = s.crystal[u];
  return Range{b, s.atom_off[b], s.atom_off[b + 1], s.shift_off[b], s.shift_off[b + 1], s.cutoffs[b]};
}

enum ScanMode { kCount = 0, kFillRadius = 1, kFillKnn = 2 };
enum Strategy { kRadius = 0, kKnn = 1 };

// One warp per atom u walks (image c, atom v) of u's own crystal in the host builder's order; 32 candidates per step, a
// ballot gives each hit its ordered slot.  Double precision with explicit round-to-nearest operations (no FMA
// contraction), the operation order of csrc/graph_host.cu: d = (shift + x_v) - x_u ; dist = sqrt((dx*dx + dy*dy) + dz*dz).
//   kCount:      cnt[u] = hits; status[b] = min over the crystal's atoms of the hit count (k-NN growth test,
//                graphs.py:166-186) or 1 if the crystal's last atom has a bond (radius growth test, graphs.py:347-350).
//   kFillRadius: bonds (u, v, fp32 displacement, optional local image index, optional fp32 image) in (u, c, v)
//                order.
//   kFillKnn:    candidates (dist, (local v << 32) | local image index) in (c, v) order.
template <int kMode>
__global__ void crystal_scan_kernel(ScanView s, int strategy, const int32_t* __restrict__ off, int32_t* __restrict__ cnt,
                                    int32_t* __restrict__ status, int32_t* __restrict__ u_out, int32_t* __restrict__ v_out,
                                    int32_t* __restrict__ c_out, float* __restrict__ r_out, float* __restrict__ img_out,
                                    double* __restrict__ dist_out, uint64_t* __restrict__ key_out) {
  const int lane = threadIdx.x & 31;
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (u >= s.n) return;
  const Range rg = range_of(s, u);
  const double* __restrict__ X = s.X;
  const double xu = X[3 * u], yu = X[3 * u + 1], zu = X[3 * u + 2];
  const int64_t last = rg.a1 - 1;
  bool last_bonded = false;
  int32_t t = kMode != kCount ? off[u] : 0;
  for (int64_t c = rg.s0; c < rg.s1; ++c) {
    const double sx = s.shifts[3 * c], sy = s.shifts[3 * c + 1], sz = s.shifts[3 * c + 2];
    for (int64_t v0 = rg.a0; v0 < rg.a1; v0 += 32) {
      const int64_t v = v0 + lane;
      bool hit = false;
      double dx = 0.0, dy = 0.0, dz = 0.0, dist = 0.0;
      if (v < rg.a1) {
        dx = __dsub_rn(__dadd_rn(sx, X[3 * v]), xu);
        dy = __dsub_rn(__dadd_rn(sy, X[3 * v + 1]), yu);
        dz = __dsub_rn(__dadd_rn(sz, X[3 * v + 2]), zu);
        dist = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
        hit = dist <= rg.cutoff && !(fabs(dist) <= s.atol);
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (kMode == kCount) last_bonded |= hit && v == last;
      if (kMode != kCount && hit) {
        const int32_t k = t + __popc(m & ((1u << lane) - 1u));
        if (kMode == kFillRadius) {
          u_out[k] = (int32_t)u; v_out[k] = (int32_t)v;
          if (c_out) c_out[k] = (int32_t)(c - rg.s0);
          r_out[3 * k] = (float)dx; r_out[3 * k + 1] = (float)dy; r_out[3 * k + 2] = (float)dz;
          if (img_out) {
            img_out[3 * k] = (float)s.cells[3 * c];
            img_out[3 * k + 1] = (float)s.cells[3 * c + 1];
            img_out[3 * k + 2] = (float)s.cells[3 * c + 2];
          }
        } else {
          dist_out[k] = dist;
          key_out[k] = ((uint64_t)(v - rg.a0) << 32) | (uint64_t)(c - rg.s0);
        }
      }
      t += __popc(m);
    }
  }
  if (kMode == kCount) {
    last_bonded = __any_sync(0xffffffffu, last_bonded) || (u == last && t > 0);
    if (lane == 0) {
      cnt[u] = t;
      if (status) {
        if (strategy == kKnn) atomicMin(&status[rg.b], t);
        else if (last_bonded) atomicOr(&status[rg.b], 1);
      }
    }
  }
}

// ---- k-NN shell selection (graphs.py:202-214) ----------------------------------------------------------------------
// One warp per atom ranks its m candidates under the key (dist, v, image): rank_i = #{j : key_j < key_i}.  The keys are
// distinct ((v, image) is unique per atom), so the ranks are a permutation and writing each candidate to its rank sorts
// them.  kth = dist at rank k-1; the kept entries are the first #{i : dist_i <= kth} of the sorted list, compared exactly
// in double as the reference does.  Candidates are staged in shared memory when they fit a warp's tile; a larger list
// (a small cell after cutoff doubling) is ranked straight from global memory.
constexpr int kShellWarps = 4;
constexpr int kShellTile = 384;

__global__ void __launch_bounds__(kShellWarps * 32)
knn_shell_kernel(const int32_t* __restrict__ off, const double* __restrict__ dist, const uint64_t* __restrict__ key, int64_t n,
                 int k, uint64_t* __restrict__ sorted_key, int32_t* __restrict__ kept) {
  __shared__ double sd[kShellWarps][kShellTile];
  __shared__ uint64_t sk[kShellWarps][kShellTile];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t u = (int64_t)blockIdx.x * kShellWarps + warp;
  if (u >= n) return;
  const int32_t p0 = off[u], m = off[u + 1] - p0;
  const bool staged = m <= kShellTile;
  if (staged) {
    for (int i = lane; i < m; i += 32) { sd[warp][i] = dist[p0 + i]; sk[warp][i] = key[p0 + i]; }
    __syncwarp();
  }
  const double* D = staged ? sd[warp] : dist + p0;
  const uint64_t* K = staged ? sk[warp] : key + p0;
  double kth = INFINITY;                   // fewer than k candidates (not produced by the growth rule): keep them all
  for (int i0 = 0; i0 < m; i0 += 32) {
    const int i = i0 + lane;
    int r = 0;
    double di = 0.0;
    if (i < m) {
      di = D[i];
      const uint64_t ki = K[i];
      for (int j = 0; j < m; ++j) {
        const double dj = D[j];
        r += (dj < di || (dj == di && K[j] < ki)) ? 1 : 0;
      }
      sorted_key[p0 + r] = ki;
    }
    const unsigned at = __ballot_sync(0xffffffffu, i < m && r == k - 1);
    if (at) kth = __shfl_sync(0xffffffffu, di, __ffs(at) - 1);
  }
  int32_t nk = 0;
  for (int i0 = 0; i0 < m; i0 += 32) {
    const int i = i0 + lane;
    nk += __popc(__ballot_sync(0xffffffffu, i < m && D[i] <= kth));
  }
  if (lane == 0) kept[u] = nk;
}

// ---- canonicalisation (graphs.py:127-152, 218-223) ------------------------------------------------------------------
// Kept entry (u, v, c) with global rank g becomes (u, v, c) if v >= u, else (v, u, -c); on the symmetric k-NN image
// table -c is index I-1-c.  Records: pair key a * n + b, the pair's atoms and image, and g itself (the sort value).
__global__ void knn_canon_kernel(ScanView s, const int32_t* __restrict__ off, const int32_t* __restrict__ koff,
                                 const uint64_t* __restrict__ sorted_key, uint64_t* __restrict__ pair_key,
                                 int32_t* __restrict__ rec_a, int32_t* __restrict__ rec_b, int32_t* __restrict__ rec_c,
                                 int32_t* __restrict__ iota) {
  const int lane = threadIdx.x & 31;
  const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (u >= s.n) return;
  const Range rg = range_of(s, u);
  const int64_t n_img = rg.s1 - rg.s0, ul = u - rg.a0;
  const int32_t g0 = koff[u], nk = koff[u + 1] - g0, p0 = off[u];
  for (int r = lane; r < nk; r += 32) {
    const uint64_t kv = sorted_key[p0 + r];
    const int64_t vl = (int64_t)(kv >> 32), c = (int64_t)(kv & 0xffffffffu);
    int64_t a, b, cc;
    if (vl >= ul) { a = u; b = rg.a0 + vl; cc = c; }
    else { a = rg.a0 + vl; b = u; cc = n_img - 1 - c; }
    const int32_t g = g0 + r;
    pair_key[g] = (uint64_t)a * (uint64_t)s.n + (uint64_t)b;
    rec_a[g] = (int32_t)a; rec_b[g] = (int32_t)b; rec_c[g] = (int32_t)cc;
    iota[g] = g;
  }
}

// After the stable sort by pair key each pair is one segment whose first record has the pair's smallest rank.
__global__ void segment_head_kernel(const uint64_t* __restrict__ pk, int64_t R, int32_t* __restrict__ head) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  head[i] = (i == 0 || pk[i] != pk[i - 1]) ? (int32_t)i : 0;
}

// second key: (smallest rank of the pair, image) -- pairs in order of first encounter, images ascending inside a pair
__global__ void order_key_kernel(const int32_t* __restrict__ head_pos, const int32_t* __restrict__ g_sorted,
                                 const int32_t* __restrict__ rec_c, int64_t R, int cbits, uint64_t* __restrict__ key2) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  const uint64_t first = (uint64_t)g_sorted[head_pos[i]];
  key2[i] = (first << cbits) | (uint64_t)rec_c[g_sorted[i]];
}

__global__ void unique_flag_kernel(const uint64_t* __restrict__ key, int64_t R, int32_t* __restrict__ flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > R) return;
  flag[i] = (i < R && (i == 0 || key[i] != key[i - 1])) ? 1 : 0;
}

// bonds before crystal b = 2 x unique (pair, image) records of crystals < b; crystal b's records are the sorted
// positions [koff[atom_off[b]], koff[atom_off[b+1]]) because every record sorts by a rank of its own crystal
__global__ void bond_offsets_kernel(const int64_t* __restrict__ atom_off, const int32_t* __restrict__ koff,
                                    const int32_t* __restrict__ uidx, int64_t B, int64_t* __restrict__ bond_off) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  bond_off[b] = 2 * (int64_t)uidx[koff[atom_off[b]]];
}

// build_undirected_edgedata (graphs.py:240-257): every unique (a, b, image) emits (a, b, d) then (b, a, -d) with
// d = ((frac_b + image) - frac_a) @ lattice in double, rounded once to fp32; both rows carry the image.  The row-vector
// product is the fused chain fma(f2, L2q, fma(f1, L1q, fma(f0, L0q, +0))): the order numpy's `@` (OpenBLAS dgemv on
// x86-64 with FMA, accumulator starting at +0) evaluates it in, so components that cancel to rounding noise (atoms on
// symmetry planes) and signed zeros match as well.
__global__ void knn_emit_kernel(ScanView s, const double* __restrict__ frac, const double* __restrict__ lat,
                                const uint64_t* __restrict__ key2, const int32_t* __restrict__ g2,
                                const int32_t* __restrict__ uidx, const int32_t* __restrict__ rec_a,
                                const int32_t* __restrict__ rec_b, const int32_t* __restrict__ rec_c, int64_t R,
                                int32_t* __restrict__ u_out, int32_t* __restrict__ v_out, float* __restrict__ r_out,
                                float* __restrict__ img_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R || (i > 0 && key2[i] == key2[i - 1])) return;
  const int64_t j = uidx[i];
  const int32_t g = g2[i], a = rec_a[g], b = rec_b[g];
  const int32_t cr = s.crystal ? s.crystal[a] : 0;
  const int64_t ci = (s.crystal ? s.shift_off[cr] : 0) + rec_c[g];
  const double* L = lat + 9 * cr;
  double f[3], img[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    img[q] = s.cells[3 * ci + q];
    f[q] = __dsub_rn(__dadd_rn(frac[3 * (int64_t)b + q], img[q]), frac[3 * (int64_t)a + q]);
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const double d = __fma_rn(f[2], L[6 + q], __fma_rn(f[1], L[3 + q], __fma_rn(f[0], L[q], 0.0)));
    const float df = (float)d;
    r_out[6 * j + q] = df;
    r_out[6 * j + 3 + q] = -df;
    img_out[6 * j + q] = (float)img[q];
    img_out[6 * j + 3 + q] = (float)img[q];
  }
  u_out[2 * j] = a; v_out[2 * j] = b;
  u_out[2 * j + 1] = b; v_out[2 * j + 1] = a;
}

// ---- host helpers -------------------------------------------------------------------------------------------------
inline bool batch_ok(const alignn_b200_crystal_batch* bt) {
  if (!bt || bt->num_crystals < 1 || bt->num_atoms < 1 || bt->num_images < 1 || bt->max_images < 1) return false;
  if (bt->num_atoms >= ((int64_t)1 << 31) - 1 || bt->num_images >= ((int64_t)1 << 31)) return false;
  if (!bt->cart_coords || !bt->shifts || !bt->cells || !bt->lattices || !bt->atom_offsets || !bt->shift_offsets ||
      !bt->crystal_of_atom || !bt->cutoffs)
    return false;
  for (int64_t b = 0; b < bt->num_crystals; ++b) {        // a crystal whose lattice has no inverse is rejected
    const double* m = bt->lattices + 9 * b;
    const double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
    if (!(det != 0.0) || !isfinite(det)) return false;
  }
  return true;
}

inline ScanView view_of(const alignn_b200_crystal_batch* bt) {
  return ScanView{bt->cart_coords, bt->shifts, bt->cells, bt->atom_offsets, bt->shift_offsets, bt->crystal_of_atom,
                  bt->cutoffs, bt->num_atoms, bt->num_images, 0.0, bt->atol};
}

size_t scan_ws_bytes(int64_t n) {
  size_t scan_b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1));
  return align256((size_t)(n + 1) * 4) + align256(scan_b);
}

// count pass + exclusive scan -> offsets[n+1] (offsets[n] = hits)
int scan_count(const ScanView& s, int strategy, int32_t* offsets, int32_t* status, int64_t B, void* ws, size_t wsb,
               cudaStream_t st) {
  int32_t* cnt = reinterpret_cast<int32_t*>(ws);
  void* cubws = reinterpret_cast<uint8_t*>(ws) + align256((size_t)(s.n + 1) * 4);
  size_t b = wsb - align256((size_t)(s.n + 1) * 4);
  cudaMemsetAsync(cnt, 0, (size_t)(s.n + 1) * 4, st);
  if (status) cudaMemsetAsync(status, strategy == kKnn ? 0x7f : 0, (size_t)B * 4, st);    // 0x7f7f7f7f: +large for min
  if (s.n > 0)
    crystal_scan_kernel<kCount><<<blocks_for(s.n * 32), kBlock, 0, st>>>(s, strategy, nullptr, cnt, status, nullptr, nullptr,
                                                                         nullptr, nullptr, nullptr, nullptr, nullptr);
  cub::DeviceScan::ExclusiveSum(cubws, b, cnt, offsets, (int)(s.n + 1), st);
  return check_launch();
}

// k-NN workspace: the candidate, sorted and record arrays are sized by the candidate count C (>= the kept count R)
struct KnnWs {
  double* cand_dist;      // [C]
  uint64_t* cand_key;     // [C]
  uint64_t* sorted_key;   // [C]  per atom: candidates in (dist, v, image) order
  int32_t* kept;          // [n+1]
  uint64_t* pair_key;     // [C]
  uint64_t* pair_sorted;  // [C]
  int32_t* iota;          // [C]
  int32_t* g_sorted;      // [C]
  int32_t* rec_a;         // [C]
  int32_t* rec_b;         // [C]
  int32_t* rec_c;         // [C]
  int32_t* head;          // [C]
  int32_t* head_pos;      // [C]
  uint64_t* key2;         // [C]
  uint64_t* key2_sorted;  // [C]
  int32_t* g2;            // [C]
  int32_t* flag;          // [C+1]
  int32_t* uidx;          // [C+1]
  double* lat;            // [B*9]
  void* cub;
  size_t cub_bytes, total;
};

KnnWs knn_ws(void* base, int64_t n, int64_t B, int64_t C) {
  KnnWs w{};
  const int items = (int)(C > 0 ? C : 1);
  size_t a = 0, b = 0, c = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, items, 0, 64);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)((n > C ? n : C) + 1));
  cub::DeviceScan::InclusiveScan(nullptr, c, (const int32_t*)nullptr, (int32_t*)nullptr, cub::Max(), items);
  w.cub_bytes = a;
  if (b > w.cub_bytes) w.cub_bytes = b;
  if (c > w.cub_bytes) w.cub_bytes = c;
  uint8_t* p = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { void* q = p + off; off += align256(bytes); return q; };
  const size_t c8 = (size_t)C * 8, c4 = (size_t)C * 4;
  w.cand_dist = (double*)take(c8);
  w.cand_key = (uint64_t*)take(c8);
  w.sorted_key = (uint64_t*)take(c8);
  w.kept = (int32_t*)take((size_t)(n + 1) * 4);
  w.pair_key = (uint64_t*)take(c8);
  w.pair_sorted = (uint64_t*)take(c8);
  w.iota = (int32_t*)take(c4);
  w.g_sorted = (int32_t*)take(c4);
  w.rec_a = (int32_t*)take(c4);
  w.rec_b = (int32_t*)take(c4);
  w.rec_c = (int32_t*)take(c4);
  w.head = (int32_t*)take(c4);
  w.head_pos = (int32_t*)take(c4);
  w.key2 = (uint64_t*)take(c8);
  w.key2_sorted = (uint64_t*)take(c8);
  w.g2 = (int32_t*)take(c4);
  w.flag = (int32_t*)take(c4 + 4);
  w.uidx = (int32_t*)take(c4 + 4);
  w.lat = (double*)take((size_t)B * 72);
  w.cub = take(w.cub_bytes);
  w.total = off;
  return w;
}

}  // namespace crystal
}  // namespace alignn

extern "C" {

// ---- single crystal: a batch of one on the scan kernel --------------------------------------------------------------
size_t alignn_b200_radius_graph_workspace_bytes(int64_t num_atoms) {
  if (num_atoms < 0 || num_atoms >= ((int64_t)1 << 31) - 1) return 0;
  return alignn::crystal::scan_ws_bytes(num_atoms);
}

int alignn_b200_radius_graph_offsets(const double* cart_coords, const double* shifts, int64_t num_atoms, int64_t num_images,
                                     double cutoff, double atol, int32_t* offsets, void* workspace, size_t workspace_bytes,
                                     alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (num_atoms < 0 || num_images < 0 || !offsets || !workspace || (num_atoms > 0 && !cart_coords) || (num_images > 0 && !shifts))
    return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < alignn_b200_radius_graph_workspace_bytes(num_atoms)) return ALIGNN_ERR_WORKSPACE;
  const ScanView s{cart_coords, shifts, nullptr, nullptr, nullptr, nullptr, nullptr, num_atoms, num_images, cutoff, atol};
  return scan_count(s, kRadius, offsets, nullptr, 1, workspace, workspace_bytes, (cudaStream_t)stream);
}

int alignn_b200_radius_graph_fill(const double* cart_coords, const double* shifts, int64_t num_atoms, int64_t num_images,
                                  double cutoff, double atol, const int32_t* offsets, int32_t* u, int32_t* v,
                                  int32_t* image_index, float* r, alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (num_atoms < 0 || num_images < 0) return ALIGNN_ERR_BAD_ARG;
  if (num_atoms == 0) return ALIGNN_OK;
  if (!cart_coords || (num_images > 0 && !shifts) || !offsets || !u || !v || !image_index || !r) return ALIGNN_ERR_BAD_ARG;
  const ScanView s{cart_coords, shifts, nullptr, nullptr, nullptr, nullptr, nullptr, num_atoms, num_images, cutoff, atol};
  crystal_scan_kernel<kFillRadius><<<blocks_for(num_atoms * 32), kBlock, 0, (cudaStream_t)stream>>>(
      s, kRadius, offsets, nullptr, nullptr, u, v, image_index, r, nullptr, nullptr, nullptr);
  return alignn::check_launch();
}

// ---- batched scan -------------------------------------------------------------------------------------------------
size_t alignn_b200_crystal_scan_workspace_bytes(int64_t num_atoms) {
  if (num_atoms < 1 || num_atoms >= ((int64_t)1 << 31) - 1) return 0;
  return alignn::crystal::scan_ws_bytes(num_atoms);
}

int alignn_b200_crystal_scan_count(const alignn_b200_crystal_batch* batch, int strategy, int32_t* offsets, int32_t* status,
                                   void* workspace, size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (!batch_ok(batch) || (strategy != kRadius && strategy != kKnn) || !offsets || !status || !workspace)
    return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < alignn_b200_crystal_scan_workspace_bytes(batch->num_atoms)) return ALIGNN_ERR_WORKSPACE;
  return scan_count(view_of(batch), strategy, offsets, status, batch->num_crystals, workspace, workspace_bytes,
                    (cudaStream_t)stream);
}

int alignn_b200_crystal_radius_fill(const alignn_b200_crystal_batch* batch, const int32_t* offsets, int32_t* u, int32_t* v,
                                    float* r, float* images, alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (!batch_ok(batch) || !offsets || !u || !v || !r || !images) return ALIGNN_ERR_BAD_ARG;
  const ScanView s = view_of(batch);
  crystal_scan_kernel<kFillRadius><<<blocks_for(s.n * 32), kBlock, 0, (cudaStream_t)stream>>>(
      s, kRadius, offsets, nullptr, nullptr, u, v, nullptr, r, images, nullptr, nullptr);
  return alignn::check_launch();
}

// ---- k-nearest neighbours -----------------------------------------------------------------------------------------
size_t alignn_b200_knn_graph_workspace_bytes(int64_t num_atoms, int64_t num_crystals, int64_t num_candidates) {
  if (num_atoms < 1 || num_crystals < 1 || num_candidates < 0 || num_atoms >= ((int64_t)1 << 31) - 1 ||
      num_candidates >= ((int64_t)1 << 31) - 1)
    return 0;
  return alignn::crystal::knn_ws(nullptr, num_atoms, num_crystals, num_candidates).total;
}

int alignn_b200_knn_graph_select(const alignn_b200_crystal_batch* batch, const int32_t* offsets, int64_t num_candidates,
                                 int max_neighbors, int32_t* kept_offsets, void* workspace, size_t workspace_bytes,
                                 alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (!batch_ok(batch) || max_neighbors < 1 || !offsets || !kept_offsets || !workspace) return ALIGNN_ERR_BAD_ARG;
  const size_t need = alignn_b200_knn_graph_workspace_bytes(batch->num_atoms, batch->num_crystals, num_candidates);
  if (need == 0) return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < need) return ALIGNN_ERR_WORKSPACE;
  const KnnWs w = knn_ws(workspace, batch->num_atoms, batch->num_crystals, num_candidates);
  const ScanView s = view_of(batch);
  cudaStream_t st = (cudaStream_t)stream;
  crystal_scan_kernel<kFillKnn><<<blocks_for(s.n * 32), kBlock, 0, st>>>(s, kKnn, offsets, nullptr, nullptr, nullptr, nullptr,
                                                                         nullptr, nullptr, nullptr, w.cand_dist, w.cand_key);
  cudaMemsetAsync(w.kept, 0, (size_t)(s.n + 1) * 4, st);
  knn_shell_kernel<<<(int)((s.n + kShellWarps - 1) / kShellWarps), kShellWarps * 32, 0, st>>>(
      offsets, w.cand_dist, w.cand_key, s.n, max_neighbors, w.sorted_key, w.kept);
  size_t b = w.cub_bytes;
  cub::DeviceScan::ExclusiveSum(w.cub, b, w.kept, kept_offsets, (int)(s.n + 1), st);
  return alignn::check_launch();
}

int alignn_b200_knn_graph_order(const alignn_b200_crystal_batch* batch, const int32_t* offsets, const int32_t* kept_offsets,
                                int64_t num_candidates, int64_t num_kept, int64_t* bond_offsets, void* workspace,
                                size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (!batch_ok(batch) || !offsets || !kept_offsets || !bond_offsets || !workspace || num_kept < 0 || num_kept > num_candidates)
    return ALIGNN_ERR_BAD_ARG;
  const size_t need = alignn_b200_knn_graph_workspace_bytes(batch->num_atoms, batch->num_crystals, num_candidates);
  if (need == 0) return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < need) return ALIGNN_ERR_WORKSPACE;
  const int pair_bits = key_bits((uint64_t)batch->num_atoms * (uint64_t)batch->num_atoms);
  const int cbits = key_bits((uint64_t)batch->max_images), rbits = key_bits((uint64_t)num_kept + 1);
  if (rbits + cbits > 64) return ALIGNN_ERR_BAD_ARG;
  const KnnWs w = knn_ws(workspace, batch->num_atoms, batch->num_crystals, num_candidates);
  const ScanView s = view_of(batch);
  const int64_t R = num_kept;
  cudaStream_t st = (cudaStream_t)stream;
  size_t b = 0;
  if (R > 0) {          // the temporary storage was sized for C items and 64 key bits; check the actual sorts fit
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b1, w.pair_key, w.pair_sorted, w.iota, w.g_sorted, (int)R, 0, pair_bits);
    cub::DeviceRadixSort::SortPairs(nullptr, b2, w.key2, w.key2_sorted, w.g_sorted, w.g2, (int)R, 0, rbits + cbits);
    if (b1 > w.cub_bytes || b2 > w.cub_bytes) return ALIGNN_ERR_WORKSPACE;
  }
  if (R > 0) {
    knn_canon_kernel<<<blocks_for(s.n * 32), kBlock, 0, st>>>(s, offsets, kept_offsets, w.sorted_key, w.pair_key, w.rec_a,
                                                              w.rec_b, w.rec_c, w.iota);
    b = w.cub_bytes;      // LSD radix sort: stable, so each pair's records stay in rank order
    cub::DeviceRadixSort::SortPairs(w.cub, b, w.pair_key, w.pair_sorted, w.iota, w.g_sorted, (int)R, 0, pair_bits, st);
    segment_head_kernel<<<blocks_for(R), kBlock, 0, st>>>(w.pair_sorted, R, w.head);
    b = w.cub_bytes;
    cub::DeviceScan::InclusiveScan(w.cub, b, w.head, w.head_pos, cub::Max(), (int)R, st);
    order_key_kernel<<<blocks_for(R), kBlock, 0, st>>>(w.head_pos, w.g_sorted, w.rec_c, R, cbits, w.key2);
    b = w.cub_bytes;
    cub::DeviceRadixSort::SortPairs(w.cub, b, w.key2, w.key2_sorted, w.g_sorted, w.g2, (int)R, 0, rbits + cbits, st);
  }
  unique_flag_kernel<<<blocks_for(R + 1), kBlock, 0, st>>>(w.key2_sorted, R, w.flag);
  b = w.cub_bytes;
  cub::DeviceScan::ExclusiveSum(w.cub, b, w.flag, w.uidx, (int)(R + 1), st);
  bond_offsets_kernel<<<blocks_for(batch->num_crystals + 1), kBlock, 0, st>>>(batch->atom_offsets, kept_offsets, w.uidx,
                                                                              batch->num_crystals, bond_offsets);
  return alignn::check_launch();
}

int alignn_b200_knn_graph_emit(const alignn_b200_crystal_batch* batch, const double* frac_coords, int64_t num_candidates,
                               int64_t num_kept, int32_t* u, int32_t* v, float* r, float* images, void* workspace,
                               size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::crystal;
  if (!batch_ok(batch) || !frac_coords || !workspace || num_kept < 0 || num_kept > num_candidates) return ALIGNN_ERR_BAD_ARG;
  if (num_kept > 0 && (!u || !v || !r || !images)) return ALIGNN_ERR_BAD_ARG;
  const size_t need = alignn_b200_knn_graph_workspace_bytes(batch->num_atoms, batch->num_crystals, num_candidates);
  if (need == 0) return ALIGNN_ERR_BAD_ARG;
  if (workspace_bytes < need) return ALIGNN_ERR_WORKSPACE;
  const KnnWs w = knn_ws(workspace, batch->num_atoms, batch->num_crystals, num_candidates);
  cudaStream_t st = (cudaStream_t)stream;
  const cudaError_t e = cudaMemcpyAsync(w.lat, batch->lattices, (size_t)batch->num_crystals * 72, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return alignn::record_cuda_error((int)e);
  if (num_kept == 0) return ALIGNN_OK;
  knn_emit_kernel<<<blocks_for(num_kept), kBlock, 0, st>>>(view_of(batch), frac_coords, w.lat, w.key2_sorted, w.g2, w.uidx,
                                                           w.rec_a, w.rec_b, w.rec_c, num_kept, u, v, r, images);
  return alignn::check_launch();
}

}  // extern "C"
