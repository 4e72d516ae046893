// Edge-gated graph convolution: gather / gate / segment-reduce / norm kernels, forward and
// backward, fp32, sm_90a.  One warp owns one destination node (one CSR segment): it walks the
// node's in-edges in sorted order, gathers the source rows by edge index, and reduces the gated
// messages in registers -- no atomics, deterministic, every global access a coalesced row.
//
// Reference math: alignn/models/alignn.py:98-127 (SURVEY.md App. B).  P is the [Nn,4d] node
// projection in the layout documented in include/alignn_b200.h: [e_src | Bh | e_dst | src_update].
#include "common.cuh"
#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {

// =============================================================================================
// Forward
// =============================================================================================
// GIM ("gate is m"): a.G already holds the pre-activation gate m = e_src[src] + e_dst[dst] + edge_gate(y), written
// (together with its batch statistics) by the gather GEMM (gemm_tc.cu).  The kernel then neither gathers
// e_src / e_dst nor writes M nor accumulates edge statistics: it is the second and last pass over the edge rows.
template <int D, bool GIM>
__global__ void __launch_bounds__(kThreads, 2)
egc_forward_kernel(alignn_b200_egc_fwd_args a) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  // norm vectors {n_w, n_b, e_w, e_b} and (STATS mode) the per-warp partial sums live in shared memory so
  // (the kernel sits at the L2-fabric limit -- G stream + row gathers -- so 2 blocks/SM are enough;
  //  3 blocks/SM were measured no faster)
  extern __shared__ __align__(16) float dyn_smem[];
  float* vec = dyn_smem;                       // [4][D]
  float* sacc = dyn_smem + 4 * D;              // [kWarpsPerBlock][4][D]   {sum m, sum m^2, sum x', sum x'^2}
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + wib;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  const bool train = a.XP != nullptr;      // (M is a null pointer for an edgeless graph, so XP marks training)
  const bool want_res = a.residual && a.y_out && a.norm_edges != ALIGNN_NORM_STATS;
  const bool stats = a.partials != nullptr;
  {
    const float* srcs[4] = {a.n_w, a.n_b, a.e_w, a.e_b};
#pragma unroll
    for (int q = 0; q < 4; ++q)
      for (int i = threadIdx.x; i < D; i += blockDim.x) vec[q * D + i] = srcs[q] ? srcs[q][i] : 0.f;
  }
  float* st = sacc + wib * 4 * D;
  if (stats)
    for (int i = lane; i < 4 * D; i += 32) st[i] = 0.f;
  __syncthreads();

  for (int64_t v = warp0; v < a.Nn; v += nwarps) {
    const int p0 = a.in_ptr[v], p1 = a.in_ptr[v + 1];
    float bv[V], accS[V], accSh[V];
    if constexpr (!GIM) ld_row<D, false>(bv, a.P + v * 4 * D + 2 * D, lane);
#pragma unroll
    for (int i = 0; i < V; ++i) { accS[i] = 0.f; accSh[i] = 0.f; }

    for (int base = p0; base < p1; base += 32) {
      const int cnt = min(32, p1 - base);
      int my_e = 0, my_s = 0;
      if (lane < cnt) {
        my_e = a.in_eid ? a.in_eid[base + lane] : base + lane;
        my_s = a.src[my_e];
      }
      // everything of one edge after its three rows have arrived
      // yr: the edge's residual row (requested together with its other rows, not after the gate math) when used
      auto edge_tail = [&](int64_t e, float (&m)[V], const float (&cv)[V], const float (&yr)[V]) {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float sg = sigmoidf_(m[k]);
          accS[k] += sg;
          accSh[k] += cv[k] * sg;
        }
        if (train && !GIM) st_row<D, true>(a.M + e * D, m, lane);   // Ne > 0 here, so M is a real buffer
        if (!GIM && a.norm_edges == ALIGNN_NORM_STATS) {
          smem_row_add<D>(st, m, lane);
#pragma unroll
          for (int k = 0; k < V; ++k) m[k] *= m[k];
          smem_row_add<D>(st + D, m, lane);
        } else if (a.y_out) {
          float o[V], ew[V], eb[V];
          ld_srow<D>(ew, vec + 2 * D, lane);
          ld_srow<D>(eb, vec + 3 * D, lane);
          if (a.norm_edges == ALIGNN_NORM_LAYER) {
            float mean, rstd;
            row_mean_rstd<D>(m, a.ln_eps, mean, rstd);
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] = silu_((m[k] - mean) * rstd * ew[k] + eb[k]);
          } else {
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] = silu_(m[k] * ew[k] + eb[k]);
          }
          if (a.residual) {
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] += yr[k];
          }
          st_row<D, true>(a.y_out + e * D, o, lane);
        }
      };
      int i = 0;
      for (; i + 1 < cnt; i += 2) {   // two edges (six row loads) in flight per warp
        const int64_t e0 = __shfl_sync(0xffffffffu, my_e, i), s0 = __shfl_sync(0xffffffffu, my_s, i);
        const int64_t e1 = __shfl_sync(0xffffffffu, my_e, i + 1), s1 = __shfl_sync(0xffffffffu, my_s, i + 1);
        float g0[V], a0[V], c0[V], g1[V], a1[V], c1[V], y0[V], y1[V];
        ld_row<D, true>(g0, a.G + e0 * D, lane);
        ld_row<D, true>(g1, a.G + e1 * D, lane);
        if (want_res) {
          ld_row<D, true>(y0, a.y + e0 * D, lane);
          ld_row<D, true>(y1, a.y + e1 * D, lane);
        }
        if constexpr (!GIM) {
          ld_row<D, false>(a0, a.P + s0 * 4 * D, lane);
          ld_row<D, false>(a1, a.P + s1 * 4 * D, lane);
        }
        ld_row<D, false>(c0, a.P + s0 * 4 * D + D, lane);
        ld_row<D, false>(c1, a.P + s1 * 4 * D + D, lane);
        if constexpr (!GIM) {
#pragma unroll
          for (int k = 0; k < V; ++k) { g0[k] += a0[k] + bv[k]; g1[k] += a1[k] + bv[k]; }
        }
        edge_tail(e0, g0, c0, y0);
        edge_tail(e1, g1, c1, y1);
      }
      if (i < cnt) {
        const int64_t e0 = __shfl_sync(0xffffffffu, my_e, i), s0 = __shfl_sync(0xffffffffu, my_s, i);
        float g0[V], a0[V], c0[V], y0[V];
        ld_row<D, true>(g0, a.G + e0 * D, lane);
        if (want_res) ld_row<D, true>(y0, a.y + e0 * D, lane);
        if constexpr (!GIM) ld_row<D, false>(a0, a.P + s0 * 4 * D, lane);
        ld_row<D, false>(c0, a.P + s0 * 4 * D + D, lane);
        if constexpr (!GIM) {
#pragma unroll
          for (int k = 0; k < V; ++k) g0[k] += a0[k] + bv[k];
        }
        edge_tail(e0, g0, c0, y0);
      }
    }
    // ---- node finalize: h = Sh/(S+eps); x' = src_update(x) + h; norm; silu; residual -----------
    float dv[V], xp[V], h[V];
    ld_row<D, false>(dv, a.P + v * 4 * D + 3 * D, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) { h[k] = accSh[k] / (accS[k] + a.gate_eps); xp[k] = dv[k] + h[k]; }
    if (train) {
      st_row<D, false>(a.XP + v * D, xp, lane);
      st_row<D, false>(a.S + v * D, accS, lane);
      st_row<D, false>(a.H + v * D, h, lane);
    }
    if (a.norm_nodes == ALIGNN_NORM_STATS) {
      smem_row_add<D>(st + 2 * D, xp, lane);
#pragma unroll
      for (int k = 0; k < V; ++k) xp[k] *= xp[k];
      smem_row_add<D>(st + 3 * D, xp, lane);
    } else {
      float o[V], nw[V], nb[V];
      ld_srow<D>(nw, vec, lane);
      ld_srow<D>(nb, vec + D, lane);
      if (a.norm_nodes == ALIGNN_NORM_LAYER) {
        float mean, rstd;
        row_mean_rstd<D>(xp, a.ln_eps, mean, rstd);
#pragma unroll
        for (int k = 0; k < V; ++k) o[k] = silu_((xp[k] - mean) * rstd * nw[k] + nb[k]);
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k) o[k] = silu_(xp[k] * nw[k] + nb[k]);
      }
      if (a.residual) {
        float xr[V];
        ld_row<D, false>(xr, a.x + v * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) o[k] += xr[k];
      }
      st_row<D, false>(a.x_out + v * D, o, lane);
    }
  }
  if (stats) {   // fixed-order sum over the block's warps -> one partial row
    __syncthreads();
    float* out_row = a.partials + (int64_t)blockIdx.x * 4 * D;
    for (int i = threadIdx.x; i < 4 * D; i += blockDim.x) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kWarpsPerBlock; ++w) t += sacc[w * 4 * D + i];
      out_row[i] = t;
    }
  }
}

// ---- forward, second pass, with the edge rows staged through shared memory -------------------------------------------
// Same arithmetic, same per-row operation order and therefore the same bits as egc_forward_kernel<D, true>; what changes
// is how the rows arrive.  Every warp owns a ring of kRing slots in shared memory; a slot holds the three rows of one
// edge (gate m, gathered Bh[src], residual y) and is filled by cp.async (LDGSTS: global -> shared without passing through
// registers), each lane copying exactly the 16-byte pieces it will read back, so completion needs no barrier -- only
// cp.async.wait_group.  The warp issues the copies of edge i + kRing - 1 before it does the gate / norm / SiLU math of
// edge i: kRing - 1 edges (9 KB at d = 256) stay in flight per warp WHILE it computes, where the register-staged kernel
// has nothing in flight during the math of its two edges.  Slot headers (edge id, node, first / last flags) are
// warp-uniform registers; the loop is unrolled over the ring so that they are indexed statically.
constexpr int kRing = 4;

template <int BYTES>
__device__ __forceinline__ void cp_async_piece(float* sdst, const float* gsrc) {
  const uint32_t sa = (uint32_t)__cvta_generic_to_shared(sdst);
  if constexpr (BYTES == 16) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gsrc) : "memory");
  else if constexpr (BYTES == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sa), "l"(gsrc) : "memory");
  else asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(gsrc) : "memory");
}
template <int D>
__device__ __forceinline__ void cp_async_row(float* srow, const float* __restrict__ grow, int lane) {
  using C = RowCfg<D>;
#pragma unroll
  for (int c = 0; c < C::CH; ++c) cp_async_piece<C::W * 4>(srow + c * 32 * C::W + lane * C::W, grow + c * 32 * C::W + lane * C::W);
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int D>
__global__ void __launch_bounds__(kThreads, 2)
egc_forward_ring_kernel(alignn_b200_egc_fwd_args a) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  constexpr int SLOT = 3 * D;
  constexpr int F_FIRST = 1, F_LAST = 2, F_EMPTY = 4, F_DONE = 8;
  extern __shared__ __align__(16) float dyn_smem[];
  float* vec = dyn_smem;                                            // [4][D]: n_w, n_b, e_w, e_b
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* ring = dyn_smem + 4 * D + wib * kRing * SLOT;              // this warp's slots
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + wib;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  const bool train = a.XP != nullptr;
  const bool edge_out = a.y_out != nullptr;
  const bool want_res = a.residual && edge_out;
  const bool nstats = a.norm_nodes == ALIGNN_NORM_STATS;
  {
    const float* srcs[4] = {a.n_w, a.n_b, a.e_w, a.e_b};
#pragma unroll
    for (int q = 0; q < 4; ++q)
      for (int i = threadIdx.x; i < D; i += blockDim.x) vec[q * D + i] = srcs[q] ? srcs[q][i] : 0.f;
  }
  __syncthreads();

  // ---- producer cursor: (node, position in its in-edge list), indices of the current 32-edge chunk ----
  // The index chain in_ptr[v] -> in_eid -> src is two or three dependent loads; it is requested one and two nodes ahead
  // (n1*, n2*) so that moving to the next node never waits for it.
  int64_t pv = warp0;
  bool pdone = pv >= a.Nn;
  int pfirst = 0, ppos = 0, pend = 0, cbase = 0, ccnt = 0, my_e = 0, my_s = 0;
  int n1first = 0, n1end = 0, n1_e = 0, n1_s = 0, n2first = 0, n2end = 0;
  auto load_ptr = [&](int64_t v, int& f, int& e) {
    if (v < a.Nn) { f = a.in_ptr[v]; e = a.in_ptr[v + 1]; } else { f = 0; e = 0; }
  };
  auto load_idx = [&](int first, int end, int& e_out, int& s_out) {
    if (lane < min(32, end - first)) {
      e_out = a.in_eid ? a.in_eid[first + lane] : first + lane;
      s_out = a.src[e_out];
    }
  };
  load_ptr(pv, pfirst, pend);
  ppos = cbase = pfirst;
  ccnt = min(32, pend - pfirst);
  load_idx(pfirst, pend, my_e, my_s);
  load_ptr(pv + nwarps, n1first, n1end);
  load_idx(n1first, n1end, n1_e, n1_s);
  load_ptr(pv + 2 * nwarps, n2first, n2end);
  int64_t hv[kRing];
  int he[kRing], hf[kRing];

  auto next_node = [&]() {
    pv += nwarps;
    pdone = pv >= a.Nn;
    pfirst = ppos = cbase = n1first; pend = n1end;
    ccnt = min(32, pend - pfirst);
    my_e = n1_e; my_s = n1_s;
    n1first = n2first; n1end = n2end;
    load_idx(n1first, n1end, n1_e, n1_s);
    load_ptr(pv + 2 * nwarps, n2first, n2end);
  };
  auto produce = [&](float* slot, int64_t& sv, int& se, int& sf) {
    if (pdone) { sf = F_DONE; cp_async_commit(); return; }
    sv = pv;
    if (pend == pfirst) {                                           // a node without in-edges still gets its tail
      se = -1; sf = F_FIRST | F_LAST | F_EMPTY;
      cp_async_commit();
      next_node();
      return;
    }
    if (ppos >= cbase + ccnt) {
      cbase = ppos;
      ccnt = min(32, pend - ppos);
      if (lane < ccnt) {
        my_e = a.in_eid ? a.in_eid[cbase + lane] : cbase + lane;
        my_s = a.src[my_e];
      }
    }
    const int e = __shfl_sync(0xffffffffu, my_e, ppos - cbase), sidx = __shfl_sync(0xffffffffu, my_s, ppos - cbase);
    cp_async_row<D>(slot, a.G + (int64_t)e * D, lane);
    cp_async_row<D>(slot + D, a.P + (int64_t)sidx * 4 * D + D, lane);
    if (want_res) cp_async_row<D>(slot + 2 * D, a.y + (int64_t)e * D, lane);
    cp_async_commit();
    se = e;
    sf = (ppos == pfirst ? F_FIRST : 0) | (ppos + 1 == pend ? F_LAST : 0);
    if (++ppos == pend) next_node();
  };

#pragma unroll
  for (int s = 0; s < kRing - 1; ++s) produce(ring + s * SLOT, hv[s], he[s], hf[s]);
  hf[kRing - 1] = F_DONE;

  float accS[V], accSh[V], dv[V], xr[V], nst[2][V];
#pragma unroll
  for (int k = 0; k < V; ++k) { accS[k] = 0.f; accSh[k] = 0.f; dv[k] = 0.f; xr[k] = 0.f; nst[0][k] = 0.f; nst[1][k] = 0.f; }

  bool running = true;
  while (running) {
#pragma unroll
    for (int s = 0; s < kRing; ++s) {
      // refill the slot consumed one step ago (slot s-1), then wait for slot s: kRing-1 groups may stay pending
      {
        const int t = (s + kRing - 1) % kRing;
        produce(ring + t * SLOT, hv[t], he[t], hf[t]);
      }
      cp_async_wait<kRing - 1>();
      const int f = hf[s];
      if (f & F_DONE) { running = false; break; }
      const int64_t v = hv[s];
      float* slot = ring + s * SLOT;
      if (f & F_FIRST) {
#pragma unroll
        for (int k = 0; k < V; ++k) { accS[k] = 0.f; accSh[k] = 0.f; }
        ld_row<D, false>(dv, a.P + v * 4 * D + 3 * D, lane);        // needed at the node's tail: requested a segment early
        if (!nstats && a.residual) ld_row<D, false>(xr, a.x + v * D, lane);
      }
      if (!(f & F_EMPTY)) {
        const int64_t e = he[s];
        float m[V], cv[V];
        ld_srow<D>(m, slot, lane);
        ld_srow<D>(cv, slot + D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float sg = sigmoidf_(m[k]);
          accS[k] += sg;
          accSh[k] += cv[k] * sg;
        }
        if (edge_out) {
          float o[V], ew[V], eb[V];
          ld_srow<D>(ew, vec + 2 * D, lane);
          ld_srow<D>(eb, vec + 3 * D, lane);
          if (a.norm_edges == ALIGNN_NORM_LAYER) {
            float mean, rstd;
            row_mean_rstd<D>(m, a.ln_eps, mean, rstd);
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] = silu_((m[k] - mean) * rstd * ew[k] + eb[k]);
          } else {
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] = silu_(m[k] * ew[k] + eb[k]);
          }
          if (a.residual) {
            float yr[V];
            ld_srow<D>(yr, slot + 2 * D, lane);
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] += yr[k];
          }
          st_row<D, true>(a.y_out + e * D, o, lane);
        }
      }
      if (f & F_LAST) {
        // ---- node tail: h = Sh/(S+eps); x' = src_update(x) + h; norm; silu; residual ----
        float xp[V], h[V];
#pragma unroll
        for (int k = 0; k < V; ++k) { h[k] = accSh[k] / (accS[k] + a.gate_eps); xp[k] = dv[k] + h[k]; }
        if (train) {
          st_row<D, false>(a.XP + v * D, xp, lane);
          st_row<D, false>(a.S + v * D, accS, lane);
          st_row<D, false>(a.H + v * D, h, lane);
        }
        if (nstats) {
#pragma unroll
          for (int k = 0; k < V; ++k) { nst[0][k] += xp[k]; nst[1][k] += xp[k] * xp[k]; }
        } else {
          float o[V], nw[V], nb[V];
          ld_srow<D>(nw, vec, lane);
          ld_srow<D>(nb, vec + D, lane);
          if (a.norm_nodes == ALIGNN_NORM_LAYER) {
            float mean, rstd;
            row_mean_rstd<D>(xp, a.ln_eps, mean, rstd);
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] = silu_((xp[k] - mean) * rstd * nw[k] + nb[k]);
          } else {
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] = silu_(xp[k] * nw[k] + nb[k]);
          }
          if (a.residual) {
#pragma unroll
            for (int k = 0; k < V; ++k) o[k] += xr[k];
          }
          st_row<D, false>(a.x_out + v * D, o, lane);
        }
      }
    }
  }
  cp_async_wait<0>();
  if (a.partials) {   // {0, 0, sum x', sum x'^2}: the edge statistics came from the gather GEMM
    __syncthreads();
    float* out_row = a.partials + (int64_t)blockIdx.x * 4 * D;
    for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) out_row[i] = 0.f;
    block_reduce_to_partials<D, 2>(nst, out_row + 2 * D, dyn_smem + 4 * D);
  }
}

// =============================================================================================
// Backward, destination-keyed pass: node-norm backward, per-edge gate backward, edge-norm
// backward, GM = dL/dm, GP[:, 2d:3d] = sum over in-edges (dL/d e_dst), GP[:, 3d:4d] = dL/dx'.
// partials row: {sum gu_e*xhat_e, sum gu_e, sum gu_n*xhat_n, sum gu_n, sum gD, sum gB}
// =============================================================================================
// vecs: 6 per-channel vectors in shared memory at stride D: {w, b, mean, rstd, c1, c2} (meaning per mode in
// include/alignn_b200.h).  They are re-read from shared memory at every use instead of living in registers.
template <int D, int mode>
__device__ __forceinline__ void norm_backward_row(const float (&r)[RowCfg<D>::VPL], const float (&go)[RowCfg<D>::VPL],
                                                  float ln_eps, const float* __restrict__ vecs,
                                                  float (&gr)[RowCfg<D>::VPL], float* __restrict__ acc_gw,
                                                  float* __restrict__ acc_gb, int lane) {
  constexpr int V = RowCfg<D>::VPL;
  float w[V], b[V];
  ld_srow<D>(w, vecs, lane);
  ld_srow<D>(b, vecs + D, lane);
  if constexpr (mode == ALIGNN_NORM_LAYER) {
    float mean, rstd;
    row_mean_rstd<D>(r, ln_eps, mean, rstd);
    float xh[V], gxh[V], t1[V], sa = 0.f, sb = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      xh[k] = (r[k] - mean) * rstd;
      const float gu = go[k] * dsilu_(xh[k] * w[k] + b[k]);
      t1[k] = gu;
      gxh[k] = gu * w[k];
      sa += gxh[k];
      sb += gxh[k] * xh[k];
    }
    smem_row_add<D>(acc_gb, t1, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) t1[k] *= xh[k];
    smem_row_add<D>(acc_gw, t1, lane);
    sa = warp_sum(sa) * (1.f / D);
    sb = warp_sum(sb) * (1.f / D);
#pragma unroll
    for (int k = 0; k < V; ++k) gr[k] = rstd * (gxh[k] - sa - xh[k] * sb);
  } else {
    // w = scale, b = shift; xhat = (r - mean_c) * rstd_c
    float mu[V], rs[V], t0[V], t1[V];
    ld_srow<D>(mu, vecs + 2 * D, lane);
    ld_srow<D>(rs, vecs + 3 * D, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float gu = go[k] * dsilu_(r[k] * w[k] + b[k]);
      const float xh = (r[k] - mu[k]) * rs[k];
      t0[k] = gu * xh;
      t1[k] = gu;
      gr[k] = w[k] * gu;
      mu[k] = xh;
    }
    smem_row_add<D>(acc_gw, t0, lane);
    smem_row_add<D>(acc_gb, t1, lane);
    if constexpr (mode == ALIGNN_NORM_STATS) {
      float c1[V], c2[V];
      ld_srow<D>(c1, vecs + 4 * D, lane);
      ld_srow<D>(c2, vecs + 5 * D, lane);
#pragma unroll
      for (int k = 0; k < V; ++k) gr[k] -= w[k] * (c1[k] + mu[k] * c2[k]);
    }
  }
}

// Node side of the destination-keyed backward for node v: node-norm backward, GP[v, 3d:4d] = dL/dx', GSh[v] = dL/dSh,
// and {dL/dSh, dL/dS} of v parked in the warp's shared segment `wseg` [2][D] for its in-edge loop (each lane re-reads
// only what it wrote).  Shared by egc_backward_dst_kernel and egc_backward_line_kernel so both produce the same bits.
template <int D, int NORM>
__device__ __forceinline__ void bwd_node_side(const alignn_b200_egc_bwd_args& a, int64_t v, const float* __restrict__ nvec,
                                              float* __restrict__ acc, float* __restrict__ wseg, int lane) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  float gsh[V], gs[V];
  float xp[V], go[V], gxp[V], sv[V], hv[V];
  ld_row<D, false>(xp, a.XP + v * D, lane);
  ld_row<D, false>(go, a.gx_out + v * D, lane);
  norm_backward_row<D, NORM>(xp, go, a.ln_eps, nvec, gxp, acc + 2 * D, acc + 3 * D, lane);
  st_row<D, false>(a.GP + v * 4 * D + 3 * D, gxp, lane);
  ld_row<D, false>(sv, a.S + v * D, lane);
  ld_row<D, false>(hv, a.H + v * D, lane);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const float inv = 1.f / (sv[k] + a.gate_eps);
    gsh[k] = gxp[k] * inv;
    gs[k] = -gxp[k] * hv[k] * inv;
  }
  smem_row_add<D>(acc + 4 * D, gxp, lane);
  st_row<D, false>(a.GSh + v * D, gsh, lane);
#pragma unroll
  for (int c = 0; c < C::CH; ++c)
#pragma unroll
    for (int j = 0; j < C::W; ++j) {
      wseg[c * 32 * C::W + lane * C::W + j] = gsh[c * C::W + j];
      wseg[D + c * 32 * C::W + lane * C::W + j] = gs[c * C::W + j];
    }
  __syncwarp();
}

// One in-edge of the destination whose segment is parked in `wseg`: edge-norm backward (when the edge output is used)
// plus the gate term, gm = dL/dm; accB += gm.  m / go: the edge's pre-activation and output-gradient rows, cv: Bh[src].
template <int D, int NORM>
__device__ __forceinline__ void bwd_edge_gm(const alignn_b200_egc_bwd_args& a, const float (&m)[RowCfg<D>::VPL],
                                           const float (&go)[RowCfg<D>::VPL], const float (&cv)[RowCfg<D>::VPL],
                                           const float* __restrict__ evec, float* __restrict__ acc,
                                           const float* __restrict__ wseg, float (&gm)[RowCfg<D>::VPL],
                                           float (&accB)[RowCfg<D>::VPL], int lane) {
  constexpr int V = RowCfg<D>::VPL;
  if (a.gy_out) {
    norm_backward_row<D, NORM>(m, go, a.ln_eps, evec, gm, acc, acc + D, lane);
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) gm[k] = 0.f;
  }
  float gsh[V], gs[V];
  ld_srow<D>(gsh, wseg, lane);
  ld_srow<D>(gs, wseg + D, lane);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const float sg = sigmoidf_(m[k]);
    gm[k] += (gsh[k] * cv[k] + gs[k]) * sg * (1.f - sg);
    accB[k] += gm[k];
  }
}

template <int D, int NORM>   // NORM: the norm mode of both bn_nodes and bn_edges (compile-time: unused vectors vanish)
__global__ void __launch_bounds__(kThreads)
egc_backward_dst_kernel(alignn_b200_egc_bwd_args a) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  // per-warp partial sums live in shared memory (6 rows of D per warp): keeping them in registers cost 48
  // registers per thread and halved the resident warps of this HBM-latency-bound kernel
  extern __shared__ __align__(16) float dyn_smem[];
  float* sacc = dyn_smem;                                  // [kWarpsPerBlock][6][D]
  float* nvec = dyn_smem + kWarpsPerBlock * 6 * D;         // node norm vectors  [6][D]
  float* sseg = nvec + 12 * D;                             // [kWarpsPerBlock][2][D]: dL/dSh, dL/dS of the warp's segment
  float* evec = nvec + 6 * D;                              // edge norm vectors  [6][D]
  {
    const float* srcs[12] = {a.n_w, a.n_b, a.n_mean, a.n_rstd, a.n_c1, a.n_c2, a.e_w, a.e_b, a.e_mean, a.e_rstd, a.e_c1, a.e_c2};
#pragma unroll
    for (int q = 0; q < 12; ++q)
      for (int i = threadIdx.x; i < D; i += blockDim.x) nvec[q * D + i] = srcs[q] ? srcs[q][i] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + wib;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float* acc = sacc + wib * 6 * D;     // acc + q*D = row q of this warp
  for (int i = lane; i < 6 * D; i += 32) acc[i] = 0.f;
  __syncwarp();

  float* wseg = sseg + wib * 2 * D;
  for (int64_t v = warp0; v < a.Nn; v += nwarps) {
    bwd_node_side<D, NORM>(a, v, nvec, acc, wseg, lane);
    float accB[V];
#pragma unroll
    for (int k = 0; k < V; ++k) accB[k] = 0.f;
    const int p0 = a.in_ptr[v], p1 = a.in_ptr[v + 1];
    for (int base = p0; base < p1; base += 32) {
      const int cnt = min(32, p1 - base);
      int my_e = 0, my_s = 0;
      if (lane < cnt) {
        my_e = a.in_eid ? a.in_eid[base + lane] : base + lane;
        my_s = a.src[my_e];
      }
      // software pipeline: the M / gy_out rows of edge i+1 are requested before edge i is processed
      float m[V], go[V];
      if (cnt > 0) {
        const int64_t e = __shfl_sync(0xffffffffu, my_e, 0);
        ld_row<D, true>(m, a.M + e * D, lane);
        if (a.gy_out) ld_row<D, true>(go, a.gy_out + e * D, lane);
      }
      for (int i = 0; i < cnt; ++i) {
        const int64_t e = __shfl_sync(0xffffffffu, my_e, i);
        const int64_t s = __shfl_sync(0xffffffffu, my_s, i);
        float cv[V], gm[V], mn[V], gon[V];
        ld_row<D, false>(cv, a.P + s * 4 * D + D, lane);
        const bool more = (i + 1 < cnt);
        if (more) {
          const int64_t en = __shfl_sync(0xffffffffu, my_e, i + 1);
          ld_row<D, true>(mn, a.M + en * D, lane);
          if (a.gy_out) ld_row<D, true>(gon, a.gy_out + en * D, lane);
        }
        bwd_edge_gm<D, NORM>(a, m, go, cv, evec, acc, wseg, gm, accB, lane);
        st_row<D, false>(a.GM + e * D, gm, lane);   // re-read by the src-keyed pass and the GEMMs
        if (more) {
#pragma unroll
          for (int k = 0; k < V; ++k) { m[k] = mn[k]; go[k] = gon[k]; }
        }
      }
    }
    st_row<D, false>(a.GP + v * 4 * D + 2 * D, accB, lane);
    smem_row_add<D>(acc + 5 * D, accB, lane);
  }
  __syncthreads();
  if (a.partials) {   // fixed-order sum over the block's warps -> one partial row
    float* out_row = a.partials + (int64_t)blockIdx.x * 6 * D;
    for (int i = threadIdx.x; i < 6 * D; i += blockDim.x) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kWarpsPerBlock; ++w) t += sacc[w * 6 * D + i];
      out_row[i] = t;
    }
  }
}

// =============================================================================================
// Backward, source-keyed pass (out-CSR): GP[:, 0:d] = sum over out-edges of GM (dL/d e_src),
// GP[:, d:2d] = sum over out-edges of GSh[dst] * sigma (dL/d Bh).
// partials row: {sum gA, sum gC}
// =============================================================================================
template <int D>
__global__ void __launch_bounds__(kThreads)
egc_backward_src_kernel(alignn_b200_egc_bwd_args a, float* __restrict__ partials_src, int partial_rows_total) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  __shared__ float red[kWarpsPerBlock * D];
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float acc[2][V];
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < V; ++i) acc[q][i] = 0.f;

  for (int64_t u = warp0; u < a.Nn; u += nwarps) {
    float accA[V], accC[V];
#pragma unroll
    for (int k = 0; k < V; ++k) { accA[k] = 0.f; accC[k] = 0.f; }
    const int p0 = a.out_ptr[u], p1 = a.out_ptr[u + 1];
    for (int base = p0; base < p1; base += 32) {
      const int cnt = min(32, p1 - base);
      int my_e = 0, my_t = 0;
      if (lane < cnt) {
        my_e = a.out_eid[base + lane];
        my_t = a.dst[my_e];
      }
      int i = 0;
      for (; i + 1 < cnt; i += 2) {   // two edges (six row loads) in flight per warp
        const int64_t e0 = __shfl_sync(0xffffffffu, my_e, i), t0 = __shfl_sync(0xffffffffu, my_t, i);
        const int64_t e1 = __shfl_sync(0xffffffffu, my_e, i + 1), t1 = __shfl_sync(0xffffffffu, my_t, i + 1);
        float gm0[V], m0[V], gs0[V], gm1[V], m1[V], gs1[V];
        ld_row<D, false>(gm0, a.GM + e0 * D, lane);
        ld_row<D, false>(gm1, a.GM + e1 * D, lane);
        ld_row<D, true>(m0, a.M + e0 * D, lane);
        ld_row<D, true>(m1, a.M + e1 * D, lane);
        ld_row<D, false>(gs0, a.GSh + t0 * D, lane);
        ld_row<D, false>(gs1, a.GSh + t1 * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) { accA[k] += gm0[k]; accC[k] = fmaf(gs0[k], sigmoidf_(m0[k]), accC[k]); }
#pragma unroll
        for (int k = 0; k < V; ++k) { accA[k] += gm1[k]; accC[k] = fmaf(gs1[k], sigmoidf_(m1[k]), accC[k]); }
      }
      if (i < cnt) {
        const int64_t e = __shfl_sync(0xffffffffu, my_e, i);
        const int64_t t = __shfl_sync(0xffffffffu, my_t, i);
        float gm[V], m[V], gsh[V];
        ld_row<D, false>(gm, a.GM + e * D, lane);
        ld_row<D, true>(m, a.M + e * D, lane);
        ld_row<D, false>(gsh, a.GSh + t * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          accA[k] += gm[k];
          accC[k] = fmaf(gsh[k], sigmoidf_(m[k]), accC[k]);
        }
      }
    }
    st_row<D, false>(a.GP + u * 4 * D, accA, lane);
    st_row<D, false>(a.GP + u * 4 * D + D, accC, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) { acc[0][k] += accA[k]; acc[1][k] += accC[k]; }
  }
  if (partials_src) {
    block_reduce_to_partials<D, 2>(acc, partials_src + (int64_t)blockIdx.x * 2 * D, red);
    const int extra = blockIdx.x + gridDim.x;              // rows [gridDim.x, partial_rows_total) belong to no block
    if (extra < partial_rows_total)
      for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) partials_src[(int64_t)extra * 2 * D + i] = 0.f;
  }
}

// =============================================================================================
// Backward on a line graph, both passes in one: one CTA per atom of the parent graph g.
// L(g) has an edge (i -> j) for every pair of bonds with dst(i) == src(j) == a, i != j, emitted destination-major with
// the sources of each j in the order of a's in-list.  So the L(g) edges at atom a are one complete bipartite block,
// sources in(a) x destinations out(a) (less the self pair of a self-loop bond), and the CTA that owns a holds ALL the
// in-edges of its destinations and ALL the out-edges of its sources: it produces GP[j, 2d:4d], GSh[j] and GM of the
// block exactly as egc_backward_dst_kernel does, and GP[i, 0:2d] exactly as egc_backward_src_kernel does, without
// reading GM / M back.
//   Warps own destinations j, kLineWarps at a time, in out-list (= ascending id) order.  The sources i are processed in
// rounds, all warps on the same source: the warp does the destination-side work of edge (i, j) and stages gm and
// sigma(m) of that edge in shared memory; after one barrier the CTA adds the staged rows over the warps in ascending j
// -- the same sequential order and the same fmaf as the source-keyed kernel -- onto the running sums GP[i, 0:2d].  When
// out(a) takes more than one chunk of warps, the running sums go back to GP[i] between chunks (only this CTA owns them).
// Edge ids: (in(a)[t], j) is L(g) edge in_ptr_lg[j] + t, minus one after the excluded self pair.
// partials: [6][D] per CTA as the destination-keyed pass; partials_src: [2][D] per CTA as the source-keyed pass.
// =============================================================================================
// 12 warps, one CTA per SM (registers): a 12 x 12 block (k = 12 neighbours) is one chunk, so the running sums never go
// back through GP and the atom's index chain and node side are paid once.  Measured faster than 6 warps x 2 CTAs and
// 4 warps x 3 CTAs per SM on the headline L(g); an L2 prefetch of the warp's next edge rows did not help.
constexpr int kLineWarps = 12;
constexpr int kLineThreads = kLineWarps * 32;

template <int D>
constexpr size_t line_bwd_smem_floats() {
  // sacc [W][6][D], nvec [12][D], wseg [W][2][D], stage [2][W][2][D], ssrc [2][D]
  return (size_t)(kLineWarps * 6 + 12 + kLineWarps * 2 + 2 * kLineWarps * 2 + 2) * D;
}

template <int D, int NORM>
__global__ void __launch_bounds__(kLineThreads, 1)
egc_backward_line_kernel(alignn_b200_egc_bwd_args a, int partial_rows_total) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  constexpr int W = kLineWarps;
  extern __shared__ __align__(16) float dyn_smem[];
  float* sacc = dyn_smem;                        // [W][6][D]: per-warp partial sums of the destination side
  float* nvec = sacc + W * 6 * D;                // node norm vectors [6][D], then edge norm vectors [6][D]
  float* evec = nvec + 6 * D;
  float* sseg = nvec + 12 * D;                   // [W][2][D]: dL/dSh, dL/dS of the warp's destination
  float* stage = sseg + W * 2 * D;               // [2][W][2][D]: gm, sigma(m) of the round's edge, double-buffered
  float* ssrc = stage + 2 * W * 2 * D;           // [2][D]: this CTA's sums of GP[:, 0:2d]
  __shared__ int sself[W];                       // per warp: round of the excluded self pair, or -1
  {
    const float* srcs[12] = {a.n_w, a.n_b, a.n_mean, a.n_rstd, a.n_c1, a.n_c2, a.e_w, a.e_b, a.e_mean, a.e_rstd, a.e_c1, a.e_c2};
#pragma unroll
    for (int q = 0; q < 12; ++q)
      for (int i = threadIdx.x; i < D; i += blockDim.x) nvec[q * D + i] = srcs[q] ? srcs[q][i] : 0.f;
  }
  for (int i = threadIdx.x; i < W * 6 * D; i += blockDim.x) sacc[i] = 0.f;
  for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) ssrc[i] = 0.f;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* acc = sacc + wib * 6 * D;
  float* wseg = sseg + wib * 2 * D;
  int round = 0;                                 // rounds run by this CTA so far: picks the stage buffer

  for (int64_t at = blockIdx.x; at < a.parent_Nn; at += gridDim.x) {
    const int ip0 = a.parent_in_ptr[at], kin = a.parent_in_ptr[at + 1] - ip0;
    const int op0 = a.parent_out_ptr[at], kout = a.parent_out_ptr[at + 1] - op0;
    if (kout == 0) {                             // sources without out-edges: GP[i, 0:2d] = 0
      for (int t = 0; t < kin; ++t) {
        const int64_t i = a.parent_in_eid[ip0 + t];
        for (int q = threadIdx.x; q < 2 * D; q += blockDim.x) a.GP[i * 4 * D + q] = 0.f;
      }
      continue;
    }
    for (int c0 = 0; c0 < kout; c0 += W) {
      const int nd = min(W, kout - c0);
      const bool last_chunk = c0 + W >= kout;
      const bool active = wib < nd;
      __syncthreads();                           // the previous chunk's round sums have read wseg / sself
      int64_t j = 0, ebase = 0;
      int selfpos = -1;
      if (active) {
        j = a.parent_out_eid[op0 + c0 + wib];
        ebase = a.in_ptr[j];
        if (a.in_ptr[j + 1] - ebase != kin) {    // j is a self-loop bond: find it in a's in-list
          for (int t0 = 0; t0 < kin; t0 += 32) {
            const bool hit = t0 + lane < kin && a.parent_in_eid[ip0 + t0 + lane] == (int)j;
            const unsigned bal = __ballot_sync(0xffffffffu, hit);
            if (bal) { selfpos = t0 + __ffs(bal) - 1; break; }
          }
        }
        if (lane == 0) sself[wib] = selfpos;
        bwd_node_side<D, NORM>(a, j, nvec, acc, wseg, lane);
      }
      auto edge_of = [&](int t) { return ebase + t - ((selfpos >= 0 && t > selfpos) ? 1 : 0); };
      // the first 32 sources, one per lane: every warp shuffles the round's source from its own copy (t < kin)
      const int my_i = lane < kin ? a.parent_in_eid[ip0 + lane] : 0;
      auto source = [&](int t) { return t < 32 ? __shfl_sync(0xffffffffu, my_i, t) : a.parent_in_eid[ip0 + t]; };
      float accB[V], m[V], go[V], cv[V];
#pragma unroll
      for (int k = 0; k < V; ++k) accB[k] = 0.f;
      // the warp's next edge: its M / gy_out rows and its source's Bh row are requested one round ahead
      int tn = selfpos == 0 ? 1 : 0;
      {
        const int64_t in_ = kin > 0 ? source(min(tn, kin - 1)) : 0;
        if (active && tn < kin) {
          const int64_t e = edge_of(tn);
          ld_row<D, true>(m, a.M + e * D, lane);
          if (a.gy_out) ld_row<D, true>(go, a.gy_out + e * D, lane);
          ld_row<D, false>(cv, a.P + in_ * 4 * D + D, lane);
        }
      }
      // this thread's 4 channels of the round sums (2d / 4 <= kLineThreads: at most one float4 per thread)
      const int q = threadIdx.x * 4;
      static_assert(2 * D <= 4 * kLineThreads, "one float4 of GP[i, 0:2d] per thread");
      for (int t = 0; t < kin; ++t, ++round) {
        const int64_t i = source(t);
        float* stg = stage + (round & 1) * W * 2 * D;
        // running sum of GP[i, q:q+4] from the previous chunks (written by this thread), requested before the edge work
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 > 0 && q < 2 * D) r = *reinterpret_cast<const float4*>(a.GP + i * 4 * D + q);
        const int tnext = (t + 1 == selfpos) ? t + 2 : t + 1;
        const int64_t inext = source(min(tnext, kin - 1));
        if (active && t != selfpos) {
          const int64_t e = edge_of(t);
          float gm[V], mn[V], gon[V], cvn[V];
          if (tnext < kin) {
            const int64_t en = edge_of(tnext);
            ld_row<D, true>(mn, a.M + en * D, lane);
            if (a.gy_out) ld_row<D, true>(gon, a.gy_out + en * D, lane);
            ld_row<D, false>(cvn, a.P + inext * 4 * D + D, lane);
          }
          bwd_edge_gm<D, NORM>(a, m, go, cv, evec, acc, wseg, gm, accB, lane);
          st_row<D, false>(a.GM + e * D, gm, lane);
          float sg[V];
#pragma unroll
          for (int k = 0; k < V; ++k) sg[k] = sigmoidf_(m[k]);
#pragma unroll
          for (int c = 0; c < C::CH; ++c)
#pragma unroll
            for (int u = 0; u < C::W; ++u) {
              stg[wib * 2 * D + c * 32 * C::W + lane * C::W + u] = gm[c * C::W + u];
              stg[wib * 2 * D + D + c * 32 * C::W + lane * C::W + u] = sg[c * C::W + u];
            }
          if (tnext < kin) {
#pragma unroll
            for (int k = 0; k < V; ++k) { m[k] = mn[k]; go[k] = gon[k]; cv[k] = cvn[k]; }
          }
        }
        __syncthreads();
        // GP[i, 0:2d] += this round's edges, warps (= destinations) in ascending order
        if (q < 2 * D) {
          if (q < D) {                           // dL/d e_src = sum GM
            for (int w = 0; w < nd; ++w) {
              if (t == sself[w]) continue;
              const float4 g = *reinterpret_cast<const float4*>(stg + w * 2 * D + q);
              r.x += g.x; r.y += g.y; r.z += g.z; r.w += g.w;
            }
          } else {                               // dL/d Bh = sum GSh[j] * sigma(m)
            for (int w = 0; w < nd; ++w) {
              if (t == sself[w]) continue;
              const float4 g = *reinterpret_cast<const float4*>(sseg + w * 2 * D + (q - D));
              const float4 sg = *reinterpret_cast<const float4*>(stg + w * 2 * D + q);
              r.x = fmaf(g.x, sg.x, r.x); r.y = fmaf(g.y, sg.y, r.y); r.z = fmaf(g.z, sg.z, r.z); r.w = fmaf(g.w, sg.w, r.w);
            }
          }
          *reinterpret_cast<float4*>(a.GP + i * 4 * D + q) = r;
          if (last_chunk) {
            float4* s4 = reinterpret_cast<float4*>(ssrc + q);
            float4 u = *s4;
            u.x += r.x; u.y += r.y; u.z += r.z; u.w += r.w;
            *s4 = u;
          }
        }
      }
      if (active) {
        st_row<D, false>(a.GP + j * 4 * D + 2 * D, accB, lane);
        smem_row_add<D>(acc + 5 * D, accB, lane);
      }
    }
  }
  __syncthreads();
  if (a.partials) {                              // fixed-order sum over the CTA's warps -> one partial row
    float* out_row = a.partials + (int64_t)blockIdx.x * 6 * D;
    for (int i = threadIdx.x; i < 6 * D; i += blockDim.x) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < W; ++w) t += sacc[w * 6 * D + i];
      out_row[i] = t;
    }
  }
  if (a.partials_src)
    for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) a.partials_src[(int64_t)blockIdx.x * 2 * D + i] = ssrc[i];
  // rows [gridDim.x, partial_rows_total) belong to no CTA
  for (int64_t r = blockIdx.x + gridDim.x; r < partial_rows_total; r += gridDim.x) {
    if (a.partials)
      for (int i = threadIdx.x; i < 6 * D; i += blockDim.x) a.partials[r * 6 * D + i] = 0.f;
    if (a.partials_src)
      for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) a.partials_src[r * 2 * D + i] = 0.f;
  }
}

// =============================================================================================
// BatchNorm train-mode helpers
// =============================================================================================
// 32 channels per block x 32 row lanes; fp64 accumulation over the per-block partial rows, fixed order
__global__ void __launch_bounds__(1024)
bn_finalize_kernel(const float* __restrict__ partials, int rows, int stride, int which, double count,
                   int d, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                   float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                   float* mean_out, float* rstd_out) {
  __shared__ double ss[32][33], sq[32][33];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double s = 0.0, q = 0.0;
  if (c < d) {
    const float* p = partials + (size_t)which * 2 * d + c;
    for (int r = rl; r < rows; r += 32) {
      s += (double)p[(size_t)r * stride];
      q += (double)p[(size_t)r * stride + d];
    }
  }
  ss[rl][cl] = s; sq[rl][cl] = q;
  __syncthreads();
  if (rl != 0 || c >= d) return;
#pragma unroll
  for (int k = 1; k < 32; ++k) { s += ss[k][cl]; q += sq[k][cl]; }
  const double mean = s / count;
  double var = q / count - mean * mean;
  if (var < 0.0) var = 0.0;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  scale[c] = g * rstd;
  shift[c] = b - (float)mean * g * rstd;
  mean_out[c] = (float)mean;
  rstd_out[c] = rstd;
  if (running_mean) {
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

template <int D>
__global__ void __launch_bounds__(kThreads)
affine_silu_residual_kernel(const float* __restrict__ R, const float* __restrict__ res, const float* __restrict__ scale,
                            const float* __restrict__ shift, float* __restrict__ out, int64_t n) {
  constexpr int V = RowCfg<D>::VPL;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float sc[V], sh[V];
  ld_vec<D>(sc, scale, lane); ld_vec<D>(sh, shift, lane);
  for (int64_t r = warp0; r < n; r += 2 * nwarps) {   // two rows in flight per warp
    const int64_t r2 = r + nwarps;
    const bool has2 = r2 < n;
    float v[V], v2[V], y[V], y2[V];
    ld_row<D, true>(v, R + r * D, lane);
    if (has2) ld_row<D, true>(v2, R + r2 * D, lane);
    if (res) {
      ld_row<D, true>(y, res + r * D, lane);
      if (has2) ld_row<D, true>(y2, res + r2 * D, lane);
    }
#pragma unroll
    for (int k = 0; k < V; ++k) v[k] = silu_(v[k] * sc[k] + sh[k]) + (res ? y[k] : 0.f);
    st_row<D, true>(out + r * D, v, lane);
    if (has2) {
#pragma unroll
      for (int k = 0; k < V; ++k) v2[k] = silu_(v2[k] * sc[k] + sh[k]) + (res ? y2[k] : 0.f);
      st_row<D, true>(out + r2 * D, v2, lane);
    }
  }
}

template <int D>
__global__ void __launch_bounds__(kThreads, 2)
bn_backward_reduce_kernel(const float* __restrict__ R, const float* __restrict__ g_out, const float* __restrict__ scale,
                          const float* __restrict__ shift, const float* __restrict__ mean, const float* __restrict__ rstd,
                          int64_t n, float* __restrict__ partials) {
  constexpr int V = RowCfg<D>::VPL;
  __shared__ float red[kWarpsPerBlock * D];
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float sc[V], sh[V], mu[V], rs[V], acc[2][V];
  ld_vec<D>(sc, scale, lane); ld_vec<D>(sh, shift, lane); ld_vec<D>(mu, mean, lane); ld_vec<D>(rs, rstd, lane);
#pragma unroll
  for (int k = 0; k < V; ++k) { acc[0][k] = 0.f; acc[1][k] = 0.f; }
  // four rows (eight row loads, 8 KB) in flight per warp: the kernel is latency-bound (stall long-scoreboard ~11 per
  // issue with two rows), and the rows are consumed in the same order as before, so the sums keep their bits
  for (int64_t r = warp0; r < n; r += 4 * nwarps) {
    float v[4][V], g[4][V];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t rj = r + j * nwarps;
      if (rj < n) {
        ld_row<D, true>(v[j], R + rj * D, lane);
        ld_row<D, true>(g[j], g_out + rj * D, lane);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (r + j * nwarps < n) {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float gu = g[j][k] * dsilu_(v[j][k] * sc[k] + sh[k]);
          acc[0][k] += gu;
          acc[1][k] += gu * (v[j][k] - mu[k]) * rs[k];
        }
      }
    }
  }
  block_reduce_to_partials<D, 2>(acc, partials + (int64_t)blockIdx.x * 2 * D, red);
}

// per-block partials {sum, sum of squares} per column of a tall [n, D] matrix: batch statistics of a
// Linear -> BatchNorm1d(train) -> SiLU embedding layer (alignn.py:170-184).  Row layout [2][D] = what bn_finalize reads.
template <int D>
__global__ void __launch_bounds__(kThreads)
rowstats_partials_kernel(const float* __restrict__ a, int64_t n, float* __restrict__ partials) {
  constexpr int V = RowCfg<D>::VPL;
  __shared__ float red[kWarpsPerBlock * D];
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float acc[2][V];
#pragma unroll
  for (int k = 0; k < V; ++k) { acc[0][k] = 0.f; acc[1][k] = 0.f; }
  for (int64_t r = warp0; r < n; r += nwarps) {
    float v[V];
    ld_row<D, false>(v, a + r * D, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) { acc[0][k] += v[k]; acc[1][k] += v[k] * v[k]; }
  }
  block_reduce_to_partials<D, 2>(acc, partials + (int64_t)blockIdx.x * 2 * D, red);
}

// BatchNorm1d(train) + SiLU backward, pass 2: gR = scale * (gu - c1 - xhat * c2), gu = g_out * silu'(R*scale+shift)
template <int D>
__global__ void __launch_bounds__(kThreads, 2)
bn_backward_apply_kernel(const float* __restrict__ R, const float* __restrict__ g_out, const float* __restrict__ scale,
                         const float* __restrict__ shift, const float* __restrict__ mean, const float* __restrict__ rstd,
                         const float* __restrict__ c1, const float* __restrict__ c2, int64_t n, float* __restrict__ gR) {
  constexpr int V = RowCfg<D>::VPL;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float sc[V], sh[V], mu[V], rs[V], k1[V], k2[V];
  ld_vec<D>(sc, scale, lane); ld_vec<D>(sh, shift, lane); ld_vec<D>(mu, mean, lane); ld_vec<D>(rs, rstd, lane);
  ld_vec<D>(k1, c1, lane); ld_vec<D>(k2, c2, lane);
  for (int64_t r = warp0; r < n; r += 2 * nwarps) {   // two rows (four row loads) in flight per warp
    const int64_t r2 = r + nwarps;
    const bool has2 = r2 < n;
    float v[V], g[V], v2[V], g2[V];
    ld_row<D, true>(v, R + r * D, lane);
    ld_row<D, true>(g, g_out + r * D, lane);
    if (has2) {
      ld_row<D, true>(v2, R + r2 * D, lane);
      ld_row<D, true>(g2, g_out + r2 * D, lane);
    }
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float gu = g[k] * dsilu_(v[k] * sc[k] + sh[k]);
      g[k] = sc[k] * (gu - k1[k] - (v[k] - mu[k]) * rs[k] * k2[k]);
    }
    st_row<D, true>(gR + r * D, g, lane);
    if (has2) {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float gu = g2[k] * dsilu_(v2[k] * sc[k] + sh[k]);
        g2[k] = sc[k] * (gu - k1[k] - (v2[k] - mu[k]) * rs[k] * k2[k]);
      }
      st_row<D, true>(gR + r2 * D, g2, lane);
    }
  }
}

// per-block partial column sums of a tall [n, D] matrix (bias gradients of the embedding Linears)
template <int D>
__global__ void __launch_bounds__(kThreads)
colsum_partials_kernel(const float* __restrict__ a, int64_t n, float* __restrict__ partials) {
  constexpr int V = RowCfg<D>::VPL;
  __shared__ float red[kWarpsPerBlock * D];
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float acc[1][V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[0][k] = 0.f;
  for (int64_t r = warp0; r < n; r += nwarps) {
    float v[V];
    ld_row<D, false>(v, a + r * D, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) acc[0][k] += v[k];
  }
  block_reduce_to_partials<D, 1>(acc, partials + (int64_t)blockIdx.x * D, red);
}

// out[c] = alpha * sum_r a[r*stride + c]; 32 columns per block x 32 row lanes, fp64, fixed order.
// Used on per-block partial buffers (rows <= kMaxBlocks).
__global__ void __launch_bounds__(1024)
colsum_kernel(const float* __restrict__ a, int64_t rows, int cols, int64_t stride, float alpha,
              float* __restrict__ out) {
  __shared__ double ss[32][33];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double s = 0.0;
  if (c < cols)
    for (int64_t r = rl; r < rows; r += 32) s += (double)a[r * stride + c];
  ss[rl][cl] = s;
  __syncthreads();
  if (rl != 0 || c >= cols) return;
#pragma unroll
  for (int k = 1; k < 32; ++k) s += ss[k][cl];
  out[c] = alpha * (float)s;
}

// Many column sums in one launch: problem p sums `cols` columns of its own partial buffer into its own output vector
// (the bias / norm-parameter gradients of every conv of a backward pass: 100+ vectors of d floats, each the fixed-order
// fp64 sum of <= 592 partial rows).  blockIdx.y = problem, blockIdx.x = 32-column chunk; same arithmetic as colsum_kernel.
struct ColsumProblem { const float* a; float* out; int64_t rows, stride; int cols; float alpha; };
constexpr int kMaxColsumProblems = 192;
struct ColsumBatch { ColsumProblem p[kMaxColsumProblems]; };
__global__ void __launch_bounds__(1024)
colsum_batch_kernel(const __grid_constant__ ColsumBatch bt) {
  __shared__ double ss[32][33];
  const ColsumProblem& q = bt.p[blockIdx.y];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double s = 0.0;
  if (c < q.cols)
    for (int64_t r = rl; r < q.rows; r += 32) s += (double)q.a[r * q.stride + c];
  ss[rl][cl] = s;
  __syncthreads();
  if (rl != 0 || c >= q.cols) return;
#pragma unroll
  for (int k = 1; k < 32; ++k) s += ss[k][cl];
  q.out[c] = q.alpha * (float)s;
}

// =============================================================================================
// Gather / segment-sum primitive (DGL u_mul_e -> sum and copy_e -> sum in one pass)
// =============================================================================================
template <int D>
__global__ void __launch_bounds__(kThreads)
gather_segment_sum_kernel(const float* __restrict__ Bh, const float* __restrict__ sigma, const int32_t* __restrict__ src,
                          const int32_t* __restrict__ in_ptr, const int32_t* __restrict__ in_eid, int64_t Nn,
                          float* __restrict__ Sh, float* __restrict__ S) {
  constexpr int V = RowCfg<D>::VPL;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  for (int64_t v = warp0; v < Nn; v += nwarps) {
    float accS[V], accSh[V];
#pragma unroll
    for (int k = 0; k < V; ++k) { accS[k] = 0.f; accSh[k] = 0.f; }
    const int p0 = in_ptr[v], p1 = in_ptr[v + 1];
    for (int base = p0; base < p1; base += 32) {
      const int cnt = min(32, p1 - base);
      int my_e = 0, my_s = 0;
      if (lane < cnt) {
        my_e = in_eid ? in_eid[base + lane] : base + lane;
        my_s = src[my_e];
      }
      int i = 0;
      for (; i + 1 < cnt; i += 2) {   // two edges in flight per warp
        const int64_t e0 = __shfl_sync(0xffffffffu, my_e, i), s0 = __shfl_sync(0xffffffffu, my_s, i);
        const int64_t e1 = __shfl_sync(0xffffffffu, my_e, i + 1), s1 = __shfl_sync(0xffffffffu, my_s, i + 1);
        float g0[V], b0[V], g1[V], b1[V];
        ld_row<D, true>(g0, sigma + e0 * D, lane);
        ld_row<D, true>(g1, sigma + e1 * D, lane);
        ld_row<D, false>(b0, Bh + s0 * D, lane);
        ld_row<D, false>(b1, Bh + s1 * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) { accS[k] += g0[k]; accSh[k] += b0[k] * g0[k]; }
#pragma unroll
        for (int k = 0; k < V; ++k) { accS[k] += g1[k]; accSh[k] += b1[k] * g1[k]; }
      }
      if (i < cnt) {
        const int64_t e0 = __shfl_sync(0xffffffffu, my_e, i), s0 = __shfl_sync(0xffffffffu, my_s, i);
        float g0[V], b0[V];
        ld_row<D, true>(g0, sigma + e0 * D, lane);
        ld_row<D, false>(b0, Bh + s0 * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) { accS[k] += g0[k]; accSh[k] += b0[k] * g0[k]; }
      }
    }
    st_row<D, true>(Sh + v * D, accSh, lane);
    st_row<D, true>(S + v * D, accS, lane);
  }
}

// =============================================================================================
// Per-graph mean pooling over node rows and its backward (block per graph)
// =============================================================================================
__global__ void segment_mean_kernel(const float* __restrict__ x, const int32_t* __restrict__ gptr, int d,
                                    float* __restrict__ out) {
  const int b = blockIdx.x;
  const int r0 = gptr[b], r1 = gptr[b + 1];
  const float inv = r1 > r0 ? 1.f / (float)(r1 - r0) : 0.f;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int r = r0; r < r1; ++r) s += x[(size_t)r * d + c];
    out[(size_t)b * d + c] = s * inv;
  }
}

__global__ void segment_mean_backward_kernel(const float* __restrict__ g_out, const int32_t* __restrict__ gptr, int d,
                                             float* __restrict__ gx) {
  const int b = blockIdx.x;
  const int r0 = gptr[b], r1 = gptr[b + 1];
  const float inv = r1 > r0 ? 1.f / (float)(r1 - r0) : 0.f;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const float g = g_out[(size_t)b * d + c] * inv;
    for (int r = r0; r < r1; ++r) gx[(size_t)r * d + c] = g;
  }
}

}  // namespace alignn

// =============================================================================================
// C ABI
// =============================================================================================
#include <atomic>
#include <mutex>
#include <unordered_map>

namespace alignn {
std::atomic<uint64_t> g_launches{0};
std::atomic<int> g_last_cuda_error{0};
int check_launch() {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { g_last_cuda_error.store((int)e); return ALIGNN_ERR_CUDA; }
  return ALIGNN_OK;
}
int record_cuda_error(int e) { g_last_cuda_error.store(e); return ALIGNN_ERR_CUDA; }
int one_wave_grid(const void* kernel, int threads, size_t dyn_smem, int wanted_blocks) {
  static std::mutex mu;
  static std::unordered_map<const void*, int> cache;
  int resident;
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(kernel);
    if (it == cache.end()) {
      int per_sm = 0, dev = 0, sms = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, dyn_smem) != cudaSuccess || per_sm < 1) {
        (void)cudaGetLastError();
        per_sm = 1;
      }
      it = cache.emplace(kernel, per_sm * (sms > 0 ? sms : kNumSMs)).first;
    }
    resident = it->second;
  }
  return wanted_blocks < resident ? wanted_blocks : resident;
}
}  // namespace alignn

namespace {
using alignn::check_launch;
using alignn::g_launches;
std::atomic<int> g_forward_ring{1};      // alignn_b200_debug_egc_flags bit 0 selects the register-staged pass 2 instead
using alignn::g_last_cuda_error;
inline bool supported_d(int d) { return d == 32 || d == 64 || d == 128 || d == 256; }
inline int grid_for_rows(int64_t n) {
  int64_t b = (n + alignn::kWarpsPerBlock - 1) / alignn::kWarpsPerBlock;
  if (b < 1) b = 1;
  if (b > alignn::kMaxBlocks) b = alignn::kMaxBlocks;
  return (int)b;
}
inline bool norm_ok(int m) { return m == ALIGNN_NORM_LAYER || m == ALIGNN_NORM_AFFINE || m == ALIGNN_NORM_STATS; }
}  // namespace

#define DISPATCH_D(d, ...)                         \
  switch (d) {                                     \
    case 32: { constexpr int D = 32; __VA_ARGS__; break; }   \
    case 64: { constexpr int D = 64; __VA_ARGS__; break; }   \
    case 128: { constexpr int D = 128; __VA_ARGS__; break; } \
    case 256: { constexpr int D = 256; __VA_ARGS__; break; } \
    default: return ALIGNN_ERR_UNSUPPORTED_D;      \
  }

extern "C" {

int alignn_b200_version(void) { return ALIGNN_B200_VERSION; }

const char* alignn_b200_strerror(int s) {
  switch (s) {
    case ALIGNN_OK: return "ok";
    case ALIGNN_ERR_BAD_ARG: return "bad argument (NULL pointer, negative size or invalid flag)";
    case ALIGNN_ERR_UNSUPPORTED_D: return "unsupported feature width d (supported: 32, 64, 128, 256)";
    case ALIGNN_ERR_STRUCT_SIZE: return "argument struct size mismatch between caller and library";
    case ALIGNN_ERR_CUDA: return "CUDA runtime error (see alignn_b200_last_cuda_error)";
    case ALIGNN_ERR_WORKSPACE: return "workspace too small";
    default: return "unknown status";
  }
}

int alignn_b200_last_cuda_error(void) { return g_last_cuda_error.load(); }
void alignn_b200_debug_egc_flags(int flags) { g_forward_ring.store((flags & 1) ? 0 : 1); }
uint64_t alignn_b200_launch_count(void) { return g_launches.load(); }

int alignn_b200_egc_partial_rows(int64_t Nn, int d) { (void)d; return grid_for_rows(Nn); }

int alignn_b200_egc_forward(const alignn_b200_egc_fwd_args* a) {
  if (!a) return ALIGNN_ERR_BAD_ARG;
  if (a->struct_size != sizeof(*a)) return ALIGNN_ERR_STRUCT_SIZE;
  if (!supported_d(a->d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (a->Nn < 0 || a->Ne < 0 || !norm_ok(a->norm_nodes) || !norm_ok(a->norm_edges)) return ALIGNN_ERR_BAD_ARG;
  if (a->Nn == 0) return ALIGNN_OK;
  if (!a->P || !a->in_ptr || (a->Ne > 0 && (!a->G || !a->src))) return ALIGNN_ERR_BAD_ARG;
  if (a->norm_nodes != ALIGNN_NORM_STATS && (!a->x_out || !a->n_w || !a->n_b)) return ALIGNN_ERR_BAD_ARG;
  if (a->norm_edges != ALIGNN_NORM_STATS && a->y_out && (!a->e_w || !a->e_b)) return ALIGNN_ERR_BAD_ARG;
  if (a->residual && ((a->norm_nodes != ALIGNN_NORM_STATS && !a->x) ||
                      (a->norm_edges != ALIGNN_NORM_STATS && a->y_out && !a->y))) return ALIGNN_ERR_BAD_ARG;
  if ((a->norm_nodes == ALIGNN_NORM_STATS || a->norm_edges == ALIGNN_NORM_STATS) && !a->partials) return ALIGNN_ERR_BAD_ARG;
  if ((a->norm_nodes == ALIGNN_NORM_STATS || a->norm_edges == ALIGNN_NORM_STATS) && !a->XP) return ALIGNN_ERR_BAD_ARG;
  if (a->XP && (!a->S || !a->H || (a->Ne > 0 && !a->M && !a->gate_is_m))) return ALIGNN_ERR_BAD_ARG;   // training: all saved buffers
  if (a->gate_is_m && a->norm_edges == ALIGNN_NORM_STATS && a->y_out) return ALIGNN_ERR_BAD_ARG;   // statistics come from the gather GEMM
  cudaStream_t st = (cudaStream_t)a->stream;
  const int grid = grid_for_rows(a->Nn);
  DISPATCH_D(a->d, {
    const size_t smem_bytes = (size_t)(4 + (a->partials ? alignn::kWarpsPerBlock * 4 : 0)) * D * sizeof(float);
    if (a->gate_is_m && g_forward_ring.load()) {
      // rows staged through a shared-memory ring (cp.async); same results as egc_forward_kernel<D, true>
      const size_t ring_bytes = (size_t)(4 + alignn::kWarpsPerBlock * alignn::kRing * 3) * D * sizeof(float);
      static alignn::DeviceOnce configured; int cfg_dev;
      if (configured.needed(&cfg_dev)) {
        cudaError_t e = cudaFuncSetAttribute(alignn::egc_forward_ring_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)ring_bytes);
        if (e != cudaSuccess) return alignn::record_cuda_error((int)e);
        configured.done(cfg_dev);
      }
      alignn::egc_forward_ring_kernel<D><<<grid, alignn::kThreads, ring_bytes, st>>>(*a);
    } else if (a->gate_is_m) alignn::egc_forward_kernel<D, true><<<grid, alignn::kThreads, smem_bytes, st>>>(*a);
    else alignn::egc_forward_kernel<D, false><<<grid, alignn::kThreads, smem_bytes, st>>>(*a);   // <= 36 KB: no opt-in needed
  });
  return check_launch();
}

int alignn_b200_bn_finalize(const float* partials, int partial_rows, int partial_stride, int which, int64_t count, int d,
                            const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                            float* running_var, float* scale, float* shift, float* mean, float* rstd,
                            alignn_stream_t stream) {
  if (!partials || !scale || !shift || !mean || !rstd || partial_rows <= 0 || d <= 0 || count <= 0 ||
      (which != 0 && which != 1) || ((running_mean == nullptr) != (running_var == nullptr)))
    return ALIGNN_ERR_BAD_ARG;
  alignn::bn_finalize_kernel<<<(d + 31) / 32, 1024, 0, (cudaStream_t)stream>>>(
      partials, partial_rows, partial_stride, which, (double)count, d, gamma, beta, eps, momentum, running_mean,
      running_var, scale, shift, mean, rstd);
  return check_launch();
}

int alignn_b200_affine_silu_residual(const float* R, const float* res, const float* scale, const float* shift, float* out,
                                     int64_t n, int d, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n < 0 || (n > 0 && (!R || !scale || !shift || !out))) return ALIGNN_ERR_BAD_ARG;
  if (n == 0) return ALIGNN_OK;
  const int grid = grid_for_rows(n);
  DISPATCH_D(d, alignn::affine_silu_residual_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(
                    R, res, scale, shift, out, n));
  return check_launch();
}

int alignn_b200_egc_backward(const alignn_b200_egc_bwd_args* a) {
  if (!a) return ALIGNN_ERR_BAD_ARG;
  if (a->struct_size != sizeof(*a)) return ALIGNN_ERR_STRUCT_SIZE;
  if (!supported_d(a->d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (a->Nn < 0 || a->Ne < 0 || !norm_ok(a->norm_nodes) || !norm_ok(a->norm_edges)) return ALIGNN_ERR_BAD_ARG;
  if (a->Nn == 0) return ALIGNN_OK;
  if (!a->P || !a->XP || !a->S || !a->H || !a->in_ptr || !a->out_ptr || !a->gx_out || !a->GP || !a->GSh ||
      !a->n_w || !a->n_b)
    return ALIGNN_ERR_BAD_ARG;
  if (a->Ne > 0 && (!a->M || !a->src || !a->dst || !a->out_eid || !a->GM)) return ALIGNN_ERR_BAD_ARG;
  if (a->norm_nodes != ALIGNN_NORM_LAYER && (!a->n_mean || !a->n_rstd)) return ALIGNN_ERR_BAD_ARG;
  if (a->norm_nodes == ALIGNN_NORM_STATS && (!a->n_c1 || !a->n_c2)) return ALIGNN_ERR_BAD_ARG;
  if (a->gy_out) {
    if (!a->e_w || !a->e_b) return ALIGNN_ERR_BAD_ARG;
    if (a->norm_edges != ALIGNN_NORM_LAYER && (!a->e_mean || !a->e_rstd)) return ALIGNN_ERR_BAD_ARG;
    if (a->norm_edges == ALIGNN_NORM_STATS && (!a->e_c1 || !a->e_c2)) return ALIGNN_ERR_BAD_ARG;
  }
  cudaStream_t st = (cudaStream_t)a->stream;
  const int grid = grid_for_rows(a->Nn);
  if (a->norm_nodes != a->norm_edges) return ALIGNN_ERR_BAD_ARG;   // both norms of a conv are of one kind (alignn.py:71-76)
  const bool line = a->parent_in_ptr || a->parent_in_eid || a->parent_out_ptr || a->parent_out_eid || a->parent_Nn;
  if (line) {
    // one pass per atom of the parent graph (egc_backward_line_kernel); `grid` partial rows, as the two-pass path
    if (!a->parent_in_ptr || !a->parent_out_ptr || a->parent_Nn <= 0 ||
        (a->Nn > 0 && (!a->parent_in_eid || !a->parent_out_eid)) || (a->Ne > 0 && (!a->M || !a->GM)))
      return ALIGNN_ERR_BAD_ARG;
#define LAUNCH_BWD_LINE(NORM)                                                                                   \
  DISPATCH_D(a->d, {                                                                                           \
    const size_t smem_bytes = alignn::line_bwd_smem_floats<D>() * sizeof(float);                               \
    static alignn::DeviceOnce configured; int cfg_dev;                                                         \
    if (configured.needed(&cfg_dev)) {                                                                         \
      cudaError_t e = cudaFuncSetAttribute(alignn::egc_backward_line_kernel<D, NORM>,                          \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);      \
      if (e != cudaSuccess) return alignn::record_cuda_error((int)e);                                          \
      configured.done(cfg_dev);                                                                                \
    }                                                                                                          \
    const int64_t want = a->parent_Nn < grid ? a->parent_Nn : grid;                                            \
    const int grid_line = alignn::one_wave_grid((const void*)alignn::egc_backward_line_kernel<D, NORM>,        \
                                                alignn::kLineThreads, smem_bytes, (int)want);                  \
    alignn::egc_backward_line_kernel<D, NORM><<<grid_line, alignn::kLineThreads, smem_bytes, st>>>(*a, grid);  \
  })
    switch (a->norm_nodes) {
      case ALIGNN_NORM_LAYER: LAUNCH_BWD_LINE(ALIGNN_NORM_LAYER); break;
      case ALIGNN_NORM_AFFINE: LAUNCH_BWD_LINE(ALIGNN_NORM_AFFINE); break;
      default: LAUNCH_BWD_LINE(ALIGNN_NORM_STATS); break;
    }
#undef LAUNCH_BWD_LINE
    return check_launch();
  }
#define LAUNCH_BWD_DST(NORM)                                                                                   \
  DISPATCH_D(a->d, {                                                                                           \
    const size_t smem_bytes = (size_t)(alignn::kWarpsPerBlock * 8 + 12) * D * sizeof(float);                   \
    static alignn::DeviceOnce configured; int cfg_dev;                                                                            \
    if (configured.needed(&cfg_dev)) {                                                                                         \
      cudaError_t e = cudaFuncSetAttribute(alignn::egc_backward_dst_kernel<D, NORM>,                           \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);      \
      if (e != cudaSuccess) return alignn::record_cuda_error((int)e);                                          \
      configured.done(cfg_dev);                                                                                       \
    }                                                                                                          \
    alignn::egc_backward_dst_kernel<D, NORM><<<grid, alignn::kThreads, smem_bytes, st>>>(*a);                  \
  })
  switch (a->norm_nodes) {
    case ALIGNN_NORM_LAYER: LAUNCH_BWD_DST(ALIGNN_NORM_LAYER); break;
    case ALIGNN_NORM_AFFINE: LAUNCH_BWD_DST(ALIGNN_NORM_AFFINE); break;
    default: LAUNCH_BWD_DST(ALIGNN_NORM_STATS); break;
  }
#undef LAUNCH_BWD_DST
  int rc = check_launch();
  if (rc != ALIGNN_OK) return rc;
  DISPATCH_D(a->d, {
    // `grid` partial rows are expected by the caller; the kernel runs as one wave and zeroes the rows no block owns
    const int grid_src = alignn::one_wave_grid((const void*)alignn::egc_backward_src_kernel<D>, alignn::kThreads, 0, grid);
    if (2 * grid_src < grid) return ALIGNN_ERR_CUDA;       // cannot happen on a device with >= 74 SMs
    alignn::egc_backward_src_kernel<D><<<grid_src, alignn::kThreads, 0, st>>>(*a, a->partials_src, grid);
  });
  return check_launch();
}

int alignn_b200_bn_backward_reduce(const float* R, const float* g_out, const float* scale, const float* shift,
                                   const float* mean, const float* rstd, int64_t n, int d, float* partials,
                                   int partial_rows, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n <= 0 || !R || !g_out || !scale || !shift || !mean || !rstd || !partials) return ALIGNN_ERR_BAD_ARG;
  const int grid = grid_for_rows(n);
  if (partial_rows < grid) return ALIGNN_ERR_WORKSPACE;
  DISPATCH_D(d, alignn::bn_backward_reduce_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(
                    R, g_out, scale, shift, mean, rstd, n, partials));
  return check_launch();
}

int alignn_b200_rowstats_partials(const float* a, int64_t n, int d, float* partials, int partial_rows, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n <= 0 || !a || !partials) return ALIGNN_ERR_BAD_ARG;
  const int grid = grid_for_rows(n);
  if (partial_rows < grid) return ALIGNN_ERR_WORKSPACE;
  DISPATCH_D(d, alignn::rowstats_partials_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(a, n, partials));
  return check_launch();
}

int alignn_b200_bn_backward_apply(const float* R, const float* g_out, const float* scale, const float* shift,
                                  const float* mean, const float* rstd, const float* c1, const float* c2, int64_t n, int d,
                                  float* gR, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n <= 0 || !R || !g_out || !scale || !shift || !mean || !rstd || !c1 || !c2 || !gR) return ALIGNN_ERR_BAD_ARG;
  DISPATCH_D(d, {
    const int grid = alignn::one_wave_grid((const void*)alignn::bn_backward_apply_kernel<D>, alignn::kThreads, 0, grid_for_rows(n));
    alignn::bn_backward_apply_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(R, g_out, scale, shift, mean, rstd, c1, c2, n, gR);
  });
  return check_launch();
}

int alignn_b200_colsum_partials(const float* a, int64_t n, int d, float* partials, int partial_rows, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n <= 0 || !a || !partials) return ALIGNN_ERR_BAD_ARG;
  const int grid = grid_for_rows(n);
  if (partial_rows < grid) return ALIGNN_ERR_WORKSPACE;
  DISPATCH_D(d, alignn::colsum_partials_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(a, n, partials));
  return check_launch();
}

int alignn_b200_colsum(const float* a, int64_t rows, int cols, int64_t stride, float alpha, float* out,
                       alignn_stream_t stream) {
  if (!a || !out || rows < 0 || cols <= 0 || stride < cols) return ALIGNN_ERR_BAD_ARG;
  alignn::colsum_kernel<<<(cols + 31) / 32, 1024, 0, (cudaStream_t)stream>>>(a, rows, cols, stride, alpha, out);
  return check_launch();
}

int alignn_b200_colsum_batch(const alignn_b200_colsum_problem* problems, int n, alignn_stream_t stream) {
  if (!problems || n < 0) return ALIGNN_ERR_BAD_ARG;
  static thread_local alignn::ColsumBatch bt;
  for (int i0 = 0; i0 < n; i0 += alignn::kMaxColsumProblems) {
    const int m = n - i0 < alignn::kMaxColsumProblems ? n - i0 : alignn::kMaxColsumProblems;
    int max_cols = 0;
    for (int i = 0; i < m; ++i) {
      const alignn_b200_colsum_problem& q = problems[i0 + i];
      if (!q.a || !q.out || q.rows < 0 || q.cols <= 0 || q.stride < q.cols) return ALIGNN_ERR_BAD_ARG;
      bt.p[i].a = q.a; bt.p[i].out = q.out; bt.p[i].rows = q.rows; bt.p[i].stride = q.stride; bt.p[i].cols = q.cols;
      bt.p[i].alpha = q.alpha;
      if (q.cols > max_cols) max_cols = q.cols;
    }
    alignn::colsum_batch_kernel<<<dim3((max_cols + 31) / 32, m), 1024, 0, (cudaStream_t)stream>>>(bt);
    int rc = check_launch();
    if (rc != ALIGNN_OK) return rc;
  }
  return ALIGNN_OK;
}

int alignn_b200_gather_segment_sum(const float* Bh, const float* sigma, const int32_t* src, const int32_t* in_ptr,
                                   const int32_t* in_eid, int64_t Nn, int64_t Ne, int d, float* Sh, float* S,
                                   alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (Nn < 0 || Ne < 0) return ALIGNN_ERR_BAD_ARG;
  if (Nn == 0) return ALIGNN_OK;
  if (!in_ptr || !Sh || !S || (Ne > 0 && (!Bh || !sigma || !src))) return ALIGNN_ERR_BAD_ARG;
  int64_t b = (Nn + alignn::kWarpsPerBlock - 1) / alignn::kWarpsPerBlock;
  const int grid = (int)(b > alignn::kNumSMs * 16 ? alignn::kNumSMs * 16 : b);
  DISPATCH_D(d, alignn::gather_segment_sum_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(
                    Bh, sigma, src, in_ptr, in_eid, Nn, Sh, S));
  return check_launch();
}

int alignn_b200_segment_mean(const float* x, const int32_t* graph_ptr, int64_t B, int d, float* out,
                             alignn_stream_t stream) {
  if (B < 0 || d <= 0) return ALIGNN_ERR_BAD_ARG;
  if (B == 0) return ALIGNN_OK;
  if (!x || !graph_ptr || !out) return ALIGNN_ERR_BAD_ARG;
  alignn::segment_mean_kernel<<<(unsigned)B, 256, 0, (cudaStream_t)stream>>>(x, graph_ptr, d, out);
  return check_launch();
}

int alignn_b200_segment_mean_backward(const float* g_out, const int32_t* graph_ptr, int64_t B, int d, float* gx,
                                      alignn_stream_t stream) {
  if (B < 0 || d <= 0) return ALIGNN_ERR_BAD_ARG;
  if (B == 0) return ALIGNN_OK;
  if (!g_out || !graph_ptr || !gx) return ALIGNN_ERR_BAD_ARG;
  alignn::segment_mean_backward_kernel<<<(unsigned)B, 256, 0, (cudaStream_t)stream>>>(g_out, graph_ptr, d, gx);
  return check_launch();
}

}  // extern "C"
