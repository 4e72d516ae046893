// Double backward of the LayerNorm edge-gated graph convolution, fp32, sm_90a: the vector-Jacobian product of the
// first backward (alignn_b200_egc_backward plus its GEMMs) that `torch.autograd.grad(..., create_graph=True)` needs
// for force training (alignn/models/alignn_atomwise.py:530-539).  Same structure as the first backward: one warp per
// node, a destination-keyed pass over the in-CSR and a source-keyed pass over the out-CSR, every reduction in
// registers or per-warp shared memory, per-block partial rows for the parameter sums -- no atomics, deterministic.
//
// Notation (include/alignn_b200.h, P = [A = e_src | C = Bh | B = e_dst | D = src_update]):
//   forward      M = y W_eg^T + A[s] + B[t],  sg = sigmoid(M),  Sh_v = sum_in C[s] sg,  S_v = sum_in sg,
//                r = 1 / (S + eps),  H = Sh r,  XP = D + H
//   first bwd    gXP = Jn(XP, gx_out),  gM0 = Je(M, gy_out)   (row-local LayerNorm + SiLU backwards)
//                gSh = gXP r,  gS = -gXP H r,  gM = gM0 + (gSh[t] C[s] + gS[t]) sg'
//                GP = [sum_out gM | sum_out gSh[t] sg | sum_in gM | gXP]
// Given the cotangents of gx = GP Wcat (+ gx_out) and gy = gM W_eg (+ gy_out), projected by the caller through the
// same weights (GPbar = gx_bar Wcat^T, GMbar = gy_bar W_eg^T), this file produces Pbar = dL/dP, Mbar = dL/dM and the
// cotangents of gx_out, gy_out and of the four LayerNorm parameters.  The caller finishes through the forward GEMMs.
#include "common.cuh"
#include "api_common.h"
#include "alignn_b200.h"

#include <type_traits>

namespace alignn {
namespace {

// lane-layout row -> per-warp shared-memory row; each lane writes (and later reads) only its own channels
template <int D>
__device__ __forceinline__ void st_srow(float* __restrict__ row, const float (&v)[RowCfg<D>::VPL], int lane) {
  using C = RowCfg<D>;
#pragma unroll
  for (int c = 0; c < C::CH; ++c)
#pragma unroll
    for (int j = 0; j < C::W; ++j) row[c * 32 * C::W + lane * C::W + j] = v[c * C::W + j];
}

// VJP of the row map (m, g_out, w, b) -> gm = d/dm [g_out . silu(LayerNorm(m) * w + b)] with cotangent `gam` on gm.
// On return: mbar (dL/dm), gob (dL/dg_out), gm (the first-backward row itself); the row's contributions to dL/dw and
// dL/db are added to the shared-memory accumulator rows acc_w / acc_b.  w, b live in shared memory.
template <int D>
__device__ __forceinline__ void ln_silu_vjp_row(const float (&m)[RowCfg<D>::VPL], const float (&go)[RowCfg<D>::VPL],
                                                const float (&gam)[RowCfg<D>::VPL], float ln_eps,
                                                const float* __restrict__ w_s, const float* __restrict__ b_s,
                                                float (&mbar)[RowCfg<D>::VPL], float (&gob)[RowCfg<D>::VPL],
                                                float (&gm)[RowCfg<D>::VPL], float* __restrict__ acc_w,
                                                float* __restrict__ acc_b, int lane) {
  constexpr int V = RowCfg<D>::VPL;
  float mean, rstd;
  row_mean_rstd<D>(m, ln_eps, mean, rstd);
  float w[V], xh[V], s1[V], s2[V], gu[V], gxh[V];
  {
    float b[V];
    ld_srow<D>(w, w_s, lane);
    ld_srow<D>(b, b_s, lane);
    float sa = 0.f, sc = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      xh[k] = (m[k] - mean) * rstd;
      const float u = xh[k] * w[k] + b[k];
      const float s = sigmoidf_(u);
      s1[k] = s * (1.f + u * (1.f - s));                       // silu'(u)
      s2[k] = s * (1.f - s) * (2.f + u * (1.f - 2.f * s));      // silu''(u)
      gu[k] = go[k] * s1[k];
      gxh[k] = gu[k] * w[k];
      sa += gxh[k];
      sc += gxh[k] * xh[k];
    }
    sa = warp_sum(sa) * (1.f / D);
    sc = warp_sum(sc) * (1.f / D);
    // gm = rstd (gxh - mean(gxh) - xh mean(gxh xh));  mbar collects its rstd * xh-free part later
    float p = 0.f, q = 0.f, rg = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      gm[k] = rstd * (gxh[k] - sa - xh[k] * sc);
      const float gp = rstd * gam[k];
      p += gp;
      q += gp * xh[k];
      rg += gam[k] * gm[k];
    }
    p = warp_sum(p) * (1.f / D);
    q = warp_sum(q) * (1.f / D);
    rg = warp_sum(rg) * (1.f / D);
    // cotangents of gxh (projected like a LayerNorm backward) and of xh (through the two means of gm)
    float e1 = 0.f, e2 = 0.f, aw[V], ab[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float gp = rstd * gam[k];
      const float gxhb = gp - p - xh[k] * q;
      float xhb = -sc * gp - q * gxh[k];
      const float gub = gxhb * w[k];
      gob[k] = gub * s1[k];
      const float ub = gub * go[k] * s2[k];
      xhb += ub * w[k];
      aw[k] = gxhb * gu[k] + ub * xh[k];
      ab[k] = ub;
      mbar[k] = xhb;
      e1 += xhb;
      e2 += xhb * xh[k];
    }
    smem_row_add<D>(acc_w, aw, lane);
    smem_row_add<D>(acc_b, ab, lane);
    e1 = warp_sum(e1) * (1.f / D);
    e2 = warp_sum(e2) * (1.f / D);
    // back through xh = (m - mean) rstd, plus the direct use of rstd in gm (d rstd / dm = -rstd^2 xh / D)
#pragma unroll
    for (int k = 0; k < V; ++k) mbar[k] = rstd * (mbar[k] - e1 - xh[k] * e2) - rstd * rg * xh[k];
  }
}

__device__ __forceinline__ float dsig_(float s) { return s * (1.f - s); }

// Destination-keyed pass.  Per node v (in-edges e, sources s):
//   Gamma_e = GMbar_e + GPbar_A[s] + GPbar_B[v]                         (cotangent of gM_e; stored for the source pass)
//   Je VJP(Gamma_e) -> Mbar_e, gy_out_bar_e;  Mbar_e += Gamma_e (gSh C[s] + gS) sg'' + GPbar_C[s] gSh sg'
//   gShb = sum_in Gamma_e C[s] sg' + GPbar_C[s] sg,   gSb = sum_in Gamma_e sg'
//   Jn VJP(GPbar_D + (gShb - gSb H) r) -> XPbar, gx_out_bar;  Hbar = XPbar - gSb gXP r,  Shbar = Hbar r,
//   Sbar = -Hbar H r - (gShb - gSb H) gXP r^2;  second sweep: Mbar_e += (Shbar C[s] + Sbar) sg'
//   Pbar_B[v] = sum_in Mbar_e,  Pbar_D[v] = XPbar
// partials row: {sum e_w-bar, sum e_b-bar, sum n_w-bar, sum n_b-bar, sum Pbar_D, sum Pbar_B}
template <int D>
__global__ void __launch_bounds__(kThreads, 1)
egc_vjp_dst_kernel(alignn_b200_egc_bwd_vjp_args a) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  extern __shared__ __align__(16) float dyn_smem[];
  float* vec = dyn_smem;                                   // [4][D]: n_w, n_b, e_w, e_b
  float* sacc = vec + 4 * D;                               // [kWarpsPerBlock][6][D]  partial sums
  float* sseg = sacc + kWarpsPerBlock * 6 * D;             // [kWarpsPerBlock][5][D]  per-node rows of the segment
  {
    const float* srcs[4] = {a.n_w, a.n_b, a.e_w, a.e_b};
#pragma unroll
    for (int q = 0; q < 4; ++q)
      for (int i = threadIdx.x; i < D; i += blockDim.x) vec[q * D + i] = srcs[q] ? srcs[q][i] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + wib;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float* acc = sacc + wib * 6 * D;
  for (int i = lane; i < 6 * D; i += 32) acc[i] = 0.f;
  // rows of the warp's segment: gSh, gS (later Shbar, Sbar), GPbar_B, and the accumulators gShb, gSb
  float* s_gsh = sseg + wib * 5 * D;
  float* s_gs = s_gsh + D;
  float* s_gbb = s_gsh + 2 * D;
  float* s_ashb = s_gsh + 3 * D;
  float* s_asb = s_gsh + 4 * D;
  __syncwarp();

  for (int64_t v = warp0; v < a.Nn; v += nwarps) {
    {
      float gsh[V], hv[V], gs[V], t[V];
      ld_row<D, false>(gsh, a.GSh + v * D, lane);
      ld_row<D, false>(hv, a.H + v * D, lane);
      ld_row<D, false>(t, a.GPbar + v * 4 * D + 2 * D, lane);
#pragma unroll
      for (int k = 0; k < V; ++k) gs[k] = -gsh[k] * hv[k];    // gS = -gXP H r = -gSh H
      st_srow<D>(s_gsh, gsh, lane);
      st_srow<D>(s_gs, gs, lane);
      st_srow<D>(s_gbb, t, lane);
#pragma unroll
      for (int k = 0; k < V; ++k) t[k] = 0.f;
      st_srow<D>(s_ashb, t, lane);
      st_srow<D>(s_asb, t, lane);
    }
    const int p0 = a.in_ptr[v], p1 = a.in_ptr[v + 1];
    // ---- sweep 1: Gamma, the edge-norm VJP and the gate terms of Mbar; segment sums gShb, gSb ----
    for (int base = p0; base < p1; base += 32) {
      const int cnt = min(32, p1 - base);
      int my_e = 0, my_s = 0;
      if (lane < cnt) {
        my_e = a.in_eid ? a.in_eid[base + lane] : base + lane;
        my_s = a.src[my_e];
      }
      for (int i = 0; i < cnt; ++i) {
        const int64_t e = __shfl_sync(0xffffffffu, my_e, i);
        const int64_t s = __shfl_sync(0xffffffffu, my_s, i);
        float m[V], gam[V], cv[V], gcb[V], mb[V];
        ld_row<D, true>(m, a.M + e * D, lane);
        ld_row<D, false>(cv, a.P + s * 4 * D + D, lane);
        ld_row<D, false>(gcb, a.GPbar + s * 4 * D + D, lane);
        {
          float gab[V], gbb[V];
          ld_row<D, false>(gab, a.GPbar + s * 4 * D, lane);
          ld_srow<D>(gbb, s_gbb, lane);
          if (a.GMbar) ld_row<D, true>(gam, a.GMbar + e * D, lane);
          else {
#pragma unroll
            for (int k = 0; k < V; ++k) gam[k] = 0.f;
          }
#pragma unroll
          for (int k = 0; k < V; ++k) gam[k] = gam[k] + gab[k] + gbb[k];
        }
        st_row<D, true>(a.Gamma + e * D, gam, lane);
        if (a.gy_out) {
          float go[V], gob[V], gm0[V];
          ld_row<D, true>(go, a.gy_out + e * D, lane);
          ln_silu_vjp_row<D>(m, go, gam, a.ln_eps, vec + 2 * D, vec + 3 * D, mb, gob, gm0, acc, acc + D, lane);
          if (a.gy_bar_res) {
            float r[V];
            ld_row<D, true>(r, a.gy_bar_res + e * D, lane);
#pragma unroll
            for (int k = 0; k < V; ++k) gob[k] += r[k];
          }
          st_row<D, true>(a.gy_out_bar + e * D, gob, lane);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) mb[k] = 0.f;
        }
        {
          float gsh[V], gs[V], ashb[V], asb[V];
          ld_srow<D>(gsh, s_gsh, lane);
          ld_srow<D>(gs, s_gs, lane);
#pragma unroll
          for (int k = 0; k < V; ++k) {
            const float sg = sigmoidf_(m[k]);
            const float sp = dsig_(sg);
            const float spp = sp * (1.f - 2.f * sg);
            mb[k] += gam[k] * (gsh[k] * cv[k] + gs[k]) * spp + gcb[k] * gsh[k] * sp;
            ashb[k] = gam[k] * cv[k] * sp + gcb[k] * sg;
            asb[k] = gam[k] * sp;
          }
          smem_row_add<D>(s_ashb, ashb, lane);
          smem_row_add<D>(s_asb, asb, lane);
        }
        st_row<D, false>(a.Mbar + e * D, mb, lane);          // completed by sweep 2 (same warp, same lanes)
      }
    }
    // ---- node: the node-norm VJP, then Hbar, Shbar, Sbar ----
    {
      float xp[V], go[V], gam[V], xpb[V], gob[V], gxp[V];
      float r[V], hv[V], shb[V], sb[V];
      ld_row<D, false>(xp, a.XP + v * D, lane);
      ld_row<D, false>(go, a.gx_out + v * D, lane);
      ld_row<D, false>(r, a.S + v * D, lane);
      ld_row<D, false>(hv, a.H + v * D, lane);
      ld_row<D, false>(gam, a.GPbar + v * 4 * D + 3 * D, lane);
      ld_srow<D>(shb, s_ashb, lane);
      ld_srow<D>(sb, s_asb, lane);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        r[k] = 1.f / (r[k] + a.gate_eps);
        shb[k] = shb[k] - sb[k] * hv[k];                      // gShb - gSb H
        gam[k] += shb[k] * r[k];
      }
      ln_silu_vjp_row<D>(xp, go, gam, a.ln_eps, vec, vec + D, xpb, gob, gxp, acc + 2 * D, acc + 3 * D, lane);
      if (a.gx_bar_res) {
        float t[V];
        ld_row<D, false>(t, a.gx_bar_res + v * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) gob[k] += t[k];
      }
      st_row<D, false>(a.gx_out_bar + v * D, gob, lane);
      st_row<D, false>(a.Pbar + v * 4 * D + 3 * D, xpb, lane);
      smem_row_add<D>(acc + 4 * D, xpb, lane);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float hb = xpb[k] - sb[k] * gxp[k] * r[k];
        const float w = shb[k];
        shb[k] = hb * r[k];
        sb[k] = -hb * hv[k] * r[k] - w * gxp[k] * r[k] * r[k];
      }
      st_row<D, false>(a.Shbar + v * D, shb, lane);
      st_srow<D>(s_gsh, shb, lane);                        // the segment rows now hold Shbar, Sbar
      st_srow<D>(s_gs, sb, lane);
    }
    // ---- sweep 2: Mbar_e += (Shbar C[s] + Sbar) sg';  Pbar_B = sum_in Mbar ----
    float accB[V];
#pragma unroll
    for (int k = 0; k < V; ++k) accB[k] = 0.f;
    for (int base = p0; base < p1; base += 32) {
      const int cnt = min(32, p1 - base);
      int my_e = 0, my_s = 0;
      if (lane < cnt) {
        my_e = a.in_eid ? a.in_eid[base + lane] : base + lane;
        my_s = a.src[my_e];
      }
      for (int i = 0; i < cnt; ++i) {
        const int64_t e = __shfl_sync(0xffffffffu, my_e, i);
        const int64_t s = __shfl_sync(0xffffffffu, my_s, i);
        float m[V], cv[V], mb[V], shb[V], sb[V];
        ld_row<D, true>(m, a.M + e * D, lane);
        ld_row<D, false>(cv, a.P + s * 4 * D + D, lane);
        ld_row<D, true>(mb, a.Mbar + e * D, lane);     // written by sweep 1 of this kernel: no read-only (nc) path
        ld_srow<D>(shb, s_gsh, lane);
        ld_srow<D>(sb, s_gs, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          mb[k] += (shb[k] * cv[k] + sb[k]) * dsig_(sigmoidf_(m[k]));
          accB[k] += mb[k];
        }
        st_row<D, false>(a.Mbar + e * D, mb, lane);
      }
    }
    st_row<D, false>(a.Pbar + v * 4 * D + 2 * D, accB, lane);
    smem_row_add<D>(acc + 5 * D, accB, lane);
    __syncwarp();
  }
  __syncthreads();
  float* out_row = a.partials + (int64_t)blockIdx.x * 6 * D;   // fixed-order sum over the block's warps
  for (int i = threadIdx.x; i < 6 * D; i += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kWarpsPerBlock; ++w) t += sacc[w * 6 * D + i];
    out_row[i] = t;
  }
}

// Source-keyed pass (out-CSR), per node u (out-edges e, destinations t):
//   Pbar_A[u] = sum_out Mbar_e,   Pbar_C[u] = sum_out (Gamma_e gSh[t] sg' + Shbar[t] sg)
// partials row: {sum Pbar_A, sum Pbar_C}
template <int D>
__global__ void __launch_bounds__(kThreads)
egc_vjp_src_kernel(alignn_b200_egc_bwd_vjp_args a) {
  using C = RowCfg<D>;
  constexpr int V = C::VPL;
  __shared__ float red[kWarpsPerBlock * D];
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float acc[2][V];
#pragma unroll
  for (int k = 0; k < V; ++k) { acc[0][k] = 0.f; acc[1][k] = 0.f; }
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
      for (int i = 0; i < cnt; ++i) {
        const int64_t e = __shfl_sync(0xffffffffu, my_e, i);
        const int64_t t = __shfl_sync(0xffffffffu, my_t, i);
        float mb[V], gam[V], m[V], gsh[V], shb[V];
        ld_row<D, true>(mb, a.Mbar + e * D, lane);
        ld_row<D, true>(gam, a.Gamma + e * D, lane);
        ld_row<D, true>(m, a.M + e * D, lane);
        ld_row<D, false>(gsh, a.GSh + t * D, lane);
        ld_row<D, false>(shb, a.Shbar + t * D, lane);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float sg = sigmoidf_(m[k]);
          accA[k] += mb[k];
          accC[k] += gam[k] * gsh[k] * dsig_(sg) + shb[k] * sg;
        }
      }
    }
    st_row<D, false>(a.Pbar + u * 4 * D, accA, lane);
    st_row<D, false>(a.Pbar + u * 4 * D + D, accC, lane);
#pragma unroll
    for (int k = 0; k < V; ++k) { acc[0][k] += accA[k]; acc[1][k] += accC[k]; }
  }
  block_reduce_to_partials<D, 2>(acc, a.partials_src + (int64_t)blockIdx.x * 2 * D, red);
}

}  // namespace
}  // namespace alignn

extern "C" int alignn_b200_egc_backward_vjp(const alignn_b200_egc_bwd_vjp_args* a) {
  if (!a) return ALIGNN_ERR_BAD_ARG;
  if (a->struct_size != sizeof(*a)) return ALIGNN_ERR_STRUCT_SIZE;
  if (a->d != 32 && a->d != 64 && a->d != 128 && a->d != 256) return ALIGNN_ERR_UNSUPPORTED_D;
  if (a->norm != ALIGNN_NORM_LAYER) return ALIGNN_ERR_BAD_ARG;      // the BatchNorm double backward is not built
  if (a->Nn < 0 || a->Ne < 0) return ALIGNN_ERR_BAD_ARG;
  if (a->Nn == 0) return ALIGNN_OK;
  if (!a->P || !a->XP || !a->S || !a->H || !a->in_ptr || !a->out_ptr || !a->n_w || !a->n_b || !a->gx_out || !a->GSh ||
      !a->GPbar || !a->Pbar || !a->gx_out_bar || !a->Shbar || !a->partials || !a->partials_src)
    return ALIGNN_ERR_BAD_ARG;
  if (a->Ne > 0 && (!a->M || !a->src || !a->dst || !a->out_eid || !a->Mbar || !a->Gamma)) return ALIGNN_ERR_BAD_ARG;
  if (a->gy_out && (!a->e_w || !a->e_b || !a->gy_out_bar)) return ALIGNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)a->stream;
  const int grid = alignn_b200_egc_partial_rows(a->Nn, a->d);
  int rc = ALIGNN_OK;
  auto launch = [&](auto dc) -> int {
    constexpr int D = decltype(dc)::value;
    const size_t smem_bytes = (size_t)(4 + alignn::kWarpsPerBlock * 11) * D * sizeof(float);
    static alignn::DeviceOnce configured;
    int cfg_dev;
    if (configured.needed(&cfg_dev)) {
      cudaError_t e = cudaFuncSetAttribute(alignn::egc_vjp_dst_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem_bytes);
      if (e != cudaSuccess) return alignn::record_cuda_error((int)e);
      configured.done(cfg_dev);
    }
    alignn::egc_vjp_dst_kernel<D><<<grid, alignn::kThreads, smem_bytes, st>>>(*a);
    int r = alignn::check_launch();
    if (r != ALIGNN_OK) return r;
    alignn::egc_vjp_src_kernel<D><<<grid, alignn::kThreads, 0, st>>>(*a);
    return alignn::check_launch();
  };
  switch (a->d) {
    case 32: rc = launch(std::integral_constant<int, 32>{}); break;
    case 64: rc = launch(std::integral_constant<int, 64>{}); break;
    case 128: rc = launch(std::integral_constant<int, 128>{}); break;
    default: rc = launch(std::integral_constant<int, 256>{}); break;
  }
  return rc;
}
