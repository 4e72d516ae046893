// Shared device helpers for the edge-gated conv kernels (sm_90a).
//
// Row-per-warp layout: a feature row of D floats is spread over the 32 lanes of a warp,
// lane l holding CH vectors of W floats: channels  c*32*W + l*W + j  (c < CH, j < W).
// Every warp-wide access to a row is one or two fully coalesced 128-bit transactions per lane
// (512 contiguous bytes per instruction for W == 4), which is what makes the row gathers by
// sorted-CSR edge index run at HBM/L2 line rate.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace alignn {

constexpr int kWarpsPerBlock = 8;
constexpr int kThreads = kWarpsPerBlock * 32;
constexpr int kNumSMs = 132;                       // H100 SXM
constexpr int kMaxBlocks = kNumSMs * 4;            // rows of per-block partials are bounded by this

template <int D>
struct RowCfg {
  static_assert(D % 32 == 0, "feature width must be a multiple of the warp size");
  static constexpr int W = (D % 128 == 0) ? 4 : ((D % 64 == 0) ? 2 : 1);
  static constexpr int CH = D / (32 * W);
  static constexpr int VPL = D / 32;               // values per lane
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- row loads / stores --------------------------------------------------------------------
// kStream = true: data touched once (edge rows) -> evict-first (ld.global.cs / st.global.cs);
// false: gathered node rows that are re-read by other edges -> default caching (L1+L2).
template <int D, bool kStream>
__device__ __forceinline__ void ld_row(float (&v)[RowCfg<D>::VPL], const float* __restrict__ row, int lane) {
  using C = RowCfg<D>;
#pragma unroll
  for (int c = 0; c < C::CH; ++c) {
    const float* p = row + c * 32 * C::W + lane * C::W;
    if constexpr (C::W == 4) {
      float4 t = kStream ? __ldcs(reinterpret_cast<const float4*>(p)) : __ldg(reinterpret_cast<const float4*>(p));
      v[c * 4 + 0] = t.x; v[c * 4 + 1] = t.y; v[c * 4 + 2] = t.z; v[c * 4 + 3] = t.w;
    } else if constexpr (C::W == 2) {
      float2 t = kStream ? __ldcs(reinterpret_cast<const float2*>(p)) : __ldg(reinterpret_cast<const float2*>(p));
      v[c * 2 + 0] = t.x; v[c * 2 + 1] = t.y;
    } else {
      v[c] = kStream ? __ldcs(p) : __ldg(p);
    }
  }
}

template <int D, bool kStream>
__device__ __forceinline__ void st_row(float* __restrict__ row, const float (&v)[RowCfg<D>::VPL], int lane) {
  using C = RowCfg<D>;
#pragma unroll
  for (int c = 0; c < C::CH; ++c) {
    float* p = row + c * 32 * C::W + lane * C::W;
    if constexpr (C::W == 4) {
      float4 t = make_float4(v[c * 4 + 0], v[c * 4 + 1], v[c * 4 + 2], v[c * 4 + 3]);
      if (kStream) __stcs(reinterpret_cast<float4*>(p), t); else *reinterpret_cast<float4*>(p) = t;
    } else if constexpr (C::W == 2) {
      float2 t = make_float2(v[c * 2 + 0], v[c * 2 + 1]);
      if (kStream) __stcs(reinterpret_cast<float2*>(p), t); else *reinterpret_cast<float2*>(p) = t;
    } else {
      if (kStream) __stcs(p, v[c]); else *p = v[c];
    }
  }
}

// per-channel parameter vector in the same lane layout (tiny, L1/L2 resident)
template <int D>
__device__ __forceinline__ void ld_vec(float (&v)[RowCfg<D>::VPL], const float* __restrict__ p, int lane) {
  if (p) ld_row<D, false>(v, p, lane);
  else {
#pragma unroll
    for (int i = 0; i < RowCfg<D>::VPL; ++i) v[i] = 0.f;
  }
}

// sigmoid in four instructions (FMUL, MUFU.EX2, FADD, MUFU.RCP; <= 2 ulp) instead of ~25 with an IEEE division and the
// denormal paths of the non-ftz approximations: the edge kernels are bound by instruction issue at 4 warps per
// scheduler, not by HBM.  exp(-x) underflowing to 0 and overflowing to +inf give
// exactly 1 and 0.
__device__ __forceinline__ float sigmoidf_(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return r;
}
// u = pre-activation after the norm; silu(u) and its derivative
__device__ __forceinline__ float silu_(float u) { return u * sigmoidf_(u); }
__device__ __forceinline__ float dsilu_(float u) { float s = sigmoidf_(u); return s * (1.f + u * (1.f - s)); }

// mean and reciprocal std of a row held across the warp (two-pass, like torch's LayerNorm)
template <int D>
__device__ __forceinline__ void row_mean_rstd(const float (&v)[RowCfg<D>::VPL], float eps, float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < RowCfg<D>::VPL; ++i) s += v[i];
  mean = warp_sum(s) * (1.f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < RowCfg<D>::VPL; ++i) { float t = v[i] - mean; q += t * t; }
  rstd = rsqrtf(warp_sum(q) * (1.f / D) + eps);
}

// row held in SHARED memory (per-channel parameter vectors staged once per block) -> lane layout
template <int D>
__device__ __forceinline__ void ld_srow(float (&v)[RowCfg<D>::VPL], const float* __restrict__ row, int lane) {
  using C = RowCfg<D>;
#pragma unroll
  for (int c = 0; c < C::CH; ++c) {
    const float* p = row + c * 32 * C::W + lane * C::W;
    if constexpr (C::W == 4) {
      const float4 t = *reinterpret_cast<const float4*>(p);
      v[c * 4 + 0] = t.x; v[c * 4 + 1] = t.y; v[c * 4 + 2] = t.z; v[c * 4 + 3] = t.w;
    } else if constexpr (C::W == 2) {
      const float2 t = *reinterpret_cast<const float2*>(p);
      v[c * 2 + 0] = t.x; v[c * 2 + 1] = t.y;
    } else {
      v[c] = *p;
    }
  }
}

// acc[lane layout] += v, for per-warp accumulator rows kept in shared memory (frees registers in the
// big backward kernel).  Each lane only ever touches its own channels: no conflicts, no atomics.
template <int D>
__device__ __forceinline__ void smem_row_add(float* __restrict__ acc_row, const float (&v)[RowCfg<D>::VPL], int lane) {
  using C = RowCfg<D>;
#pragma unroll
  for (int c = 0; c < C::CH; ++c) {
    float* p = acc_row + c * 32 * C::W + lane * C::W;
    if constexpr (C::W == 4) {
      float4 t = *reinterpret_cast<float4*>(p);
      t.x += v[c * 4 + 0]; t.y += v[c * 4 + 1]; t.z += v[c * 4 + 2]; t.w += v[c * 4 + 3];
      *reinterpret_cast<float4*>(p) = t;
    } else if constexpr (C::W == 2) {
      float2 t = *reinterpret_cast<float2*>(p);
      t.x += v[c * 2 + 0]; t.y += v[c * 2 + 1];
      *reinterpret_cast<float2*>(p) = t;
    } else {
      *p += v[c];
    }
  }
}

// Sum the per-warp accumulators of a block in a fixed order and write one partial row.
// acc: NQ quantities of VPL per lane.  out row layout: [NQ][D].  smem: [kWarpsPerBlock][D].
template <int D, int NQ>
__device__ __forceinline__ void block_reduce_to_partials(const float (&acc)[NQ][RowCfg<D>::VPL], float* __restrict__ out_row,
                                                         float* smem) {
  using C = RowCfg<D>;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
#pragma unroll
    for (int c = 0; c < C::CH; ++c)
#pragma unroll
      for (int j = 0; j < C::W; ++j)
        smem[warp * D + c * 32 * C::W + lane * C::W + j] = acc[q][c * C::W + j];
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kWarpsPerBlock; ++w) s += smem[w * D + i];
      out_row[q * D + i] = s;
    }
    __syncthreads();
  }
}

}  // namespace alignn
