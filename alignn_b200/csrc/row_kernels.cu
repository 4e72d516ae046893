// Row-wise kernels around the conv stack, fp32, sm_90a (HBM-bound: every row is read once and written once,
// one warp per row, 512 contiguous bytes per warp instruction -- common.cuh).
//
//   ln_silu_forward / ln_silu_backward: the LayerNorm -> SiLU tail of the embedding layers of the LayerNorm model
//     (Linear -> LayerNorm -> SiLU, alignn/models/alignn_atomwise.py:249-268 `MLPLayer`), applied to the output of the
//     tensor-core Linear.  T = 276 480 angle rows per batch go through two of these layers (alignn_atomwise.py:315-329).
//   adamw_flat: torch.optim.AdamW's update (the optimizer alignn/train.py:253-263 builds by default) over ONE flat fp32
//     parameter / gradient / moment buffer, step count on the device so that the launch can be replayed inside a CUDA
//     graph.
#include <atomic>
#include "common.cuh"
#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {

// out[r] = silu(LayerNorm(h[r]) * gamma + beta); rowstat[r] = {mean, rstd}
template <int D>
__global__ void __launch_bounds__(kThreads)
ln_silu_forward_kernel(const float* __restrict__ h, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                       int64_t n, float* __restrict__ out, float2* __restrict__ rowstat) {
  constexpr int V = RowCfg<D>::VPL;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float w[V], b[V];
  ld_vec<D>(w, gamma, lane); ld_vec<D>(b, beta, lane);
  for (int64_t r = warp0; r < n; r += 2 * nwarps) {      // two rows in flight per warp
    const int64_t r2 = r + nwarps;
    const bool has2 = r2 < n;
    float v[V], v2[V];
    ld_row<D, true>(v, h + r * D, lane);
    if (has2) ld_row<D, true>(v2, h + r2 * D, lane);
    float mean, rstd;
    row_mean_rstd<D>(v, eps, mean, rstd);
#pragma unroll
    for (int k = 0; k < V; ++k) v[k] = silu_((v[k] - mean) * rstd * w[k] + b[k]);
    st_row<D, true>(out + r * D, v, lane);
    if (lane == 0) rowstat[r] = make_float2(mean, rstd);
    if (has2) {
      row_mean_rstd<D>(v2, eps, mean, rstd);
#pragma unroll
      for (int k = 0; k < V; ++k) v2[k] = silu_((v2[k] - mean) * rstd * w[k] + b[k]);
      st_row<D, true>(out + r2 * D, v2, lane);
      if (lane == 0) rowstat[r2] = make_float2(mean, rstd);
    }
  }
}

// gh[r] = rstd * (gx - mean_c(gx) - xhat * mean_c(gx * xhat)),  gx = g_out * silu'(u) * gamma,  u = xhat * gamma + beta;
// partials[block] = {sum_r g_out silu'(u) xhat  (-> d gamma),  sum_r g_out silu'(u)  (-> d beta)}
template <int D>
__global__ void __launch_bounds__(kThreads, 2)
ln_silu_backward_kernel(const float* __restrict__ h, const float* __restrict__ g_out, const float2* __restrict__ rowstat,
                        const float* __restrict__ gamma, const float* __restrict__ beta, int64_t n, float* __restrict__ gh,
                        float* __restrict__ partials, int partial_rows_total) {
  constexpr int V = RowCfg<D>::VPL;
  __shared__ float red[kWarpsPerBlock * D];
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  float w[V], b[V], acc[2][V];
  ld_vec<D>(w, gamma, lane); ld_vec<D>(b, beta, lane);
#pragma unroll
  for (int k = 0; k < V; ++k) { acc[0][k] = 0.f; acc[1][k] = 0.f; }
  auto one_row = [&](int64_t r, float (&v)[V], float (&g)[V]) {
    const float2 st = __ldg(rowstat + r);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float xh = (v[k] - st.x) * st.y;
      const float gu = g[k] * dsilu_(xh * w[k] + b[k]);
      acc[0][k] += gu * xh;
      acc[1][k] += gu;
      const float gx = gu * w[k];
      v[k] = xh; g[k] = gx;
      s1 += gx; s2 += gx * xh;
    }
    s1 = warp_sum(s1) * (1.f / D);
    s2 = warp_sum(s2) * (1.f / D);
#pragma unroll
    for (int k = 0; k < V; ++k) g[k] = st.y * (g[k] - s1 - v[k] * s2);
    st_row<D, true>(gh + r * D, g, lane);
  };
  for (int64_t r = warp0; r < n; r += 2 * nwarps) {        // two rows (four row loads) in flight per warp
    const int64_t r2 = r + nwarps;
    const bool has2 = r2 < n;
    float v[V], g[V], v2[V], g2[V];
    ld_row<D, true>(v, h + r * D, lane);
    ld_row<D, true>(g, g_out + r * D, lane);
    if (has2) {
      ld_row<D, true>(v2, h + r2 * D, lane);
      ld_row<D, true>(g2, g_out + r2 * D, lane);
    }
    one_row(r, v, g);
    if (has2) one_row(r2, v2, g2);
  }
  block_reduce_to_partials<D, 2>(acc, partials + (int64_t)blockIdx.x * 2 * D, red);
  const int extra = blockIdx.x + gridDim.x;                // rows [gridDim.x, partial_rows_total) belong to no block
  if (extra < partial_rows_total)
    for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) partials[(int64_t)extra * 2 * D + i] = 0.f;
}

// torch.optim.AdamW (amsgrad = False, maximize = False), element by element:
//   p *= 1 - lr * wd;  m += (1 - b1) (g - m);  v = b2 v + (1 - b2) g^2;  p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// t = *step + 1; the last block to finish stores t back (integer ticket: no float atomics, deterministic).
__global__ void __launch_bounds__(256)
adamw_flat_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n4,
                  int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int zero_grad,
                  int64_t* __restrict__ step, unsigned int* __restrict__ ticket) {
  const int64_t t = *reinterpret_cast<volatile int64_t*>(step) + 1;
  const double bc1 = 1.0 - pow((double)beta1, (double)t), bc2 = 1.0 - pow((double)beta2, (double)t);
  const float step_size = (float)((double)lr / bc1);
  const float inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
  const float decay = 1.f - lr * weight_decay;
  const float omb1 = 1.f - beta1, omb2 = 1.f - beta2;
  auto upd = [&](float& pp, float gg, float& mm, float& vv) {
    pp *= decay;
    mm += omb1 * (gg - mm);
    vv = beta2 * vv + omb2 * gg * gg;
    pp -= step_size * mm / (sqrtf(vv) * inv_sqrt_bc2 + eps);
  };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 P = reinterpret_cast<float4*>(p)[i], G = __ldcs(reinterpret_cast<const float4*>(g) + i);
    float4 M = reinterpret_cast<float4*>(m)[i], Vv = reinterpret_cast<float4*>(v)[i];
    upd(P.x, G.x, M.x, Vv.x); upd(P.y, G.y, M.y, Vv.y); upd(P.z, G.z, M.z, Vv.z); upd(P.w, G.w, M.w, Vv.w);
    reinterpret_cast<float4*>(p)[i] = P; reinterpret_cast<float4*>(m)[i] = M; reinterpret_cast<float4*>(v)[i] = Vv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (blockIdx.x == 0)
    for (int64_t i = 4 * n4 + threadIdx.x; i < n; i += blockDim.x) {      // tail when n is not a multiple of 4
      upd(p[i], g[i], m[i], v[i]);
      if (zero_grad) g[i] = 0.f;
    }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) { *step = t; *ticket = 0u; __threadfence(); }
  }
}

}  // namespace alignn

namespace {
inline bool supported_d(int d) { return d == 32 || d == 64 || d == 128 || d == 256; }
inline int rows_grid(int64_t n) {
  int64_t b = (n + alignn::kWarpsPerBlock - 1) / alignn::kWarpsPerBlock;
  if (b < 1) b = 1;
  if (b > alignn::kMaxBlocks) b = alignn::kMaxBlocks;
  return (int)b;
}
}  // namespace

#define ROW_DISPATCH_D(d, ...)                     \
  switch (d) {                                     \
    case 32: { constexpr int D = 32; __VA_ARGS__; break; }   \
    case 64: { constexpr int D = 64; __VA_ARGS__; break; }   \
    case 128: { constexpr int D = 128; __VA_ARGS__; break; } \
    case 256: { constexpr int D = 256; __VA_ARGS__; break; } \
    default: return ALIGNN_ERR_UNSUPPORTED_D;      \
  }

extern "C" {

int alignn_b200_ln_silu_forward(const float* h, const float* gamma, const float* beta, float eps, int64_t n, int d, float* out,
                                float* rowstat, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n < 0 || (n > 0 && (!h || !gamma || !beta || !out || !rowstat))) return ALIGNN_ERR_BAD_ARG;
  if (n == 0) return ALIGNN_OK;
  ROW_DISPATCH_D(d, {
    const int grid = alignn::one_wave_grid((const void*)alignn::ln_silu_forward_kernel<D>, alignn::kThreads, 0, rows_grid(n));
    alignn::ln_silu_forward_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(h, gamma, beta, eps, n, out,
                                                                                         reinterpret_cast<float2*>(rowstat));
  });
  return alignn::check_launch();
}

int alignn_b200_ln_silu_backward(const float* h, const float* g_out, const float* rowstat, const float* gamma, const float* beta,
                                 int64_t n, int d, float* gh, float* partials, int partial_rows, alignn_stream_t stream) {
  if (!supported_d(d)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n < 0 || (n > 0 && (!h || !g_out || !rowstat || !gamma || !beta || !gh || !partials))) return ALIGNN_ERR_BAD_ARG;
  if (n == 0) return ALIGNN_OK;
  if (partial_rows != rows_grid(n)) return ALIGNN_ERR_WORKSPACE;
  ROW_DISPATCH_D(d, {
    const int grid = alignn::one_wave_grid((const void*)alignn::ln_silu_backward_kernel<D>, alignn::kThreads, 0, partial_rows);
    if (2 * grid < partial_rows) return ALIGNN_ERR_CUDA;
    alignn::ln_silu_backward_kernel<D><<<grid, alignn::kThreads, 0, (cudaStream_t)stream>>>(
        h, g_out, reinterpret_cast<const float2*>(rowstat), gamma, beta, n, gh, partials, partial_rows);
  });
  return alignn::check_launch();
}

int alignn_b200_adamw_flat(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1,
                           float beta2, float eps, float weight_decay, int zero_grad, int64_t* step, uint32_t* ticket,
                           alignn_stream_t stream) {
  if (n < 0 || (n > 0 && (!param || !grad || !exp_avg || !exp_avg_sq)) || !step || !ticket) return ALIGNN_ERR_BAD_ARG;
  if (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) return ALIGNN_ERR_BAD_ARG;
  const int64_t n4 = n / 4;
  int64_t blocks = (n4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > alignn::kNumSMs * 8) blocks = alignn::kNumSMs * 8;
  alignn::adamw_flat_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, n4, n, lr, beta1,
                                                                          beta2, eps, weight_decay, zero_grad, step, ticket);
  return alignn::check_launch();
}

}  // extern "C"
