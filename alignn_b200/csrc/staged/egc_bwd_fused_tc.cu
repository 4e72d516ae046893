// STAGED WORK (see egc_fused.h): backward edge side of EdgeGatedGraphConv for train-mode BatchNorm in one persistent
// wgmma kernel -- the per-edge part of egc_backward_dst_kernel fused with the data-gradient GEMM  gy = GM * W_eg.
//
//   gu_e  = gy_out_e * silu'(M_e * scale + shift) ;  xhat_e = (M_e - mean) * rstd                 (BatchNorm + SiLU backward)
//   gm0_e = scale * gu_e - scale * (c1 + xhat_e * c2)
//   sig_e = sigmoid(M_e) ;  gm_e = gm0_e + (GSh[dst_e] * P[src_e, d:2d] + GS[dst_e]) * sig_e * (1 - sig_e)   (gate backward)
//   GM = gm ;  gy = GM * W_eg (+ gy_out) ;  GPB_v = sum_{e -> v} gm_e ;  partials = column sums of gm
//
// Warp roles: warps 0-3 = MMA warpgroup (accumulator tile in scratch, acc_sm90.cuh); warps 4-7 = epilogue; warps 8-23 = PRODUCERS.  A producer thread owns
// one tile row and two 4-column fragments of every 128 x 32 chunk: it loads M, gy_out and the three gathered node-row
// slices (all L2 hits: the next tile's M / gy_out rows are bulk-prefetched into L2 one tile ahead), forms gm, stores it
// to GM and writes the bf16 hi/lo split of the same values into the operand planes -- the A operand never exists in
// HBM in converted form and GM is written exactly once.  The epilogue drains the accumulator (+ residual) as gemm_tc.cu does
// and then sums the tile's GM rows per destination segment (read back through L2: the producers fence once per tile
// before their last arrival).  Tiles are the segment-aligned tiles of the forward kernel, so the segment sums need no
// atomics and have a fixed order.
#include <atomic>

#include "../tc_common.cuh"
#include "acc_sm90.cuh"
#include "alignn_b200.h"
#include "egc_fused.h"

namespace alignn {
namespace fused { extern std::atomic<int> g_last_cuda_error; }
namespace fusedb {

constexpr int BM = ALIGNN_FUSED_TILE_ROWS;
constexpr int BK = 32;
constexpr int STAGES = 3;
constexpr int EPI_WARPS = 4;
constexpr int EPI_THREADS = 32 * EPI_WARPS;
constexpr int PROD_WARPS = 16;
constexpr int NF = 32 / PROD_WARPS;           // fragments per producer thread and chunk: 2
constexpr int THREADS = 32 * (4 + EPI_WARPS + PROD_WARPS);   // 768
constexpr uint32_t LBO = 128;
constexpr uint32_t SBO = (BK / 8) * 128;
constexpr int EPI_COLS = 128;
constexpr int EPI_STRIDE = EPI_COLS + 4;
constexpr int kSMs = 132;

template <int D>
struct Cfg {
  static constexpr int A_PLANE = BM * BK * 2;
  static constexpr int B_PLANE = D * BK * 2;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int PIPE_BYTES = STAGES * STAGE;
  static constexpr int EC = D < EPI_COLS ? D : EPI_COLS;
  static constexpr int EPI_OFF = PIPE_BYTES;                   // [EPI_WARPS][32][EPI_STRIDE] floats
  static constexpr int EPI_BYTES = EPI_WARPS * 32 * EPI_STRIDE * 4;
  static constexpr int STAT_OFF = EPI_OFF + EPI_BYTES;         // [EPI_WARPS][D] column sums of gm
  static constexpr int STAT_BYTES = EPI_WARPS * D * 4;
  static constexpr int VEC_OFF = STAT_OFF + STAT_BYTES;        // scale | shift | A | B (see gm_elem)
  static constexpr int VEC_BYTES = 4 * D * 4;
  static constexpr int SEG_OFF = VEC_OFF + VEC_BYTES;          // [BM + 1] segment starts, then [BM] edge ids of the rows
  static constexpr int SEG_BYTES = ((2 * BM + 1) * 4 + 15) / 16 * 16;
  static constexpr int BAR_OFF = SEG_OFF + SEG_BYTES;
  static constexpr int SMEM = BAR_OFF + 128;
  static_assert(SMEM <= 232448, "shared memory budget of one sm_90 CTA");
};

__host__ __device__ constexpr int plane_off(int r, int k) { return (r >> 3) * (int)SBO + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2; }

__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory"); }

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float dsilu_(float u) { const float s = sigmoidf_(u); return s * (1.f + u * (1.f - s)); }

// dL/dm of one element (train-mode BatchNorm on the edge side).  Per channel: w = scale, b = shift and the folded
// constants  A = w c1 - B mean,  B = w c2 rstd,  so that  w (c1 + xhat c2) = A + B m  with xhat = (m - mean) rstd.
// has_go == false: dead edge output, no norm term.
__device__ __forceinline__ float gm_elem(float m, float go, bool has_go, float cv, float gsh, float gs, float w, float b,
                                         float A, float B) {
  float gr = 0.f;
  if (has_go) gr = w * (go * dsilu_(m * w + b)) - (A + B * m);
  const float sg = sigmoidf_(m);
  return gr + (gsh * cv + gs) * sg * (1.f - sg);
}

template <int D>
__global__ void __launch_bounds__(THREADS, 1)
egc_backward_fused_kernel(const alignn_b200_egc_bwd_fused_args a, float* __restrict__ scratch_all) {
  using F = Cfg<D>;
  extern __shared__ __align__(128) uint8_t smem[];
  float* stat = reinterpret_cast<float*>(smem + F::STAT_OFF);
  float* vec = reinterpret_cast<float*>(smem + F::VEC_OFF);
  int* seg = reinterpret_cast<int*>(smem + F::SEG_OFF);
  int* erow = seg + BM + 1;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  uint64_t* empty = full + STAGES;
  uint64_t* tfull = empty + STAGES;
  uint64_t* tempty = tfull + 2;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int nk = D / BK;
  const int total = a.num_tiles;
  const int4* tiles = reinterpret_cast<const int4*>(a.tiles);    // {v0, nseg, p0, rows}

  // per-channel vectors for the producers (staged before the role split): scale, shift and the folded constants
  for (int i = tid; i < D; i += THREADS) {
    const float w = a.e_w ? a.e_w[i] : 0.f;
    const float B = a.e_w ? w * a.e_c2[i] * a.e_rstd[i] : 0.f;
    vec[i] = w;
    vec[D + i] = a.e_b ? a.e_b[i] : 0.f;
    vec[2 * D + i] = a.e_w ? w * a.e_c1[i] - B * a.e_mean[i] : 0.f;
    vec[3 * D + i] = B;
  }
  for (int i = tid; i < EPI_WARPS * D; i += THREADS) stat[i] = 0.f;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full[s], PROD_WARPS + 1); tc::mbar_init(&empty[s], 4); }
    for (int b = 0; b < 2; ++b) { tc::mbar_init(&tfull[b], 128); tc::mbar_init(&tempty[b], EPI_WARPS); }
    tc::mbar_fence_init();
  }
  __syncthreads();
  const uint32_t tmem = 0;                                  // accumulator "address": see acc_sm90.cuh
  float* const scr = scratch_all + (size_t)blockIdx.x * staged_acc::kRows * 2 * D;

  if (warp >= 4 + EPI_WARPS) {
    // ================= producers: gm per element -> GM (HBM) and bf16 hi/lo planes (smem) =================
    // Thread -> ONE tile row and two (4-column) fragments of every chunk: row = 8 * warp + ((lane >> 1) & 7),
    // float4 index kq_i = 4 i + 2 (lane >> 4) + (lane & 1).  A half-warp covers 8 rows x 2 adjacent float4 per
    // fragment: conflict-free 64-bit plane stores and full 32-byte sectors on every global access.
    // No register prefetch ring (the register budget of 21 warps is 80): the NEXT tile's M / gy_out rows are pulled
    // into L2 by bulk prefetches one tile ahead, so every load below is an L2 hit and the 4 warps per scheduler cover it.
    const int pt = tid - 32 * (4 + EPI_WARPS);          // 0..511
    const int pw = pt >> 5;
    const bool has_go = a.gy_out != nullptr;
    const int prow = pw * 8 + ((lane >> 1) & 7);
    int fkq[NF], soff[NF];
#pragma unroll
    for (int i = 0; i < NF; ++i) {
      fkq[i] = i * 4 + (lane >> 4) * 2 + (lane & 1);
      soff[i] = plane_off(prow, fkq[i] * 4);
    }
    const bool prefetcher = (lane & 17) == 0;            // one of the four threads that share the row
    const int my_tiles = (total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    int n_e = 0, n_s = 0, n_t = 0;
    bool n_v = false;
    auto fetch_row = [&](int tile) {                     // row metadata of `tile`, and its rows on their way into L2
      n_v = false;
      if (tile < total) {
        const int4 d4 = __ldg(tiles + tile);
        n_v = prow < d4.w;
        const int p = d4.z + prow;
        n_e = n_v ? (a.in_eid ? __ldg(a.in_eid + p) : p) : 0;
        n_s = n_v ? __ldg(a.src + n_e) : 0;
        n_t = n_v ? __ldg(a.dst + n_e) : 0;
        if (n_v && prefetcher) {
          tc::bulk_prefetch_l2(a.M + (int64_t)n_e * D, (uint32_t)D * 4u);
          if (has_go) tc::bulk_prefetch_l2(a.gy_out + (int64_t)n_e * D, (uint32_t)D * 4u);
        }
      }
    };
    fetch_row(blockIdx.x);
    int s = 0, ph = 0, c = 0;
    const uint8_t* wimg = reinterpret_cast<const uint8_t*>(a.w_image);
    for (int lt = 0; lt < my_tiles; ++lt) {
      const int tile = blockIdx.x + lt * gridDim.x;
      const bool valid = n_v;
      const int64_t e = n_e, sr = n_s, tr = n_t;
      fetch_row(tile + gridDim.x);
      const float* pm = a.M + e * D;
      const float* pg = has_go ? a.gy_out + e * D : nullptr;
      const float* pc = a.P + sr * 4 * D + D;
      const float* ph_ = a.GSh + tr * D;
      const float* ps = a.GS + tr * D;
      float* pgm = a.GM + e * D;
#pragma unroll 1
      for (int kc = 0; kc < nk; ++kc, ++c) {
        // all global loads of this chunk first (two fragments x five arrays), then the waits and the math
        float4 mm[NF], go[NF], cv[NF], gh[NF], gs[NF];
#pragma unroll
        for (int i = 0; i < NF; ++i) {
          const int col = kc * BK + fkq[i] * 4;
          const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
          mm[i] = valid ? __ldcs(reinterpret_cast<const float4*>(pm + col)) : z4;
          go[i] = (valid && has_go) ? __ldcs(reinterpret_cast<const float4*>(pg + col)) : z4;
          cv[i] = valid ? __ldg(reinterpret_cast<const float4*>(pc + col)) : z4;
          gh[i] = valid ? __ldg(reinterpret_cast<const float4*>(ph_ + col)) : z4;
          gs[i] = valid ? __ldg(reinterpret_cast<const float4*>(ps + col)) : z4;
        }
        if (c >= STAGES) tc::mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + s * F::STAGE;
        if (pt == 0) {   // weight chunk: one contiguous bulk copy (both planes), counted in bytes on full[s]
          tc::mbar_arrive_expect_tx(&full[s], 2 * F::B_PLANE);
          staged_acc::copy_weight_chunk<D, nk>(st + 2 * F::A_PLANE, wimg, kc, &full[s]);
        }
#pragma unroll
        for (int i = 0; i < NF; ++i) {
          const int col = kc * BK + fkq[i] * 4;
          const float4 w4 = *reinterpret_cast<const float4*>(vec + col);
          const float4 b4 = *reinterpret_cast<const float4*>(vec + D + col);
          const float4 A4 = *reinterpret_cast<const float4*>(vec + 2 * D + col);
          const float4 B4 = *reinterpret_cast<const float4*>(vec + 3 * D + col);
          float4 gm;
          gm.x = gm_elem(mm[i].x, go[i].x, has_go, cv[i].x, gh[i].x, gs[i].x, w4.x, b4.x, A4.x, B4.x);
          gm.y = gm_elem(mm[i].y, go[i].y, has_go, cv[i].y, gh[i].y, gs[i].y, w4.y, b4.y, A4.y, B4.y);
          gm.z = gm_elem(mm[i].z, go[i].z, has_go, cv[i].z, gh[i].z, gs[i].z, w4.z, b4.z, A4.z, B4.z);
          gm.w = gm_elem(mm[i].w, go[i].w, has_go, cv[i].w, gh[i].w, gs[i].w, w4.w, b4.w, A4.w, B4.w);
          if (!valid) gm = make_float4(0.f, 0.f, 0.f, 0.f);               // rows past the tile's end: zero operand rows
          else *reinterpret_cast<float4*>(pgm + col) = gm;
          uint2 hi, lo;
          tc::split4(gm, hi, lo);
          *reinterpret_cast<uint2*>(st + soff[i]) = hi;
          *reinterpret_cast<uint2*>(st + F::A_PLANE + soff[i]) = lo;
        }
        if (kc == nk - 1) __threadfence();          // this tile's GM rows are visible before the epilogue re-reads them
        tc::fence_async_smem();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&full[s]);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ================= epilogue: gy = acc (+ gy_out), then per-segment sums of the tile's GM rows =================
    const int q = warp & 3;
    const int et = q * 32 + lane;
    float* stg = reinterpret_cast<float*>(smem + F::EPI_OFF) + (warp - 4) * 32 * EPI_STRIDE;
    float* wstat = stat + (warp - 4) * D;
    int4 n_desc = make_int4(0, 0, 0, 0);
    int n_e = 0, n_seg = 0, n_seg_last = 0;
    auto fetch_meta = [&](int tile) {
      if (tile < total) {
        n_desc = __ldg(tiles + tile);
        const int p = n_desc.z + et;
        n_e = (et < n_desc.w) ? (a.in_eid ? __ldg(a.in_eid + p) : p) : 0;
        n_seg = (et <= n_desc.y) ? __ldg(a.in_ptr + n_desc.x + et) - n_desc.z : 0;
        n_seg_last = (et == 0 && n_desc.y == BM) ? __ldg(a.in_ptr + n_desc.x + BM) - n_desc.z : 0;
      }
    };
    fetch_meta(blockIdx.x);
    uint32_t lt = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x, ++lt) {
      const int acc = lt & 1;
      const int4 desc = n_desc;
      const int v0 = desc.x, nseg = desc.y, rows = desc.w;
      epi_bar();                                         // the previous tile's segment pass is done with seg[] / erow[]
      if (et <= nseg) seg[et] = n_seg;
      if (et == 0 && nseg == BM) seg[BM] = n_seg_last;
      erow[et] = n_e;
      fetch_meta(tile + gridDim.x);
      epi_bar();
      tc::mbar_wait(&tfull[acc], (lt >> 1) & 1);
            if (a.gy) {
        constexpr int EC = F::EC;
#pragma unroll 1
        for (int c0 = 0; c0 < D; c0 += EC) {
#pragma unroll 1
          for (int cc = 0; cc < EC; cc += 32) {
            float v[32];
            staged_acc::ld<32>(scr, 2 * D, tmem + ((uint32_t)(q * 32) << 16) + (uint32_t)(acc * D + c0 + cc), v);
#pragma unroll
            for (int j = 0; j < 32; j += 4)
              *reinterpret_cast<float4*>(stg + lane * EPI_STRIDE + cc + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
          }
          __syncwarp();
          constexpr int LPR = EC / 4;                        // lanes per row (float4 each)
          constexpr int RPI = 32 / LPR;                      // rows per store instruction
          const int c4 = (lane % LPR) * 4;
          const bool res = a.residual && a.gy_out;
          constexpr int RB = 8;
#pragma unroll 1
          for (int rb = 0; rb < 32; rb += RB * RPI) {
            float4 qv[RB];
#pragma unroll
            for (int u = 0; u < RB; ++u) {
              const int r = q * 32 + rb + u * RPI + lane / LPR;
              qv[u] = (res && r < rows) ? __ldcs(reinterpret_cast<const float4*>(a.gy_out + (int64_t)erow[r] * D + c0 + c4))
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < RB; ++u) {
              const int rl = rb + u * RPI + lane / LPR;
              const int r = q * 32 + rl;
              float4 o = *reinterpret_cast<const float4*>(stg + rl * EPI_STRIDE + c4);
              o.x += qv[u].x; o.y += qv[u].y; o.z += qv[u].z; o.w += qv[u].w;
              if (r < rows) *reinterpret_cast<float4*>(a.gy + (int64_t)erow[r] * D + c0 + c4) = o;
            }
          }
          __syncwarp();
        }
      }
      __threadfence_block();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&tempty[acc]);      // accumulator drained: the next tile's MMAs may start
      // ---- per-segment sums of this tile's GM rows (written by the producers, read back through L2) ----
      constexpr int VPL = D / 32;                          // values per lane, row spread over the warp
      constexpr int W = (D % 128 == 0) ? 4 : ((D % 64 == 0) ? 2 : 1);
      constexpr int CH = D / (32 * W);
      for (int j = warp - 4; j < nseg; j += EPI_WARPS) {
        float accb[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) accb[k] = 0.f;
        for (int r = seg[j]; r < seg[j + 1]; ++r) {
          const float* row = a.GM + (int64_t)erow[r] * D;
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const float* p = row + c * 32 * W + lane * W;
            if constexpr (W == 4) {
              const float4 t = __ldcg(reinterpret_cast<const float4*>(p));
              accb[c * 4] += t.x; accb[c * 4 + 1] += t.y; accb[c * 4 + 2] += t.z; accb[c * 4 + 3] += t.w;
            } else if constexpr (W == 2) {
              const float2 t = __ldcg(reinterpret_cast<const float2*>(p));
              accb[c * 2] += t.x; accb[c * 2 + 1] += t.y;
            } else {
              accb[c] += __ldcg(p);
            }
          }
        }
        float* out = a.GPB + (int64_t)(v0 + j) * a.ld_gpb;
#pragma unroll
        for (int c = 0; c < CH; ++c)
#pragma unroll
          for (int k = 0; k < W; ++k) {
            const int ch = c * 32 * W + lane * W + k;
            out[ch] = accb[c * W + k];
            wstat[ch] += accb[c * W + k];                  // each lane owns its channels of its warp's row: no conflicts
          }
      }
    }
    epi_bar();
    if (a.partials) {                                      // fixed-order sum over the four warps -> one partial row per CTA
      float* out_row = a.partials + (int64_t)blockIdx.x * D;
      for (int i = et; i < D; i += EPI_THREADS) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < EPI_WARPS; ++w) t += stat[w * D + i];
        out_row[i] = t;
      }
    }
  } else {
    // ================= MMA warpgroup (warps 0-3): the accumulator tile in scratch =================
    // 64-column blocks: 768 threads leave 80 registers per thread
    staged_acc::mma_warpgroup<D, F::STAGE, F::A_PLANE, STAGES, (D < 64 ? D : 64)>(smem, full, empty, tfull, tempty, scr, total);
  }
}

template <int D>
int launch(const alignn_b200_egc_bwd_fused_args& a) {
  using F = Cfg<D>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(egc_backward_fused_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM);
    if (e != cudaSuccess) { fused::g_last_cuda_error.store((int)e); return ALIGNN_ERR_CUDA; }
    configured = true;
  }
  const int grid = a.num_tiles < kSMs ? a.num_tiles : kSMs;
  cudaError_t se;
  float* scr = staged_acc::scratch((size_t)grid * staged_acc::kRows * 2 * D * sizeof(float), &se);
  if (!scr) { fused::g_last_cuda_error.store((int)se); return ALIGNN_ERR_CUDA; }
  egc_backward_fused_kernel<D><<<grid, THREADS, F::SMEM, (cudaStream_t)a.stream>>>(a, scr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { fused::g_last_cuda_error.store((int)e); return ALIGNN_ERR_CUDA; }
  return ALIGNN_OK;
}

}  // namespace fusedb
}  // namespace alignn

extern "C" int alignn_b200_egc_backward_fused(const alignn_b200_egc_bwd_fused_args* a) {
  if (!a) return ALIGNN_ERR_BAD_ARG;
  if (a->struct_size != sizeof(*a)) return ALIGNN_ERR_STRUCT_SIZE;
  if (a->d != 64 && a->d != 128 && a->d != 256) return ALIGNN_ERR_UNSUPPORTED_D;   // d = 32 keeps the two-kernel path
  if (a->Nn < 0 || a->Ne < 0 || a->num_tiles < 0) return ALIGNN_ERR_BAD_ARG;
  if (a->Nn == 0) return ALIGNN_OK;
  if (a->num_tiles == 0 || !a->tiles || !a->in_ptr || !a->w_image || !a->GPB || a->ld_gpb < a->d) return ALIGNN_ERR_BAD_ARG;
  if (a->Ne > 0 && (!a->M || !a->P || !a->GSh || !a->GS || !a->src || !a->dst || !a->GM)) return ALIGNN_ERR_BAD_ARG;
  if (a->gy_out && (!a->e_w || !a->e_b || !a->e_mean || !a->e_rstd || !a->e_c1 || !a->e_c2)) return ALIGNN_ERR_BAD_ARG;
  if (((uintptr_t)a->tiles & 15) != 0) return ALIGNN_ERR_BAD_ARG;
  switch (a->d) {
    case 256: return alignn::fusedb::launch<256>(*a);
    case 128: return alignn::fusedb::launch<128>(*a);
    default: return alignn::fusedb::launch<64>(*a);
  }
}
