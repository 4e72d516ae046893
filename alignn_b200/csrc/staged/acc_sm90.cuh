// The accumulator of the staged kernels on sm_90.  The kernels were written around a [128 x 2D] fp32 accumulator (two
// tile buffers) that the epilogue reads row by row; on Hopper the 128 x 256 tile does not fit next to the pipeline in
// registers or shared memory, so it lives in a per-CTA scratch tile in global memory (L2-resident):
//   element (row, column) at scr[row * 2D + column],  "address" = (first row << 16) | column.
// One warpgroup computes it with wgmma, chunk by chunk, in 64-row x BN-column blocks, reloading the block's partial sums
// between chunks.  With BN = min(D, 128), the column tile of gemm_tc.cu, the MMAs and their order (lo*hi, hi*lo, hi*hi
// per K = 16 step, starting from zero) are those of gemm_tc.cu, so the accumulators are bit-identical to the shipped GEMM.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../tc_common.cuh"

namespace alignn {
namespace staged_acc {

constexpr int kRows = 128;

// one warp: rows (taddr >> 16) + lane, columns (taddr & 0xffff) .. + N
template <int N>
__device__ __forceinline__ void ld(const float* scr, int ld_cols, uint32_t taddr, float (&v)[N]) {
  const int row = (int)(taddr >> 16) + (threadIdx.x & 31), col = (int)(taddr & 0xffffu);
  const float4* p = reinterpret_cast<const float4*>(scr + (size_t)row * ld_cols + col);
#pragma unroll
  for (int i = 0; i < N / 4; ++i) {
    const float4 x = __ldcg(p + i);
    v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
  }
}
template <int N>
__device__ __forceinline__ void st(float* scr, int ld_cols, uint32_t taddr, const float (&v)[N]) {
  const int row = (int)(taddr >> 16) + (threadIdx.x & 31), col = (int)(taddr & 0xffffu);
  float4* p = reinterpret_cast<float4*>(scr + (size_t)row * ld_cols + col);
#pragma unroll
  for (int i = 0; i < N / 4; ++i) __stcg(p + i, make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]));
}

// Warpgroup (threads 0..127 of the CTA).  Stage s of the ring: A planes [hi, lo][128 x 32] at s * STAGE, then the weight
// chunk as D / min(D, 128) column tiles of [hi, lo][BN x 32] (K-major core-matrix order, LBO = 128, SBO = 512).  Per tile:
// waits until the epilogue released accumulator buffer lt & 1, accumulates all D / 32 chunks, arrives on tfull (count
// 128: every thread releases its own stores).
template <int D, int STAGE, int A_PLANE, int STAGES, int BN = (D < 128 ? D : 128)>
__device__ __forceinline__ void mma_warpgroup(uint8_t* smem, uint64_t* full, uint64_t* empty, uint64_t* tfull, uint64_t* tempty,
                                              float* scr, int total) {
  constexpr int IBN = D < 128 ? D : 128, WBP = IBN * 32 * 2, NK = D / 32;   // column tile of the weight image
  constexpr uint32_t LBO = 128, SBO = 512;
  static_assert(IBN % BN == 0, "MMA blocks inside one image tile");
  const int t = threadIdx.x, w = t >> 5, lane = t & 31;
  const uint32_t base = tc::smem_u32(smem);
  uint32_t lt = 0;
  int s = 0, ph = 0;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x, ++lt) {
    const int acc = lt & 1;
    if (lt >= 2) tc::mbar_wait(&tempty[acc], ((lt >> 1) - 1) & 1);
    for (int kc = 0; kc < NK; ++kc) {
      tc::mbar_wait(&full[s], ph);
      const uint32_t sa = base + s * STAGE;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
#pragma unroll 1
        for (int cb = 0; cb < D / BN; ++cb) {
          float r[BN / 2];
          float* p = scr + (size_t)(h * 64 + w * 16 + (lane >> 2)) * (2 * D) + acc * D + cb * BN + 2 * (lane & 3);
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2) {    // r[4j + 2hh + e] = (row + 8 hh, column 8 j + e)
            const float2 x = kc ? __ldcg(reinterpret_cast<const float2*>(p + ((i >> 1) & 1) * 8 * (2 * D) + 8 * (i >> 2)))
                                : make_float2(0.f, 0.f);
            r[i] = x.x; r[i + 1] = x.y;
          }
          tc::wgmma_fence();
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint32_t a_hi = sa + h * 8 * SBO + j * 2 * LBO;
            const uint32_t b_hi = sa + 2 * A_PLANE + (cb * BN / IBN) * 2 * WBP + ((cb * BN) % IBN) / 8 * SBO + j * 2 * LBO;
            const uint64_t dah = tc::smem_desc(a_hi, LBO, SBO), dal = tc::smem_desc(a_hi + A_PLANE, LBO, SBO);
            const uint64_t dbh = tc::smem_desc(b_hi, LBO, SBO), dbl = tc::smem_desc(b_hi + WBP, LBO, SBO);
            tc::Wgmma<BN>::template mma<0, 0>(r, dal, dbh, 1);   // same order as gemm_tc.cu
            tc::Wgmma<BN>::template mma<0, 0>(r, dah, dbl, 1);
            tc::Wgmma<BN>::template mma<0, 0>(r, dah, dbh, 1);
          }
          tc::wgmma_commit();
          tc::wgmma_wait_all();
#pragma unroll
          for (int i = 0; i < BN / 2; i += 2)
            __stcg(reinterpret_cast<float2*>(p + ((i >> 1) & 1) * 8 * (2 * D) + 8 * (i >> 2)), make_float2(r[i], r[i + 1]));
        }
      }
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&empty[s]);           // count: the four warps of the group
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    __threadfence_block();
    tc::mbar_arrive(&tfull[acc]);
  }
}

// weight chunk kc of an image with D columns (gemm_prepare_table layout, column tiles of BN) -> the stage's B region
template <int D, int NK>
__device__ __forceinline__ void copy_weight_chunk(uint8_t* dst, const uint8_t* wimg, int kc, uint64_t* bar) {
  constexpr int BN = D < 128 ? D : 128, WBP = BN * 32 * 2;
#pragma unroll
  for (int nt = 0; nt < D / BN; ++nt)
    tc::bulk_g2s(dst + nt * 2 * WBP, wimg + ((int64_t)nt * NK + kc) * 2 * WBP, 2 * WBP, bar);
}

// Scratch for the accumulators, shared by the staged kernels of this process (grown on demand; not graph-capturable).
inline float* scratch(size_t bytes, cudaError_t* err) {
  static float* buf = nullptr;
  static size_t cap = 0;
  *err = cudaSuccess;
  if (bytes > cap) {
    if (buf) cudaFree(buf);
    buf = nullptr;
    cap = 0;
    *err = cudaMalloc(&buf, bytes);
    if (*err != cudaSuccess) return nullptr;
    cap = bytes;
  }
  return buf;
}

}  // namespace staged_acc
}  // namespace alignn
