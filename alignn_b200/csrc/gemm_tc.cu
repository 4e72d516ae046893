// Linear layers in fp32 parity on the Hopper tensor cores: wgmma (bf16 x bf16 -> fp32 in registers) with the bf16x3
// operand split (tc_common.cuh).
//
//   C[r, :] = A[r, :] * W^T (+ bias) (+ add0[i0(r), :]) (+ add1[i1(r), :])                                  r < M
//   stats[cta][0/1][c] = partial sums over the CTA's tiles of C[r, c] and C[r, c]^2                         (optional)
//
// gemm_nt is the plain form (add0 = the residual, no index).  gemm_gather is the edge-gate kernel of the conv path: with
// A = edge features y, add0 = P[src, 0:d] (e_src), add1 = P[dst, 2d:3d] (e_dst + both biases) it is the pre-activation
// gate  m = e_src[src] + e_dst[dst] + edge_gate(y)  of alignn/models/alignn.py:98-101 in ONE pass over y, plus the
// per-channel batch statistics BatchNorm1d(m) needs (alignn.py:123).  With add0 = the incoming gradient it is the
// data-gradient GEMM of the backward (residual in the epilogue).
//
// A is the fp32 activation matrix, read once per column tile: the producer warps copy its K-chunks global -> shared with
// cp.async into a ring of fp32 stages (the bytes in flight are set by shared memory, not by registers) and split them
// into the bf16 hi/lo planes of a ring of plane stages.  W is pre-split once per step into an image that already has the
// GMMA core-matrix order (gemm_prepare_table), so a K-chunk of it is ONE contiguous bulk copy (cp.async.bulk) signalled
// on the plane stage's mbarrier.
//
// Persistent, warp-specialised CTA (one per SM), 128 x BN output tiles, BN <= 128, three warpgroups:
//   warps 0-3, 4-7 : two consumer warpgroups, ping-pong: local tile i of the CTA belongs to warpgroup i % 2, which runs
//                    both m64 row halves of it (wgmma m64nBNk16, BN accumulator registers per thread) and then its
//                    epilogue -- while one warpgroup is in its epilogue the other runs the MMAs of the next tile
//   warps 8-11     : producer: cp.async of A, fp32 -> bf16 hi/lo split, bulk copy of W
// setmaxnreg moves registers from the producer to the consumers.  The chunks of consecutive tiles pass through the
// stage ring in tile order, and a consumer starts the mainloop of local tile i only once the other one has issued the
// MMAs of tile i - 1's last chunk: the MMAs of the two warpgroups do not interleave, and a consumer never waits on a
// stage barrier more than one phase ahead of it (an mbarrier parity wait cannot tell phase k from phase k + 2).
// Mainloop: one wgmma group stays in flight; a stage is released once the MMAs of the next chunk have been issued.
// Epilogue: the wgmma fragment of one consumer warp is 16 whole rows of each row half, so each warp stages its own rows
// through a private shared-memory tile (no block barrier), one half after the other, and then works row by row: a row is
// BN / 4 lanes with one float4 each, the addend rows of several rows are loaded before the first store, and C is written
// as contiguous row segments.  The addend rows are read through __restrict__ pointers: C must not overlap A, add0, add1
// or the bias.
#include "common.cuh"
#include "tc_common.cuh"
#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace gemm {

constexpr int BM = 128;       // rows per tile (two m64 warpgroup MMAs)
constexpr int BK = 32;        // K per pipeline stage (2 MMA K=16 steps)
constexpr int STAGES = 2;     // bf16 hi/lo plane stages (producer -> MMAs)
constexpr int FSTAGES = 4;    // fp32 stages of A (cp.async -> producer): up to 64 KB in flight per CTA
constexpr int MMA_WARPS = 8;  // two consumer warpgroups
constexpr int LOAD_WARPS = 4; // one producer warpgroup
constexpr int THREADS = 32 * (MMA_WARPS + LOAD_WARPS);   // 384
constexpr int LOAD_REGS = 40, MMA_REGS = 232;            // setmaxnreg: 128 x 40 + 256 x 232 <= 64 K registers
static_assert(128 * LOAD_REGS + 256 * MMA_REGS <= 65536, "register file of one SM");
constexpr uint32_t LBO = 128;               // next 8-element K chunk
constexpr uint32_t SBO = (BK / 8) * 128;    // next 8-row group (chunk-local image): 512 B
constexpr int kMaxStatN = 256;              // widest output with column statistics
constexpr int WARP_ROWS = 16;               // tile rows of one consumer warp's wgmma fragment (per row half)
constexpr int STAT_ROWS = 8;                // column partials: one per (row half, warp of the warpgroup)

template <int BN>
struct Cfg {
  static constexpr int A_PLANE = BM * BK * 2;   // bytes of one bf16 plane of the A chunk
  static constexpr int B_PLANE = BN * BK * 2;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int PIPE_BYTES = STAGES * STAGE;
  // fp32 stage: 128 rows x 128 bytes, 32 rows (4 KB) per producer warp
  static constexpr int FSTAGE = BM * BK * 4;
  static constexpr int FP_OFF = PIPE_BYTES;
  // accumulator staging, fp32, 16 rows per consumer warp, rows padded by 8 floats: the fragment stores (8 rows x 4 lane
  // pairs per instruction) then fill all 32 banks twice, the minimum for 256 bytes
  static constexpr int PITCH = BN + 8;
  static constexpr int STG_OFF = FP_OFF + FSTAGES * FSTAGE;
  static constexpr int STG_BYTES = MMA_WARPS * WARP_ROWS * PITCH * 4;
  static constexpr int STAT_OFF = STG_OFF + STG_BYTES;
  static constexpr int STAT_BYTES = STAT_ROWS * 2 * kMaxStatN * 4;   // [STAT_ROWS][2][N] column partials
  static constexpr int BAR_OFF = STAT_OFF + STAT_BYTES;
  static constexpr int SMEM = BAR_OFF + 128;
  static_assert(SMEM <= 232448, "shared memory budget of one sm_90 CTA");
  // row-oriented epilogue: LPR lanes per row (one float4 each), RPI rows per warp instruction, ITERS instructions
  // for the warp's rows, G rows whose addends are in flight before the first store
  static constexpr int LPR = BN / 4;
  static constexpr int RPI = 32 / LPR;
  static constexpr int ITERS = WARP_ROWS / RPI;
  static constexpr int G = ITERS < 8 ? ITERS : 8;
};

struct Params {
  const float* A; int64_t lda;
  const uint8_t* w_image;
  int M, N, K;
  const float* bias;
  const float* add0; int64_t ld0; const int32_t* idx0;   // addend rows: add0[idx0 ? idx0[r] : r][0 .. N)
  const float* add1; int64_t ld1; const int32_t* idx1;
  float* C; int64_t ldc;
  float* stats;                                          // [gridDim.x][2][N] or NULL (requires N <= kMaxStatN)
};

// byte offset of element (r, k) inside one chunk plane (rows x BK, core-matrix order)
__host__ __device__ constexpr int plane_off(int r, int k) { return (r >> 3) * (int)SBO + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2; }

__device__ __forceinline__ float4 ld4(const float* __restrict__ p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4s(const float* p) {          // 4 scalars: vectors of any 4-byte alignment
  return p ? make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3)) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// One consumer warp's WARP_ROWS rows of the tile, from its staged accumulator rows `stg` (row pitch Cfg::PITCH):
//   C[r, col .. col + 3] = (acc + bias) + (add0[i0(r)] + add1[i1(r)]),   r = row0 + rw
// i0 / i1 of row rw sit in lane rw (-1: no addend); col = n0 + 4 (lane % LPR).  s / q collect this lane's column
// sums of C and C^2 over its valid rows in row order.
template <int BN>
__device__ __forceinline__ void epilogue_rows(const float* stg, float* __restrict__ C, int64_t ldc,
                                              const float* __restrict__ add0, int64_t ld0,
                                              const float* __restrict__ add1, int64_t ld1, int i0, int i1, int row0,
                                              int M, int col, int lane, float4 b, float4& s, float4& q) {
  using F = Cfg<BN>;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const int lr = lane / F::LPR, c = (lane % F::LPR) * 4;
#pragma unroll 1   // unrolled, the row groups of BN = 128 spill at the 128-register cap
  for (int g0 = 0; g0 < F::ITERS; g0 += F::G) {
    float4 va[F::G], vb[F::G];
#pragma unroll
    for (int g = 0; g < F::G; ++g) {                         // every addend row of the group is requested first
      const int rw = (g0 + g) * F::RPI + lr;
      const int ia = __shfl_sync(0xffffffffu, i0, rw), ib = __shfl_sync(0xffffffffu, i1, rw);
      va[g] = ia >= 0 ? ld4(add0 + (int64_t)ia * ld0 + col) : z4;
      vb[g] = ib >= 0 ? ld4(add1 + (int64_t)ib * ld1 + col) : z4;
    }
#pragma unroll
    for (int g = 0; g < F::G; ++g) {
      const int rw = (g0 + g) * F::RPI + lr;
      if (row0 + rw >= M) continue;
      const float4 a = *reinterpret_cast<const float4*>(stg + rw * F::PITCH + c);
      const float4 a0 = va[g], a1 = vb[g];
      float4 o;
      o.x = (a.x + b.x) + (a0.x + a1.x);
      o.y = (a.y + b.y) + (a0.y + a1.y);
      o.z = (a.z + b.z) + (a0.z + a1.z);
      o.w = (a.w + b.w) + (a0.w + a1.w);
      *reinterpret_cast<float4*>(C + (int64_t)(row0 + rw) * ldc + col) = o;
      s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
      q.x = fmaf(o.x, o.x, q.x); q.y = fmaf(o.y, o.y, q.y); q.z = fmaf(o.z, o.z, q.z); q.w = fmaf(o.w, o.w, q.w);
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16x3_kernel(const Params p) {
  using F = Cfg<BN>;
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  uint64_t* empty = full + STAGES;
  uint64_t* stat_bar = empty + STAGES;                       // [4]: tile order of the column-partial updates
  uint64_t* mma_turn = stat_bar + 4;                         // [4]: tile order of the consumers' mainloops

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int M = p.M, N = p.N, nk = p.K / BK;
  const int n_tiles = N / BN;
  const int m_tiles = (M + BM - 1) / BM;
  const int total = m_tiles * n_tiles;
  const bool do_stats = p.stats != nullptr;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full[s], LOAD_WARPS + 1); tc::mbar_init(&empty[s], MMA_WARPS / 2); }
    for (int w = 0; w < 4; ++w) { tc::mbar_init(&stat_bar[w], 1); tc::mbar_init(&mma_turn[w], 1); }
    tc::mbar_fence_init();
  }
  if (do_stats) {
    float* stat = reinterpret_cast<float*>(smem + F::STAT_OFF);
    for (int i = tid; i < STAT_ROWS * 2 * N; i += THREADS) stat[i] = 0.f;
  }
  __syncthreads();

  if (warp >= MMA_WARPS) {
    // ================= producer =================
    tc::setmaxnreg_dec<LOAD_REGS>();
    // The CTA's work is the stream of chunks c = (local tile, kc).  Producer warp pw owns rows 32 pw .. 32 pw + 31 of
    // every chunk: it copies them into its own 4 KB of the fp32 stage (one cp.async instruction = 4 rows x 128 bytes)
    // and splits them into the planes (a half-warp = 8 rows x 2 adjacent float4 -> one 128-byte core matrix).  Float4
    // f of row r sits at r * 128 + ((f + 2 r) % 8) * 16 of the warp's block: the copies and the converting reads are
    // both free of bank conflicts.  Only the warp touches its block, so the lanes' own cp.async.wait_group and a
    // __syncwarp order the copies before the reads, and the reads before the next copy into the stage.  Rows at or
    // beyond M are not read; their copies zero-fill the slot.
    const int pw = warp - MMA_WARPS;
    const int my_tiles = (total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int nchunks = my_tiles * nk;
    uint8_t* blk = smem + F::FP_OFF + pw * 32 * 128;
    int f_tile = blockIdx.x, f_kc = 0;                       // next chunk to fetch
    auto fetch = [&](int c) {                                // chunk c into fp32 stage c % FSTAGES; one commit group
      if (c < nchunks) {
        uint8_t* fs = blk + (c % FSTAGES) * F::FSTAGE;
        const int r0 = (f_tile / n_tiles) * BM + pw * 32 + (lane >> 3);
        const float* src = p.A + (int64_t)r0 * p.lda + f_kc * BK + (lane & 7) * 4;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = i * 4 + (lane >> 3);
          const bool rv = r0 + i * 4 < M;
          tc::cp_async16_zfill(fs + row * 128 + (((lane & 7) + 2 * row) & 7) * 16, rv ? src : p.A, rv);
          src += 4 * p.lda;
        }
        if (++f_kc == nk) { f_kc = 0; f_tile += gridDim.x; }
      }
      tc::cp_async_commit();
    };
    const int e_l = (lane >> 1) & 7, oq = (lane >> 4) * 2 + (lane & 1);
#pragma unroll
    for (int c = 0; c < FSTAGES - 1; ++c) fetch(c);
    int s = 0, ph = 0, w_kc = 0, w_tile = blockIdx.x;
    const uint8_t* wsrc = p.w_image + (int64_t)(w_tile % n_tiles) * nk * 2 * F::B_PLANE;
    for (int c = 0; c < nchunks; ++c) {
      fetch(c + FSTAGES - 1);                                // into the fp32 stage this warp read in iteration c - 1
      tc::cp_async_wait<FSTAGES - 1>();                      // this lane's copies of chunk c have landed
      __syncwarp();                                          // ... and every lane's
      if (c >= STAGES) tc::mbar_wait(&empty[s], ph ^ 1);
      uint8_t* st = smem + s * F::STAGE;
      if (pw == 0 && lane == 0) {   // W chunk: one contiguous bulk copy (both planes), counted in bytes on full[s]
        tc::mbar_arrive_expect_tx(&full[s], 2 * F::B_PLANE);
        tc::bulk_g2s(st + 2 * F::A_PLANE, wsrc, 2 * F::B_PLANE, &full[s]);
      }
      const uint8_t* fs = blk + (c % FSTAGES) * F::FSTAGE;
#pragma unroll
      for (int eg = 0; eg < 4; ++eg) {
        const int row = eg * 8 + e_l;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int f = h * 4 + oq;
          uint2 hi, lo;
          tc::split4(*reinterpret_cast<const float4*>(fs + row * 128 + ((f + 2 * row) & 7) * 16), hi, lo);
          const int off = plane_off(pw * 32 + row, f * 4);
          *reinterpret_cast<uint2*>(st + off) = hi;
          *reinterpret_cast<uint2*>(st + F::A_PLANE + off) = lo;
        }
      }
      tc::fence_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&full[s]);              // one arrival per warp
      wsrc += 2 * F::B_PLANE;
      if (++w_kc == nk) {
        w_kc = 0; w_tile += gridDim.x;
        wsrc = p.w_image + (int64_t)(w_tile % n_tiles) * nk * 2 * F::B_PLANE;
      }
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    return;   // no block-wide barrier follows
  }

  // ================= consumers: MMA + epilogue, local tiles wg, wg + 2, ... =================
  tc::setmaxnreg_inc<MMA_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  const int wrow = wq * WARP_ROWS;                           // this warp's fragment: rows wrow .. wrow + 15 of each half
  float* stg = reinterpret_cast<float*>(smem + F::STG_OFF) + warp * WARP_ROWS * F::PITCH;   // this warp's staged rows
  // Column partials: row h * 4 + wq sums rows 64 h + wrow .. + 15 of every tile of the CTA, tile after tile in tile
  // order.  The two warpgroups' warps wq share the rows and take turns: stat_bar[wq] completes one phase per tile.
  float* stat = reinterpret_cast<float*>(smem + F::STAT_OFF);
  const uint32_t sbase = tc::smem_u32(smem);
  int li = wg;                                               // local tile index
  for (int tile = blockIdx.x + wg * gridDim.x; tile < total; tile += 2 * gridDim.x, li += 2) {
    const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
    // addend row indices of the warp's rows, one per lane and half, requested before the mainloop
    int i0[2] = {-1, -1}, i1[2] = {-1, -1};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gr = m0 + h * 64 + wrow + lane;
      if (lane < WARP_ROWS && gr < M) {
        if (p.add0) i0[h] = p.idx0 ? __ldg(p.idx0 + gr) : gr;
        if (p.add1) i1[h] = p.idx1 ? __ldg(p.idx1 + gr) : gr;
      }
    }
    const int g = li * nk;                                   // first chunk of this tile in the ring
    int s = g % STAGES, ph = (g / STAGES) & 1;
    float acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
    // Warp wq of the other warpgroup has waited for the last chunk of local tile li - 1.  Both hand-off barriers are per
    // warp pair, one arrival per phase: a warp's own arrival completes the phase before the one it waits for next.
    if (li > 0) tc::mbar_wait(&mma_turn[wq], (li - 1) & 1);
    int prev = -1;
    for (int kc = 0; kc < nk; ++kc) {
      tc::mbar_wait(&full[s], ph);
      const uint32_t sa = sbase + s * F::STAGE;
      tc::wgmma_fence();
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint32_t b_hi = sa + 2 * F::A_PLANE + j * 2 * LBO;
        const uint64_t dbh = tc::smem_desc(b_hi, LBO, SBO), dbl = tc::smem_desc(b_hi + F::B_PLANE, LBO, SBO);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t a_hi = sa + h * 8 * SBO + j * 2 * LBO;
          const uint64_t dah = tc::smem_desc(a_hi, LBO, SBO), dal = tc::smem_desc(a_hi + F::A_PLANE, LBO, SBO);
          tc::Wgmma<BN>::template mma<0, 0>(acc[h], dal, dbh, 1);   // small terms first
          tc::Wgmma<BN>::template mma<0, 0>(acc[h], dah, dbl, 1);
          tc::Wgmma<BN>::template mma<0, 0>(acc[h], dah, dbh, 1);
        }
      }
      tc::wgmma_commit();
      tc::wgmma_wait<1>();                                   // the MMAs of chunk kc - 1 are complete
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty[prev]);        // this warp is done reading that stage
      }
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    if (tile + (int)gridDim.x < total) {                     // local tile li + 1 may start its mainloop
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&mma_turn[wq]);
    }
    tc::wgmma_wait_all();
    __syncwarp();
    if (lane == 0 && prev >= 0) tc::mbar_arrive(&empty[prev]);
    // ---- epilogue, one row half after the other: stage the fragment (thread holds acc[h][4 j + 2 e + t] = row
    //      lane / 4 + 8 e, column 8 j + 2 (lane % 4) + t of the warp's rows), then row by row:
    //      (acc + bias) + (addend0 + addend1) ----
    const int col = n0 + (lane % F::LPR) * 4;
    const float4 b = ld4s(p.bias ? p.bias + col : nullptr);
    float4 s4[2], q4[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          *reinterpret_cast<float2*>(stg + ((lane >> 2) + 8 * e) * F::PITCH + 8 * j + 2 * (lane & 3)) =
              make_float2(acc[h][4 * j + 2 * e], acc[h][4 * j + 2 * e + 1]);
      __syncwarp();
      s4[h] = make_float4(0.f, 0.f, 0.f, 0.f); q4[h] = s4[h];
      epilogue_rows<BN>(stg, p.C, p.ldc, p.add0, p.ld0, p.add1, p.ld1, i0[h], i1[h], m0 + h * 64 + wrow, M, col, lane,
                        b, s4[h], q4[h]);
      __syncwarp();                                          // staged rows read before they are overwritten
    }
    if (do_stats) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // lanes lane % LPR hold the same columns for different rows: fold them, fixed order
#pragma unroll
        for (int o = F::LPR; o < 32; o <<= 1) {
          s4[h].x += __shfl_xor_sync(0xffffffffu, s4[h].x, o); s4[h].y += __shfl_xor_sync(0xffffffffu, s4[h].y, o);
          s4[h].z += __shfl_xor_sync(0xffffffffu, s4[h].z, o); s4[h].w += __shfl_xor_sync(0xffffffffu, s4[h].w, o);
          q4[h].x += __shfl_xor_sync(0xffffffffu, q4[h].x, o); q4[h].y += __shfl_xor_sync(0xffffffffu, q4[h].y, o);
          q4[h].z += __shfl_xor_sync(0xffffffffu, q4[h].z, o); q4[h].w += __shfl_xor_sync(0xffffffffu, q4[h].w, o);
        }
      }
      if (li > 0) tc::mbar_wait(&stat_bar[wq], (li - 1) & 1);   // the other warpgroup has added local tile li - 1
      if (lane < F::LPR) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* st = stat + (h * 4 + wq) * 2 * N;
          st[col] += s4[h].x; st[col + 1] += s4[h].y; st[col + 2] += s4[h].z; st[col + 3] += s4[h].w;
          st[N + col] += q4[h].x; st[N + col + 1] += q4[h].y; st[N + col + 2] += q4[h].z; st[N + col + 3] += q4[h].w;
        }
      }
      if (tile + (int)gridDim.x < total) {                   // hand the rows to the warp that owns local tile li + 1
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&stat_bar[wq]);
      }
    }
  }
  if (do_stats) {
    // one partial row per CTA: the eight column partials summed in a fixed order
    asm volatile("bar.sync 1, %0;" ::"n"(MMA_WARPS * 32) : "memory");
    float* out_row = p.stats + (int64_t)blockIdx.x * 2 * N;
    for (int i = tid; i < 2 * N; i += MMA_WARPS * 32) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < STAT_ROWS; ++w) t += stat[w * 2 * N + i];
      out_row[i] = t;
    }
  }
}

// Weight images: W[N,K] fp32 (or W^T of a [K,N] array) -> [N/BN tiles][K/32 chunks][hi, lo][BN x 32 bf16 in
// core-matrix order].  Every table entry converts one source block into its place inside a (possibly larger) image, so
// all operand images of a model -- [W_sg; W_du; W_dg; W_su] stacked along N, its transpose stacked along K, the
// edge gate and its transpose, the embedding Linears (K zero-padded) -- are refreshed by ONE launch per step.
// blockIdx.y = entry; thread = one 8-element K group of one image row inside the entry's block.
__global__ void prepare_weights_table_kernel(const alignn_b200_image_entry* __restrict__ entries) {
  const alignn_b200_image_entry e = entries[blockIdx.y];
  const int Ne = e.transpose ? e.cols : e.rows, Ke = e.transpose ? e.rows : e.cols;   // block shape in image coordinates
  const int k8n = (Ke + 7) / 8;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)Ne * k8n) return;
  const int nl = (int)(t / k8n), k8 = (int)(t % k8n);
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int kl = k8 * 8 + j;
    v[j] = kl < Ke ? (e.transpose ? e.W[(int64_t)kl * e.ldw + nl] : e.W[(int64_t)nl * e.ldw + kl]) : 0.f;
  }
  uint2 h0, l0, h1, l1;
  tc::split4(make_float4(v[0], v[1], v[2], v[3]), h0, l0);
  tc::split4(make_float4(v[4], v[5], v[6], v[7]), h1, l1);
  const int bn = (e.N % 128 == 0) ? 128 : (e.N % 64 == 0) ? 64 : 32;   // pick_bn
  const int n = e.n_off + nl, k = e.k_off + k8 * 8;          // image coordinates (k_off is a multiple of 8)
  const int nt = n / bn, r = n % bn, kc = k / BK, kk = (k % BK) / 8;
  const int64_t b_plane = (int64_t)bn * BK * 2;
  const int64_t chunk = ((int64_t)nt * (e.K / BK) + kc) * 2 * b_plane;
  const int off = plane_off(r, kk * 8);
  uint8_t* img = reinterpret_cast<uint8_t*>(e.image);
  *reinterpret_cast<uint4*>(img + chunk + off) = make_uint4(h0.x, h0.y, h1.x, h1.y);
  *reinterpret_cast<uint4*>(img + chunk + b_plane + off) = make_uint4(l0.x, l0.y, l1.x, l1.y);
}

// dst[j] = a[j] (+ b[j]): the stacked / folded bias vectors that go with the images (blockIdx.y = entry)
__global__ void prepare_bias_table_kernel(const alignn_b200_bias_entry* __restrict__ entries) {
  const alignn_b200_bias_entry e = entries[blockIdx.y];
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < e.n; j += gridDim.x * blockDim.x)
    e.dst[j] = e.a[j] + (e.b ? e.b[j] : 0.f);
}

// widest column tile that divides N: the accumulator of a 128 x BN tile is BN / 2 registers per consumer thread
inline int pick_bn(int N) { return (N % 128 == 0) ? 128 : (N % 64 == 0) ? 64 : (N % 32 == 0) ? 32 : 0; }

inline int num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    sms = n > 0 ? n : kNumSMs;
  }
  return sms;
}

template <int BN>
int launch_bn(const Params& p, int grid, cudaStream_t st) {
  using F = Cfg<BN>;
  static alignn::DeviceOnce configured; int cfg_dev;   // idempotent attribute; a benign race sets it twice
  if (configured.needed(&cfg_dev)) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16x3_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM);
    if (e != cudaSuccess) return record_cuda_error((int)e);
    configured.done(cfg_dev);
  }
  gemm_bf16x3_kernel<BN><<<grid, THREADS, F::SMEM, st>>>(p);
  return check_launch();
}

inline int launch(const Params& p, int grid, cudaStream_t st) {
  switch (pick_bn(p.N)) {
    case 128: return launch_bn<128>(p, grid, st);
    case 64: return launch_bn<64>(p, grid, st);
    case 32: return launch_bn<32>(p, grid, st);
    default: return ALIGNN_ERR_UNSUPPORTED_D;
  }
}

}  // namespace gemm
}  // namespace alignn

extern "C" {

size_t alignn_b200_gemm_weight_image_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || alignn::gemm::pick_bn(N) == 0 || K % alignn::gemm::BK != 0) return 0;
  return (size_t)N * K * 2 * 2;   // two bf16 planes
}

int alignn_b200_gemm_prepare_table(const alignn_b200_image_entry* entries, int n_entries, int64_t max_units,
                                   const alignn_b200_bias_entry* bias_entries, int n_bias, alignn_stream_t stream) {
  if (n_entries < 0 || n_bias < 0 || (n_entries > 0 && (!entries || max_units <= 0)) || (n_bias > 0 && !bias_entries))
    return ALIGNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (n_entries > 0) {
    const unsigned bx = (unsigned)((max_units + 255) / 256);
    alignn::gemm::prepare_weights_table_kernel<<<dim3(bx, (unsigned)n_entries), 256, 0, st>>>(entries);
    int rc = alignn::check_launch();
    if (rc != ALIGNN_OK) return rc;
  }
  if (n_bias > 0) {
    alignn::gemm::prepare_bias_table_kernel<<<dim3(4, (unsigned)n_bias), 256, 0, st>>>(bias_entries);
    return alignn::check_launch();
  }
  return ALIGNN_OK;
}

int alignn_b200_gemm_nt(const float* A, int64_t lda, const void* w_image, int64_t M, int N, int K, const float* bias,
                        const float* R, int64_t ldr, float* C, int64_t ldc, alignn_stream_t stream) {
  using namespace alignn::gemm;
  if (M < 0 || N <= 0 || K <= 0 || K % BK != 0 || lda < K || ldc < N || (R && ldr < N)) return ALIGNN_ERR_BAD_ARG;
  if (M == 0) return ALIGNN_OK;
  if (!A || !w_image || !C || M > 0x7fffffff) return ALIGNN_ERR_BAD_ARG;
  if ((lda % 4) || (ldc % 4) || (R && (ldr % 4))) return ALIGNN_ERR_BAD_ARG;   // 16-byte row alignment
  if (((uintptr_t)A & 15) || ((uintptr_t)C & 15) || ((uintptr_t)R & 15)) return ALIGNN_ERR_BAD_ARG;
  const int bn = pick_bn(N);
  if (bn == 0) return ALIGNN_ERR_UNSUPPORTED_D;
  Params p = {};
  p.A = A; p.lda = lda; p.w_image = reinterpret_cast<const uint8_t*>(w_image);
  p.M = (int)M; p.N = N; p.K = K;
  p.bias = bias;
  p.add0 = R; p.ld0 = ldr;
  p.C = C; p.ldc = ldc;
  const int total = ((p.M + BM - 1) / BM) * (N / bn);
  const int grid = total < num_sms() ? total : num_sms();   // persistent: one CTA per SM
  return launch(p, grid, (cudaStream_t)stream);
}

int alignn_b200_gemm_gather_stat_rows(int64_t M, int N) {
  using namespace alignn::gemm;
  const int bn = pick_bn(N);
  if (bn == 0 || M <= 0) return 0;
  // CTAs of the launch, one partial row each
  const int64_t total = (M + BM - 1) / BM * (N / bn);
  return (int)(total < alignn::kNumSMs ? total : alignn::kNumSMs);
}

int alignn_b200_gemm_gather(const alignn_b200_gemm_gather_args* a) {
  using namespace alignn::gemm;
  if (!a) return ALIGNN_ERR_BAD_ARG;
  if (a->struct_size != sizeof(*a)) return ALIGNN_ERR_STRUCT_SIZE;
  if (a->M < 0 || a->N <= 0 || a->K <= 0 || a->K % BK != 0 || a->lda < a->K || a->ldc < a->N) return ALIGNN_ERR_BAD_ARG;
  if (a->M == 0) return ALIGNN_OK;
  if (!a->A || !a->w_image || !a->C || a->M > 0x7fffffff) return ALIGNN_ERR_BAD_ARG;
  if ((a->lda % 4) || (a->ldc % 4) || ((uintptr_t)a->A & 15) || ((uintptr_t)a->C & 15)) return ALIGNN_ERR_BAD_ARG;
  if (a->add0 && ((a->ld0 % 4) || a->ld0 < a->N || ((uintptr_t)a->add0 & 15))) return ALIGNN_ERR_BAD_ARG;
  if (a->add1 && ((a->ld1 % 4) || a->ld1 < a->N || ((uintptr_t)a->add1 & 15))) return ALIGNN_ERR_BAD_ARG;
  if ((a->idx0 && !a->add0) || (a->idx1 && !a->add1)) return ALIGNN_ERR_BAD_ARG;
  const int bn = pick_bn(a->N);
  if (bn == 0) return ALIGNN_ERR_UNSUPPORTED_D;
  if (a->stats && a->N > kMaxStatN) return ALIGNN_ERR_BAD_ARG;   // column partials of every warp live in shared memory
  Params p;
  p.A = a->A; p.lda = a->lda;
  p.M = (int)a->M; p.N = a->N; p.K = a->K;
  p.w_image = reinterpret_cast<const uint8_t*>(a->w_image);
  p.bias = a->bias;
  p.add0 = a->add0; p.ld0 = a->ld0; p.idx0 = a->idx0;
  p.add1 = a->add1; p.ld1 = a->ld1; p.idx1 = a->idx1;
  p.C = a->C; p.ldc = a->ldc; p.stats = a->stats;
  const int total = ((p.M + BM - 1) / BM) * (p.N / bn);
  int grid = total < num_sms() ? total : num_sms();
  if (p.stats) grid = alignn_b200_gemm_gather_stat_rows(p.M, p.N);   // the caller sized `stats` for this many CTAs
  return launch(p, grid, (cudaStream_t)a->stream);
}

}  // extern "C"
