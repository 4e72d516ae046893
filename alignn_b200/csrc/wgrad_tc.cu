// Weight gradients of the Linear layers: C[g][o][i] = sum_r A[r, g*DA + o] * B[r, i], r over the rows
// (edges or nodes) of the batch -- a DA x DB output with a very long reduction (K = 276 480 rows for the
// edge gate on L(g)).  Tensor cores via wgmma (bf16 x bf16 -> fp32 in registers), bf16x3 split (tc_common.cuh).
//
// Both operands are "MN-major" for this product (the contraction index is the ROW of the row-major
// activations), so the loader threads convert fp32 -> bf16 hi/lo and store the canonical MN-major
// SWIZZLE_NONE GMMA layout:  addr(mn, k) = (mn/8)*SBO + (k/8)*LBO + (k%8)*16 + (mn%8)*2,
// SBO = 128 (next 8 channels), LBO = (rows_of_plane/8)*128 (next 8 rows of the contraction).
//
// Mainloop, per CTA: the fp32 rows travel global -> shared by cp.async into a ring of FSTAGES fp32 stages (the bytes
// in flight are set by shared memory, not by registers); the loader warps split each fp32 stage into a bf16 hi/lo
// plane stage (ring of STAGES); the two consumer warpgroups keep one wgmma group in flight and release a plane stage
// once the next chunk's MMAs are issued.
//
// Output tiles: a CTA owns a 128 x TN block of the DA x DB output (TN = min(DB, 128)), held in the registers of two
// consumer warpgroups (rows 0-63 / 64-127, TN / 2 floats per thread); DA = 256 or DB = 256 take 2 or 4 CTAs per row
// slab, each reading only its channels.  Split-K: CTA c of group g reduces a contiguous slab of rows into its block
// and writes it into a partial tile; the partials are then summed in a fixed order (deterministic, no float atomics).
#include <cooperative_groups.h>

#include "common.cuh"
#include "tc_common.cuh"
#include "api_common.h"
#include "alignn_b200.h"

namespace alignn {
namespace wgrad {

constexpr int BK = 32;          // contraction rows per stage (2 MMA K=16 steps)
// Shared memory at TA = TN = 128: 2 plane stages of 32 KB, 3 fp32 stages of 32 KB and the 64 KB of running sums, 224 KB.
// (3 plane stages with 2 fp32 stages measured 6 % slower on the bench's weight-gradient launch on H100.)
constexpr int STAGES = 2;       // bf16 hi/lo plane stages (loaders -> MMAs)
constexpr int FSTAGES = 3;      // fp32 stages (cp.async -> loaders): up to 64 KB in flight per CTA while it converts
constexpr int LOAD_WARPS = 8;
constexpr int MMA_WARPS = 8;    // two consumer warpgroups
constexpr int THREADS = 32 * (MMA_WARPS + LOAD_WARPS);
constexpr uint32_t SBO = 128;
constexpr int kNumSMsWgrad = kNumSMs;
// Contraction rows a wgmma accumulator sums before it is added into the fp32 running sum in shared memory: the tensor
// core's own accumulation over the thousands of rows of one slab loses more than the 2e-5 budget allows.
constexpr int PROMOTE_CHUNKS = 8;

__host__ __device__ constexpr int tiles_of(int DA, int DB) { return (DA > 128 ? DA / 128 : 1) * (DB > 128 ? DB / 128 : 1); }

template <int DA, int DB>   // A: [K, groups*DA] (output-gradient side), B: [K, DB] (input side); out DA x DB
struct Cfg {
  static constexpr int TA = DA < 128 ? DA : 128;      // A channels of one CTA's block (plane padded to 128 rows)
  static constexpr int TN = DB <= 128 ? DB : 128;     // B channels of one CTA's block
  static constexpr int NT = DB / TN;
  static constexpr int TILES = tiles_of(DA, DB);
  static constexpr int A_PLANE = 128 * BK * 2;
  static constexpr int B_PLANE = TN * BK * 2;
  static constexpr uint32_t LBO_A = (128 / 8) * 128;
  static constexpr uint32_t LBO_B = (TN / 8) * 128;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int PIPE = STAGES * STAGE;
  static constexpr int NBA = TA / 32, NBB = TN / 32;         // 32-channel blocks of A and B: one loader warp each
  static constexpr int FSTAGE = LOAD_WARPS * BK * 128;        // fp32 stage: 4 KB (32 rows x 32 channels) per loader warp
  static constexpr int ACC_OFF = PIPE + FSTAGES * FSTAGE;
  static constexpr int ACC = MMA_WARPS * 32 * (TN / 2) * 4;   // running sums, one column per consumer thread
  static constexpr int BAR_OFF = ACC_OFF + ACC;
  static constexpr int SMEM = BAR_OFF + 128;
  static_assert(TILES * TA * TN == DA * DB, "output blocks cover the output");
  static_assert(SMEM <= 232448, "shared memory budget of one sm_90 CTA");
  static_assert(TA % 32 == 0 && TN % 32 == 0 && NBA + NBB <= LOAD_WARPS, "one loader warp per 32-channel block");
};

// The pipeline of one CTA over consecutive chunks of contraction rows, shared by the single-problem and the batch
// kernels: loader warps fill the stage ring, the consumer warpgroups accumulate; the caller brackets it.
template <int DA, int DB>
struct Pipe {
  using F = Cfg<DA, DB>;
  uint8_t* smem;
  uint64_t* full;
  uint64_t* empty;

  // loader warps: rows [r_begin, r_end) of A (channels a0 .. a0 + TA) and B (channels b0 .. b0 + TN), chunks numbered
  // from g0 in the plane ring.  Loader warp w < NBA + NBB owns one 32-channel block of the chunk (A's blocks first, then
  // B's), all 32 rows: it copies the block into its own 4 KB of the fp32 stage (one cp.async instruction = 4 rows x
  // 128 bytes) and converts it into the planes (a half-warp = 8 contraction rows x 2 adjacent float4 -> one 128-byte
  // core matrix).  Float4 f of row r sits at r * 128 + ((f + 2 r) % 8) * 16 of the warp's block: the copies and the
  // converting reads are both free of bank conflicts.  Only the warp touches its block, so the lanes' own
  // cp.async.wait_group and a __syncwarp order the copies before the reads, and the reads before the next copy into
  // the stage.  Rows at or beyond r_end are not read; their copies zero-fill the slot.
  __device__ __forceinline__ void load(const float* __restrict__ Ag, int64_t lda, const float* __restrict__ Bg, int64_t ldb,
                                       int64_t r_begin, int64_t r_end, int nk, int g0, int warp, int lane) {
    const bool isA = warp < F::NBA, active = warp < F::NBA + F::NBB;
    const int cb = isA ? warp : warp - F::NBA;                         // 32-channel block of the operand
    const float* __restrict__ src = (isA ? Ag : Bg) + cb * 32 + (lane & 7) * 4;
    const int64_t ld = isA ? lda : ldb;
    uint8_t* blk = smem + F::PIPE + warp * BK * 128;
    auto fetch = [&](int kc) {                 // chunk kc into fp32 stage kc % FSTAGES; one commit group per call
      if (active && kc < nk) {
        uint8_t* fs = blk + (kc % FSTAGES) * F::FSTAGE;
#pragma unroll
        for (int i = 0; i < BK / 4; ++i) {
          const int row = i * 4 + (lane >> 3);
          const int64_t r = r_begin + (int64_t)kc * BK + row;
          const bool rv = r < r_end;
          tc::cp_async16_zfill(fs + row * 128 + (((lane & 7) + 2 * row) & 7) * 16, src + (rv ? r : r_begin) * ld, rv);
        }
      }
      tc::cp_async_commit();
    };
    const int e_l = (lane >> 1) & 7, oq = (lane >> 4) * 2 + (lane & 1);
    const int lbo = isA ? (int)F::LBO_A : (int)F::LBO_B, plane = isA ? F::A_PLANE : F::B_PLANE;
#pragma unroll
    for (int kc = 0; kc < FSTAGES - 1; ++kc) fetch(kc);
    for (int kc = 0; kc < nk; ++kc) {
      fetch(kc + FSTAGES - 1);                 // into the stage this warp converted from in iteration kc - 1
      tc::cp_async_wait<FSTAGES - 1>();        // this lane's copies of chunk kc have landed
      __syncwarp();                            // ... and every lane's
      const int gc = g0 + kc, s = gc % STAGES;
      if (gc >= STAGES) tc::mbar_wait(&empty[s], ((gc / STAGES) - 1) & 1);
      if (active) {
        const uint8_t* fs = blk + (kc % FSTAGES) * F::FSTAGE;
        uint8_t* base = smem + s * F::STAGE + (isA ? 0 : 2 * F::A_PLANE);
#pragma unroll
        for (int eg = 0; eg < 4; ++eg) {
          const int edge = eg * 8 + e_l;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int f = h * 4 + oq, o4 = cb * 8 + f;
            uint2 hi, lo;
            tc::split4(*reinterpret_cast<const float4*>(fs + edge * 128 + ((f + 2 * edge) & 7) * 16), hi, lo);
            const int off = (o4 >> 1) * (int)SBO + (edge >> 3) * lbo + (edge & 7) * 16 + (o4 & 1) * 8;
            *reinterpret_cast<uint2*>(base + off) = hi;
            *reinterpret_cast<uint2*>(base + plane + off) = lo;
          }
        }
      }
      tc::fence_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&full[s]);          // one arrival per warp
    }
  }

  // consumer warpgroup wg: acc = its 64 rows of the block summed over nk chunks numbered from g0.  One wgmma group
  // stays in flight: the stage of chunk kc - 1 is released once the MMAs of chunk kc are issued and kc - 1's are
  // complete; the queue drains only where the accumulator is read (promotion into the running sum).
  __device__ __forceinline__ void mma(float (&acc)[F::TN / 2], int nk, int g0, int wg, int lane) {
    const uint32_t base0 = tc::smem_u32(smem);
    float* run = reinterpret_cast<float*>(smem + F::ACC_OFF) + wg * 128 + (threadIdx.x & 127);
#pragma unroll
    for (int i = 0; i < F::TN / 2; ++i) { run[i * MMA_WARPS * 32] = 0.f; acc[i] = 0.f; }
    // The chunks go in runs of PROMOTE_CHUNKS: the full drain sits after a run's loop, never on a branch inside it (a
    // wgmma wait on a branch makes ptxas serialize every wgmma of the kernel).
    for (int k0 = 0; k0 < nk; k0 += PROMOTE_CHUNKS) {
      const int k1 = k0 + PROMOTE_CHUNKS < nk ? k0 + PROMOTE_CHUNKS : nk;
      int prev = -1;                                     // stage whose MMAs may still be in flight
      for (int kc = k0; kc < k1; ++kc) {
        const int g = g0 + kc, s = g % STAGES;
        tc::mbar_wait(&full[s], (g / STAGES) & 1);
        const uint32_t base = base0 + s * F::STAGE;
        tc::wgmma_fence();
#pragma unroll
        for (int j = 0; j < BK / 16; ++j) {
          const uint64_t b_hi = tc::smem_desc(base + 2 * F::A_PLANE + j * 2 * F::LBO_B, F::LBO_B, SBO);
          const uint64_t b_lo = tc::smem_desc(base + 2 * F::A_PLANE + F::B_PLANE + j * 2 * F::LBO_B, F::LBO_B, SBO);
          const uint32_t ao = j * 2 * F::LBO_A + wg * 8 * SBO;
          const uint64_t a_hi = tc::smem_desc(base + ao, F::LBO_A, SBO);
          const uint64_t a_lo = tc::smem_desc(base + F::A_PLANE + ao, F::LBO_A, SBO);
          tc::Wgmma<F::TN>::template mma<1, 1>(acc, a_lo, b_hi, 1);
          tc::Wgmma<F::TN>::template mma<1, 1>(acc, a_hi, b_lo, 1);
          tc::Wgmma<F::TN>::template mma<1, 1>(acc, a_hi, b_hi, 1);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<1>();                             // the MMAs of chunk kc - 1 are complete
        __syncwarp();
        if (lane == 0 && prev >= 0) tc::mbar_arrive(&empty[prev]);
        prev = s;
      }
      tc::wgmma_wait_all();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&empty[prev]);
#pragma unroll
      for (int i = 0; i < F::TN / 2; ++i) { run[i * MMA_WARPS * 32] += acc[i]; acc[i] = 0.f; }
    }
#pragma unroll
    for (int i = 0; i < F::TN / 2; ++i) acc[i] = run[i * MMA_WARPS * 32];
  }

  // Partial tiles are a private workspace, stored BLOCKED: element (o, c) at ((c / 32) * DA + o) * 32 + c % 32; the
  // reduction un-blocks.  Block (mt, nt) of the output, consumer thread (warp, lane).
  __device__ __forceinline__ static void store(const float (&acc)[F::TN / 2], float* out, int mt, int nt, int warp, int lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (r >= F::TA) continue;
      const int o = mt * F::TA + r;
#pragma unroll
      for (int j = 0; j < F::TN / 8; ++j) {
        const int c = nt * F::TN + 8 * j + 2 * (lane & 3);
        *reinterpret_cast<float2*>(out + ((int64_t)(c >> 5) * DA + o) * 32 + (c & 31)) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
};

template <int DA, int DB>
__device__ __forceinline__ void pipe_init(uint8_t* smem, uint64_t* full, uint64_t* empty) {
  using F = Cfg<DA, DB>;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full[s], LOAD_WARPS); tc::mbar_init(&empty[s], MMA_WARPS); }
    tc::mbar_fence_init();
  }
  if (F::TA < 128) {   // padded A rows [TA, 128) are never written by the loaders: zero the planes once
    for (int i = threadIdx.x; i < F::PIPE / 16; i += THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  }
  tc::fence_async_smem();
  __syncthreads();
}

// grid (ctas, groups, TILES): CTA (c, g, t) reduces rows [c * rows_per_cta, ...) of group g into output block t
template <int DA, int DB>
__global__ void __launch_bounds__(THREADS, 1)
wgrad_bf16x3_kernel(const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb, int64_t K,
                    int rows_per_cta, float* __restrict__ partials, float* __restrict__ out, int64_t ld_out) {
  using F = Cfg<DA, DB>;
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  Pipe<DA, DB> pipe{smem, full, full + STAGES};
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x, group = blockIdx.y, mt = blockIdx.z / F::NT, nt = blockIdx.z % F::NT;
  const int64_t r_begin = (int64_t)cta * rows_per_cta;
  const int64_t r_end = (r_begin + rows_per_cta < K) ? r_begin + rows_per_cta : K;
  const int nk = r_end > r_begin ? (int)((r_end - r_begin + BK - 1) / BK) : 0;
  pipe_init<DA, DB>(smem, full, full + STAGES);

  if (warp >= MMA_WARPS) {
    pipe.load(A + (int64_t)group * DA + mt * F::TA, lda, B + nt * F::TN, ldb, r_begin, r_end, nk, 0, warp - MMA_WARPS, lane);
  } else {
    float acc[F::TN / 2];
    pipe.mma(acc, nk, 0, warp >> 2, lane);
    Pipe<DA, DB>::store(acc, partials + ((int64_t)group * gridDim.x + cta) * DA * DB, mt, nt, warp, lane);
  }
  if (out) {
    // Split-K reduction inside the kernel (cooperative launch: every CTA is resident): once all partial tiles are
    // written, the CTAs of a group sum slices of the DA x DB output over the group's partials in a fixed order.
    __threadfence();
    cooperative_groups::this_grid().sync();
    const int ctas = gridDim.x;
    const int64_t rank = (int64_t)blockIdx.z * gridDim.x + cta, parts = (int64_t)gridDim.z * gridDim.x;
    constexpr int64_t tile = (int64_t)DA * DB;
    const float* p = partials + (int64_t)group * ctas * tile;
    for (int64_t idx = (rank * THREADS + tid) * 4; idx < tile; idx += parts * THREADS * 4) {
      // 16 partials per batch: the loads of a batch are independent (latency paid once per batch), the adds keep one
      // fixed order
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
      int c = 0;
      for (; c + 16 <= ctas; c += 16) {
        float4 v[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) v[u] = __ldcg(reinterpret_cast<const float4*>(p + (int64_t)(c + u) * tile + idx));
#pragma unroll
        for (int u = 0; u < 16; ++u) { s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w; }
      }
      for (; c < ctas; ++c) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(p + (int64_t)c * tile + idx));
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
      const int64_t o = (idx >> 5) % DA, i = (idx >> 5) / DA * 32 + (idx & 31);     // blocked -> row-major
      *reinterpret_cast<float4*>(out + ((int64_t)group * DA + o) * ld_out + i) = s;
    }
  }
}

// ---- many weight gradients in ONE launch ---------------------------------------------------------------------------
// A training step of the 4+4 stack needs 24 square weight gradients (4 with K = T bond pairs, 12 with K = E bonds, 8 x 4
// with K = N atoms); none of them is on the critical path of the backward pass, and launched one by one the small ones
// cost a prologue, one partial tile per CTA and a grid barrier each.  The batch kernel takes all of them as a list of
// problems, cuts the concatenated rows into slabs of equal cost, one sequence of slabs per CTA column (blockIdx.x; the
// TILES CTAs of a column, blockIdx.y, own the output blocks), and runs the same loader / MMA / store pipeline slab after
// slab; every slab leaves one partial tile, and after the grid barrier all CTAs sum each problem's partial tiles in slab
// order (fixed order: deterministic).
constexpr int kMaxProblems = 64;
constexpr int kMaxSlabs = 320;

struct Problem {
  const float* A; const float* B; float* out;
  int64_t lda, ldb, ld_out, K;
  int slab_first, slab_count;
};
struct Slab { int prob, chunk_begin, chunks; };     // rows [chunk_begin*BK, min(K, (chunk_begin+chunks)*BK)) of the problem
struct Batch {
  Problem prob[kMaxProblems];
  Slab slab[kMaxSlabs];
  int cta_first[kNumSMsWgrad + 1];                  // CTA column c runs slabs [cta_first[c], cta_first[c+1])
  int nprob;
};

template <int DA, int DB>
__global__ void __launch_bounds__(THREADS, 1)
wgrad_batch_kernel(const __grid_constant__ Batch bt, float* __restrict__ partials) {
  using F = Cfg<DA, DB>;
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  Pipe<DA, DB> pipe{smem, full, full + STAGES};
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x, mt = blockIdx.y / F::NT, nt = blockIdx.y % F::NT;
  const int s_first = bt.cta_first[cta], s_last = bt.cta_first[cta + 1];
  pipe_init<DA, DB>(smem, full, full + STAGES);

  int g = 0;                                     // chunks this CTA has pushed through the stage ring so far
  for (int si = s_first; si < s_last; ++si) {
    const Slab sl = bt.slab[si];
    const Problem& pr = bt.prob[sl.prob];
    const int nk = sl.chunks;
    if (warp >= MMA_WARPS) {
      const int64_t r_begin = (int64_t)sl.chunk_begin * BK;
      const int64_t r_end = (r_begin + (int64_t)sl.chunks * BK < pr.K) ? r_begin + (int64_t)sl.chunks * BK : pr.K;
      pipe.load(pr.A + mt * F::TA, pr.lda, pr.B + nt * F::TN, pr.ldb, r_begin, r_end, nk, g, warp - MMA_WARPS, lane);
    } else {
      float acc[F::TN / 2];
      pipe.mma(acc, nk, g, warp >> 2, lane);
      Pipe<DA, DB>::store(acc, partials + (int64_t)si * DA * DB, mt, nt, warp, lane);
    }
    g += nk;
  }
  // ---- all partial tiles are written: every CTA sums a share of every problem's output, slabs in order ----
  __threadfence();
  cooperative_groups::this_grid().sync();
  constexpr int64_t tile = (int64_t)DA * DB;
  constexpr int64_t tile4 = tile / 4;
  const int64_t items = (int64_t)bt.nprob * tile4;
  const int64_t rank = (int64_t)blockIdx.y * gridDim.x + cta, parts = (int64_t)gridDim.y * gridDim.x;
  for (int64_t it = rank * THREADS + tid; it < items; it += parts * THREADS) {
    const int pi = (int)(it / tile4);
    const int64_t idx = (it - (int64_t)pi * tile4) * 4;
    const Problem& pr = bt.prob[pi];
    const float* p = partials + (int64_t)pr.slab_first * tile + idx;
    const int n = pr.slab_count;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    int c = 0;
    for (; c + 8 <= n; c += 8) {
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldcg(reinterpret_cast<const float4*>(p + (int64_t)(c + u) * tile));
#pragma unroll
      for (int u = 0; u < 8; ++u) { s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w; }
    }
    for (; c < n; ++c) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(p + (int64_t)c * tile));
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    const int64_t o = (idx >> 5) % DA, i = (idx >> 5) / DA * 32 + (idx & 31);     // blocked -> row-major
    *reinterpret_cast<float4*>(pr.out + o * pr.ld_out + i) = s;
  }
}

// Cut the problems into slabs: every CTA gets about the same cost, cost(slab) = its chunks + kSlabCost (the fixed price
// of a slab: accumulator drain and a DA x DB partial tile to write and re-read, about the time of 6 chunks of rows).
// The per-CTA budget starts at total / ctas and grows until the cut fits `ctas` CTA columns (kNumSMs / TILES: every
// column is TILES CTAs, one per output block; a problem cut in two pays the slab price twice, so the first guess can be
// short).  Returns the number of slabs, or -1 if the batch does not fit the
// tables (the caller then splits the batch).
constexpr int kSlabCost = 6;
inline int cut_batch(const int64_t* K, int n, int64_t target, int ctas, Batch* bt) {
  int ns = 0, cta = 0;
  int64_t budget = target;
  if (bt) bt->cta_first[0] = 0;
  for (int p = 0; p < n; ++p) {
    int64_t left = (K[p] + BK - 1) / BK, begin = 0;
    const int first = ns;
    while (left > 0) {
      if (budget <= kSlabCost + 2) {                                  // not worth a slab here: next CTA
        if (++cta >= ctas) return -2;                                  // budget too small for the CTAs
        budget = target;
        if (bt) bt->cta_first[cta] = ns;
      }
      int64_t take = budget - kSlabCost;
      if (take > left) take = left;
      if (ns >= kMaxSlabs) return -1;
      if (bt) { bt->slab[ns].prob = p; bt->slab[ns].chunk_begin = (int)begin; bt->slab[ns].chunks = (int)take; }
      ++ns;
      begin += take; left -= take; budget -= take + kSlabCost;
    }
    if (bt) { bt->prob[p].slab_first = first; bt->prob[p].slab_count = ns - first; }
  }
  if (bt) {
    for (int c = cta + 1; c <= kNumSMsWgrad; ++c) bt->cta_first[c] = ns;
    bt->nprob = n;
  }
  return ns;
}
inline int plan_batch(const int64_t* K, int n, int ctas, Batch* bt) {
  if (n < 1 || n > kMaxProblems) return -1;
  int64_t total = 0;
  for (int p = 0; p < n; ++p) total += (K[p] + BK - 1) / BK + kSlabCost;
  int64_t target = (total + ctas - 1) / ctas;
  if (target < 8 * kSlabCost) target = 8 * kSlabCost;                 // never spread a small batch thinner than this
  for (;;) {
    const int ns = cut_batch(K, n, target, ctas, nullptr);
    if (ns == -1) return -1;
    if (ns >= 0) break;
    target += (target + 31) / 32;                                     // +3 % and try again
  }
  return cut_batch(K, n, target, ctas, bt);
}

// out[g*DA + o][i] = sum_c partials[g][c][o][i]  (fixed order)
__global__ void wgrad_reduce_kernel(const float* __restrict__ partials, int ctas, int64_t tile, float* __restrict__ out,
                                    int64_t ld_out, int DA, int DB) {
  const int64_t idx = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int g = blockIdx.y;
  if (idx >= tile) return;
  const float* p = partials + (int64_t)g * ctas * tile + idx;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < ctas; ++c) {
    const float4 v = __ldcs(reinterpret_cast<const float4*>(p + (int64_t)c * tile));
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  const int64_t o = (idx >> 5) % DA, i = (idx >> 5) / DA * 32 + (idx & 31);         // blocked -> row-major (see the epilogue)
  *reinterpret_cast<float4*>(out + ((int64_t)g * DA + o) * ld_out + i) = s;
}

inline int ctas_for(int64_t K, int groups, int tiles) {
  int per_group = kNumSMsWgrad / (groups * tiles);
  if (per_group < 1) per_group = 1;
  const int64_t chunks = (K + BK - 1) / BK;
  // every CTA column writes (and the reduction re-reads) a full DA x DB partial tile -- 256 KB at D = 256 -- so a short
  // reduction is not spread thinner than 4 pipeline chunks (128 rows) per CTA.
  const int64_t want = (chunks + 3) / 4;
  if (want < per_group) per_group = (int)(want < 1 ? 1 : want);
  return per_group;
}

template <int DA, int DB>
int launch(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t K, int groups, float* out, int64_t ld_out,
           float* ws, cudaStream_t st) {
  using F = Cfg<DA, DB>;
  static alignn::DeviceOnce configured; int cfg_dev;
  if (configured.needed(&cfg_dev)) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_bf16x3_kernel<DA, DB>, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM);
    if (e != cudaSuccess) return record_cuda_error((int)e);
    configured.done(cfg_dev);
  }
  const int ctas = ctas_for(K, groups, F::TILES);
  int64_t rows = (K + ctas - 1) / ctas;
  rows = (rows + BK - 1) / BK * BK;               // slabs start on a stage boundary
  // cooperative launch: ctas * groups * TILES <= kNumSMs CTAs of one per SM, so the in-kernel grid barrier before the
  // split-K reduction is legal; if the device cannot co-schedule them (MPS slice, smaller part) fall back to two launches
  static int coop_ok = -1;
  if (coop_ok < 0) {
    int dev = 0, sms = 0, per_sm = 0, coop = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wgrad_bf16x3_kernel<DA, DB>, THREADS, F::SMEM);
    coop_ok = (coop && (int64_t)sms * per_sm >= kNumSMsWgrad) ? 1 : 0;
  }
  int rows_i = (int)rows;
  if (coop_ok) {
    float* ws_p = ws;
    void* args[] = {(void*)&A, (void*)&lda, (void*)&B, (void*)&ldb, (void*)&K, (void*)&rows_i, (void*)&ws_p, (void*)&out, (void*)&ld_out};
    cudaError_t e = cudaLaunchCooperativeKernel((const void*)wgrad_bf16x3_kernel<DA, DB>, dim3(ctas, groups, F::TILES), dim3(THREADS), args,
                                                (size_t)F::SMEM, st);
    if (e != cudaSuccess) return record_cuda_error((int)e);
    return check_launch();
  }
  wgrad_bf16x3_kernel<DA, DB><<<dim3(ctas, groups, F::TILES), THREADS, F::SMEM, st>>>(A, lda, B, ldb, K, rows_i, ws, nullptr, 0);
  int rc = check_launch();
  if (rc != ALIGNN_OK) return rc;
  const int64_t tile = (int64_t)DA * DB;
  wgrad_reduce_kernel<<<dim3((unsigned)((tile / 4 + 255) / 256), groups), 256, 0, st>>>(ws, ctas, tile, out, ld_out, DA, DB);
  return check_launch();
}

// supported (DA, DB): square conv shapes and the embedding-MLP shapes (inputs zero-padded to a multiple of 32)
inline bool shape_ok(int DA, int DB) {
  if (DA == DB) return DA == 32 || DA == 64 || DA == 128 || DA == 256;
  return (DA == 256 && (DB == 64 || DB == 96)) || (DA == 64 && (DB == 96 || DB == 32)) || (DA == 32 && (DB == 64 || DB == 96));
}

}  // namespace wgrad
}  // namespace alignn

constexpr int kBatchNeedsFallback = -1000;     // internal: cooperative launch refused, run the problems one by one

template <int D>
static int launch_batch(const alignn::wgrad::Batch& bt, float* ws, cudaStream_t st) {
  using namespace alignn::wgrad;
  using F = Cfg<D, D>;
  static alignn::DeviceOnce configured; int cfg_dev;
  if (configured.needed(&cfg_dev)) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_batch_kernel<D, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM);
    if (e != cudaSuccess) return alignn::record_cuda_error((int)e);
    configured.done(cfg_dev);
  }
  void* args[] = {(void*)&bt, (void*)&ws};
  cudaError_t e = cudaLaunchCooperativeKernel((const void*)wgrad_batch_kernel<D, D>, dim3(kNumSMsWgrad / F::TILES, F::TILES), dim3(THREADS), args,
                                              (size_t)F::SMEM, st);
  if (e == cudaErrorCooperativeLaunchTooLarge) {     // the device cannot co-schedule the grid right now (MPS slice, ...)
    (void)cudaGetLastError();
    return kBatchNeedsFallback;
  }
  if (e != cudaSuccess) return alignn::record_cuda_error((int)e);
  return alignn::check_launch();
}

extern "C" {

size_t alignn_b200_wgrad_workspace_bytes(int64_t K, int DA, int DB, int groups) {
  if (K < 0 || groups < 1 || !alignn::wgrad::shape_ok(DA, DB)) return 0;
  return (size_t)alignn::wgrad::ctas_for(K, groups, alignn::wgrad::tiles_of(DA, DB)) * groups * DA * DB * sizeof(float);
}

size_t alignn_b200_wgrad_batch_workspace_bytes(const alignn_b200_wgrad_problem* problems, int n, int D) {
  using namespace alignn::wgrad;
  if (!problems || n < 1 || n > kMaxProblems || !shape_ok(D, D)) return 0;
  int64_t K[kMaxProblems];
  for (int p = 0; p < n; ++p) { if (problems[p].K < 0) return 0; K[p] = problems[p].K; }
  const int ns = plan_batch(K, n, kNumSMsWgrad / tiles_of(D, D), nullptr);
  return ns < 0 ? 0 : (size_t)(ns > 0 ? ns : 1) * D * D * sizeof(float);
}

int alignn_b200_wgrad_batch(const alignn_b200_wgrad_problem* problems, int n, int D, void* workspace, size_t workspace_bytes,
                            alignn_stream_t stream) {
  using namespace alignn::wgrad;
  if (!problems || n < 1) return ALIGNN_ERR_BAD_ARG;
  if (!shape_ok(D, D)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (n > kMaxProblems) return ALIGNN_ERR_BAD_ARG;
  int64_t K[kMaxProblems];
  static thread_local Batch bt;
  for (int p = 0; p < n; ++p) {
    const alignn_b200_wgrad_problem& q = problems[p];
    if (q.K < 0 || !q.out || q.ld_out < D || (q.ld_out % 4) || ((uintptr_t)q.out & 15)) return ALIGNN_ERR_BAD_ARG;
    if (q.K > 0 && (!q.A || !q.B || q.lda < D || q.ldb < D || (q.lda % 4) || (q.ldb % 4) || ((uintptr_t)q.A & 15) || ((uintptr_t)q.B & 15)))
      return ALIGNN_ERR_BAD_ARG;
    if (q.K >= ((int64_t)1 << 31) * BK) return ALIGNN_ERR_BAD_ARG;
    K[p] = q.K;
    bt.prob[p].A = q.A; bt.prob[p].B = q.B; bt.prob[p].out = q.out;
    bt.prob[p].lda = q.lda; bt.prob[p].ldb = q.ldb; bt.prob[p].ld_out = q.ld_out; bt.prob[p].K = q.K;
  }
  const int ns = plan_batch(K, n, kNumSMsWgrad / tiles_of(D, D), &bt);
  if (ns < 0) return ALIGNN_ERR_BAD_ARG;
  if (!workspace || workspace_bytes < (size_t)(ns > 0 ? ns : 1) * D * D * sizeof(float)) return ALIGNN_ERR_WORKSPACE;
  static int coop_ok = -1;
  if (coop_ok < 0) {
    int dev = 0, sms = 0, coop = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    coop_ok = (coop && sms >= kNumSMsWgrad) ? 1 : 0;
  }
  auto one_by_one = [&]() -> int {   // no co-scheduled grid on this device: one launch per problem through the single-problem path
    for (int p = 0; p < n; ++p) {
      const alignn_b200_wgrad_problem& q = problems[p];
      if (workspace_bytes < alignn_b200_wgrad_workspace_bytes(q.K, D, D, 1)) return ALIGNN_ERR_WORKSPACE;
      int rc = alignn_b200_wgrad(q.A, q.lda, q.B, q.ldb, q.K, D, D, 1, q.out, q.ld_out, workspace, workspace_bytes, stream);
      if (rc != ALIGNN_OK) return rc;
    }
    return ALIGNN_OK;
  };
  if (!coop_ok) return one_by_one();
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = reinterpret_cast<float*>(workspace);
  int rc = ALIGNN_ERR_UNSUPPORTED_D;
  switch (D) {
    case 256: rc = launch_batch<256>(bt, ws, st); break;
    case 128: rc = launch_batch<128>(bt, ws, st); break;
    case 64: rc = launch_batch<64>(bt, ws, st); break;
    case 32: rc = launch_batch<32>(bt, ws, st); break;
  }
  if (rc == kBatchNeedsFallback) {
    coop_ok = 0;
    return one_by_one();
  }
  return rc;
}

int alignn_b200_wgrad(const float* A, int64_t lda, const float* B, int64_t ldb, int64_t K, int DA, int DB, int groups,
                      float* out, int64_t ld_out, void* workspace, size_t workspace_bytes, alignn_stream_t stream) {
  using namespace alignn::wgrad;
  if (K < 0 || groups < 1 || !out || ld_out < DB || (ld_out % 4)) return ALIGNN_ERR_BAD_ARG;
  if (!shape_ok(DA, DB)) return ALIGNN_ERR_UNSUPPORTED_D;
  if (K > 0 && (!A || !B || lda < (int64_t)groups * DA || ldb < DB || (lda % 4) || (ldb % 4) || ((uintptr_t)A & 15) ||
                ((uintptr_t)B & 15)))
    return ALIGNN_ERR_BAD_ARG;
  if (K >= ((int64_t)1 << 31) * BK) return ALIGNN_ERR_BAD_ARG;
  if (!workspace || workspace_bytes < alignn_b200_wgrad_workspace_bytes(K, DA, DB, groups)) return ALIGNN_ERR_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = reinterpret_cast<float*>(workspace);
#define WG(a, b) if (DA == a && DB == b) return launch<a, b>(A, lda, B, ldb, K, groups, out, ld_out, ws, st)
  WG(256, 256); WG(128, 128); WG(64, 64); WG(32, 32);
  WG(256, 64); WG(256, 96); WG(64, 96); WG(64, 32); WG(32, 64); WG(32, 96);
#undef WG
  return ALIGNN_ERR_UNSUPPORTED_D;
}

}  // extern "C"
