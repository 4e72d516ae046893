// STAGED WORK (see egc_fused.h): edge-gate GEMM + gate + segment sums in ONE persistent wgmma kernel.
//
//   m_e   = edge_gate(y)_e + P[src_e, 0:d] + P[dst_e, 2d:3d]            (alignn.py:100-101)
//   sig_e = sigmoid(m_e)                                                  (:103)
//   S_v   = sum_{e -> v} sig_e ;  Sh_v = sum_{e -> v} sig_e * P[src_e, d:2d]     (:105-108)
//   h_v   = Sh_v / (S_v + eps) ;  x'_v = P[v, 3d:4d] + h_v                (:109-110)
//   edge tail: M = m (training), BatchNorm column sums, or y_out = y + silu(norm(m)) (:123,:127)
//
// Tiles are SEGMENT ALIGNED: a tile is up to 128 consecutive rows of the destination-sorted edge list that form
// whole in-edge segments (host packer below), so every segment sum is finished inside one CTA -- no atomics, fixed
// summation order (the same order as the shipped row-per-warp kernel, which makes M / S / H / x' bit-identical to it).
//
// Warp roles: warps 0-3 = MMA warpgroup (accumulator tile in scratch, acc_sm90.cuh), then the epilogue warps, then 8 loaders
// (gather y rows by edge id, fp32 -> bf16 hi/lo planes; the weight image arrives by cp.async.bulk).
// Epilogue, per 32-column chunk of the [128 x d] accumulator:
//   row phase    (thread = edge row): accumulator row, gather the three P slices of the row (128 B each),
//                m, M store, sigmoid; sigma / Bh / m go to a padded smem staging tile;
//   column phase (thread = column x row group): per-segment sums over consecutive staged rows -> S, H, x' rows
//                (coalesced 128 B), BatchNorm column sums of m, m^2 into per-warp smem accumulators.
// LayerNorm: m is written back into the accumulator during the row phase, then two more accumulator passes
// give the two-pass variance and the normalised output, all by the thread that owns the row.
#include <atomic>

#include "../tc_common.cuh"
#include "acc_sm90.cuh"
#include "alignn_b200.h"
#include "egc_fused.h"

namespace alignn {
namespace fused {

constexpr int BM = ALIGNN_FUSED_TILE_ROWS;
constexpr int BK = 32;
constexpr int STAGES = 3;
constexpr int LOAD_WARPS = 8;
constexpr int GROUP_THREADS = 128;            // one epilogue group = 4 warps = one thread per tile row
constexpr uint32_t LBO = 128;
constexpr uint32_t SBO = (BK / 8) * 128;
constexpr int kSMs = 132;

std::atomic<int> g_last_cuda_error{0};   // shared with egc_bwd_fused_tc.cu

// EG = number of epilogue groups.  With two groups the column chunks alternate between them, so one group's row
// phase (L2 gathers, MUFU) overlaps the other's column phase; chunks are then 16 columns wide to keep the staging
// tiles inside the shared-memory budget.
template <int D, int EG>
struct Cfg {
  static constexpr int EPI_WARPS = 4 * EG;
  static constexpr int THREADS = 32 * (4 + EPI_WARPS + LOAD_WARPS);   // 512 / 640
  static constexpr int CC = 32 / EG;            // columns per epilogue chunk
  static constexpr int NG = GROUP_THREADS / CC; // row groups of the column phase (4 / 8)
  static constexpr int STG = CC + 4;            // staging row stride in floats (16-byte rows, conflict-free both ways)
  static constexpr int A_PLANE = BM * BK * 2;
  static constexpr int B_PLANE = D * BK * 2;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int PIPE_BYTES = STAGES * STAGE;
  static constexpr int STG_OFF = PIPE_BYTES;                    // per group: sigma | Bh | m   [3][BM][STG] floats
  static constexpr int STG_GROUP = 3 * BM * STG * 4;
  static constexpr int STAT_OFF = STG_OFF + EG * STG_GROUP;     // [NG][2][D] floats (a column belongs to one group)
  static constexpr int STAT_BYTES = NG * 2 * D * 4;
  static constexpr int VEC_OFF = STAT_OFF + STAT_BYTES;         // bias | e_w | e_b
  static constexpr int VEC_BYTES = 3 * D * 4;
  static constexpr int SEG_OFF = VEC_OFF + VEC_BYTES;           // per group: [BM + 1] tile-local segment starts
  static constexpr int SEG_GROUP = ((BM + 1) * 4 + 15) / 16 * 16;
  static constexpr int XCH_OFF = SEG_OFF + EG * SEG_GROUP;      // [EG][BM] floats: LayerNorm row statistics exchange
  static constexpr int XCH_BYTES = EG * BM * 4;
  static constexpr int BAR_OFF = XCH_OFF + XCH_BYTES;
  static constexpr int SMEM = BAR_OFF + 128;
  static_assert(SMEM <= 232448, "shared memory budget of one sm_90 CTA");
  static_assert(D % (EG * CC) == 0, "chunks must tile the row");
};

__host__ __device__ constexpr int plane_off(int r, int k) { return (r >> 3) * (int)SBO + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2; }

// loader thread -> (row, float4 index along K) of the 128 x 32 fp32 chunk for its i-th load (gemm_tc.cu mapping)
__device__ __forceinline__ void a_coord(int i, int lt, int& row, int& kq) {
  const int w = lt >> 5, lane = lt & 31;
  const int u = i * LOAD_WARPS + w;
  row = (u >> 1) * 8 + ((lane >> 1) & 7);
  kq = (u & 1) * 4 + (lane >> 4) * 2 + (lane & 1);
}

// named barriers: 1 + group for one epilogue group, 3 for all epilogue warps
__device__ __forceinline__ void group_bar(int grp) { asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(GROUP_THREADS) : "memory"); }
template <int EG>
__device__ __forceinline__ void all_epi_bar() { asm volatile("bar.sync 3, %0;" ::"n"(EG * GROUP_THREADS) : "memory"); }

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }   // as common.cuh
__device__ __forceinline__ float silu_(float u) { return u * sigmoidf_(u); }

template <int D, int EG>
__global__ void __launch_bounds__(Cfg<D, EG>::THREADS, 1)
egc_forward_fused_kernel(const alignn_b200_egc_fused_fwd_args a, float* __restrict__ scratch_all) {
  using F = Cfg<D, EG>;
  constexpr int CC = F::CC, STG = F::STG, NG = F::NG, EPI_WARPS = F::EPI_WARPS;
  extern __shared__ __align__(128) uint8_t smem[];
  float* stat = reinterpret_cast<float*>(smem + F::STAT_OFF);
  float* vec = reinterpret_cast<float*>(smem + F::VEC_OFF);
  float* xch = reinterpret_cast<float*>(smem + F::XCH_OFF);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + F::BAR_OFF);
  uint64_t* empty = full + STAGES;
  uint64_t* tfull = empty + STAGES;
  uint64_t* tempty = tfull + 2;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int nk = D / BK;
  const int total = a.num_tiles;
  const int4* tiles = reinterpret_cast<const int4*>(a.tiles);    // {v0, nseg, p0, rows}

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full[s], LOAD_WARPS + 1); tc::mbar_init(&empty[s], 4); }
    for (int b = 0; b < 2; ++b) { tc::mbar_init(&tfull[b], 128); tc::mbar_init(&tempty[b], EPI_WARPS); }
    tc::mbar_fence_init();
  }
  __syncthreads();
  const uint32_t tmem = 0;                                  // accumulator "address": see acc_sm90.cuh
  float* const scr = scratch_all + (size_t)blockIdx.x * staged_acc::kRows * 2 * D;

  if (warp >= 4 + EPI_WARPS) {
    // ================= loaders: gather y rows by edge id, split to bf16 hi/lo planes =================
    const int lt = tid - 32 * (4 + EPI_WARPS);          // 0..255
    constexpr int PF = 3;
    float4 buf[PF][4];
    int soff[4], arow[4], akq[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      a_coord(i, lt, arow[i], akq[i]);
      soff[i] = plane_off(arow[i], akq[i] * 4);
    }
    const int my_tiles = (total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int nchunks = my_tiles * nk;
    int l_tile = blockIdx.x, l_kc = 0;
    const float* lp[4];
    bool lval[4];
    // edge ids of the NEXT tile are fetched while the current one streams (descriptor -> in_eid is a dependent chain)
    int ne[4];
    bool nv[4];
    auto fetch_rows = [&](int tile) {
      if (tile < total) {
        const int4 t = __ldg(tiles + tile);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          nv[i] = arow[i] < t.w;
          const int p = t.z + arow[i];
          ne[i] = nv[i] ? (a.in_eid ? __ldg(a.in_eid + p) : p) : 0;
        }
      }
    };
    auto set_tile_ptrs = [&]() {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        lval[i] = nv[i];
        lp[i] = a.y + (int64_t)ne[i] * D + akq[i] * 4;
      }
    };
    auto load_next = [&](float4 (&v)[4]) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[i] = lval[i] ? __ldcs(reinterpret_cast<const float4*>(lp[i])) : make_float4(0.f, 0.f, 0.f, 0.f);
        lp[i] += BK;
      }
      if (++l_kc == nk) {
        l_kc = 0;
        l_tile += gridDim.x;
        if (l_tile < total) { set_tile_ptrs(); fetch_rows(l_tile + gridDim.x); }
      }
    };
    if (nchunks > 0) { fetch_rows(l_tile); set_tile_ptrs(); fetch_rows(l_tile + gridDim.x); }
#pragma unroll
    for (int j = 0; j < PF; ++j)
      if (j < nchunks) load_next(buf[j]);
    int s = 0, ph = 0, s_kc = 0;
    const uint8_t* wimg = reinterpret_cast<const uint8_t*>(a.w_image);
    for (int c0 = 0; c0 < nchunks; c0 += PF) {
#pragma unroll
      for (int j = 0; j < PF; ++j) {
        const int c = c0 + j;
        if (c < nchunks) {
          if (c >= STAGES) tc::mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * F::STAGE;
          if (lt == 0) {   // weight chunk: one contiguous bulk copy (both planes), counted in bytes on full[s]
            tc::mbar_arrive_expect_tx(&full[s], 2 * F::B_PLANE);
            staged_acc::copy_weight_chunk<D, nk>(st + 2 * F::A_PLANE, wimg, s_kc, &full[s]);
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint2 hi, lo;
            tc::split4(buf[j][i], hi, lo);
            *reinterpret_cast<uint2*>(st + soff[i]) = hi;
            *reinterpret_cast<uint2*>(st + F::A_PLANE + soff[i]) = lo;
          }
          if (c + PF < nchunks) load_next(buf[j]);
          tc::fence_async_smem();
          __syncwarp();
          if ((lt & 31) == 0) tc::mbar_arrive(&full[s]);
          if (++s_kc == nk) s_kc = 0;
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ================= epilogue =================
    const int q = warp & 3;                   // this warp's 32 tile rows of the accumulator
    const int grp = (warp - 4) >> 2;          // epilogue group: owns chunks grp, grp + EG, ...
    const int et = q * 32 + lane;             // tile row owned in the row phase (and: which seg[] entry it fills)
    const int ea = grp * GROUP_THREADS + et;  // index among all epilogue threads
    const int col = et % CC;                  // column phase: this thread's column inside the chunk ...
    const int rg = et / CC;                   // ... and its row group (segments rg, rg + NG, ...; stat rows of group rg)
    float* sig = reinterpret_cast<float*>(smem + F::STG_OFF + grp * F::STG_GROUP);
    float* sgc = sig + BM * STG;
    float* mst = sig + 2 * BM * STG;
    int* seg = reinterpret_cast<int*>(smem + F::SEG_OFF + grp * F::SEG_GROUP);
    float* bias_s = vec;
    float* ew_s = vec + D;
    float* eb_s = vec + 2 * D;
    const bool stats = a.norm_edges == ALIGNN_NORM_STATS && a.partials != nullptr;
    const bool affine_out = a.norm_edges == ALIGNN_NORM_AFFINE && a.y_out != nullptr;
    const bool layer_out = a.norm_edges == ALIGNN_NORM_LAYER && a.y_out != nullptr;
    for (int i = ea; i < D; i += EG * GROUP_THREADS) {
      bias_s[i] = a.bias ? a.bias[i] : 0.f;
      ew_s[i] = a.e_w ? a.e_w[i] : 0.f;
      eb_s[i] = a.e_b ? a.e_b[i] : 0.f;
    }
    for (int i = ea; i < NG * 2 * D; i += EG * GROUP_THREADS) stat[i] = 0.f;
    all_epi_bar<EG>();                        // vec / stat initialised for every group

    // per-tile row metadata, fetched one tile ahead (descriptor -> in_eid -> src/dst is a dependent chain)
    int4 n_desc = make_int4(0, 0, 0, 0);
    int n_e = 0, n_s = 0, n_t = 0, n_seg = 0, n_seg_last = 0;
    auto fetch_meta = [&](int tile) {
      if (tile < total) {
        n_desc = __ldg(tiles + tile);
        const bool valid = et < n_desc.w;
        const int p = n_desc.z + et;
        n_e = valid ? (a.in_eid ? __ldg(a.in_eid + p) : p) : 0;
        n_s = valid ? __ldg(a.src + n_e) : 0;
        n_t = valid ? __ldg(a.dst + n_e) : 0;
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
      const bool valid = et < rows;
      const int64_t e = n_e, s = n_s, t = n_t;
      // (the group's last barrier of the previous tile already fenced its reads of seg[])
      if (et <= nseg) seg[et] = n_seg;
      if (et == 0 && nseg == BM) seg[BM] = n_seg_last;
      fetch_meta(tile + gridDim.x);
      tc::mbar_wait(&tfull[acc], (lt >> 1) & 1);
            const uint32_t trow = tmem + ((uint32_t)(q * 32) << 16) + (uint32_t)(acc * D);
      const float* pa = a.P + s * 4 * D;              // [e_src | Bh] of the source row
      const float* pb = a.P + t * 4 * D + 2 * D;      // e_dst of the destination row
      float row_sum = 0.f;
#pragma unroll 1
      for (int c0 = grp * CC; c0 < D; c0 += EG * CC) {
        // ---------------- row phase ----------------
        float v[CC];
        staged_acc::ld<CC>(scr, 2 * D, trow + (uint32_t)c0, v);
        float* srow = sig + et * STG;
        float* crow = sgc + et * STG;
        float* mrow = mst + et * STG;
        if (valid) {
#pragma unroll
          for (int j = 0; j < CC; j += 4) {
            const float4 a4 = __ldg(reinterpret_cast<const float4*>(pa + c0 + j));
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(pb + c0 + j));
            const float4 bi = *reinterpret_cast<const float4*>(bias_s + c0 + j);
            // same association as the shipped path: (acc + bias) from the GEMM epilogue, then + (e_src + e_dst)
            v[j] = (v[j] + bi.x) + (a4.x + b4.x);
            v[j + 1] = (v[j + 1] + bi.y) + (a4.y + b4.y);
            v[j + 2] = (v[j + 2] + bi.z) + (a4.z + b4.z);
            v[j + 3] = (v[j + 3] + bi.w) + (a4.w + b4.w);
          }
          if (a.M) {
            float4* mo = reinterpret_cast<float4*>(a.M + e * D + c0);
#pragma unroll
            for (int j = 0; j < CC; j += 4) __stcs(mo + j / 4, make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]));
          }
          if (affine_out) {
            float4* yo = reinterpret_cast<float4*>(a.y_out + e * D + c0);
            const float4* yi = reinterpret_cast<const float4*>(a.y + e * D + c0);
#pragma unroll
            for (int j = 0; j < CC; j += 4) {
              const float4 w4 = *reinterpret_cast<const float4*>(ew_s + c0 + j);
              const float4 s4 = *reinterpret_cast<const float4*>(eb_s + c0 + j);
              float4 o = make_float4(silu_(v[j] * w4.x + s4.x), silu_(v[j + 1] * w4.y + s4.y),
                                     silu_(v[j + 2] * w4.z + s4.z), silu_(v[j + 3] * w4.w + s4.w));
              if (a.residual) {
                const float4 r4 = __ldcs(yi + j / 4);
                o.x += r4.x; o.y += r4.y; o.z += r4.z; o.w += r4.w;
              }
              __stcs(yo + j / 4, o);
            }
          }
          if (layer_out) {
#pragma unroll
            for (int j = 0; j < CC; ++j) row_sum += v[j];
          }
          if (stats) {
#pragma unroll
            for (int j = 0; j < CC; j += 4) *reinterpret_cast<float4*>(mrow + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
          }
#pragma unroll
          for (int j = 0; j < CC; j += 4) {
            const float4 c4 = __ldg(reinterpret_cast<const float4*>(pa + D + c0 + j));
            const float4 g4 = make_float4(sigmoidf_(v[j]), sigmoidf_(v[j + 1]), sigmoidf_(v[j + 2]), sigmoidf_(v[j + 3]));
            *reinterpret_cast<float4*>(srow + j) = g4;
            *reinterpret_cast<float4*>(crow + j) = c4;   // the product is formed by the FMA of the column phase
          }
        } else if (stats) {                    // rows past the tile's end must not count in the column sums
#pragma unroll
          for (int j = 0; j < CC; j += 4) *reinterpret_cast<float4*>(mrow + j) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // LayerNorm: keep m in the accumulator for the two passes below.  The store is per warp
        // (.sync.aligned), so it sits outside the `valid` branch; rows past the tile's end store junk nobody reads.
        if (layer_out) staged_acc::st<CC>(scr, 2 * D, trow + (uint32_t)c0, v);
        group_bar(grp);
        // ---------------- column phase: thread = (column `col`, row group `rg`) ----------------
        for (int j = rg; j < nseg; j += NG) {
          const int64_t vtx = v0 + j;
          const float dv = __ldg(a.P + vtx * 4 * D + 3 * D + c0 + col);
          const int r0 = seg[j], r1 = seg[j + 1];
          float s1 = 0.f, s2 = 0.f;
          for (int r = r0; r < r1; ++r) {
            const float g = sig[r * STG + col];
            s1 += g;
            s2 = fmaf(sgc[r * STG + col], g, s2);   // Bh * sigma, fused and in edge order like the row-per-warp kernel
          }
          const float h = s2 / (s1 + a.gate_eps);
          a.XP[vtx * D + c0 + col] = dv + h;
          if (a.S) {
            a.S[vtx * D + c0 + col] = s1;
            a.H[vtx * D + c0 + col] = h;
          }
        }
        if (stats) {
          float t1 = 0.f, t2 = 0.f;
#pragma unroll 8
          for (int r = rg * (BM / NG); r < (rg + 1) * (BM / NG); ++r) {
            const float x = mst[r * STG + col];
            t1 += x;
            t2 += x * x;
          }
          stat[(rg * 2 + 0) * D + c0 + col] += t1;
          stat[(rg * 2 + 1) * D + c0 + col] += t2;
        }
        group_bar(grp);                        // staging tile (and, after the last chunk, seg[]) free again
      }
      if (layer_out) {
        // two more passes over the row in the accumulator: variance about the mean (two-pass, like torch), then the output.
        // Every lane runs the per-warp accumulator load; only rows inside the tile store.  With two groups each
        // holds the statistics of its own chunks: exchange through shared memory.
        float mean;
        if constexpr (EG == 1) {
          mean = row_sum * (1.f / D);
        } else {
          xch[grp * BM + et] = row_sum;
          all_epi_bar<EG>();
          float tot = 0.f;
#pragma unroll
          for (int g2 = 0; g2 < EG; ++g2) tot += xch[g2 * BM + et];
          mean = tot * (1.f / D);
          all_epi_bar<EG>();
        }
        float qsum = 0.f;
#pragma unroll 1
        for (int c0 = grp * CC; c0 < D; c0 += EG * CC) {
          float v[CC];
          staged_acc::ld<CC>(scr, 2 * D, trow + (uint32_t)c0, v);
#pragma unroll
          for (int j = 0; j < CC; ++j) { const float dlt = v[j] - mean; qsum += dlt * dlt; }
        }
        if constexpr (EG > 1) {
          xch[grp * BM + et] = qsum;
          all_epi_bar<EG>();
          qsum = 0.f;
#pragma unroll
          for (int g2 = 0; g2 < EG; ++g2) qsum += xch[g2 * BM + et];
          all_epi_bar<EG>();
        }
        const float rstd = rsqrtf(qsum * (1.f / D) + a.ln_eps);
#pragma unroll 1
        for (int c0 = grp * CC; c0 < D; c0 += EG * CC) {
          float v[CC];
          staged_acc::ld<CC>(scr, 2 * D, trow + (uint32_t)c0, v);
          if (valid) {
            float4* yo = reinterpret_cast<float4*>(a.y_out + e * D + c0);
            const float4* yi = reinterpret_cast<const float4*>(a.y + e * D + c0);
#pragma unroll
            for (int j = 0; j < CC; j += 4) {
              const float4 w4 = *reinterpret_cast<const float4*>(ew_s + c0 + j);
              const float4 s4 = *reinterpret_cast<const float4*>(eb_s + c0 + j);
              float4 o = make_float4(silu_((v[j] - mean) * rstd * w4.x + s4.x), silu_((v[j + 1] - mean) * rstd * w4.y + s4.y),
                                     silu_((v[j + 2] - mean) * rstd * w4.z + s4.z), silu_((v[j + 3] - mean) * rstd * w4.w + s4.w));
              if (a.residual) {
                const float4 r4 = __ldcs(yi + j / 4);
                o.x += r4.x; o.y += r4.y; o.z += r4.z; o.w += r4.w;
              }
              __stcs(yo + j / 4, o);
            }
          }
        }
      }
      __threadfence_block();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&tempty[acc]);
    }
    if (stats) {                               // fixed-order sum over the row groups -> one partial row per CTA
      all_epi_bar<EG>();
      float* out_row = a.partials + (int64_t)blockIdx.x * 2 * D;
      for (int i = ea; i < 2 * D; i += EG * GROUP_THREADS) {
        const int which = i / D, c = i % D;
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < NG; ++w) t += stat[(w * 2 + which) * D + c];
        out_row[i] = t;
      }
    }
  } else {
    // ================= MMA warpgroup (warps 0-3): the accumulator tile in scratch =================
    staged_acc::mma_warpgroup<D, F::STAGE, F::A_PLANE, STAGES>(smem, full, empty, tfull, tempty, scr, total);
  }
}

template <int D, int EG>
int launch(const alignn_b200_egc_fused_fwd_args& a) {
  using F = Cfg<D, EG>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(egc_forward_fused_kernel<D, EG>, cudaFuncAttributeMaxDynamicSharedMemorySize, F::SMEM);
    if (e != cudaSuccess) { g_last_cuda_error.store((int)e); return ALIGNN_ERR_CUDA; }
    configured = true;
  }
  const int grid = a.num_tiles < kSMs ? a.num_tiles : kSMs;
  cudaError_t se;
  float* scr = staged_acc::scratch((size_t)grid * staged_acc::kRows * 2 * D * sizeof(float), &se);
  if (!scr) { g_last_cuda_error.store((int)se); return ALIGNN_ERR_CUDA; }
  egc_forward_fused_kernel<D, EG><<<grid, F::THREADS, F::SMEM, (cudaStream_t)a.stream>>>(a, scr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { g_last_cuda_error.store((int)e); return ALIGNN_ERR_CUDA; }
  return ALIGNN_OK;
}

}  // namespace fused
}  // namespace alignn

extern "C" {

int64_t alignn_b200_segment_tiles_host(const int32_t* in_ptr, int64_t num_nodes, int32_t* tiles, int64_t capacity) {
  if (num_nodes < 0 || (num_nodes > 0 && !in_ptr) || capacity < 0) return -1;
  constexpr int R = ALIGNN_FUSED_TILE_ROWS;
  int64_t n = 0, v0 = 0;
  while (v0 < num_nodes) {
    int64_t v1 = v0;
    int32_t rows = 0;
    while (v1 < num_nodes && v1 - v0 < R) {
      const int32_t deg = in_ptr[v1 + 1] - in_ptr[v1];
      if (deg < 0) return -1;
      if (rows + deg > R) break;
      rows += deg;
      ++v1;
    }
    if (v1 == v0) return -2;                 // one node with more than 128 in-edges: no segment-aligned tile holds it
    if (tiles) {
      if (n >= capacity) return -1;
      tiles[4 * n + 0] = (int32_t)v0;
      tiles[4 * n + 1] = (int32_t)(v1 - v0);
      tiles[4 * n + 2] = in_ptr[v0];
      tiles[4 * n + 3] = rows;
    }
    ++n;
    v0 = v1;
  }
  return n;
}

int alignn_b200_egc_fused_partial_rows(int32_t num_tiles) { return num_tiles < alignn::fused::kSMs ? num_tiles : alignn::fused::kSMs; }

int alignn_b200_staged_last_cuda_error(void) { return alignn::fused::g_last_cuda_error.load(); }

int alignn_b200_egc_forward_fused(const alignn_b200_egc_fused_fwd_args* a) {
  if (!a) return ALIGNN_ERR_BAD_ARG;
  if (a->struct_size != sizeof(*a)) return ALIGNN_ERR_STRUCT_SIZE;
  if (a->d != 32 && a->d != 64 && a->d != 128 && a->d != 256) return ALIGNN_ERR_UNSUPPORTED_D;
  if (a->Nn < 0 || a->Ne < 0 || a->num_tiles < 0) return ALIGNN_ERR_BAD_ARG;
  if (a->norm_edges != ALIGNN_NORM_STATS && a->norm_edges != ALIGNN_NORM_AFFINE && a->norm_edges != ALIGNN_NORM_LAYER)
    return ALIGNN_ERR_BAD_ARG;
  if (a->Nn == 0) return ALIGNN_OK;
  if (a->num_tiles == 0 || !a->tiles || !a->P || !a->in_ptr || !a->w_image || !a->XP) return ALIGNN_ERR_BAD_ARG;
  if ((a->S == nullptr) != (a->H == nullptr)) return ALIGNN_ERR_BAD_ARG;
  if (a->Ne > 0 && (!a->y || !a->src || !a->dst)) return ALIGNN_ERR_BAD_ARG;
  if (a->norm_edges == ALIGNN_NORM_STATS && (!a->partials || (a->Ne > 0 && !a->M))) return ALIGNN_ERR_BAD_ARG;
  if (a->y_out && (!a->e_w || !a->e_b)) return ALIGNN_ERR_BAD_ARG;
  if (((uintptr_t)a->tiles & 15) != 0) return ALIGNN_ERR_BAD_ARG;   // descriptors are read as int4
  if (a->epilogue_groups != 1 && a->epilogue_groups != 2) return ALIGNN_ERR_BAD_ARG;
#define ALIGNN_FUSED_LAUNCH(DD) (a->epilogue_groups == 2 ? alignn::fused::launch<DD, 2>(*a) : alignn::fused::launch<DD, 1>(*a))
  switch (a->d) {
    case 256: return ALIGNN_FUSED_LAUNCH(256);
    case 128: return ALIGNN_FUSED_LAUNCH(128);
    case 64: return ALIGNN_FUSED_LAUNCH(64);
    default: return ALIGNN_FUSED_LAUNCH(32);
  }
#undef ALIGNN_FUSED_LAUNCH
}

}  // extern "C"
