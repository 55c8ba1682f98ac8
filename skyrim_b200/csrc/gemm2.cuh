// TMA-fed persistent wgmma GEMM (v2 data flow), k_gemm2 / k_gemm2_pair:
//
//   D[M, N] = A[M, K] * W[N, K]^T -> fused epilogue        (optionally per batch)
//
// Both operands arrive as pre-built SWIZZLE_128B "tile images" and are fetched by ONE thread
// with 1-D bulk copies through the TMA engine (cp.async.bulk + mbarrier complete_tx):
//   A image  [ceil(M/128)][K/64][128 rows x 128 B]   fp16 activations, written in this layout
//                                                     by the epilogue of the producing kernel
//   W image  [N/BLOCK_N][K/64][BLOCK_N rows x 128 B]  packed once at weight load
// so no warp ever touches the operands with ld/st.  A schedule (SchedW here, SchedTB in gemm_tb.cuh) decides which
// images a tile's k-blocks come from; the pipeline is the same for all.  Warp roles: 0..7 = two consumer warpgroups,
// 8 = loader.  Warpgroup g issues the wgmma products of rows 64g .. 64g+63 of the 128-row tile
// over all BLOCK_N columns (fp32 accumulators in registers, BLOCK_N / 2 per thread).  At the end of
// a tile both warpgroups stage their accumulators in shared memory — over the operand ring, which
// is drained by then — and the same eight warps run the row-owner epilogue on the staged tile
// (warp%4 selects the 32-row quarter, warp/4 the column partition).  Epilogues re-tile their 32x32
// accumulator blocks through a padded smem patch so that every global access is a full
// 64/128-byte row segment.
#pragma once
#include <climits>
#include <type_traits>

#include "../../include/skyrim_b200.h"
#include "pangu_ops.cuh"
#include "wgmma_ops.cuh"

namespace sky {

constexpr int G2_BLOCK_M = 128;
constexpr int G2_A_BYTES = G2_BLOCK_M * 128;
constexpr int G2_PATCH_LD = 33;    // scalar accessors (odd stride: conflict-free column reads)
constexpr int G2_PATCH_FLOATS = 32 * G2_PATCH_LD;
constexpr int G2_PATCHV_BYTES = 4096;   // 128-bit accessors: 32 rows x 128 B, 16-byte chunk index XOR (row & 7)

// element (row, col) of an fp16 tile image with nkb k-blocks per row tile -> byte offset
__device__ __forceinline__ size_t img_offset(long long row, int col, int nkb) {
  long long tile = row >> 7;
  uint32_t r = (uint32_t)(row & 127);
  return ((size_t)tile * nkb + (col >> 6)) * (size_t)G2_A_BYTES + sw128_offset(r, (col & 63) >> 3) + (col & 7) * 2;
}

// A operand: up to 6 fp16 tile images concatenated along K, so that a concatenation is never materialised (patch
// recovery: concat(skip, x); GraphCast's mesh2grid node update: [v | e0 | e1 | e2]; SFNO: the 3-term fp16 split
// A = [hi | lo | hi], DESIGN.md §2, and the decoder's concat(x, input)).  In a batched launch every segment has its own
// image per batch, batch_stride bytes apart.
struct AOperand {
  const uint8_t* seg[6] = {};
  int nkb[6] = {};                 // k-blocks per row tile of each segment
  long long batch_stride[6] = {};  // bytes between batches of each segment
  int nseg = 0;
  AOperand() = default;
  AOperand(const uint8_t* img, int k) { add(img, k); }
  // appends a segment of k k-blocks per row tile
  AOperand& add(const uint8_t* img, int k, long long bstride = 0) {
    seg[nseg] = img; nkb[nseg] = k; batch_stride[nseg] = bstride; ++nseg;
    return *this;
  }
  // The loader calls this once per k-block, so it is kept short: a single image needs no walk, and the walk over several
  // is done by selects (unused segments have nkb = 0), without branches.
  __device__ const uint8_t* kblock(int batch, int mt, int kb) const {
    if (nseg == 1) return seg[0] + (size_t)batch * batch_stride[0] + ((size_t)mt * nkb[0] + kb) * G2_A_BYTES;
    const uint8_t* p = seg[0];
    long long bs = batch_stride[0];
    int n = nkb[0];
#pragma unroll
    for (int s = 1; s < 6; ++s)
      if (kb >= n) { kb -= n; p = seg[s]; bs = batch_stride[s]; n = nkb[s]; }
    return p + (size_t)batch * bs + ((size_t)mt * n + kb) * G2_A_BYTES;
  }
};

template <int BLOCK_N, int EPI_WARPS>
struct G2Cfg {
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = G2_A_BYTES + B_BYTES;
  static constexpr int PATCH_BYTES = EPI_WARPS * G2_PATCH_FLOATS * 4;
  static constexpr int VEC_BYTES = 3 * 512 * 4;  // smem copies of bias | gamma | beta (LN epilogues), <= 512 floats each
  static constexpr int FIXED = 1024 /*align*/ + 256 /*barriers*/ + PATCH_BYTES + VEC_BYTES;
  static constexpr int MAXS = (232448 - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = MAXS > 6 ? 6 : MAXS;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  // accumulator staging over the drained ring: all 128 rows when they fit, else 64 rows (one warpgroup) at a time
  static constexpr int STG_LD = (BLOCK_N + 31) / 32 * 32 + 4;
  static constexpr int STG_ROWS = 128 * STG_LD * 4 <= RING_BYTES ? 128 : 64;
  static constexpr int SMEM_BYTES = RING_BYTES + FIXED;
  static constexpr int THREADS = (EPI_WARPS + 1) * 32;
  static_assert(BLOCK_N % 8 == 0 && BLOCK_N <= 384, "wgmma N, accumulator registers");
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static_assert(STAGES >= 2, "pipeline depth");
  static_assert(STG_ROWS * STG_LD * 4 <= RING_BYTES, "accumulator staging");
  static_assert(EPI_WARPS == 8, "two consumer warpgroups");
};

struct EpiCtx {
  long long row0;   // first row of this warp's 32-row group
  long long M;
  int lane;
  int batch = 0;    // batch of the tile (batched launches; 0 otherwise)
  int n0;           // first column of the tile in the full N
  int part, nparts; // column-chunk partition among the warps sharing a lane quarter
  float* patch;     // [32][33] floats, private to the warp
  uint32_t patch_s;    // the same patch as a shared-space address
  uint32_t svec_s;     // shared-space address of bias | gamma | beta, vstride floats apart (LN epilogues)
  int vstride = 512;
  int patch_stride = G2_PATCH_FLOATS * 4;   // bytes between the patches of consecutive warps
  // per-row-group scratch an epilogue may cache across the n-tiles of one m-tile (EpiQkvWin: destination row of this lane)
  mutable long long aux_row0 = -1;
  mutable int aux = 0, aux2 = 0;
  // row-statistics exchange with the peer CTA of a column-split pair (k_gemm2_pair); x_own_bar == nullptr elsewhere
  uint64_t* x_own_bar = nullptr;   // completes when the peer's 32 (sum, sum of squares) pairs of this lane quarter landed
  uint32_t x_own_stat = 0;         // shared-space address of this CTA's slot: 32 x {float s, ss}
  uint32_t x_peer_stat = 0, x_peer_bar = 0;   // shared::cluster addresses of the same slot / barrier in the peer CTA
  uint32_t x_parity = 0;
};

// ---------------------------------------------------------------------------------------------------------------
// consumer side shared by the wgmma GEMM kernels
// ---------------------------------------------------------------------------------------------------------------
// Accumulators of warpgroup wg: rows 64 wg .. 64 wg + 63 of the 128-row tile, all BN columns (N > 256: two products of N/2).
template <int BN, bool kBMN = false>
struct WgAcc {
  static constexpr int NI = BN <= 256 ? BN : BN / 2;
  static constexpr int NS = BN / NI;
  float d[NS][NI / 2];
  // zeroed at the start of every tile (rather than a scale-d = 0 first product): the registers are then dead between the
  // staging of one tile and the main loop of the next, i.e. free for the epilogue
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int ni = 0; ni < NS; ++ni)
#pragma unroll
      for (int i = 0; i < NI / 2; ++i) d[ni][i] = 0.f;
  }
  // one k-block: A = 128 rows x 64 halves at a_addr; B = BN rows x 64 halves, K-major, at b_addr, or (kBMN) 64 k-rows x BN
  // columns in 64-column atoms 8 KB apart
  __device__ __forceinline__ void kblock(uint32_t a_addr, uint32_t b_addr, int wg) {
    wgmma_fence();
    const uint64_t da = make_desc_sw128(a_addr + (uint32_t)wg * 8192u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
      for (int ni = 0; ni < NS; ++ni) {
        const uint64_t db = kBMN ? make_desc_sw128_mn(b_addr, 8192) + (uint64_t)(k * (2048 >> 4))
                                 : make_desc_sw128(b_addr + (uint32_t)(ni * NI * 128)) + (uint64_t)(2 * k);
        Wgmma<NI, kBMN>::mma(d[ni], da + 2 * k, db);
      }
    }
    wgmma_commit();
  }
  __device__ __forceinline__ void settle() {
    wgmma_wait<0>();
#pragma unroll
    for (int ni = 0; ni < NS; ++ni) wgmma_fence_operands(d[ni]);
  }
  // fragment -> staging (row-major, ld floats per row); row_off = first row of this warpgroup minus the staging's first row
  __device__ __forceinline__ void dump(uint32_t stg_s, int ld, int row_off) const {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    const uint32_t r = (uint32_t)(16 * w + (l >> 2) + row_off);
    const uint32_t a0 = stg_s + (r * (uint32_t)ld + 2u * (uint32_t)(l & 3)) * 4u, a8 = a0 + 8u * (uint32_t)ld * 4u;
#pragma unroll
    for (int ni = 0; ni < NS; ++ni) {
#pragma unroll
      for (int i = 0; i < NI / 8; ++i) {
        const uint32_t o = (uint32_t)(ni * NI + 8 * i) * 4u;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0 + o), "f"(d[ni][4 * i]), "f"(d[ni][4 * i + 1]) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a8 + o), "f"(d[ni][4 * i + 2]), "f"(d[ni][4 * i + 3]) : "memory");
      }
    }
  }
};

// Main loop of one tile over the stage ring (stage = A tile | B tile).  One wgmma group stays in flight: the stage of
// k-block kb - 1 is released once the products of kb are issued.  empty[] counts the eight consumer warps.
template <int STAGES, int STAGE_BYTES, class Acc>
__device__ __forceinline__ void wg_mainloop(Acc& acc, uint8_t* smem, uint64_t* full, uint64_t* empty, int& s, uint32_t& ph,
                                            int num_kb, int wg, int lane) {
  int prev = -1;
  acc.zero();
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full[s], ph);
    const uint32_t a = smem_u32(smem + s * STAGE_BYTES);
    acc.kblock(a, a + G2_A_BYTES, wg);
    wgmma_wait<1>();
    if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
  acc.settle();
  if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
}

// Stage the accumulators at the base of the (drained) ring and run fn(AccSmem) in every consumer warp whose 32-row quarter
// (warp % 4) is staged; STG_ROWS = 64 stages and finishes one warpgroup's rows at a time.  The caller signals the loader
// afterwards (the ring is free again).
template <int STG_ROWS, class Acc, class Fn>
__device__ __forceinline__ void wg_epilogue(const Acc& acc, uint8_t* smem, int ld, int wg, int warp, int lane, Fn&& fn) {
  const uint32_t stg = smem_u32(smem);
  const int q = warp & 3;
  named_bar_sync(1, 256);   // both warpgroups' products have completed: no wgmma still reads the ring the staging overwrites
#pragma unroll 1
  for (int h = 0; h < 128 / STG_ROWS; ++h) {
    if (STG_ROWS == 128 || wg == h) acc.dump(stg, ld, 64 * wg - h * STG_ROWS);
    named_bar_sync(1, 256);
    if (q * 32 >= h * STG_ROWS && q * 32 < (h + 1) * STG_ROWS)
      fn(AccSmem{stg + (uint32_t)((q * 32 + lane - h * STG_ROWS) * ld) * 4u});
    named_bar_sync(1, 256);
  }
  fence_proxy_async_smem();   // the staging's generic accesses are ordered before the next bulk copies into the ring
}

// ---------------------------------------------------------------------------------------------------------------
// Per-channel statistics of the CTA (SFNO epilogues with kCtaStats)
// ---------------------------------------------------------------------------------------------------------------
// Epilogues that gather per-channel statistics keep them in shared memory for the CTA's whole (persistent) life and flush
// them with ONE fp64 atomic per channel and CTA at kernel end: per-chunk global atomics (26 M on 768 addresses for a
// full-resolution GEMM) were the bottleneck of those epilogues (ncu r2b: 2.0 ms against 1.07 ms for the same GEMM with a
// plain store).  Layout of the CTA accumulators (fp64): sums at [0, 384), sums of squares at [384, 768) of the bias region.
template <class E, class = void> struct has_cta_stats : std::false_type {};
template <class E> struct has_cta_stats<E, std::void_t<decltype(E::kCtaStats)>> : std::true_type {};
constexpr int CTA_STATS_MAX = 384;   // channels: 2 x 384 fp64 accumulators fill the 6 KB bias region
// fp64 accumulators: the order in which the warps of a CTA (and then the CTAs) add their fp32 partial sums is not fixed;
// in fp64 the order changes the result by ~1e-16 relative, i.e. the fp32 scale / shift derived from it are reproducible
// from run to run (fp32 accumulators were not: 1e-7 differences in the statistics)
__device__ __forceinline__ void red_shared_f64(uint32_t addr, double v) {
  asm volatile("red.shared.add.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
template <class Epi>
__device__ __forceinline__ void cta_stats_flush(const Epi& epi, const float* sbias) {
  if constexpr (has_cta_stats<Epi>::value) {
    if (epi.sums) {
      const double* acc = reinterpret_cast<const double*>(sbias);
      for (int i = threadIdx.x; i < 2 * epi.n_valid; i += blockDim.x)
        atomicAdd(epi.sums + i, acc[(i < epi.n_valid ? 0 : CTA_STATS_MAX) + (i < epi.n_valid ? i : i - epi.n_valid)]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Schedules: which bytes the loader fetches for a tile.  The kernel walks the tiles of D[batches][M, N] (n-tile fastest)
// persistently; a schedule maps a tile to (batch, m-tile, n-tile, skip) and issues the bulk copies of its k-blocks.
// ---------------------------------------------------------------------------------------------------------------
struct G2Grid {
  long long M;
  int num_m_tiles, num_n_tiles, batches;
  __host__ __device__ long long num_tiles() const { return (long long)num_m_tiles * num_n_tiles * batches; }
};
struct G2Tile {
  int b, mt, nt;
  bool skip;
  __device__ static G2Tile at(const G2Grid& g, int tile) {
    const int tiles_per_batch = g.num_m_tiles * g.num_n_tiles;
    const int b = tile / tiles_per_batch, t = tile % tiles_per_batch;
    return {b, t / g.num_n_tiles, t % g.num_n_tiles, false};
  }
};

// Weights: D_b = A_b W_b^T with A an AOperand and W the image [batches][N / BLOCK_N][num_kb - w_rep][BLOCK_N rows x 128 B]
// packed at weight load.  w_rep > 0: W = [hi | lo] with w_rep k-blocks each, consumed as hi, hi, lo against A = [hi | lo | hi]
// (the 3-term split of the SFNO GEMMs).
// kTri: batch b only has rows 0 .. b (degree l of a spectrum holds orders m <= l): row tiles that start past row b are
// skipped by every role (their output is multiplied by zeros downstream).  A compile-time choice: the run-time test in
// the consumers' tile loop alone costs registers (and spills) in every other instantiation.
template <bool kTri = false>
struct SchedW {
  static constexpr bool kBMN = false;
  AOperand A;
  const uint8_t* W;
  int num_kb;
  long long w_batch_stride = 0;   // bytes
  int w_rep = 0;
  struct Tile : G2Tile {
    const uint8_t* w;   // the tile's W image: k-block 0 of its batch and n-tile
  };
  template <int BN>
  __device__ Tile tile(const G2Grid& g, int i) const {
    Tile t{G2Tile::at(g, i), nullptr};
    t.skip = kTri && t.mt * G2_BLOCK_M > t.b;
    t.w = W + (size_t)t.b * w_batch_stride + (size_t)t.nt * (num_kb - w_rep) * (BN * 128);
    return t;
  }
  template <int BN>
  __device__ __forceinline__ void issue(uint8_t* dst, uint64_t* full, const Tile& t, int kb, int lane) const {
    constexpr int B_BYTES = BN * 128;
    if (lane == 0) {
      mbar_arrive_expect_tx(full, G2_A_BYTES + B_BYTES);
      bulk_g2s(dst, A.kblock(t.b, t.mt, kb), G2_A_BYTES, full);
      bulk_g2s(dst + G2_A_BYTES, t.w + (size_t)(kb < w_rep ? kb : kb - w_rep) * B_BYTES, B_BYTES, full);
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------
// The TMA-fed persistent GEMM.  One loader warp fills the stage ring (stage = A tile | B tile) through the schedule; two
// consumer warpgroups run the main loop and the epilogue of each tile.  The loader starts the next tile's copies once the
// previous tile's epilogue has left the ring (stg_free); a tile the schedule skips counts for no role.
// kPair (k_gemm2_pair): the two CTAs of a cluster take the same m-tile and n-tiles 0 / 1 (N = 2 BLOCK_N; the persistent
// walk over 2 n-tiles with an even grid gives CTA rank r exactly the tiles (mt, r)), and exchange LayerNorm row statistics
// through distributed shared memory (EpiCtx::x_*).  A 128 x 512 fp32 accumulator is the whole register file of an SM;
// this way the epilogue still sees whole rows.  Exchange slots and barriers are double buffered by tile parity; a CTA
// runs at most one tile ahead of its peer, because its next statistics wait needs the peer's sums of that tile.
// ---------------------------------------------------------------------------------------------------------------
constexpr int G2_EPI_WARPS = 8;
constexpr int G2_PAIR_SMEM = 2048;   // the pair's exchange slots, behind the barrier block

template <class Sched, class Epi, int BLOCK_N, bool kPair>
__device__ __forceinline__ void gemm2_body(const Sched& sc, const Epi& epi, const G2Grid& g) {
  constexpr int EPI_WARPS = G2_EPI_WARPS;
  using Cfg = G2Cfg<BLOCK_N, EPI_WARPS>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* patches = reinterpret_cast<float*>(smem + Cfg::RING_BYTES);
  float* sbias = patches + EPI_WARPS * G2_PATCH_FLOATS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + 3 * 512);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* stg_free = bars + 2 * Cfg::STAGES;   // consumers -> loader: the tile's epilogue has left the ring
  uint64_t* xbar = bars + 2 * Cfg::STAGES + 1;                                          // pair: [2 tile parities][4 lane quarters]
  float* xstat = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);     // pair: [2][4][32 lanes][2]
  static_assert(!kPair || (2 * Cfg::STAGES + 1 + 8) * 8 <= 256, "barrier block");

  // warp index through a shuffle: provably warp-uniform, so the role branches are uniform control flow
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;
  const uint32_t rank = kPair ? cluster_ctarank() : 0u;
  const int num_tiles = (int)g.num_tiles();   // < 2^31 (launch_gemm2)
  constexpr int LOADER = EPI_WARPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], EPI_WARPS); }
    mbar_init(stg_free, EPI_WARPS);
    if (kPair) for (int i = 0; i < 8; ++i) mbar_init(&xbar[i], 1);
    mbar_fence_init();
  }
  if constexpr (Epi::kNeedsBias) if (threadIdx.x < EPI_WARPS * 32)
    for (int i = threadIdx.x; i < BLOCK_N; i += EPI_WARPS * 32) {
      const uint32_t c = rank * BLOCK_N + i;   // this CTA's columns
      sbias[i] = epi.bias[c]; sbias[512 + i] = epi.gamma[c]; sbias[1024 + i] = epi.beta[c];
    }
  if constexpr (has_cta_stats<Epi>::value)
    for (int i = threadIdx.x; i < 3 * 512; i += blockDim.x) sbias[i] = 0.f;
  __syncthreads();
  if (kPair) cluster_sync_all();   // the peer's exchange barriers exist before anything is posted to them

  if (warp == LOADER) {
    int s = 0; uint32_t ph = 0; int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const auto t = sc.template tile<BLOCK_N>(g, tile);
      if (t.skip) continue;
      // the tile's indices are computed while the previous tile's epilogue still runs, not after it has left the ring
      asm volatile("" ::"r"(t.b), "r"(t.mt), "r"(t.nt));
      if (it > 0) mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
      ++it;
      for (int kb = 0; kb < sc.num_kb; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        sc.template issue<BLOCK_N>(smem + s * Cfg::STAGE_BYTES, &full[s], t, kb, lane);
        __syncwarp();
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // ---------------- consumer warpgroups: MMA, then epilogue ----------------
    const int q = warp & 3, part = warp >> 2, wg = warp >> 2;
    EpiCtx ctx;
    ctx.M = g.M; ctx.lane = lane; ctx.part = part; ctx.nparts = EPI_WARPS / 4;
    ctx.patch = patches + warp * G2_PATCH_FLOATS;
    ctx.patch_s = smem_u32(ctx.patch);
    ctx.svec_s = smem_u32(sbias);
    WgAcc<BLOCK_N, Sched::kBMN> acc;
    int s = 0; uint32_t ph = 0; int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const auto t = sc.template tile<BLOCK_N>(g, tile);
      if (t.skip) continue;
      ctx.batch = t.b;
      ctx.row0 = (long long)t.mt * G2_BLOCK_M + q * 32;
      ctx.n0 = t.nt * BLOCK_N;
      if constexpr (kPair) {
        const int buf = it & 1;
        ctx.x_own_bar = &xbar[buf * 4 + q];
        ctx.x_own_stat = smem_u32(xstat + (buf * 4 + q) * 64);
        ctx.x_peer_stat = mapa_u32(ctx.x_own_stat, rank ^ 1u);
        ctx.x_peer_bar = mapa_u32(smem_u32(ctx.x_own_bar), rank ^ 1u);
        ctx.x_parity = (uint32_t)(it >> 1) & 1;
      }
      ++it;
      if constexpr (Epi::kNeedsBias) epi.template prefetch<BLOCK_N>(ctx);  // LN + residual epilogues
      wg_mainloop<Cfg::STAGES, Cfg::STAGE_BYTES>(acc, smem, full, empty, s, ph, sc.num_kb, wg, lane);
      wg_epilogue<Cfg::STG_ROWS>(acc, smem, Cfg::STG_LD, wg, warp, lane, [&](AccSmem a) { epi.template run<BLOCK_N>(a, ctx); });
      __syncwarp();
      if (lane == 0) mbar_arrive(stg_free);
    }
  }
  if constexpr (kPair) {
    __syncthreads();
    cluster_sync_all();   // nobody leaves while the peer may still post into this CTA's slots
  }
  if constexpr (has_cta_stats<Epi>::value) {
    __syncthreads();
    cta_stats_flush(epi, sbias);
  }
}

template <class Sched, class Epi, int BLOCK_N>
__global__ void __launch_bounds__((G2_EPI_WARPS + 1) * 32, 1) k_gemm2(const Sched sc, const Epi epi, const G2Grid g) {
  gemm2_body<Sched, Epi, BLOCK_N, false>(sc, epi, g);
}
template <class Sched, class Epi, int BLOCK_N>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__((G2_EPI_WARPS + 1) * 32, 1)
k_gemm2_pair(const Sched sc, const Epi epi, const G2Grid g) {
  gemm2_body<Sched, Epi, BLOCK_N, true>(sc, epi, g);
}

// D[batches][M, N] through schedule sc.  kPair: N = 2 BLOCK_N on the column-split CTA pairs (W packed as two BLOCK_N-row
// halves: 256 for GraphCast's 512-wide latents, 192 for Pangu's C = 384 projection and fc2).
template <int BLOCK_N, bool kPair = false, class Sched, class Epi>
int launch_gemm2(const Sched& sc, const Epi& epi, long long M, int N, int batches, int num_sms, cudaStream_t st) {
  using Cfg = G2Cfg<BLOCK_N, G2_EPI_WARPS>;
  constexpr int SMEM = Cfg::SMEM_BYTES + (kPair ? G2_PAIR_SMEM : 0);
  static_assert(SMEM <= 232448, "smem budget");
  auto kern = [] {   // instantiates only the entry that is launched
    if constexpr (kPair) return k_gemm2_pair<Sched, Epi, BLOCK_N>;
    else return k_gemm2<Sched, Epi, BLOCK_N>;
  }();
  static std::atomic<uint64_t> configured{0};   // one bit per device: the attribute is per (function, device)
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(kern), SMEM)) return rc;
  const G2Grid g{M, (int)((M + G2_BLOCK_M - 1) / G2_BLOCK_M), N / BLOCK_N, batches};
  const long long tiles = g.num_tiles();
  if (N % BLOCK_N || (kPair && N != 2 * BLOCK_N) || tiles > INT_MAX) {
    set_error("internal: GEMM shape M=%lld N=%d BN=%d batches=%d%s", M, N, BLOCK_N, batches, kPair ? " (pair)" : "");
    return SKY_ERR_STATE;
  }
  int grid;
  if (kPair) {
    const int pairs = g.num_m_tiles < num_sms / 2 ? g.num_m_tiles : num_sms / 2;
    grid = 2 * pairs;
  } else {
    grid = (int)(tiles < num_sms ? tiles : num_sms);
  }
  kern<<<grid, Cfg::THREADS, SMEM, st>>>(sc, epi, g);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

// ======================================================================================
// v2 epilogues.  acc.load32(c, v): this lane's row (ctx.row0 + lane), columns [c, c+32).
// The 32x32 block is re-tiled through ctx.patch so global accesses run along rows.
// ======================================================================================
__device__ __forceinline__ void patch_put(float* patch, int lane, const float (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) patch[lane * G2_PATCH_LD + j] = v[j];
}
__device__ __forceinline__ void patch_put_s(uint32_t patch_s, int lane, const float (&v)[32]) {
  const uint32_t a = patch_s + lane * (G2_PATCH_LD * 4);
#pragma unroll
  for (int j = 0; j < 32; ++j) sts_f32(a + 4 * j, v[j]);
}
// 32x32 fp32 block in the swizzled vector layout (G2_PATCHV_BYTES): row r is 128 bytes, its 16-byte chunk k sits at
// position k ^ (r & 7).  Row-owner writes (lane = row, all chunks) and re-tiled reads (8 lanes = the 8 chunks of one
// row) are both conflict-free per quarter warp, with no padding: 16 patches fit in 64 KB.
__device__ __forceinline__ uint32_t patchv_addr(uint32_t patch_s, int r, int k) {
  return patch_s + (uint32_t)r * 128u + ((uint32_t)(k ^ (r & 7)) << 4);
}
__device__ __forceinline__ void patch_put_v(uint32_t patch_s, int lane, const float (&v)[32]) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(patchv_addr(patch_s, lane, k)), "f"(v[4 * k]), "f"(v[4 * k + 1]),
                 "f"(v[4 * k + 2]), "f"(v[4 * k + 3])
                 : "memory");
}
// 8 consecutive floats of patch row rr starting at column c8 -> 8 halves
__device__ __forceinline__ uint4 patch_get_h8(uint32_t patch_s, int rr, int c8) {
  const uint32_t a = patch_s + (rr * G2_PATCH_LD + c8) * 4;
  uint4 pk;
  pk.x = pack_half2(lds_f32(a), lds_f32(a + 4));
  pk.y = pack_half2(lds_f32(a + 8), lds_f32(a + 12));
  pk.z = pack_half2(lds_f32(a + 16), lds_f32(a + 20));
  pk.w = pack_half2(lds_f32(a + 24), lds_f32(a + 28));
  return pk;
}

// fp16 output, optional GELU: row-major [M, ldo] (kImage = false) or tile image with nkb
// k-blocks per row tile (kImage = true).  16-byte stores: lane -> (row = it*8 + lane/4,
// 8-column chunk = lane%4), so four lanes cover 64 contiguous bytes of one row.
template <bool kGelu, bool kImage>
struct Epi2F16 {
  static constexpr bool kNeedsBias = false;
  __half* out; int ldo; int nkb; const float* bias;
  const float* gamma = nullptr; const float* beta = nullptr;  // unused (uniform epilogue interface)
#ifdef SKY_EXPERIMENTS
  int exp = 0;  // timing experiments only (results invalid): 2 = no global stores
#else
  static constexpr int exp = 0;
#endif
  // head_major (row-major mode only): column block j of 32 goes to out[j][row][0..32), i.e. (part, head, token, 32) for
  // the QKV projection.  A warp store then covers 8 consecutive tokens x 64 B = 512 contiguous bytes instead of 8
  // half lines 2*ldo bytes apart, and the attention kernel reads 64-byte rows that are contiguous along longitude.
  int head_major = 0;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& x) const {
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    const uint32_t r0 = (uint32_t)(x.row0 & 127);
    for (int c = x.part * 32; c < BN; c += 32 * x.nparts) {
      // this lane's 8 output columns are the same for all its rows: their bias is loaded once, ahead of the accumulator read
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + x.n0 + c + ch * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + x.n0 + c + ch * 8 + 4));
      {
        float v[32];
        acc.load32(c, v);
        if (kGelu) {
          // activation in the row domain: 32 independent dependency chains per thread
          const float4* bp = reinterpret_cast<const float4*>(bias + x.n0 + c);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 b = __ldg(bp + j);
            gelu_erf_x2(v[4 * j], v[4 * j + 1], b.x, b.y);
            gelu_erf_x2(v[4 * j + 2], v[4 * j + 3], b.z, b.w);
          }
        }
        patch_put_v(x.patch_s, x.lane, v);
      }
      __syncwarp();
      const int col = x.n0 + c;  // first column of the chunk
      uint8_t* ibase = nullptr;
      if (kImage)
        ibase = reinterpret_cast<uint8_t*>(out) + ((size_t)(x.row0 >> 7) * nkb + (col >> 6)) * (size_t)G2_A_BYTES + r0 * 128;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + rsub;
        float4 t0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
        float4 t1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
        if (!kGelu) {
          t0.x += b0.x; t0.y += b0.y; t0.z += b0.z; t0.w += b0.w;
          t1.x += b1.x; t1.y += b1.y; t1.z += b1.z; t1.w += b1.w;
        }
        uint4 pk;
        pk.x = pack_half2(t0.x, t0.y); pk.y = pack_half2(t0.z, t0.w);
        pk.z = pack_half2(t1.x, t1.y); pk.w = pack_half2(t1.z, t1.w);
        if (x.row0 + rr < x.M && !(exp & 2)) {
          if (kImage)
            *reinterpret_cast<uint4*>(ibase + rr * 128 + (((((col & 63) >> 3) + ch) ^ (rr & 7)) << 4)) = pk;
          else if (head_major)
            *reinterpret_cast<uint4*>(out + ((size_t)((col + ch * 8) >> 5) * x.M + (x.row0 + rr)) * 32 + ((col + ch * 8) & 31)) = pk;
          else
            *reinterpret_cast<uint4*>(out + (x.row0 + rr) * ldo + col + ch * 8) = pk;
        } else if (exp & 2) {
          asm volatile("" ::"r"(pk.x), "r"(pk.y), "r"(pk.z), "r"(pk.w));   // keep the value alive
        }
      }
      __syncwarp();
    }
  }
};

// xf32[row, n0+col] (=|+=) f(acc)  and the fp16 tile image of the new rows.
//   kLn:       y = LayerNorm(acc + bias) * gamma + beta  (tile spans the feature width: n0 == 0)
//   kResidual: x += y, else x = y  (bias, if any, is applied when !kLn as well)
// Global traffic is 128-bit: lane -> (row = it*4 + lane/8, float4 column group = lane%8), i.e.
// eight lanes cover one 128-byte row segment.  bias / gamma / beta come from shared memory.
// kImgStream: the rows exist ONLY as their fp16 operand image — the residual is read from `img` (in place), the sum is formed in
// fp32 and rounded once back into `img`; nothing is read from or written to x.  Round 2 (late): on the oracle an fp16-only
// residual stream moves the Pangu step error from 5.3e-4 to 5.9e-4 (tests/test_oracle_cpu.py) and removes 8 of the 12 bytes
// per token and feature that the projection / MLP epilogues move through HBM.
template <bool kLn, bool kResidual, bool kImgStream = false>
struct Epi2F32Img {
  static constexpr bool kNeedsBias = kLn;
  float* x; int ldx;            // fp32 row-major (unused when kImgStream)
  uint8_t* img; int nkb;        // fp16 image of the same rows (may be null unless kImgStream)
  const float* bias; const float* gamma; const float* beta; float eps;  // bias may be null when !kLn
#ifdef SKY_EXPERIMENTS
  int exp = 0;  // timing experiments only (results invalid): 1 = no residual loads, 2 = no fp32 stores, 4 = no image stores
#else
  static constexpr int exp = 0;
#endif
  // Pull this warp's residual rows into L2 ahead of time, while the tile's main loop runs.
  // four residual values of row (row0 + rr) at tile column n0 + c + 4 * c4, read from the fp16 image
  __device__ __forceinline__ uint2 img_res_raw(const EpiCtx& e, int rr, int c, int c4) const {
    const int col = e.n0 + c + c4 * 4;
    return *reinterpret_cast<const uint2*>(img + ((size_t)(e.row0 >> 7) * nkb + (col >> 6)) * (size_t)G2_A_BYTES +
                                           ((uint32_t)(e.row0 & 127) + rr) * 128 + ((((uint32_t)(col & 63) >> 3) ^ (uint32_t)(rr & 7)) << 4) + (c4 & 1) * 8);
  }
  static __device__ __forceinline__ float4 h4_to_f4(const uint2& u) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  template <int BN>
  __device__ void prefetch(const EpiCtx& e) const {
    if (!kResidual) return;
    const long long row = e.row0 + e.lane;
    if (row >= e.M) return;
    if (kImgStream) {
      const char* p = reinterpret_cast<const char*>(img) + ((size_t)(e.row0 >> 7) * nkb + (e.n0 >> 6)) * (size_t)G2_A_BYTES +
                      ((uint32_t)(e.row0 & 127) + e.lane) * 128;
#pragma unroll
      for (int i = e.part; i < BN / 64; i += e.nparts) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (size_t)i * G2_A_BYTES));
      return;
    }
    const char* p = reinterpret_cast<const char*>(x + row * ldx + e.n0);
#pragma unroll
    for (int i = e.part; i < BN * 4 / 128; i += e.nparts) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + i * 128));
  }
  // Per 32x32 block: the row-owner lanes drop the raw accumulator into the warp's patch with 128-bit
  // stores, then every lane works on (row = it*4 + lane/8, 4 columns = lane%8) pieces: 8 lanes cover a
  // full 128-byte row segment of x, so residual loads and stores are coalesced 128-bit accesses.  The
  // LayerNorm statistics of the 8 rows a lane touches come from their owner lanes by shuffle; the
  // fp16 image chunks (8 columns = 16 bytes) are assembled from lane pairs by shuffle, not through
  // shared memory.  Every warp reduces the statistics of its own column groups only; the warps that
  // share a lane quarter exchange partial sums through their patches.
  // kPrefetch: load the residual of the next column group while this one is processed (32 more registers)
  template <int BN, bool kPrefetch = true, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    constexpr int NG = BN / 32;
    const int rsub4 = e.lane >> 3, c4 = e.lane & 7;
    const long long rows_left = e.M - e.row0;          // >= 32 for every tile but the last
    float* xp = x + e.row0 * ldx + e.n0 + c4 * 4;
    const bool ld_on = kResidual && !(exp & 1);
    float4 xin[8];
    if constexpr (kImgStream) {
      uint2 raw[8];
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        raw[it] = (kPrefetch && ld_on && rr < rows_left && e.part < NG) ? img_res_raw(e, rr, e.part * 32, c4) : make_uint2(0u, 0u);
      }
#pragma unroll
      for (int it = 0; it < 8; ++it) xin[it] = h4_to_f4(raw[it]);
    } else {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        xin[it] = (kPrefetch && ld_on && rr < rows_left && e.part < NG) ? *reinterpret_cast<const float4*>(xp + (size_t)rr * ldx + e.part * 32)
                                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    float rs[8], ns[8];   // rstd and -mean*rstd of row it*4 + rsub4
#pragma unroll
    for (int it = 0; it < 8; ++it) { rs[it] = 1.f; ns[it] = 0.f; }
    if (kLn) {
      float s = 0.f, ss = 0.f;
      for (int g = e.part; g < NG; g += e.nparts) {
        float v[32];
        acc.load32(g * 32, v);
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 b = lds_f32x4_ro(e.svec_s + (g * 32 + j) * 4);
          const float y0 = v[j] + b.x, y1 = v[j + 1] + b.y, y2 = v[j + 2] + b.z, y3 = v[j + 3] + b.w;
          s += (y0 + y1) + (y2 + y3);
          ss += (y0 * y0 + y1 * y1) + (y2 * y2 + y3 * y3);
        }
      }
      if (e.nparts > 1) {
        const uint32_t slot = e.patch_s + e.lane * 8;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(slot), "f"(s), "f"(ss) : "memory");
        const int q = (int)((e.row0 >> 5) & 3);
        asm volatile("bar.sync %0, %1;" ::"r"(8 + q), "r"(32 * e.nparts) : "memory");
        for (int p = 0; p < e.nparts; ++p) {
          if (p == e.part) continue;
          float ps, pss;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(ps), "=f"(pss) : "r"(slot + (p - e.part) * 4 * e.patch_stride));
          s += ps; ss += pss;
        }
        asm volatile("bar.sync %0, %1;" ::"r"(8 + q), "r"(32 * e.nparts) : "memory");   // the patches are reused below
      }
      float width = (float)BN;
      if (e.x_own_bar) {
        // column-split CTA pair (k_gemm2_pair): the other half of these rows is in the peer CTA — post this CTA's sums into
        // the peer's slot (st.async completes the peer's mbarrier transaction), wait for the peer's, add
        if (e.part == 0) {
          if (e.lane == 0) mbar_arrive_expect_tx(e.x_own_bar, 32 * 8);
          __syncwarp();
          asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];" ::"r"(e.x_peer_stat + e.lane * 8),
                       "f"(s), "f"(ss), "r"(e.x_peer_bar)
                       : "memory");
        }
        mbar_wait(e.x_own_bar, e.x_parity);   // CTA-scope acquire: the peer's sums arrive in THIS CTA's shared memory through st.async, whose completion the barrier phase carries (as for bulk copies); the cluster-scope wait added an L1 invalidate (CCTL.IVALL) per tile
        float ps, pss;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(ps), "=f"(pss) : "r"(e.x_own_stat + e.lane * 8));
        s += ps; ss += pss;
        width = (float)(2 * BN);
      }
      const float mean = s / width;
      const float rstd = rsqrtf(fmaxf(ss / width - mean * mean, 0.f) + eps);
      const float nmr = -mean * rstd;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        rs[it] = __shfl_sync(0xffffffffu, rstd, it * 4 + rsub4);
        ns[it] = __shfl_sync(0xffffffffu, nmr, it * 4 + rsub4);
      }
    }
    const uint32_t r0 = (uint32_t)(e.row0 & 127);
    const int odd = e.lane & 1;
    for (int g = e.part; g < NG; g += e.nparts) {
      const int c = g * 32;
      if (!kPrefetch && kResidual) {
        if constexpr (kImgStream) {
          uint2 raw[8];
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int rr = it * 4 + rsub4;
            raw[it] = (ld_on && rr < rows_left) ? img_res_raw(e, rr, c, c4) : make_uint2(0u, 0u);
          }
#pragma unroll
          for (int it = 0; it < 8; ++it) xin[it] = h4_to_f4(raw[it]);
        } else {
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int rr = it * 4 + rsub4;
            xin[it] = (ld_on && rr < rows_left) ? *reinterpret_cast<const float4*>(xp + (size_t)rr * ldx + c) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(e.patch_s, e.lane, v);
      }
      __syncwarp();
      float4 bs = make_float4(0.f, 0.f, 0.f, 0.f), ga = make_float4(1.f, 1.f, 1.f, 1.f), be = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kLn) {
        bs = lds_f32x4_ro(e.svec_s + (c + c4 * 4) * 4);
        ga = lds_f32x4_ro(e.svec_s + (e.vstride + c + c4 * 4) * 4);
        be = lds_f32x4_ro(e.svec_s + (2 * e.vstride + c + c4 * 4) * 4);
      } else if (bias) {
        bs = __ldg(reinterpret_cast<const float4*>(bias + e.n0 + c + c4 * 4));
      }
      const bool more = g + e.nparts < NG;
      float4 xnext[kPrefetch ? 8 : 1];
      if constexpr (kResidual && kPrefetch) {
        if constexpr (kImgStream) {
          uint2 raw[8];
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int rr = it * 4 + rsub4;
            raw[it] = (more && ld_on && rr < rows_left) ? img_res_raw(e, rr, c + 32 * e.nparts, c4) : make_uint2(0u, 0u);
          }
#pragma unroll
          for (int it = 0; it < 8; ++it) xnext[it] = h4_to_f4(raw[it]);
        } else {
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int rr = it * 4 + rsub4;
            xnext[it] = (more && ld_on && rr < rows_left) ? *reinterpret_cast<const float4*>(xp + (size_t)rr * ldx + c + 32 * e.nparts)
                                                          : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
      const int col = e.n0 + c;
      uint8_t* ibase = img ? img + ((size_t)(e.row0 >> 7) * nkb + (col >> 6)) * (size_t)G2_A_BYTES + r0 * 128 : nullptr;
      const uint32_t cb = (((uint32_t)col & 63u) >> 3) + (uint32_t)(c4 >> 1);   // 16-byte chunk of this lane pair inside the image row
#pragma unroll
      for (int it2 = 0; it2 < 8; it2 += 2) {
        uint2 h[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int it = it2 + u;
          const int rr = it * 4 + rsub4;
          const float4 t = lds_f32x4(patchv_addr(e.patch_s, rr, c4));
          float4 y;
          y.x = fmaf(fmaf(t.x + bs.x, rs[it], ns[it]), ga.x, be.x); y.y = fmaf(fmaf(t.y + bs.y, rs[it], ns[it]), ga.y, be.y);
          y.z = fmaf(fmaf(t.z + bs.z, rs[it], ns[it]), ga.z, be.z); y.w = fmaf(fmaf(t.w + bs.w, rs[it], ns[it]), ga.w, be.w);
          if (kResidual) { y.x += xin[it].x; y.y += xin[it].y; y.z += xin[it].z; y.w += xin[it].w; }
          if (!kImgStream && rr < rows_left && !(exp & 2)) *reinterpret_cast<float4*>(xp + (size_t)rr * ldx + c) = y;
          h[u].x = pack_half2(y.x, y.y); h[u].y = pack_half2(y.z, y.w);
        }
        if (ibase && !(exp & 4)) {
          // even lane assembles the chunk of row it2, odd lane the chunk of row it2+1: swap the other halves
          const uint2 send = odd ? h[0] : h[1];
          uint2 recv;
          recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
          recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
          const int rr = (it2 + odd) * 4 + rsub4;
          const uint4 pk = odd ? make_uint4(recv.x, recv.y, h[1].x, h[1].y) : make_uint4(h[0].x, h[0].y, recv.x, recv.y);
          if (rr < rows_left) *reinterpret_cast<uint4*>(ibase + rr * 128 + ((cb ^ (uint32_t)(rr & 7)) << 4)) = pk;
        }
      }
      __syncwarp();
      if constexpr (kResidual && kPrefetch) {
#pragma unroll
        for (int it = 0; it < 8; ++it) xin[it] = xnext[it];
      }
    }
  }
};

// post-norm residual of the attention projection and of the MLP: fp32 row-major token stream (EpiLnRes) or the stream kept
// only as its fp16 operand image (EpiLnResImg); the engine picks one per handle (pangu_engine.cu, "fp32_stream")
using EpiLnRes = Epi2F32Img<true, true, false>;
using EpiLnResImg = Epi2F32Img<true, true, true>;

// up-sample linear1 (N = 4C as (hs, ws, C); one n-tile = one sub-position): LayerNorm over
// the C features of the tile, written as fp16 image rows of the FINE token
// (z, 2*h2+hs, 2*w2+ws) when it survives the crop.
struct Epi2UpShuffle {
  static constexpr bool kNeedsBias = false;
  uint8_t* img; int nkb; int C; const float* gamma; const float* beta; float eps; const float* bias;  // bias unused
  int H, W, H2, W2;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    float s = 0.f, ss = 0.f;
    for (int c = 0; c < BN; c += 32) {
      float v[32];
      acc.load32(c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) { s += v[j]; ss += v[j] * v[j]; }
    }
    const float mean = s / BN, rstd = rsqrtf(fmaxf(ss / BN - mean * mean, 0.f) + eps);
    const int sub = e.n0 / C, hs = sub >> 1, ws = sub & 1;
    long long dst = -1;
    {
      const long long row = e.row0 + e.lane;
      if (row < e.M) {
        int w2 = (int)(row % W2); long long qq = row / W2;
        int h2 = (int)(qq % H2); qq /= H2;  // member*Z + z
        int h = 2 * h2 + hs, w = 2 * w2 + ws;
        if (h < H) dst = (qq * H + h) * W + w;
      }
    }
    const int cp = 2 * (e.lane & 15), hr = e.lane >> 4;
    for (int c = e.part * 32; c < BN; c += 32 * e.nparts) {
      float v[32];
      acc.load32(c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = (v[j] - mean) * rstd;
      patch_put(e.patch, e.lane, v);
      __syncwarp();
      const float g0 = __ldg(gamma + c + cp), g1 = __ldg(gamma + c + cp + 1);
      const float b0 = __ldg(beta + c + cp), b1 = __ldg(beta + c + cp + 1);
#pragma unroll 8
      for (int it = 0; it < 16; ++it) {
        const int rr = 2 * it + hr;
        const long long d = __shfl_sync(0xffffffffu, dst, rr);
        if (d >= 0)
          *reinterpret_cast<uint32_t*>(img + img_offset(d, c + cp, nkb)) =
              pack_half2(e.patch[rr * G2_PATCH_LD + cp] * g0 + b0, e.patch[rr * G2_PATCH_LD + cp + 1] * g1 + b1);
      }
      __syncwarp();
    }
  }
};

// patch recovery over ALL tokens with N = 160 (upper, cols ((v*2+dz)*4+dh)*4+dw) + 64
// (surface, cols 160 + (v*4+dh)*4+dw): a token of slab z == 0 takes the surface columns, the
// others the upper-air ones.  Consecutive lanes are consecutive longitudes, so the float4
// stores of a warp already form contiguous 512-byte runs: no re-tiling needed.
struct Epi2Recover {
  static constexpr bool kNeedsBias = false;
  float* out; const float* bias /*[5+4]*/; const float* mean; const float* stdv;
  int nlat, nlon, nch, nup, nlev, H, W, T;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    const long long row = e.row0 + e.lane;
    const bool ok = row < e.M;
    long long b = 0; int z = 0, h = 0, w = 0;
    if (ok) {
      int t = (int)(row % T); b = row / T;
      w = t % W; int q2 = t / W; h = q2 % H; z = q2 / H;
    }
    for (int c = e.part * 32; c < BN; c += 32 * e.nparts) {
      float v[32];
      acc.load32(c, v);
      if (!ok) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = c + 4 * j;
        int ch, lat, vv;
        if (col < 160) {
          if (z == 0) continue;
          int dh = (col >> 2) & 3, dz = (col >> 4) & 1;
          vv = col >> 5;
          int lev = 2 * (z - 1) + dz;
          lat = 4 * h + dh;
          if (lev >= nlev) continue;
          ch = vv * nlev + lev;
        } else {
          if (z != 0) continue;
          int cs = col - 160;
          int dh = (cs >> 2) & 3;
          vv = 5 + (cs >> 4);
          lat = 4 * h + dh;
          ch = nup + (cs >> 4);
        }
        if (lat >= nlat) continue;
        const float bsv = __ldg(bias + vv), mu = __ldg(mean + ch), sd = __ldg(stdv + ch);
        float4 t4;
        t4.x = (v[4 * j + 0] + bsv) * sd + mu; t4.y = (v[4 * j + 1] + bsv) * sd + mu;
        t4.z = (v[4 * j + 2] + bsv) * sd + mu; t4.w = (v[4 * j + 3] + bsv) * sd + mu;
        *reinterpret_cast<float4*>(out + ((b * nch + ch) * (long long)nlat + lat) * nlon + 4 * w) = t4;
      }
    }
  }
};

}  // namespace sky
