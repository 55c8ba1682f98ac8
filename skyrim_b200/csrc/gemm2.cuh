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
// 8 = loader.  One schedule has no A image: under SchedProd four more warps (9..12) gather and convert A straight into
// the ring (Pangu's patch embedding) and the loader fetches only W.  Warpgroup g issues the wgmma products of rows
// 64g .. 64g+63 of the 128-row tile over all BLOCK_N columns (fp32 accumulators in registers, BLOCK_N / 2 per thread).
// At the end of a tile both warpgroups stage their accumulators in shared memory — over the operand ring, which
// is drained by then — and the same eight warps run the row-owner epilogue on the staged tile
// (warp%4 selects the 32-row quarter, warp/4 the column partition).  Epilogues re-tile their 32x32
// accumulator blocks through a padded smem patch so that every global access is a full
// 64/128-byte row segment.  Epilogues wrapped in FragEpi run on the accumulator registers instead and leave through a
// dedicated output tile that the loader bulk-stores, so the ring keeps streaming under them (Pangu's QKV projection, fc1,
// projection, fc2).
#pragma once
#include <climits>
#include <type_traits>

#include "../../include/skyrim_b200.h"
#include "sky_common.cuh"
#include "wgmma_ops.cuh"

namespace sky {

constexpr int G2_BLOCK_M = 128;
constexpr int G2_A_BYTES = G2_BLOCK_M * 128;
constexpr int G2_PATCH_LD = 33;    // scalar accessors (odd stride: conflict-free column reads)
constexpr int G2_PATCH_FLOATS = 32 * G2_PATCH_LD;
constexpr int G2_PATCHV_BYTES = 4096;   // 128-bit accessors: 32 rows x 128 B, 16-byte chunk index XOR (row & 7)
constexpr int G2_VEC_FLOATS = 512;      // shared-memory copies of bias | gamma | beta (LN epilogues), this many floats apart

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
  // appends a segment of k k-blocks per row tile; a seventh segment is not stored and marks the operand invalid
  // (launch_gemm2 refuses it)
  AOperand& add(const uint8_t* img, int k, long long bstride = 0) {
    if (nseg >= 6) { nseg = 7; return *this; }
    seg[nseg] = img; nkb[nseg] = k; batch_stride[nseg] = bstride; ++nseg;
    return *this;
  }
  bool valid() const { return nseg >= 1 && nseg <= 6; }
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

// kFrag: the epilogue runs on the accumulator fragments (FragEpi below); the patches give way to the output tile,
// BLOCK_N / 64 blocks of 128 rows x 128 B laid out as the destination image's blocks.  PROD_WARPS: the A producer warps
// of the schedule (SchedProd), 0 for image-fed A.
template <int BLOCK_N, int EPI_WARPS, bool kFrag = false, int PROD_WARPS = 0>
struct G2Cfg {
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = G2_A_BYTES + B_BYTES;
  static constexpr int OUT_BYTES = BLOCK_N / 64 * G2_A_BYTES;
  static constexpr int PATCH_BYTES = kFrag ? OUT_BYTES : EPI_WARPS * G2_PATCH_FLOATS * 4;
  static constexpr int VEC_BYTES = 3 * G2_VEC_FLOATS * 4;
  static constexpr int FIXED = 1024 /*align*/ + 256 /*barriers*/ + PATCH_BYTES + VEC_BYTES;
  static constexpr int MAXS = (232448 - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = MAXS > 6 ? 6 : MAXS;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  // accumulator staging over the drained ring: all 128 rows at once
  static constexpr int STG_LD = (BLOCK_N + 31) / 32 * 32 + 4;
  static constexpr int SMEM_BYTES = RING_BYTES + FIXED;
  static constexpr int THREADS = (EPI_WARPS + 1 + PROD_WARPS) * 32;   // consumers, loader, A producers
  static_assert(BLOCK_N % 8 == 0 && BLOCK_N <= 256, "wgmma N, accumulator registers");
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static_assert(STAGES >= 2, "pipeline depth");
  static_assert(kFrag || 128 * STG_LD * 4 <= RING_BYTES, "accumulator staging");
  static_assert(!kFrag || BLOCK_N % 64 == 0, "output tile of whole 64-column blocks");
  static_assert(EPI_WARPS == 8, "two consumer warpgroups");
};

// Epilogue on the accumulator fragments: FragEpi<E> runs E::frag instead of E::run.  Each consumer thread applies the
// epilogue to its own wgmma fragment (rows 64 wg + 16 w + l/4 and + 8, columns 8 i + 2 (l & 3) + {0, 1}) and writes the
// fp16 results into the output tile, which the loader warp bulk-stores to E::tile_image.  Nothing is staged over the
// ring, so the loader streams the next tile's k-blocks in under the epilogue.  E::kLoadsTile: the loader first fills the
// output tile with the destination's current bytes (the residual of an in-place update).
template <class E>
struct FragEpi : E {
  static constexpr bool kFragment = true;
};
template <class E, class = void> struct is_fragment_epi : std::false_type {};
template <class E> struct is_fragment_epi<E, std::void_t<decltype(E::kFragment)>> : std::true_type {};
// E::kScatter: the tile's rows do not land as three contiguous blocks at E::tile_image.  The loader looks up the destination
// row of each tile row with E::dest_row (while it waits for the ring, ahead of the tile's epilogue), publishes the 128 rows
// as a 512-byte map over the bias region (E::kNeedsBias is false), opens the output tile, and stores it later with
// E::frag_store, which reads the same map.  The map is overwritten only after the previous tile's epilogue has finished
// (stg_free) and that tile has been stored.
template <class E, class = void> struct is_scatter_epi : std::false_type {};
template <class E> struct is_scatter_epi<E, std::void_t<decltype(E::kScatter)>> : std::true_type {};

// LayerNorm statistics of a row, or of a part of its columns: the mean and m2, the sum of squared deviations from that
// mean.  Every LayerNorm epilogue takes the statistics of the values a thread holds about their mean (two passes, or the
// staged path's one pass about a nearby shift) and merges the partials of disjoint column sets with Chan's formula; one
// pass over (sum, sum of squares) loses the variance to cancellation once |mean| / std reaches ~100 (ss / n - mean^2 in
// fp32 keeps 2^-24 mean^2 / var of it).
struct LnStat {
  float mean, m2;
};
// merge of the partials a (na columns) and b (nb columns): bit for bit symmetric in (a, na) and (b, nb), so the lanes of a
// quad, the warps of a lane quarter and the two CTAs of a pair that merge the same partials agree exactly
__device__ __forceinline__ LnStat ln_merge(LnStat a, float na, LnStat b, float nb) {
  const float n = na + nb, d = b.mean - a.mean;
  return {(na / n) * a.mean + (nb / n) * b.mean, (a.m2 + b.m2) + d * d * (na * nb / n)};
}

// LayerNorm row statistics of a column-split CTA pair (k_gemm2_pair): the two CTAs hold the two column halves of the same
// 128 rows.  For each tile and 32-row group, a CTA posts its rows' LnStat (mean, m2 of its half) into the peer's slot and
// reads the peer's from its own.  Slots [tile parity][32-row group][row % 32][mean, m2] and one barrier per (tile parity,
// group) follow the barrier block (gemm2_body).  own_bar == nullptr outside a pair.
struct PairStats {
  uint64_t* own_bar = nullptr;            // completes when the peer's 32 rows of this group have landed
  uint32_t own_stat = 0;                  // shared-space address of this CTA's slot
  uint32_t peer_stat = 0, peer_bar = 0;   // shared::cluster addresses of the same slot / barrier in the peer CTA
  uint32_t parity = 0;
  // 32-row group q of the CTA's it-th tile
  __device__ __forceinline__ static PairStats at(uint64_t* xbar, float* xstat, int it, int q, uint32_t rank) {
    PairStats p;
    const int buf = it & 1;
    p.own_bar = &xbar[buf * 4 + q];
    p.own_stat = smem_u32(xstat + (buf * 4 + q) * 64);
    p.peer_stat = mapa_u32(p.own_stat, rank ^ 1u);
    p.peer_bar = mapa_u32(smem_u32(p.own_bar), rank ^ 1u);
    p.parity = (uint32_t)(it >> 1) & 1;
    return p;
  }
  // one lane per group and tile: announces the bytes of the peer's 32 posts
  __device__ __forceinline__ void expect() const { mbar_arrive_expect_tx(own_bar, 32 * 8); }
  // tile row r's statistics into the peer's slot.  st.async itself completes the peer's barrier transaction: no fence, no
  // release arrive.
  __device__ __forceinline__ void post(int r, LnStat v) const {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];" ::"r"(
                     peer_stat + (uint32_t)(r & 31) * 8u),
                 "f"(v.mean), "f"(v.m2), "r"(peer_bar)
                 : "memory");
  }
  // CTA-scope acquire: the peer's statistics arrive in THIS CTA's shared memory through st.async, whose completion the
  // barrier phase carries (as for bulk copies); a cluster-scope wait added an L1 invalidate (CCTL.IVALL) per tile
  __device__ __forceinline__ void wait() const { mbar_wait(own_bar, parity); }
  // after wait(): merges the peer's statistics of tile row r (its half: n columns, as many as this CTA's) into v.  Both
  // CTAs of the pair end with the same statistics (ln_merge is symmetric).
  __device__ __forceinline__ void merge_peer(int r, LnStat& v, float n) const {
    LnStat p;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(p.mean), "=f"(p.m2) : "r"(own_stat + (uint32_t)(r & 31) * 8u));
    v = ln_merge(v, n, p, n);
  }
};

// What a fragment epilogue sees of its tile
struct FragCtx {
  int row;              // the thread's first fragment row in the tile (64 wg + 16 w + l/4); the second is row + 8
  int c2;               // 2 (l & 3): the thread's first column inside each 8-column group
  int n0;               // first column of the tile in the full N
  uint32_t out_s;       // shared-space address of the output tile
  uint32_t svec_s;      // bias | gamma | beta of this CTA's columns, G2_VEC_FLOATS apart (LN epilogues)
  uint64_t* out_ready;  // completes when the output tile may be written (and, kLoadsTile, holds the destination's bytes)
  uint32_t ready_parity;
  PairStats pair;       // the thread's 32-row group (k_gemm2_pair)
  bool post_bar = false;   // this warp announces the pair's transaction bytes (one of the group's two warps)
  // byte offset inside the output tile of fragment row `row` (+ 8 with hi), 8-column group i
  __device__ __forceinline__ uint32_t offset(int i, bool hi) const {
    const uint32_t r = (uint32_t)(row + (hi ? 8 : 0));
    return (uint32_t)(i >> 3) * G2_A_BYTES + r * 128u + ((((uint32_t)i & 7u) ^ (r & 7u)) << 4) + (uint32_t)c2 * 2u;
  }
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
  uint32_t svec_s;     // shared-space address of bias | gamma | beta, G2_VEC_FLOATS apart (LN epilogues)
  PairStats pair;      // the warp's 32-row group (k_gemm2_pair)
};

// ---------------------------------------------------------------------------------------------------------------
// consumer side shared by the wgmma GEMM kernels
// ---------------------------------------------------------------------------------------------------------------
// Accumulators of warpgroup wg: rows 64 wg .. 64 wg + 63 of the 128-row tile, all BN columns.
template <int BN, bool kBMN = false>
struct WgAcc {
  float d[BN / 2];
  // zeroed at the start of every tile (rather than a scale-d = 0 first product): the registers are then dead between the
  // staging of one tile and the main loop of the next, i.e. free for the epilogue
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  }
  // one k-block: A = 128 rows x 64 halves at a_addr; B = BN rows x 64 halves, K-major, at b_addr, or (kBMN) 64 k-rows x BN
  // columns in 64-column atoms 8 KB apart
  __device__ __forceinline__ void kblock(uint32_t a_addr, uint32_t b_addr, int wg) {
    wgmma_fence();
    const uint64_t da = make_desc_sw128(a_addr + (uint32_t)wg * 8192u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t db = kBMN ? make_desc_sw128_mn(b_addr, 8192) + (uint64_t)(k * (2048 >> 4))
                               : make_desc_sw128(b_addr) + (uint64_t)(2 * k);
      Wgmma<BN, kBMN>::mma(d, da + 2 * k, db);
    }
    wgmma_commit();
  }
  __device__ __forceinline__ void settle() {
    wgmma_wait<0>();
    wgmma_fence_operands(d);
  }
  // fragment -> staging (row-major, ld floats per row, 128 rows); this warpgroup's rows start at 64 wg
  __device__ __forceinline__ void dump(uint32_t stg_s, int ld, int wg) const {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    const uint32_t r = (uint32_t)(64 * wg + 16 * w + (l >> 2));
    const uint32_t a0 = stg_s + (r * (uint32_t)ld + 2u * (uint32_t)(l & 3)) * 4u, a8 = a0 + 8u * (uint32_t)ld * 4u;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const uint32_t o = (uint32_t)(8 * i) * 4u;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0 + o), "f"(d[4 * i]), "f"(d[4 * i + 1]) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a8 + o), "f"(d[4 * i + 2]), "f"(d[4 * i + 3]) : "memory");
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

// Stage all 128 rows of accumulators at the base of the (drained) ring and run fn(AccSmem) in every consumer warp on its
// 32-row quarter (warp % 4).  The caller signals the loader afterwards (the ring is free again).
template <class Acc, class Fn>
__device__ __forceinline__ void wg_epilogue(const Acc& acc, uint8_t* smem, int ld, int wg, int warp, int lane, Fn&& fn) {
  const uint32_t stg = smem_u32(smem);
  named_bar_sync(1, 256);   // both warpgroups' products have completed: no wgmma still reads the ring the staging overwrites
  acc.dump(stg, ld, wg);
  named_bar_sync(1, 256);
  fn(AccSmem{stg + (uint32_t)(((warp & 3) * 32 + lane) * ld) * 4u});
  named_bar_sync(1, 256);
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
  bool valid() const { return A.valid(); }
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

// Producer-fed A: the A tile of every k-block is written into the ring by kProdWarps producer warps, one tile row per
// thread, through prod.prep(row) (once per tile) and prod.load8(info, k) (the 8 halves at columns k .. k + 7, zeros past
// M and past the valid K).  Only W, packed as for SchedW, is bulk-copied.  Staged epilogues only.
template <class Prod>
struct SchedProd {
  static constexpr bool kBMN = false;
  static constexpr int kProdWarps = 4;
  Prod prod;
  const uint8_t* W;
  int num_kb;
  bool valid() const { return true; }
  template <int BN>
  __device__ G2Tile tile(const G2Grid& g, int i) const { return G2Tile::at(g, i); }
  template <int BN>
  __device__ __forceinline__ void issue(uint8_t* dst, uint64_t* full, const G2Tile& t, int kb, int lane) const {
    constexpr int B_BYTES = BN * 128;
    if (lane == 0) {
      mbar_arrive_expect_tx(full, B_BYTES);
      bulk_g2s(dst + G2_A_BYTES, W + ((size_t)t.nt * num_kb + kb) * B_BYTES, B_BYTES, full);
    }
  }
};
// producer warps of a schedule: S::kProdWarps, none for the image-fed schedules
template <class S, class = void> struct sched_prod_warps : std::integral_constant<int, 0> {};
template <class S> struct sched_prod_warps<S, std::void_t<decltype(S::kProdWarps)>> : std::integral_constant<int, S::kProdWarps> {};

// ---------------------------------------------------------------------------------------------------------------
// The TMA-fed persistent GEMM.  One loader warp fills the stage ring (stage = A tile | B tile) through the schedule; two
// consumer warpgroups run the main loop and the epilogue of each tile.  The loader starts the next tile's copies once the
// previous tile's epilogue has left the ring (stg_free); a tile the schedule skips counts for no role.  Under a producer
// schedule the producer warps fill the A half of each stage on the same protocol, and full[s] also counts their arrivals.
// kPair (k_gemm2_pair): the two CTAs of a cluster take the same m-tile and n-tiles 0 / 1 (N = 2 BLOCK_N; the persistent
// walk over 2 n-tiles with an even grid gives CTA rank r exactly the tiles (mt, r)), and exchange LayerNorm row statistics
// through distributed shared memory (PairStats).  A 128 x 512 fp32 accumulator is the whole register file of an SM;
// this way the epilogue still sees whole rows.  Exchange slots and barriers are double buffered by tile parity; a CTA
// runs at most one tile ahead of its peer, because its next statistics wait needs the peer's sums of that tile.
// ---------------------------------------------------------------------------------------------------------------
constexpr int G2_EPI_WARPS = 8;
constexpr int G2_PAIR_SMEM = 2048;   // the pair's exchange slots, behind the barrier block
template <class Sched, class Epi, int BLOCK_N>
using G2CfgOf = G2Cfg<BLOCK_N, G2_EPI_WARPS, is_fragment_epi<Epi>::value, sched_prod_warps<Sched>::value>;

// Fragment epilogues (FragEpi): the loader warp stores the output tile of tile `t` (a finished tile) to the destination
// image.  The three 16 KB blocks of a tile are contiguous there (n0 is a multiple of BLOCK_N); a partial last m-tile is
// stored row by row, so that rows >= M are never written.  Every lane waits until its copies have read the tile.  (Scatter
// epilogues, E::kScatter, store the tile with E::frag_store instead.)
template <class Cfg, class Epi, class Tile>
__device__ __forceinline__ void frag_store(const Epi& epi, const Tile& t, uint32_t out_s, long long M, int bn, int lane) {
  uint8_t* dst = epi.tile_image(t.mt, t.nt * bn);
  const long long rows = M - (long long)t.mt * G2_BLOCK_M;
  if (rows >= G2_BLOCK_M) {
    if (lane == 0) bulk_s2g(dst, out_s, Cfg::OUT_BYTES);
  } else {
    for (int r = lane; r < rows; r += 32)
      for (int j = 0; j < Cfg::OUT_BYTES / G2_A_BYTES; ++j)
        bulk_s2g(dst + j * G2_A_BYTES + r * 128, out_s + (uint32_t)(j * G2_A_BYTES + r * 128), 128);
  }
  bulk_commit();
  bulk_wait_read<0>();
}

template <class Sched, class Epi, int BLOCK_N, bool kPair>
__device__ __forceinline__ void gemm2_body(const Sched& sc, const Epi& epi, const G2Grid& g) {
  constexpr int EPI_WARPS = G2_EPI_WARPS;
  constexpr bool kFrag = is_fragment_epi<Epi>::value;
  constexpr bool kScatter = is_scatter_epi<Epi>::value;
  if constexpr (kScatter) static_assert(kFrag && !Epi::kNeedsBias && !Epi::kLoadsTile, "scatter: fragment path, map over the bias region");
  constexpr int PROD_WARPS = sched_prod_warps<Sched>::value;
  static_assert(PROD_WARPS == 0 || (!kFrag && !kPair && PROD_WARPS * 32 == G2_BLOCK_M),
                "producer schedules: staged epilogue, one CTA, one tile row per producer thread");
  using Cfg = G2CfgOf<Sched, Epi, BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* patches = reinterpret_cast<float*>(smem + Cfg::RING_BYTES);
  float* sbias = reinterpret_cast<float*>(smem + Cfg::RING_BYTES + Cfg::PATCH_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + 3 * G2_VEC_FLOATS);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* stg_free = bars + 2 * Cfg::STAGES;   // consumers -> loader: the tile's epilogue has left the ring
  uint64_t* xbar = bars + 2 * Cfg::STAGES + 1;                                          // pair: [2 tile parities][4 lane quarters]
  float* xstat = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);     // pair: [2][4][32 lanes][2]
  static_assert(!kPair || (2 * Cfg::STAGES + 1 + 8) * 8 <= 256, "barrier block");
  // fragment path: stg_free becomes out_full (consumers -> loader: the output tile is written), and out_ready (loader ->
  // consumers: the output tile may be written) follows the pair's barriers
  uint64_t* out_ready = bars + 2 * Cfg::STAGES + 9;
  static_assert(!kFrag || (2 * Cfg::STAGES + 10) * 8 <= 256, "barrier block");

  // warp index through a shuffle: provably warp-uniform, so the role branches are uniform control flow
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;
  const uint32_t rank = kPair ? cluster_ctarank() : 0u;
  const int num_tiles = (int)g.num_tiles();   // < 2^31 (launch_gemm2)
  constexpr int LOADER = EPI_WARPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1 + PROD_WARPS * 32); mbar_init(&empty[s], EPI_WARPS); }
    mbar_init(stg_free, EPI_WARPS);
    if (kPair) for (int i = 0; i < 8; ++i) mbar_init(&xbar[i], 1);
    if constexpr (kFrag) mbar_init(out_ready, 1);
    mbar_fence_init();
  }
  if constexpr (Epi::kNeedsBias) if (threadIdx.x < EPI_WARPS * 32)
    for (int i = threadIdx.x; i < BLOCK_N; i += EPI_WARPS * 32) {
      const uint32_t c = rank * BLOCK_N + i;   // this CTA's columns
      sbias[i] = epi.bias[c]; sbias[G2_VEC_FLOATS + i] = epi.gamma[c]; sbias[2 * G2_VEC_FLOATS + i] = epi.beta[c];
    }
  if constexpr (has_cta_stats<Epi>::value)
    for (int i = threadIdx.x; i < 3 * G2_VEC_FLOATS; i += blockDim.x) sbias[i] = 0.f;
  __syncthreads();
  if (kPair) cluster_sync_all();   // the peer's exchange barriers exist before anything is posted to them

  const uint32_t out_s = smem_u32(patches);   // fragment path: the output tile
  if constexpr (kFrag) {
    int it = 0;
    if (warp == LOADER) {
      // The first min(num_kb, STAGES) k-blocks of a tile only wait for ring slots that the previous tile's main loop
      // releases.  After them the loader hands the output tile over: it stores the previous tile's once that epilogue is
      // done (stg_free), then opens it for this tile (out_ready), after loading the destination's bytes if the epilogue
      // reads them.  The rest of the tile's k-blocks follow.
      const int head = sc.num_kb < Cfg::STAGES ? sc.num_kb : Cfg::STAGES;
      int s = 0; uint32_t ph = 0;
      decltype(sc.template tile<BLOCK_N>(g, 0)) prev{};
      const uint32_t map_s = smem_u32(sbias);   // kScatter: destination row of tile row r at map_s + 4 r
      int dst_row[4];                           // kScatter: of tile rows lane + 32 k
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const auto t = sc.template tile<BLOCK_N>(g, tile);
        if (t.skip) continue;
        // the destination's bytes of this tile are pulled into L2 a main loop ahead of their load into the output tile
        if constexpr (Epi::kLoadsTile) if (lane == 0) bulk_prefetch_l2(epi.tile_image(t.mt, t.nt * BLOCK_N), Cfg::OUT_BYTES);
        if constexpr (kScatter)
#pragma unroll
          for (int k = 0; k < 4; ++k) dst_row[k] = epi.dest_row((long long)t.mt * G2_BLOCK_M + lane + 32 * k, g.M);
        for (int kb = 0; kb < sc.num_kb; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          sc.template issue<BLOCK_N>(smem + s * Cfg::STAGE_BYTES, &full[s], t, kb, lane);
          __syncwarp();
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
          if (kb + 1 != head) continue;
          if (it > 0) {
            mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
            if constexpr (kScatter) epi.frag_store(prev.nt * BLOCK_N, out_s, map_s, lane);
            else frag_store<Cfg>(epi, prev, out_s, g.M, BLOCK_N, lane);
          }
          if constexpr (kScatter)
#pragma unroll
            for (int k = 0; k < 4; ++k)
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(map_s + (uint32_t)(lane + 32 * k) * 4u), "r"(dst_row[k]) : "memory");
          __syncwarp();
          if (lane == 0) {
            if constexpr (Epi::kLoadsTile) {
              mbar_arrive_expect_tx(out_ready, Cfg::OUT_BYTES);
              bulk_g2s(patches, epi.tile_image(t.mt, t.nt * BLOCK_N), Cfg::OUT_BYTES, out_ready);
            } else {
              mbar_arrive(out_ready);
            }
          }
        }
        prev = t;
        ++it;
      }
      if (it > 0) {
        mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
        if constexpr (kScatter) epi.frag_store(prev.nt * BLOCK_N, out_s, map_s, lane);
        else frag_store<Cfg>(epi, prev, out_s, g.M, BLOCK_N, lane);
        bulk_wait<0>();
      }
    } else {
      const int wg = warp >> 2, w = warp & 3;
      FragCtx x;
      x.row = 64 * wg + 16 * w + (lane >> 2);
      x.c2 = 2 * (lane & 3);
      x.out_s = out_s;
      x.svec_s = smem_u32(sbias);
      x.out_ready = out_ready;
      x.post_bar = (w & 1) == 0;
      WgAcc<BLOCK_N, Sched::kBMN> acc;
      int s = 0; uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const auto t = sc.template tile<BLOCK_N>(g, tile);
        if (t.skip) continue;
        x.n0 = t.nt * BLOCK_N;
        x.ready_parity = (uint32_t)it & 1;
        if constexpr (kPair) x.pair = PairStats::at(xbar, xstat, it, x.row >> 5, rank);
        ++it;
        wg_mainloop<Cfg::STAGES, Cfg::STAGE_BYTES>(acc, smem, full, empty, s, ph, sc.num_kb, wg, lane);
        epi.template frag<BLOCK_N>(acc, x);
        fence_proxy_async_smem();   // the tile's generic writes are ordered before the loader's bulk store
        __syncwarp();
        if (lane == 0) mbar_arrive(stg_free);
      }
    }
  } else if (warp == LOADER) {
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
  } else if (PROD_WARPS > 0 && warp > LOADER) {
    // ---------------- A producers (SchedProd) ----------------
    // thread = tile row, the 8 chunks of a k-block in sequence: for one chunk the 32 lanes of a warp are 32 consecutive
    // rows (for the patch embedding 32 consecutive tokens, i.e. one contiguous 512-byte run of the source field per load
    // instruction), and the 16-byte shared-memory stores of a quarter warp fall into 8 different swizzled chunk slots
    if constexpr (PROD_WARPS > 0) {
      const int row = threadIdx.x - (LOADER + 1) * 32;
      int s = 0; uint32_t ph = 0; int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const auto t = sc.template tile<BLOCK_N>(g, tile);
        if (t.skip) continue;
        const auto ri = sc.prod.prep((long long)t.mt * G2_BLOCK_M + row);
        if (it > 0) mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
        ++it;
        for (int kb = 0; kb < sc.num_kb; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* a_s = smem + s * Cfg::STAGE_BYTES;
          uint4 v[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = sc.prod.load8(ri, kb * 64 + i * 8);
#pragma unroll
          for (int i = 0; i < 8; ++i) *reinterpret_cast<uint4*>(a_s + sw128_offset(row, i)) = v[i];
          fence_proxy_async_smem();
          mbar_arrive(&full[s]);
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
        }
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
      if constexpr (kPair) ctx.pair = PairStats::at(xbar, xstat, it, q, rank);
      ++it;
      if constexpr (Epi::kNeedsBias) epi.template prefetch<BLOCK_N>(ctx);  // LN + residual epilogues
      wg_mainloop<Cfg::STAGES, Cfg::STAGE_BYTES>(acc, smem, full, empty, s, ph, sc.num_kb, wg, lane);
      wg_epilogue(acc, smem, Cfg::STG_LD, wg, warp, lane, [&](AccSmem a) { epi.template run<BLOCK_N>(a, ctx); });
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
__global__ void __launch_bounds__(G2CfgOf<Sched, Epi, BLOCK_N>::THREADS, 1) k_gemm2(const Sched sc, const Epi epi, const G2Grid g) {
  gemm2_body<Sched, Epi, BLOCK_N, false>(sc, epi, g);
}
template <class Sched, class Epi, int BLOCK_N>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(G2CfgOf<Sched, Epi, BLOCK_N>::THREADS, 1)
k_gemm2_pair(const Sched sc, const Epi epi, const G2Grid g) {
  gemm2_body<Sched, Epi, BLOCK_N, true>(sc, epi, g);
}

// D[batches][M, N] through schedule sc.  kPair: N = 2 BLOCK_N on the column-split CTA pairs (W packed as two BLOCK_N-row
// halves: 256 for GraphCast's 512-wide latents, 192 for Pangu's C = 384 projection and fc2).
template <int BLOCK_N, bool kPair = false, class Sched, class Epi>
int launch_gemm2(const Sched& sc, const Epi& epi, long long M, int N, int batches, int num_sms, cudaStream_t st) {
  using Cfg = G2CfgOf<Sched, Epi, BLOCK_N>;
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
  if (!sc.valid()) {   // an operand the loader cannot walk: more than 6 A segments, a misaligned data batch (SchedTB)
    set_error("internal: GEMM operands (M=%lld N=%d BN=%d): schedule rejected", M, N, BLOCK_N);
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
        if (x.row0 + rr < x.M) {
          if (kImage)
            *reinterpret_cast<uint4*>(ibase + rr * 128 + (((((col & 63) >> 3) + ch) ^ (rr & 7)) << 4)) = pk;
          else
            *reinterpret_cast<uint4*>(out + (x.row0 + rr) * ldo + col + ch * 8) = pk;
        }
      }
      __syncwarp();
    }
  }
  // FragEpi (tile image only): the same arithmetic on the accumulator fragments, into the output tile
  static constexpr bool kLoadsTile = false;
  __device__ uint8_t* tile_image(int mt, int n0) const {
    return reinterpret_cast<uint8_t*>(out) + ((size_t)mt * nkb + (n0 >> 6)) * (size_t)G2_A_BYTES;
  }
  template <int BN, class Acc>
  __device__ void frag(Acc& acc, const FragCtx& x) const {
    static_assert(kImage, "fragment path: tile image output");
    const float* bp = bias + x.n0 + x.c2;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(bp + 8 * i));
      float* d = acc.d + 4 * i;
      if (kGelu) {
        gelu_erf_x2(d[0], d[1], b.x, b.y);
        gelu_erf_x2(d[2], d[3], b.x, b.y);
      } else {
        d[0] += b.x; d[1] += b.y; d[2] += b.x; d[3] += b.y;
      }
    }
    mbar_wait(x.out_ready, x.ready_parity);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(x.out_s + x.offset(i, false)), "r"(pack_half2(acc.d[4 * i], acc.d[4 * i + 1])) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(x.out_s + x.offset(i, true)), "r"(pack_half2(acc.d[4 * i + 2], acc.d[4 * i + 3])) : "memory");
    }
  }
};

// The staged LayerNorm / residual epilogue: Pangu's projection, fc2 and the second GEMMs of down- and up-sample, and every
// GraphCast LayerNorm MLP.  For each row of the tile
//   y   = LayerNorm(acc + bias) * gamma + beta   (kLn: the tile spans the row, or one column half of it in a CTA pair)
//   y   = acc + bias                             (!kLn: no statistics; bias may be null)
//   sum = res + y                                (kRes: the residual source, 0 none, 1 fp32 rows, 2 an fp16 tile image)
// and it writes any of xout (fp32 rows of sum), img (fp16 tile image of sum: the A operand of the next GEMM) and yimg (fp16
// tile image of y: what GraphCast's aggregation sums).  Each destination may be null; res may be one of them (an in-place
// update).  The residual source is a template argument because a run-time branch per load serialised the loads and cost
// the kernel 10 - 50 %.
// A stream kept only as its fp16 image (Pangu by default, GraphCast's grid nodes and mesh edges) passes res = img and
// xout = null: the sum is formed in fp32 and rounded once back into img.  On the oracle that moves the Pangu step error
// from 5.3e-4 to 5.9e-4 (tests/test_oracle_cpu.py) and GraphCast's tendency error over 16 layers from 7.66e-4 to 7.95e-4
// (tests/test_graphcast_cpu.py); it removes 8 of the 12 bytes per row and feature that Pangu's projection / MLP
// epilogues move through HBM, and 3 KB per row and launch of GraphCast's.
// Global traffic is 128-bit: lane -> (row = it*4 + lane/8, float4 column group = lane%8), i.e. eight lanes cover one
// 128-byte row segment.  bias / gamma / beta come from shared memory (kLn) or bias from global memory (!kLn).
template <bool kLn, int kRes>
struct Epi2F32Img {
  static_assert(kRes >= 0 && kRes <= 2, "residual source: none, fp32 rows, fp16 image");
  static constexpr bool kNeedsBias = kLn;
  const void* res;              // residual: fp32 rows ldx floats apart (kRes 1), or a tile image with nkb k-blocks (kRes 2)
  float* xout; int ldx;         // fp32 rows of the sum, ldx floats apart
  uint8_t* img; int nkb;        // fp16 tile image of the sum, nkb k-blocks per row tile
  uint8_t* yimg;                // fp16 tile image of y, in img's layout
  const float* bias; const float* gamma; const float* beta; float eps;
  // residual of the lane's eight (row, 4-column) pieces of the 32-column group at tile column c: all eight loads are
  // issued before any is used
  __device__ __forceinline__ void residual8(const EpiCtx& e, int c, int rsub4, int c4, size_t rowoff, long long rows_left, bool on,
                                            float4 (&r)[8]) const {
    if constexpr (kRes == 1) {
      const float* xin = static_cast<const float*>(res);
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        r[it] = (on && rr < rows_left) ? *reinterpret_cast<const float4*>(xin + rowoff + (size_t)rr * ldx + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else if constexpr (kRes == 2) {
      const int col = e.n0 + c + c4 * 4;
      const uint8_t* base = static_cast<const uint8_t*>(res) + ((size_t)(e.row0 >> 7) * nkb + (col >> 6)) * (size_t)G2_A_BYTES +
                            (uint32_t)(e.row0 & 127) * 128 + (c4 & 1) * 8;
      const uint32_t chunk = (uint32_t)(col & 63) >> 3;
      uint2 u[8];
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        u[it] = (on && rr < rows_left) ? *reinterpret_cast<const uint2*>(base + rr * 128 + ((chunk ^ (uint32_t)(rr & 7)) << 4)) : make_uint2(0u, 0u);
      }
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u[it].x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u[it].y));
        r[it] = make_float4(a.x, a.y, b.x, b.y);
      }
    } else {
#pragma unroll
      for (int it = 0; it < 8; ++it) r[it] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // Pull this warp's residual rows into L2 ahead of time, while the tile's main loop runs.
  template <int BN>
  __device__ void prefetch(const EpiCtx& e) const {
    if (kRes == 0) return;
    const long long row = e.row0 + e.lane;
    if (row >= e.M) return;
    if (kRes == 2) {
      const char* p = static_cast<const char*>(res) + ((size_t)(e.row0 >> 7) * nkb + (e.n0 >> 6)) * (size_t)G2_A_BYTES +
                      ((uint32_t)(e.row0 & 127) + e.lane) * 128;
#pragma unroll
      for (int i = e.part; i < BN / 64; i += e.nparts) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (size_t)i * G2_A_BYTES));
      return;
    }
    const char* p = reinterpret_cast<const char*>(static_cast<const float*>(res) + row * ldx + e.n0);
#pragma unroll
    for (int i = e.part; i < BN * 4 / 128; i += e.nparts) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + i * 128));
  }
  // The 16-byte image chunk (8 columns) of a lane pair: the even lane assembles the chunk of row it2, the odd lane that of
  // row it2 + 1, and the pair swaps the other halves by shuffle.  h: this lane's 4 columns of rows it2, it2 + 1.
  static __device__ __forceinline__ uint4 pair_chunk(const uint2 (&h)[2], int odd) {
    const uint2 send = odd ? h[0] : h[1];
    uint2 recv;
    recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
    recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
    return odd ? make_uint4(recv.x, recv.y, h[1].x, h[1].y) : make_uint4(h[0].x, h[0].y, recv.x, recv.y);
  }
  // Per 32x32 block: the row-owner lanes drop the raw accumulator into the warp's patch with 128-bit stores, then every
  // lane works on (row = it*4 + lane/8, 4 columns = lane%8) pieces.  The LayerNorm statistics of the 8 rows a lane touches
  // come from their owner lanes by shuffle; the fp16 image chunks are assembled from lane pairs by shuffle, not through
  // shared memory.  Every warp reduces the statistics of its own column groups only; the warps that share a lane quarter
  // exchange partial sums through their patches.  The residual of the next column group is loaded while this one is
  // processed (32 more registers).
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    constexpr int NG = BN / 32;
    static_assert(NG >= 2, "a column group for each warp of a lane quarter");
    const int rsub4 = e.lane >> 3, c4 = e.lane & 7;
    const long long rows_left = e.M - e.row0;          // >= 32 for every tile but the last
    const size_t rowoff = (size_t)e.row0 * ldx + e.n0 + c4 * 4;   // fp32 rows: this lane's columns in row row0
    const size_t ld4 = (size_t)4 * ldx;                             // from the lane's row it * 4 + rsub4 to its next
    // residual rows of the first column group: requested before the statistics pass (they come from L2: prefetch())
    float4 xr[8];
    residual8(e, e.part * 32, rsub4, c4, rowoff, rows_left, true, xr);
    float rs[8], ns[8];   // rstd and -mean*rstd of row it*4 + rsub4
#pragma unroll
    for (int it = 0; it < 8; ++it) { rs[it] = 1.f; ns[it] = 0.f; }
    if (kLn) {
      // columns of the row this warp's lane holds: the column groups part, part + nparts, ...
      const auto cols = [&](int p) { return (float)(32 * ((NG - p + e.nparts - 1) / e.nparts)); };
      // One pass over the staged tile (a second pass that re-read it cost a GraphCast step 1.5 %, H100 80GB HBM3 at
      // 700 W): sums about k, the mean of the lane's first 32-column group, which is in registers.  (k - mean)^2 <= m2 / 32,
      // so the sum of squares about k is at most (1 + cols / 32) m2 whatever |mean| / std is.
      float k = 0.f, s = 0.f, ss = 0.f;
      for (int g = e.part; g < NG; g += e.nparts) {
        float v[32];
        acc.load32(g * 32, v);
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 b = lds_f32x4_ro(e.svec_s + (g * 32 + j) * 4);
          v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
        }
        if (g == e.part) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) k += (v[j] + v[j + 1]) + (v[j + 2] + v[j + 3]);
          k *= 1.f / 32.f;
        }
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float y0 = v[j] - k, y1 = v[j + 1] - k, y2 = v[j + 2] - k, y3 = v[j + 3] - k;
          s += (y0 + y1) + (y2 + y3);
          ss += (y0 * y0 + y1 * y1) + (y2 * y2 + y3 * y3);
        }
      }
      const float d = s / cols(e.part);
      LnStat st{k + d, fmaxf(ss - s * d, 0.f)};
      if (e.nparts > 1) {
        // the warps of a lane quarter are 4 warps apart, and so are their patches.  Every warp merges all parts in the
        // same order, so all hold the same statistics.
        const uint32_t slot = e.patch_s + e.lane * 8;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(slot), "f"(st.mean), "f"(st.m2) : "memory");
        const int q = (int)((e.row0 >> 5) & 3);
        asm volatile("bar.sync %0, %1;" ::"r"(8 + q), "r"(32 * e.nparts) : "memory");
        float n = 0.f;
        for (int p = 0; p < e.nparts; ++p) {
          LnStat o;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(o.mean), "=f"(o.m2) : "r"(slot + (p - e.part) * 4 * (G2_PATCH_FLOATS * 4)));
          st = p ? ln_merge(st, n, o, cols(p)) : o;
          n += cols(p);
        }
        asm volatile("bar.sync %0, %1;" ::"r"(8 + q), "r"(32 * e.nparts) : "memory");   // the patches are reused below
      }
      float width = (float)BN;
      if (e.pair.own_bar) {   // column-split CTA pair: the other half of these rows is in the peer CTA
        if (e.part == 0) {
          if (e.lane == 0) e.pair.expect();
          __syncwarp();
          e.pair.post(e.lane, st);
        }
        e.pair.wait();
        e.pair.merge_peer(e.lane, st, (float)BN);
        width = (float)(2 * BN);
      }
      const float mean = st.mean;
      const float rstd = rsqrtf(st.m2 / width + eps);
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
      float4 xn[8];   // the next group's residual, in flight while this group is normalised and stored
      residual8(e, c + 32 * e.nparts, rsub4, c4, rowoff, rows_left, g + e.nparts < NG, xn);
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(e.patch_s, e.lane, v);
      }
      __syncwarp();
      float4 bs = make_float4(0.f, 0.f, 0.f, 0.f), ga = make_float4(1.f, 1.f, 1.f, 1.f), be = make_float4(0.f, 0.f, 0.f, 0.f);
      if (kLn) {
        bs = lds_f32x4_ro(e.svec_s + (c + c4 * 4) * 4);
        ga = lds_f32x4_ro(e.svec_s + (G2_VEC_FLOATS + c + c4 * 4) * 4);
        be = lds_f32x4_ro(e.svec_s + (2 * G2_VEC_FLOATS + c + c4 * 4) * 4);
      } else if (bias) {
        bs = __ldg(reinterpret_cast<const float4*>(bias + e.n0 + c + c4 * 4));
      }
      const int col = e.n0 + c;
      const size_t tile_off = ((size_t)(e.row0 >> 7) * nkb + (col >> 6)) * (size_t)G2_A_BYTES + r0 * 128;
      const uint32_t cb = (((uint32_t)col & 63u) >> 3) + (uint32_t)(c4 >> 1);   // 16-byte chunk of this lane pair inside the image row
      size_t xo = rowoff + (size_t)rsub4 * ldx + c;   // xout offset of the lane's row it * 4 + rsub4: one add per row
#pragma unroll
      for (int it2 = 0; it2 < 8; it2 += 2) {
        uint2 hs[2], hy[2];   // fp16 of the sum and of y, rows it2 and it2 + 1
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int it = it2 + u;
          const int rr = it * 4 + rsub4;
          const float4 t = lds_f32x4(patchv_addr(e.patch_s, rr, c4));
          float4 y;
          y.x = fmaf(fmaf(t.x + bs.x, rs[it], ns[it]), ga.x, be.x); y.y = fmaf(fmaf(t.y + bs.y, rs[it], ns[it]), ga.y, be.y);
          y.z = fmaf(fmaf(t.z + bs.z, rs[it], ns[it]), ga.z, be.z); y.w = fmaf(fmaf(t.w + bs.w, rs[it], ns[it]), ga.w, be.w);
          hy[u].x = pack_half2(y.x, y.y); hy[u].y = pack_half2(y.z, y.w);
          if (kRes) { y.x += xr[it].x; y.y += xr[it].y; y.z += xr[it].z; y.w += xr[it].w; }
          if (xout && rr < rows_left) *reinterpret_cast<float4*>(xout + xo) = y;
          xo += ld4;
          hs[u].x = pack_half2(y.x, y.y); hs[u].y = pack_half2(y.z, y.w);
        }
        const int rr = (it2 + odd) * 4 + rsub4;
        const uint32_t coff = rr * 128 + ((cb ^ (uint32_t)(rr & 7)) << 4);
        if (img) {
          const uint4 pk = pair_chunk(hs, odd);
          if (rr < rows_left) *reinterpret_cast<uint4*>(img + tile_off + coff) = pk;
        }
        if (yimg) {
          const uint4 pk = pair_chunk(hy, odd);
          if (rr < rows_left) *reinterpret_cast<uint4*>(yimg + tile_off + coff) = pk;
        }
      }
      __syncwarp();
      if (kRes) {
#pragma unroll
        for (int it = 0; it < 8; ++it) xr[it] = xn[it];
      }
    }
  }
  // FragEpi: the same arithmetic on the accumulator fragments, only for LayerNorm with the residual read in place from the
  // fp16 image (kLn, kRes == 2, res == img; xout and yimg are not written).  The loader fills the output tile with img's
  // bytes, which are the residual, and the sum overwrites them.  A warpgroup holds whole rows, so a row's statistics are
  // the thread's sums added across its lane quad (and, in a CTA pair, the peer's).
  static constexpr bool kLoadsTile = kRes == 2;
  __device__ uint8_t* tile_image(int mt, int n0) const { return img + ((size_t)mt * nkb + (n0 >> 6)) * (size_t)G2_A_BYTES; }
  template <int BN, class Acc>
  __device__ void frag(Acc& acc, const FragCtx& x) const {
    static_assert(kLn && kRes == 2, "fragment path: LayerNorm with the fp16 image's in-place residual");
    constexpr float kCols = (float)(BN / 4);        // columns of a row in one thread
    // rows x.row, x.row + 8; each pass adds the even and the odd 8-column groups in two independent chains, which halves
    // the latency the second pass puts in front of the next tile's main loop
    LnStat st[2];
    float a[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      float2 b;
      asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b.x), "=f"(b.y) : "r"(x.svec_s + (uint32_t)(8 * i + x.c2) * 4u));
      float* d = acc.d + 4 * i;
      d[0] += b.x; d[1] += b.y; d[2] += b.x; d[3] += b.y;
      a[0][i & 1] += d[0] + d[1];
      a[1][i & 1] += d[2] + d[3];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      st[h].mean = (a[h][0] + a[h][1]) * (1.f / kCols);
      a[h][0] = a[h][1] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < BN / 8; ++i)   // second pass, about the thread's mean
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float y0 = acc.d[4 * i + 2 * h] - st[h].mean, y1 = acc.d[4 * i + 2 * h + 1] - st[h].mean;
        a[h][i & 1] += y0 * y0 + y1 * y1;
      }
#pragma unroll
    for (int h = 0; h < 2; ++h) st[h].m2 = a[h][0] + a[h][1];
    // the lane quad holds the whole row: two merges of equal halves
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        const LnStat p{__shfl_xor_sync(0xffffffffu, st[h].mean, o), __shfl_xor_sync(0xffffffffu, st[h].m2, o)};
        st[h] = ln_merge(st[h], kCols * o, p, kCols * o);
      }
    float width = (float)BN;
    if (x.pair.own_bar) {
      // column-split CTA pair: lane (l & 3) == h of each quad posts row x.row + 8 h; the two warps of a 32-row group share
      // one barrier, whose transaction bytes one of them announces
      const int lane = threadIdx.x & 31, h = lane & 3;
      if (x.post_bar && lane == 0) x.pair.expect();
      __syncwarp();
      if (h < 2) x.pair.post(x.row + 8 * h, h ? st[1] : st[0]);
      x.pair.wait();
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) x.pair.merge_peer(x.row + 8 * hh, st[hh], (float)BN);
      width = (float)(2 * BN);
    }
    float rs[2], ns[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rs[h] = rsqrtf(st[h].m2 / width + eps);
      ns[h] = -st[h].mean * rs[h];
    }
    mbar_wait(x.out_ready, x.ready_parity);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      float2 ga, be;
      asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(ga.x), "=f"(ga.y) : "r"(x.svec_s + (uint32_t)(G2_VEC_FLOATS + 8 * i + x.c2) * 4u));
      asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(be.x), "=f"(be.y) : "r"(x.svec_s + (uint32_t)(2 * G2_VEC_FLOATS + 8 * i + x.c2) * 4u));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t a = x.out_s + x.offset(i, h);
        const float* d = acc.d + 4 * i + 2 * h;
        float y0 = fmaf(fmaf(d[0], rs[h], ns[h]), ga.x, be.x), y1 = fmaf(fmaf(d[1], rs[h], ns[h]), ga.y, be.y);
        uint32_t r;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r) : "r"(a));
        const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(&r));
        y0 += rf.x; y1 += rf.y;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack_half2(y0, y1)) : "memory");
      }
    }
  }
};

// up-sample linear1 (N = 4C as (hs, ws, C); one n-tile = one sub-position): LayerNorm over
// the C features of the tile, written as fp16 image rows of the FINE token
// (z, 2*h2+hs, 2*w2+ws) when it survives the crop.
struct Epi2UpShuffle {
  static constexpr bool kNeedsBias = false;
  uint8_t* img; int nkb; int C; const float* gamma; const float* beta; float eps; const float* bias;  // bias unused
  int H, W, H2, W2;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    // the lane holds its whole row: two passes, the mean, then m2 about it (LnStat)
    float mean = 0.f, m2 = 0.f;
    for (int c = 0; c < BN; c += 32) {
      float v[32];
      acc.load32(c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) mean += v[j];
    }
    mean /= BN;
    for (int c = 0; c < BN; c += 32) {
      float v[32];
      acc.load32(c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j) { const float t = v[j] - mean; m2 += t * t; }
    }
    const float rstd = rsqrtf(m2 / BN + eps);
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
