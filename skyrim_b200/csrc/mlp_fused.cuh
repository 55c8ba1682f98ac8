// Pangu's MLP as one persistent wgmma kernel per 128-row tile (k_mlp_fused):
//
//   xh <- xh + LayerNorm(GELU(xh W1^T + b1) W2^T + b2) * gamma + beta
//
// The two-GEMM path writes the 4C-wide hidden activation to HBM as fc1's fp16 image and fc2 reads it back: at C = 192 that
// is 800 MB per block and member, which makes fc2 HBM-bound.  Here the hidden activation never leaves the SM.  Per tile,
// the loader bulk-loads the tile's C / 64 k-blocks of xh once (the x tile, resident for the whole tile), and the 4C hidden
// columns are walked in chunks of 64.  For chunk j each consumer warpgroup
//   fc1   computes its 64 rows x 64 hidden columns with m64n64k16 over the x tile's k-blocks, against W1's 64-row slice j
//         (W1 packed at BLOCK_N 64: the slice's k-blocks are one contiguous 24 KB run);
//   GELU  adds the bias and applies GELU on the fragment with the arithmetic of Epi2F16<true, true>::frag, rounds once to
//         fp16 and writes its 64 rows into the H k-block (128 rows x 128 B, SWIZZLE_128B, the A operand layout);
//   fc2   accumulates H W2[:, 64 j : 64 j + 64]^T into its 64 x 192 accumulator with the m64n192k16 products of the
//         two-GEMM path's fc2 (k-block j of W2, packed at BLOCK_N 192, is one contiguous 24 KB run).
// After the last chunk FragEpi<Epi2F32Img<true, 2>>::frag runs unchanged on the fc2 accumulator (LayerNorm over the
// row, residual read in place from the output tile, which the loader filled from xh) and the loader bulk-stores the tile.
//
// The fc2 accumulation visits hidden k-blocks 0 .. 4C/64 - 1 in order with the same instructions on the same fp16 values,
// and fc1's m64n64k16 products give, column by column, the sums of the two-GEMM path's m64n192k16 ones: the result is
// bit for bit that of fc1 + fc2 (tests/test_pangu_mlp_fused_gpu.py).
//
// The ring carries only weights, in 24 KB stages: W1 slice j, then W2 k-block j, for every chunk.  One H k-block is
// enough: a warpgroup writes chunk j's H only after the wgmma_wait<0> that fc1 of chunk j needs anyway, and that wait also
// completes fc2 of chunk j - 1, the last reader of H.  Each warpgroup reads and writes only its own 64 rows of H, so the
// hand-over from the GELU's generic stores to the wgmma's async-proxy reads is a proxy fence and a barrier among the
// warpgroup's 128 threads.
#pragma once
#include "gemm2.cuh"

namespace sky {

// Shared memory of k_mlp_fused at C = NKB * 64 (C = 192: x 48 KB, H 16 KB, output tile 48 KB, vectors and barriers
// 6.25 KB, 4 ring stages of 24 KB).
template <int NKB>
struct MlpCfg {
  static constexpr int C = NKB * 64;
  static constexpr int NCHUNK = 4 * NKB;                        // hidden chunks of 64 columns
  static constexpr int W1_KB_BYTES = 64 * 128;                  // one k-block of W1's 64-row slice
  static constexpr int W1_CHUNK_BYTES = NKB * W1_KB_BYTES;      // W1 slice j: all C / 64 k-blocks
  static constexpr int W2_KB_BYTES = C * 128;                   // W2 k-block j: all C rows
  static constexpr int STAGE_BYTES = W1_CHUNK_BYTES > W2_KB_BYTES ? W1_CHUNK_BYTES : W2_KB_BYTES;
  static constexpr int X_BYTES = NKB * G2_A_BYTES;
  static constexpr int H_BYTES = G2_A_BYTES;
  static constexpr int OUT_BYTES = NKB * G2_A_BYTES;            // the output tile: the stream's C columns of the tile
  static constexpr int VEC_BYTES = 3 * G2_VEC_FLOATS * 4;       // fc2 bias | gamma | beta
  static constexpr int BAR_BYTES = 256;
  static constexpr int FIXED = 1024 /*align*/ + X_BYTES + H_BYTES + OUT_BYTES + VEC_BYTES + BAR_BYTES;
  static constexpr int MAXS = (232448 - FIXED) / STAGE_BYTES;
  static constexpr int STAGES = MAXS > 6 ? 6 : MAXS;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = RING_BYTES + FIXED;
  static constexpr int THREADS = (G2_EPI_WARPS + 1) * 32;      // two consumer warpgroups, one loader warp
  // offsets from the 1024-byte aligned base
  static constexpr int X_OFF = RING_BYTES, H_OFF = X_OFF + X_BYTES, OUT_OFF = H_OFF + H_BYTES, VEC_OFF = OUT_OFF + OUT_BYTES,
                       BAR_OFF = VEC_OFF + VEC_BYTES;
  static_assert(NKB == 3, "one CTA holds the whole 192-column fc2 accumulator of its rows (96 registers per thread)");
  static_assert(STAGE_BYTES % 1024 == 0 && X_OFF % 1024 == 0 && H_OFF % 1024 == 0 && OUT_OFF % 1024 == 0, "SWIZZLE_128B alignment");
  static_assert(STAGES >= 3, "pipeline depth");
  static_assert((2 * STAGES + 4) * 8 <= BAR_BYTES, "barrier block");
  static_assert(SMEM_BYTES <= 232448, "smem budget");
};

struct MlpArgs {
  uint8_t* xh;           // the stream's fp16 image, NKB k-blocks per row tile: A operand of fc1 and residual, updated in place
  const uint8_t* w1;     // fc1 weight image at BLOCK_N 64: [4C / 64][C / 64][64 rows x 128 B]
  const uint8_t* w2;     // fc2 weight image at BLOCK_N 192: [1][4C / 64][C rows x 128 B]
  const float* b1;       // fc1 bias [4C]
  FragEpi<Epi2F32Img<true, 2>> ln;   // fc2's epilogue: bias, gamma, beta, eps; res = img = xh
  long long M;
};

// Chunk epilogue of fc1: bias + GELU on the thread's fc1 fragment (rows row and row + 8, columns 8 i + c2 + {0, 1} of the
// chunk), with the arithmetic of Epi2F16<true, true>::frag, rounded once to fp16 into the H k-block at h_s (SWIZZLE_128B).
// bp: the fc1 bias of the thread's first column.
__device__ __forceinline__ void gelu_into_h(WgAcc<64>& acc1, const float* bp, uint32_t h_s, int row, int c2) {
  const uint32_t r0 = (uint32_t)row, r8 = r0 + 8u;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(bp + 8 * i));
    float* d = acc1.d + 4 * i;
    gelu_erf_x2(d[0], d[1], b.x, b.y);
    gelu_erf_x2(d[2], d[3], b.x, b.y);
    const uint32_t o0 = r0 * 128u + ((((uint32_t)i) ^ (r0 & 7u)) << 4) + (uint32_t)c2 * 2u;
    const uint32_t o8 = r8 * 128u + ((((uint32_t)i) ^ (r8 & 7u)) << 4) + (uint32_t)c2 * 2u;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(h_s + o0), "r"(pack_half2(d[0], d[1])) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(h_s + o8), "r"(pack_half2(d[2], d[3])) : "memory");
  }
}

template <int NKB>
__global__ void __launch_bounds__(MlpCfg<NKB>::THREADS, 1) k_mlp_fused(const MlpArgs a) {
  using Cfg = MlpCfg<NKB>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xs = smem + Cfg::X_OFF;
  uint8_t* outs = smem + Cfg::OUT_OFF;
  float* sbias = reinterpret_cast<float*>(smem + Cfg::VEC_OFF);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* x_full = bars + 2 * Cfg::STAGES;       // loader -> consumers: the tile's x k-blocks have landed
  uint64_t* x_free = x_full + 1;                   // consumers -> loader: the tile's last fc1 products have read the x tile
  uint64_t* out_full = x_full + 2;                 // consumers -> loader: the output tile is written
  uint64_t* out_ready = x_full + 3;                // loader -> consumers: the output tile holds the residual

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;
  const G2Grid g{a.M, (int)((a.M + G2_BLOCK_M - 1) / G2_BLOCK_M), 1, 1};
  const int num_tiles = g.num_m_tiles;
  constexpr int LOADER = G2_EPI_WARPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], G2_EPI_WARPS); }
    mbar_init(x_full, 1); mbar_init(x_free, G2_EPI_WARPS);
    mbar_init(out_full, G2_EPI_WARPS); mbar_init(out_ready, 1);
    mbar_fence_init();
  }
  for (int i = threadIdx.x; i < Cfg::C; i += blockDim.x) {
    sbias[i] = a.ln.bias[i]; sbias[G2_VEC_FLOATS + i] = a.ln.gamma[i]; sbias[2 * G2_VEC_FLOATS + i] = a.ln.beta[i];
  }
  __syncthreads();

  int it = 0;
  if (warp == LOADER) {
    // Per tile: the x tile once x_free says the previous tile's fc1 is done with it, then W1 slice j and W2 k-block j for
    // every chunk.  After the first STAGES weight blocks (which only wait for ring slots) the output tile is handed over:
    // the previous tile's is stored once its epilogue is done, and this tile's is filled with the residual.
    int s = 0; uint32_t ph = 0;
    G2Tile prev{};
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const G2Tile t{0, tile, 0, false};
      const uint8_t* xsrc = a.xh + (size_t)tile * Cfg::X_BYTES;
      if (lane == 0) {
        // the next tile's x is pulled into L2 a tile ahead of its load (and of the residual's, which reads it again)
        if (tile + (int)gridDim.x < num_tiles) bulk_prefetch_l2(xsrc + (size_t)gridDim.x * Cfg::X_BYTES, Cfg::X_BYTES);
        if (it > 0) mbar_wait(x_free, (uint32_t)(it - 1) & 1);
        mbar_arrive_expect_tx(x_full, Cfg::X_BYTES);
        bulk_g2s(xs, xsrc, Cfg::X_BYTES, x_full);
      }
      __syncwarp();
      for (int i = 0; i < 2 * Cfg::NCHUNK; ++i) {
        mbar_wait(&empty[s], ph ^ 1);
        if (lane == 0) {
          const int j = i >> 1;
          const uint8_t* src = (i & 1) ? a.w2 + (size_t)j * Cfg::W2_KB_BYTES : a.w1 + (size_t)j * Cfg::W1_CHUNK_BYTES;
          const uint32_t bytes = (i & 1) ? Cfg::W2_KB_BYTES : Cfg::W1_CHUNK_BYTES;
          mbar_arrive_expect_tx(&full[s], bytes);
          bulk_g2s(smem + s * Cfg::STAGE_BYTES, src, bytes, &full[s]);
        }
        __syncwarp();
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
        if (i + 1 != Cfg::STAGES) continue;
        if (it > 0) {
          mbar_wait(out_full, (uint32_t)(it - 1) & 1);
          frag_store<Cfg>(a.ln, prev, smem_u32(outs), a.M, 0, lane);
        }
        if (lane == 0) {
          mbar_arrive_expect_tx(out_ready, Cfg::OUT_BYTES);
          bulk_g2s(outs, xsrc, Cfg::OUT_BYTES, out_ready);
        }
        __syncwarp();
      }
      prev = t;
    }
    if (it > 0) {
      mbar_wait(out_full, (uint32_t)(it - 1) & 1);
      frag_store<Cfg>(a.ln, prev, smem_u32(outs), a.M, 0, lane);
      bulk_wait<0>();
    }
  } else {
    const int wg = warp >> 2, w = warp & 3;
    FragCtx x;
    x.row = 64 * wg + 16 * w + (lane >> 2);
    x.c2 = 2 * (lane & 3);
    x.n0 = 0;
    x.out_s = smem_u32(outs);
    x.svec_s = smem_u32(sbias);
    x.out_ready = out_ready;
    const uint32_t ring_s = smem_u32(smem), x_s = smem_u32(xs) + (uint32_t)wg * 8192u;
    const uint32_t h_s = smem_u32(smem + Cfg::H_OFF);
    const uint64_t da_h = make_desc_sw128(h_s + (uint32_t)wg * 8192u);
    WgAcc<64> acc1;
    WgAcc<Cfg::C> acc2;
    int s = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      x.ready_parity = (uint32_t)it & 1;
      mbar_wait(x_full, (uint32_t)it & 1);
      acc2.zero();
      acc1.zero();
      wgmma_fence_operands(acc1.d);
      int prev2 = -1;   // ring stage of the previous chunk's W2 k-block, released once its products have completed
      for (int j = 0; j < Cfg::NCHUNK; ++j) {
        // ---- fc1: 64 rows x 64 hidden columns over the x tile ----
        mbar_wait(&full[s], ph);
        wgmma_fence();
        const uint32_t w1s = ring_s + (uint32_t)(s * Cfg::STAGE_BYTES);
#pragma unroll
        for (int kb = 0; kb < NKB; ++kb) {
          const uint64_t da = make_desc_sw128(x_s + (uint32_t)(kb * G2_A_BYTES)), db = make_desc_sw128(w1s + (uint32_t)(kb * Cfg::W1_KB_BYTES));
#pragma unroll
          for (int k = 0; k < 4; ++k) Wgmma<64, false>::mma(acc1.d, da + 2 * k, db + 2 * k);
        }
        wgmma_commit();
        wgmma_wait<0>();   // fc1 of chunk j and fc2 of chunk j - 1 have completed
        wgmma_fence_operands(acc1.d);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&empty[s]);
          if (prev2 >= 0) mbar_arrive(&empty[prev2]);
          if (j == Cfg::NCHUNK - 1) mbar_arrive(x_free);
        }
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
        // ---- bias + GELU, one fp16 rounding, into H ----
        gelu_into_h(acc1, a.b1 + 64 * j + x.c2, h_s, x.row, x.c2);
        // zeroed for the next chunk here, while no product is in flight: zeroing registers under fc2's products would
        // make ptxas wait for them before fc1's
        acc1.zero();
        wgmma_fence_operands(acc1.d);   // keeps ptxas from sinking the zeroing to the products
        fence_proxy_async_smem();
        named_bar_sync(2 + wg, 128);   // the warpgroup's 64 rows of H are written before its wgmma reads them
        // ---- fc2: one k-block, H against W2 k-block j ----
        mbar_wait(&full[s], ph);
        wgmma_fence();
        const uint64_t db2 = make_desc_sw128(ring_s + (uint32_t)(s * Cfg::STAGE_BYTES));
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<Cfg::C, false>::mma(acc2.d, da_h + 2 * k, db2 + 2 * k);
        wgmma_commit();
        prev2 = s;
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
      acc2.settle();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev2]);
      a.ln.template frag<Cfg::C>(acc2, x);
      fence_proxy_async_smem();   // the tile's generic writes are ordered before the loader's bulk store
      __syncwarp();
      if (lane == 0) mbar_arrive(out_full);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// C = 384 on column-split CTA pairs (k_mlp_fused_pair).  A 128 x 384 fc2 accumulator does not fit one CTA, so as for fc2
// (k_gemm2_pair) the two CTAs of a cluster take the same 128-row tile and 192 fc2 columns each, and cross their LayerNorm row
// statistics through PairStats.  Both need every hidden chunk; CTA r computes fc1 only for the chunks j = r (mod 2) and
// sends each one to the peer: after writing its rows of H slot r, a warpgroup bulk-copies them (8 KB) into the same rows of
// the peer's slot r, completing the peer's h_full barrier.  Slot r is written again two chunks later, once the peer has
// arrived (remotely) on this CTA's h_cons barrier: that arrival follows the peer's fc2 of the chunk, hence also the end of
// the copy that read the slot.  Per warpgroup and CTA, fc1 runs 12 times per tile (K = 384 over two ring stages) and fc2 24.
// The x tile (96 KB, resident for the tile) holds the output tile too: CTA r's 192 columns are its k-blocks 3r .. 3r + 2, the
// residual of the epilogue, which overwrites them in place; the next tile's x is loaded once the loader has stored them.
// Shared memory: ring 3 x 24 KB, x 96 KB, H 2 x 16 KB, vectors 6 KB, barriers 256 B, pair slots 2 KB, alignment 1 KB.
// ---------------------------------------------------------------------------------------------------------------
struct MlpPairCfg {
  static constexpr int NKB = 6, C = 384, HALF = 192, NCHUNK = 24;
  static constexpr int STAGE_BYTES = 3 * 64 * 128;        // three 8 KB k-blocks of a W1 slice, or one W2 k-block (192 rows)
  static constexpr int X_BYTES = NKB * G2_A_BYTES;
  static constexpr int OUT_BYTES = 3 * G2_A_BYTES;         // frag_store: the CTA's three column blocks of the tile
  static constexpr int H_BYTES = 2 * G2_A_BYTES;
  static constexpr int VEC_BYTES = 3 * G2_VEC_FLOATS * 4;
  static constexpr int BAR_BYTES = 256;
  static constexpr int FIXED = 1024 + X_BYTES + H_BYTES + VEC_BYTES + BAR_BYTES + G2_PAIR_SMEM;
  static constexpr int STAGES = (232448 - FIXED) / STAGE_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = RING_BYTES + FIXED;
  static constexpr int THREADS = (G2_EPI_WARPS + 1) * 32;
  static constexpr int X_OFF = RING_BYTES, H_OFF = X_OFF + X_BYTES, VEC_OFF = H_OFF + H_BYTES, BAR_OFF = VEC_OFF + VEC_BYTES,
                       STAT_OFF = BAR_OFF + BAR_BYTES;
  static_assert(STAGES >= 3, "a W1 slice (two stages) beside the W2 k-block still in flight");
  static_assert(X_OFF % 1024 == 0 && H_OFF % 1024 == 0, "SWIZZLE_128B alignment");
  static_assert((2 * STAGES + 2 + 4 + 8) * 8 <= BAR_BYTES, "barrier block");
  static_assert(SMEM_BYTES <= 232448, "smem budget");
};

__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "SKY_WAITC_%=:\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra SKY_DONEC_%=;\n\t"
      "bra SKY_WAITC_%=;\n\t"
      "SKY_DONEC_%=:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(0x989680)
      : "memory");
}

// 288 threads put three warps on one SM sub-partition, whose 16K registers allow 168 per thread: ptxas keeps the two
// accumulator sets (128 registers) and spills about 20 loop-invariant values (84 bytes), reloaded from L1.
template <int NKB>   // 6: a template only so that every translation unit that launches it may instantiate it
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(MlpPairCfg::THREADS, 1) k_mlp_fused_pair(const MlpArgs a) {
  using Cfg = MlpPairCfg;
  static_assert(NKB == Cfg::NKB, "C = 384");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xs = smem + Cfg::X_OFF;
  float* sbias = reinterpret_cast<float*>(smem + Cfg::VEC_OFF);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* x_full = bars + 2 * Cfg::STAGES;   // loader -> consumers: x (and with it the output tile's residual) has landed
  uint64_t* out_full = x_full + 1;             // consumers -> loader: the output tile is written
  uint64_t* h_full = x_full + 2;               // [wg]: the peer's rows of its chunk have landed in slot rank ^ 1
  uint64_t* h_cons = x_full + 4;               // [wg]: the peer's fc2 has consumed this CTA's last chunk (remote arrive)
  uint64_t* xbar = x_full + 6;                 // PairStats barriers [2][4]
  float* xstat = reinterpret_cast<float*>(smem + Cfg::STAT_OFF);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;
  const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
  const int num_tiles = (int)((a.M + G2_BLOCK_M - 1) / G2_BLOCK_M);
  const int pair0 = blockIdx.x >> 1, npairs = gridDim.x >> 1;
  constexpr int LOADER = G2_EPI_WARPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], G2_EPI_WARPS); }
    mbar_init(x_full, 1); mbar_init(out_full, G2_EPI_WARPS);
    for (int g = 0; g < 2; ++g) { mbar_init(&h_full[g], 1); mbar_init(&h_cons[g], 1); }
    for (int i = 0; i < 8; ++i) mbar_init(&xbar[i], 1);
    mbar_fence_init();
  }
  for (int i = threadIdx.x; i < Cfg::HALF; i += blockDim.x) {
    const int c = (int)rank * Cfg::HALF + i;
    sbias[i] = a.ln.bias[c]; sbias[G2_VEC_FLOATS + i] = a.ln.gamma[c]; sbias[2 * G2_VEC_FLOATS + i] = a.ln.beta[c];
  }
  __syncthreads();
  cluster_sync_all();   // the peer's barriers exist before anything is copied or posted to them

  const uint32_t out_s = smem_u32(xs) + rank * (uint32_t)Cfg::OUT_BYTES;
  int it = 0;
  if (warp == LOADER) {
    // Per tile: the first STAGES weight blocks only wait for ring slots; then the previous tile's output tile is stored once
    // its epilogue is done, the x tile (which holds it) is reloaded for this tile, and the rest of the weights follow: for
    // chunk j, W1 slice j in two stages if this CTA computes it, then k-block j of this CTA's half of W2.
    int s = 0; uint32_t ph = 0;
    G2Tile prev{};
    const uint8_t* w2 = a.w2 + (size_t)rank * Cfg::NCHUNK * Cfg::STAGE_BYTES;
    auto put = [&](const uint8_t* src) {
      mbar_wait(&empty[s], ph ^ 1);
      if (lane == 0) {
        mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
        bulk_g2s(smem + s * Cfg::STAGE_BYTES, src, Cfg::STAGE_BYTES, &full[s]);
      }
      __syncwarp();
      if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
    };
    for (int tile = pair0; tile < num_tiles; tile += npairs, ++it) {
      int n = 0;
      for (int j = 0; j < Cfg::NCHUNK; ++j) {
        for (int part = 0; part < 3; ++part) {
          if (part < 2 && (j & 1) != (int)rank) continue;
          put(part < 2 ? a.w1 + ((size_t)j * 2 + part) * Cfg::STAGE_BYTES : w2 + (size_t)j * Cfg::STAGE_BYTES);
          if (++n != Cfg::STAGES) continue;
          if (it > 0) {
            mbar_wait(out_full, (uint32_t)(it - 1) & 1);
            frag_store<Cfg>(a.ln, prev, out_s, a.M, Cfg::HALF, lane);
          }
          if (lane == 0) {
            const uint8_t* xsrc = a.xh + (size_t)tile * Cfg::X_BYTES;
            mbar_arrive_expect_tx(x_full, Cfg::X_BYTES);
            bulk_g2s(xs, xsrc, Cfg::X_BYTES, x_full);
            if (tile + npairs < num_tiles) bulk_prefetch_l2(xsrc + (size_t)npairs * Cfg::X_BYTES, Cfg::X_BYTES);
          }
          __syncwarp();
        }
      }
      prev = G2Tile{0, tile, (int)rank, false};
    }
    if (it > 0) {
      mbar_wait(out_full, (uint32_t)(it - 1) & 1);
      frag_store<Cfg>(a.ln, prev, out_s, a.M, Cfg::HALF, lane);
      bulk_wait<0>();
    }
  } else {
    const int wg = warp >> 2, w = warp & 3;
    const bool leader = w == 0 && lane == 0;   // the warpgroup's copies, expectations and remote arrivals
    FragCtx x;
    x.row = 64 * wg + 16 * w + (lane >> 2);
    x.c2 = 2 * (lane & 3);
    x.n0 = (int)rank * Cfg::HALF;
    x.out_s = out_s;
    x.svec_s = smem_u32(sbias);
    x.out_ready = x_full;
    x.post_bar = (w & 1) == 0;
    const uint32_t ring_s = smem_u32(smem), x_s = smem_u32(xs) + (uint32_t)wg * 8192u;
    const uint32_t h_own = smem_u32(smem + Cfg::H_OFF) + rank * (uint32_t)G2_A_BYTES;
    const uint32_t h_peer = smem_u32(smem + Cfg::H_OFF) + peer * (uint32_t)G2_A_BYTES;
    const uint64_t da_own = make_desc_sw128(h_own + (uint32_t)wg * 8192u), da_peer = make_desc_sw128(h_peer + (uint32_t)wg * 8192u);
    const uint32_t h_own_remote = mapa_u32(h_own + (uint32_t)wg * 8192u, peer);    // the same rows of slot rank in the peer
    const uint32_t h_full_remote = mapa_u32(smem_u32(&h_full[wg]), peer);
    const uint32_t h_cons_remote = mapa_u32(smem_u32(&h_cons[wg]), peer);
    WgAcc<64> acc1;
    WgAcc<Cfg::HALF> acc2;
    int s = 0; uint32_t ph = 0;
    uint32_t n_own = 0, n_peer = 0;   // chunks computed here / received, over the CTA's life
    bool consumed = false;            // a received chunk's fc2 has been issued but not yet reported to the peer
    int pend = -1;                    // ring stage of the last W2 k-block whose products may still be in flight
    auto release = [&](int st) { if (st >= 0 && lane == 0) mbar_arrive(&empty[st]); };
    auto fc2 = [&](uint64_t da) {
      mbar_wait(&full[s], ph);
      wgmma_fence();
      const uint64_t db = make_desc_sw128(ring_s + (uint32_t)(s * Cfg::STAGE_BYTES));
#pragma unroll
      for (int k = 0; k < 4; ++k) Wgmma<Cfg::HALF, false>::mma(acc2.d, da + 2 * k, db + 2 * k);
      wgmma_commit();
    };
    for (int tile = pair0; tile < num_tiles; tile += npairs, ++it) {
      x.ready_parity = (uint32_t)it & 1;
      x.pair = PairStats::at(xbar, xstat, it, x.row >> 5, rank);
      mbar_wait(x_full, (uint32_t)it & 1);
      acc2.zero();
      acc1.zero();
      wgmma_fence_operands(acc1.d);
      for (int j = 0; j < Cfg::NCHUNK; ++j) {
        if ((j & 1) == (int)rank) {
          // ---- fc1 of chunk j over the x tile: k-blocks 0-2 from one stage, 3-5 from the next ----
          const int sa = s;
          mbar_wait(&full[s], ph);
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
          const int sb = s;
          mbar_wait(&full[s], ph);
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
          wgmma_fence();
#pragma unroll
          for (int kb = 0; kb < Cfg::NKB; ++kb) {
            const uint32_t wst = ring_s + (uint32_t)((kb < 3 ? sa : sb) * Cfg::STAGE_BYTES + (kb % 3) * 64 * 128);
            const uint64_t da = make_desc_sw128(x_s + (uint32_t)(kb * G2_A_BYTES)), db = make_desc_sw128(wst);
#pragma unroll
            for (int k = 0; k < 4; ++k) Wgmma<64, false>::mma(acc1.d, da + 2 * k, db + 2 * k);
          }
          wgmma_commit();
          wgmma_wait<0>();   // fc1 of chunk j and every earlier fc2 have completed
          wgmma_fence_operands(acc1.d);
          __syncwarp();
          release(sa); release(sb); release(pend);
          pend = -1;
          if (consumed) {
            if (leader) asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(h_cons_remote) : "memory");
            consumed = false;
          }
          // slot rank is free here once the peer has consumed this CTA's previous chunk (and so the copy has read it)
          if (n_own > 0) mbar_wait_cluster(&h_cons[wg], (n_own - 1) & 1);
          gelu_into_h(acc1, a.b1 + 64 * j + x.c2, h_own, x.row, x.c2);
          acc1.zero();
          wgmma_fence_operands(acc1.d);
          fence_proxy_async_smem();
          named_bar_sync(2 + wg, 128);   // the warpgroup's 64 rows of H are written
          if (leader)
            asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(h_own_remote),
                         "r"(h_own + (uint32_t)wg * 8192u), "r"(8192), "r"(h_full_remote)
                         : "memory");
          ++n_own;
          fc2(da_own);
          pend = s;
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
        } else {
          // ---- the peer's chunk: its rows arrive in slot peer ----
          if (leader) mbar_arrive_expect_tx(&h_full[wg], 8192);
          mbar_wait(&h_full[wg], n_peer & 1);
          ++n_peer;
          fc2(da_peer);
          wgmma_wait<1>();   // the previous chunk's fc2 has completed: its W2 stage goes back to the ring
          __syncwarp();
          release(pend);
          pend = s;
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
          consumed = true;
        }
      }
      acc2.settle();
      __syncwarp();
      release(pend);
      pend = -1;
      if (consumed) {
        if (leader) asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(h_cons_remote) : "memory");
        consumed = false;
      }
      a.ln.template frag<Cfg::HALF>(acc2, x);
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(out_full);
    }
  }
  __syncthreads();
  cluster_sync_all();   // nobody leaves while the peer may still copy, arrive or post into this CTA
}

// fc1 + GELU + fc2 + LayerNorm + residual on the stream image xh (in place) for M tokens at C = NKB * 64.
template <int NKB>
int launch_mlp_fused(const MlpArgs& a, int num_sms, cudaStream_t st) {
  using Cfg = MlpCfg<NKB>;
  auto kern = k_mlp_fused<NKB>;
  static std::atomic<uint64_t> configured{0};
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(kern), Cfg::SMEM_BYTES)) return rc;
  const long long tiles = (a.M + G2_BLOCK_M - 1) / G2_BLOCK_M;
  if (a.M < 1 || tiles > INT_MAX || num_sms < 1) {
    set_error("internal: fused MLP shape M=%lld on %d SMs", a.M, num_sms);
    return SKY_ERR_STATE;
  }
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(a);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

// The same at C = 384 on CTA pairs: W1 at BLOCK_N 64, W2 at BLOCK_N 192 as the two column halves fc2's pair kernel reads.
inline int launch_mlp_fused_pair(const MlpArgs& a, int num_sms, cudaStream_t st) {
  using Cfg = MlpPairCfg;
  static std::atomic<uint64_t> configured{0};
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(k_mlp_fused_pair<6>), Cfg::SMEM_BYTES)) return rc;
  const long long tiles = (a.M + G2_BLOCK_M - 1) / G2_BLOCK_M;
  if (a.M < 1 || tiles > INT_MAX || num_sms < 2) {
    set_error("internal: fused MLP (pair) shape M=%lld on %d SMs", a.M, num_sms);
    return SKY_ERR_STATE;
  }
  const long long pairs = tiles < num_sms / 2 ? tiles : num_sms / 2;
  k_mlp_fused_pair<6><<<(int)(2 * pairs), Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(a);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
