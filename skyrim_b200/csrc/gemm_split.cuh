// Column-split CTA pairs for GEMMs whose epilogue needs whole rows wider than one CTA's accumulators hold (GraphCast:
// second MLP layer + LayerNorm over 512 columns; Pangu: attention projection + LayerNorm at C = 384):
//
//     D[M, 2 BLOCK_N] = A[M, K] W[2 BLOCK_N, K]^T  ->  epilogue over full rows
//
// A 128 x 512 fp32 accumulator is the whole register file of an SM.  Here the two CTAs of a cluster take the SAME 128-row
// tile and BLOCK_N output columns each (k_gemm2's pipeline: two consumer warpgroups, accumulators staged over the drained
// ring for the epilogue), and the only coupling is the LayerNorm statistics: per lane quarter and tile, 32 (sum, sum of
// squares) pairs cross to the peer through distributed shared memory (st.async completing the peer's mbarrier; gemm2.cuh
// EpiCtx::x_*).  Slots and barriers are double buffered by tile parity; a CTA can run at most one tile ahead of its peer,
// because its next statistics wait needs the peer's sums of that tile.
#pragma once
#include "gemm2.cuh"

namespace sky {

template <class Epi, int EPI_WARPS, int BLOCK_N = 256>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__((EPI_WARPS + 1) * 32, 1)
k_gemm_split(const AImage A, const Epi epi, const uint8_t* __restrict__ Wimg, long long M, int num_kb, int num_m_tiles) {
  using Cfg = G2Cfg<BLOCK_N, EPI_WARPS>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* patches = reinterpret_cast<float*>(smem + Cfg::RING_BYTES);
  float* sbias = patches + EPI_WARPS * G2_PATCH_FLOATS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + 3 * 512);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* stg_free = bars + 2 * Cfg::STAGES;
  uint64_t* xbar = bars + 2 * Cfg::STAGES + 1;                          // [2 tile parities][4 lane quarters]
  float* xstat = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);   // [2][4][32 lanes][2]
  static_assert((2 * Cfg::STAGES + 1 + 8) * 8 <= 256, "barrier block");

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;
  const uint32_t rank = cluster_ctarank();
  const int pair = blockIdx.x >> 1, npairs = gridDim.x >> 1;
  constexpr int LOADER = EPI_WARPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], EPI_WARPS); }
    mbar_init(stg_free, EPI_WARPS);
    for (int i = 0; i < 8; ++i) mbar_init(&xbar[i], 1);
    mbar_fence_init();
  }
  if (threadIdx.x < EPI_WARPS * 32)
    for (int i = threadIdx.x; i < BLOCK_N; i += EPI_WARPS * 32) {
      sbias[i] = epi.bias[rank * BLOCK_N + i]; sbias[512 + i] = epi.gamma[rank * BLOCK_N + i]; sbias[1024 + i] = epi.beta[rank * BLOCK_N + i];
    }
  __syncthreads();
  cluster_sync_all();   // the peer's exchange barriers exist before anything is posted to them

  if (warp == LOADER) {
    int s = 0; uint32_t ph = 0; int it = 0;
    const uint8_t* wsrc = Wimg + (size_t)rank * num_kb * Cfg::B_BYTES;
    for (int mt = pair; mt < num_m_tiles; mt += npairs, ++it) {
      if (it > 0) mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        if (lane == 0) {
          uint8_t* dst = smem + s * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
          bulk_g2s(dst, A.kblock(mt, kb), G2_A_BYTES, &full[s]);
          bulk_g2s(dst + G2_A_BYTES, wsrc + (size_t)kb * Cfg::B_BYTES, Cfg::B_BYTES, &full[s]);
        }
        __syncwarp();
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    const int q = warp & 3, part = warp >> 2, wg = warp >> 2;
    EpiCtx ctx;
    ctx.M = M; ctx.lane = lane; ctx.part = part; ctx.nparts = EPI_WARPS / 4;
    ctx.patch = patches + warp * G2_PATCH_FLOATS;
    ctx.patch_s = smem_u32(ctx.patch);
    ctx.svec_s = smem_u32(sbias);
    ctx.n0 = (int)rank * BLOCK_N;
    WgAcc<BLOCK_N> acc;
    int s = 0; uint32_t ph = 0; int it = 0;
    for (int mt = pair; mt < num_m_tiles; mt += npairs, ++it) {
      const int buf = it & 1;
      const uint32_t use = (uint32_t)(it >> 1);
      ctx.row0 = (long long)mt * G2_BLOCK_M + q * 32;
      ctx.x_own_bar = &xbar[buf * 4 + q];
      ctx.x_own_stat = smem_u32(xstat + (buf * 4 + q) * 64);
      ctx.x_peer_stat = mapa_u32(ctx.x_own_stat, rank ^ 1u);
      ctx.x_peer_bar = mapa_u32(smem_u32(ctx.x_own_bar), rank ^ 1u);
      ctx.x_parity = use & 1;
      epi.template prefetch<BLOCK_N>(ctx);
      wg_mainloop<Cfg::STAGES, Cfg::STAGE_BYTES>(acc, smem, full, empty, s, ph, num_kb, wg, lane);
      wg_epilogue<Cfg::STG_ROWS>(acc, smem, Cfg::STG_LD, wg, warp, lane, [&](AccSmem a) { epi.template run<BLOCK_N>(a, ctx); });
      __syncwarp();
      if (lane == 0) mbar_arrive(stg_free);
    }
  }
  __syncthreads();
  cluster_sync_all();   // nobody leaves while the peer may still post into this CTA's slots
}

// Wimg: [2][K/64][BLOCK_N rows x 128 B] (weight packed with BLOCK_N = half of the row width: 256 for GraphCast's 512-wide
// latents, 192 for Pangu's C = 384 projection)
template <class Epi, int EPI_WARPS, int BLOCK_N = 256>
int launch_gemm_split(const AImage& A, const Epi& epi, const uint8_t* Wimg, long long M, int Kp, int num_sms, cudaStream_t st) {
  using Cfg = G2Cfg<BLOCK_N, EPI_WARPS>;
  constexpr int SMEM = Cfg::SMEM_BYTES + 2048;
  static_assert(SMEM <= 232448, "smem budget");
  auto kern = k_gemm_split<Epi, EPI_WARPS, BLOCK_N>;
  static std::atomic<uint64_t> configured{0};
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(kern), SMEM)) return rc;
  const int num_m_tiles = (int)((M + G2_BLOCK_M - 1) / G2_BLOCK_M);
  const int pairs = num_m_tiles < num_sms / 2 ? num_m_tiles : num_sms / 2;
  kern<<<2 * pairs, Cfg::THREADS, SMEM, st>>>(A, epi, Wimg, M, Kp / 64, num_m_tiles);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
