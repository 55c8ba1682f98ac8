// Persistent warp-specialised wgmma GEMM for sm_90a:
//
//      D[M, N] = A(prod)[M, K] * W[N, K]^T  ->  epilogue(epi)
//
//   * A operand: gathered / normalised / converted fp32->fp16 by four producer warps
//     straight into a SWIZZLE_128B K-major smem tile (no intermediate HBM copy of the
//     windowed / im2col'd activations ever exists);
//   * B operand: weights pre-packed at load time as the exact smem tile image
//     (k_pack_weight), fetched with one 1-D bulk copy (TMA engine, cp.async.bulk +
//     mbarrier complete_tx) per k-block;
//   * two consumer warpgroups issue the wgmma products (gemm2.cuh WgAcc) and stage the
//     accumulator in shared memory; warps 0..3 then run the row-owner epilogue on it.
#pragma once
#include "gemm2.cuh"

namespace sky {

constexpr int TC_BLOCK_M = 128;
constexpr int TC_BLOCK_K = 64;                      // halves: one 128-byte swizzle row
constexpr int TC_A_BYTES = TC_BLOCK_M * 128;        // 16 KB
constexpr int TC_THREADS = 416;                     // 8 consumer + 4 producer + B-loader warps
constexpr int TC_NUM_PRODUCER_THREADS = 128;

template <int BLOCK_N>
struct TcCfg {
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES;
  static constexpr int STAGES = (200 * 1024) / STAGE_BYTES >= 6 ? 6 : (200 * 1024) / STAGE_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int STG_LD = (BLOCK_N + 31) / 32 * 32 + 4;
  static constexpr int SMEM_BYTES = RING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(BLOCK_N % 32 == 0 && BLOCK_N <= 256, "wgmma N");
  static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
  static_assert(128 * STG_LD * 4 <= RING_BYTES, "accumulator staging");
};

template <class Prod, class Epi, int BLOCK_N>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_gemm_tc(const Prod prod, const Epi epi, const uint8_t* __restrict__ Wimg, long long M,
          int num_kb, int num_m_tiles, int num_n_tiles) {
  using Cfg = TcCfg<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::RING_BYTES);
  uint64_t* full = bars;                       // [STAGES]  producers(128) + B loader(1 + tx)
  uint64_t* empty = bars + Cfg::STAGES;        // [STAGES]  the 8 consumer warps
  uint64_t* stg_free = bars + 2 * Cfg::STAGES; // consumers -> producers / B loader: the epilogue has left the ring

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;  // provably warp-uniform
  const int num_tiles = num_m_tiles * num_n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full[s], TC_NUM_PRODUCER_THREADS + 1);
      mbar_init(&empty[s], 8);
    }
    mbar_init(stg_free, 8);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 8 && warp < 12) {
    // ============================ A producers ============================
    // thread = tile row, the 8 chunks of a k-block in sequence: for one chunk the 32 lanes of a warp are 32
    // consecutive tokens, i.e. one contiguous 512-byte run of the source field per load instruction, and the
    // 16-byte shared-memory stores of a quarter warp fall into 8 different swizzled chunk slots
    const int row = threadIdx.x - 256;
    int s = 0; uint32_t ph = 0; int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const long long m0 = (long long)(tile / num_n_tiles) * TC_BLOCK_M;
      const RowInfo ri = prod.prep(m0 + row);
      if (it > 0) mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* a_s = smem + s * Cfg::STAGE_BYTES;
        uint4 v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = prod.load8(ri, kb * TC_BLOCK_K + i * 8);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<uint4*>(a_s + sw128_offset(row, i)) = v[i];
        fence_proxy_async_smem();
        mbar_arrive(&full[s]);
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp == 12) {
    // ============================ B loader (TMA engine) ============================
    int s = 0; uint32_t ph = 0; int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int nt = tile % num_n_tiles;
      const uint8_t* src = Wimg + (size_t)nt * num_kb * Cfg::B_BYTES;
      if (it > 0) mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        if (lane == 0) {
          mbar_arrive_expect_tx(&full[s], Cfg::B_BYTES);
          bulk_g2s(smem + s * Cfg::STAGE_BYTES + TC_A_BYTES, src + (size_t)kb * Cfg::B_BYTES, Cfg::B_BYTES,
                   &full[s]);
        }
        __syncwarp();
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // ============================ consumer warpgroups: MMA, then epilogue in warps 0..3 ============================
    const int wg = warp >> 2;
    WgAcc<BLOCK_N> acc;
    int s = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const long long m0 = (long long)(tile / num_n_tiles) * TC_BLOCK_M;
      const int n0 = (tile % num_n_tiles) * BLOCK_N;
      wg_mainloop<Cfg::STAGES, Cfg::STAGE_BYTES>(acc, smem, full, empty, s, ph, num_kb, wg, lane);
      wg_epilogue(acc, smem, Cfg::STG_LD, wg, warp, lane, [&](AccSmem a) {
        if (warp < 4) epi.run(a, m0 + warp * 32 + lane, n0, BLOCK_N);
      });
      __syncwarp();
      if (lane == 0) mbar_arrive(stg_free);
    }
  }
}

template <class Prod, class Epi, int BLOCK_N>
int launch_gemm_tc(const Prod& prod, const Epi& epi, const uint8_t* Wimg, long long M, int N, int Kp,
                   int num_sms, cudaStream_t st) {
  using Cfg = TcCfg<BLOCK_N>;
  auto kern = k_gemm_tc<Prod, Epi, BLOCK_N>;
  static std::atomic<uint64_t> configured{0};   // one bit per device: the attribute is per (function, device)
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(kern), Cfg::SMEM_BYTES)) return rc;
  const int num_m_tiles = (int)((M + TC_BLOCK_M - 1) / TC_BLOCK_M);
  const int num_n_tiles = N / BLOCK_N;
  const int tiles = num_m_tiles * num_n_tiles;
  const int grid = tiles < num_sms ? tiles : num_sms;
  kern<<<grid, TC_THREADS, Cfg::SMEM_BYTES, st>>>(prod, epi, Wimg, M, Kp / TC_BLOCK_K, num_m_tiles, num_n_tiles);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
