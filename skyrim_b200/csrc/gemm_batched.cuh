// Batched, K-segmented variant of the TMA-fed wgmma GEMM (gemm2.cuh), used by the SFNO path:
//
//   for b in batches:  D_b[M, N] = A_b[M, Ktot] * W_b[N, Ktot]^T      -> fused epilogue
//
// The A operand is a concatenation along K of up to 6 image segments, which is how the
// 3-term fp16 split (a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo, DESIGN.md §2) and the decoder's
// concat(x, input) are expressed without touching the kernel: A = [hi | lo | hi] (the same
// image twice), W = one image packed as [hi | hi | lo].  Every batch has its own A and W
// images at fixed byte strides (Legendre transforms: one per zonal wavenumber m; the spectral
// channel mixing: one per degree l).
#pragma once
#include <type_traits>
#include "gemm2.cuh"

namespace sky {

struct AOperand {
  const uint8_t* seg[6];
  int nkb[6];                 // k-blocks of each segment
  long long batch_stride[6];  // bytes between batches of each segment
  int nseg;
  int m_tiles_per_batch;      // row tiles of one batch inside a segment image
  int tri = 0;                // 1: batch b only has rows 0 .. b (degree l of a spectrum holds orders m <= l): row tiles that
                              // start past row b are skipped by every role (their output is multiplied by zeros downstream)
  __device__ const uint8_t* kblock(int batch, int mt, int kb) const {
#pragma unroll
    for (int s = 0; s < 6; ++s) {
      if (s < nseg) {
        if (kb < nkb[s]) return seg[s] + (size_t)batch * batch_stride[s] + ((size_t)mt * nkb[s] + kb) * G2_A_BYTES;
        kb -= nkb[s];
      }
    }
    return seg[0];
  }
};

struct EpiCtxB : EpiCtx {
  int batch;
};

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

template <class Epi, int BLOCK_N, int EPI_WARPS>
__global__ void __launch_bounds__((EPI_WARPS + 1) * 32, 1)
k_gemm_batched(const AOperand A, const Epi epi, const uint8_t* __restrict__ Wimg, long long w_batch_stride,
               long long M, int num_kb, int num_m_tiles, int num_n_tiles, int batches) {
  using Cfg = G2Cfg<BLOCK_N, EPI_WARPS>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* patches = reinterpret_cast<float*>(smem + Cfg::RING_BYTES);
  float* sbias = patches + EPI_WARPS * G2_PATCH_FLOATS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + 3 * 512);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* stg_free = bars + 2 * Cfg::STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x / 32, 0), lane = threadIdx.x % 32;
  const int tiles_per_batch = num_m_tiles * num_n_tiles;
  const long long num_tiles = (long long)tiles_per_batch * batches;
  constexpr int LOADER = EPI_WARPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], EPI_WARPS); }
    mbar_init(stg_free, EPI_WARPS);
    mbar_fence_init();
  }
  if constexpr (has_cta_stats<Epi>::value)
    for (int i = threadIdx.x; i < 3 * 512; i += blockDim.x) sbias[i] = 0.f;
  __syncthreads();

  if (warp == LOADER) {
    int s = 0; uint32_t ph = 0; int it = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int b = (int)(tile / tiles_per_batch), t = (int)(tile % tiles_per_batch);
      const int mt = t / num_n_tiles, nt = t % num_n_tiles;
      if (A.tri && mt * G2_BLOCK_M > b) continue;
      if (it > 0) mbar_wait(stg_free, (uint32_t)(it - 1) & 1);
      ++it;
      // W image = [hi | lo] (nkw k-blocks each), consumed as hi, hi, lo against A = hi, lo, hi
      const int nkw = num_kb / 3;
      const uint8_t* wsrc = Wimg + (size_t)b * w_batch_stride + (size_t)nt * (2 * nkw) * Cfg::B_BYTES;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        if (lane == 0) {
          uint8_t* dst = smem + s * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
          bulk_g2s(dst, A.kblock(b, mt, kb), G2_A_BYTES, &full[s]);
          bulk_g2s(dst + G2_A_BYTES, wsrc + (size_t)(kb < nkw ? kb : kb - nkw) * Cfg::B_BYTES, Cfg::B_BYTES, &full[s]);
        }
        __syncwarp();
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    const int q = warp & 3, part = warp >> 2, wg = warp >> 2;
    EpiCtxB ctx;
    ctx.M = M; ctx.lane = lane; ctx.part = part; ctx.nparts = EPI_WARPS / 4;
    ctx.patch = patches + warp * G2_PATCH_FLOATS;
    ctx.patch_s = smem_u32(ctx.patch);
    ctx.svec_s = smem_u32(sbias);
    WgAcc<BLOCK_N> acc;
    int s = 0; uint32_t ph = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int b = (int)(tile / tiles_per_batch), t = (int)(tile % tiles_per_batch);
      if (A.tri && (t / num_n_tiles) * G2_BLOCK_M > b) continue;
      ctx.batch = b;
      ctx.row0 = (long long)(t / num_n_tiles) * G2_BLOCK_M + q * 32;
      ctx.n0 = (t % num_n_tiles) * BLOCK_N;
      wg_mainloop<Cfg::STAGES, Cfg::STAGE_BYTES>(acc, smem, full, empty, s, ph, num_kb, wg, lane);
      wg_epilogue<Cfg::STG_ROWS>(acc, smem, Cfg::STG_LD, wg, warp, lane, [&](AccSmem a) { epi.template run<BLOCK_N>(a, ctx); });
      __syncwarp();
      if (lane == 0) mbar_arrive(stg_free);
    }
  }
  __syncthreads();
  cta_stats_flush(epi, sbias);
}

template <class Epi, int BLOCK_N, int EPI_WARPS>
int launch_gemm_batched(const AOperand& A, const Epi& epi, const uint8_t* Wimg, long long w_batch_stride, long long M,
                        int N, int Ktot, int batches, int num_sms, cudaStream_t st) {
  using Cfg = G2Cfg<BLOCK_N, EPI_WARPS>;
  auto kern = k_gemm_batched<Epi, BLOCK_N, EPI_WARPS>;
  static std::atomic<uint64_t> configured{0};   // one bit per device: the attribute is per (function, device)
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(kern), Cfg::SMEM_BYTES)) return rc;
  const int num_m_tiles = (int)((M + G2_BLOCK_M - 1) / G2_BLOCK_M);
  const int num_n_tiles = N / BLOCK_N;
  const long long tiles = (long long)num_m_tiles * num_n_tiles * batches;
  const int grid = (int)(tiles < num_sms ? tiles : num_sms);
  kern<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(A, epi, Wimg, w_batch_stride, M, Ktot / 64, num_m_tiles, num_n_tiles,
                                                   batches);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

// out[batch][row, n0+col] (=|+=) acc (+ bias[col]) — fp32 row-major, 128-bit accesses on full
// row segments (same re-tiling as Epi2F32Img).  kAccumulate adds to what the buffer holds
// (pre-filled by the caller with a residual / positional / spectral term).
template <bool kAccumulate>
struct EpiF32Batched {
  static constexpr bool kNeedsBias = false;
  float* out; int ldo; long long batch_stride /*floats*/; const float* bias /*may be null*/;
  int n_valid;  // columns >= n_valid are padding and are not stored
  const float* add = nullptr;   // optional addend with the layout of `out` (residual / positional term): out = acc + bias + add
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtxB& e) const {
    const int rsub4 = e.lane >> 3, c4 = e.lane & 7;
    const int step = 32 * e.nparts;
    const long long rows_left = e.M - e.row0;
    float* xp = out + (size_t)e.batch * batch_stride + e.row0 * ldo + e.n0 + c4 * 4;
    const float* ap = add ? add + (size_t)e.batch * batch_stride + e.row0 * ldo + e.n0 + c4 * 4 : nullptr;
    for (int c = e.part * 32; c < BN; c += step) {
      const int col = e.n0 + c + c4 * 4;
      // BN need not be a multiple of 32 (16, 80, 240): the 32-column accumulator read then runs past the tile; those columns
      // belong to the NEXT n-tile (another CTA's work) and must not be stored from here (round-1 bug: they were, and
      // raced with the owner's store whenever N had more than one such tile, e.g. nlon = 1440 or lmax = 240)
      const bool act = col < n_valid && c + c4 * 4 < BN;
      // all global reads of the chunk (previous value / addend) are issued before the accumulator fetch: written as
      // load -> add -> store per row they serialise into 8 DRAM round trips per chunk, because the compiler may not move
      // a load above the preceding store to `out` (ncu r2a: 82 % long-scoreboard stalls, 33 k cycles per 128x192 tile
      // against 7 k of MMA time)
      float4 o[8];
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        o[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (act && rr < rows_left) {
          if (kAccumulate) o[it] = *reinterpret_cast<const float4*>(xp + (size_t)rr * ldo + c);
          if (ap) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(ap + (size_t)rr * ldo + c));
            o[it].x += a.x; o[it].y += a.y; o[it].z += a.z; o[it].w += a.w;
          }
        }
      }
      float v[32];
      acc.load32(c, v);
      patch_put_s(e.patch_s, e.lane, v);
      __syncwarp();
      if (act) {
        float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (bias) b = __ldg(reinterpret_cast<const float4*>(bias + col));
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int rr = it * 4 + rsub4;
          if (rr < rows_left) {
            const uint32_t pa = e.patch_s + (rr * G2_PATCH_LD + c4 * 4) * 4;
            const float4 y = make_float4(lds_f32(pa) + b.x + o[it].x, lds_f32(pa + 4) + b.y + o[it].y,
                                         lds_f32(pa + 8) + b.z + o[it].z, lds_f32(pa + 12) + b.w + o[it].w);
            *reinterpret_cast<float4*>(xp + (size_t)rr * ldo + c) = y;
          }
        }
      }
      __syncwarp();
    }
  }
};

// Inverse longitude DFT: rows = (lat, c) with c fastest (E channels, E % 32 == 0), columns = lon.  Stores the result
// PIXEL-MAJOR, out[(lat * W + lon) * E + c], straight from the accumulator registers: lane = row = channel c0 + lane, so for
// every column (longitude) the warp's 32 lanes hold 32 consecutive channels of ONE pixel = one 128-byte store.
// Replaces the fp32 [(lat, c)][lon] buffer and the k_transpose pass that used to follow this GEMM.
struct EpiF32PixelMajor {
  static constexpr bool kNeedsBias = false;
  float* out; int E; int W; int n_valid;
  const float* chan_bias = nullptr;   // optional per-channel constant (the folded inner skip's bias)
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtxB& e) const {
    const long long r0 = e.row0;                       // 32-aligned and E % 32 == 0: the 32 rows share their latitude
    const bool ok = r0 < e.M;
    const long long lat = r0 / E;
    const int c0 = (int)(r0 - lat * E);
    float* obase = out + (size_t)lat * W * E + c0 + e.lane;
    const float cb = (chan_bias && ok) ? __ldg(chan_bias + c0 + e.lane) : 0.f;
    for (int c = e.part * 32; c < BN; c += 32 * e.nparts) {
      float v[32];
      acc.load32(c, v);
      if (!ok) continue;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int lon = e.n0 + c + j;
        if (lon < n_valid && c + j < BN) obase[(size_t)lon * E] = v[j] + cb;
      }
    }
  }
};

// acc (+ bias, optional GELU) -> hi / lo fp16 operand images of the NEXT GEMM (K = this GEMM's N): the 3-term split is
// produced where the value is produced, instead of an fp32 round trip through HBM and a separate pack pass.
// Same re-tiling as Epi2F16<.., kImage = true>: lane -> (row = it*8 + lane/4, 8-column chunk = lane%4), 16-byte stores.
template <bool kGelu>
struct EpiSplitImg {
  static constexpr bool kNeedsBias = false;
  uint8_t* hi; uint8_t* lo; int nkb;   // k-blocks per row tile of the destination images
  const float* bias; int n_valid;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtxB& x) const {
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    const uint32_t r0 = (uint32_t)(x.row0 & 127);
    for (int c = x.part * 32; c < BN; c += 32 * x.nparts) {
      const int col = x.n0 + c + ch * 8;                       // first of this lane's 8 columns
      const bool cols_ok = c + ch * 8 < BN && col < n_valid;   // BN need not be a multiple of 32
      float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
      if (!kGelu && cols_ok) { b0 = __ldg(reinterpret_cast<const float4*>(bias + col)); b1 = __ldg(reinterpret_cast<const float4*>(bias + col + 4)); }
      {
        float v[32];
        acc.load32(c, v);
        if (kGelu) {   // activation in the row domain: 32 independent chains per thread
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int cj = x.n0 + c + 4 * j;
            const float4 b = cj < n_valid ? __ldg(reinterpret_cast<const float4*>(bias + cj)) : make_float4(0.f, 0.f, 0.f, 0.f);
            gelu_erf_x2(v[4 * j], v[4 * j + 1], b.x, b.y);
            gelu_erf_x2(v[4 * j + 2], v[4 * j + 3], b.z, b.w);
          }
        }
        patch_put_v(x.patch_s, x.lane, v);
      }
      __syncwarp();
      const size_t tbase = ((size_t)(x.row0 >> 7) * nkb + (size_t)((x.n0 + c) >> 6)) * (size_t)G2_A_BYTES + (size_t)r0 * 128;
      const uint32_t cb = (((uint32_t)(x.n0 + c) & 63u) >> 3) + (uint32_t)ch;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + rsub;
        float4 t0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
        float4 t1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
        if (!kGelu) {
          t0.x += b0.x; t0.y += b0.y; t0.z += b0.z; t0.w += b0.w;
          t1.x += b1.x; t1.y += b1.y; t1.z += b1.z; t1.w += b1.w;
        }
        const float f[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
        __half h[8], l[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) { h[e] = __float2half_rn(f[e]); l[e] = __float2half_rn(f[e] - __half2float(h[e])); }
        if (cols_ok && x.row0 + rr < x.M) {
          const size_t off = tbase + (size_t)rr * 128 + ((cb ^ (uint32_t)((r0 + rr) & 7)) << 4);
          *reinterpret_cast<uint4*>(hi + off) = *reinterpret_cast<const uint4*>(h);
          *reinterpret_cast<uint4*>(lo + off) = *reinterpret_cast<const uint4*>(l);
        }
      }
      __syncwarp();
    }
  }
};

}  // namespace sky
