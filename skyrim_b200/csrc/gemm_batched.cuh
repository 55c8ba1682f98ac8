// Epilogues of the batched SFNO GEMMs (k_gemm2 with SchedW over batches, gemm2.cuh):
//
//   for b in batches:  D_b[M, N] = A_b[M, Ktot] * W_b[N, Ktot]^T      -> fused epilogue
//
// A is the 3-term fp16 split (a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo, DESIGN.md §2): A = [hi | lo | hi] (the same
// image twice), W = one image packed as [hi | lo], read as hi, hi, lo.  Every batch has its own A and W images at fixed
// byte strides (Legendre transforms: one per zonal wavenumber m; the spectral channel mixing: one per degree l).
#pragma once
#include "gemm2.cuh"

namespace sky {

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
  __device__ void run(Acc& acc, const EpiCtx& e) const {
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
  __device__ void run(Acc& acc, const EpiCtx& e) const {
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
  __device__ void run(Acc& acc, const EpiCtx& x) const {
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
