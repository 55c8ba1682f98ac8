// "Table x data" schedule of the wgmma GEMM k_gemm2 (gemm2.cuh) and its epilogues (SFNO transforms):
//
//   for b in batches:  D_b[M, N] = T_b[M, Ktot] * X_b[Ktot, N]        -> fused epilogue
//
// A = a TABLE (DFT matrix, Legendre table of one zonal wavenumber): K-major tile image packed [hi | lo] along K (read as
//     hi, hi, lo), 128-row tiles (a W3 image with BN = 128), optionally one table per batch.
// B = the DATA, used where it lies: an fp16 tile image whose ROWS are the contraction index (pixels of one latitude,
//     latitudes, degrees l, (m, re/im)) and whose 128-byte row chunks hold 64 consecutive channels.  Those bytes are a
//     valid MN-MAJOR SWIZZLE_128B B operand (atoms of [64 k-rows][128 B] stacked along N with the atom stride in the
//     descriptor's LBO field, sky_common.cuh make_desc_sw128_mn), so no transposing pack pass is needed between two
//     contractions over different indices: each GEMM's epilogue writes its fp16 hi / lo result rows straight into the
//     next GEMM's data image (EpiSplitRemap), K-concatenated as [hi | lo | hi] by reading the hi image twice.
//
// One k-block = 64 data rows x BLOCK_N channels = BLOCK_N/64 atoms of 8 KB; a batch may start at any multiple of 8 rows
// of the image (latitude y of a pixel image starts at row y*W), so a k-block is fetched as one or two bulk copies per atom.
// Rows past the valid K of a batch are read (they belong to the next batch or to zero padding) and multiplied by the
// table's zero K-padding: they must be finite, which every producer of these images guarantees.
#pragma once
#include "gemm_batched.cuh"

namespace sky {

struct BData {
  const uint8_t* hi; const uint8_t* lo;
  int nkb_img;                 // 64-channel column blocks per 128-row tile of the image
  long long rows_per_batch;    // batch b starts at image row b * rows_per_batch (batches inside one image), and / or
  long long batch_bytes;       // at byte offset b * batch_bytes (one image per batch)
};

// Schedule of k_gemm2 (gemm2.cuh) for T_b x X_b.  T: [batches][M/128][hi | lo: 2 x num_kb/3 k-blocks][128 rows x 128 B],
// t_batch_stride bytes apart (0: one table for all batches).
struct SchedTB {
  static constexpr bool kBMN = true;   // B = the data, MN-major
  const uint8_t* T; long long t_batch_stride;
  BData B;
  int num_kb;                          // 3 x the k-blocks of one table segment
  // a batch starts at a multiple of 8 data rows: the MN-major swizzle atom is 8 rows, and the bulk copies of a k-block
  // split at a 128-row tile boundary only on an 8-row boundary
  bool valid() const { return num_kb > 0 && num_kb % 3 == 0 && B.rows_per_batch % 8 == 0; }
  template <int BN>
  __device__ G2Tile tile(const G2Grid& g, int i) const { return G2Tile::at(g, i); }
  template <int BN>
  __device__ __forceinline__ void issue(uint8_t* dst, uint64_t* full, const G2Tile& t, int kb, int lane) const {
    static_assert(BN % 64 == 0 && BN <= 256, "whole 64-channel atoms, one MMA per k-step");
    constexpr int ATOMS = BN / 64;
    const int nkb = num_kb / 3;
    if (lane == 0) {
      const uint8_t* tsrc = T + (size_t)t.b * t_batch_stride + (size_t)t.mt * (2 * nkb) * G2_A_BYTES;   // [hi | lo] image
      mbar_arrive_expect_tx(full, G2_A_BYTES + BN * 128);
      bulk_g2s(dst, tsrc + (size_t)(kb < nkb ? kb : kb - nkb) * G2_A_BYTES, G2_A_BYTES, full);   // hi, hi, lo
    }
    __syncwarp();
    // data rows [r0, r0 + 64) of segment hi | lo | hi; lanes 0 .. ATOMS-1 fetch one 64-channel atom each
    const int seg = kb / nkb;
    const long long r0 = (long long)t.b * B.rows_per_batch + (long long)(kb - seg * nkb) * 64;
    const long long rt = r0 >> 7;
    const uint32_t off = (uint32_t)(r0 & 127);
    const uint32_t rows1 = off <= 64 ? 64u : 128u - off;
    if (lane < ATOMS) {
      const uint8_t* img = (seg == 1 ? B.lo : B.hi) + (size_t)t.b * B.batch_bytes;
      const size_t cb = (size_t)t.nt * ATOMS + lane;
      uint8_t* d = dst + G2_A_BYTES + lane * 8192;
      bulk_g2s(d, img + ((size_t)rt * B.nkb_img + cb) * G2_A_BYTES + off * 128u, rows1 * 128u, full);
      if (rows1 < 64u)
        bulk_g2s(d + rows1 * 128u, img + ((size_t)(rt + 1) * B.nkb_img + cb) * G2_A_BYTES, (64u - rows1) * 128u, full);
    }
  }
};

// acc -> hi / lo fp16 rows of the NEXT contraction's data (or A) image, with the index roles permuted:
//   source element (batch b, row r, column c)  ->  image of batch' = r / bdiv,
//                                                  row'  = b * rb + (c / kdiv),
//                                                  k'    = (r % bdiv) * kmul + (c % kdiv)
// (forward DFT -> Legendre data: bdiv 2, kmul E;  Legendre -> mixing A image and mixing -> inverse Legendre data: a plain
//  batch <-> row swap;  inverse Legendre -> inverse DFT data: kdiv E, rb 2).  Same re-tiling as EpiSplitImg: 16-byte stores.
struct EpiSplitRemap {
  static constexpr bool kNeedsBias = false;
  uint8_t* hi; uint8_t* lo;
  long long img_batch_bytes;   // bytes between destination batch images
  int nkb;                     // 64-wide k-blocks per 128-row tile of a destination image
  int bdiv, kmul, kdiv, rb;
  int n_valid;
  int same = 0;                // 1: no permutation (batch' = b, row' = r, k' = c): the same spectrum laid out for an inverse
  // optional instance-norm affine of the DATA folded behind the (linear) transform:  T (sc x + sh 1) = sc (T x) + sh (T 1):
  // per-column scale / shift and the table's row sums t1[r] (forward DFT: only the m = 0 real row is non-zero)
  const float* csc = nullptr; const float* csh = nullptr; const float* t1 = nullptr;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& x) const {
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    for (int c = x.part * 32; c < BN; c += 32 * x.nparts) {
      const int col = x.n0 + c + ch * 8;
      const bool cols_ok = c + ch * 8 < BN && col < n_valid;
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(x.patch_s, x.lane, v);
      }
      __syncwarp();
      if (cols_ok) {
        const int cq = col / kdiv, cr = col - cq * kdiv;
        float sc[8], sh[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) { sc[e] = 1.f; sh[e] = 0.f; }
        if (csc) {
          const float4 s0 = __ldg(reinterpret_cast<const float4*>(csc + col)), s1 = __ldg(reinterpret_cast<const float4*>(csc + col + 4));
          const float4 h0 = __ldg(reinterpret_cast<const float4*>(csh + col)), h1 = __ldg(reinterpret_cast<const float4*>(csh + col + 4));
          sc[0] = s0.x; sc[1] = s0.y; sc[2] = s0.z; sc[3] = s0.w; sc[4] = s1.x; sc[5] = s1.y; sc[6] = s1.z; sc[7] = s1.w;
          sh[0] = h0.x; sh[1] = h0.y; sh[2] = h0.z; sh[3] = h0.w; sh[4] = h1.x; sh[5] = h1.y; sh[6] = h1.z; sh[7] = h1.w;
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 8 + rsub;
          const long long r = x.row0 + rr;
          if (r < x.M) {
            const float4 q0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
            const float4 q1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
            float f[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
            if (csc) {
              const float tr = __ldg(t1 + r);
#pragma unroll
              for (int e = 0; e < 8; ++e) f[e] = fmaf(f[e], sc[e], sh[e] * tr);
            }
            __half h[8], l[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) { h[e] = __float2half_rn(f[e]); l[e] = __float2half_rn(f[e] - __half2float(h[e])); }
            long long db, drow; int k;
            if (same) { db = x.batch; drow = r; k = col; }
            else { db = r / bdiv; drow = (long long)x.batch * rb + cq; k = (int)(r - db * bdiv) * kmul + cr; }
            const size_t o = (size_t)db * img_batch_bytes + ((size_t)(drow >> 7) * nkb + (size_t)(k >> 6)) * G2_A_BYTES +
                             sw128_offset((uint32_t)(drow & 127), (k & 63) >> 3);
            *reinterpret_cast<uint4*>(hi + o) = *reinterpret_cast<const uint4*>(h);
            *reinterpret_cast<uint4*>(lo + o) = *reinterpret_cast<const uint4*>(l);
          }
        }
      }
      __syncwarp();
    }
  }
};

// y = acc (+ bias[col]) (+ addend[pixel][col]);  g = GELU(y)  ->  hi / lo fp16 rows of the pixel image of g (the next
// pointwise GEMM's A operand) AND per-channel sum / sum of squares of g (instance-norm statistics of the following norm,
// whose affine is folded into that GEMM's weights once the statistics are final).  Replaces: fp32 store of y, a
// statistics pass over it, and the GELU + normalise + split pack pass.  Pixel row = batch * rows_per_batch + row.
struct EpiGeluStatsImg {
  static constexpr bool kNeedsBias = false;
  static constexpr bool kCtaStats = true;   // n_valid <= CTA_STATS_MAX
  uint8_t* hi; uint8_t* lo; int nkb;
  const float* bias;          // per column, may be null
  const float* add; int ld;   // fp32 addend [pixel][ld], may be null
  long long rows_per_batch;
  double* sums;               // [n_valid] sums, then [n_valid] sums of squares
  int n_valid;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& x) const {
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    const long long p0 = (long long)x.batch * rows_per_batch + x.row0;   // pixel row of this warp's first accumulator row
    for (int c = x.part * 32; c < BN; c += 32 * x.nparts) {
      const int col = x.n0 + c + ch * 8;
      const bool cols_ok = c + ch * 8 < BN && col < n_valid;
      float4 a0[4], a1[4];
#pragma unroll
      for (int it = 0; it < 4; ++it) {   // all global reads of the chunk first (see EpiF32Batched)
        const int rr = it * 8 + rsub;
        a0[it] = a1[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (add && cols_ok && x.row0 + rr < x.M) {
          const float* ap = add + (size_t)(p0 + rr) * ld + col;
          a0[it] = __ldg(reinterpret_cast<const float4*>(ap));
          a1[it] = __ldg(reinterpret_cast<const float4*>(ap + 4));
        }
      }
      float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
      if (bias && cols_ok) { b0 = __ldg(reinterpret_cast<const float4*>(bias + col)); b1 = __ldg(reinterpret_cast<const float4*>(bias + col + 4)); }
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(x.patch_s, x.lane, v);
      }
      __syncwarp();
      float s[8], q[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + rsub;
        const float4 t0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
        const float4 t1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
        float f[8] = {t0.x + a0[it].x, t0.y + a0[it].y, t0.z + a0[it].z, t0.w + a0[it].w,
                      t1.x + a1[it].x, t1.y + a1[it].y, t1.z + a1[it].z, t1.w + a1[it].w};
        gelu_erf_x2(f[0], f[1], b0.x, b0.y); gelu_erf_x2(f[2], f[3], b0.z, b0.w);
        gelu_erf_x2(f[4], f[5], b1.x, b1.y); gelu_erf_x2(f[6], f[7], b1.z, b1.w);
        if (cols_ok && x.row0 + rr < x.M) {
          __half h[8], l[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            h[e] = __float2half_rn(f[e]); l[e] = __float2half_rn(f[e] - __half2float(h[e]));
            s[e] += f[e]; q[e] = fmaf(f[e], f[e], q[e]);
          }
          const long long p = p0 + rr;
          const size_t o = ((size_t)(p >> 7) * nkb + (size_t)(col >> 6)) * G2_A_BYTES + sw128_offset((uint32_t)(p & 127), (col & 63) >> 3);
          *reinterpret_cast<uint4*>(hi + o) = *reinterpret_cast<const uint4*>(h);
          *reinterpret_cast<uint4*>(lo + o) = *reinterpret_cast<const uint4*>(l);
        }
      }
      // the 8 lanes that share a column group (same lane & 3) hold 4 rows each: butterfly over lane bits 2..4, then one
      // fp64 atomic per column and statistic from the lanes with rsub == 0
#pragma unroll
      for (int e = 0; e < 8; ++e) {
#pragma unroll
        for (int d = 4; d < 32; d <<= 1) {
          s[e] += __shfl_xor_sync(0xffffffffu, s[e], d);
          q[e] += __shfl_xor_sync(0xffffffffu, q[e], d);
        }
      }
      if (rsub == 0 && cols_ok) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          red_shared_f64(x.svec_s + (uint32_t)(col + e) * 8u, (double)s[e]);
          red_shared_f64(x.svec_s + (uint32_t)(CTA_STATS_MAX + col + e) * 8u, (double)q[e]);
        }
      }
      __syncwarp();
    }
  }
};

// x_out = acc + bias[col] + addend, where addend = asc[col] * add[pixel][col] + ash[col] (the outer skip: norm0 of the block
// input, evaluated on the fly) or plain add[pixel][col] (positional embedding, resampled residual).  Writes the fp32 state
// (the next block's skip source), its hi / lo pixel image (the next block's transform data and inner-skip operand, or the
// decoder's input) and per-channel sum / sum of squares (the next block's norm0) in one pass.  With stat_shift set, the
// statistics are those of x_out - stat_shift[col]: the variance comes from E[d^2] - E[d]^2, which cancels catastrophically
// when |mean| >> std, so the engine passes the bias, which carries a channel's constant offset (k_finalize_norm adds the
// shift back to the mean).
struct EpiF32ImgStats {
  static constexpr bool kNeedsBias = false;
  static constexpr bool kCtaStats = true;   // n_valid <= CTA_STATS_MAX
  float* out; int ld;          // out may be null when nothing reads the fp32 state (the image is always written)
  uint8_t* hi; uint8_t* lo; int nkb;
  const float* bias;
  const float* add; const float* asc; const float* ash;   // add may be null; asc / ash null = plain addend
  double* sums;                                           // may be null (last block: no norm follows)
  int n_valid;
  const float* stat_shift = nullptr;                      // per column, may be null: the statistics are of x_out - shift
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& x) const {
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    for (int c = x.part * 32; c < BN; c += 32 * x.nparts) {
      const int col = x.n0 + c + ch * 8;
      const bool cols_ok = c + ch * 8 < BN && col < n_valid;
      float4 a0[4], a1[4];
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + rsub;
        a0[it] = a1[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (add && cols_ok && x.row0 + rr < x.M) {
          const float* ap = add + (size_t)(x.row0 + rr) * ld + col;
          a0[it] = __ldg(reinterpret_cast<const float4*>(ap));
          a1[it] = __ldg(reinterpret_cast<const float4*>(ap + 4));
        }
      }
      float bb[8], sc[8], sb[8];   // sb: the statistics' shift
#pragma unroll
      for (int e = 0; e < 8; ++e) { bb[e] = 0.f; sc[e] = 1.f; sb[e] = 0.f; }
      if (cols_ok) {
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + col)), b1 = __ldg(reinterpret_cast<const float4*>(bias + col + 4));
        bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w; bb[4] = b1.x; bb[5] = b1.y; bb[6] = b1.z; bb[7] = b1.w;
        if (stat_shift) {
          const float4 t0 = __ldg(reinterpret_cast<const float4*>(stat_shift + col)), t1 = __ldg(reinterpret_cast<const float4*>(stat_shift + col + 4));
          sb[0] = t0.x; sb[1] = t0.y; sb[2] = t0.z; sb[3] = t0.w; sb[4] = t1.x; sb[5] = t1.y; sb[6] = t1.z; sb[7] = t1.w;
        }
        if (asc) {
          const float4 s0 = __ldg(reinterpret_cast<const float4*>(asc + col)), s1 = __ldg(reinterpret_cast<const float4*>(asc + col + 4));
          const float4 h0 = __ldg(reinterpret_cast<const float4*>(ash + col)), h1 = __ldg(reinterpret_cast<const float4*>(ash + col + 4));
          sc[0] = s0.x; sc[1] = s0.y; sc[2] = s0.z; sc[3] = s0.w; sc[4] = s1.x; sc[5] = s1.y; sc[6] = s1.z; sc[7] = s1.w;
          bb[0] += h0.x; bb[1] += h0.y; bb[2] += h0.z; bb[3] += h0.w; bb[4] += h1.x; bb[5] += h1.y; bb[6] += h1.z; bb[7] += h1.w;
        }
      }
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(x.patch_s, x.lane, v);
      }
      __syncwarp();
      float s[8], q[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + rsub;
        const long long p = x.row0 + rr;
        if (cols_ok && p < x.M) {
          const float4 t0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
          const float4 t1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
          const float av[8] = {a0[it].x, a0[it].y, a0[it].z, a0[it].w, a1[it].x, a1[it].y, a1[it].z, a1[it].w};
          float f[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
          __half h[8], l[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            f[e] = f[e] + fmaf(av[e], sc[e], bb[e]);
            h[e] = __float2half_rn(f[e]); l[e] = __float2half_rn(f[e] - __half2float(h[e]));
            const float d = f[e] - sb[e];
            s[e] += d; q[e] = fmaf(d, d, q[e]);
          }
          if (out) {
            float* op = out + (size_t)p * ld + col;
            *reinterpret_cast<float4*>(op) = make_float4(f[0], f[1], f[2], f[3]);
            *reinterpret_cast<float4*>(op + 4) = make_float4(f[4], f[5], f[6], f[7]);
          }
          const size_t o = ((size_t)(p >> 7) * nkb + (size_t)(col >> 6)) * G2_A_BYTES + sw128_offset((uint32_t)(p & 127), (col & 63) >> 3);
          *reinterpret_cast<uint4*>(hi + o) = *reinterpret_cast<const uint4*>(h);
          *reinterpret_cast<uint4*>(lo + o) = *reinterpret_cast<const uint4*>(l);
        }
      }
      if (sums) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
#pragma unroll
          for (int d = 4; d < 32; d <<= 1) {
            s[e] += __shfl_xor_sync(0xffffffffu, s[e], d);
            q[e] += __shfl_xor_sync(0xffffffffu, q[e], d);
          }
        }
        if (rsub == 0 && cols_ok) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            red_shared_f64(x.svec_s + (uint32_t)(col + e) * 8u, (double)s[e]);
            red_shared_f64(x.svec_s + (uint32_t)(CTA_STATS_MAX + col + e) * 8u, (double)q[e]);
          }
        }
      }
      __syncwarp();
    }
  }
};

}  // namespace sky
