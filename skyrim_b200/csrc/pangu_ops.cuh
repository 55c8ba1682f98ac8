// Pangu-Weather step: the token geometry, and the patch embedding's A-operand producers
// (gather + normalise + fp32->fp16) and epilogue.  Both the producer-fed wgmma GEMM
// (gemm_tc.cuh) and the plain reference GEMM (gemm_ref.cuh, test infrastructure on the
// device) are templated on these, so the index arithmetic is written once.  The epilogues
// of the TMA-fed GEMM are in gemm2.cuh and attention_tc.cuh.
//
// Architecture restated from SURVEY.md Appendix A; the reference reaches it through
// /root/reference/skyrim/core/models/pangu.py:45-46.
#pragma once
#include "sky_common.cuh"

namespace sky {

// token grid of one resolution level
struct Geo {
  int Z, H, W, C;
  int Hp;             // H padded to a multiple of the window
  int nWz, nWh, nWw;  // windows along each axis
  int T;              // tokens per member  = Z*H*W
  int nWin;           // windows per member = nWz*nWh*nWw
  int heads;
};
constexpr int WZ = 2, WH = 6, WW = 12, WIN_TOK = WZ * WH * WW;  // 144
constexpr int SZ = WZ / 2, SH = WH / 2, SW = WW / 2;

struct RowInfo {
  long long base;  // element offset of the row's source, or -1 (row contributes zeros)
  int aux;
};

__device__ __forceinline__ uint4 f32x8_to_h8(float4 a, float4 b) {
  uint4 r;
  r.x = pack_half2(a.x, a.y); r.y = pack_half2(a.z, a.w);
  r.z = pack_half2(b.x, b.y); r.w = pack_half2(b.z, b.w);
  return r;
}

// ======================================================================================
// A-operand producers:  prep(row) once per row, load8(info, k) -> 8 halves (k multiple of 8)
// ======================================================================================
// patch embedding, upper-air: row = (member, zt, h, w), k = ((v*2+dz)*4+dh)*4+dw  (K=160)
struct ProdEmbedUpper {
  const float* state;            // (B, nch, nlat, nlon)
  const float* mean; const float* stdv;
  int nlat, nlon, nlev, nvar, nch, H, W, nzt; long long M;
  __device__ RowInfo prep(long long row) const {
    if (row >= M) return {-1, 0};
    int w = (int)(row % W); long long q = row / W;
    int h = (int)(q % H); q /= H;
    int zt = (int)(q % nzt); long long b = q / nzt;
    long long base = (b * nch) * (long long)nlat * nlon + (long long)(4 * h) * nlon + 4 * w;
    return {base, (zt << 16) | h};
  }
  __device__ uint4 load8(const RowInfo& ri, int k) const {
    if (ri.base < 0 || k >= nvar * 32) return make_uint4(0, 0, 0, 0);
    int zt = ri.aux >> 16, h = ri.aux & 0xffff;
    int dh = (k >> 2) & 3, dz = (k >> 4) & 1, v = k >> 5;
    int lev = 2 * zt + dz;
    float4 a = make_float4(0, 0, 0, 0), b = a;
    if (lev < nlev) {
      int ch = v * nlev + lev;
      float mu = __ldg(mean + ch), rs = 1.0f / __ldg(stdv + ch);
      const float* p = state + ri.base + ((long long)ch * nlat + dh) * nlon;
      if (4 * h + dh < nlat) {
        a = __ldg(reinterpret_cast<const float4*>(p));
        a.x = (a.x - mu) * rs; a.y = (a.y - mu) * rs; a.z = (a.z - mu) * rs; a.w = (a.w - mu) * rs;
      }
      if (4 * h + dh + 1 < nlat) {
        b = __ldg(reinterpret_cast<const float4*>(p + nlon));
        b.x = (b.x - mu) * rs; b.y = (b.y - mu) * rs; b.z = (b.z - mu) * rs; b.w = (b.w - mu) * rs;
      }
    }
    return f32x8_to_h8(a, b);
  }
};

// patch embedding, surface: row = (member, h, w), k = (c*4+dh)*4+dw, c<4 state, c>=4 const masks
struct ProdEmbedSurf {
  const float* state; const float* masks;  // masks (3, nlat, nlon)
  const float* mean; const float* stdv;
  int nlat, nlon, nch, ch0, nsurf, nmask, H, W; long long M;
  __device__ RowInfo prep(long long row) const {
    if (row >= M) return {-1, 0};
    int w = (int)(row % W); long long q = row / W;
    int h = (int)(q % H); long long b = q / H;
    return {b, (h << 16) | w};
  }
  __device__ uint4 load8(const RowInfo& ri, int k) const {
    if (ri.base < 0 || k >= (nsurf + nmask) * 16) return make_uint4(0, 0, 0, 0);
    int h = ri.aux >> 16, w = ri.aux & 0xffff;
    int dh = (k >> 2) & 3, c = k >> 4;
    const float* p; float mu = 0.f, rs = 1.f;
    if (c < nsurf) {
      int ch = ch0 + c;
      mu = __ldg(mean + ch); rs = 1.0f / __ldg(stdv + ch);
      p = state + ((ri.base * nch + ch) * (long long)nlat + 4 * h + dh) * nlon + 4 * w;
    } else {
      p = masks + ((long long)(c - nsurf) * nlat + 4 * h + dh) * nlon + 4 * w;
    }
    float4 a = make_float4(0, 0, 0, 0), b = a;
    if (4 * h + dh < nlat) {
      a = __ldg(reinterpret_cast<const float4*>(p));
      a.x = (a.x - mu) * rs; a.y = (a.y - mu) * rs; a.z = (a.z - mu) * rs; a.w = (a.w - mu) * rs;
    }
    if (4 * h + dh + 1 < nlat) {
      b = __ldg(reinterpret_cast<const float4*>(p + nlon));
      b.x = (b.x - mu) * rs; b.y = (b.y - mu) * rs; b.z = (b.z - mu) * rs; b.w = (b.w - mu) * rs;
    }
    return f32x8_to_h8(a, b);
  }
};

// ======================================================================================
// Epilogues.  Model: one lane owns one accumulator row; `acc.load32(col, v)` is a
// warp-collective read of 32 consecutive columns of the lane's row (staged accumulator or scratch).
// `row` may be >= M (tail tile): loads still execute, stores are predicated off.
// n0 = first column of this tile in the full N, BN = tile width.
// ======================================================================================

// out_f32[dstrow, n0+col] = acc + bias  (+ the fp16 tile image of the same rows)   (patch embedding)
struct EpiStoreF32 {
  float* out; int ldo; const float* bias;  // bias may be null
  long long M;
  // dst row = member*T + zoff*HW + (row % rows_per_member); identity when rows_per_member==0
  int T; int HW; int zoff; long long rows_per_member;
  uint8_t* img; int nkb;  // optional fp16 image (SWIZZLE_128B tiles of 128 rows x 64 cols)
  template <class Acc>
  __device__ void run(Acc& acc, long long row, int n0, int BN) const {
    long long dst = row;
    if (rows_per_member > 0) dst = (row / rows_per_member) * T + (long long)zoff * HW + row % rows_per_member;
    for (int c = 0; c < BN; c += 32) {
      float v[32];
      acc.load32(c, v);
      if (row < M) {
        if (bias) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + n0 + c) + j);
            v[4 * j] += bb.x; v[4 * j + 1] += bb.y; v[4 * j + 2] += bb.z; v[4 * j + 3] += bb.w;
          }
        }
        // the lane owns its row: 256-bit stores, one full 32-byte sector per lane and instruction
        if (out) {   // null with the image-only token stream: nothing reads the fp32 rows
          float* o = out + dst * ldo + n0 + c;
#pragma unroll
          for (int j = 0; j < 4; ++j) stg_f32x8(o + 8 * j, v + 8 * j);
        }
        if (img) {
          const int col = n0 + c;
          uint8_t* base = img + ((size_t)(dst >> 7) * nkb + (col >> 6)) * 16384 + (size_t)(dst & 127) * 128;
          const uint32_t r7 = (uint32_t)dst & 7u, cb = ((uint32_t)col & 63u) >> 3;   // cb = 0 or 4
          // SWIZZLE_128B permutes 16-byte chunks by XOR with (row & 7): an aligned chunk pair stays an aligned pair
          // (halves swapped when bit 0 of the row is set), so two chunks go out as one 32-byte store
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            uint4 c0, c1;
            c0.x = pack_half2(v[16 * m], v[16 * m + 1]); c0.y = pack_half2(v[16 * m + 2], v[16 * m + 3]);
            c0.z = pack_half2(v[16 * m + 4], v[16 * m + 5]); c0.w = pack_half2(v[16 * m + 6], v[16 * m + 7]);
            c1.x = pack_half2(v[16 * m + 8], v[16 * m + 9]); c1.y = pack_half2(v[16 * m + 10], v[16 * m + 11]);
            c1.z = pack_half2(v[16 * m + 12], v[16 * m + 13]); c1.w = pack_half2(v[16 * m + 14], v[16 * m + 15]);
            const uint32_t pr = ((cb >> 1) + m) ^ (r7 >> 1);
            if (r7 & 1u) stg_b32x8(base + pr * 32, c1, c0); else stg_b32x8(base + pr * 32, c0, c1);
          }
        }
      }
    }
  }
};

}  // namespace sky
