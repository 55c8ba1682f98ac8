// Earth-specific 3-D window attention on the tensor cores (mma.sync m16n8k16, fp16 operands, fp32 accumulation).
//
//     O = softmax(scale * Q K^T + B[type, head] + shift_mask) V      per (window, head); 144 tokens, head_dim 32
//
// Data layout (written by EpiQkvWin, the QKV projection's epilogue, and k_qkv_fill_pad):
//   qkv "window image"  [part q|k|v][member][window][head pair] -> tile of 144 rows x 128 B
//     row j    = position in the (rolled) window, (zj, hj, wj) order
//     128 B    = [head 2p: 32 halves | head 2p+1: 32 halves], 16-byte chunk c stored at c ^ (j & 7)
//   Windowing, the cyclic shift and the latitude padding were applied by the producer, so one work item is three
//   contiguous 18 KB tiles.
//
// One CTA per item (window, head pair), nine warps: warp w owns query rows 16w .. 16w+15 of both heads.  The q, k, v
// tiles and the pair's two compact bias tables are copied to shared memory once; per head the warp computes its 16 x 144
// score block in registers (ldmatrix + mma.sync), adds the bias gathered from the compact table (shift mask folded in,
// in fp16), takes exp2 against the row max, and multiplies P (fp16, straight from the score registers) by V
// (ldmatrix.trans).  1/sum is applied to the 32 outputs of each row, which go to the projection's operand image.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "gemm2.cuh"

namespace sky {

constexpr int AT_TABLE = (2 * WW - 1) * WH * WH * WZ * WZ;   // 3312 entries of the compact bias table per (type, head)
constexpr int AT_TILE_B = WIN_TOK * 128;                     // 18432: one (window, head pair) tile of q, k or v
constexpr int AT_OFF_TAB = 3 * AT_TILE_B;                    // q | k | v tiles, then the two heads' compact tables (fp16)
constexpr int AT_OFF_KEY = AT_OFF_TAB + 2 * AT_TABLE * 2;    // per key: table offset and shift-region flags (int32 each)
constexpr int AT_SMEM_BYTES = AT_OFF_KEY + 2 * WIN_TOK * 4;
constexpr int AT_THREADS = 32 * (WIN_TOK / 16);              // one warp per 16 query rows
static_assert(WIN_TOK % 16 == 0 && (2 * AT_TABLE * 2) % 16 == 0, "tile shapes");

struct AttnArgs {
  const uint8_t* qkv;        // window image, 3 parts
  long long part_stride;     // bytes between the q, k and v parts
  uint8_t* att_img; int att_nkb;   // output: fp16 tile image of (tokens, C) in natural token order
  const __half* bias_tab;    // (n_type, heads, 3312) fp16, pre-scaled by log2 e
  Geo g; int roll; int B; int pairs;
  float sl2;                 // head_dim^-0.5 * log2 e
  float mask_l2;             // mask value * log2 e
  long long items;           // B * nWin * pairs
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// c (16 x 8, fp32) += a (16 x 16, fp16, row-major fragment) * b (16 x 8, fp16, column fragment)
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// shared address of 16-byte chunk c of row j of a window tile (swizzled: chunk c sits at c ^ (j & 7))
__device__ __forceinline__ uint32_t at_chunk(uint32_t tile_s, int j, int c) {
  return tile_s + (uint32_t)j * 128u + ((uint32_t)(c ^ (j & 7)) << 4);
}

// window position (wz, wh, ww, row j) -> natural token of member b, or -1 for a latitude-padding row
__device__ __forceinline__ long long at_row_token(const Geo& g, int roll, int b, int wz, int wh, int ww, int j) {
  const int wj = j % WW, hj = (j / WW) % WH, zj = j / (WW * WH);
  int z = wz * WZ + zj, h = wh * WH + hj, w = ww * WW + wj;
  if (roll) {
    z += SZ; if (z >= g.Z) z -= g.Z;
    h += SH; if (h >= g.Hp) h -= g.Hp;
    w += SW; if (w >= g.W) w -= g.W;
  }
  if (h >= g.H) return -1;
  return (long long)b * g.T + ((long long)z * g.H + h) * g.W + w;
}

// ---------------------------------------------------------------------------------------------------------------
// QKV projection epilogue: accumulator (tokens in natural order) -> fp16 window image.  Re-tiled through the warp's
// swizzled patch exactly like Epi2F16; only the destination address differs: row (window, j) of tile (part, pair).
// A warp store covers 8 token rows x 64 B (one head of each row).
// ---------------------------------------------------------------------------------------------------------------
struct EpiQkvWin {
  static constexpr bool kNeedsBias = false;
  uint8_t* out; long long part_stride; const float* bias; Geo g; int roll; int C; int pairs;
  const float* gamma = nullptr; const float* beta = nullptr;   // unused (uniform epilogue interface)
#ifdef SKY_EXPERIMENTS
  int exp = 0;
#else
  static constexpr int exp = 0;
#endif
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& x) const {
    // this lane's own token row -> index of its 128-byte row inside a part, pair 0 (tile stride = 144 rows); computed once
    // per row group and cached in the context across the n-tiles of the m-tile (the divisions are by run-time values)
    if (x.aux_row0 != x.row0) {
      int myrow = -1;
      const long long row = x.row0 + x.lane;
      if (row < x.M) {
        const unsigned ur = (unsigned)row;             // members * tokens < 2^31
        const unsigned b = ur / (unsigned)g.T, t = ur - b * (unsigned)g.T;
        const unsigned q2 = t / (unsigned)g.W;
        int w = (int)(t - q2 * (unsigned)g.W);
        int z = (int)(q2 / (unsigned)g.H), h = (int)(q2 - (unsigned)z * (unsigned)g.H);
        if (roll) {   // natural -> rolled-grid coordinates
          z -= SZ; if (z < 0) z += g.Z;
          h -= SH; if (h < 0) h += g.Hp;
          w -= SW; if (w < 0) w += g.W;
        }
        const int wz = z / WZ, zj = z % WZ, wh = h / WH, hj = h % WH, ww = w / WW, wj = w % WW;
        const int win = (int)b * g.nWin + (wz * g.nWh + wh) * g.nWw + ww;
        myrow = win * pairs * WIN_TOK + (zj * WH + hj) * WW + wj;     // < 2^31 for members * windows * pairs * 144
      }
      x.aux = myrow;
      x.aux_row0 = x.row0;
    }
    const int myrow = x.aux;
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    for (int c = x.part * 32; c < BN; c += 32 * x.nparts) {
      const int col = x.n0 + c;                       // first of the 32 columns = one head of one part
      const int part = col / C, hd = (col - part * C) >> 5;
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + col + ch * 8));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + col + ch * 8 + 4));
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(x.patch_s, x.lane, v);
      }
      __syncwarp();
      uint8_t* pbase = out + (size_t)part * part_stride + (size_t)(hd >> 1) * AT_TILE_B;
      const uint32_t cpos = (uint32_t)((hd & 1) * 4 + ch);
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + rsub;
        float4 t0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
        float4 t1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
        t0.x += b0.x; t0.y += b0.y; t0.z += b0.z; t0.w += b0.w;
        t1.x += b1.x; t1.y += b1.y; t1.z += b1.z; t1.w += b1.w;
        uint4 pk;
        pk.x = pack_half2(t0.x, t0.y); pk.y = pack_half2(t0.z, t0.w);
        pk.z = pack_half2(t1.x, t1.y); pk.w = pack_half2(t1.z, t1.w);
        const int drow = __shfl_sync(0xffffffffu, myrow, rr);
        if (drow >= 0 && !(exp & 2))
          *reinterpret_cast<uint4*>(pbase + (size_t)drow * 128 + ((cpos ^ ((uint32_t)drow & 7u)) << 4)) = pk;
      }
      __syncwarp();
    }
  }
};

// latitude-padding rows of the window image (tokens with x = 0): q, k, v = the projection's bias
__global__ void __launch_bounds__(256) k_qkv_fill_pad(uint8_t* __restrict__ out, long long part_stride, const float* __restrict__ bias,
                                                      Geo g, int roll, int B, int pairs, int C, long long total) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int chunk = (int)(t & 7); t >>= 3;
  const int pair = (int)(t % pairs); t /= pairs;
  int w = (int)(t % g.W); t /= g.W;
  const int npad = g.Hp - g.H;
  int h = g.H + (int)(t % npad); t /= npad;
  int z = (int)(t % g.Z); t /= g.Z;
  const int b = (int)(t % B); const int part = (int)(t / B);
  if (roll) {
    z -= SZ; if (z < 0) z += g.Z;
    h -= SH; if (h < 0) h += g.Hp;
    w -= SW; if (w < 0) w += g.W;
  }
  const int wz = z / WZ, zj = z % WZ, wh = h / WH, hj = h % WH, ww = w / WW, wj = w % WW;
  const long long win = (long long)b * g.nWin + ((long long)wz * g.nWh + wh) * g.nWw + ww;
  const int j = (zj * WH + hj) * WW + wj;
  const float* bp = bias + part * C + pair * 64 + chunk * 8;
  uint4 pk;
  pk.x = pack_half2(bp[0], bp[1]); pk.y = pack_half2(bp[2], bp[3]);
  pk.z = pack_half2(bp[4], bp[5]); pk.w = pack_half2(bp[6], bp[7]);
  *reinterpret_cast<uint4*>(out + (size_t)part * part_stride + ((size_t)(win * pairs + pair) * WIN_TOK + j) * 128 +
                            (((uint32_t)chunk ^ ((uint32_t)j & 7u)) << 4)) = pk;
}

// ---------------------------------------------------------------------------------------------------------------
// the attention kernel
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AT_THREADS) k_window_attention_tc(const AttnArgs a) {
  extern __shared__ __align__(1024) uint8_t at_smem[];
  const Geo& g = a.g;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // item n = ((type * pairs + pair) * B + b) * nWw + ww
  const long long n = blockIdx.x;
  const long long key = n / ((long long)a.B * g.nWw);
  const int type = (int)(key / a.pairs), pair = (int)(key % a.pairs);
  const int wz = type / g.nWh, wh = type % g.nWh;
  const int ww = (int)(n % g.nWw), b = (int)((n / g.nWw) % a.B);
  const uint8_t* src = a.qkv + ((size_t)(((long long)b * g.nWin + (long long)type * g.nWw + ww) * a.pairs + pair)) * AT_TILE_B;

  // ---- q, k, v tiles and the pair's two compact bias tables -> shared memory ----
  for (int i = tid; i < 3 * AT_TILE_B / 16; i += AT_THREADS) {
    const int part = i / (AT_TILE_B / 16), off = i - part * (AT_TILE_B / 16);
    reinterpret_cast<uint4*>(at_smem)[i] = __ldg(reinterpret_cast<const uint4*>(src + (size_t)part * a.part_stride) + off);
  }
  {
    const uint4* tsrc = reinterpret_cast<const uint4*>(a.bias_tab + ((long long)type * g.heads + 2 * pair) * AT_TABLE);
    for (int i = tid; i < 2 * AT_TABLE * 2 / 16; i += AT_THREADS) reinterpret_cast<uint4*>(at_smem + AT_OFF_TAB)[i] = __ldg(tsrc + i);
  }
  int* kpart = reinterpret_cast<int*>(at_smem + AT_OFF_KEY);
  int* kflag = kpart + WIN_TOK;
  for (int j = tid; j < WIN_TOK; j += AT_THREADS) {
    const int wj = j % WW, hj = (j / WW) % WH, zj = j / (WW * WH);
    kpart[j] = (WZ * zj) * ((2 * WW - 1) * WH * WH) + (WH * hj) * (2 * WW - 1) - wj;
    kflag[j] = (zj >= WZ - SZ ? 1 : 0) | (hj >= WH - SH ? 2 : 0);
  }
  __syncthreads();

  const uint32_t q_s = smem_u32(at_smem), k_s = q_s + AT_TILE_B, v_s = q_s + 2 * AT_TILE_B;
  const __half* tabs = reinterpret_cast<const __half*>(at_smem + AT_OFF_TAB);
  const int fmask = a.roll ? ((wz == g.nWz - 1 ? 1 : 0) | (wh == g.nWh - 1 ? 2 : 0)) : 0;
  const __half mask_h = __float2half_rn(a.mask_l2);
  // this thread's two query rows (fragment rows l/4 and l/4 + 8 of the warp's 16)
  int row[2], rpart[2], rflag[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int i = 16 * warp + (lane >> 2) + 8 * u;
    const int wi = i % WW, hi = (i / WW) % WH, zi = i / (WW * WH);
    row[u] = i;
    rpart[u] = zi * ((2 * WW - 1) * WH * WH) + hi * (2 * WW - 1) + wi + (WW - 1);
    rflag[u] = (zi >= WZ - SZ ? 1 : 0) | (hi >= WH - SH ? 2 : 0);
  }
  const int c2 = 2 * (lane & 3);   // first of this thread's two columns in every 8-column fragment

#pragma unroll 1
  for (int hd = 0; hd < 2; ++hd) {
    // ---- S = Q K^T: 16 rows x 144 keys, K = 32 (two k16 steps = the head's four 16-byte chunks) ----
    uint32_t qa[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      ldsm_x4(at_chunk(q_s, 16 * warp + (lane & 7) + 8 * ((lane >> 3) & 1), hd * 4 + 2 * ks + (lane >> 4)), qa[ks]);
    float s[WIN_TOK / 8][4];
#pragma unroll
    for (int j = 0; j < WIN_TOK / 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
      uint32_t kb[4];   // keys 8j .. 8j+7: dims 0-7 | 8-15 | 16-23 | 24-31
      ldsm_x4(at_chunk(k_s, 8 * j + (lane & 7), hd * 4 + (lane >> 3)), kb);
      mma_16816(s[j], qa[0], kb[0], kb[1]);
      mma_16816(s[j], qa[1], kb[2], kb[3]);
    }
    // ---- scale + bias (+ shift mask), row max ----
    const __half* tab = tabs + hd * AT_TABLE;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < WIN_TOK / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int u = e >> 1, col = 8 * j + c2 + (e & 1);
        __half bh = tab[rpart[u] + kpart[col]];
        if ((rflag[u] ^ kflag[col]) & fmask) bh = __hadd(bh, mask_h);
        s[j][e] = fmaf(s[j][e], a.sl2, __half2float(bh));
        mx[u] = fmaxf(mx[u], s[j][e]);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      mx[u] = fmaxf(mx[u], __shfl_xor_sync(0xffffffffu, mx[u], 1));
      mx[u] = fmaxf(mx[u], __shfl_xor_sync(0xffffffffu, mx[u], 2));
    }
    // ---- P = exp2(s - max) in (0, 1]: fp16 into the tensor core, fp32 row sums ----
    uint32_t p[WIN_TOK / 8][2];
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < WIN_TOK / 8; ++j) {
      const float e0 = mufu_ex2(s[j][0] - mx[0]), e1 = mufu_ex2(s[j][1] - mx[0]);
      const float e2 = mufu_ex2(s[j][2] - mx[1]), e3 = mufu_ex2(s[j][3] - mx[1]);
      sum[0] += e0 + e1; sum[1] += e2 + e3;
      p[j][0] = pack_half2(e0, e1); p[j][1] = pack_half2(e2, e3);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], 1);
      sum[u] += __shfl_xor_sync(0xffffffffu, sum[u], 2);
    }
    // ---- O = P V: K = 144 keys (nine k16 steps), N = 32 dims (four n8 fragments) ----
    float o[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c) o[c][0] = o[c][1] = o[c][2] = o[c][3] = 0.f;
#pragma unroll
    for (int t = 0; t < WIN_TOK / 16; ++t) {
      const uint32_t pa[4] = {p[2 * t][0], p[2 * t][1], p[2 * t + 1][0], p[2 * t + 1][1]};
      uint32_t v0[4], v1[4];   // keys 16t .. 16t+7 | 16t+8 .. 16t+15, dims 8c .. 8c+7 in register c
      ldsm_x4_t(at_chunk(v_s, 16 * t + (lane & 7), hd * 4 + (lane >> 3)), v0);
      ldsm_x4_t(at_chunk(v_s, 16 * t + 8 + (lane & 7), hd * 4 + (lane >> 3)), v1);
#pragma unroll
      for (int c = 0; c < 4; ++c) mma_16816(o[c], pa, v0[c], v1[c]);
    }
    // ---- 1/sum -> fp16 -> 64 bytes of the projection's operand image per row ----
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long tok = at_row_token(g, a.roll, b, wz, wh, ww, row[u]);
      if (tok < 0) continue;
      const float inv = 1.f / sum[u];
      uint8_t* dst = a.att_img + ((size_t)(tok >> 7) * a.att_nkb + pair) * (size_t)G2_A_BYTES + (size_t)(tok & 127) * 128;
      const uint32_t r7 = (uint32_t)tok & 7u;
#pragma unroll
      for (int c = 0; c < 4; ++c)
        *reinterpret_cast<uint32_t*>(dst + ((((uint32_t)(hd * 4 + c)) ^ r7) << 4) + 2 * c2) =
            pack_half2(o[c][2 * u] * inv, o[c][2 * u + 1] * inv);
    }
  }
}

#ifdef SKY_EXPERIMENTS
// CUDA-core reference of the same operator on the same window image (development library, SKY_ATTN=ref): one thread
// per query row, fp32 scores, bias gathered from the compact table.  Bisects "window image / index arithmetic" from
// "tensor pipeline" failures; never benchmarked.
__global__ void __launch_bounds__(WIN_TOK) k_window_attention_ref(const AttnArgs a) {
  const Geo& g = a.g;
  const long long item = blockIdx.x;
  const int hd = blockIdx.y;   // 0 / 1 of the pair
  const long long key = item / (a.B * g.nWw);
  const int type = (int)(key / a.pairs), pair = (int)(key % a.pairs), wz = type / g.nWh, wh = type % g.nWh;
  const int ww = (int)(item % g.nWw), b = (int)((item / g.nWw) % a.B);
  const uint8_t* src = a.qkv + ((size_t)(((long long)b * g.nWin + (long long)type * g.nWw + ww) * a.pairs + pair)) * AT_TILE_B;
  __shared__ float ks[WIN_TOK][33], vs[WIN_TOK][33];
  const int i = threadIdx.x;
  auto elem = [&](int part, int row, int d) {
    const uint32_t c = (uint32_t)(hd * 4 + d / 8);
    return __half2float(*reinterpret_cast<const __half*>(src + (size_t)part * a.part_stride + (size_t)row * 128 + ((c ^ ((uint32_t)row & 7u)) << 4) + (d % 8) * 2));
  };
  float q[32];
  for (int d = 0; d < 32; ++d) { q[d] = elem(0, i, d); ks[i][d] = elem(1, i, d); vs[i][d] = elem(2, i, d); }
  __syncthreads();
  const int fmask = a.roll ? ((wz == g.nWz - 1 ? 1 : 0) | (wh == g.nWh - 1 ? 2 : 0)) : 0;
  const int wi = i % WW, hi = (i / WW) % WH, zi = i / (WW * WH);
  const int rflag = (zi >= WZ - SZ ? 1 : 0) | (hi >= WH - SH ? 2 : 0);
  const __half* tab = a.bias_tab + ((long long)type * g.heads + 2 * pair + hd) * AT_TABLE;
  float sc[WIN_TOK], mx = -INFINITY;
  for (int j = 0; j < WIN_TOK; ++j) {
    float d = 0.f;
    for (int e = 0; e < 32; ++e) d += q[e] * ks[j][e];
    const int wj = j % WW, hj = (j / WW) % WH, zj = j / (WW * WH);
    const int idx = (zi + WZ * zj) * ((2 * WW - 1) * WH * WH) + (hi + WH * hj) * (2 * WW - 1) + wi - wj + WW - 1;
    const int cflag = (zj >= WZ - SZ ? 1 : 0) | (hj >= WH - SH ? 2 : 0);
    d = d * a.sl2 + __half2float(tab[idx]) + (((rflag ^ cflag) & fmask) ? a.mask_l2 : 0.f);
    sc[j] = d; mx = fmaxf(mx, d);
  }
  float sum = 0.f, o[32];
  for (int e = 0; e < 32; ++e) o[e] = 0.f;
  for (int j = 0; j < WIN_TOK; ++j) {
    const float p = exp2f(sc[j] - mx);
    sum += p;
    const float ph = __half2float(__float2half_rn(p));
    for (int e = 0; e < 32; ++e) o[e] += ph * vs[j][e];
  }
  const long long tok = at_row_token(g, a.roll, b, wz, wh, ww, i);
  if (tok < 0) return;
  uint8_t* row = a.att_img + ((size_t)(tok >> 7) * a.att_nkb + pair) * (size_t)G2_A_BYTES + (size_t)(tok & 127) * 128;
  for (int e = 0; e < 32; ++e)
    *reinterpret_cast<__half*>(row + ((((uint32_t)(hd * 4 + e / 8)) ^ ((uint32_t)tok & 7u)) << 4) + (e % 8) * 2) = __float2half_rn(o[e] / sum);
}
#endif

inline int launch_window_attention_tc(const AttnArgs& a, int num_sms, cudaStream_t st) {
  (void)num_sms;
  static std::atomic<uint64_t> configured{0};
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(k_window_attention_tc), AT_SMEM_BYTES)) return rc;
  if (a.items <= 0) return 0;
  k_window_attention_tc<<<(unsigned)a.items, AT_THREADS, AT_SMEM_BYTES, st>>>(a);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
