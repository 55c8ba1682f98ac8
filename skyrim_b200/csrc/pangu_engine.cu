// Pangu-Weather 6-h step operator on sm_90a: weight repacking + the per-step kernel
// sequence.  Replaces the two ONNX Runtime sessions that Skyrim's Pangu model
// (skyrim/core/models/pangu.py) loads and steps.
//
// Data flow (v2): every token matrix lives in NATURAL token order (member, z, lat, lon).
//   x   fp32 row-major (rows, C)                  the residual stream
//   xh  fp16 "tile image" [rows/128][C/64][128x128B SWIZZLE_128B]   = the A operand of the next
//       GEMM, written by the epilogue that produced x and fetched by 1-D bulk copies
// Windowing / cyclic shift / padding exist only as index arithmetic inside the attention kernel.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "attention_tc.cuh"
#include "engine.h"
#include "gemm2.cuh"
#include "mlp_fused.cuh"
#include "pangu_ops.cuh"

namespace sky {

// ======================================================================================
// weight repacking (runs once, at load)
// ======================================================================================
// fp32 W (logical [Nsrc, K]; stored [Nsrc,K] or, if transposed, [K,Nsrc]) -> rows
// [n_off, n_off+Nsrc) of the fp16 tile image [Ntot/BN][Kp/64][BN rows x 128 B, SWIZZLE_128B]
__global__ void k_pack_weight(const float* __restrict__ W, int Nsrc, int K, int Kp, int BN, int transposed,
                              int n_off, uint8_t* __restrict__ img) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one 8-half chunk each
  int chunks_per_row = Kp / 8;
  if (idx >= (long long)Nsrc * chunks_per_row) return;
  int ns = (int)(idx / chunks_per_row), kc = (int)(idx % chunks_per_row);
  __half h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    int k = kc * 8 + e;
    float v = 0.f;
    if (k < K) v = transposed ? W[(long long)k * Nsrc + ns] : W[(long long)ns * K + k];
    h[e] = __float2half_rn(v);
  }
  uint4 pk = *reinterpret_cast<uint4*>(h);
  const int n = n_off + ns;
  int nt = n / BN, nr = n % BN, kb = kc / 8, ch = kc % 8;
  size_t tile = ((size_t)nt * (Kp / 64) + kb) * (size_t)BN * 128;
  *reinterpret_cast<uint4*>(img + tile + sw128_offset(nr, ch)) = pk;
}

// earth-specific bias (3312, n_type, heads) -> (n_type, heads, 3312), pre-scaled by log2(e)
// (the attention kernel computes its softmax with exp2)
__global__ void k_pack_bias_table(const float* __restrict__ src, __half* __restrict__ dst, int L, int n_type,
                                  int heads) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long tot = (long long)L * n_type * heads;
  if (idx >= tot) return;
  int l = (int)(idx % L);
  long long th = idx / L;  // type*heads + head
  dst[idx] = __float2half_rn(src[(long long)l * n_type * heads + th] * 1.4426950408889634f);
}

int launch_pack_bias_table(const float* src, __half* dst, int n_type, int heads, cudaStream_t st) {
  const long long tot = (long long)AT_TABLE * n_type * heads;
  if (tot <= 0) return 0;
  k_pack_bias_table<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(src, dst, AT_TABLE, n_type, heads);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

// ======================================================================================
// window image fill and window attention (layout, AttnArgs and EpiQkvWin: attention_tc.cuh)
// ======================================================================================
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

int launch_qkv_fill_pad(uint8_t* out, long long part_stride, const float* bias, const Geo& g, int roll, int B, int pairs,
                        cudaStream_t st) {
  const long long total = 3LL * B * g.Z * (g.Hp - g.H) * g.W * pairs * 8;
  if (total <= 0) return 0;
  k_qkv_fill_pad<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(out, part_stride, bias, g, roll, B, pairs, g.C, total);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// the attention kernel (work split, warp roles and shared-memory layout: attention_tc.cuh)
// ---------------------------------------------------------------------------------------------------------------
// item n = ((type * pairs + pair) * B + b) * nWw + ww; a CTA decodes its first item and steps through the rest
struct AtItem {
  int type, pair, b, ww;
  __device__ AtItem(const AttnArgs& a, long long n) {
    const long long key = n / ((long long)a.B * a.g.nWw);
    type = (int)(key / a.pairs); pair = (int)(key % a.pairs); b = (int)((n / a.g.nWw) % a.B); ww = (int)(n % a.g.nWw);
  }
  __device__ void next(const AttnArgs& a) {
    if (++ww < a.g.nWw) return;
    ww = 0;
    if (++b < a.B) return;
    b = 0;
    if (++pair < a.pairs) return;
    pair = 0; ++type;
  }
};

__global__ void __launch_bounds__(AT_THREADS, 1) k_window_attention_tc(const AttnArgs a) {
  extern __shared__ __align__(1024) uint8_t at_smem[];
  const Geo& g = a.g;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* full = reinterpret_cast<uint64_t*>(at_smem + AT_OFF_BAR);
  uint64_t* empty = full + AT_STAGES;
  if (threadIdx.x == 0) {
    for (int s = 0; s < AT_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], AT_WARPS); }
    mbar_fence_init();
  }
  __syncthreads();
  const long long n0 = a.items * blockIdx.x / gridDim.x, n1 = a.items * (blockIdx.x + 1) / gridDim.x;

  if (warp == AT_WARPS) {   // ---- producer: the q, k, v tiles of each item -> ring slot ----
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      AtItem it(a, n0);
      for (long long n = n0; n < n1; ++n, it.next(a)) {
        const uint8_t* src =
            a.qkv + (size_t)(((long long)it.b * g.nWin + (long long)it.type * g.nWw + it.ww) * a.pairs + it.pair) * AT_TILE_B;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], AT_SLOT_B);
        for (int p = 0; p < 3; ++p)
          bulk_g2s(at_smem + s * AT_SLOT_B + p * AT_TILE_B, src + (size_t)p * a.part_stride, AT_TILE_B, &full[s]);
        if (++s == AT_STAGES) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  const int c2 = 2 * (lane & 3);   // first of this thread's two columns in every 8-column fragment
  // this thread's nine 16-byte entries of the warp's head-0 bias slice, 512 bytes apart (head 1: + AT_BIAS_HEAD_B)
  const uint32_t bias_s = smem_u32(at_smem + AT_OFF_BIAS + warp * AT_BIAS_WARP_B) + 16u * lane;
  int held = -1;   // type * pairs + pair of the bias the slice holds
  int slot = 0; uint32_t ph = 0;

  AtItem it(a, n0);
#pragma unroll 1
  for (long long n = n0; n < n1; ++n, it.next(a)) {
    const int wz = it.type / g.nWh, wh = it.type % g.nWh;
    if (it.type * a.pairs + it.pair != held) {
      // ---- bias slice of both heads: compact table entry (+ shift mask, in fp16) of every (row, key) this thread's
      // score fragments hold, in the order the score loop consumes them.  A thread reads back only what it wrote, so
      // the refill needs no barrier.  Runs while the item's tiles are in flight ----
      held = it.type * a.pairs + it.pair;
      const int fmask = a.roll ? ((wz == g.nWz - 1 ? 1 : 0) | (wh == g.nWh - 1 ? 2 : 0)) : 0;
      const __half mask_h = __float2half_rn(a.mask_l2);
      int rpart[2], rflag[2];   // this thread's two query rows (fragment rows l/4 and l/4 + 8 of the warp's 16)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = 16 * warp + (lane >> 2) + 8 * u;
        const int wi = i % WW, hi = (i / WW) % WH, zi = i / (WW * WH);
        rpart[u] = zi * ((2 * WW - 1) * WH * WH) + hi * (2 * WW - 1) + wi + (WW - 1);
        rflag[u] = (zi >= WZ - SZ ? 1 : 0) | (hi >= WH - SH ? 2 : 0);
      }
#pragma unroll 1
      for (int hd = 0; hd < 2; ++hd) {
        const __half* tab = a.bias_tab + ((long long)it.type * g.heads + 2 * it.pair + hd) * AT_TABLE;
#pragma unroll 1
        for (int i = 0; i < WIN_TOK / 16; ++i) {   // not unrolled: 72 loads in flight at once spill the score registers
          uint32_t w[4];
#pragma unroll
          for (int x = 0; x < 4; ++x) {   // word x: keys 8j + c2, 8j + c2 + 1 of row u, j = 2i + x/2, u = x%2
            const int j = 2 * i + (x >> 1), u = x & 1;
            __half bh[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * j + c2 + e;
              const int wj = col % WW, hj = (col / WW) % WH, zj = col / (WW * WH);
              const int kpart = (WZ * zj) * ((2 * WW - 1) * WH * WH) + (WH * hj) * (2 * WW - 1) - wj;
              const int kflag = (zj >= WZ - SZ ? 1 : 0) | (hj >= WH - SH ? 2 : 0);
              bh[e] = __ldg(tab + rpart[u] + kpart);
              if ((rflag[u] ^ kflag) & fmask) bh[e] = __hadd(bh[e], mask_h);
            }
            w[x] = (uint32_t)__half_as_ushort(bh[0]) | ((uint32_t)__half_as_ushort(bh[1]) << 16);
          }
          sts_b32x4(bias_s + hd * AT_BIAS_HEAD_B + i * 512, w);
        }
      }
    }

    mbar_wait(&full[slot], ph);
    const uint32_t q_s = smem_u32(at_smem + slot * AT_SLOT_B), k_s = q_s + AT_TILE_B, v_s = q_s + 2 * AT_TILE_B;
    // the warp's 16 q rows stage its output rows, same swizzle: head hd's outputs overwrite exactly the chunks that held
    // head hd's q, after the warp has them in registers
    const uint32_t stage = q_s + 16 * warp * 128;

#pragma unroll 1
    for (int hd = 0; hd < 2; ++hd) {
      // ---- S = Q K^T: 16 rows x 144 keys, K = 32 (two k16 steps = the head's four 16-byte chunks) ----
      uint32_t qa[2][4];
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
        ldsm_x4(at_chunk(q_s, 16 * warp + (lane & 7) + 8 * ((lane >> 3) & 1), hd * 4 + 2 * ks + (lane >> 4)), qa[ks]);
      __syncwarp();
      float s[WIN_TOK / 8][4];
#pragma unroll
      for (int j = 0; j < WIN_TOK / 8; ++j) {
        s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
        uint32_t kb[4];   // keys 8j .. 8j+7: dims 0-7 | 8-15 | 16-23 | 24-31
        ldsm_x4(at_chunk(k_s, 8 * j + (lane & 7), hd * 4 + (lane >> 3)), kb);
        mma_16816(s[j], qa[0], kb[0], kb[1]);
        mma_16816(s[j], qa[1], kb[2], kb[3]);
      }
      // ---- scale + bias, row max.  Half x of entry i: s[2i + x/4][x%4] ----
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < WIN_TOK / 16; ++i) {
        uint32_t bw[4];
        lds_b32x4(bias_s + hd * AT_BIAS_HEAD_B + i * 512, bw);
#pragma unroll
        for (int x = 0; x < 8; ++x) {
          const int j = 2 * i + (x >> 2), e = x & 3;
          const __half bh = __ushort_as_half((unsigned short)(bw[x >> 1] >> (16 * (x & 1))));
          s[j][e] = fmaf(s[j][e], a.sl2, __half2float(bh));
          mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
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
      // ---- 1/sum -> fp16 -> the head's 64 bytes of the two staged rows ----
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int r = (lane >> 2) + 8 * u;
        const float inv = 1.f / sum[u];
#pragma unroll
        for (int c = 0; c < 4; ++c)
          sts_b32(stage + r * 128 + (((hd * 4 + c) ^ (r & 7)) << 4) + 2 * c2, pack_half2(o[c][2 * u] * inv, o[c][2 * u + 1] * inv));
      }
    }
    __syncwarp();
    // ---- staged rows -> 128-byte lines of k-block `pair` of the projection's operand image, eight lanes per token row;
    // latitude-padding rows are skipped ----
    const long long my_tok = at_row_token(g, a.roll, it.b, wz, wh, it.ww, 16 * warp + (lane & 15));   // token of row lane % 16
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = 4 * k + (lane >> 3), ch = lane & 7;
      const long long tok = __shfl_sync(0xffffffffu, my_tok, r);
      if (tok < 0) continue;
      uint32_t v[4];
      lds_b32x4(stage + r * 128 + ((ch ^ (r & 7)) << 4), v);
      *reinterpret_cast<uint4*>(a.att_img + ((size_t)(tok >> 7) * a.att_nkb + it.pair) * (size_t)G2_A_BYTES +
                                (size_t)(tok & 127) * 128 + (((uint32_t)ch ^ ((uint32_t)tok & 7u)) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
    }
    fence_proxy_async_smem();   // the staging's generic writes are ordered before the next bulk copy into the slot
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[slot]);
    if (++slot == AT_STAGES) { slot = 0; ph ^= 1; }
  }
}

int launch_window_attention_tc(const AttnArgs& a, int num_sms, cudaStream_t st) {
  static std::atomic<uint64_t> configured{0};
  if (int rc = smem_opt_in(configured, reinterpret_cast<const void*>(k_window_attention_tc), AT_SMEM_BYTES)) return rc;
  if (a.items <= 0) return 0;
  if (num_sms <= 0) {
    int dev = 0;
    SKY_CUDA_OK(cudaGetDevice(&dev));
    SKY_CUDA_OK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const long long grid = a.items < num_sms ? a.items : num_sms;
  k_window_attention_tc<<<(unsigned)grid, AT_THREADS, AT_SMEM_BYTES, st>>>(a);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

// DownSample front end: 2x2 (lat, lon) merge + zero pad + LayerNorm(4C) -> fp16 tile image.
// One warp per output row; NPL = (4C)/32 values per lane.
template <int NPL>
__global__ void __launch_bounds__(256) k_down_merge_ln(const float* __restrict__ x, const uint8_t* __restrict__ ximg, uint8_t* __restrict__ img,
                                                       const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, int H, int W,
                                                       int C, int H2, int W2, long long rows) {
  long long row = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  int lane = threadIdx.x % 32;
  if (row >= rows) return;
  int w2 = (int)(row % W2); long long q = row / W2;
  int h2 = (int)(q % H2); q /= H2;  // q = member*Z + z
  // lane owns 4 consecutive features per 128-feature slab: 128-bit loads, 64-bit image stores
  static_assert(NPL % 4 == 0, "features per lane");
  float v[NPL];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NPL / 4; ++i) {
    const int e = 4 * lane + 128 * i;  // feature index in (hs, ws, c); C % 4 == 0, so the four share (hs, ws)
    const int sub = e / C, c = e % C;
    const int h = 2 * h2 + (sub >> 1), w = 2 * w2 + (sub & 1);
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h < H) {
      const long long src = (q * H + h) * W + w;
      if (ximg) {   // the token stream exists only as its fp16 operand image: 4 features = 8 bytes
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(ximg + img_offset(src, c, C / 64)));
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b2 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        t = make_float4(a.x, a.y, b2.x, b2.y);
      } else {
        t = __ldg(reinterpret_cast<const float4*>(x + src * C + c));
      }
    }
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    s += (t.x + t.y) + (t.z + t.w);
  }
  float mean = warp_sum(s) / (NPL * 32);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NPL; ++i) { float d = v[i] - mean; ss += d * d; }
  float rstd = rsqrtf(warp_sum(ss) / (NPL * 32) + eps);
#pragma unroll
  for (int i = 0; i < NPL / 4; ++i) {
    const int e = 4 * lane + 128 * i;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + e)), b = __ldg(reinterpret_cast<const float4*>(beta + e));
    uint2 pk;
    pk.x = pack_half2((v[4 * i] - mean) * rstd * g.x + b.x, (v[4 * i + 1] - mean) * rstd * g.y + b.y);
    pk.y = pack_half2((v[4 * i + 2] - mean) * rstd * g.z + b.z, (v[4 * i + 3] - mean) * rstd * g.w + b.w);
    *reinterpret_cast<uint2*>(img + img_offset(row, e, NPL / 2)) = pk;
  }
}

// test tap: fp16 image -> fp32 row-major
__global__ void k_image_to_rows(const uint8_t* __restrict__ img, int nkb, float* __restrict__ out, long long rows,
                                int cols) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  long long r = idx / cols; int c = (int)(idx % cols);
  out[idx] = __half2float(*reinterpret_cast<const __half*>(img + img_offset(r, c, nkb)));
}

// ======================================================================================
// engine
// ======================================================================================
struct GemmW {
  uint8_t* img = nullptr;
  int N = 0, K = 0, Kp = 0, BN = 0;
};
struct BlockW {
  GemmW qkv, proj, fc1, fc2;   // all at BLOCK_N 192: at C = 384 projection and fc2 are the two halves of a CTA pair
  GemmW fc1c;                   // C = 192: fc1 again at BLOCK_N 64, W1's 64-row slices of the fused MLP (mlp_fused.cuh)
  const float *qkv_b, *proj_b, *fc1_b, *fc2_b, *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  __half* bias_tab;  // (n_type, heads, 3312), fp16, pre-scaled by log2 e
};

struct PanguEngine : Engine {
  sky_pangu_config_t cfg;
  Geo g1, g2;
  int nch, nup;
  // Token stream storage (sky_model_debug_set "fp32_stream"): true = only the fp16 operand image (default: 8 of the 12 bytes
  // per token and feature of the projection / MLP epilogues disappear; step error 5.8e-4 instead of 5.1e-4 at 721x1440),
  // false = fp32 rows beside the image (round-1 / early round-2 data flow; for weights whose error margin is tighter)
  bool img_stream = true;
  std::vector<void*> owned;
  GemmW embed_u, embed_s, down, up1, up2, rec;
  std::vector<BlockW> blocks[4];
  const float *mean, *stdv, *masks, *embed_u_b, *embed_s_b, *down_g, *down_b, *up_g, *up_b;
  float* rec_b = nullptr;  // 5 upper + 4 surface

  PanguEngine(const sky_pangu_config_t& c, int dev) : cfg(c) {
    device = dev;
    nup = 5 * c.n_levels;
    nch = nup + 4;
    auto mk = [&](int H, int W, int C, int heads) {
      Geo g;
      g.Z = (c.n_levels + 1) / 2 + 1;
      g.H = H; g.W = W; g.C = C;
      g.Hp = (H + WH - 1) / WH * WH;
      g.nWz = g.Z / WZ; g.nWh = g.Hp / WH; g.nWw = W / WW;
      g.T = g.Z * H * W; g.nWin = g.nWz * g.nWh * g.nWw; g.heads = heads;
      return g;
    };
    int H = (c.nlat + 3) / 4, W = c.nlon / 4;
    g1 = mk(H, W, c.dim, c.heads[0]);
    g2 = mk((H + 1) / 2, W / 2, 2 * c.dim, c.heads[1]);
  }
  ~PanguEngine() override {
    for (void* p : owned) cudaFree(p);
  }

  template <class T>
  T* dalloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * sizeof(T)) != cudaSuccess) { set_error("cudaMalloc(%zu) failed", n * sizeof(T)); return nullptr; }
    owned.push_back(p);
    return reinterpret_cast<T*>(p);
  }

  int pack_alloc(GemmW& g, int N, int K, int BN) {
    g.N = N; g.K = K; g.Kp = (K + 63) / 64 * 64; g.BN = BN;
    if (N % BN) { set_error("N=%d not a multiple of BLOCK_N=%d", N, BN); return SKY_ERR_ARG; }
    g.img = dalloc<uint8_t>((size_t)N * g.Kp * 2);
    return g.img ? 0 : SKY_ERR_NOMEM;
  }
  int pack_rows(GemmW& g, const char* name, int Nsrc, int n_off, bool transposed, cudaStream_t st) {
    const float* w = param(name, (uint64_t)Nsrc * g.K);
    if (!w) return SKY_ERR_ARG;
    long long chunks = (long long)Nsrc * g.Kp / 8;
    k_pack_weight<<<(unsigned)((chunks + 255) / 256), 256, 0, st>>>(w, Nsrc, g.K, g.Kp, g.BN, transposed ? 1 : 0, n_off, g.img);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }
  int pack(GemmW& g, const char* name, int N, int K, int BN, bool transposed, cudaStream_t st) {
    int rc = pack_alloc(g, N, K, BN);
    return rc ? rc : pack_rows(g, name, N, 0, transposed, st);
  }

  int prepare(cudaStream_t st) override {
    const int C = cfg.dim;
#define P(dst, name, cnt) if (!((dst) = keep(name, (uint64_t)(cnt), st))) return SKY_ERR_ARG;   // persistent copies
    P(mean, "norm.mean", nch); P(stdv, "norm.std", nch);
    P(masks, "const.masks", 3LL * cfg.nlat * cfg.nlon);
    P(embed_u_b, "embed.upper.b", C); P(embed_s_b, "embed.surf.b", C);
    P(down_g, "down.ln.g", 4 * C); P(down_b, "down.ln.b", 4 * C);
    P(up_g, "up.ln.g", C); P(up_b, "up.ln.b", C);
    const float *ru = param("recover.upper.b", 5), *rs = param("recover.surf.b", 4);
    if (!ru || !rs) return SKY_ERR_ARG;
    rec_b = dalloc<float>(16);
    if (!rec_b) return SKY_ERR_NOMEM;
    SKY_CUDA_OK(cudaMemcpyAsync(rec_b, ru, 5 * 4, cudaMemcpyDeviceToDevice, st));
    SKY_CUDA_OK(cudaMemcpyAsync(rec_b + 5, rs, 4 * 4, cudaMemcpyDeviceToDevice, st));
    int rc;
    if ((rc = pack(embed_u, "embed.upper.w", C, 160, 192, false, st))) return rc;
    if ((rc = pack(embed_s, "embed.surf.w", C, 112, 192, false, st))) return rc;
    if ((rc = pack(down, "down.w", 2 * C, 4 * C, 192, false, st))) return rc;
    if ((rc = pack(up1, "up.w1", 4 * C, 2 * C, 192, false, st))) return rc;
    if ((rc = pack(up2, "up.w2", C, C, 192, false, st))) return rc;
    // patch recovery: one N = 160 + 64 weight (upper-air | surface columns)
    if ((rc = pack_alloc(rec, 224, 2 * C, 224))) return rc;
    if ((rc = pack_rows(rec, "recover.upper.w", 160, 0, true, st))) return rc;
    if ((rc = pack_rows(rec, "recover.surf.w", 64, 160, true, st))) return rc;
    for (int li = 0; li < 4; ++li) {
      const Geo& g = (li == 0 || li == 3) ? g1 : g2;
      const int c = g.C, heads = cfg.heads[li], n_type = g.nWz * g.nWh;
      blocks[li].resize(cfg.depths[li]);
      for (int bi = 0; bi < cfg.depths[li]; ++bi) {
        BlockW& b = blocks[li][bi];
        char nm[96];
        auto N = [&](const char* s) { snprintf(nm, sizeof nm, "layer%d.block%d.%s", li, bi, s); return nm; };
        if ((rc = pack(b.qkv, N("qkv.w"), 3 * c, c, 192, false, st))) return rc;
        if ((rc = pack(b.proj, N("proj.w"), c, c, 192, false, st))) return rc;
        if ((rc = pack(b.fc1, N("fc1.w"), 4 * c, c, 192, false, st))) return rc;
        if ((rc = pack(b.fc2, N("fc2.w"), c, 4 * c, 192, false, st))) return rc;
        if (c == 192 && (rc = pack(b.fc1c, N("fc1.w"), 4 * c, c, 64, false, st))) return rc;
        P(b.qkv_b, N("qkv.b"), 3 * c); P(b.proj_b, N("proj.b"), c);
        P(b.fc1_b, N("fc1.b"), 4 * c); P(b.fc2_b, N("fc2.b"), c);
        P(b.ln1_g, N("ln1.g"), c); P(b.ln1_b, N("ln1.b"), c);
        P(b.ln2_g, N("ln2.g"), c); P(b.ln2_b, N("ln2.b"), c);
        long long tot = (long long)AT_TABLE * n_type * heads;
        const float* bt = param(N("bias_table"), (uint64_t)tot);   // transient: repacked below
        if (!bt) return SKY_ERR_ARG;
        b.bias_tab = dalloc<__half>((size_t)tot);
        if (!b.bias_tab) return SKY_ERR_NOMEM;
        if ((rc = launch_pack_bias_table(bt, b.bias_tab, n_type, heads, st))) return rc;
        count_launch();
      }
    }
#undef P
    SKY_CUDA_OK(cudaGetLastError());
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }

  // ---- workspace carving -----------------------------------------------------------------
  struct Ws {
    float *x1, *x2;
    uint8_t *x1h, *skiph, *x2h, *atth, *hidh;
    uint8_t* qkv;
    size_t x1h_bytes;
    size_t total;
  };
  static size_t tiles(long long rows) { return (size_t)((rows + 127) / 128); }
  Ws carve(void* base, int B) const {
    Ws w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 1023) / 1024 * 1024; return (char*)base + o; };
    const size_t C = cfg.dim;
    const long long R1 = (long long)B * g1.T, R2 = (long long)B * g2.T;
    const size_t t1 = tiles(R1), t2 = tiles(R2);
    w.x1 = (float*)take((size_t)R1 * C * 4);
    w.x2 = (float*)take((size_t)R2 * 2 * C * 4);
    w.x1h_bytes = t1 * (C / 64) * G2_A_BYTES;
    w.x1h = (uint8_t*)take(w.x1h_bytes);
    w.skiph = (uint8_t*)take(w.x1h_bytes);
    w.x2h = (uint8_t*)take(t2 * (2 * C / 64) * G2_A_BYTES);
    // q | k | v window images (attention_tc.cuh): one 144-row x 128-byte tile per (member, window, head pair) and part
    const size_t wt1 = (size_t)B * g1.nWin * (g1.heads / 2), wt2 = (size_t)B * g2.nWin * (g2.heads / 2);
    w.qkv = (uint8_t*)take(3 * (wt1 > wt2 ? wt1 : wt2) * AT_TILE_B);
    size_t att_b = t1 * (C / 64) > t2 * (2 * C / 64) ? t1 * (C / 64) : t2 * (2 * C / 64);
    w.atth = (uint8_t*)take(att_b * G2_A_BYTES);
    size_t hid_b = t1 * (4 * C / 64) > t2 * (8 * C / 64) ? t1 * (4 * C / 64) : t2 * (8 * C / 64);
    w.hidh = (uint8_t*)take(hid_b * G2_A_BYTES);  // MLP hidden; also the down-sample / up-sample staging images
    w.total = off;
    return w;
  }
  size_t workspace_bytes(int batch) const override { return carve(nullptr, batch).total; }

  // ---- GEMM dispatch -----------------------------------------------------------------------
  // kPair: N = 2 BN on the column-split CTA pairs (k_gemm2_pair).  sc reads the weight w.
  template <int BN, bool kPair = false, class Sched, class Epi>
  int gemm2(int tag, const Sched& sc, const Epi& epi, const GemmW& w, long long M, cudaStream_t st) {
    if (w.BN != BN) { set_error("internal: weight packed for BLOCK_N=%d used with %d", w.BN, BN); return SKY_ERR_STATE; }
    prof_begin(tag, st);
    count_launch();
    const int rc = launch_gemm2<BN, kPair>(sc, epi, M, w.N, 1, num_sms, st);
    prof_end(tag, st);
    return rc;
  }
  template <int BN, bool kPair = false, class Epi>
  int gemm2(int tag, const AOperand& A, const Epi& epi, const GemmW& w, long long M, cudaStream_t st) {
    return gemm2<BN, kPair>(tag, SchedW<>{A, w.img, w.Kp / 64}, epi, w, M, st);
  }

  // IMG: the token stream of this handle lives only as its fp16 operand image (img_stream) — the LayerNorm epilogues then read
  // the residual from xh and write xh in place; otherwise x (fp32 rows) is read-modify-written beside the image.
  int run_block(float* x, uint8_t* xh, const Geo& g, const BlockW& b, int roll, int B, const Ws& ws, cudaStream_t st) {
    return img_stream ? run_block_t<true>(x, xh, g, b, roll, B, ws, st) : run_block_t<false>(x, xh, g, b, roll, B, ws, st);
  }
  // ---- test tap: stop inside the step ---------------------------------------------------------------------------
  // debug_set "stop_launch" n: the step returns after its n-th unit, counted in program order over the whole step: the
  // embedding; per block QKV (GEMM + padding fill), attention, projection, then the fused MLP or fc1 and fc2; the
  // down-sample, the up-sample and the recovery.  -1 (the default) never stops.  debug_copy then reads the buffers the
  // unit wrote (the workspace is reused).  A stopped step is never captured (Engine::step_cached), and the counter is host
  // state only: the launch sequence of an unstopped step is unchanged.
  static constexpr int PG_STOPPED = 1 << 20;   // not an error code: step() swallows it
  int units_done = 0;
  const Geo* stop_geo = nullptr;   // grid level of the unit the step stopped after
  bool stop_on_skip = false;       // the image-only token stream was the skip image there (embedding and layer 0)
  int unit_done(const Geo& g, bool on_skip) {
    if (stop_launch < 0 || !loaded || ++units_done < stop_launch) return 0;
    stop_geo = &g; stop_on_skip = on_skip;
    return PG_STOPPED;
  }

  template <bool IMG>
  int run_block_t(float* x, uint8_t* xh, const Geo& g, const BlockW& b, int roll, int B, const Ws& ws, cudaStream_t st) {
    const bool on_skip = xh == ws.skiph;
    // projection and fc2: the epilogue runs on the accumulator fragments on the fp16 stream (the fp32 rows stay staged).
    // Both update the stream in place: the residual is what the epilogue overwrites.
    using ELn = std::conditional_t<IMG, FragEpi<Epi2F32Img<true, 2>>, Epi2F32Img<true, 1>>;
    const void* res = IMG ? static_cast<const void*>(xh) : x;
    float* xout = IMG ? nullptr : x;
    const int C = g.C, nkb = C / 64;
    const long long R = (long long)B * g.T;
    int rc;
    const int pairs = g.heads / 2;
    const long long part_stride = (long long)B * g.nWin * pairs * AT_TILE_B;
    {  // QKV projection: natural-order tokens in, window image out (windowing / shift / padding applied by the epilogue)
      AOperand A(xh, nkb);
      FragEpi<EpiQkvWin> e{{ws.qkv, part_stride, b.qkv_b, g, roll, C, pairs}};
      if ((rc = gemm2<192>(KT_QKV, A, e, b.qkv, R, st))) return rc;
      if (g.Hp > g.H) {   // latitude-padding tokens (x = 0): their q, k, v rows are the projection's bias.  (Writing them from
                          // the GEMM epilogue of the neighbouring tokens instead cost the GEMM 0.5 ms/step: measured, reverted.)
        prof_begin(KT_QKV, st);
        rc = launch_qkv_fill_pad(ws.qkv, part_stride, b.qkv_b, g, roll, B, pairs, st);
        prof_end(KT_QKV, st);
        count_launch();
        if (rc) return rc;
      }
      if ((rc = unit_done(g, on_skip))) return rc;
    }
    {
      AttnArgs a{ws.qkv, part_stride, ws.atth, nkb, b.bias_tab, g, roll, B, pairs,
                 rsqrtf(32.f) * 1.4426950408889634f, cfg.mask_value * 1.4426950408889634f, (long long)B * g.nWin * pairs};
      prof_begin(KT_ATTN, st);
      count_launch();
      rc = launch_window_attention_tc(a, num_sms, st);
      prof_end(KT_ATTN, st);
      if (rc || (rc = unit_done(g, on_skip))) return rc;
    }
    {  // projection + LayerNorm + residual.  At C = 384 a 128 x 384 accumulator would take 192 registers per consumer thread:
       // the two CTAs of a cluster take 192 columns each of the same 128 rows, LayerNorm statistics cross through DSMEM
      AOperand A(ws.atth, nkb);
      ELn e{res, xout, C, xh, nkb, nullptr, b.proj_b, b.ln1_g, b.ln1_b, cfg.ln_eps};
      rc = C == 192 ? gemm2<192>(KT_PROJ, A, e, b.proj, R, st) : gemm2<192, true>(KT_PROJ, A, e, b.proj, R, st);
      if (rc || (rc = unit_done(g, on_skip))) return rc;
    }
    if (IMG && C == 192) {   // MLP in one kernel: the hidden activation stays on the SM (mlp_fused.cuh).  At C = 384 the
                             // fused CTA-pair kernel measured 2.4x slower than fc1 + fc2 (DESIGN.md section 4)
      const MlpArgs m{xh, b.fc1c.img, b.fc2.img, b.fc1_b,
                      {Epi2F32Img<true, 2>{xh, nullptr, C, xh, nkb, nullptr, b.fc2_b, b.ln2_g, b.ln2_b, cfg.ln_eps}}, R};
      prof_begin(KT_MLP, st);
      count_launch();
      rc = launch_mlp_fused<3>(m, num_sms, st);
      prof_end(KT_MLP, st);
      if (rc || (rc = unit_done(g, on_skip))) return rc;
    } else {  // MLP: fc1 + GELU into the fp16 hidden image, then fc2 + LayerNorm + residual
      AOperand A(xh, nkb);
      FragEpi<Epi2F16<true, true>> e{reinterpret_cast<__half*>(ws.hidh), 0, 4 * nkb, b.fc1_b};
      if ((rc = gemm2<192>(KT_FC1, A, e, b.fc1, R, st)) || (rc = unit_done(g, on_skip))) return rc;
      AOperand A2(ws.hidh, 4 * nkb);
      ELn e2{res, xout, C, xh, nkb, nullptr, b.fc2_b, b.ln2_g, b.ln2_b, cfg.ln_eps};
      rc = C == 192 ? gemm2<192>(KT_FC2, A2, e2, b.fc2, R, st) : gemm2<192, true>(KT_FC2, A2, e2, b.fc2, R, st);
      if (rc || (rc = unit_done(g, on_skip))) return rc;
    }
    if (range_guard) {   // fp16 operand images of this block (whole tiles only: the tail rows of the last tile are never written)
      const size_t full = (size_t)(R / 128) * nkb * G2_A_BYTES;
      if ((rc = range_scan(0, xh, full, st))) return rc;
      if ((rc = range_scan(1, ws.qkv, (size_t)3 * part_stride, st))) return rc;
      if ((rc = range_scan(2, ws.atth, full, st))) return rc;
    }
    return 0;
  }

  int step(const float* x_in, float* x_out, int B, void* wsp, size_t ws_bytes, cudaStream_t st) override {
    units_done = 0;
    stop_geo = nullptr;
    const int rc = step_units(x_in, x_out, B, wsp, ws_bytes, st);
    return rc == PG_STOPPED ? 0 : rc;
  }
  int step_units(const float* x_in, float* x_out, int B, void* wsp, size_t ws_bytes, cudaStream_t st) {
    if (!loaded) { set_error("weights not loaded"); return SKY_ERR_STATE; }
    Ws ws = carve(wsp, B);
    if (ws_bytes < ws.total) { set_error("workspace too small: %zu < %zu", ws_bytes, ws.total); return SKY_ERR_ARG; }
    const int C = cfg.dim, HW = g1.H * g1.W, nzt = g1.Z - 1;
    const long long R1 = (long long)B * g1.T, R2 = (long long)B * g2.T;
    int rc;
    // test tap (sky_model_debug_set "stop_after"): return early so that debug_copy can read the token buffers
    // (0 embed, 1 layer0, 2 down, 3 layer1, 4 layer2, 5 up, 6 layer3; default 99 = whole step)
    const int stop = stop_after;
    // ---- patch embedding: producer warps gather and normalise the fp32 state into the A tiles (im2col) ----
    {
      long long M = (long long)B * nzt * HW;
      ProdEmbedUpper p{x_in, mean, stdv, cfg.nlat, cfg.nlon, cfg.n_levels, 5, nch, g1.H, g1.W, nzt, M};
      EpiStoreF32 e{img_stream ? nullptr : ws.x1, C, embed_u_b, g1.T, HW, 1, (long long)nzt * HW, ws.skiph, C / 64};
      if ((rc = gemm2<192>(KT_EMBED, SchedProd<ProdEmbedUpper>{p, embed_u.img, embed_u.Kp / 64}, e, embed_u, M, st))) return rc;
      long long Ms = (long long)B * HW;
      ProdEmbedSurf ps{x_in, masks, mean, stdv, cfg.nlat, cfg.nlon, nch, nup, 4, 3, g1.H, g1.W, Ms};
      EpiStoreF32 es{img_stream ? nullptr : ws.x1, C, embed_s_b, g1.T, HW, 0, (long long)HW, ws.skiph, C / 64};
      if ((rc = gemm2<192>(KT_EMBED, SchedProd<ProdEmbedSurf>{ps, embed_s.img, embed_s.Kp / 64}, es, embed_s, Ms, st))) return rc;
      if ((rc = unit_done(g1, true))) return rc;
    }
    if (stop == 0) return 0;
    for (size_t i = 0; i < blocks[0].size(); ++i)
      if ((rc = run_block(ws.x1, ws.skiph, g1, blocks[0][i], (int)(i & 1), B, ws, st))) return rc;
    if (stop == 1) return 0;
    // the first layer works in place on the skip image: its final operand image IS the skip connection that patch
    // recovery concatenates, the up-sample path writes the other image (x1h) — no copy
    // ---- down-sample ----
    {
      prof_begin(KT_DOWN, st);
      k_down_merge_ln<24><<<(unsigned)((R2 + 7) / 8), 256, 0, st>>>(ws.x1, img_stream ? ws.skiph : nullptr, ws.hidh, down_g, down_b,
                                                                 cfg.ln_eps, g1.H, g1.W, C, g2.H, g2.W, R2);
      prof_end(KT_DOWN, st);
      count_launch();
      SKY_CUDA_OK(cudaGetLastError());
      AOperand A(ws.hidh, 4 * C / 64);
      Epi2F32Img<false, 0> e{nullptr, img_stream ? nullptr : ws.x2, 2 * C, ws.x2h, 2 * C / 64, nullptr, nullptr, nullptr, nullptr, 0.f};
      if ((rc = gemm2<192>(KT_DOWN, A, e, down, R2, st))) return rc;
      if ((rc = range_scan(3, ws.x2h, (size_t)(R2 / 128) * (2 * C / 64) * G2_A_BYTES, st))) return rc;
      if ((rc = unit_done(g2, false))) return rc;
    }
    if (stop == 2) return 0;
    for (int li = 1; li <= 2; ++li) {
      for (size_t i = 0; i < blocks[li].size(); ++i)
        if ((rc = run_block(ws.x2, ws.x2h, g2, blocks[li][i], (int)(i & 1), B, ws, st))) return rc;
      if (stop == 2 + li) return 0;
    }
    // ---- up-sample ----
    {
      AOperand A(ws.x2h, 2 * C / 64);
      Epi2UpShuffle e{ws.hidh, C / 64, C, up_g, up_b, cfg.ln_eps, nullptr, g1.H, g1.W, g2.H, g2.W};
      if ((rc = gemm2<192>(KT_UP, A, e, up1, R2, st))) return rc;
      AOperand A2(ws.hidh, C / 64);
      Epi2F32Img<false, 0> e2{nullptr, img_stream ? nullptr : ws.x1, C, ws.x1h, C / 64, nullptr, nullptr, nullptr, nullptr, 0.f};
      if ((rc = gemm2<192>(KT_UP, A2, e2, up2, R1, st)) || (rc = unit_done(g1, false))) return rc;
    }
    if (stop == 5) return 0;
    for (size_t i = 0; i < blocks[3].size(); ++i)
      if ((rc = run_block(ws.x1, ws.x1h, g1, blocks[3][i], (int)(i & 1), B, ws, st))) return rc;
    if (stop == 6) return 0;
    // ---- patch recovery: concat(skip, x) along K, one GEMM for upper-air + surface ----
    {
      const AOperand A = AOperand(ws.skiph, C / 64).add(ws.x1h, C / 64);
      Epi2Recover e{x_out, rec_b, mean, stdv, cfg.nlat, cfg.nlon, nch, nup, cfg.n_levels, g1.H, g1.W, g1.T};
      if ((rc = gemm2<224>(KT_RECOVER, A, e, rec, R1, st))) return rc;
    }
    return unit_done(g1, false);
  }

  int debug_set(const char* key, long long value) override {
    if (!strcmp(key, "fp32_stream")) { img_stream = value == 0; drop_graphs(); return 0; }
    return Engine::debug_set(key, value);
  }

  int debug_copy(const char* what, float* dst, uint64_t max_floats, void* wsp, int B, cudaStream_t st) override {
    Ws ws = carve(wsp, B);
    const float* src = nullptr;
    uint64_t n = 0;
    const long long R1 = (long long)B * g1.T, R2 = (long long)B * g2.T;
    if (!strcmp(what, "qkv") || !strcmp(what, "att_h") || !strcmp(what, "hid_h") || !strcmp(what, "stream_h")) {
      // raw taps after a stop_launch stop: the buffer as it lies in memory at the stopped unit's grid level (decoded on the
      // host), the whole of it: q | k | v window image (3 part_stride bytes), attention output, MLP hidden and token
      // stream images (every 128-row tile, the rows past B T included)
      if (!stop_geo) { set_error("debug buffer '%s' needs a step stopped by stop_launch", what); return SKY_ERR_STATE; }
      const Geo& g = *stop_geo;
      const long long R = (long long)B * g.T;
      const size_t img = tiles(R) * (g.C / 64) * G2_A_BYTES;
      const uint8_t* p = what[0] == 'q' ? ws.qkv : what[0] == 'a' ? ws.atth : what[0] == 'h' ? ws.hidh
                       : &g == &g2 ? ws.x2h : stop_on_skip ? ws.skiph : ws.x1h;
      const size_t bytes = what[0] == 'q' ? 3 * (size_t)B * g.nWin * (g.heads / 2) * AT_TILE_B : what[0] == 'h' ? 4 * img : img;
      if (bytes != max_floats * sizeof(float)) {
        set_error("debug buffer '%s' is %zu floats, destination %llu", what, bytes / sizeof(float), (unsigned long long)max_floats);
        return SKY_ERR_ARG;
      }
      SKY_CUDA_OK(cudaMemcpyAsync(dst, p, bytes, cudaMemcpyDeviceToDevice, st));
      return 0;
    }
    const bool stream_tap = img_stream && (!strcmp(what, "tokens1") || !strcmp(what, "tokens2"));
    if (!stream_tap && !strcmp(what, "tokens1")) { src = ws.x1; n = (uint64_t)R1 * cfg.dim; }
    else if (!stream_tap && !strcmp(what, "tokens2")) { src = ws.x2; n = (uint64_t)R2 * 2 * cfg.dim; }
    else if (stream_tap || !strcmp(what, "tokens1_h") || !strcmp(what, "tokens2_h") || !strcmp(what, "skip_h")) {
      // the fp16 operand image, expanded to fp32 rows.  With the image-only token stream "tokens1" is the skip image until the
      // down-sample (embedding and first layer work in place on it) and the x1 image from the up-sample on.
      const bool two = what[6] == '2';
      const bool on_skip = stop_geo ? stop_on_skip : stop_after <= 1;
      const uint8_t* img = two ? ws.x2h : ((!strcmp(what, "skip_h") || (stream_tap && on_skip)) ? ws.skiph : ws.x1h);
      const long long rows = two ? R2 : R1;
      const int cols = two ? 2 * cfg.dim : cfg.dim;
      if ((uint64_t)rows * cols > max_floats) { set_error("destination too small"); return SKY_ERR_ARG; }
      k_image_to_rows<<<(unsigned)((rows * cols + 255) / 256), 256, 0, st>>>(img, cols / 64, dst, rows, cols);
      SKY_CUDA_OK(cudaGetLastError());
      return 0;
    } else if (!strcmp(what, "range")) {
      if (!range_dev || max_floats < 8) { set_error("range guard is off (debug_set range_guard 1) or destination < 8 floats"); return SKY_ERR_STATE; }
      src = range_dev; n = 8;
    } else { set_error("unknown debug buffer '%s'", what); return SKY_ERR_ARG; }
    if (n > max_floats) n = max_floats;
    SKY_CUDA_OK(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
};

Engine* make_pangu_engine(const sky_pangu_config_t& cfg, int device) {
  if (cfg.nlon % 96 || cfg.nlat < 8 || cfg.n_levels != 13 || cfg.dim != 192) {
    set_error("unsupported Pangu shape: nlat=%d nlon=%d (need nlon %% 96 == 0) levels=%d dim=%d", cfg.nlat, cfg.nlon,
              cfg.n_levels, cfg.dim);
    return nullptr;
  }
  for (int i = 0; i < 4; ++i) {
    int c = (i == 0 || i == 3) ? cfg.dim : 2 * cfg.dim;
    if (cfg.heads[i] * 32 != c) { set_error("head_dim must be 32"); return nullptr; }
  }
  return new PanguEngine(cfg, device);
}

}  // namespace sky
