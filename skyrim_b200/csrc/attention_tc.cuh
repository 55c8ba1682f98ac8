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
// Work item n = ((type * pairs + pair) * B + b) * nWw + ww, one (window, head pair).  The kernel is persistent: CTA c
// walks the contiguous item range [c items / G, (c+1) items / G) of a grid of G = min(items, SMs) CTAs, so consecutive
// items of a CTA share their window type and head pair for B nWw items at a time.  Ten warps:
//   * warp 9, the producer: one lane streams each item's q, k, v tiles (three contiguous 18 KB bulk copies) into a
//     two-slot ring, so the next item's loads run under the current item's compute;
//   * warps 0-8 compute: warp w owns query rows 16w .. 16w+15 of both heads.  Per head the warp computes its 16 x 144
//     score block in registers (ldmatrix + mma.sync), adds the bias, takes exp2 against the row max, and multiplies P
//     (fp16, straight from the score registers) by V (ldmatrix.trans).  1/sum is applied to the 32 outputs of each row.
// The bias (compact table entry + shift mask, added in fp16) depends only on (type, head) and the thread's fragment
// position, so each warp expands its 16 x 144 slice of both heads into shared memory in the order the score loop
// consumes it (nine 16-byte loads per head) and rebuilds it only when the item's (type, pair) changes.  Once a warp
// holds its q fragments in registers, its 16 q rows of the slot are free: the output rows are staged there and leave as
// full 128-byte lines of the projection's operand image.
// This header holds the layout, EpiQkvWin and the device helpers; the kernels themselves are in pangu_engine.cu.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "gemm2.cuh"

namespace sky {

constexpr int AT_TABLE = (2 * WW - 1) * WH * WH * WZ * WZ;   // 3312 entries of the compact bias table per (type, head)
constexpr int AT_TILE_B = WIN_TOK * 128;                     // 18432: one (window, head pair) tile of q, k or v
constexpr int AT_WARPS = WIN_TOK / 16;                       // compute warps, one per 16 query rows
constexpr int AT_THREADS = 32 * (AT_WARPS + 1);              // + the producer warp
constexpr int AT_STAGES = 2;                                 // ring slots
constexpr int AT_SLOT_B = 3 * AT_TILE_B;                     // one item's q | k | v tiles
constexpr int AT_BIAS_WARP_B = AT_WARPS * 32 * 16;           // a warp's 16 x 144 fp16 bias slice: uint4 [i < 9][lane]
constexpr int AT_BIAS_HEAD_B = AT_WARPS * AT_BIAS_WARP_B;    // one head: 144 x 144 fp16
constexpr int AT_OFF_BIAS = AT_STAGES * AT_SLOT_B;           // ring, then the bias [head][warp][i][lane], then the barriers
constexpr int AT_OFF_BAR = AT_OFF_BIAS + 2 * AT_BIAS_HEAD_B;
constexpr int AT_SMEM_BYTES = AT_OFF_BAR + 2 * AT_STAGES * 8;
static_assert(WIN_TOK % 16 == 0 && AT_SMEM_BYTES <= 227 * 1024, "tile shapes");

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

// Host launchers of k_qkv_fill_pad, k_window_attention_tc and k_pack_bias_table.  The kernels and launchers are defined
// in pangu_engine.cu only; the engine and the kernel-level probe (pangu_probe.cu) both launch them through these.
int launch_qkv_fill_pad(uint8_t* out, long long part_stride, const float* bias, const Geo& g, int roll, int B, int pairs,
                        cudaStream_t st);
int launch_window_attention_tc(const AttnArgs& a, int num_sms, cudaStream_t st);
int launch_pack_bias_table(const float* src, __half* dst, int n_type, int heads, cudaStream_t st);

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

// shared-space 32- and 128-bit accesses (volatile: the bias slice and the staged rows are rewritten between reads)
__device__ __forceinline__ void sts_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_b32x4(uint32_t addr, const uint32_t (&v)[4]) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
}
__device__ __forceinline__ void lds_b32x4(uint32_t addr, uint32_t (&v)[4]) {
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr) : "memory");
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
        if (drow >= 0)
          *reinterpret_cast<uint4*>(pbase + (size_t)drow * 128 + ((cpos ^ ((uint32_t)drow & 7u)) << 4)) = pk;
      }
      __syncwarp();
    }
  }
};


}  // namespace sky
