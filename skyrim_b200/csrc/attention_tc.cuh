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
#include "pangu_ops.cuh"

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

// natural token row (member b = row / T) -> row of its tile of the window image at head pair 0: win * pairs * 144 + j, win
// the member's window and j the position in it, on the rolled grid when roll is set.  members * tokens < 2^31, and
// members * windows * pairs * 144 < 2^31 (checked by the callers).
__device__ __forceinline__ int qkv_window_row(const Geo& g, int roll, int pairs, unsigned row) {
  const unsigned b = row / (unsigned)g.T, t = row - b * (unsigned)g.T;
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
  return win * pairs * WIN_TOK + (zj * WH + hj) * WW + wj;
}

// ---------------------------------------------------------------------------------------------------------------
// QKV projection epilogue, on the accumulator fragments (FragEpi<EpiQkvWin>, BLOCK_N 192): accumulator (tokens in
// natural order) + bias -> fp16 window image.  C is a multiple of 192, so an n-tile is three consecutive head pairs
// hp0 .. hp0 + 2 of one part (q, k or v at C = 192; half a part at C = 384).  The output tile holds them as
// [pair p < 3][tile row r < 128][128 B], and row r of block p is byte for byte destination row drow (qkv_window_row of the
// tile's row r) of pair hp0 + p: its 16-byte chunk c sits at c ^ (drow & 7), the swizzle of the destination row, not of r.
// The loader stores the tile in runs of consecutive drow (kScatter): a run breaks at a window edge, at the end of a latitude
// row or level, at a member boundary and at the roll's wrap, so most runs are one window row (12 rows, 1.5 KB) and a tile
// has 10 to 15 of them.  One bulk copy per (run, pair) instead of one per (row, pair) is 30 to 45 copies instead of 384.
// ---------------------------------------------------------------------------------------------------------------
struct EpiQkvWin {
  static constexpr bool kNeedsBias = false, kLoadsTile = false, kScatter = true;
  uint8_t* out; long long part_stride; const float* bias; Geo g; int roll; int C; int pairs;
  const float* gamma = nullptr; const float* beta = nullptr;   // unused (uniform epilogue interface)
  // The loader, not the consumers, computes the destination rows: it has the time while it waits for ring slots, and
  // the divisions by the grid's run-time sizes stay off the epilogue that keeps the tensor cores waiting.  -1: row >= M.
  __device__ __forceinline__ int dest_row(long long row, long long M) const {
    return row < M ? qkv_window_row(g, roll, pairs, (unsigned)row) : -1;
  }
  template <int BN, class Acc>
  __device__ void frag(Acc& acc, const FragCtx& x) const {
    static_assert(BN == 192, "an n-tile is three head pairs");
    const float* bp = bias + x.n0 + x.c2;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(bp + 8 * i));
      float* d = acc.d + 4 * i;
      d[0] += b.x; d[1] += b.y; d[2] += b.x; d[3] += b.y;
    }
    mbar_wait(x.out_ready, x.ready_parity);   // also publishes the loader's map of destination rows (svec_s)
    uint32_t row_s[2], sw[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t r = (uint32_t)(x.row + 8 * h);
      uint32_t drow;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(drow) : "r"(x.svec_s + r * 4u) : "memory");
      sw[h] = drow & 7u;
      row_s[h] = x.out_s + r * 128u + (uint32_t)x.c2 * 2u;
    }
#pragma unroll
    for (int i = 0; i < BN / 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        sts_b32(row_s[h] + (uint32_t)(i >> 3) * G2_A_BYTES + ((((uint32_t)i & 7u) ^ sw[h]) << 4),
                pack_half2(acc.d[4 * i + 2 * h], acc.d[4 * i + 2 * h + 1]));
  }
  // Loader warp: store the output tile of the n-tile at column n0, with tile row r going to destination row map[r]
  // (map_s + 4 r; -1 past M, those rows are not written).  Lane l looks at rows l + 32 k; every lane issues the copies of
  // the runs that start at its rows and waits until they have read the tile.
  __device__ void frag_store(int n0, uint32_t out_s, uint32_t map_s, int lane) const {
    const int part = n0 / C, hp0 = (n0 - part * C) >> 6;
    uint8_t* dst = out + (size_t)part * part_stride + (size_t)hp0 * AT_TILE_B;
    int d[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) asm volatile("ld.shared.b32 %0, [%1];" : "=r"(d[k]) : "r"(map_s + (uint32_t)(lane + 32 * k) * 4u) : "memory");
    // bit l of brk[k]: row 32 k + l does not continue the run of the row before it (it starts a run, or is past M)
    uint32_t brk[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int prev = __shfl_up_sync(0xffffffffu, d[k], 1);
      const int last = __shfl_sync(0xffffffffu, d[k > 0 ? k - 1 : 0], 31);
      if (lane == 0) prev = k > 0 ? last : -1;
      brk[k] = __ballot_sync(0xffffffffu, d[k] < 0 || prev < 0 || d[k] != prev + 1);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (d[k] < 0 || !((brk[k] >> lane) & 1u)) continue;
      const int r = 32 * k + lane;
      int end = G2_BLOCK_M;   // the next break after row r
#pragma unroll
      for (int kk = 3; kk >= k; --kk) {
        const uint32_t m = kk == k ? brk[kk] & (0xfffffffeu << lane) : brk[kk];
        if (m) end = 32 * kk + __ffs((int)m) - 1;
      }
      const uint32_t bytes = (uint32_t)(end - r) * 128u;
#pragma unroll
      for (int p = 0; p < 3; ++p)
        bulk_s2g(dst + (size_t)p * AT_TILE_B + (size_t)d[k] * 128, out_s + (uint32_t)(p * G2_A_BYTES + r * 128), bytes);
    }
    bulk_commit();
    bulk_wait_read<0>();
  }
};

}  // namespace sky
