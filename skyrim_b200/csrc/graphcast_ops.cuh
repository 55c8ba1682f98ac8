// GraphCast step: device pieces that are not GEMM main loops — epilogue functors for k_gemm2 (gemm2.cuh), the feature
// builder, the CSR aggregation and small set-up kernels.  Latent width is fixed at 512 (GC_L).
//
// Data layout (per member): every latent matrix (grid nodes, mesh nodes, the three edge sets) is an fp16 tile image
// [rows/128][8][128 x 128 B, SWIZZLE_128B] — byte for byte the A operand of the next GEMM.  Of the three residual streams
// only the mesh nodes keep an fp32 row-major copy; grid nodes and mesh edges are read-modify-written in their images
// (EpiGcLn<2>).  Per-node first-layer partial products ("tables": v W1_s^T, v W1_r^T) are fp16 row-major and are gathered
// by edge index inside the hidden GEMM's epilogue.
#pragma once
#include "gemm2.cuh"

namespace sky {

constexpr int GC_L = 512;
constexpr int GC_NKB = GC_L / 64;

__device__ __forceinline__ float silu_f(float x) {
  // x * sigmoid(x); exp through ex2: one MUFU.EX2 + one MUFU.RCP per element
  return x * mufu_rcp(1.f + mufu_ex2(-1.4426950408889634f * x));
}
// table rows are re-read by many edges while operand / hidden images stream through L2 once: keep the tables
// (L2 cache-hint policies; the plain .L2::evict_* qualifiers exist for 256-bit accesses only)
__device__ __forceinline__ uint64_t l2_policy_keep() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_stream() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint4 ldg_hint(const void* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void stg_hint(void* p, const uint4& v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void add_h8(float* v, const uint4& p) {
  const __half2* h = reinterpret_cast<const __half2*>(&p);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(h[i]);
    v[2 * i] += f.x; v[2 * i + 1] += f.y;
  }
}

// hidden = swish(acc + bias + Ta[ia[row]] + Tb[ib[row]])  ->  fp16 tile image (GC_NKB k-blocks per row tile).
// kG = number of gathered tables (0, 1, 2).  Everything after the accumulator read happens in the RE-TILED domain (lane ->
// row = it * 8 + lane / 4, 8 columns = lane % 4): there four lanes read 64 contiguous bytes of one table row, so a gather
// instruction touches 8 cache lines instead of 32.  A gather is an L2 round trip, so the table rows of TWO 32-column
// chunks are requested together, in front of the first chunk's accumulator read; the second chunk then finds its rows in
// registers.  A warp handles 4 chunks per 256-column tile: 2 exposed round trips instead of 4.
template <int kG>
struct EpiGcSiluImg {
  static constexpr bool kNeedsBias = false;
  uint8_t* out; const float* bias;
  const float* gamma = nullptr; const float* beta = nullptr;   // unused (uniform epilogue interface)
  const __half* ta = nullptr; int lda = 0; const int* ia = nullptr;
  const __half* tb = nullptr; int ldb = 0; const int* ib = nullptr;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& x) const {
    const int rsub = x.lane >> 2, ch = x.lane & 3;
    const uint32_t r0 = (uint32_t)(x.row0 & 127);
    const uint64_t pol_keep = l2_policy_keep(), pol_stream = l2_policy_stream();
    // table rows of the four rows this lane finishes (it * 8 + rsub): indices come from the row-owner lanes by shuffle
    const __half* pa[kG >= 1 ? 4 : 1]; const __half* pb[kG >= 2 ? 4 : 1];
    {
      const long long row = x.row0 + x.lane;
      const bool valid = row < x.M;
      const int ja = (kG >= 1 && valid) ? __ldg(ia + row) : 0;
      const int jb = (kG >= 2 && valid) ? __ldg(ib + row) : 0;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        if (kG >= 1) pa[it] = ta + (size_t)__shfl_sync(0xffffffffu, ja, it * 8 + rsub) * lda + x.n0 + ch * 8;
        if (kG >= 2) pb[it] = tb + (size_t)__shfl_sync(0xffffffffu, jb, it * 8 + rsub) * ldb + x.n0 + ch * 8;
      }
    }
    const int cstep = 32 * x.nparts;
    for (int c0 = x.part * 32; c0 < BN; c0 += 2 * cstep) {
      uint4 ga[kG >= 1 ? 8 : 1], gb[kG >= 2 ? 8 : 1];     // [chunk u][it]
      const bool two = c0 + cstep < BN;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int cu = (u && !two) ? c0 : c0 + u * cstep;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          if (kG >= 1) ga[u * 4 + it] = ldg_hint(pa[it] + cu, pol_keep);
          if (kG >= 2) gb[u * 4 + it] = ldg_hint(pb[it] + cu, pol_keep);
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = c0 + u * cstep;
        if (u && !two) break;
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + x.n0 + c + ch * 8));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + x.n0 + c + ch * 8 + 4));
        {
          float v[32];
          acc.load32(c, v);
          patch_put_v(x.patch_s, x.lane, v);
        }
        __syncwarp();
        const int col = x.n0 + c;
        uint8_t* ibase = out + ((size_t)(x.row0 >> 7) * GC_NKB + (col >> 6)) * (size_t)G2_A_BYTES + r0 * 128;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 8 + rsub;
          const float4 t0 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch));
          const float4 t1 = lds_f32x4(patchv_addr(x.patch_s, rr, 2 * ch + 1));
          float v[8] = {t0.x + b0.x, t0.y + b0.y, t0.z + b0.z, t0.w + b0.w, t1.x + b1.x, t1.y + b1.y, t1.z + b1.z, t1.w + b1.w};
          if (kG >= 1) add_h8(v, ga[u * 4 + it]);
          if (kG >= 2) add_h8(v, gb[u * 4 + it]);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = silu_f(v[j]);
          uint4 pk;
          pk.x = pack_half2(v[0], v[1]); pk.y = pack_half2(v[2], v[3]);
          pk.z = pack_half2(v[4], v[5]); pk.w = pack_half2(v[6], v[7]);
          if (x.row0 + rr < x.M)
            stg_hint(ibase + rr * 128 + (((((col & 63) >> 3) + ch) ^ (rr & 7)) << 4), pk, pol_stream);
        }
        __syncwarp();
      }
    }
  }
};

// y = LayerNorm(acc + bias) * gamma + beta over the full 512-wide row, then any of
//   xout[row] = residual + y                  fp32 row-major (ld 512); residual = xin (fp32 rows, may equal xout) or
//                                             xin_img (the fp16 operand image of the stream, may equal img) or nothing
//   img       = fp16 tile image of that sum   (the A operand of the next GEMM)
//   yimg      = fp16 tile image of y itself   (what the aggregation sums: the update BEFORE the residual)
// Grid-node and mesh-edge latents live ONLY as fp16 images (residual read from xin_img, sum formed in fp32, rounded once
// into img): their consumers round to fp16 anyway, and the measured cost on the oracle is a tendency error of 7.95e-4
// instead of 7.66e-4 over 16 layers (tests/test_graphcast_cpu.py); it saves 3 KB of HBM traffic per row and launch.
// Structure follows Epi2F32Img (gemm2.cuh): statistics in the row-owner domain, then 32x32 blocks re-tiled through the
// warp's patch so that every global access is a 128-bit access on a full 128-byte row segment.
// kRes: residual source, a compile-time choice (a run-time branch per load serialised the loads and cost 10 - 50 % of the
// kernel): 0 none, 1 fp32 rows (xin), 2 the stream's fp16 image (xin_img)
template <int kRes>
struct EpiGcLn {
  static constexpr bool kNeedsBias = true;
  const float* xin; float* xout; uint8_t* img; uint8_t* yimg;
  const float* bias; const float* gamma; const float* beta; float eps;
  const uint8_t* xin_img = nullptr;
  // residual values of the lane's eight (row, 4-column) pieces of the 32-column group at local column c: all eight
  // loads are issued before any is used
  __device__ __forceinline__ void residual8(const EpiCtx& e, int c, int rsub4, int c4, size_t rowoff, long long rows_left, bool on,
                                            float4 (&x)[8]) const {
    if constexpr (kRes == 1) {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        x[it] = (on && rr < rows_left) ? *reinterpret_cast<const float4*>(xin + rowoff + (size_t)rr * GC_L + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else if constexpr (kRes == 2) {
      const int col = e.n0 + c + c4 * 4;
      const uint8_t* base = xin_img + ((size_t)(e.row0 >> 7) * GC_NKB + (col >> 6)) * (size_t)G2_A_BYTES + (uint32_t)(e.row0 & 127) * 128 + (c4 & 1) * 8;
      const uint32_t chunk = (uint32_t)(col & 63) >> 3;
      uint2 u[8];
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + rsub4;
        u[it] = (on && rr < rows_left) ? *reinterpret_cast<const uint2*>(base + rr * 128 + ((chunk ^ (uint32_t)(rr & 7)) << 4)) : make_uint2(0u, 0u);
      }
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u[it].x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u[it].y));
        x[it] = make_float4(a.x, a.y, b.x, b.y);
      }
    } else {
#pragma unroll
      for (int it = 0; it < 8; ++it) x[it] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  template <int BN>
  __device__ void prefetch(const EpiCtx& e) const {
    if (kRes == 0) return;
    const long long row = e.row0 + e.lane;
    if (row >= e.M) return;
    if (kRes == 2) {
      const char* p = reinterpret_cast<const char*>(xin_img) + ((size_t)(e.row0 >> 7) * GC_NKB + (e.n0 >> 6)) * (size_t)G2_A_BYTES +
                      ((uint32_t)(e.row0 & 127) + e.lane) * 128;
#pragma unroll
      for (int i = e.part; i < BN / 64; i += e.nparts) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (size_t)i * G2_A_BYTES));
      return;
    }
    if (!xin) return;
    const char* p = reinterpret_cast<const char*>(xin + row * GC_L + e.n0);
#pragma unroll
    for (int i = e.part; i < BN * 4 / 128; i += e.nparts) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + i * 128));
  }
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    static_assert(BN == GC_L || 2 * BN == GC_L, "the tile is the full latent width, or one half of a column-split CTA pair");
    constexpr int NG = BN / 32;
    const int rsub4 = e.lane >> 3, c4 = e.lane & 7;
    const long long rows_left = e.M - e.row0;
    const size_t rowoff = (size_t)e.row0 * GC_L + e.n0 + c4 * 4;
    // residual rows of the first column group: requested before the statistics pass (they come from L2: prefetch())
    float4 xr[8];
    residual8(e, e.part * 32, rsub4, c4, rowoff, rows_left, true, xr);
    float s = 0.f, ss = 0.f;
    for (int g = e.part; g < NG; g += e.nparts) {
      float v[32];
      acc.load32(g * 32, v);
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 b = lds_f32x4_ro(e.svec_s + (g * 32 + j) * 4);
        const float y0 = v[j] + b.x, y1 = v[j + 1] + b.y, y2 = v[j + 2] + b.z, y3 = v[j + 3] + b.w;
        s += (y0 + y1) + (y2 + y3);
        ss += (y0 * y0 + y1 * y1) + (y2 * y2 + y3 * y3);
      }
    }
    if (e.nparts > 1) {
      const uint32_t slot = e.patch_s + e.lane * 8;
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(slot), "f"(s), "f"(ss) : "memory");
      const int q = (int)((e.row0 >> 5) & 3);
      asm volatile("bar.sync %0, %1;" ::"r"(8 + q), "r"(32 * e.nparts) : "memory");
      for (int p = 0; p < e.nparts; ++p) {
        if (p == e.part) continue;
        float ps, pss;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(ps), "=f"(pss) : "r"(slot + (p - e.part) * 4 * e.patch_stride));
        s += ps; ss += pss;
      }
      asm volatile("bar.sync %0, %1;" ::"r"(8 + q), "r"(32 * e.nparts) : "memory");
    }
    if (e.x_own_bar) {
      // column-split pair: the other half of these rows lives in the peer CTA.  Part 0 posts this CTA's sums into the
      // peer's slot with st.async (the store itself completes the peer's mbarrier transaction: no fence, no release
      // arrive), then every warp of the lane quarter waits for the peer's sums in its own slot.
      if (e.part == 0) {
        if (e.lane == 0) mbar_arrive_expect_tx(e.x_own_bar, 32 * 8);
        __syncwarp();
        asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];" ::"r"(e.x_peer_stat + e.lane * 8),
                     "f"(s), "f"(ss), "r"(e.x_peer_bar)
                     : "memory");
      }
      mbar_wait(e.x_own_bar, e.x_parity);   // CTA-scope acquire: the peer's sums arrive in THIS CTA's shared memory through st.async, whose completion the barrier phase carries (as for bulk copies); the cluster-scope wait added an L1 invalidate (CCTL.IVALL) per tile
      float ps, pss;
      asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(ps), "=f"(pss) : "r"(e.x_own_stat + e.lane * 8));
      s += ps; ss += pss;
    }
    float rs[8], ns[8];
    {
      const float mean = s / GC_L;
      const float rstd = rsqrtf(fmaxf(ss / GC_L - mean * mean, 0.f) + eps);
      const float nmr = -mean * rstd;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        rs[it] = __shfl_sync(0xffffffffu, rstd, it * 4 + rsub4);
        ns[it] = __shfl_sync(0xffffffffu, nmr, it * 4 + rsub4);
      }
    }
    const uint32_t r0 = (uint32_t)(e.row0 & 127);
    const int odd = e.lane & 1;
    for (int g = e.part; g < NG; g += e.nparts) {
      const int c = g * 32;
      float4 xn[8];   // next group's residual rows in flight while this group is normalised and stored
      residual8(e, c + 32 * e.nparts, rsub4, c4, rowoff, rows_left, g + e.nparts < NG, xn);
      {
        float v[32];
        acc.load32(c, v);
        patch_put_v(e.patch_s, e.lane, v);
      }
      __syncwarp();
      const float4 bs = lds_f32x4_ro(e.svec_s + (c + c4 * 4) * 4);
      const float4 ga = lds_f32x4_ro(e.svec_s + (e.vstride + c + c4 * 4) * 4);
      const float4 be = lds_f32x4_ro(e.svec_s + (2 * e.vstride + c + c4 * 4) * 4);
      const size_t tile_off = ((size_t)(e.row0 >> 7) * GC_NKB + ((e.n0 + c) >> 6)) * (size_t)G2_A_BYTES + r0 * 128;
      const uint32_t cb = (((uint32_t)c & 63u) >> 3) + (uint32_t)(c4 >> 1);
#pragma unroll
      for (int it2 = 0; it2 < 8; it2 += 2) {
        uint2 hx[2], hy[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int it = it2 + u;
          const int rr = it * 4 + rsub4;
          const float4 t = lds_f32x4(patchv_addr(e.patch_s, rr, c4));
          float4 y;
          y.x = fmaf(fmaf(t.x + bs.x, rs[it], ns[it]), ga.x, be.x); y.y = fmaf(fmaf(t.y + bs.y, rs[it], ns[it]), ga.y, be.y);
          y.z = fmaf(fmaf(t.z + bs.z, rs[it], ns[it]), ga.z, be.z); y.w = fmaf(fmaf(t.w + bs.w, rs[it], ns[it]), ga.w, be.w);
          hy[u].x = pack_half2(y.x, y.y); hy[u].y = pack_half2(y.z, y.w);
          if (kRes) { y.x += xr[it].x; y.y += xr[it].y; y.z += xr[it].z; y.w += xr[it].w; }
          if (xout && rr < rows_left) *reinterpret_cast<float4*>(xout + rowoff + (size_t)rr * GC_L + c) = y;
          hx[u].x = pack_half2(y.x, y.y); hx[u].y = pack_half2(y.z, y.w);
        }
        // even lane assembles the 16-byte chunk of row it2, odd lane the chunk of row it2 + 1
        const int rr = (it2 + odd) * 4 + rsub4;
        const uint32_t coff = rr * 128 + ((cb ^ (uint32_t)(rr & 7)) << 4);
        if (img) {
          const uint2 send = odd ? hx[0] : hx[1];
          uint2 recv;
          recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
          recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
          const uint4 pk = odd ? make_uint4(recv.x, recv.y, hx[1].x, hx[1].y) : make_uint4(hx[0].x, hx[0].y, recv.x, recv.y);
          if (rr < rows_left) *reinterpret_cast<uint4*>(img + tile_off + coff) = pk;
        }
        if (yimg) {
          const uint2 send = odd ? hy[0] : hy[1];
          uint2 recv;
          recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
          recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
          const uint4 pk = odd ? make_uint4(recv.x, recv.y, hy[1].x, hy[1].y) : make_uint4(hy[0].x, hy[0].y, recv.x, recv.y);
          if (rr < rows_left) *reinterpret_cast<uint4*>(yimg + tile_off + coff) = pk;
        }
      }
      __syncwarp();
      if (kRes) {
#pragma unroll
        for (int it = 0; it < 8; ++it) xr[it] = xn[it];
      }
    }
  }
};

// output head: x_out[c][g] = x_in[c][g] + diff_std[c] * (acc[g][c] + bias[c]) for the prognostic channels c < nprog.
// Rows are grid points in state order, so a warp's 32 lanes write 128 contiguous bytes of one channel plane.
struct EpiGcOut {
  static constexpr bool kNeedsBias = false;
  float* xout; const float* xin; const float* bias; const float* dstd; long long plane; int nprog;
  const float* gamma = nullptr; const float* beta = nullptr;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    const long long row = e.row0 + e.lane;
    const bool ok = row < e.M;
    for (int c = e.part * 32; c < BN; c += 32 * e.nparts) {
      if (c >= nprog) break;
      float xi[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) xi[j] = (ok && c + j < nprog) ? __ldg(xin + (size_t)(c + j) * plane + row) : 0.f;
      float v[32];
      acc.load32(c, v);
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (ok && c + j < nprog) xout[(size_t)(c + j) * plane + row] = fmaf(__ldg(dstd + c + j), v[j] + __ldg(bias + c + j), xi[j]);
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------
// set-up kernels (weight / table packing; run once at load)
// ---------------------------------------------------------------------------------------------------------------
// columns [c0, c0 + K) of fp32 W (N rows, leading dimension ldw) -> columns [k_off, k_off + K) of rows [n_off, n_off + N)
// of a weight tile image [Ntot/BN][Kp/64][BN x 128 B].  One 8-half chunk per thread; k_off % 8 == 0; the image is
// zero-initialised by the caller (padding columns / rows).
__global__ void k_gc_pack_w(const float* __restrict__ W, int ldw, int c0, int N, int K, int k_off, int Kp, int BN, int n_off,
                            uint8_t* __restrict__ img) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int cpr = (K + 7) / 8;
  if (idx >= (long long)N * cpr) return;
  const int ns = (int)(idx / cpr), kc = (int)(idx % cpr);
  __half h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kc * 8 + e;
    h[e] = __float2half_rn(k < K ? W[(long long)ns * ldw + c0 + k] : 0.f);
  }
  const int n = n_off + ns, kd = k_off + kc * 8;
  const int nt = n / BN, nr = n % BN, kb = kd / 64, chk = (kd % 64) / 8;
  *reinterpret_cast<uint4*>(img + ((size_t)nt * (Kp / 64) + kb) * (size_t)BN * 128 + sw128_offset(nr, chk)) = *reinterpret_cast<uint4*>(h);
}

// fp32 row-major (rows, F <= 64) -> fp16 tile image with ONE k-block per row tile (static edge / node features)
__global__ void k_gc_pack_rows(const float* __restrict__ src, long long rows, int F, uint8_t* __restrict__ img) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one 8-half chunk each
  if (idx >= rows * 8) return;
  const long long r = idx >> 3; const int chk = (int)(idx & 7);
  __half h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = chk * 8 + e;
    h[e] = __float2half_rn(k < F ? src[r * F + k] : 0.f);
  }
  *reinterpret_cast<uint4*>(img + (size_t)(r >> 7) * G2_A_BYTES + sw128_offset((uint32_t)(r & 127), chk)) = *reinterpret_cast<uint4*>(h);
}

// index tables arrive as fp32 arena entries (every value < 2^24 is exact)
__global__ void k_gc_f2i(const float* __restrict__ src, int* __restrict__ dst, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (int)src[i];
}
// mesh2grid rows are k-major with each segment padded to a whole number of row tiles: row = k * ngp + g
__global__ void k_gc_m2g_index(const float* __restrict__ senders, int* __restrict__ si, int* __restrict__ ri, long long ng, long long ngp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * ngp) return;
  const long long k = i / ngp, g = i % ngp;
  si[i] = g < ng ? (int)senders[k * ng + g] : 0;
  ri[i] = g < ng ? (int)g : 0;
}
// edge features (E, 4) of the k-major mesh2grid rows -> padded rows
__global__ void k_gc_m2g_feat(const float* __restrict__ src, float* __restrict__ dst, long long ng, long long ngp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * ngp) return;
  const long long k = i / ngp, g = i % ngp;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (g < ng) v = *reinterpret_cast<const float4*>(src + (k * ng + g) * 4);
  *reinterpret_cast<float4*>(dst + i * 4) = v;
}

// test tap: fp16 tile image (GC_NKB k-blocks per row tile) -> fp32 row-major (rows, 512)
__global__ void k_gc_img_to_rows(const uint8_t* __restrict__ img, float* __restrict__ out, long long rows) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one 8-column chunk each
  if (idx >= rows * (GC_L / 8)) return;
  const long long r = idx / (GC_L / 8); const int j = (int)(idx % (GC_L / 8));
  const uint4 p = *reinterpret_cast<const uint4*>(img + (size_t)(r >> 7) * GC_NKB * G2_A_BYTES + (size_t)(j >> 3) * G2_A_BYTES +
                                                  sw128_offset((uint32_t)(r & 127), (uint32_t)(j & 7)));
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  add_h8(v, p);
#pragma unroll
  for (int k = 0; k < 8; ++k) out[r * GC_L + j * 8 + k] = v[k];
}

// ---------------------------------------------------------------------------------------------------------------
// per-step kernels
// ---------------------------------------------------------------------------------------------------------------
struct GcClock {        // derived from the device clock once per step (k_gc_clock), read by k_gc_features / k_gc_toa
  float ysin[3], ycos[3], dfrac[3];   // year-progress sin / cos and UTC day fraction at t-6h, t, t+6h
  float sdec, cdec, flux;             // sin / cos of the solar declination and S0 (1 + 0.033 cos g) 3600 at t+6h
};
__device__ __forceinline__ void gc_clock_terms(double t, float& ys, float& yc, float& df) {
  const double days = t / 86400.0;
  const double yp = days / 365.24219;
  const double g = 6.283185307179586 * (yp - floor(yp));
  ys = (float)sin(g); yc = (float)cos(g);
  df = (float)(days - floor(days));
}
__device__ __forceinline__ void gc_solar_terms(double t, float& sdec, float& cdec, float& flux) {
  const double yp = t / 86400.0 / 365.24219;
  const double g = 6.283185307179586 * (yp - floor(yp));
  const double d = 0.4093 * sin(g - 1.405);
  sdec = (float)sin(d); cdec = (float)cos(d);
  flux = (float)(1361.0 * (1.0 + 0.033 * cos(g)) * 3600.0);
}
// clock[0] = valid time of the state's LAST slice (unix seconds).  Derives the step's scalar forcings, then advances
// the clock by dt: the whole step is stream ordered and replayable as a CUDA graph.
__global__ void k_gc_clock(double* clock, GcClock* out, double dt, int advance) {
  if (threadIdx.x || blockIdx.x) return;
  const double t = clock[0];
  GcClock c;
  for (int k = 0; k < 3; ++k) gc_clock_terms(t + (k - 1) * dt, c.ysin[k], c.ycos[k], c.dfrac[k]);
  gc_solar_terms(t + dt, c.sdec, c.cdec, c.flux);
  *out = c;
  if (advance) clock[0] = t + dt;
}
__device__ __forceinline__ float gc_toa(float sdec, float cdec, float flux, float sinlat, float coslat, float dfrac, float lonfrac) {
  float dp = dfrac + lonfrac;
  dp -= floorf(dp);
  const float h = 6.2831853071795865f * dp - 3.14159265358979323846f;
  const float cosz = sinlat * sdec + coslat * cdec * cosf(h);
  return flux * fmaxf(cosz, 0.f);
}
// stand-alone toa field at time t (C-ABI sky_toa_radiation: the host fills the forcing channel of an initial condition)
__global__ void k_gc_toa(float* __restrict__ out, int nlat, int nlon, double t) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nlat * nlon) return;
  const int la = (int)(i / nlon), lo = (int)(i % nlon);
  float sdec, cdec, flux, ys, yc, df;
  gc_solar_terms(t, sdec, cdec, flux);
  gc_clock_terms(t, ys, yc, df);
  const float lat = (90.f - 180.f * (float)la / (float)(nlat - 1)) * 0.017453292519943295f;
  out[i] = gc_toa(sdec, cdec, flux, sinf(lat), cosf(lat), df, (float)lo / (float)nlon);
}

constexpr int GC_FEAT_KP = 192;   // 184 features padded to three k-blocks

// state (2 x n_state planes at t-6h, t) -> grid-node feature image [n_grid/128][3][128 x 128 B]; also writes the two
// slices of the next state that do not depend on the network: x_out[slice 0] = x_in[slice 1], x_out[slice 1][forcing]
// = toa(t+6h).  One CTA = one row tile of 128 consecutive grid points (consecutive in every channel plane: coalesced
// plane reads); the tile is transposed through shared memory and stored as swizzled 16-byte chunks.
__global__ void __launch_bounds__(128) k_gc_features(const float* __restrict__ xin, float* __restrict__ xout, uint8_t* __restrict__ img,
                                                     const float* __restrict__ mean, const float* __restrict__ stdv,
                                                     const float* __restrict__ statics, const GcClock* __restrict__ clk,
                                                     int nlat, int nlon, int nstate, int nprog, int nstatic) {
  constexpr int TS = 186;   // row stride in halves: 93 words (odd) -> conflict-free row-owner writes; 47.6 KB static
  __shared__ __half tile[128][TS];
  __shared__ GcClock c;
  const long long plane = (long long)nlat * nlon;
  const long long g = (long long)blockIdx.x * 128 + threadIdx.x;
  const bool ok = g < plane;
  if (threadIdx.x == 0) c = *clk;
  __syncthreads();
  __half* my = tile[threadIdx.x];
  int f = 0;
  if (ok) {
    // eight independent plane reads in flight per thread (16 warps per SM: latency has to be covered by the thread itself)
    for (int s = 0; s < 2; ++s)
      for (int c0 = 0; c0 < nprog; c0 += 8) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = c0 + j < nprog ? __ldg(xin + (size_t)(s * nstate + c0 + j) * plane + g) : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (c0 + j < nprog) {
            my[f++] = __float2half_rn((v[j] - __ldg(mean + c0 + j)) / __ldg(stdv + c0 + j));
            if (s == 1) xout[(size_t)(c0 + j) * plane + g] = v[j];
          }
      }
    // prognostic channels of slice 0 of the next state come from slice 1 (written above); slice 0 itself is dropped
    const int la = (int)(g / nlon), lo = (int)(g % nlon);
    const float lat = (90.f - 180.f * (float)la / (float)(nlat - 1)) * 0.017453292519943295f;
    const float lonfrac = (float)lo / (float)nlon;
    const float sinlat = sinf(lat), coslat = cosf(lat);
    const float fm = __ldg(mean + nstate - 1), fs = __ldg(stdv + nstate - 1);
    const float toa0 = __ldg(xin + (size_t)(nstate - 1) * plane + g), toa1 = __ldg(xin + (size_t)(2 * nstate - 1) * plane + g);
    const float toa2 = gc_toa(c.sdec, c.cdec, c.flux, sinlat, coslat, c.dfrac[2], lonfrac);
    xout[(size_t)(nstate - 1) * plane + g] = toa1;        // n_state = n_prog + 1: the forcing is the last channel of a slice
    xout[(size_t)(2 * nstate - 1) * plane + g] = toa2;
    my[f++] = __float2half_rn((toa0 - fm) / fs);
    my[f++] = __float2half_rn((toa1 - fm) / fs);
    my[f++] = __float2half_rn((toa2 - fm) / fs);
    for (int k = 0; k < 3; ++k) {
      float dp = c.dfrac[k] + lonfrac;
      dp -= floorf(dp);
      float sn, cs;
      sincosf(6.2831853071795865f * dp, &sn, &cs);
      my[f++] = __float2half_rn(c.ysin[k]); my[f++] = __float2half_rn(c.ycos[k]);
      my[f++] = __float2half_rn(sn); my[f++] = __float2half_rn(cs);
    }
    for (int k = 0; k < nstatic; ++k) my[f++] = __float2half_rn(__ldg(statics + (size_t)k * plane + g));
    float sl, cl;
    sincosf(6.2831853071795865f * lonfrac, &sl, &cl);
    my[f++] = __float2half_rn(coslat); my[f++] = __float2half_rn(sl); my[f++] = __float2half_rn(cl);
  }
  for (; f < TS; ++f) my[f] = __float2half_rn(0.f);
  __syncthreads();
  // 128 rows x 24 chunks of 16 bytes
  uint8_t* dst = img + (size_t)blockIdx.x * (GC_FEAT_KP / 64) * G2_A_BYTES;
  for (int i = threadIdx.x; i < 128 * (GC_FEAT_KP / 8); i += 128) {
    const int r = i / (GC_FEAT_KP / 8), ck = i % (GC_FEAT_KP / 8);
    uint4 pk = make_uint4(0u, 0u, 0u, 0u);
    __half* s = &tile[r][ck * 8];
    if (ck * 8 + 8 <= TS) {
      pk.x = *reinterpret_cast<uint32_t*>(s); pk.y = *reinterpret_cast<uint32_t*>(s + 2);
      pk.z = *reinterpret_cast<uint32_t*>(s + 4); pk.w = *reinterpret_cast<uint32_t*>(s + 6);
    } else if (ck * 8 < TS) {
      pk.x = *reinterpret_cast<uint32_t*>(s);   // columns 184, 185 (zero padding; n_features = 184)
    }
    *reinterpret_cast<uint4*>(dst + (size_t)(ck >> 3) * G2_A_BYTES + sw128_offset((uint32_t)r, (uint32_t)(ck & 7))) = pk;
  }
}

// agg[n] = sum over the incoming edges [ptr[n], ptr[n+1]) of the y image rows -> fp16 tile image; fp32 accumulation in a
// FIXED order (deterministic, no atomics).  The receiver degrees are very uneven (grid2mesh at 0.25 deg: median 29, the
// mesh nodes at the poles 4320), so the segments are cut into chunks of <= GC_SEG_CHUNK edges (table built at load):
// one warp per chunk, a lane owns two 16-byte chunks of the 64 per row, four edges in flight.  A node with a single chunk
// is finished here; the others leave fp32 partial rows that k_gc_segsum_fin adds in chunk order.
constexpr int GC_SEG_CHUNK = 64;
struct GcSegChunk { int node, e0, e1, part; };   // part < 0: single-chunk node; else row of the partial buffer

__device__ __forceinline__ uint4 gc_img_ld(const uint8_t* img, int row, int j) {
  return __ldg(reinterpret_cast<const uint4*>(img + (size_t)(row >> 7) * GC_NKB * G2_A_BYTES + (size_t)(j >> 3) * G2_A_BYTES +
                                              sw128_offset((uint32_t)(row & 127), (uint32_t)(j & 7))));
}
__device__ __forceinline__ void gc_img_st(uint8_t* img, int row, int j, const float* a) {
  uint4 pk;
  pk.x = pack_half2(a[0], a[1]); pk.y = pack_half2(a[2], a[3]); pk.z = pack_half2(a[4], a[5]); pk.w = pack_half2(a[6], a[7]);
  *reinterpret_cast<uint4*>(img + (size_t)(row >> 7) * GC_NKB * G2_A_BYTES + (size_t)(j >> 3) * G2_A_BYTES +
                            sw128_offset((uint32_t)(row & 127), (uint32_t)(j & 7))) = pk;
}
__global__ void __launch_bounds__(256) k_gc_segsum(const uint8_t* __restrict__ yimg, const GcSegChunk* __restrict__ chunks, int n_chunks,
                                                   uint8_t* __restrict__ out, float* __restrict__ partial) {
  const int ci = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (ci >= n_chunks) return;
  const GcSegChunk c = chunks[ci];
  float a[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = 0.f;
  int e = c.e0;
  for (; e + 4 <= c.e1; e += 4) {
    uint4 p[8];
#pragma unroll
    for (int u = 0; u < 4; ++u) { p[2 * u] = gc_img_ld(yimg, e + u, lane); p[2 * u + 1] = gc_img_ld(yimg, e + u, lane + 32); }
#pragma unroll
    for (int u = 0; u < 4; ++u) { add_h8(a, p[2 * u]); add_h8(a + 8, p[2 * u + 1]); }
  }
  for (; e < c.e1; ++e) { add_h8(a, gc_img_ld(yimg, e, lane)); add_h8(a + 8, gc_img_ld(yimg, e, lane + 32)); }
  if (c.part < 0) {
    gc_img_st(out, c.node, lane, a);
    gc_img_st(out, c.node, lane + 32, a + 8);
  } else {
    float* d = partial + (size_t)c.part * GC_L;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      *reinterpret_cast<float4*>(d + (lane + 32 * h) * 8) = make_float4(a[8 * h], a[8 * h + 1], a[8 * h + 2], a[8 * h + 3]);
      *reinterpret_cast<float4*>(d + (lane + 32 * h) * 8 + 4) = make_float4(a[8 * h + 4], a[8 * h + 5], a[8 * h + 6], a[8 * h + 7]);
    }
  }
}
struct GcSegMulti { int node, p0, p1; };   // a node whose segment was cut: partial rows [p0, p1)
__global__ void __launch_bounds__(256) k_gc_segsum_fin(const float* __restrict__ partial, const GcSegMulti* __restrict__ multi, int n_multi,
                                                       uint8_t* __restrict__ out) {
  const int mi = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (mi >= n_multi) return;
  const GcSegMulti m = multi[mi];
  float a[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = 0.f;
  for (int p = m.p0; p < m.p1; ++p) {
    const float* s = partial + (size_t)p * GC_L;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 u = __ldg(reinterpret_cast<const float4*>(s + (lane + 32 * h) * 8));
      const float4 v = __ldg(reinterpret_cast<const float4*>(s + (lane + 32 * h) * 8 + 4));
      a[8 * h] += u.x; a[8 * h + 1] += u.y; a[8 * h + 2] += u.z; a[8 * h + 3] += u.w;
      a[8 * h + 4] += v.x; a[8 * h + 5] += v.y; a[8 * h + 6] += v.z; a[8 * h + 7] += v.w;
    }
  }
  gc_img_st(out, m.node, lane, a);
  gc_img_st(out, m.node, lane + 32, a + 8);
}

}  // namespace sky
