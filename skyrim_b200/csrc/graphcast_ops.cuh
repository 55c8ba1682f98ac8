// GraphCast step: device pieces that are not GEMM main loops — the hidden-layer and output-head epilogue functors for
// k_gemm2 (gemm2.cuh), the feature builder, the CSR aggregation and small set-up kernels.  Latent width is fixed at 512
// (GC_L).  The LayerNorm layer of every MLP uses gemm2.cuh's Epi2F32Img on the column-split CTA pairs.
//
// Data layout (per member): every latent matrix (grid nodes, mesh nodes, the three edge sets) is an fp16 tile image
// [rows/128][8][128 x 128 B, SWIZZLE_128B] — byte for byte the A operand of the next GEMM.  Of the three residual streams
// only the mesh nodes keep an fp32 row-major copy; grid nodes and mesh edges are read-modify-written in their images
// (Epi2F32Img<true, 2>).  Per-node first-layer partial products ("tables": v W1_s^T, v W1_r^T) are fp16 row-major and are
// gathered by edge index inside the hidden GEMM's epilogue.
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

#ifndef SKY_GC_EPILOGUES_ONLY   // the GEMM epilogues above are all a test build of the GEMM (gemm_probe.cu) takes
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
constexpr int GC_FEAT_TS = 186;   // halves k_gc_features stages per grid point: the most features a configuration may have

// state (2 x n_state planes at t-6h, t) -> grid-node feature image [n_grid/128][3][128 x 128 B]; also writes the two
// slices of the next state that do not depend on the network: x_out[slice 0] = x_in[slice 1], x_out[slice 1][forcing]
// = toa(t+6h).  One CTA = one row tile of 128 consecutive grid points (consecutive in every channel plane: coalesced
// plane reads); the tile is transposed through shared memory and stored as swizzled 16-byte chunks.
__global__ void __launch_bounds__(128) k_gc_features(const float* __restrict__ xin, float* __restrict__ xout, uint8_t* __restrict__ img,
                                                     const float* __restrict__ mean, const float* __restrict__ stdv,
                                                     const float* __restrict__ statics, const GcClock* __restrict__ clk,
                                                     int nlat, int nlon, int nstate, int nprog, int nstatic) {
  constexpr int TS = GC_FEAT_TS;   // row stride in halves: 93 words (odd) -> conflict-free row-owner writes; 47.6 KB static
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

#endif  // SKY_GC_EPILOGUES_ONLY
}  // namespace sky
