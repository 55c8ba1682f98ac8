// FourCastNet-v2-small SFNO 6-h step operator on sm_90a.  Replaces what Skyrim's FourCastNet-v2
// model (skyrim/core/models/fourcastnet_v2.py) loads (earth2mip fcnv2_sm: torch + torch_harmonics)
// and what models/utils.py steps.  Architecture: SURVEY.md Appendix B,
// free choices in DESIGN.md §2; oracle: oracle/sfno_ref.py.
//
// Every contraction of the step — per-pixel MLPs, the truncated longitude DFT, the Legendre
// transforms (one GEMM per zonal wavenumber m), the per-degree complex channel mixing (one GEMM
// per l) and their inverses — runs on the TMA-fed wgmma GEMM (gemm2.cuh: batched weights; gemm_tb.cuh: table x data) with
// 3-term fp16 splitting (a_hi*w_hi + a_lo*w_hi + a_hi*w_lo, ~22-bit mantissa: single-pass fp16
// misses the 1e-3 budget on this network, DESIGN.md §2).
// The spherical transforms are a chain of four "table x data" GEMMs around the mixing GEMM; the data is always the
// MN-major B operand, read where the previous epilogue wrote it as fp16 hi / lo rows (no fp32 intermediates, no
// transposing pack passes):
//   pixel image [(lat,lon)][c] --DFT per lat--> [m][lat][(ri,c)] --Legendre per m--> [l][m][(ri,c)] --mixing per l-->
//   [m][l][(ro,o)] --inverse Legendre per m--> [lat][(m,ro)][o] --inverse DFT per lat--> fp32 pixel-major [(lat,lon)][o]
// "Pack" kernels remain where a normalisation needs global statistics first (instance norms) and for the state input.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "engine.h"
#include "gemm_tb.cuh"

namespace sky {

static inline int pad_to(int x, int m) { return (x + m - 1) / m * m; }

// ======================================================================================
// generic re-indexing pack: fp32 tensor -> hi / lo fp16 tile images (+ optional fp32 copy)
//   dest element (batch b, row r = r1*R0 + r0, col k), rows < rows_valid, k < k_valid
//   source offset = b*s_b + r1*s_r1 + r0*s_r0 + (k>>1)*s_kh + (k&1)*s_kl
//   value = affine(act(v)):  act: 0 none, 1 GELU ;  affine: y*sc[i] + sh[i], i by aff_mode
//           (0 none, 1 r1, 2 k)
// thread order: digits (chunk, r0, r1, batch) peeled from the linear thread id in the order
// given by `ord` (fastest first) so that the SOURCE side is read coalesced.
// ======================================================================================
struct PackDesc {
  const float* src;
  long long s_b, s_r1, s_r0, s_kh, s_kl;
  int R0, R1, batches;           // rows = R1*R0
  int k_valid, Kp;               // columns, padded columns (multiple of 64)
  int rows_pad;                  // rows per batch in the image (multiple of 128)
  const float* sc; const float* sh; int aff_mode; int act;
  uint8_t* hi; uint8_t* lo;      // images [batch][rows_pad/128][Kp/64][16 KB]
  float* f32; long long f32_ld;  // optional fp32 row-major copy of the transformed values (batch 0 only)
  int ord[4];                    // permutation of {0: chunk, 1: r0, 2: r1, 3: batch}
};

__global__ void __launch_bounds__(256) k_pack_img(PackDesc d, long long total) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int ext[4] = {d.Kp / 8, d.R0, d.R1, d.batches};
  int dig[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int w = d.ord[i];
    dig[w] = (int)(t % ext[w]);
    t /= ext[w];
  }
  const int chunk = dig[0], r0 = dig[1], r1 = dig[2], b = dig[3];
  const long long r = (long long)r1 * d.R0 + r0;
  const long long base = (long long)b * d.s_b + (long long)r1 * d.s_r1 + (long long)r0 * d.s_r0;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = chunk * 8 + e;
    float x = 0.f;
    if (k < d.k_valid) {
      x = d.src[base + (long long)(k >> 1) * d.s_kh + (long long)(k & 1) * d.s_kl];
      if (d.act == 1) x = gelu_erf(x);
      if (d.aff_mode == 1) x = x * d.sc[r1] + d.sh[r1];
      else if (d.aff_mode == 2) x = x * d.sc[k] + d.sh[k];
    }
    v[e] = x;
  }
  if (d.f32 && b == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (chunk * 8 + e < d.k_valid) d.f32[r * d.f32_ld + chunk * 8 + e] = v[e];
  }
  __half h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    h[e] = __float2half_rn(v[e]);
    l[e] = __float2half_rn(v[e] - __half2float(h[e]));
  }
  const int nkb = d.Kp / 64;
  const size_t off = (size_t)b * (d.rows_pad / 128) * nkb * G2_A_BYTES + ((size_t)(r >> 7) * nkb + (chunk >> 3)) * G2_A_BYTES +
                     sw128_offset((uint32_t)(r & 127), chunk & 7);
  *reinterpret_cast<uint4*>(d.hi + off) = *reinterpret_cast<uint4*>(h);
  *reinterpret_cast<uint4*>(d.lo + off) = *reinterpret_cast<uint4*>(l);
}

// Tiled variant for the packs that TRANSPOSE (the source is contiguous along a row index, not along k): a block moves a
// 32 (source-contiguous index d) x 64 (k) tile through shared memory, so the reads are 128-byte coalesced along d and
// every image row receives its 64 k-values as one 128-byte run (hi) + one (lo).  FAST selects which index is d:
//   1 = r0, 2 = r1, 3 = batch, 4 = (batch, r0) combined (r0 fastest; s_b == R0 * s_r0, e.g. (m, re/im))
// The generic kernel above wrote 16-byte chunks 128..2048 bytes apart and ran at ~1.8 TB/s (profiles/r2_sfno.md).
template <int FAST>
__global__ void __launch_bounds__(256) k_pack_tile(PackDesc d, int ext_d, int n_kb) {
  __shared__ float tile[32][65];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int dt = blockIdx.x / n_kb, kb = blockIdx.x % n_kb;
  const int y = blockIdx.y;
  // decode (b, r1, r0) of element dd of this tile
  auto coords = [&](int dd, int& b, int& r1, int& r0) {
    if (FAST == 1) { r0 = dd; r1 = y % d.R1; b = y / d.R1; }
    else if (FAST == 2) { r1 = dd; r0 = y % d.R0; b = y / d.R0; }
    else if (FAST == 3) { b = dd; r0 = y % d.R0; r1 = y / d.R0; }
    else { b = dd / d.R0; r0 = dd % d.R0; r1 = y; }
  };
  {
    const int dd = dt * 32 + tx;
    int b, r1, r0;
    coords(dd, b, r1, r0);
    const long long base = (long long)b * d.s_b + (long long)r1 * d.s_r1 + (long long)r0 * d.s_r0;
    const float a_sc = (d.aff_mode == 1 && dd < ext_d) ? d.sc[r1] : 1.f, a_sh = (d.aff_mode == 1 && dd < ext_d) ? d.sh[r1] : 0.f;
#pragma unroll
    for (int kk = ty; kk < 64; kk += 8) {
      const int k = kb * 64 + kk;
      float x = 0.f;
      if (dd < ext_d && k < d.k_valid) {
        x = __ldg(d.src + base + (long long)(k >> 1) * d.s_kh + (long long)(k & 1) * d.s_kl);
        if (d.act == 1) x = gelu_erf(x);
        if (d.aff_mode == 1) x = x * a_sc + a_sh;
        else if (d.aff_mode == 2) x = x * d.sc[k] + d.sh[k];
      }
      tile[tx][kk] = x;
    }
  }
  __syncthreads();
  {
    const int dv = threadIdx.x >> 3, ch = threadIdx.x & 7;
    const int dd = dt * 32 + dv;
    if (dd >= ext_d) return;
    int b, r1, r0;
    coords(dd, b, r1, r0);
    const long long r = (long long)r1 * d.R0 + r0;
    __half h[8], l[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float v = tile[dv][ch * 8 + e];
      h[e] = __float2half_rn(v);
      l[e] = __float2half_rn(v - __half2float(h[e]));
    }
    const int nkb = d.Kp / 64;
    const size_t off = (size_t)b * (d.rows_pad / 128) * nkb * G2_A_BYTES + ((size_t)(r >> 7) * nkb + kb) * G2_A_BYTES +
                       sw128_offset((uint32_t)(r & 127), ch);
    *reinterpret_cast<uint4*>(d.hi + off) = *reinterpret_cast<uint4*>(h);
    *reinterpret_cast<uint4*>(d.lo + off) = *reinterpret_cast<uint4*>(l);
  }
}

// ======================================================================================
// weights / tables -> split W images  [batch][N/BN][2*Kp/64][BN x 128 B]   ([hi | lo] along K; the GEMM loaders read
// the k-blocks in the order hi, hi, lo against the data's hi, lo, hi: the second pass over hi comes from L2)
//   mode 0: src[b*s_b + n*s_n + k*s_k]            (n < n_valid, k < k_valid)
//   mode 1: complex channel mixing: src = W[l][o][i][2]; row n = (ro, o), col k = (ri, i)  (re/im-major: the spectra
//           are stored as [.., (ri, c)] so that 64 consecutive channels share a 128-byte row):
//           (ro,ri)=(0,0) Wr, (0,1) -Wi, (1,0) Wi, (1,1) Wr
// ======================================================================================
struct WPackDesc {
  const float* src; long long s_b, s_n, s_k;
  int n_valid, k_valid, N, Kp, BN, batches, mode, E;
  uint8_t* img;
  const float* kscale;   // optional per-k factor (an instance-norm scale folded into the weights), mode 0
};
__global__ void __launch_bounds__(256) k_pack_w3(WPackDesc d, long long total) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int cpr = d.Kp / 8;
  const int kc = (int)(t % cpr); t /= cpr;
  const int n = (int)(t % d.N); const int b = (int)(t / d.N);
  __half h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kc * 8 + e;
    float v = 0.f;
    if (n < d.n_valid && k < d.k_valid) {
      if (d.mode == 0) {
        v = d.src[(long long)b * d.s_b + (long long)n * d.s_n + (long long)k * d.s_k];
        if (d.kscale) v *= d.kscale[k];
      } else {
        const int ro = n / d.E, o = n - ro * d.E, ri = k / d.E, i = k - ri * d.E;
        const float* w = d.src + (((long long)b * d.E + o) * d.E + i) * 2;
        v = ro == ri ? w[0] : (ro == 1 ? w[1] : -w[1]);
      }
    }
    h[e] = __float2half_rn(v);
    l[e] = __float2half_rn(v - __half2float(h[e]));
  }
  const int nkb = d.Kp / 64, nkb2 = 2 * nkb;
  const int nt = n / d.BN, nr = n % d.BN, kb = kc / 8, ch = kc % 8;
  const size_t tile_bytes = (size_t)d.BN * 128;
  uint8_t* base = d.img + (size_t)b * (d.N / d.BN) * nkb2 * tile_bytes + (size_t)nt * nkb2 * tile_bytes;
  const uint32_t o = sw128_offset(nr, ch);
  *reinterpret_cast<uint4*>(base + (size_t)kb * tile_bytes + o) = *reinterpret_cast<uint4*>(h);
  *reinterpret_cast<uint4*>(base + (size_t)(nkb + kb) * tile_bytes + o) = *reinterpret_cast<uint4*>(l);
}

// per-column sums of (optionally GELU'd) fp32 [P, E]:  sums[c], sums[E + c]  (instance norm).
// Block = 32 lanes x 8 row-lanes; a lane owns FOUR consecutive columns (128-bit loads: a warp reads 512 contiguous
// bytes of a row), strides over its rows, the 8 partials of a column meet in shared memory, one fp64 atomic per
// (block, column).  E % 4 == 0.
// Grid-changing blocks (first: 721x1440 -> 240x480, last: back): the inner skip acts on residual = iSHT(X), X the block's
// own forward spectrum, and a 1x1 convolution commutes with the (linear, per-channel) inverse transform:
//   iSHT(W_l X) + V iSHT(X) = iSHT((W_l + V) X)
// so V is added to the real part of every degree's mixing matrix once, at load time, and the pixel-space GEMM over the
// output grid (1.04 M pixels for the last block) and the operand pack feeding it disappear.  spec: (l, out, in, re/im).
__global__ void k_fold_inner_into_spec(float* __restrict__ spec, const float* __restrict__ inner, long long total, int EE) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) spec[2 * i] += inner[i % EE];
}

__global__ void __launch_bounds__(256) k_colstats(const float* __restrict__ x, long long P, int E, int act,
                                                  double* __restrict__ sums, int rows_per_block) {
  __shared__ float4 red[2][8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const int c = (blockIdx.x * 32 + cx) * 4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), ss = s;
  if (c < E) {
    long long rend = r0 + rows_per_block;
    if (rend > P) rend = P;
#pragma unroll 4
    for (long long r = r0 + ry; r < rend; r += 8) {
      float4 v = __ldg(reinterpret_cast<const float4*>(x + r * E + c));
      if (act) { v.x = gelu_erf(v.x); v.y = gelu_erf(v.y); v.z = gelu_erf(v.z); v.w = gelu_erf(v.w); }
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      ss.x += v.x * v.x; ss.y += v.y * v.y; ss.z += v.z * v.z; ss.w += v.w * v.w;
    }
  }
  red[0][ry][cx] = s; red[1][ry][cx] = ss;
  __syncthreads();
  if (ry == 0 && c < E) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 u = red[0][i][cx], w = red[1][i][cx];
      a.x += u.x; a.y += u.y; a.z += u.z; a.w += u.w; b.x += w.x; b.y += w.y; b.z += w.z; b.w += w.w;
    }
    atomicAdd(&sums[c], (double)a.x); atomicAdd(&sums[c + 1], (double)a.y); atomicAdd(&sums[c + 2], (double)a.z); atomicAdd(&sums[c + 3], (double)a.w);
    atomicAdd(&sums[E + c], (double)b.x); atomicAdd(&sums[E + c + 1], (double)b.y); atomicAdd(&sums[E + c + 2], (double)b.z); atomicAdd(&sums[E + c + 3], (double)b.w);
  }
}
// sc = gamma * rstd, sh = beta - mean * sc
__global__ void k_finalize_norm(const double* __restrict__ sums, const float* __restrict__ g,
                                const float* __restrict__ b, float eps, long long P, int E, float* __restrict__ sc,
                                float* __restrict__ sh) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= E) return;
  const double mean = sums[c] / (double)P;
  const double var = fmax(sums[E + c] / (double)P - mean * mean, 0.0);
  const float s = g[c] * (float)(1.0 / sqrt(var + (double)eps));
  sc[c] = s;
  sh[c] = b[c] - (float)mean * s;
}
// bias'[n] = bias[n] + sum_k W[n][k] * shift[k]   (the shift of a folded instance norm); one warp per output
__global__ void k_fold_bias(const float* __restrict__ W, const float* __restrict__ shift, const float* __restrict__ bias,
                            float* __restrict__ out, int N, int K) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (n >= N) return;
  float a = 0.f;
  for (int k = lane; k < K; k += 32) a = fmaf(W[(size_t)n * K + k], shift[k], a);
#pragma unroll
  for (int d = 16; d; d >>= 1) a += __shfl_xor_sync(0xffffffffu, a, d);
  if (lane == 0) out[n] = bias[n] + a;
}
// t1[r] = sum_k T[r][k]  (row sums of a transform table: what the transform makes of a constant field)
__global__ void k_row_sums(const float* __restrict__ T, int rows, int K, float* __restrict__ out) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (r >= rows) return;
  float a = 0.f;
  for (int k = lane; k < K; k += 32) a += T[(size_t)r * K + k];
#pragma unroll
  for (int d = 16; d; d >>= 1) a += __shfl_xor_sync(0xffffffffu, a, d);
  if (lane == 0) out[r] = a;
}
__global__ void k_input_affine(const float* __restrict__ mean, const float* __restrict__ stdv, int C,
                               float* __restrict__ sc, float* __restrict__ sh) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  sc[c] = 1.f / stdv[c];
  sh[c] = -mean[c] / stdv[c];
}

// batched 2-D transpose  in[b][R][C] -> out[b][C][R]  (+= when accumulate)
__global__ void k_transpose(const float* __restrict__ in, float* __restrict__ out, int R, int C, int accumulate) {
  __shared__ float tile[32][33];
  const long long boff = (long long)blockIdx.z * R * C;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < C) ? in[boff + (long long)r * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < C) {
      float* o = out + boff + (long long)c * R + r;
      *o = accumulate ? *o + tile[threadIdx.x][i] : tile[threadIdx.x][i];
    }
  }
}

// decoder output: rows = pixels, cols = channels (< C): state[c][p] = (acc + b[c]) * std[c] + mean[c]
struct EpiStateOut {
  static constexpr bool kNeedsBias = false;
  float* out; long long P; int C; const float* bias; const float* mean; const float* stdv;
  template <int BN, class Acc>
  __device__ void run(Acc& acc, const EpiCtx& e) const {
    const long long row = e.row0 + e.lane;
    for (int c = e.part * 32; c < BN; c += 32 * e.nparts) {
      float v[32];
      acc.load32(c, v);
      if (row < e.M) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int ch = e.n0 + c + j;
          if (ch < C) out[(long long)ch * P + row] = (v[j] + __ldg(bias + ch)) * __ldg(stdv + ch) + __ldg(mean + ch);
        }
      }
    }
  }
};

// ======================================================================================
struct W3 {   // a packed 3-term weight image
  uint8_t* img = nullptr;
  int N = 0, Kp = 0, BN = 0, batches = 1;
  long long batch_stride = 0;  // bytes
};
struct Img2 {  // hi / lo activation images
  uint8_t *hi = nullptr, *lo = nullptr;
  size_t bytes = 0;
};

struct SfnoEngine : Engine {
  sky_sfno_config_t cfg;
  int E, Cin, L, H1, W1, H2, W2, lmax, mmax;
  long long P1, P2;
  std::vector<void*> owned;
  // weights
  W3 enc1, enc2, dec1, dec2;
  // transform tables as A operands (128-row tiles): forward DFT [(m,ri)][lon], forward Legendre [m][l][lat],
  // inverse Legendre [m][lat][l], inverse DFT [lon][(m,ri)]
  W3 tdf_big, tdf_int, tdi_big, tdi_int, tpf_big, tpf_int, tpi_big, tpi_int;
  struct Blk { W3 spec, inner, fc1, fc2; const float *n0g, *n0b, *n1g, *n1b, *inner_b, *fc1_b, *fc2_b, *fc1_w, *inner_w; };
  float *fc1_bs = nullptr, *inner_bs = nullptr;   // biases with a folded norm's shift (rewritten per block and step)
  float *n0_sc = nullptr, *n0_sh = nullptr;       // norm0 scale / shift of the current block (n_sc / n_sh: norm1)
  float *t1_big = nullptr, *t1_int = nullptr;     // row sums of the forward DFT tables
  double* sums0 = nullptr;                        // statistics of the NEXT block's input, gathered by the epilogue that writes it
  std::vector<Blk> blk;
  const float *mean, *stdv, *enc1_b, *enc2_b, *dec1_b, *dec2_b;
  float* pos_pm = nullptr;  // [P1, E]
  float *in_sc, *in_sh, *n_sc, *n_sh;
  double* sums;
  // scratch (engine owned, one member at a time)
  float *X, *Xn, *F1, *Rpm;
  Img2 I_a, I_b, I_in, I_x;   // hidden / GELU'd / input-state / block-input pixel images
  // spectral-chain data images: LI [m][lat][(ri,c)], SI [l][m][(ri,c)], MI / MI2 [m][l][(ro,o)], DI [lat][(m,ro)][o]
  Img2 LI, SI, MI, MI2, DI;
  bool scratch_ready = false;

  SfnoEngine(const sky_sfno_config_t& c, int dev) : cfg(c) {
    device = dev;
    E = c.embed; Cin = c.n_channels; L = c.layers;
    H1 = c.nlat; W1 = c.nlon; H2 = c.nlat / c.scale_factor; W2 = c.nlon / c.scale_factor;
    lmax = H2; mmax = W2 / 2 + 1;
    P1 = (long long)H1 * W1; P2 = (long long)H2 * W2;
  }
  ~SfnoEngine() override { for (void* p : owned) cudaFree(p); }

  template <class T>
  T* dalloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n * sizeof(T) + 256) != cudaSuccess) { set_error("cudaMalloc(%zu) failed", n * sizeof(T)); return nullptr; }
    owned.push_back(p);
    return reinterpret_cast<T*>(p);
  }
  bool img_alloc(Img2& im, size_t bytes) {
    im.bytes = bytes;
    im.hi = dalloc<uint8_t>(bytes); im.lo = dalloc<uint8_t>(bytes);
    if (!im.hi || !im.lo) return false;
    cudaMemset(im.hi, 0, bytes); cudaMemset(im.lo, 0, bytes);
    return true;
  }
  static size_t img_bytes(long long rows, int K, int batches = 1) {
    return (size_t)batches * (size_t)(pad_to((int)rows, 128) / 128) * (pad_to(K, 64) / 64) * G2_A_BYTES;
  }

  // BLOCK_N policies (must match the template dispatch in gemm())
  int bn_point(int N) const { return N % 192 == 0 ? 192 : 64; }
  int bn_small(int N) const { return N >= 240 && N % 240 == 0 ? 240 : (N % 192 == 0 ? 192 : (N % 64 == 0 ? 64 : (N % 32 == 0 ? 32 : 16))); }

  int pack_w(W3& w, const float* src, int mode, int n_valid, int k_valid, int N, int BN, int batches, long long s_b,
             long long s_n, long long s_k, cudaStream_t st) {
    w.N = N; w.Kp = pad_to(k_valid, 64); w.BN = BN; w.batches = batches;
    if (N % BN) { set_error("internal: N=%d not a multiple of BN=%d", N, BN); return SKY_ERR_STATE; }
    w.batch_stride = (long long)N * 2 * w.Kp * 2;   // [hi | lo]
    w.img = dalloc<uint8_t>((size_t)w.batch_stride * batches);
    if (!w.img) return SKY_ERR_NOMEM;
    return fill_w(w, src, mode, n_valid, k_valid, s_b, s_n, s_k, nullptr, st);
  }
  // (re)write the image of an allocated W3; kscale: per-k factor folded into the weights (per step, after the statistics)
  int fill_w(const W3& w, const float* src, int mode, int n_valid, int k_valid, long long s_b, long long s_n, long long s_k,
             const float* kscale, cudaStream_t st) {
    WPackDesc d{src, s_b, s_n, s_k, n_valid, k_valid, w.N, w.Kp, w.BN, w.batches, mode, E, w.img, kscale};
    const long long total = (long long)w.batches * w.N * (w.Kp / 8);
    k_pack_w3<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d, total);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }
  // instance norm folded into the pointwise GEMM that follows it:  W (sc * g + sh) + b = (W diag(sc)) g + (W sh + b)
  int fold_norm(const W3& dst, float* bias_out, const float* Wsrc, const float* bias, int N, int K, const float* sc,
                const float* sh, cudaStream_t st) {
    int rc;
    if ((rc = fill_w(dst, Wsrc, 0, N, K, 0, K, 1, sc, st))) return rc;
    k_fold_bias<<<(N * 32 + 255) / 256, 256, 0, st>>>(Wsrc, sh, bias, bias_out, N, K);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }

  int prepare(cudaStream_t st) override {
    if (E % 64) { set_error("embed must be a multiple of 64"); return SKY_ERR_ARG; }
    int rc;
    // P: transient view into the fp32 arena (repacked below, the arena is freed after prepare); KEEP: persistent copy
#define P(dst, name, cnt) if (!((dst) = param(name, (uint64_t)(cnt)))) return SKY_ERR_ARG;
#define KEEP(dst, name, cnt) if (!((dst) = keep(name, (uint64_t)(cnt), st))) return SKY_ERR_ARG;
    const float *w_e1, *w_e2, *w_d1, *w_d2, *pos, *t;
    KEEP(mean, "norm.mean", Cin); KEEP(stdv, "norm.std", Cin);
    P(w_e1, "enc.fc1.w", (long long)E * Cin); KEEP(enc1_b, "enc.fc1.b", E);
    P(w_e2, "enc.fc2.w", (long long)E * E); KEEP(enc2_b, "enc.fc2.b", E);
    P(pos, "pos_embed", (long long)E * P1);
    P(w_d1, "dec.fc1.w", (long long)E * (E + Cin)); KEEP(dec1_b, "dec.fc1.b", E);
    P(w_d2, "dec.fc2.w", (long long)Cin * E); KEEP(dec2_b, "dec.fc2.b", Cin);
    const int CinP = pad_to(Cin, 64);
    if ((rc = pack_w(enc1, w_e1, 0, E, Cin, E, bn_point(E), 1, 0, Cin, 1, st))) return rc;
    if ((rc = pack_w(enc2, w_e2, 0, E, E, E, bn_point(E), 1, 0, E, 1, st))) return rc;
    // decoder fc1: K = [x (E) | input (Cin -> CinP)] — plain [E, E+Cin] padded works because E % 64 == 0
    if ((rc = pack_w(dec1, w_d1, 0, E, E + Cin, E, bn_point(E), 1, 0, E + Cin, 1, st))) return rc;
    if (dec1.Kp != E + CinP) { set_error("internal: decoder K padding"); return SKY_ERR_STATE; }
    const int NoutP = pad_to(Cin, 16);
    if ((rc = pack_w(dec2, w_d2, 0, Cin, E, NoutP, NoutP, 1, 0, E, 1, st))) return rc;
    // transform tables as A operands (128-row tiles, [hi | hi | lo] along K)
    {
      const int r_dft = pad_to(2 * mmax, 128), r_l = pad_to(lmax, 128);
      t1_big = dalloc<float>(r_dft); t1_int = dalloc<float>(r_dft);
      if (!t1_big || !t1_int) return SKY_ERR_NOMEM;
      P(t, "dft.fwd_big", 2LL * mmax * W1);   // [(m,ri)][lon]
      if ((rc = pack_w(tdf_big, t, 0, 2 * mmax, W1, r_dft, 128, 1, 0, W1, 1, st))) return rc;
      k_row_sums<<<(2 * mmax * 32 + 255) / 256, 256, 0, st>>>(t, 2 * mmax, W1, t1_big);
      P(t, "dft.fwd_int", 2LL * mmax * W2);
      if ((rc = pack_w(tdf_int, t, 0, 2 * mmax, W2, r_dft, 128, 1, 0, W2, 1, st))) return rc;
      k_row_sums<<<(2 * mmax * 32 + 255) / 256, 256, 0, st>>>(t, 2 * mmax, W2, t1_int);
      count_launch(2);
      P(t, "dft.inv_big", 2LL * mmax * W1);   // [lon][(m,ri)]
      if ((rc = pack_w(tdi_big, t, 0, W1, 2 * mmax, pad_to(W1, 128), 128, 1, 0, 2 * mmax, 1, st))) return rc;
      P(t, "dft.inv_int", 2LL * mmax * W2);
      if ((rc = pack_w(tdi_int, t, 0, W2, 2 * mmax, pad_to(W2, 128), 128, 1, 0, 2 * mmax, 1, st))) return rc;
      P(t, "sht.fwd_big", (long long)mmax * lmax * H1);   // [m][l][lat]
      if ((rc = pack_w(tpf_big, t, 0, lmax, H1, r_l, 128, mmax, (long long)lmax * H1, H1, 1, st))) return rc;
      P(t, "sht.fwd_int", (long long)mmax * lmax * H2);
      if ((rc = pack_w(tpf_int, t, 0, lmax, H2, r_l, 128, mmax, (long long)lmax * H2, H2, 1, st))) return rc;
      P(t, "sht.inv_big", (long long)mmax * lmax * H1);   // [m][lat][l]
      if ((rc = pack_w(tpi_big, t, 0, H1, lmax, pad_to(H1, 128), 128, mmax, (long long)lmax * H1, lmax, 1, st))) return rc;
      P(t, "sht.inv_int", (long long)mmax * lmax * H2);
      if ((rc = pack_w(tpi_int, t, 0, H2, lmax, pad_to(H2, 128), 128, mmax, (long long)lmax * H2, lmax, 1, st))) return rc;
    }
    blk.resize(L);
    for (int i = 0; i < L; ++i) {
      Blk& b = blk[i];
      char nm[96];
      auto N = [&](const char* s) { snprintf(nm, sizeof nm, "blk%d.%s", i, s); return nm; };
      const float* w;
      KEEP(b.n0g, N("norm0.g"), E); KEEP(b.n0b, N("norm0.b"), E); KEEP(b.n1g, N("norm1.g"), E); KEEP(b.n1b, N("norm1.b"), E);
      const float* wi;
      P(w, N("spec.w"), (long long)lmax * E * E * 2);
      P(wi, N("inner.w"), (long long)E * E); KEEP(b.inner_b, N("inner.b"), E);
      if ((i == 0) != (i == L - 1)) {   // grid-changing block (run_block: Hi != Ho): inner skip folded into the mixing matrices
        const long long total = (long long)lmax * E * E;
        k_fold_inner_into_spec<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(const_cast<float*>(w), wi, total, E * E);
        count_launch();
        SKY_CUDA_OK(cudaGetLastError());
      } else {   // re-packed every step with norm0's scale folded in (fold_norm): keep the fp32 weights
        KEEP(b.inner_w, N("inner.w"), (long long)E * E);
        if ((rc = pack_w(b.inner, b.inner_w, 0, E, E, E, bn_point(E), 1, 0, E, 1, st))) return rc;
      }
      if ((rc = pack_w(b.spec, w, 1, 2 * E, 2 * E, 2 * E, bn_point(2 * E), lmax, 0, 0, 0, st))) return rc;
      const int Hd = cfg.mlp_ratio * E;
      // fc1 is re-packed every step with norm1's scale folded in (fold_norm): keep the fp32 weights
      KEEP(b.fc1_w, N("fc1.w"), (long long)Hd * E); KEEP(b.fc1_b, N("fc1.b"), Hd);
      if ((rc = pack_w(b.fc1, b.fc1_w, 0, Hd, E, Hd, bn_point(Hd), 1, 0, E, 1, st))) return rc;
      P(w, N("fc2.w"), (long long)E * Hd); KEEP(b.fc2_b, N("fc2.b"), E);
      if ((rc = pack_w(b.fc2, w, 0, E, Hd, E, bn_point(E), 1, 0, Hd, 1, st))) return rc;
    }
#undef P
#undef KEEP
    // positional embedding in pixel-major order
    pos_pm = dalloc<float>((size_t)P1 * E);
    if (!pos_pm) return SKY_ERR_NOMEM;
    {
      dim3 g((unsigned)((P1 + 31) / 32), (unsigned)((E + 31) / 32), 1), bdim(32, 8);
      k_transpose<<<g, bdim, 0, st>>>(pos, pos_pm, E, (int)P1, 0);
      count_launch();
    }
    in_sc = dalloc<float>(512); in_sh = dalloc<float>(512); n_sc = dalloc<float>(E); n_sh = dalloc<float>(E);
    sums = dalloc<double>(2 * E);
    fc1_bs = dalloc<float>((size_t)cfg.mlp_ratio * E); inner_bs = dalloc<float>(E);
    n0_sc = dalloc<float>(E); n0_sh = dalloc<float>(E); sums0 = dalloc<double>(2 * E);
    if (!in_sc || !in_sh || !n_sc || !n_sh || !sums || !fc1_bs || !inner_bs || !n0_sc || !n0_sh || !sums0) return SKY_ERR_NOMEM;
    k_input_affine<<<1, 128, 0, st>>>(mean, stdv, Cin, in_sc, in_sh);
    count_launch();
    // ---- scratch ----
    const size_t Hd = (size_t)cfg.mlp_ratio * E;
    X = dalloc<float>((size_t)P1 * E); Xn = dalloc<float>((size_t)P1 * E);
    F1 = dalloc<float>((size_t)P1 * E);
    Rpm = dalloc<float>((size_t)P1 * E);
    if (!X || !Xn || !F1 || !Rpm) return SKY_ERR_NOMEM;
    // one spare row tile: the last latitude's final k-block of the per-latitude DFT reads (and multiplies by the table's
    // zero padding) up to 63 rows past the grid
    const size_t ab = img_bytes(P1 + 128, (int)Hd);
    if (!img_alloc(I_a, ab) || !img_alloc(I_b, ab)) return SKY_ERR_NOMEM;
    if (!img_alloc(I_in, img_bytes(P1, Cin)) || !img_alloc(I_x, img_bytes(P1 + 128, E))) return SKY_ERR_NOMEM;
    if (!img_alloc(LI, img_bytes(H1, 2 * E, mmax))) return SKY_ERR_NOMEM;
    if (!img_alloc(SI, img_bytes(mmax, 2 * E, lmax))) return SKY_ERR_NOMEM;
    if (!img_alloc(MI, img_bytes(lmax, 2 * E, mmax)) || !img_alloc(MI2, img_bytes(lmax, 2 * E, mmax))) return SKY_ERR_NOMEM;
    if (!img_alloc(DI, img_bytes(2 * mmax, E, H1))) return SKY_ERR_NOMEM;
    SKY_CUDA_OK(cudaGetLastError());
    SKY_CUDA_OK(cudaStreamSynchronize(st));
    scratch_ready = true;
    return 0;
  }

  size_t workspace_bytes(int) const override { return 256; }  // scratch is engine owned

  // ---- helpers -------------------------------------------------------------------------
  int pack(int tag, const float* src, Img2& im, int batches, int R1, int R0, int k_valid, long long s_b, long long s_r1,
           long long s_r0, long long s_kh, long long s_kl, int aff_mode, const float* sc, const float* sh, int act,
           int o0, int o1, int o2, int o3, cudaStream_t st, float* f32 = nullptr, long long f32_ld = 0) {
    PackDesc d;
    d.src = src; d.s_b = s_b; d.s_r1 = s_r1; d.s_r0 = s_r0; d.s_kh = s_kh; d.s_kl = s_kl;
    d.R0 = R0; d.R1 = R1; d.batches = batches; d.k_valid = k_valid; d.Kp = pad_to(k_valid, 64);
    d.rows_pad = pad_to(R1 * R0, 128);
    d.sc = sc; d.sh = sh; d.aff_mode = aff_mode; d.act = act; d.hi = im.hi; d.lo = im.lo; d.f32 = f32; d.f32_ld = f32_ld;
    d.ord[0] = o0; d.ord[1] = o1; d.ord[2] = o2; d.ord[3] = o3;
    const size_t need = (size_t)batches * (d.rows_pad / 128) * (d.Kp / 64) * G2_A_BYTES;
    if (need > im.bytes) { set_error("internal: image buffer too small (%zu > %zu)", need, im.bytes); return SKY_ERR_STATE; }
    const long long total = (long long)batches * R1 * R0 * (d.Kp / 8);
    prof_begin(tag, st);
    // choose the tiled (transposing) kernel when the source is contiguous along a row index rather than along k
    const int n_kb = d.Kp / 64;
    const bool k_contig = s_kh == 2 && s_kl == 1;
    int fast = 0, ext = 0; long long ny = 0;
    if (!k_contig && !f32) {
      if (s_r0 == 1 && R0 >= 32) { fast = 1; ext = R0; ny = (long long)batches * R1; }
      else if (s_r1 == 1 && R1 >= 32) { fast = 2; ext = R1; ny = (long long)batches * R0; }
      else if (s_b == 1 && batches >= 32) { fast = 3; ext = batches; ny = (long long)R1 * R0; }
      else if (s_r0 == 1 && s_b == R0 && batches * R0 >= 32) { fast = 4; ext = batches * R0; ny = R1; }
      if (ny > 65535) fast = 0;
    }
    if (fast) {
      dim3 grid((unsigned)(((ext + 31) / 32) * n_kb), (unsigned)ny);
      switch (fast) {
        case 1: k_pack_tile<1><<<grid, 256, 0, st>>>(d, ext, n_kb); break;
        case 2: k_pack_tile<2><<<grid, 256, 0, st>>>(d, ext, n_kb); break;
        case 3: k_pack_tile<3><<<grid, 256, 0, st>>>(d, ext, n_kb); break;
        default: k_pack_tile<4><<<grid, 256, 0, st>>>(d, ext, n_kb); break;
      }
    } else {
      k_pack_img<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d, total);
    }
    prof_end(tag, st);
    count_launch();
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }

  // D[batch][M, N] (=|+=) [hi|lo|hi](A) * W3^T (+bias)
  template <bool kTri = false, class Epi>
  int gemm_epi(int tag, const Img2& A, int nkbA, long long a_bstride, const Epi& epi, const W3& w, long long M, cudaStream_t st) {
    AOperand a;
    a.add(A.hi, nkbA, a_bstride).add(A.lo, nkbA, a_bstride).add(A.hi, nkbA, a_bstride);
    if (nkbA * 64 != w.Kp) { set_error("internal: K mismatch (A %d vs W %d)", nkbA * 64, w.Kp); return SKY_ERR_STATE; }
    return gemm_op<kTri>(tag, a, epi, w, M, st);
  }
  template <bool kTri = false, class Epi>
  int gemm_op(int tag, const AOperand& a, const Epi& epi, const W3& w, long long M, cudaStream_t st) {
    int rc;
    prof_begin(tag, st);
    count_launch();
    const SchedW<kTri> sc{a, w.img, 3 * w.Kp / 64, w.batch_stride, w.Kp / 64};   // W = [hi | lo], read as hi, hi, lo
#define SKY_BN(bn) case bn: rc = launch_gemm2<bn>(sc, epi, M, w.N, w.batches, num_sms, st); break;
    switch (w.BN) {
      SKY_BN(16) SKY_BN(32) SKY_BN(64) SKY_BN(80) SKY_BN(192) SKY_BN(240) SKY_BN(256)
      default: set_error("internal: unsupported BLOCK_N %d", w.BN); rc = SKY_ERR_STATE;
    }
#undef SKY_BN
    prof_end(tag, st);
    return rc;
  }
  int gemm(int tag, const Img2& A, int K, long long a_bstride_bytes, long long rows_per_batch, float* out, int ldo,
           long long out_bstride, const float* bias, bool accumulate, const W3& w, long long M, cudaStream_t st,
           const float* add = nullptr) {
    const int nkb = pad_to(K, 64) / 64;
    const int mt = pad_to((int)rows_per_batch, 128) / 128;
    if (accumulate) {
      EpiF32Batched<true> e{out, ldo, out_bstride, bias, w.N, add};
      return gemm_epi(tag, A, nkb, a_bstride_bytes, e, w, M, st);
    }
    EpiF32Batched<false> e{out, ldo, out_bstride, bias, w.N, add};
    return gemm_epi(tag, A, nkb, a_bstride_bytes, e, w, M, st);
  }

  // D (+bias, optional GELU) written directly as the hi / lo operand images of the next GEMM (no fp32 round trip, no pack)
  int gemm_to_img(int tag, const Img2& A, int K, long long rows, Img2& out, int Nout, const float* bias, bool gelu,
                  const W3& w, cudaStream_t st) {
    const int nkb = pad_to(K, 64) / 64, mt = pad_to((int)rows, 128) / 128;
    const size_t need = (size_t)mt * (pad_to(Nout, 64) / 64) * G2_A_BYTES;
    if (need > out.bytes || Nout % 64) { set_error("internal: split-image epilogue target (%zu > %zu, N=%d)", need, out.bytes, Nout); return SKY_ERR_STATE; }
    if (gelu) { EpiSplitImg<true> e{out.hi, out.lo, Nout / 64, bias, w.N}; return gemm_epi(tag, A, nkb, 0, e, w, rows, st); }
    EpiSplitImg<false> e{out.hi, out.lo, Nout / 64, bias, w.N};
    return gemm_epi(tag, A, nkb, 0, e, w, rows, st);
  }

  int norm_stats(const float* x, long long P, int act, const float* g, const float* b, cudaStream_t st) {
    prof_begin(KT_SFNO_MISC, st);
    SKY_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * E * sizeof(double), st));
    const int rpb = 256;
    dim3 grid((unsigned)((E / 4 + 31) / 32), (unsigned)((P + rpb - 1) / rpb));
    k_colstats<<<grid, 256, 0, st>>>(x, P, E, act, sums, rpb);
    k_finalize_norm<<<(E + 127) / 128, 128, 0, st>>>(sums, g, b, cfg.eps, P, E, n_sc, n_sh);
    prof_end(KT_SFNO_MISC, st);
    count_launch(2);
    SKY_CUDA_OK(cudaGetLastError());
    return 0;
  }

  // ---- spherical transforms: table x data GEMMs (gemm_tb.cuh) ----
  template <class Epi>
  int gemm_tb(int tag, const W3& T, const BData& B, const Epi& epi, long long M, int N, int batches, cudaStream_t st) {
    int rc;
    prof_begin(tag, st);
    count_launch();
    const SchedTB sc{T.img, T.batches > 1 ? T.batch_stride : 0, B, 3 * T.Kp / 64};
    const int bn = N % 256 == 0 ? 256 : (N % 192 == 0 ? 192 : (N % 128 == 0 ? 128 : 64));
#define SKY_TB(v) case v: rc = launch_gemm2<v>(sc, epi, M, N, batches, num_sms, st); break;
    if (T.N % 128 || T.Kp % 64) { set_error("internal: gemm_tb shape N=%d BN=%d rows=%d Kp=%d", N, bn, T.N, T.Kp); rc = SKY_ERR_STATE; }
    else switch (bn) { SKY_TB(64) SKY_TB(128) SKY_TB(192) default: rc = launch_gemm2<256>(sc, epi, M, N, batches, num_sms, st); }
#undef SKY_TB
    prof_end(tag, st);
    return rc;
  }
  static long long tile_img_bytes(int rows, int K) { return (long long)(pad_to(rows, 128) / 128) * (pad_to(K, 64) / 64) * G2_A_BYTES; }

  // forward SHT of the pixel image D (normalised block input on grid (Hi, Wi)):
  //   per latitude  F[(m,ri)][c] = Tf[(m,ri)][lon] * D[lon][c]            -> LI[m][lat][(ri,c)]
  //   per m         S[l][(ri,c)] = Pf_m[l][lat]  * LI_m[lat][(ri,c)]      -> `to_mixing` as [l][m][(ri,c)] (A images of the
  //                 mixing GEMM) and / or `to_inverse` as [m][l][(ri,c)] (data of an inverse transform: the residual of a
  //                 grid-changing block); the second layout costs a second pass of the (cheap) Legendre GEMM
  int forward_sht(const Img2& D, int Hi, int Wi, const float* csc, const float* csh, Img2* to_mixing, Img2* to_inverse,
                  cudaStream_t st) {
    const bool big = Hi == H1;
    const int n2 = 2 * E;
    int rc;
    const long long li_b = tile_img_bytes(Hi, n2);
    {
      BData bd{D.hi, D.lo, E / 64, Wi, 0};
      // D holds the RAW block input; its instance norm (per-channel affine) is applied behind the linear transform
      EpiSplitRemap e{LI.hi, LI.lo, li_b, n2 / 64, 2, E, 1 << 30, 1, E, 0, csc, csh, big ? t1_big : t1_int};
      if ((rc = gemm_tb(KT_SFNO_SHT, big ? tdf_big : tdf_int, bd, e, 2 * mmax, E, Hi, st))) return rc;
    }
    BData bd{LI.hi, LI.lo, n2 / 64, 0, li_b};
    if (to_mixing) {   // batch' = l (source row), row' = m (source batch)
      EpiSplitRemap e{to_mixing->hi, to_mixing->lo, tile_img_bytes(mmax, n2), n2 / 64, 1, 0, 1 << 30, 1, n2};
      if ((rc = gemm_tb(KT_SFNO_SHT, big ? tpf_big : tpf_int, bd, e, lmax, n2, mmax, st))) return rc;
    }
    if (to_inverse) {
      EpiSplitRemap e{to_inverse->hi, to_inverse->lo, tile_img_bytes(lmax, n2), n2 / 64, 1, 0, 1 << 30, 1, n2, 1};
      if ((rc = gemm_tb(KT_SFNO_SHT, big ? tpf_big : tpf_int, bd, e, lmax, n2, mmax, st))) return rc;
    }
    return 0;
  }

  // inverse SHT of the spectrum image S ([m][l][(ro,o)]) onto grid (Ho, Wo); `e_out` is the epilogue of the last GEMM
  // (batch = latitude, row = longitude, column = channel: fp32 pixel-major store, or GELU + statistics + pixel image)
  //   per m         G[lat][(ro,o)] = Pi_m[lat][l] * S_m[l][(ro,o)]          -> DI[lat][(m,ro)][o]
  //   per latitude  y[lon][o]      = Ti[lon][(m,ro)] * DI_lat[(m,ro)][o]    -> e_out
  template <class EpiOut>
  int inverse_sht(const Img2& S, int Ho, int Wo, const EpiOut& e_out, cudaStream_t st) {
    const bool big = Ho == H1;
    const int n2 = 2 * E;
    int rc;
    const long long di_b = tile_img_bytes(2 * mmax, E);
    {
      BData bd{S.hi, S.lo, n2 / 64, 0, tile_img_bytes(lmax, n2)};
      EpiSplitRemap e{DI.hi, DI.lo, di_b, E / 64, 1, 0, E, 2, n2};
      if ((rc = gemm_tb(KT_SFNO_ISHT, big ? tpi_big : tpi_int, bd, e, Ho, n2, mmax, st))) return rc;
    }
    BData bd{DI.hi, DI.lo, E / 64, 0, di_b};
    return gemm_tb(KT_SFNO_ISHT, big ? tdi_big : tdi_int, bd, e_out, Wo, E, Ho, st);
  }
  EpiF32Batched<false> to_field(float* out_pm, int Wo) const { return EpiF32Batched<false>{out_pm, E, (long long)Wo * E, nullptr, E, nullptr}; }

  int run_block(int i, float*& xin, float*& xout, cudaStream_t st) {
    const Blk& b = blk[i];
    const bool in_big = i == 0, out_big = i == L - 1;
    const int Hi = in_big ? H1 : H2, Wi = in_big ? W1 : W2, Ho = out_big ? H1 : H2, Wo = out_big ? W1 : W2;
    const long long Pi = (long long)Hi * Wi, Po = (long long)Ho * Wo;
    const int n2 = 2 * E, Hd = cfg.mlp_ratio * E;
    int rc;
    // norm0 of the block input: its statistics were gathered by the epilogue that wrote xin (encoder fc2 / previous fc2);
    // the affine is applied behind the forward DFT, inside the inner skip's weights and inside the outer skip's addend
    prof_begin(KT_SFNO_MISC, st);
    k_finalize_norm<<<(E + 127) / 128, 128, 0, st>>>(sums0, b.n0g, b.n0b, cfg.eps, Pi, E, n0_sc, n0_sh);
    count_launch();
    prof_end(KT_SFNO_MISC, st);
    if (Hi == Ho) {
      if ((rc = forward_sht(I_x, Hi, Wi, n0_sc, n0_sh, &SI, nullptr, st))) return rc;
      prof_begin(KT_SFNO_MISC, st);
      rc = fold_norm(b.inner, inner_bs, b.inner_w, b.inner_b, E, E, n0_sc, n0_sh, st);
      prof_end(KT_SFNO_MISC, st);
      if (rc) return rc;
    } else {
      if ((rc = forward_sht(I_x, Hi, Wi, n0_sc, n0_sh, &SI, &MI2, st))) return rc;
      // only the OUTER skip needs the resampled residual as a field; the inner skip lives in the mixing matrices
      if ((rc = inverse_sht(MI2, Ho, Wo, to_field(Rpm, Wo), st))) return rc;
    }
    // spectral channel mixing, one GEMM per degree l: rows m, K = (ri, i); written as the inverse Legendre's data [m][l][(ro,o)]
    {
      EpiSplitRemap e{MI.hi, MI.lo, tile_img_bytes(lmax, n2), n2 / 64, 1, 0, 1 << 30, 1, n2};
      // degree l only has orders m <= l: row tiles past l are skipped (what they would write meets zeros of the inverse
      // Legendre table)
      if ((rc = gemm_epi<true>(KT_SFNO_SPEC, SI, n2 / 64, tile_img_bytes(mmax, n2), e, b.spec, mmax, st))) return rc;
    }
    // g = GELU(iSHT(mixed) + inner_skip(residual) + bias) -> pixel image I_b + norm1 statistics, from the epilogue that
    // produces y (the inner-skip GEMM on an unchanged grid, the inverse DFT when the inner skip is folded)
    SKY_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * E * sizeof(double), st));
    if (Hi == Ho) {
      if ((rc = inverse_sht(MI, Ho, Wo, to_field(F1, Wo), st))) return rc;
      EpiGeluStatsImg e{I_b.hi, I_b.lo, E / 64, inner_bs, F1, E, 0, sums, E};
      if ((rc = gemm_epi(KT_SFNO_MLP, I_x, E / 64, 0, e, b.inner, Po, st))) return rc;
    } else {
      EpiGeluStatsImg e{I_b.hi, I_b.lo, E / 64, b.inner_b, nullptr, E, Wo, sums, E};
      if ((rc = inverse_sht(MI, Ho, Wo, e, st))) return rc;
    }
    // norm1 folded into fc1:  fc1(norm1(g)) = (W1 diag(sc)) g + (W1 sh + b1)
    prof_begin(KT_SFNO_MISC, st);
    k_finalize_norm<<<(E + 127) / 128, 128, 0, st>>>(sums, b.n1g, b.n1b, cfg.eps, Po, E, n_sc, n_sh);
    count_launch();
    if ((rc = fold_norm(b.fc1, fc1_bs, b.fc1_w, b.fc1_b, Hd, E, n_sc, n_sh, st))) return rc;
    prof_end(KT_SFNO_MISC, st);
    // GELU(fc1) goes straight into the operand images of fc2 (I_a: the residual image it held was consumed by the inner skip)
    if ((rc = gemm_to_img(KT_SFNO_MLP, I_b, E, Po, I_a, Hd, fc1_bs, true, b.fc1, st))) return rc;
    // x_out = residual + fc2(...): fp32 state + its pixel image (next block's data / the decoder's input) + the next
    // block's norm0 statistics, all from this epilogue; the residual is norm0(xin) evaluated on the fly (unchanged grid) or
    // the resampled field
    SKY_CUDA_OK(cudaMemsetAsync(sums0, 0, 2 * E * sizeof(double), st));
    {
      const bool same = Hi == Ho;
      EpiF32ImgStats e{i + 1 < L ? xout : nullptr, E, I_x.hi, I_x.lo, E / 64, b.fc2_b, same ? xin : Rpm, same ? n0_sc : nullptr, same ? n0_sh : nullptr,
                       i + 1 < L ? sums0 : nullptr, E};
      if ((rc = gemm_epi(KT_SFNO_MLP, I_a, Hd / 64, 0, e, b.fc2, Po, st))) return rc;
    }
    if (range_guard) {   // fp16 (hi) operand images this block produced: pixel images, hidden image, spectral images
      if ((rc = range_scan(4, I_x.hi, (size_t)(Po / 128) * (E / 64) * G2_A_BYTES, st))) return rc;
      if ((rc = range_scan(4, I_b.hi, (size_t)(Po / 128) * (E / 64) * G2_A_BYTES, st))) return rc;
      if ((rc = range_scan(5, I_a.hi, (size_t)(Po / 128) * (Hd / 64) * G2_A_BYTES, st))) return rc;
      if ((rc = range_scan(6, SI.hi, SI.bytes, st))) return rc;
      if ((rc = range_scan(6, MI.hi, MI.bytes, st))) return rc;
      if ((rc = range_scan(6, LI.hi, (size_t)mmax * tile_img_bytes(Hi, n2), st))) return rc;
      if ((rc = range_scan(6, DI.hi, (size_t)Ho * tile_img_bytes(2 * mmax, E), st))) return rc;
    }
    float* tmp = xin; xin = xout; xout = tmp;
    return 0;
  }

  int step_one(const float* x_in, float* x_out, cudaStream_t st) {
    int rc;
    // encoder
    if ((rc = pack(KT_SFNO_ENC, x_in, I_in, 1, 1, (int)P1, Cin, 0, 0, 1, 2LL * P1, P1, 2, in_sc, in_sh, 0, 1, 0, 2, 3, st))) return rc;
    if ((rc = gemm_to_img(KT_SFNO_ENC, I_in, Cin, P1, I_a, E, enc1_b, true, enc1, st))) return rc;   // GELU(fc1) -> split images
    SKY_CUDA_OK(cudaMemsetAsync(sums0, 0, 2 * E * sizeof(double), st));
    {   // + positional embedding; fp32 state, pixel image and the first block's norm0 statistics from one epilogue
      // (the fp32 copy is only read by an unchanged-grid first block's outer skip, i.e. when there is a single block)
      EpiF32ImgStats e{L > 1 ? nullptr : X, E, I_x.hi, I_x.lo, E / 64, enc2_b, pos_pm, nullptr, nullptr, sums0, E};
      if ((rc = gemm_epi(KT_SFNO_ENC, I_a, E / 64, 0, e, enc2, P1, st))) return rc;
    }
    float *a = X, *b = Xn;
    for (int i = 0; i < L; ++i)
      if ((rc = run_block(i, a, b, st))) return rc;
    // decoder on concat(x, normalised input): x is already there as the last fc2's pixel image
    {
      const int kx = E / 64, ki = pad_to(Cin, 64) / 64;
      const AOperand op = AOperand(I_x.hi, kx).add(I_in.hi, ki).add(I_x.lo, kx).add(I_in.lo, ki).add(I_x.hi, kx).add(I_in.hi, ki);
      EpiSplitImg<true> e{I_b.hi, I_b.lo, E / 64, dec1_b, dec1.N};   // GELU(fc1) -> operand images of fc2
      if ((rc = gemm_op(KT_SFNO_DEC, op, e, dec1, P1, st))) return rc;
    }
    {
      EpiStateOut e{x_out, P1, Cin, dec2_b, mean, stdv};
      if ((rc = gemm_epi(KT_SFNO_DEC, I_b, E / 64, 0, e, dec2, P1, st))) return rc;
    }
    return 0;
  }

  int step(const float* x_in, float* x_out, int B, void*, size_t, cudaStream_t st) override {
    if (!loaded || !scratch_ready) { set_error("weights not loaded"); return SKY_ERR_STATE; }
    for (int m = 0; m < B; ++m) {
      int rc = step_one(x_in + (size_t)m * Cin * P1, x_out + (size_t)m * Cin * P1, st);
      if (rc) return rc;
    }
    return 0;
  }

  int debug_copy(const char* what, float* dst, uint64_t max_floats, void*, int, cudaStream_t st) override {
    if (!strcmp(what, "range")) {
      if (!range_dev || max_floats < 8) { set_error("range guard is off (debug_set range_guard 1) or destination < 8 floats"); return SKY_ERR_STATE; }
      SKY_CUDA_OK(cudaMemcpyAsync(dst, range_dev, 8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
      return 0;
    }
    set_error("unknown debug buffer '%s'", what);
    return SKY_ERR_ARG;
  }
};

Engine* make_sfno_engine(const sky_sfno_config_t& cfg, int device) {
  if (cfg.embed > CTA_STATS_MAX) { set_error("unsupported SFNO shape: embed %d > %d", cfg.embed, CTA_STATS_MAX); return nullptr; }
  if (cfg.embed % 64 || cfg.nlat % cfg.scale_factor == 0 /* nlat = s*h + 1 */ || cfg.nlon % cfg.scale_factor ||
      (cfg.nlon / cfg.scale_factor) % 32 || (cfg.nlat / cfg.scale_factor) % 16 || cfg.n_channels > 128) {
    set_error("unsupported SFNO shape: nlat=%d nlon=%d embed=%d scale=%d", cfg.nlat, cfg.nlon, cfg.embed, cfg.scale_factor);
    return nullptr;
  }
  return new SfnoEngine(cfg, device);
}

}  // namespace sky
