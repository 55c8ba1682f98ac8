// Spherical Gaussian random field perturbation of an initial condition (DESIGN.md section 5).
//
// For every (member g, channel c) field with sigma_c != 0:
//     a_lm  = s_l z0                    (m = 0)        z0, z1: Box-Muller (fp64) of Philox4x32-10 words 0, 1 with
//           = s_l (z0 + i z1) / sqrt 2  (m > 0)        key = seed, counter = (l | m << 16, "GRF1", c, g)
//     F_m(theta_k) = sum_{l=m..L} Pbar_l^m(cos theta_k) a_lm                     (k_grf_legendre)
//     x[g, c, k, j] += amp sigma_c (F_0 + 2 sum_{m>=1} Re(F_m e^{i m lambda_j}))  (k_grf_longitude)
// which is torch-harmonics' inverse real SHT on the equiangular grid (skyrim_b200/sht.py RealSHT.inverse).  The
// Legendre table comes from the host (sht.legpoly, fp32, triangular in (m, l)); this file contains no Legendre code.
//
// Determinism: a draw depends only on (seed, g, c, l, m); every output is one thread's sequential sum in a fixed order
// (l ascending, then m' = 2m + re/im ascending), and there are no atomics, so a member's field is bitwise the same
// whether it runs alone or in a batch, in any chunk.
#include <algorithm>

#include "engine.h"
#include "philox.cuh"
#include "sky_common.cuh"

namespace sky {
namespace {

constexpr size_t kGrfWsCap = size_t(512) << 20;   // workspace cap: fields are processed in chunks that fit
constexpr uint32_t kGrfTag = 0x47524631u;         // "GRF1": second Philox counter word (K11 uses 0 there)

__host__ __device__ __forceinline__ long long tri_off(int m, int lmax) {   // first (m, l = m) entry of the (m, l) triangle
  return (long long)m * (lmax + 1) - (long long)m * (m - 1) / 2;
}
__host__ __device__ __forceinline__ long long tri_size(int lmax) { return (long long)(lmax + 1) * (lmax + 2) / 2; }
inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// coefficients a[field][tri(m, l)] (float2 re, im) for fields f0 .. f0 + gridDim.x - 1; block = one (field, m)
__global__ void __launch_bounds__(64) k_grf_draw(float2* __restrict__ a, const float* __restrict__ spec_std, uint64_t seed,
                                                 int member0, int channels, int f0, int lmax) {
  const int fl = blockIdx.x, m = blockIdx.y, fg = f0 + fl;
  const uint32_t c = (uint32_t)(fg % channels), g = (uint32_t)(member0 + fg / channels);
  float2* out = a + (long long)fl * tri_size(lmax) + tri_off(m, lmax) - m;
  for (int l = m + threadIdx.x; l <= lmax; l += blockDim.x) {
    uint32_t ctr[4] = {(uint32_t)l | ((uint32_t)m << 16), kGrfTag, c, g};
    philox4x32_10(ctr, (uint32_t)seed, (uint32_t)(seed >> 32));
    const double u0 = ((double)ctr[0] + 0.5) * 2.3283064365386963e-10, u1 = ((double)ctr[1] + 0.5) * 2.3283064365386963e-10;
    const double r = sqrt(-2.0 * log(u0));
    double sn, cs;
    sincos(6.283185307179586 * u1, &sn, &cs);
    const double s = (double)spec_std[l];
    out[l] = m == 0 ? make_float2((float)(s * (r * cs)), 0.f)
                    : make_float2((float)(s * (r * cs) * 0.7071067811865476), (float)(s * (r * sn) * 0.7071067811865476));
  }
}

// (cos, sin)(2 pi j / nlon), j < nlon: the longitude basis is read from here at index (m j) mod nlon, so it has no phase drift
__global__ void k_grf_twiddle(float2* __restrict__ tw, int nlon) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nlon) return;
  double s, c;
  sincospi(2.0 * j / nlon, &s, &c);
  tw[j] = make_float2((float)c, (float)s);
}

// F[field][2m + {0, 1}][k] = sum_{l=m..L} P[m][k][l - m] a[field][tri(m, l)]   (re, im planes)
// grid (lat tiles of 64, field tiles of 32, m); block 256 = 16 field lanes x 16 lat lanes, 2 x 4 complex outputs each
constexpr int LG_F = 32, LG_K = 64, LG_L = 16;
__global__ void __launch_bounds__(256) k_grf_legendre(float* __restrict__ F, const float2* __restrict__ a,
                                                      const float* __restrict__ leg, int fields, int nlat, int lmax) {
  __shared__ float sre[LG_L][LG_F], sim[LG_L][LG_F], sp[LG_L][LG_K + 1];
  const int m = blockIdx.z, k0 = blockIdx.x * LG_K, fb = blockIdx.y * LG_F;
  const int t = threadIdx.x, tf = t >> 4, tk = t & 15;
  const int km = lmax + 1 - m;                                   // degrees l = m .. L
  const long long T = tri_size(lmax), toff = tri_off(m, lmax);
  const float* P = leg + (long long)nlat * toff;                 // P[m] block: nlat rows of km entries
  float re[2][4] = {}, im[2][4] = {};
  for (int l0 = 0; l0 < km; l0 += LG_L) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = t + 256 * r, f = i >> 4, ll = i & 15;
      float2 v = make_float2(0.f, 0.f);
      if (fb + f < fields && l0 + ll < km) v = a[(long long)(fb + f) * T + toff + l0 + ll];
      sre[ll][f] = v.x; sim[ll][f] = v.y;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = t + 256 * r, kk = i >> 4, ll = i & 15;
      sp[ll][kk] = (k0 + kk < nlat && l0 + ll < km) ? P[(long long)(k0 + kk) * km + l0 + ll] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int ll = 0; ll < LG_L; ++ll) {
      float p[4], ar[2], ai[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) p[i] = sp[ll][tk + 16 * i];
#pragma unroll
      for (int j = 0; j < 2; ++j) { ar[j] = sre[ll][tf + 16 * j]; ai[j] = sim[ll][tf + 16 * j]; }
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) { re[j][i] = fmaf(p[i], ar[j], re[j][i]); im[j][i] = fmaf(p[i], ai[j], im[j][i]); }
    }
    __syncthreads();
  }
  const long long plane = (long long)2 * (lmax + 1) * nlat;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int f = fb + tf + 16 * j;
    if (f >= fields) continue;
    float* o = F + f * plane + (long long)2 * m * nlat;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + tk + 16 * i;
      if (k < nlat) { o[k] = re[j][i]; o[nlat + k] = im[j][i]; }
    }
  }
}

// x[row, j] += amp sigma_c sum_{m'} A[row, m'] B[m', j] over the chunk's rows (row = field * nlat + k):
//   A[row, 2m + ri] = F[field][2m + ri][k],  B[2m, j] = w_m cos(2 pi (m j mod nlon) / nlon),
//   B[2m + 1, j] = -w_m sin(...), w_0 = 1 (Im F_0 is ignored, as irfft does), w_m = 2.
// 128 x 128 output tile per block, 16-deep k-steps staged in shared memory, 8 x 8 outputs per thread, the next
// k-step's operands held in registers while the current one is multiplied.  Two blocks per SM (128 registers, with a
// 12-byte spill).
constexpr int LN_M = 128, LN_N = 128, LN_K = 16;
__global__ void __launch_bounds__(256, 2) k_grf_longitude(float* __restrict__ x, const float* __restrict__ F,
                                                       const float2* __restrict__ tw, const float* __restrict__ sigma,
                                                       float amp, int f0, int fields, int channels, int nlat, int nlon,
                                                       int lmax) {
  __shared__ __align__(16) float sa[LN_K][LN_M], sb[LN_K][LN_N];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const long long rows = (long long)fields * nlat;
  const long long r0 = (long long)blockIdx.x * LN_M;
  const int n0 = blockIdx.y * LN_N;
  const int K = 2 * (lmax + 1);
  // operand loads: this thread always stages A row (r0 + t % 128) and B column (n0 + t % 128), k-rows t / 128 + 2 r
  const int lr = t & 127, lk = t >> 7;
  const long long arow = r0 + lr;
  const bool a_ok = arow < rows;
  const float* ap = F;
  if (a_ok) {
    const long long f = arow / nlat;
    ap = F + f * (long long)K * nlat + (arow - f * nlat);
  }
  const int bj = n0 + lr;
  const bool b_ok = bj < nlon;
  // k-row mk = kb + lk + 2r holds order m = kb / 2 + r, so (m bj) mod nlon advances by bj per r and by 8 bj per k-step:
  // kept incrementally, without a division in the loop
  const int step = (int)((long long)(LN_K / 2) * bj % nlon);
  int mj = 0;                                                    // (kb / 2) bj mod nlon
  float ra[LN_K / 2], rb[LN_K / 2];
  auto load = [&](int kb) {
    int idx = mj;
#pragma unroll
    for (int r = 0; r < LN_K / 2; ++r) {
      const int mk = kb + lk + 2 * r;
      ra[r] = (a_ok && mk < K) ? ap[(long long)mk * nlat] : 0.f;
      float b = 0.f;
      if (b_ok && mk < K) {
        const int m = mk >> 1;
        const float2 c = tw[idx];
        b = (mk & 1) ? (m ? -2.f * c.y : 0.f) : (m ? 2.f * c.x : c.x);
      }
      rb[r] = b;
      idx += bj;
      if (idx >= nlon) idx -= nlon;
    }
    mj += step;
    if (mj >= nlon) mj -= nlon;
  };
  float acc[8][8] = {};
  load(0);
  for (int kb = 0; kb < K; kb += LN_K) {
#pragma unroll
    for (int r = 0; r < LN_K / 2; ++r) { sa[lk + 2 * r][lr] = ra[r]; sb[lk + 2 * r][lr] = rb[r]; }
    __syncthreads();
    if (kb + LN_K < K) load(kb + LN_K);
#pragma unroll
    for (int kk = 0; kk < LN_K; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&sa[kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&sa[kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&sb[kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&sb[kk][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* xc = x + (long long)f0 * nlat * nlon;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long row = r0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
    if (row >= rows) continue;
    const int c = (int)((f0 + row / nlat) % channels);
    const float sc = sigma[c];
    if (sc == 0.f) continue;                                     // forcings and static channels stay bit-identical
    const float s = amp * sc;
    float* xr = xc + row * nlon;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
      if (col < nlon) xr[col] += s * acc[i][j];
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
struct GrfLayout {
  long long fields = 0, chunk = 0;
  size_t tw_bytes = 0, a_bytes = 0, f_bytes = 0, total = 0;   // per-chunk regions
};
GrfLayout grf_layout(long long fields, int nlat, int nlon, int lmax) {
  GrfLayout L;
  L.fields = fields;
  L.tw_bytes = align256((size_t)nlon * sizeof(float2));
  const size_t a_field = (size_t)tri_size(lmax) * sizeof(float2), f_field = (size_t)2 * (lmax + 1) * nlat * sizeof(float);
  const size_t per_field = a_field + f_field;
  const long long fit = kGrfWsCap > L.tw_bytes + 512 ? (long long)((kGrfWsCap - L.tw_bytes - 512) / per_field) : 0;
  L.chunk = std::max(1LL, std::min({fields, fit, 65535LL * LG_F}));   // k_grf_legendre: field tiles on grid y
  L.a_bytes = align256(a_field * L.chunk);
  L.f_bytes = align256(f_field * L.chunk);
  L.total = L.tw_bytes + L.a_bytes + L.f_bytes;
  return L;
}

bool grf_shape_ok(int members, int channels, int nlat, int nlon, int lmax) {
  if (members <= 0 || channels <= 0) { set_error("members (%d) and channels (%d) must be positive", members, channels); return false; }
  if ((long long)members * channels > (1 << 24)) { set_error("members x channels = %lld fields is too many", (long long)members * channels); return false; }
  if (lmax < 1 || lmax > 32767) { set_error("lmax = %d must lie in [1, 32767]", lmax); return false; }
  if (nlat < 2 || lmax >= nlat) { set_error("lmax = %d must be below nlat = %d", lmax, nlat); return false; }
  if (nlon < 2 * lmax + 1) { set_error("nlon = %d must be at least 2 lmax + 1 = %d", nlon, 2 * lmax + 1); return false; }
  return true;
}

int launch_draw(float2* a, const float* spec_std, uint64_t seed, int member0, int channels, long long f0, long long n,
                int lmax, cudaStream_t st) {
  k_grf_draw<<<dim3((unsigned)n, lmax + 1), 64, 0, st>>>(a, spec_std, seed, member0, channels, (int)f0, lmax);
  count_launch(1);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace sky

using namespace sky;

extern "C" {

size_t sky_grf_workspace_bytes(int32_t members, int32_t channels, int32_t nlat, int32_t nlon, int32_t lmax) {
  if (!grf_shape_ok(members, channels, nlat, nlon, lmax)) return 0;
  return grf_layout((long long)members * channels, nlat, nlon, lmax).total;
}

int sky_grf_draw(float* coeffs, const float* spec_std, uint64_t seed, int32_t member0, int32_t members, int32_t channels,
                 int32_t lmax, void* stream) {
  if (members <= 0 || channels <= 0 || member0 < 0 || lmax < 1 || lmax > 32767 ||
      (long long)members * channels > (1 << 24)) {
    set_error("bad argument (members %d, channels %d, member0 %d, lmax %d)", members, channels, member0, lmax);
    return SKY_ERR_ARG;
  }
  int dev = -1, rc;
  if ((rc = device_of(coeffs, "coeffs", &dev)) || (rc = device_of(spec_std, "spec_std", &dev))) return rc;
  DeviceGuard guard(dev);
  return launch_draw(reinterpret_cast<float2*>(coeffs), spec_std, seed, member0, channels, 0, (long long)members * channels,
                     lmax, (cudaStream_t)stream);
}

int sky_perturb_ic_grf(float* x, const float* sigma_c, float amp, uint64_t seed, int32_t member0, int32_t members,
                       int32_t channels, int32_t nlat, int32_t nlon, int32_t lmax, const float* spec_std,
                       const float* legendre, void* ws, size_t ws_bytes, void* stream) {
  if (!grf_shape_ok(members, channels, nlat, nlon, lmax)) return SKY_ERR_ARG;
  if (member0 < 0) { set_error("member0 = %d must be non-negative", member0); return SKY_ERR_ARG; }
  const GrfLayout L = grf_layout((long long)members * channels, nlat, nlon, lmax);
  if (ws_bytes < L.total) { set_error("workspace of %zu bytes, %zu needed", ws_bytes, L.total); return SKY_ERR_ARG; }
  int dev = -1, rc;
  if ((rc = device_of(x, "x", &dev)) || (rc = device_of(sigma_c, "sigma_c", &dev)) ||
      (rc = device_of(spec_std, "spec_std", &dev)) || (rc = device_of(legendre, "legendre", &dev)) ||
      (rc = device_of(ws, "workspace", &dev)))
    return rc;
  DeviceGuard guard(dev);   // launch on the device that owns the state, whatever the caller's current device is
  cudaStream_t st = (cudaStream_t)stream;
  char* w = static_cast<char*>(ws);
  float2* tw = reinterpret_cast<float2*>(w);
  float2* a = reinterpret_cast<float2*>(w + L.tw_bytes);
  float* F = reinterpret_cast<float*>(w + L.tw_bytes + L.a_bytes);
  k_grf_twiddle<<<(nlon + 255) / 256, 256, 0, st>>>(tw, nlon);
  count_launch(1);
  SKY_CUDA_OK(cudaGetLastError());
  for (long long f0 = 0; f0 < L.fields; f0 += L.chunk) {
    const long long n = std::min(L.chunk, L.fields - f0);
    if ((rc = launch_draw(a, spec_std, seed, member0, channels, f0, n, lmax, st))) return rc;
    k_grf_legendre<<<dim3((nlat + LG_K - 1) / LG_K, (unsigned)((n + LG_F - 1) / LG_F), lmax + 1), 256, 0, st>>>(
        F, a, legendre, (int)n, nlat, lmax);
    const long long rows = n * nlat;
    k_grf_longitude<<<dim3((unsigned)((rows + LN_M - 1) / LN_M), (nlon + LN_N - 1) / LN_N), 256, 0, st>>>(
        x, F, tw, sigma_c, amp, (int)f0, (int)n, channels, nlat, nlon, lmax);
    count_launch(2);
    SKY_CUDA_OK(cudaGetLastError());
  }
  return SKY_OK;
}

}  // extern "C"
