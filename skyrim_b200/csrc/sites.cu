// Forecasts at sites and their verification against station observations (DESIGN.md section 5).
//
// Site table.  sky_sites_create builds, on the host and in fp64, a 4-entry stencil per site on the equiangular grid
// (rows 90 -> -90 degrees, dphi = 180 / (nlat - 1); columns from 0 degrees, dlam = 360 / nlon):
//   lam' = fmod(lam, 360) (+ 360 if negative), u = lam' / dlam, j = floor(u), b = u - j, j0 = j mod nlon,
//   j1 = (j0 + 1) mod nlon, t = (90 - phi) / dphi;
//   bilinear: i0 = min(floor(t), nlat - 2), a = t - i0, weights ((1-a)(1-b), (1-a) b, a (1-b), a b) on (i0, j0), (i0, j1),
//             (i0 + 1, j0), (i0 + 1, j1);
//   nearest:  (floor(t + 0.5), floor(u + 0.5) mod nlon) with weight 1, the three other entries weight 0.
// Each weight is one rounded operation on rounded operands (no product is added to anything), so the host compiler has
// nothing to contract.  Every index is checked against the plane here, and the table is uploaded once: no index a kernel
// reads comes from anywhere else.  The table stores the stencil as structure of arrays (entry k of site i at k n + i), so
// a warp's loads of one entry are coalesced.
//
// Sampling (k_sample_sites).  One thread per (site, selected channel); it loads its stencil once and, for every member,
// adds w_k x_k in stencil order in fp64 (__dmul_rn / __dadd_rn, no contraction), skipping entries of weight exactly 0
// (they are not read, so a NaN beside a nearest-neighbour site does not leak in), and rounds the sum once to fp32.  The
// output is [members][n_sel][n_sites], sites along threads: the writes are coalesced, and sky_ensemble_stats over it with
// plane = n_sites gives the site statistics.
//
// Scores (k_site_partial, k_site_final).  One thread per (channel, site) reads the site's members, takes ens_point_terms
// (point_terms.cuh) against the observation and forms the six terms 1, e = xb - y, e^2, var, mae / M, G.  A NaN
// observation is missing: the thread adds nothing.  A NaN member at a site with an observation makes terms 1..5 NaN.
// Each thread adds its terms once to the site's fp64 accumulators; the block adds its threads' terms in thread order into
// one partial per (channel, term, block), and launch 2 adds the partials of each (channel, term) in block order.  The
// partial layout depends on n_sites alone, so the sums are bitwise reproducible, and no atomics are used.
#include <algorithm>
#include <cmath>

#include "engine.h"
#include "member_fields.h"
#include "point_terms.cuh"
#include "sky_common.cuh"

struct sky_sites {
  int device;
  int n_sites, nlat, nlon, method;
  int32_t* idx;   // device [4][n_sites] flat plane indices
  double* w;      // device [4][n_sites] weights
};

namespace sky {
namespace {

constexpr int kStencil = 4, kSiteTerms = 6, kThreads = SKY_SITES_THREADS, kMaxSites = 1 << 20;

// the stencil of one site, as the file comment defines it; false if an index falls outside the grid
bool site_stencil(double lat, double lon, int nlat, int nlon, int method, int32_t idx[kStencil], double w[kStencil]) {
  const double dphi = 180.0 / (nlat - 1), dlam = 360.0 / nlon;
  double lp = std::fmod(lon, 360.0);
  if (lp < 0.0) lp += 360.0;
  const double u = lp / dlam, t = (90.0 - lat) / dphi;
  long long i0, j0, j1;
  if (method == SKY_SITES_NEAREST) {
    i0 = (long long)std::floor(t + 0.5);
    j0 = (long long)std::floor(u + 0.5) % nlon;
    if (i0 < 0 || i0 >= nlat || j0 < 0) return false;
    for (int k = 0; k < kStencil; ++k) {
      idx[k] = (int32_t)(i0 * nlon + j0);
      w[k] = k == 0 ? 1.0 : 0.0;
    }
    return true;
  }
  const double jf = std::floor(u), b = u - jf;
  j0 = (long long)jf % nlon;
  j1 = (j0 + 1) % nlon;
  i0 = std::min((long long)std::floor(t), (long long)nlat - 2);
  const double a = t - (double)i0;
  if (i0 < 0 || j0 < 0) return false;
  const long long r0 = i0 * nlon, r1 = (i0 + 1) * nlon;
  idx[0] = (int32_t)(r0 + j0);
  idx[1] = (int32_t)(r0 + j1);
  idx[2] = (int32_t)(r1 + j0);
  idx[3] = (int32_t)(r1 + j1);
  w[0] = (1.0 - a) * (1.0 - b);
  w[1] = (1.0 - a) * b;
  w[2] = a * (1.0 - b);
  w[3] = a * b;
  return true;
}

struct SampleParams {
  const float* x;          // member m, selected channel s at x + m member_stride + chan[s] plane
  const int32_t* idx;
  const double* w;
  float* values;           // [members][n_sel][n_sites]
  long long member_stride;
  int plane, n_sites, members, n_sel;
  int chan[kMaxSel];
};

__global__ void __launch_bounds__(kThreads) k_sample_sites(const __grid_constant__ SampleParams P) {
  const int i = blockIdx.x * kThreads + threadIdx.x, s = blockIdx.y, n = P.n_sites;
  if (i >= n) return;
  int32_t idx[kStencil];
  double w[kStencil];
#pragma unroll
  for (int k = 0; k < kStencil; ++k) {
    idx[k] = P.idx[k * n + i];
    w[k] = P.w[k * n + i];
  }
  const float* xs = P.x + (long long)P.chan[s] * P.plane;
  float* out = P.values + (long long)s * n + i;
  for (int m = 0; m < P.members; ++m) {
    const float* xm = xs + m * P.member_stride;
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < kStencil; ++k)
      if (w[k] != 0.0) acc = __dadd_rn(acc, __dmul_rn(w[k], (double)xm[idx[k]]));
    out[(long long)m * P.n_sel * n] = __double2float_rn(acc);
  }
}

struct ScoreParams {
  const float* values;     // [members][n_sel][n_sites]
  const float* obs;        // [n_sel][n_sites]
  double* acc;             // [n_sel][n_sites][6]
  double* partial;         // [n_sel][6][blocks]
  double* sums;            // [n_sel][6]
  int n_sites, members, n_sel, blocks;
};

template <int MP>
__global__ void __launch_bounds__(kThreads) k_site_partial(const __grid_constant__ ScoreParams P) {
  const int tid = threadIdx.x, b = blockIdx.x, s = blockIdx.y, M = P.members, n = P.n_sites;
  const int i = b * kThreads + tid;
  __shared__ double col[kSiteTerms][kThreads];
  double term[kSiteTerms] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  const float yf = i < n ? P.obs[(long long)s * n + i] : __int_as_float(0x7fc00000);
  if (yf == yf) {   // an observation: a NaN one is missing and adds nothing
    float v[MP];
#pragma unroll
    for (int m = 0; m < MP; ++m) v[m] = m < M ? P.values[((long long)m * P.n_sel + s) * n + i] : __int_as_float(0x7f800000);
    const double y = yf;
    const EnsPointTerms q = ens_point_terms(v, M, y, false);
    const double e = q.xb - y, qnan = __longlong_as_double(0x7ff8000000000000ll);
    term[0] = 1.0;
    term[1] = q.nan ? qnan : e;
    term[2] = q.nan ? qnan : e * e;
    term[3] = q.nan ? qnan : q.var;
    term[4] = q.nan ? qnan : q.mae * (1.0 / M);
    term[5] = q.nan ? qnan : q.g;
    double* a = P.acc + ((long long)s * n + i) * kSiteTerms;
#pragma unroll
    for (int t = 0; t < kSiteTerms; ++t) a[t] += term[t];
  }
#pragma unroll
  for (int t = 0; t < kSiteTerms; ++t) col[t][tid] = term[t];
  __syncthreads();
  if (tid < kSiteTerms) {   // fixed order: thread t adds term t of every thread in thread order
    double a = 0.0;
    for (int k = 0; k < kThreads; ++k) a += col[tid][k];
    P.partial[((long long)s * kSiteTerms + tid) * P.blocks + b] = a;
  }
}

__global__ void __launch_bounds__(kThreads) k_site_final(const __grid_constant__ ScoreParams P) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= P.n_sel * kSiteTerms) return;
  const double* src = P.partial + (long long)i * P.blocks;
  double a = 0.0;
  for (int b = 0; b < P.blocks; ++b) a += src[b];
  P.sums[i] = a;
}

}  // namespace
}  // namespace sky

using namespace sky;

extern "C" {

int sky_sites_create(sky_sites_t** out, const double* lat, const double* lon, int32_t n_sites, int32_t nlat, int32_t nlon,
                     int32_t method, int device) {
  if (!out || !lat || !lon) { set_error("out, lat and lon must not be null"); return SKY_ERR_ARG; }
  *out = nullptr;
  if (n_sites < 1 || n_sites > kMaxSites) { set_error("n_sites = %d must lie in [1, 2^20]", n_sites); return SKY_ERR_ARG; }
  if (nlat < 2 || nlon < 1 || (int64_t)nlat * nlon > INT32_MAX) {
    set_error("nlat = %d must be at least 2 and nlon = %d at least 1, with nlat x nlon < 2^31", nlat, nlon);
    return SKY_ERR_ARG;
  }
  if (method != SKY_SITES_BILINEAR && method != SKY_SITES_NEAREST) {
    set_error("method = %d is neither SKY_SITES_BILINEAR (0) nor SKY_SITES_NEAREST (1)", method);
    return SKY_ERR_ARG;
  }
  std::vector<int32_t> idx((size_t)kStencil * n_sites);
  std::vector<double> w((size_t)kStencil * n_sites);
  for (int i = 0; i < n_sites; ++i) {
    if (!std::isfinite(lat[i]) || !std::isfinite(lon[i]) || lat[i] < -90.0 || lat[i] > 90.0) {
      set_error("site %d at (%g, %g): lat must lie in [-90, 90] and both must be finite", i, lat[i], lon[i]);
      return SKY_ERR_ARG;
    }
    int32_t si[kStencil];
    double sw[kStencil];
    if (!site_stencil(lat[i], lon[i], nlat, nlon, method, si, sw)) {
      set_error("site %d at (%g, %g) falls outside the %d x %d grid", i, lat[i], lon[i], nlat, nlon);
      return SKY_ERR_ARG;
    }
    for (int k = 0; k < kStencil; ++k) {
      if (si[k] < 0 || (int64_t)si[k] >= (int64_t)nlat * nlon) {
        set_error("site %d: stencil index %d outside the plane", i, si[k]);
        return SKY_ERR_ARG;
      }
      idx[(size_t)k * n_sites + i] = si[k];
      w[(size_t)k * n_sites + i] = sw[k];
    }
  }
  DeviceGuard guard(device);
  sky_sites_t* s = new sky_sites_t{device, n_sites, nlat, nlon, method, nullptr, nullptr};
  cudaError_t e = cudaMalloc(&s->idx, idx.size() * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&s->w, w.size() * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(s->idx, idx.data(), idx.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(s->w, w.data(), w.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error("site table upload failed: %s", cudaGetErrorString(e));
    if (s->idx) cudaFree(s->idx);
    if (s->w) cudaFree(s->w);
    delete s;
    return e == cudaErrorMemoryAllocation ? SKY_ERR_NOMEM : SKY_ERR_CUDA;
  }
  *out = s;
  return SKY_OK;
}

int sky_sites_destroy(sky_sites_t* s) {
  if (!s) return SKY_OK;
  DeviceGuard guard(s->device);
  cudaFree(s->idx);
  cudaFree(s->w);
  delete s;
  return SKY_OK;
}

int sky_sample_sites(const sky_sites_t* s, const float* x, int32_t members, int64_t member_stride, int32_t channel_count,
                     const int32_t* channels, int32_t n_sel, float* values, void* stream) {
  if (!s) { set_error("null site table"); return SKY_ERR_ARG; }
  SampleParams P{};
  int rc;
  if ((rc = check_members(members, member_stride, (int64_t)s->nlat * s->nlon, channel_count, channels, n_sel, P.chan)))
    return rc;
  if (!x || !values) { set_error("x and values must not be null"); return SKY_ERR_ARG; }
  int dev = s->device;
  if ((rc = device_of(x, "x", &dev)) || (rc = device_of(values, "values", &dev))) return rc;
  P.x = x;
  P.idx = s->idx;
  P.w = s->w;
  P.values = values;
  P.member_stride = member_stride;
  P.plane = s->nlat * s->nlon;
  P.n_sites = s->n_sites;
  P.members = members;
  P.n_sel = n_sel;
  DeviceGuard guard(dev);
  const dim3 grid((unsigned)((s->n_sites + kThreads - 1) / kThreads), (unsigned)n_sel);
  k_sample_sites<<<grid, kThreads, 0, (cudaStream_t)stream>>>(P);
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

int sky_site_scores(const float* values, int32_t members, int32_t n_sel, int32_t n_sites, const float* obs, double* acc,
                    double* partial, uint64_t partial_bytes, double* sums, void* stream) {
  if (members < 1 || members > kMaxMembers) { set_error("members = %d must lie in [1, %d]", members, kMaxMembers); return SKY_ERR_ARG; }
  if (n_sel < 1 || n_sel > kMaxSel) { set_error("n_sel = %d must lie in [1, %d]", n_sel, kMaxSel); return SKY_ERR_ARG; }
  if (n_sites < 1 || n_sites > kMaxSites) { set_error("n_sites = %d must lie in [1, 2^20]", n_sites); return SKY_ERR_ARG; }
  const int blocks = (n_sites + kThreads - 1) / kThreads;
  const uint64_t need = (uint64_t)n_sel * kSiteTerms * blocks * sizeof(double);
  if (partial_bytes < need) {
    set_error("partial_bytes = %llu is below %llu (n_sel x 6 x ceil(n_sites / %d) doubles)",
              (unsigned long long)partial_bytes, (unsigned long long)need, kThreads);
    return SKY_ERR_ARG;
  }
  if (!values || !obs || !acc || !partial || !sums) {
    set_error("values, obs, acc, partial and sums must not be null");
    return SKY_ERR_ARG;
  }
  int dev = -1, rc;
  if ((rc = device_of(values, "values", &dev)) || (rc = device_of(obs, "obs", &dev)) || (rc = device_of(acc, "acc", &dev)) ||
      (rc = device_of(partial, "partial", &dev)) || (rc = device_of(sums, "sums", &dev)))
    return rc;
  ScoreParams P{values, obs, acc, partial, sums, n_sites, members, n_sel, blocks};
  DeviceGuard guard(dev);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_padding<1>(members, [&](auto mp) { k_site_partial<mp><<<dim3(blocks, n_sel), kThreads, 0, st>>>(P); });
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  k_site_final<<<(n_sel * kSiteTerms + kThreads - 1) / kThreads, kThreads, 0, st>>>(P);
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

}  // extern "C"
