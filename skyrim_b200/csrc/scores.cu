// Forecast verification sums on the device (DESIGN.md section 5; the metrics are formed in skyrim_b200/scores.py).
//
// For members x_1..x_M of one selected channel, truth y, optional climatology k, ensemble mean xb (fp64, summed in member
// order: the unrounded mean of k_ens_stats) and latitude-band regions r with row weights w_r[i], this writes per
// (region, selected channel) the nine fp64 sums over the points p of the plane (row i = p / nlon) with w_r[i] > 0:
//     0  sum w                           1  sum w e,  e = xb - y          2  sum w e^2
//     3  sum w sum_m (x_m - xb)^2        4  sum w (1/M) sum_m |x_m - y|
//     5  sum w G,  G = sum_{m<k} |x_m - x_k| = sum_i (2i - M + 1) (x_(i) - x_(0)) over the sorted values (i from 0)
//     6  sum w f'o'   7  sum w f'^2   8  sum w o'^2,  f' = xb - k, o' = y - k  (NaN without a climatology)
// A NaN member, truth or climatology value at a point makes its terms 1..8 NaN; a region reads no point whose weight in it
// is 0 (a point with weight 0 in every region is not loaded at all).
//
// One thread owns one (channel, point) at a time (U of them per pass, loaded together) and holds its M values in
// registers, padded to MP (8, 16, 32, 64) with +inf, as k_ens_stats does; the mean, var, mae and G come from
// ens_point_terms (point_terms.cuh), which the per-point score maps share.  No atomics.  Launch 1: a fixed grid of
// kBlocks x n_sel blocks; block b takes rows b, b + kBlocks, ... in order, thread j sums the terms of points j,
// j + kThreads, ... of a row, then adds the row's sums, weighted per region, to its running sums; the block adds its
// threads' sums in thread order and writes one partial per (region, channel, term, block).  Launch 2 sums the kBlocks partials of each (region, channel, term) in block order.  The
// partial layout does not depend on the SM count, so the sums are bitwise reproducible and a channel's or a region's sums
// do not depend on the rest of the request.  sky_forecast_scores_multi runs the same kernels over members pooled from
// several sources (member_reader.cuh): only the loads of the members differ.
#include <cmath>

#include "engine.h"
#include "member_fields.h"
#include "member_reader.cuh"
#include "point_terms.cuh"
#include "sky_common.cuh"

namespace sky {
namespace {

constexpr int kTerms = 9, kThreads = 128, kBlocks = SKY_SCORES_BLOCKS;

struct ScoresParams {
  const float* x;              // member m, selected channel s at x + m member_stride + chan[s] plane
  const float* truth;          // [n_sel][plane]
  const float* clim;           // [n_sel][plane] or null
  const double* roww;          // [n_reg][nlat]
  double* partial;             // [n_reg][n_sel][kTerms][kBlocks]
  double* sums;                // [n_reg][n_sel][kTerms]
  long long member_stride;
  int plane, nlat, nlon, members, n_sel, n_reg;
  int chan[kMaxSel];
  static constexpr bool kPooled = false;
};

// sky_forecast_scores_multi's block: the source table, then ScoresParams' other fields
struct PooledScoresParams {
  PooledSources src;
  const float* truth;
  const float* clim;
  const double* roww;
  double* partial;
  double* sums;
  int plane, nlat, nlon, members, n_sel, n_reg;   // members: all sources' together
  static constexpr bool kPooled = true;
};
// 2712 bytes: inside the 4 KB every sm_90 launch accepts without the large-parameter path
static_assert(sizeof(PooledScoresParams) == 2712, "keep the header comment of sky_forecast_scores_multi in step");

template <class Params, int MP, int U>
__global__ void __launch_bounds__(kThreads) k_scores_partial(const __grid_constant__ Params P) {
  const int s = blockIdx.y, b = blockIdx.x, M = P.members, R = P.n_reg, tid = threadIdx.x;
  const double invM = 1.0 / M;
  __shared__ const float* base[Params::kPooled ? kMaxMembers : 1];
  const auto xs = members_of(P, s, base);
  const float* ys = P.truth + (long long)s * P.plane;
  const float* ks = P.clim ? P.clim + (long long)s * P.plane : nullptr;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  // each thread's running sums per (region, term) live in its own shared-memory column: registers hold the members
  __shared__ double acc[kMaxRegions * kTerms][kThreads];
  for (int i = 0; i < R * kTerms; ++i) acc[i][tid] = 0.0;

  for (int row = b; row < P.nlat; row += kBlocks) {
    double w[kMaxRegions];
    bool any = false;
#pragma unroll
    for (int r = 0; r < kMaxRegions; ++r) {
      w[r] = r < R ? P.roww[r * P.nlat + row] : 0.0;
      any |= w[r] > 0.0;
    }
    if (!any) continue;   // a row outside every region is not read
    double ra[kTerms];
#pragma unroll
    for (int t = 0; t < kTerms; ++t) ra[t] = 0.0;
    for (int j0 = tid; j0 < P.nlon; j0 += U * kThreads) {
      // U points per thread per pass: all their loads are issued before the arithmetic of the first one
      float v[U][MP], yf[U], kf[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = j0 + u * kThreads;
        const bool in = j < P.nlon;
        const long long p = (long long)row * P.nlon + (in ? j : 0);
#pragma unroll
        for (int m = 0; m < MP; ++m) v[u][m] = m < M && in ? xs(m, p) : __int_as_float(0x7f800000);
        yf[u] = in ? ys[p] : 0.f;
        kf[u] = in && ks ? ks[p] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (j0 + u * kThreads >= P.nlon) break;
        const double y = yf[u];
        const EnsPointTerms q = ens_point_terms(v[u], M, y, yf[u] != yf[u] || kf[u] != kf[u]);
        const bool nan = q.nan;
        const double xb = q.xb, e = xb - y;
        double term[kTerms];
        term[0] = 1.0;
        term[1] = e;
        term[2] = e * e;
        term[3] = q.var;
        term[4] = q.mae * invM;
        term[5] = q.g;
        if (ks) {
          const double k = kf[u], f = xb - k, o = y - k;
          term[6] = f * o;
          term[7] = f * f;
          term[8] = o * o;
        } else {
          term[6] = term[7] = term[8] = qnan;
        }
#pragma unroll
        for (int t = 0; t < kTerms; ++t) ra[t] += (nan && t > 0) ? qnan : term[t];
      }
    }
#pragma unroll
    for (int r = 0; r < kMaxRegions; ++r)
      if (w[r] > 0.0) {
#pragma unroll
        for (int t = 0; t < kTerms; ++t) acc[r * kTerms + t][tid] += w[r] * ra[t];
      }
  }
  __syncthreads();
  // fixed order: thread i sums column i of every thread in thread order
  if (tid < R * kTerms) {
    double a = 0.0;
    for (int k = 0; k < kThreads; ++k) a += acc[tid][k];
    const int r = tid / kTerms, t = tid % kTerms;
    P.partial[(((long long)r * P.n_sel + s) * kTerms + t) * kBlocks + b] = a;
  }
}

template <class Params>
__global__ void __launch_bounds__(kThreads) k_scores_final(const __grid_constant__ Params P) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= P.n_reg * P.n_sel * kTerms) return;
  const double* src = P.partial + (long long)i * kBlocks;
  double a = 0.0;
  for (int b = 0; b < kBlocks; ++b) a += src[b];
  P.sums[i] = a;
}

// points per thread per pass: enough loads in flight at the occupancy each padding allows
template <int MP, class Params>
void launch(const Params& P, cudaStream_t st) {
  constexpr int U = MP <= 8 ? 4 : MP == 16 ? 2 : 1;
  k_scores_partial<Params, MP, U><<<dim3(kBlocks, P.n_sel), kThreads, 0, st>>>(P);
}

// Both entries, once P's members are set and checked (x_given: the members' pointers are not null): the region, workspace
// and null-pointer checks (no CUDA call), then member_device(&dev) and the device checks of the other buffers, then the
// two launches on the members' device.
template <class Params, class MemberDevice>
int run_scores(Params& P, int nlat, int nlon, int n_sel, const float* truth, const float* clim, const double* row_weights,
               int n_regions, double* partial, uint64_t partial_bytes, double* sums, bool x_given,
               MemberDevice&& member_device, void* stream) {
  if (n_regions < 1 || n_regions > kMaxRegions) { set_error("n_regions = %d must lie in [1, %d]", n_regions, kMaxRegions); return SKY_ERR_ARG; }
  const uint64_t need = (uint64_t)n_regions * n_sel * kTerms * kBlocks * sizeof(double);
  if (partial_bytes < need) {
    set_error("partial_bytes = %llu is below %llu (n_regions x n_sel x 9 x %d doubles)", (unsigned long long)partial_bytes,
              (unsigned long long)need, kBlocks);
    return SKY_ERR_ARG;
  }
  if (!x_given || !truth || !row_weights || !partial || !sums) {
    set_error("x, truth, row_weights, partial and sums must not be null");
    return SKY_ERR_ARG;
  }
  int dev = -1, rc;
  if ((rc = member_device(&dev)) || (rc = device_of(truth, "truth", &dev)) || (clim && (rc = device_of(clim, "clim", &dev))) ||
      (rc = device_of(row_weights, "row_weights", &dev)) || (rc = device_of(partial, "partial", &dev)) ||
      (rc = device_of(sums, "sums", &dev)))
    return rc;
  P.truth = truth;
  P.clim = clim;
  P.roww = row_weights;
  P.partial = partial;
  P.sums = sums;
  P.plane = nlat * nlon;
  P.nlat = nlat;
  P.nlon = nlon;
  P.n_sel = n_sel;
  P.n_reg = n_regions;
  DeviceGuard guard(dev);   // launch on the device that owns the members, whatever the caller's current device is
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_padding<1>(P.members, [&](auto mp) { launch<mp>(P, st); });
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  k_scores_final<<<(n_regions * n_sel * kTerms + kThreads - 1) / kThreads, kThreads, 0, st>>>(P);
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

}  // namespace
}  // namespace sky

using namespace sky;

extern "C" {

int sky_forecast_scores(const float* x, int32_t members, int64_t member_stride, int32_t nlat, int32_t nlon,
                        int32_t channel_count, const int32_t* channels, int32_t n_sel, const float* truth, const float* clim,
                        const double* row_weights, int32_t n_regions, double* partial, uint64_t partial_bytes, double* sums,
                        void* stream) {
  ScoresParams P{};
  int rc;
  if ((rc = check_grid(nlat, nlon)) ||
      (rc = check_members(members, member_stride, (int64_t)nlat * nlon, channel_count, channels, n_sel, P.chan)))
    return rc;
  P.x = x;
  P.member_stride = member_stride;
  P.members = members;
  return run_scores(P, nlat, nlon, n_sel, truth, clim, row_weights, n_regions, partial, partial_bytes, sums, x != nullptr,
                    [&](int* dev) { return device_of(x, "x", dev); }, stream);
}

int sky_forecast_scores_multi(int32_t n_sources, const float* const* x, const int32_t* members, const int64_t* member_stride,
                              const int32_t* channel_count, const int32_t* channels, int32_t n_sel, int32_t nlat,
                              int32_t nlon, const float* truth, const float* clim, const double* row_weights,
                              int32_t n_regions, double* partial, uint64_t partial_bytes, double* sums, void* stream) {
  PooledScoresParams P{};
  int rc;
  if ((rc = check_grid(nlat, nlon)) ||
      (rc = check_sources(n_sources, x, members, member_stride, channel_count, channels, n_sel, (int64_t)nlat * nlon, P.src,
                          &P.members)))
    return rc;
  return run_scores(P, nlat, nlon, n_sel, truth, clim, row_weights, n_regions, partial, partial_bytes, sums, true,
                    [&](int* dev) { return sources_device(n_sources, x, dev); }, stream);
}

}  // extern "C"
