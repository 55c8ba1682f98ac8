// Per-point verification on the device (DESIGN.md section 5): the rank histogram of the truth among the members and the
// per-point score-map accumulators, for the members, channels and truth that sky_forecast_scores reads.
//
// Rank histogram.  At point p of selected channel s, with L = #{x_m < y} and E = #{x_m = y}, the truth's rank is
// L + floor(u (E + 1)) with u = w0 / 2^32 uniform in [0, 1), w0 the first word of Philox4x32-10 at key (seed, date index),
// counter (p, "RNK1", chan[s], lead index): ties are broken at random (Hamill 2001), and the draw is taken only when E > 0
// (floor(u) = 0).  A point's rank depends on nothing but its own values and those four numbers.  Launch 1
// (k_rank_counts): one block per (row, channel) counts the points of the row per rank in shared-memory integer counters,
// plus one counter of NaN points, and writes the row's counts; a row outside every region is not read.  Launch 2
// (k_rank_final): one thread per (region, channel, rank) adds w_r[row] x count over the rows of positive weight in row
// order and divides by nlon.  Integer counts and a fixed row order make the histogram bitwise reproducible, independent
// of the SM count, of the launch geometry and of which other channels or regions are requested.  No atomics on floats.
//
// Score maps.  One thread per (channel, point) holds the members in registers, takes ens_point_terms (point_terms.cuh,
// shared with k_scores_partial) and adds e = xb - y, e^2, var, mae / M and G to the point's five fp64 accumulators, once
// per call: each accumulator sees its terms in call order, so the maps are bitwise reproducible.
//
// The *_multi entries run the same kernels over members pooled from several sources (member_reader.cuh); the Philox
// channel word of a pooled histogram is source 0's plane index of the selected channel.
#include <cmath>

#include "engine.h"
#include "member_fields.h"
#include "member_reader.cuh"
#include "philox.cuh"
#include "point_terms.cuh"
#include "sky_common.cuh"

namespace sky {
namespace {

constexpr int kMapTerms = 5, kRankThreads = 256, kMapThreads = 128;
constexpr uint32_t kRankTag = 0x524E4B31u;   // "RNK1": second Philox counter word (K11 uses 0 there, the GRF "GRF1")

struct PointParams {
  const float* x;              // member m, selected channel s at x + m member_stride + chan[s] plane
  const float* truth;          // [n_sel][plane]
  const double* roww;          // [n_reg][nlat] (histogram only)
  int* counts;                 // [n_sel][nlat][members + 2]: rows' points per rank, then NaN points (histogram only)
  double* out;                 // hist [n_reg][n_sel][members + 1] or maps [n_sel][5][plane]
  long long member_stride;
  int plane, nlat, nlon, members, n_sel, n_reg;
  uint32_t seed, date, lead;
  int chan[kMaxSel];
  static constexpr bool kPooled = false;
  __device__ uint32_t philox_chan(int s) const { return (uint32_t)chan[s]; }
};

// the block of the *_multi entries: the source table, then PointParams' other fields
struct PooledPointParams {
  PooledSources src;
  const float* truth;
  const double* roww;
  int* counts;
  double* out;
  int plane, nlat, nlon, members, n_sel, n_reg;   // members: all sources' together
  uint32_t seed, date, lead;
  static constexpr bool kPooled = true;
  __device__ uint32_t philox_chan(int s) const { return (uint32_t)src.chan[0][s]; }
};
// 2720 bytes: inside the 4 KB every sm_90 launch accepts without the large-parameter path
static_assert(sizeof(PooledPointParams) == 2720, "keep the header comments of the *_multi entries in step");

template <class Params>
__global__ void __launch_bounds__(kRankThreads) k_rank_counts(const __grid_constant__ Params P) {
  const int row = blockIdx.x, s = blockIdx.y, M = P.members, tid = threadIdx.x;
  bool any = false;
  for (int r = 0; r < P.n_reg; ++r) any |= P.roww[r * P.nlat + row] > 0.0;
  if (!any) return;   // the same for the whole block: a row outside every region is not read
  __shared__ int cnt[kMaxMembers + 2];
  __shared__ const float* base[Params::kPooled ? kMaxMembers : 1];
  for (int i = tid; i < M + 2; i += kRankThreads) cnt[i] = 0;
  const auto xs = members_of(P, s, base);   // synchronises the block when pooled
  __syncthreads();
  const long long p0 = (long long)row * P.nlon;
  const float* ys = P.truth + (long long)s * P.plane + p0;
  for (int j = tid; j < P.nlon; j += kRankThreads) {
    const float y = ys[j];
    int lt = 0, eq = 0;
    bool nan = y != y;
#pragma unroll 16
    for (int m = 0; m < M; ++m) {
      const float xm = xs(m, p0 + j);
      lt += xm < y;
      eq += xm == y;
      nan |= xm != xm;
    }
    int bin = M + 1;
    if (!nan) {
      bin = lt;
      if (eq > 0) {
        uint32_t c[4] = {(uint32_t)(p0 + j), kRankTag, P.philox_chan(s), P.lead};
        philox4x32_10(c, P.seed, P.date);
        bin += (int)(((uint64_t)c[0] * (uint32_t)(eq + 1)) >> 32);   // floor(u (E + 1)), u = c0 / 2^32
      }
    }
    atomicAdd(&cnt[bin], 1);
  }
  __syncthreads();
  int* dst = P.counts + ((long long)s * P.nlat + row) * (M + 2);
  for (int i = tid; i < M + 2; i += kRankThreads) dst[i] = cnt[i];
}

template <class Params>
__global__ void __launch_bounds__(kRankThreads) k_rank_final(const __grid_constant__ Params P) {
  const int bins = P.members + 1, i = blockIdx.x * kRankThreads + threadIdx.x;
  if (i >= P.n_reg * P.n_sel * bins) return;
  const int r = i / (P.n_sel * bins), s = i / bins % P.n_sel, k = i % bins;
  const int* c = P.counts + (long long)s * P.nlat * (bins + 1);
  double a = 0.0;
  bool nan = false;
  for (int row = 0; row < P.nlat; ++row, c += bins + 1) {
    const double w = P.roww[r * P.nlat + row];
    if (w > 0.0) {
      a += w * (double)c[k];
      nan |= c[bins] != 0;
    }
  }
  P.out[i] = nan ? __longlong_as_double(0x7ff8000000000000ll) : a / P.nlon;
}

template <class Params, int MP>
__global__ void __launch_bounds__(kMapThreads) k_score_maps(const __grid_constant__ Params P) {
  const int s = blockIdx.y, M = P.members;
  const long long p = (long long)blockIdx.x * kMapThreads + threadIdx.x;
  __shared__ const float* base[Params::kPooled ? kMaxMembers : 1];
  const auto xs = members_of(P, s, base);   // every thread, before any returns
  if (p >= P.plane) return;
  float v[MP];
#pragma unroll
  for (int m = 0; m < MP; ++m) v[m] = m < M ? xs(m, p) : __int_as_float(0x7f800000);
  const float yf = P.truth[(long long)s * P.plane + p];
  const double y = yf;
  const EnsPointTerms q = ens_point_terms(v, M, y, yf != yf);
  const bool nan = q.nan;
  const double e = q.xb - y;
  const double term[kMapTerms] = {e, e * e, q.var, q.mae * (1.0 / M), q.g};
  double* o = P.out + (long long)s * kMapTerms * P.plane + p;
#pragma unroll
  for (int t = 0; t < kMapTerms; ++t) o[t * (long long)P.plane] += nan ? __longlong_as_double(0x7ff8000000000000ll) : term[t];
}

// The histogram of both entries, once P's members are set and checked (x_given: their pointers are not null): the region,
// key, workspace and null-pointer checks (no CUDA call), then member_device(&dev) and the other buffers' device checks.
template <class Params, class MemberDevice>
int run_rank_histogram(Params& P, int nlat, int nlon, int n_sel, const float* truth, const double* row_weights,
                       int n_regions, uint64_t seed, int date_index, int lead_index, int32_t* counts, uint64_t counts_bytes,
                       double* hist, bool x_given, MemberDevice&& member_device, void* stream) {
  const int members = P.members;
  if (n_regions < 1 || n_regions > kMaxRegions) { set_error("n_regions = %d must lie in [1, %d]", n_regions, kMaxRegions); return SKY_ERR_ARG; }
  if (seed > UINT32_MAX) { set_error("seed = %llu must lie in [0, 2^32)", (unsigned long long)seed); return SKY_ERR_ARG; }
  if (date_index < 0 || lead_index < 0) {
    set_error("date_index = %d and lead_index = %d must not be negative", date_index, lead_index);
    return SKY_ERR_ARG;
  }
  const uint64_t need = (uint64_t)n_sel * nlat * (members + 2) * sizeof(int32_t);
  if (counts_bytes < need) {
    set_error("counts_bytes = %llu is below %llu (n_sel x nlat x (members + 2) int32)", (unsigned long long)counts_bytes,
              (unsigned long long)need);
    return SKY_ERR_ARG;
  }
  if (!x_given || !truth || !row_weights || !counts || !hist) {
    set_error("x, truth, row_weights, counts and hist must not be null");
    return SKY_ERR_ARG;
  }
  int dev = -1, rc;
  if ((rc = member_device(&dev)) || (rc = device_of(truth, "truth", &dev)) ||
      (rc = device_of(row_weights, "row_weights", &dev)) || (rc = device_of(counts, "counts", &dev)) ||
      (rc = device_of(hist, "hist", &dev)))
    return rc;
  P.truth = truth;
  P.plane = nlat * nlon;
  P.nlat = nlat;
  P.nlon = nlon;
  P.n_sel = n_sel;
  P.roww = row_weights;
  P.counts = counts;
  P.out = hist;
  P.n_reg = n_regions;
  P.seed = (uint32_t)seed;
  P.date = (uint32_t)date_index;
  P.lead = (uint32_t)lead_index;
  DeviceGuard guard(dev);   // launch on the device that owns the members, whatever the caller's current device is
  cudaStream_t st = (cudaStream_t)stream;
  k_rank_counts<<<dim3(nlat, n_sel), kRankThreads, 0, st>>>(P);
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  const int n_out = n_regions * n_sel * (members + 1);
  k_rank_final<<<(n_out + kRankThreads - 1) / kRankThreads, kRankThreads, 0, st>>>(P);
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

// The maps of both entries, as run_rank_histogram
template <class Params, class MemberDevice>
int run_score_maps(Params& P, int nlat, int nlon, int n_sel, const float* truth, double* maps, bool x_given,
                   MemberDevice&& member_device, void* stream) {
  if (!x_given || !truth || !maps) { set_error("x, truth and maps must not be null"); return SKY_ERR_ARG; }
  int dev = -1, rc;
  if ((rc = member_device(&dev)) || (rc = device_of(truth, "truth", &dev)) || (rc = device_of(maps, "maps", &dev)))
    return rc;
  P.truth = truth;
  P.out = maps;
  P.plane = nlat * nlon;
  P.n_sel = n_sel;
  DeviceGuard guard(dev);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)((P.plane + kMapThreads - 1) / kMapThreads), (unsigned)n_sel);
  dispatch_padding<1>(P.members, [&](auto mp) { k_score_maps<Params, mp><<<grid, kMapThreads, 0, st>>>(P); });
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

}  // namespace
}  // namespace sky

using namespace sky;

extern "C" {

int sky_forecast_rank_histogram(const float* x, int32_t members, int64_t member_stride, int32_t nlat, int32_t nlon,
                                int32_t channel_count, const int32_t* channels, int32_t n_sel, const float* truth,
                                const double* row_weights, int32_t n_regions, uint64_t seed, int32_t date_index,
                                int32_t lead_index, int32_t* counts, uint64_t counts_bytes, double* hist, void* stream) {
  PointParams P{};
  int rc;
  if ((rc = check_grid(nlat, nlon)) ||
      (rc = check_members(members, member_stride, (int64_t)nlat * nlon, channel_count, channels, n_sel, P.chan)))
    return rc;
  P.x = x;
  P.member_stride = member_stride;
  P.members = members;
  return run_rank_histogram(P, nlat, nlon, n_sel, truth, row_weights, n_regions, seed, date_index, lead_index, counts,
                            counts_bytes, hist, x != nullptr, [&](int* dev) { return device_of(x, "x", dev); }, stream);
}

int sky_forecast_rank_histogram_multi(int32_t n_sources, const float* const* x, const int32_t* members,
                                      const int64_t* member_stride, const int32_t* channel_count, const int32_t* channels,
                                      int32_t n_sel, int32_t nlat, int32_t nlon, const float* truth,
                                      const double* row_weights, int32_t n_regions, uint64_t seed, int32_t date_index,
                                      int32_t lead_index, int32_t* counts, uint64_t counts_bytes, double* hist,
                                      void* stream) {
  PooledPointParams P{};
  int rc;
  if ((rc = check_grid(nlat, nlon)) ||
      (rc = check_sources(n_sources, x, members, member_stride, channel_count, channels, n_sel, (int64_t)nlat * nlon, P.src,
                          &P.members)))
    return rc;
  return run_rank_histogram(P, nlat, nlon, n_sel, truth, row_weights, n_regions, seed, date_index, lead_index, counts,
                            counts_bytes, hist, true, [&](int* dev) { return sources_device(n_sources, x, dev); }, stream);
}

int sky_forecast_score_maps(const float* x, int32_t members, int64_t member_stride, int32_t nlat, int32_t nlon,
                            int32_t channel_count, const int32_t* channels, int32_t n_sel, const float* truth, double* maps,
                            void* stream) {
  PointParams P{};
  int rc;
  if ((rc = check_grid(nlat, nlon)) ||
      (rc = check_members(members, member_stride, (int64_t)nlat * nlon, channel_count, channels, n_sel, P.chan)))
    return rc;
  P.x = x;
  P.member_stride = member_stride;
  P.members = members;
  return run_score_maps(P, nlat, nlon, n_sel, truth, maps, x != nullptr, [&](int* dev) { return device_of(x, "x", dev); },
                        stream);
}

int sky_forecast_score_maps_multi(int32_t n_sources, const float* const* x, const int32_t* members,
                                  const int64_t* member_stride, const int32_t* channel_count, const int32_t* channels,
                                  int32_t n_sel, int32_t nlat, int32_t nlon, const float* truth, double* maps, void* stream) {
  PooledPointParams P{};
  int rc;
  if ((rc = check_grid(nlat, nlon)) ||
      (rc = check_sources(n_sources, x, members, member_stride, channel_count, channels, n_sel, (int64_t)nlat * nlon, P.src,
                          &P.members)))
    return rc;
  return run_score_maps(P, nlat, nlon, n_sel, truth, maps, true, [&](int* dev) { return sources_device(n_sources, x, dev); },
                        stream);
}

}  // extern "C"
