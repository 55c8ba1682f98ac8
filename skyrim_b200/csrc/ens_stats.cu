// Per-step ensemble statistics of the M members resident on one GPU (DESIGN.md section 5).
//
// For each selected channel c and grid point p, over members m < M (fp64 inside, each output rounded once to fp32):
//     mean      sum_m x_m / M, summed in member order
//     spread    sqrt(sum_m (x_m - mu)^2 / M), mu the unrounded fp64 mean (two passes over the registers: population std)
//     q_j       numpy quantile(method="linear"): h = q_j (M - 1), lo = floor h, hi = min(lo + 1, M - 1), g = h - lo, then
//               numpy's lerp of the sorted x_(lo), x_(hi) (a + (b - a) g, or b - (b - a)(1 - g) when g >= 0.5), unfused
//     P(x > t)  count(x_m > t_e) / M, strict
// A NaN member makes every output at that point NaN.
//
// One thread owns one (channel, point) and holds its M values in registers, padded to MP (8, 16, 32, 64) with +inf; the
// padding is excluded from every statistic and sorts behind the members.  Consecutive threads take consecutive points, so
// each member's load is coalesced.  Quantiles come from a fully unrolled bitonic network (min / max on registers only,
// sort_net.cuh); the QUANT = false instantiation skips it.  No atomics: each output is one thread's fixed-order computation, so results
// are bitwise reproducible and a channel's outputs do not depend on which other channels are selected.
// k_ens_stats_multi pools the members of up to four models (sources) with their own channel layouts and also writes
// each model's own mean; the per-point reduction is the same code.
#include <algorithm>
#include <cmath>

#include "engine.h"
#include "member_fields.h"
#include "sky_common.cuh"
#include "sort_net.cuh"

namespace sky {
namespace {

constexpr int kMaxQ = 8, kMaxEvents = 64, kThreads = 128;

// travels by value (kernel parameter space): the host validates everything before any CUDA call
struct EnsStatsParams {
  const float* x;              // base: member m, selected channel s at x + m member_stride + chan[s] plane
  float* stats;                // [2 + n_q][n_sel][plane]
  float* prob;                 // [n_events][plane]
  long long member_stride, plane;
  int members, n_sel, n_q, n_events;
  int chan[kMaxSel];
  int q_lo[kMaxQ], q_hi[kMaxQ];
  double q_g[kMaxQ];
  int ev_sel[kMaxEvents];
  float ev_thr[kMaxEvents];
};

// sky_ensemble_stats_multi's block: the source table (member_fields.h), then the fields reduce_point reads, with
// EnsStatsParams' names
struct MultiStatsParams {
  PooledSources src;
  float* stats;
  float* prob;
  float* means;                          // [n_src][n_sel][plane], or null
  long long plane;
  int members, n_sel, n_q, n_events;
  int q_lo[kMaxQ], q_hi[kMaxQ];
  double q_g[kMaxQ];
  int ev_sel[kMaxEvents];
  float ev_thr[kMaxEvents];
};
// 3336 bytes: inside the 4 KB every sm_90 launch accepts without the large-parameter path
static_assert(sizeof(MultiStatsParams) == 3336, "keep the header comment of sky_ensemble_stats_multi in step");

// The statistics of one (selected channel s, point p) from its members v[0, M), padded to MP with +inf.  Shared by both
// kernels: P is either parameter block (same field names), v is sorted in place when QUANT.
template <int MP, bool QUANT, class Params>
__device__ __forceinline__ void reduce_point(float (&v)[MP], const Params& P, int s, long long p) {
  const int M = P.members;
  double sum = 0.0;
  bool nan = false;
#pragma unroll
  for (int m = 0; m < MP; ++m)
    if (m < M) { sum = __dadd_rn(sum, (double)v[m]); nan |= v[m] != v[m]; }
  const double mu = __ddiv_rn(sum, (double)M);
  double ss = 0.0;
#pragma unroll
  for (int m = 0; m < MP; ++m)
    if (m < M) { const double d = __dsub_rn((double)v[m], mu); ss = __dadd_rn(ss, __dmul_rn(d, d)); }
  const long long sp = (long long)P.n_sel * P.plane;
  float* out = P.stats + (long long)s * P.plane + p;
  out[0] = (float)mu;
  out[sp] = (float)__dsqrt_rn(__ddiv_rn(ss, (double)M));

  const float qnan = __int_as_float(0x7fc00000);
  for (int e = 0; e < P.n_events; ++e) {
    if (P.ev_sel[e] != s) continue;
    const float t = P.ev_thr[e];
    int cnt = 0;
#pragma unroll
    for (int m = 0; m < MP; ++m) cnt += (m < M && v[m] > t) ? 1 : 0;
    P.prob[(long long)e * P.plane + p] = nan ? qnan : (float)__ddiv_rn((double)cnt, (double)M);
  }

  if constexpr (QUANT) {
    bitonic_sort(v);
    for (int q = 0; q < P.n_q; ++q) {
      const int lo = P.q_lo[q], hi = P.q_hi[q];
      float a = 0.f, b = 0.f;
#pragma unroll
      for (int i = 0; i < MP; ++i) { a = i == lo ? v[i] : a; b = i == hi ? v[i] : b; }
      const double g = P.q_g[q], da = a, db = b, d = __dsub_rn(db, da);
      const double r = g >= 0.5 ? __dsub_rn(db, __dmul_rn(d, __dsub_rn(1.0, g))) : __dadd_rn(da, __dmul_rn(d, g));
      out[(2 + q) * sp] = nan ? qnan : (float)r;
    }
  }
}

template <int MP, bool QUANT>
__global__ void __launch_bounds__(kThreads) k_ens_stats(const __grid_constant__ EnsStatsParams P) {
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= P.plane) return;
  const int s = blockIdx.y, M = P.members;
  const float* xp = P.x + (long long)P.chan[s] * P.plane + p;
  float v[MP];
#pragma unroll
  for (int m = 0; m < MP; ++m) v[m] = m < M ? xp[m * P.member_stride] : __int_as_float(0x7f800000);
  reduce_point<MP, QUANT>(v, P, s, p);
}

// Several sources (models) pooled: member m (source-then-member order) starts at src.member[m], a pointer of the host's
// table, and its selected channel s is the plane src.chan[src.member_src[m]][s] of its own source.  v[] is indexed by unrolled constants
// only, so it stays in registers.  With means set, the mean of each source's own members, summed in member order (the
// arithmetic of k_ens_stats over that source alone), goes to means[k][s][p]; it is taken before reduce_point sorts v.
template <int MP, bool QUANT>
__global__ void __launch_bounds__(kThreads) k_ens_stats_multi(const __grid_constant__ MultiStatsParams P) {
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= P.plane) return;
  const int s = blockIdx.y, M = P.members;
  float v[MP];
#pragma unroll
  for (int m = 0; m < MP; ++m)
    v[m] = m < M ? P.src.member[m][(long long)P.src.chan[P.src.member_src[m]][s] * P.plane + p] : __int_as_float(0x7f800000);
  if (P.means) {
#pragma unroll
    for (int k = 0; k < kMaxSources; ++k) {
      if (k >= P.src.n_src) break;
      double sum = 0.0;
#pragma unroll
      for (int m = 0; m < MP; ++m)
        if (m < M && P.src.member_src[m] == k) sum = __dadd_rn(sum, (double)v[m]);
      P.means[((long long)k * P.n_sel + s) * P.plane + p] = (float)__ddiv_rn(sum, (double)P.src.src_members[k]);
    }
  }
  reduce_point<MP, QUANT>(v, P, s, p);
}

template <int MP>
void launch(const EnsStatsParams& P, dim3 grid, cudaStream_t st) {
  if (P.n_q > 0) k_ens_stats<MP, true><<<grid, kThreads, 0, st>>>(P);
  else k_ens_stats<MP, false><<<grid, kThreads, 0, st>>>(P);
}

template <int MP>
void launch(const MultiStatsParams& P, dim3 grid, cudaStream_t st) {
  if (P.n_q > 0) k_ens_stats_multi<MP, true><<<grid, kThreads, 0, st>>>(P);
  else k_ens_stats_multi<MP, false><<<grid, kThreads, 0, st>>>(P);
}

// quantile positions and events, checked and stored the way both entry points need them
template <class Params>
int set_quantiles_events(Params& P, int members, int n_sel, const double* quantiles, int n_q, const int32_t* event_sel,
                         const float* event_thr, int n_events) {
  if (n_q < 0 || n_q > kMaxQ || (n_q && !quantiles)) { set_error("n_q = %d quantiles must lie in [0, %d]", n_q, kMaxQ); return SKY_ERR_ARG; }
  if (n_events < 0 || n_events > kMaxEvents || (n_events && (!event_sel || !event_thr))) {
    set_error("n_events = %d events must lie in [0, %d]", n_events, kMaxEvents);
    return SKY_ERR_ARG;
  }
  P.n_q = n_q;
  P.n_events = n_events;
  for (int q = 0; q < n_q; ++q) {
    const double v = quantiles[q];
    if (!(v >= 0.0 && v <= 1.0)) { set_error("quantile %g is outside [0, 1]", v); return SKY_ERR_ARG; }
    const double h = (double)(members - 1) * v, lo = std::floor(h);
    P.q_lo[q] = (int)lo;
    P.q_hi[q] = std::min((int)lo + 1, members - 1);
    P.q_g[q] = h - lo;
  }
  for (int e = 0; e < n_events; ++e) {
    if (event_sel[e] < 0 || event_sel[e] >= n_sel) { set_error("event_sel[%d] = %d is outside [0, %d)", e, event_sel[e], n_sel); return SKY_ERR_ARG; }
    if (e > 0 && event_sel[e] < event_sel[e - 1]) { set_error("event_sel decreases at %d", e); return SKY_ERR_ARG; }
    if (!std::isfinite(event_thr[e])) { set_error("event threshold %d is not finite", e); return SKY_ERR_ARG; }
    P.ev_sel[e] = event_sel[e];
    P.ev_thr[e] = event_thr[e];
  }
  return 0;
}

}  // namespace
}  // namespace sky

using namespace sky;

extern "C" {

int sky_ensemble_stats(const float* x, int32_t members, int64_t member_stride, int64_t plane, int32_t channel_count,
                       const int32_t* channels, int32_t n_sel, const double* quantiles, int32_t n_q,
                       const int32_t* event_sel, const float* event_thr, int32_t n_events, float* stats, float* prob,
                       void* stream) {
  EnsStatsParams P{};
  int rc;
  if ((rc = check_members(members, member_stride, plane, channel_count, channels, n_sel, P.chan)) ||
      (rc = set_quantiles_events(P, members, n_sel, quantiles, n_q, event_sel, event_thr, n_events)))
    return rc;
  if (!x || !stats || (n_events && !prob)) { set_error("x, stats and (with events) prob must not be null"); return SKY_ERR_ARG; }
  int dev = -1;
  if ((rc = device_of(x, "x", &dev)) || (rc = device_of(stats, "stats", &dev)) ||
      (n_events && (rc = device_of(prob, "prob", &dev))))
    return rc;
  P.x = x;
  P.stats = stats;
  P.prob = prob;
  P.member_stride = member_stride;
  P.plane = plane;
  P.members = members;
  P.n_sel = n_sel;
  DeviceGuard guard(dev);   // launch on the device that owns the members, whatever the caller's current device is
  const dim3 grid((unsigned)((plane + kThreads - 1) / kThreads), (unsigned)n_sel);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_padding<8>(members, [&](auto mp) { launch<mp>(P, grid, st); });
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

int sky_ensemble_stats_multi(int32_t n_sources, const float* const* x, const int32_t* members, const int64_t* member_stride,
                             const int32_t* channel_count, const int32_t* channels, int32_t n_sel, int64_t plane,
                             const double* quantiles, int32_t n_q, const int32_t* event_sel, const float* event_thr,
                             int32_t n_events, float* stats, float* prob, float* means, void* stream) {
  MultiStatsParams P{};
  int total = 0, rc;
  if ((rc = check_sources(n_sources, x, members, member_stride, channel_count, channels, n_sel, plane, P.src, &total)) ||
      (rc = set_quantiles_events(P, total, n_sel, quantiles, n_q, event_sel, event_thr, n_events)))
    return rc;
  P.plane = plane;
  P.members = total;
  P.n_sel = n_sel;
  if (!stats || (n_events && !prob)) { set_error("stats and (with events) prob must not be null"); return SKY_ERR_ARG; }
  int dev = -1;
  if ((rc = sources_device(n_sources, x, &dev)) || (rc = device_of(stats, "stats", &dev)) || (n_events && (rc = device_of(prob, "prob", &dev))) ||
      (means && (rc = device_of(means, "means", &dev))))
    return rc;
  P.stats = stats;
  P.prob = prob;
  P.means = means;
  DeviceGuard guard(dev);
  const dim3 grid((unsigned)((plane + kThreads - 1) / kThreads), (unsigned)n_sel);
  cudaStream_t st = (cudaStream_t)stream;
  dispatch_padding<8>(total, [&](auto mp) { launch<mp>(P, grid, st); });
  count_launch();
  SKY_CUDA_OK(cudaGetLastError());
  return SKY_OK;
}

}  // extern "C"
