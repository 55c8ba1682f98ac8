// Per-point ensemble verification terms, shared by the forecast scores' weighted sums (scores.cu) and the per-point
// score maps (score_points.cu), so both read the same arithmetic: for the M members of one point, padded to MP with +inf,
//   xb  = (sum_m x_m) / M, summed in member order in fp64 (the unrounded mean of k_ens_stats)
//   var = sum_m (x_m - xb)^2,   mae = sum_m |x_m - y|,   g = G = sum_{m<k} |x_m - x_k| = sum_i (2i - M + 1) (x_(i) - x_(0))
// with var, mae and g taken from the sorted values (bitonic_sort; the M = 1 instantiation does no sort), all in fp64.
// nan is set when a member or one of the caller's inputs (truth, climatology) is NaN.
#pragma once
#include "sort_net.cuh"

namespace sky {

struct EnsPointTerms {
  double xb, var, mae, g;
  bool nan;
};

// v: the point's members in member order, +inf beyond M; sorted on return.  nan: the caller's own inputs are NaN
template <int MP>
__device__ __forceinline__ EnsPointTerms ens_point_terms(float (&v)[MP], int M, double y, bool nan) {
  EnsPointTerms t;
  t.nan = nan;
  double sum = 0.0;
#pragma unroll
  for (int m = 0; m < MP; ++m)
    if (m < M) { sum = __dadd_rn(sum, (double)v[m]); t.nan |= v[m] != v[m]; }
  t.xb = __ddiv_rn(sum, (double)M);
  // the remaining terms do not depend on the member order: take them from the sorted values
  if constexpr (MP > 1) bitonic_sort(v);
  const double lo = v[0];
  double var = 0.0, mae = 0.0, g = 0.0, c = 1.0 - M;
#pragma unroll
  for (int m = 0; m < MP; ++m)
    if (m < M) {
      const double xm = v[m], d = xm - t.xb;
      var += d * d;
      mae += fabs(xm - y);
      g += c * (xm - lo);   // G = sum_i (2i - M + 1) x_(i), shifted by x_(0): no cancellation
      c += 2.0;
    }
  t.var = var;
  t.mae = mae;
  t.g = g;
  return t;
}

}  // namespace sky
