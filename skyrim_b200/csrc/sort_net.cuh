// Ascending in-register sort of MP floats (MP a power of two): a fully unrolled bitonic network, min / max on registers
// only, so v[] stays in registers.  +inf padding sorts behind every finite value.  Shared by the ensemble statistics'
// quantiles (ens_stats.cu) and the CRPS spread term of the forecast scores and score maps (point_terms.cuh).
#pragma once

namespace sky {

template <int MP>
__device__ __forceinline__ void bitonic_sort(float (&v)[MP]) {
  static_assert((MP & (MP - 1)) == 0, "MP must be a power of two");
#pragma unroll
  for (int k = 2; k <= MP; k <<= 1)
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1)
#pragma unroll
      for (int i = 0; i < MP; ++i) {
        const int l = i ^ j;
        if (l > i) {
          const float a = v[i], b = v[l];
          const bool up = (i & k) == 0;
          v[i] = up ? fminf(a, b) : fmaxf(a, b);
          v[l] = up ? fmaxf(a, b) : fminf(a, b);
        }
      }
}

}  // namespace sky
