// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants), shared by the two initial-condition perturbations,
// K11's per-grid-point Gaussian noise (sky_abi.cu) and the spherical Gaussian random field (perturb_grf.cu), and by the
// rank histogram's tie-breaking draws (score_points.cu).  The counter layouts never meet, whatever the keys:
//   K11          key seed,                 counter (quad index, its high half = 0 on every grid this project runs, channel,
//                                                   member)
//   GRF          key seed,                 counter (l | m << 16, "GRF1", channel, member)
//   rank ties    key (seed, date index),   counter (point, "RNK1", channel, lead index)
// The second counter word tells them apart: 0, "GRF1" (0x47524631) or "RNK1" (0x524E4B31).
#pragma once
#include <stdint.h>

namespace sky {

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
  uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
  uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
  c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

}  // namespace sky
