// Token grid of a kernel-level probe case (gemm_probe.cu, pangu_probe.cu; tests only).  A case that names a Pangu
// geometry is refused on the host unless the grid is one the engine's make_geo could build: the index arithmetic of
// the windowing kernels divides by these fields and addresses the window image through them, so an inconsistent grid
// would read or write outside its buffers.
#pragma once
#include <cstdint>

#include "pangu_ops.cuh"

extern "C" {
typedef struct {
  int32_t Z, H, W, C, Hp, nWz, nWh, nWw, T, nWin, heads;   // the fields of sky::Geo, in its order
} sky_probe_geo_t;
}

namespace sky {

// nullptr if consistent, else what is wrong
inline const char* probe_geo_error(const sky_probe_geo_t& g, int pairs) {
  if (g.Z < WZ || g.Z % WZ) return "Z is not a positive multiple of the window (2)";
  if (g.H < 1 || g.W < WW || g.W % WW) return "H < 1, or W is not a positive multiple of the window (12)";
  if (g.Hp != (g.H + WH - 1) / WH * WH) return "Hp is not H rounded up to the window (6)";
  if (g.nWz != g.Z / WZ || g.nWh != g.Hp / WH || g.nWw != g.W / WW) return "window counts do not match Z, Hp, W";
  if ((long long)g.T != (long long)g.Z * g.H * g.W) return "T != Z H W";
  if ((long long)g.nWin != (long long)g.nWz * g.nWh * g.nWw) return "nWin != nWz nWh nWw";
  if (pairs < 1 || g.heads != 2 * pairs) return "heads != 2 pairs";
  if (g.C != 32 * g.heads) return "C != 32 heads (head_dim 32)";
  return nullptr;
}

inline Geo probe_geo(const sky_probe_geo_t& p) {
  Geo g;
  g.Z = p.Z; g.H = p.H; g.W = p.W; g.C = p.C; g.Hp = p.Hp;
  g.nWz = p.nWz; g.nWh = p.nWh; g.nWw = p.nWw; g.T = p.T; g.nWin = p.nWin; g.heads = p.heads;
  return g;
}

}  // namespace sky
