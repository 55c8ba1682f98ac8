// The field of ensemble members that the statistics and verification entries read (ens_stats.cu, scores.cu,
// score_points.cu): member m, selected channel s at x + m member_stride + channels[s] plane.  The checks here make no
// CUDA call, so an entry refuses a bad field before it inspects any pointer.
#pragma once
#include <stdint.h>

#include <type_traits>

#include "engine.h"

namespace sky {

constexpr int kMaxMembers = 64, kMaxSel = 128, kMaxRegions = 4;

// members in [1, kMaxMembers], member_stride at least channel_count x plane, n_sel in [1, kMaxSel] and every channel in
// [0, channel_count); the channels are copied to chan_out
inline int check_members(int members, int64_t member_stride, int64_t plane, int channel_count, const int32_t* channels,
                         int n_sel, int* chan_out) {
  if (members < 1 || members > kMaxMembers) { set_error("members = %d must lie in [1, %d]", members, kMaxMembers); return SKY_ERR_ARG; }
  if (plane < 1 || channel_count < 1) { set_error("plane (%lld) and channel_count (%d) must be positive", (long long)plane, channel_count); return SKY_ERR_ARG; }
  if (member_stride < (int64_t)channel_count * plane) {
    set_error("member_stride = %lld is below channel_count x plane = %lld", (long long)member_stride, (long long)channel_count * plane);
    return SKY_ERR_ARG;
  }
  if (n_sel < 1 || n_sel > kMaxSel || !channels) { set_error("n_sel = %d channels must lie in [1, %d]", n_sel, kMaxSel); return SKY_ERR_ARG; }
  for (int s = 0; s < n_sel; ++s) {
    if (channels[s] < 0 || channels[s] >= channel_count) { set_error("channel %d is outside [0, %d)", channels[s], channel_count); return SKY_ERR_ARG; }
    chan_out[s] = channels[s];
  }
  return 0;
}

// the verification entries index a plane of nlat x nlon points with int
inline int check_grid(int nlat, int nlon) {
  if (nlat < 1 || nlon < 1 || (int64_t)nlat * nlon > INT32_MAX) {
    set_error("nlat = %d and nlon = %d must be positive with nlat x nlon < 2^31", nlat, nlon);
    return SKY_ERR_ARG;
  }
  return 0;
}

// Calls f(std::integral_constant<int, MP>{}) with the members' register padding MP: the least of 8, 16, 32 and 64 that
// holds them, or 1 for a single member when MinPad is 1.  Each MP is one kernel instantiation, so this decides which
// instantiations exist and how many member registers a thread holds.
template <int MinPad, class F>
void dispatch_padding(int members, F&& f) {
  static_assert(MinPad == 1 || MinPad == 8, "the padding starts at 1 or 8 members");
  if constexpr (MinPad == 1) {
    if (members == 1) return f(std::integral_constant<int, 1>{});
  }
  if (members <= 8) f(std::integral_constant<int, 8>{});
  else if (members <= 16) f(std::integral_constant<int, 16>{});
  else if (members <= 32) f(std::integral_constant<int, 32>{});
  else f(std::integral_constant<int, 64>{});
}

}  // namespace sky
