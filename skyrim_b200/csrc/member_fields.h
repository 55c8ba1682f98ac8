// The field of ensemble members that the statistics and verification entries read (ens_stats.cu, scores.cu,
// score_points.cu): member m, selected channel s at x + m member_stride + channels[s] plane, or members pooled from several
// such fields (PooledSources).  The checks here make no CUDA call, so an entry refuses a bad field before it inspects any
// pointer; sources_device, the one exception, is the device-pointer check that follows them.
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

constexpr int kMaxSources = 4;

// Members pooled from up to kMaxSources sources (the members of several models on one device, each model with its own
// channel layout), in source-then-member order: member m starts at member[m] (its source's base + j member_stride),
// belongs to source member_src[m], and its selected channel s is the plane chan[member_src[m]][s] of that source.
// Travels by value inside the multi entries' parameter blocks (2648 bytes).
struct PooledSources {
  const float* member[kMaxMembers];
  int chan[kMaxSources][kMaxSel];
  int src_members[kMaxSources];
  int n_src;
  unsigned char member_src[kMaxMembers];
};
static_assert(sizeof(PooledSources) == 2648, "keep the parameter-block sizes of the multi entries in step");

// The source arguments of the multi entries, checked and stored in T: n_sources in [1, kMaxSources] with every host array
// given, plane positive, members[k] in [1, kMaxMembers] summing to at most kMaxMembers (returned in *total),
// channel_count[k] positive, member_stride[k] at least channel_count[k] x plane, n_sel in [1, kMaxSel], every channel of
// source k in [0, channel_count[k]) (channels is [n_sources][n_sel]) and no null x[k].  No CUDA call.
inline int check_sources(int n_sources, const float* const* x, const int32_t* members, const int64_t* member_stride,
                         const int32_t* channel_count, const int32_t* channels, int n_sel, int64_t plane, PooledSources& T,
                         int* total) {
  if (n_sources < 1 || n_sources > kMaxSources || !x || !members || !member_stride || !channel_count) {
    set_error("n_sources = %d must lie in [1, %d], with x, members, member_stride and channel_count given", n_sources, kMaxSources);
    return SKY_ERR_ARG;
  }
  if (plane < 1) { set_error("plane = %lld must be positive", (long long)plane); return SKY_ERR_ARG; }
  int sum = 0;
  for (int k = 0; k < n_sources; ++k) {
    if (members[k] < 1 || members[k] > kMaxMembers) { set_error("members[%d] = %d must lie in [1, %d]", k, members[k], kMaxMembers); return SKY_ERR_ARG; }
    sum += members[k];
    if (channel_count[k] < 1) { set_error("channel_count[%d] = %d must be positive", k, channel_count[k]); return SKY_ERR_ARG; }
    if (member_stride[k] < (int64_t)channel_count[k] * plane) {
      set_error("member_stride[%d] = %lld is below channel_count x plane = %lld", k, (long long)member_stride[k],
                (long long)channel_count[k] * plane);
      return SKY_ERR_ARG;
    }
  }
  if (sum > kMaxMembers) { set_error("total members = %d exceed %d", sum, kMaxMembers); return SKY_ERR_ARG; }
  if (n_sel < 1 || n_sel > kMaxSel || !channels) { set_error("n_sel = %d channels must lie in [1, %d]", n_sel, kMaxSel); return SKY_ERR_ARG; }
  T.n_src = n_sources;
  for (int k = 0; k < n_sources; ++k) {
    T.src_members[k] = members[k];
    for (int s = 0; s < n_sel; ++s) {
      const int c = channels[k * n_sel + s];
      if (c < 0 || c >= channel_count[k]) { set_error("channel %d of source %d is outside [0, %d)", c, k, channel_count[k]); return SKY_ERR_ARG; }
      T.chan[k][s] = c;
    }
  }
  for (int k = 0; k < n_sources; ++k)
    if (!x[k]) { set_error("x[%d] must not be null", k); return SKY_ERR_ARG; }
  for (int k = 0, m = 0; k < n_sources; ++k)
    for (int j = 0; j < members[k]; ++j, ++m) {
      T.member[m] = x[k] + j * member_stride[k];
      T.member_src[m] = (unsigned char)k;
    }
  *total = sum;
  return 0;
}

// device_of over the n sources' pointers: 0 when all are device memory on one device (*dev, or the first one's)
inline int sources_device(int n_sources, const float* const* x, int* dev) {
  for (int k = 0; k < n_sources; ++k) {
    const int rc = device_of(x[k], "x[k]", dev);
    if (rc) return rc;
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
