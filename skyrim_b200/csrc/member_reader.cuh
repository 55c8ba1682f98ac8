// How the verification kernels (scores.cu, score_points.cu) read member m of their block's selected channel s.  Each kernel
// body is a template over its parameter block; the block's kPooled picks the reader:
//   OneSource      the single-source entries: member m at x + m member_stride + chan[s] plane, the loads of a plain
//                  strided tensor;
//   PooledMembers  the *_multi entries: members pooled from several sources (PooledSources, member_fields.h).  The block
//                  forms the M base pointers of its channel, member[m] + chan[member_src[m]][s] plane, once in shared
//                  memory (pooled_bases), so the point loop loads base[m][p] and never looks up the table.
// Both are called as r(m, p) with p the point's offset in the plane.
#pragma once
#include "member_fields.h"

namespace sky {

struct OneSource {
  const float* xs;             // member 0 of the block's channel
  long long stride;
  __device__ __forceinline__ float operator()(int m, long long p) const { return xs[m * stride + p]; }
};

struct PooledMembers {
  const float* const volatile* base;   // shared memory: member m's plane of the block's channel
  // volatile: re-read (a broadcast shared load) at every point instead of 64 pointers held in registers across the loops
  __device__ __forceinline__ float operator()(int m, long long p) const { return base[m][p]; }
};

// Fills base[0, M) with the planes of selected channel s and synchronises the block; every thread of the block calls it.
__device__ __forceinline__ void pooled_bases(const PooledSources& T, int M, int s, long long plane, const float** base) {
  for (int m = threadIdx.x; m < M; m += blockDim.x) base[m] = T.member[m] + (long long)T.chan[T.member_src[m]][s] * plane;
  __syncthreads();
}

// The reader of the block's selected channel s.  base: the block's shared table of kMaxMembers pointers, read only when
// pooled; every thread of the block calls this, before any of them returns.
template <class Params>
__device__ __forceinline__ auto members_of(const Params& P, int s, const float** base) {
  if constexpr (Params::kPooled) {
    pooled_bases(P.src, P.members, s, P.plane, base);
    return PooledMembers{base};
  } else {
    return OneSource{P.x + (long long)P.chan[s] * P.plane, P.member_stride};
  }
}

}  // namespace sky
