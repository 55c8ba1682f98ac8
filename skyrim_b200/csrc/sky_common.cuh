// Common device helpers for the sm_90a kernels: mbarrier, bulk-copy (TMA engine), wgmma
// descriptors and fences, swizzle math, small math utilities.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace sky {

// ---------------------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define SKY_CUDA_OK(expr)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      ::sky::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,   \
                       __LINE__);                                                          \
      return -2;                                                                           \
    }                                                                                      \
  } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-(function, device) attribute: opt in once per device the
// function is launched on (`mask` is the launch site's own static bit set, one bit per device ordinal).
inline int smem_opt_in(std::atomic<uint64_t>& mask, const void* kern, int bytes) {
  int dev = 0;
  SKY_CUDA_OK(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (mask.load(std::memory_order_acquire) & bit) return 0;
  SKY_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  mask.fetch_or(bit, std::memory_order_release);
  return 0;
}
// RAII: make `dev` current for the duration of a C-ABI call and restore the caller's device afterwards
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// ---------------------------------------------------------------------------------------
// small device utilities
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}
// erf-GELU (PyTorch default), division free:
//     gelu(x) = relu(x) - |x| h(|x|),   h(a) = Phi(-a) = 0.5 erfcx(a/sqrt 2) exp(-a^2/2)
// with 0.5 erfcx(a/sqrt 2) replaced by a degree-7 polynomial fitted on [0, 6] under the weight
// exp(-a^2/2) (tools/fit_gelu.py): max abs error 1.2e-5, 20x below the fp16 rounding the value
// receives next.  One MUFU (ex2) per element instead of an rcp + ex2 pair.
__device__ __forceinline__ float mufu_rcp(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float mufu_ex2(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
#define SKY_GELU_C0 4.999848197e-01f
#define SKY_GELU_C1 -3.985058804e-01f
#define SKY_GELU_C2 2.469212325e-01f
#define SKY_GELU_C3 -1.237550324e-01f
#define SKY_GELU_C4 4.792390463e-02f
#define SKY_GELU_C5 -1.291761998e-02f
#define SKY_GELU_C6 2.073202457e-03f
#define SKY_GELU_C7 -1.453669241e-04f
#define SKY_GELU_EC (-0.5f * 1.4426950408889634f)
__device__ __forceinline__ float gelu_erf(float x) {
  const float a = fabsf(x);
  const float e = mufu_ex2(x * x * SKY_GELU_EC);
  float p = SKY_GELU_C7;
  p = fmaf(p, a, SKY_GELU_C6); p = fmaf(p, a, SKY_GELU_C5); p = fmaf(p, a, SKY_GELU_C4);
  p = fmaf(p, a, SKY_GELU_C3); p = fmaf(p, a, SKY_GELU_C2); p = fmaf(p, a, SKY_GELU_C1);
  p = fmaf(p, a, SKY_GELU_C0);
  return fmaf(-a, p * e, fmaxf(x, 0.f));
}
// (x0, x1) <- gelu(x0 + b0), gelu(x1 + b1)
__device__ __forceinline__ void gelu_erf_x2(float& x0, float& x1, float b0, float b1) {
  x0 = gelu_erf(x0 + b0);
  x1 = gelu_erf(x1 + b1);
}

// explicit shared-space accessors (a generic LD/ST through a pointer kept in a struct costs a
// long-scoreboard round trip; these compile to LDS/STS)
__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ float4 lds_f32x4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
// read-only variant (bias / gamma / beta vectors that are written once before the role
// dispatch): not volatile, so the compiler may batch and hoist these loads
__device__ __forceinline__ float4 lds_f32x4_ro(uint32_t a) {
  float4 v;
  asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
}

// 32-byte global accesses as two 128-bit halves.  Used by the row-owner epilogues, where lane i
// owns token row i and the warp touches 32 different lines.
__device__ __forceinline__ void ldg_f32x8(const float* p, float* v) {
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "l"(p));
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7]) : "l"(p + 4));
}
__device__ __forceinline__ void stg_f32x8(float* p, const float* v) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p + 4), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7]) : "memory");
}
__device__ __forceinline__ void stg_b32x8(void* p, uint4 lo, uint4 hi) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(static_cast<char*>(p) + 16), "r"(hi.x), "r"(hi.y), "r"(hi.z),
               "r"(hi.w)
               : "memory");
}

// Byte offset of element (row, 16-byte chunk) inside a K-major SWIZZLE_128B tile whose rows
// are 128 bytes (64 halves): Swizzle<3,4,3> — chunk index XOR (row mod 8).
__device__ __host__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk) {
  return row * 128u + ((chunk ^ (row & 7u)) << 4);
}

// ---------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Blocking wait.  try_wait suspends the warp in hardware up to the time hint, so a waiting
// role warp does not burn issue slots of the epilogue warps that share its scheduler
// (the v1 C-level spin loop cost ~30% of all executed instructions: profiles/r1_mlp_v1.md).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "SKY_WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra SKY_DONE_%=;\n\t"
      "bra SKY_WAIT_%=;\n\t"
      "SKY_DONE_%=:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(0x989680)
      : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (wgmma / bulk copy)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------------------------------
// bulk copy global -> shared through the TMA engine (1-D, no tensor map needed).
// dst/src 16-byte aligned, bytes multiple of 16; completion is signalled on `bar`.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// bulk copy shared -> global (same alignment rules), tracked by the issuing thread's bulk async-groups: after
// bulk_commit(), bulk_wait_read<0>() returns once the source bytes have been read (the shared memory may be rewritten),
// bulk_wait<0>() once the writes are done
__device__ __forceinline__ void bulk_s2g(void* gdst, uint32_t smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// bulk prefetch of global memory into L2 (16-byte aligned, bytes multiple of 16)
__device__ __forceinline__ void bulk_prefetch_l2(const void* gsrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}

// ---------------------------------------------------------------------------------------
// wgmma (warpgroup MMA).  A warpgroup of four consecutive warps issues m64nNk16 products
// (wgmma_ops.cuh) with both operands read from shared memory through 64-bit descriptors and
// fp32 accumulators in its registers: thread (warp w of the group, lane l) holds, per 8-column
// group i, rows 16w + l/4 and 16w + l/4 + 8, columns 8i + 2(l%4) and 8i + 2(l%4) + 1.
// ---------------------------------------------------------------------------------------
// K-major operand, SWIZZLE_128B, rows of 128 bytes, 8-row groups 1024 bytes apart (SBO);
// +2 in the address field = +32 B = one K=16 step inside the swizzle row
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr_bytes & 0x3FFFFu) >> 4);  // start address  [0,14)
  d |= (uint64_t)1 << 16;                              // LBO (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                    // SBO = 1024 B
  d |= (uint64_t)1 << 62;                              // layout type SWIZZLE_128B
  return d;
}
// MN-major operand, SWIZZLE_128B: atoms of [8 k-rows][64 elements = 128 B], 8-row K groups SBO = 1024 B apart,
// 64-element MN blocks `lbo` bytes apart; +128 in the address field = +2048 B = one K=16 step
__device__ __forceinline__ uint64_t make_desc_sw128_mn(uint32_t smem_addr_bytes, uint32_t lbo) {
  uint64_t d = make_desc_sw128(smem_addr_bytes);
  return (d & ~((uint64_t)0x3FFF << 16)) | ((uint64_t)(lbo >> 4) << 16);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pin accumulator registers behind the preceding wait (register reads may not be hoisted above it)
template <int N>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Accumulator tile staged in shared memory, row-major fp32 with `ld` floats per row (ld % 32 == 4: the
// row-owner reads of a quarter warp hit 8 different bank quads).  acc.load32(c, v): the calling lane's
// row, columns [c, c+32) — the interface every epilogue is written against.
struct AccSmem {
  uint32_t row_s;  // shared-space address of the lane's row
  __device__ void load32(int c, float (&v)[32]) const {
    const uint32_t a = row_s + (uint32_t)c * 4u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(v[4 * j]), "=f"(v[4 * j + 1]), "=f"(v[4 * j + 2]), "=f"(v[4 * j + 3])
                   : "r"(a + 16u * j));
    }
  }
};

// ---------------------------------------------------------------------------------------
// clusters: distributed shared memory and cluster-scope barriers
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `local_smem_addr` in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}

}  // namespace sky
