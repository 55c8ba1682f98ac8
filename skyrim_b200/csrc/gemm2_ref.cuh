// CUDA-core twin of gemm2.cuh (same image operands, same epilogue functors).
// DEVICE-SIDE TEST INFRASTRUCTURE: SKY_GEMM=ref runs the step on these to bisect a parity
// failure between "epilogue / index arithmetic" and "TMA + wgmma pipeline".  Never the
// benchmarked path.
#pragma once
#include "gemm2.cuh"

namespace sky {

// scratch[M, N] = A(image)[M, Kp] * W[N, Kp]^T   (W plain fp16 row-major, K zero-padded)
__global__ void __launch_bounds__(256) k_gemm2_ref(AImage A, const __half* __restrict__ W,
                                                   float* __restrict__ scratch, long long M, int N, int Kp) {
  constexpr int BM = 64, BN = 64, BK = 32;
  __shared__ float As[BK][BM + 1];
  __shared__ float Bs[BK][BN + 1];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int tx = tid % 16, ty = tid / 16;
  float acc[4][4] = {};
  const int lr = tid / 4, lc = tid % 4;
  for (int k0 = 0; k0 < Kp; k0 += BK) {
    uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
    const long long row = m0 + lr;
    if (row < M) {
      const int k = k0 + lc * 8;
      const uint8_t* kbp = A.kblock((int)(row >> 7), k >> 6);
      a = __ldg(reinterpret_cast<const uint4*>(kbp + sw128_offset((uint32_t)(row & 127), (k & 63) >> 3)));
    }
    if (n0 + lr < N) b = __ldg(reinterpret_cast<const uint4*>(W + (long long)(n0 + lr) * Kp + k0 + lc * 8));
    const __half* ah = reinterpret_cast<const __half*>(&a);
    const __half* bh = reinterpret_cast<const __half*>(&b);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      As[lc * 8 + e][lr] = __half2float(ah[e]);
      Bs[lc * 8 + e][lr] = __half2float(bh[e]);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[kk][ty * 4 + i]; bv[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += av[i] * bv[j];
    }
    __syncthreads();
  }
  for (int i = 0; i < 4; ++i) {
    long long r = m0 + ty * 4 + i;
    if (r >= M) continue;
    for (int j = 0; j < 4; ++j) {
      int c = n0 + tx * 4 + j;
      if (c < N) scratch[r * N + c] = acc[i][j];
    }
  }
}

struct AccScratch2 {
  const float* p;
  __device__ void load32(int c, float (&v)[32]) const {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = p ? p[c + j] : 0.f;
  }
};

// one warp per (32 rows, n-tile); single column partition
template <class Epi, int BLOCK_N>
__global__ void __launch_bounds__(128) k_epi2_ref(Epi epi, const float* __restrict__ scratch, long long M, int N) {
  __shared__ float patches[4 * G2_PATCH_FLOATS];
  __shared__ float sbias[3 * 512];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int n0 = blockIdx.y * BLOCK_N;
  if constexpr (Epi::kNeedsBias)
    for (int i = threadIdx.x; i < BLOCK_N; i += 128) { sbias[i] = epi.bias[i]; sbias[512 + i] = epi.gamma[i]; sbias[1024 + i] = epi.beta[i]; }
  __syncthreads();
  EpiCtx ctx;
  ctx.row0 = ((long long)blockIdx.x * 4 + warp) * 32;
  ctx.M = M; ctx.lane = lane; ctx.n0 = n0; ctx.part = 0; ctx.nparts = 1;
  ctx.patch = patches + warp * G2_PATCH_FLOATS;
  ctx.patch_s = smem_u32(ctx.patch);
  ctx.svec_s = smem_u32(sbias);
  const long long row = ctx.row0 + lane;
  AccScratch2 acc{row < M ? scratch + row * N + n0 : nullptr};
  epi.template run<BLOCK_N>(acc, ctx);
}

template <class Epi, int BLOCK_N>
int launch_gemm2_ref(const AImage& A, const Epi& epi, const __half* Wplain, float* scratch, long long M, int N,
                     int Kp, cudaStream_t st) {
  dim3 g1((unsigned)((M + 63) / 64), (unsigned)((N + 63) / 64));
  k_gemm2_ref<<<g1, 256, 0, st>>>(A, Wplain, scratch, M, N, Kp);
  dim3 g2((unsigned)((M + 127) / 128), (unsigned)(N / BLOCK_N));
  k_epi2_ref<Epi, BLOCK_N><<<g2, 128, 0, st>>>(epi, scratch, M, N);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
