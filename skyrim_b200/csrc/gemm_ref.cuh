// Plain CUDA-core GEMM with the same producers / epilogues as the wgmma kernel.
// DEVICE-SIDE TEST INFRASTRUCTURE: selected with SKY_GEMM=ref to bisect a parity failure
// between "index arithmetic / epilogue" and "tensor-core pipeline".  Same numerics contract
// (fp16 operands, fp32 accumulate); never the benchmarked path.
#pragma once
#include "pangu_ops.cuh"

namespace sky {

// scratch[M, N] = A(prod)[M, Kp] * W[N, Kp]^T     (W plain fp16 row-major, K zero-padded)
template <class Prod>
__global__ void __launch_bounds__(256) k_gemm_ref(Prod prod, const __half* __restrict__ W,
                                                  float* __restrict__ scratch, long long M, int N,
                                                  int Kp) {
  constexpr int BM = 64, BN = 64, BK = 32;
  __shared__ float As[BK][BM + 1];
  __shared__ float Bs[BK][BN + 1];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int tx = tid % 16, ty = tid / 16;
  float acc[4][4] = {};
  // loader mapping: 64 rows x 4 chunks(8 halves) = 256 chunks -> one per thread
  const int lr = tid / 4, lc = tid % 4;
  RowInfo ri = prod.prep(m0 + lr);
  for (int k0 = 0; k0 < Kp; k0 += BK) {
    uint4 a = prod.load8(ri, k0 + lc * 8);
    uint4 b = make_uint4(0, 0, 0, 0);
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

struct AccScratch {
  const float* p;  // this lane's row, at the tile's first column (nullptr for tail rows)
  __device__ void load32(int c, float (&v)[32]) const {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = p ? p[c + j] : 0.f;
  }
};

// one warp per (32 rows, n-tile)
template <class Epi>
__global__ void __launch_bounds__(128) k_epi_ref(Epi epi, const float* __restrict__ scratch,
                                                 long long M, int N, int BN) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const long long row = ((long long)blockIdx.x * 4 + warp) * 32 + lane;
  const int n0 = blockIdx.y * BN;
  AccScratch acc{row < M ? scratch + row * N + n0 : nullptr};
  epi.run(acc, row, n0, BN);
}

template <class Prod, class Epi>
int launch_gemm_ref(const Prod& prod, const Epi& epi, const __half* Wplain, float* scratch,
                    long long M, int N, int Kp, int BN, cudaStream_t st) {
  dim3 g1((unsigned)((M + 63) / 64), (unsigned)((N + 63) / 64));
  k_gemm_ref<Prod><<<g1, 256, 0, st>>>(prod, Wplain, scratch, M, N, Kp);
  dim3 g2((unsigned)((M + 127) / 128), (unsigned)(N / BN));
  k_epi_ref<Epi><<<g2, 128, 0, st>>>(epi, scratch, M, N, BN);
  SKY_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sky
