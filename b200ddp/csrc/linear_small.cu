// Linear layers whose dims are far below one wgmma tile (reference model.py:11-13: 10->10->5 at
// batch 32; the smallest MMA atom is 64x8x16 and TMA needs 16-byte row pitches, which a 10-wide
// bf16 row does not have).  These are latency problems, not FLOP problems: one CTA, operands in
// shared memory, fused bias + ReLU forward, and ONE backward launch producing dx, dw and db (with
// the ReLU mask recomputed from the saved output).  Larger, aligned shapes go to gemm_wgmma.cu.
#include "ops.h"

namespace b200 {
namespace {

constexpr int kSmallThreads = 256;

__global__ void __launch_bounds__(kSmallThreads) small_linear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                         const float* __restrict__ b, float* __restrict__ y, int M, int N,
                                                                         int K, int relu) {
  extern __shared__ float sw[];   // [N][K+1]
  for (int i = threadIdx.x; i < N * K; i += blockDim.x) sw[(i / K) * (K + 1) + (i % K)] = w[i];
  __syncthreads();
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < M * N; o += gridDim.x * blockDim.x) {
    const int m = o / N, n = o % N;
    const float* xr = x + (size_t)m * K;
    const float* wr = sw + n * (K + 1);
    float acc = b ? b[n] : 0.f;
    for (int k = 0; k < K; ++k) acc = fmaf(xr[k], wr[k], acc);
    y[o] = relu ? fmaxf(acc, 0.f) : acc;
  }
}

// grid.x = 1 CTA computes everything (M*N, N*K, M*K all tiny).  dz = dy * (y > 0) if relu.
__global__ void __launch_bounds__(kSmallThreads) small_linear_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                         const float* __restrict__ w, const float* __restrict__ y,
                                                                         float* __restrict__ dx, float* __restrict__ dw, float* __restrict__ db,
                                                                         int M, int N, int K, int relu, int accumulate) {
  extern __shared__ float sm[];   // dz [M][N]
  float* dz = sm;
  for (int i = threadIdx.x; i < M * N; i += blockDim.x) {
    float g = dy[i];
    if (relu && !(y[i] > 0.f)) g = 0.f;
    dz[i] = g;
  }
  __syncthreads();
  // dw[n][k] = sum_m dz[m][n] x[m][k]
  for (int o = threadIdx.x; o < N * K; o += blockDim.x) {
    const int n = o / K, k = o % K;
    float acc = 0.f;
    for (int m = 0; m < M; ++m) acc = fmaf(dz[m * N + n], x[(size_t)m * K + k], acc);
    dw[o] = accumulate ? dw[o] + acc : acc;
  }
  if (db) {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      float acc = 0.f;
      for (int m = 0; m < M; ++m) acc += dz[m * N + n];
      db[n] = accumulate ? db[n] + acc : acc;
    }
  }
  if (dx) {
    for (int o = threadIdx.x; o < M * K; o += blockDim.x) {
      const int m = o / K, k = o % K;
      float acc = 0.f;
      for (int n = 0; n < N; ++n) acc = fmaf(dz[m * N + n], w[(size_t)n * K + k], acc);
      dx[o] = acc;
    }
  }
}

}  // namespace

void launch_small_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int relu, cudaStream_t s) {
  const size_t smem = (size_t)N * (K + 1) * sizeof(float);
  if (smem > 48 * 1024) throw std::runtime_error("small_linear_fwd: weight does not fit the small-shape kernel");
  int blocks = (M * N + kSmallThreads - 1) / kSmallThreads;
  if (blocks > kNumSMs) blocks = kNumSMs;
  small_linear_fwd_kernel<<<blocks, kSmallThreads, smem, s>>>(x, w, b, y, M, N, K, relu);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_small_linear_bwd(const float* dy, const float* x, const float* w, const float* y, float* dx, float* dw, float* db, int M, int N,
                             int K, int relu, int accumulate, cudaStream_t s) {
  const size_t smem = (size_t)M * N * sizeof(float);
  if (smem > 48 * 1024) throw std::runtime_error("small_linear_bwd: activation gradient does not fit the small-shape kernel");
  small_linear_bwd_kernel<<<1, kSmallThreads, smem, s>>>(dy, x, w, y, dx, dw, db, M, N, K, relu, accumulate);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
