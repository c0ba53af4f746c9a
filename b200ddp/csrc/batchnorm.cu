// Fused training BatchNorm (+ residual add) (+ ReLU) for channels_last activations.
//
// Why: in the ResNet-50 bf16 step the stock path (ATen batch_norm_collect_statistics / transform_input /
// backward_reduce / backward_elemt + separate ReLU, residual-add and threshold_backward kernels + per-layer
// num_batches_tracked / running-stat updates) is the largest share of the ResNet-50 step outside the convolutions and
// runs far below the HBM roofline at batch 32.  A [N,C,H,W] channels_last tensor is a row-major [R = N*H*W, C]
// matrix, so every per-channel quantity is a column reduction:
//
//   forward : bn_stats      column sum / sum-of-squares -> mean, rstd, scale = gamma*rstd, shift = beta - mean*scale,
//                           running statistics and num_batches_tracked updated by the last block (deterministic)
//             bn_apply      y = relu(x*scale + shift + residual)            one pass, 16-byte accesses
//   backward: bn_bwd_reduce sum(dy*), sum(dy* * xhat); the ReLU mask is a 1-bit/element bitmap written by bn_apply
//                           (1/16 of re-reading y in bf16, twice); dgamma/dbeta
//             bn_bwd_apply  dx = scale*(dy* - mean(dy*) - xhat*mean(dy* xhat)), and the residual branch's grad
//
// Threads own 8 consecutive channels (one 16-byte vector of bf16); rows are strided across the block and
// across gridDim.y "row splits"; partial sums land in a [splits, C] workspace and the last block of each
// channel tile finishes the reduction in a fixed order (no float atomics -> bitwise reproducible).
//
// Resident kernels (bf16, the default wherever the shape fits): one cooperative launch per direction that reads every
// activation from HBM ONCE.  The persistent grid (<= one CTA per SM, ~200 KB of shared memory each) cuts [R, C] into
// 64-channel tiles and row slabs; a wave of tiles is TMA-loaded into shared memory (x, or dy and x), reduced to per-CTA
// partials, a grid barrier makes the partials visible, every CTA reduces its tile's partials in a fixed order and then
// normalises / applies the gradient straight from shared memory, writing the result back in place and TMA-storing it.
#include "ops.h"
#include "drv.h"
#include "tc_primitives.cuh"

#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>
#include <utility>

namespace b200 {
namespace {

constexpr int kBnThreads = 256;
constexpr int kVec = 8;              // channels per thread

template <typename T> __device__ __forceinline__ void bn_load8(const T* p, float* f);
template <> __device__ __forceinline__ void bn_load8<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
  unpack8(*reinterpret_cast<const Bf16x8*>(p), f);
}
template <> __device__ __forceinline__ void bn_load8<float>(const float* p, float* f) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <typename T> __device__ __forceinline__ void bn_store8(T* p, const float* f);
template <> __device__ __forceinline__ void bn_store8<__nv_bfloat16>(__nv_bfloat16* p, const float* f) {
  *reinterpret_cast<Bf16x8*>(p) = pack8(f);
}
template <> __device__ __forceinline__ void bn_store8<float>(float* p, const float* f) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}

struct Tile {
  int cvb;       // channel vectors handled by a block (threads along x)
  int ty;        // rows handled per block iteration
  int grid_x;    // channel tiles
  int grid_y;    // row splits
};

// Block-level reduction over the `ty` row-lanes of two 8-wide accumulators; result valid for threads with row-lane 0.
template <int NACC>
__device__ __forceinline__ void reduce_rows(float (*acc)[kVec], float* smem, int tx, int tyi, int cvb, int ty) {
  // smem layout: [NACC][ty][cvb*8]
  const int width = cvb * kVec;
#pragma unroll
  for (int a = 0; a < NACC; ++a)
#pragma unroll
    for (int i = 0; i < kVec; ++i) smem[(a * ty + tyi) * width + tx * kVec + i] = acc[a][i];
  __syncthreads();
  for (int idx = threadIdx.x; idx < NACC * width; idx += blockDim.x) {
    const int a = idx / width, c = idx % width;
    float s = 0.f;
    for (int r = 0; r < ty; ++r) s += smem[(a * ty + r) * width + c];
    smem[(a * ty) * width + c] = s;       // row-lane 0 slot now holds the block total
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void bn_apply_rows(const T* __restrict__ x, const T* __restrict__ residual, T* __restrict__ y,
                                              unsigned char* __restrict__ mask, const float* __restrict__ scale,
                                              const float* __restrict__ shift, int C, int cv, int r0, int r1, int tyi, int ty, int relu);

// Programmatic dependent launch (opt-in, B200DDP_PDL=1): the producer lets the dependent grid start scheduling once its
// main loop is done; the dependent blocks at griddepcontrol.wait until the producer grid has completed and flushed.
__device__ __forceinline__ void bn_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void bn_wait_producer() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// release/acquire on the per-tile generation word used by the fused (single-launch) variants
__device__ __forceinline__ void bn_st_release(unsigned int* p, unsigned int v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned int bn_ld_acquire(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// bounded spin (2 s): a scheduling surprise must degrade into a wrong number, never into a hung GPU
__device__ __forceinline__ void bn_wait_generation(const unsigned int* p, unsigned int gen0) {
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while (bn_ld_acquire(p) == gen0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (t - t0 > 2000000000ull) break;
  }
}

// FUSED = true: statistics AND normalisation in ONE launch.  All blocks of a channel tile rendezvous on a
// generation word after the tile's last block has finished the statistics (the grid is sized to be co-resident:
// <= 2 blocks per SM), then every block normalises exactly the rows it has just read (L2-hot).
template <typename T, bool FUSED, bool PDL = false>
__global__ void __launch_bounds__(kBnThreads, 2) bn_stats_kernel(const T* __restrict__ x, int R, int C, int cvb, int ty,
                                                             float* __restrict__ partial /*[2][S][C]*/, unsigned int* __restrict__ counters,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* __restrict__ running_mean, float* __restrict__ running_var,
                                                             long long* __restrict__ num_batches, float* __restrict__ save_mean,
                                                             float* __restrict__ save_rstd, float* __restrict__ scale, float* __restrict__ shift,
                                                             float eps, float momentum, const T* __restrict__ residual, T* __restrict__ y,
                                                             unsigned char* __restrict__ mask, int relu) {
  extern __shared__ float smem[];
  __shared__ bool is_last;
  unsigned int* gen = counters + gridDim.x;             // [grid_x] generation words behind the [grid_x] ticket counters
  unsigned int gen0 = 0;
  if (FUSED && threadIdx.x == 0) gen0 = *reinterpret_cast<volatile unsigned int*>(&gen[blockIdx.x]);   // read BEFORE taking a ticket
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;                 // channel-vector index
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  float acc[2][kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  if (cv * kVec < C) {
    const T* base = x + (size_t)cv * kVec;
    int r = r0 + tyi;
    for (; r + 3 * ty < r1; r += 4 * ty) {              // 4 independent 16-byte loads in flight
      float f[4][kVec];
#pragma unroll
      for (int u = 0; u < 4; ++u) bn_load8<T>(base + (size_t)(r + u * ty) * C, f[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int i = 0; i < kVec; ++i) { acc[0][i] += f[u][i]; acc[1][i] = fmaf(f[u][i], f[u][i], acc[1][i]); }
    }
    for (; r < r1; r += ty) {
      float f[kVec];
      bn_load8<T>(base + (size_t)r * C, f);
#pragma unroll
      for (int i = 0; i < kVec; ++i) { acc[0][i] += f[i]; acc[1][i] = fmaf(f[i], f[i], acc[1][i]); }
    }
  }
  if constexpr (PDL) bn_launch_dependents();       // the apply kernel may start scheduling; it still waits for this whole grid
  reduce_rows<2>(acc, smem, tx, tyi, cvb, ty);
  const int width = cvb * kVec;
  const int c0 = blockIdx.x * width;
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    if (c0 + c < C) {
      partial[(size_t)(0 * S + blockIdx.y) * C + c0 + c] = smem[c];
      partial[(size_t)(1 * S + blockIdx.y) * C + c0 + c] = smem[ty * width + c];
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(&counters[blockIdx.x], 1u);
    is_last = (ticket == (unsigned int)S - 1);
  }
  __syncthreads();
  if (!FUSED && !is_last) return;
  if (is_last) {
    __threadfence();
    const float inv_r = 1.f / (float)R;
    // finish: `lanes` threads per channel each sum a strided subset of the S partials (independent loads in flight),
    // then a fixed-order combine through shared memory
    const int lanes = max(1, (int)blockDim.x / width);
    {
      const int c = threadIdx.x % width, l = threadIdx.x / width;
      float ps = 0.f, pq = 0.f;
      if (l < lanes && c0 + c < C) {
  #pragma unroll 4
        for (int k = l; k < S; k += lanes) { ps += __ldcg(&partial[(size_t)(0 * S + k) * C + c0 + c]); pq += __ldcg(&partial[(size_t)(1 * S + k) * C + c0 + c]); }
      }
      __syncthreads();
      if (l < lanes) { smem[l * width + c] = ps; smem[(lanes + l) * width + c] = pq; }
      __syncthreads();
    }
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      const int ch = c0 + c;
      if (ch >= C) continue;
      float s = 0.f, q = 0.f;
      for (int l = 0; l < lanes; ++l) { s += smem[l * width + c]; q += smem[(lanes + l) * width + c]; }
      const float mean = s * inv_r;
      const float var = fmaxf(q * inv_r - mean * mean, 0.f);     // biased variance (normalisation)
      const float rstd = rsqrtf(var + eps);
      const float sc = gamma[ch] * rstd;
      save_mean[ch] = mean;
      save_rstd[ch] = rstd;
      scale[ch] = sc;
      shift[ch] = beta[ch] - mean * sc;
      if (running_mean != nullptr) {
        const float unbiased = R > 1 ? var * ((float)R / (float)(R - 1)) : var;
        running_mean[ch] = (1.f - momentum) * running_mean[ch] + momentum * mean;
        running_var[ch] = (1.f - momentum) * running_var[ch] + momentum * unbiased;
      }
    }

    __syncthreads();
    if (threadIdx.x == 0) {
      counters[blockIdx.x] = 0u;                                 // ready for the next launch (graph replay safe)
      if (blockIdx.x == 0 && num_batches != nullptr) *num_batches += 1;
      if (FUSED) { __threadfence(); bn_st_release(&gen[blockIdx.x], gen0 + 1u); }
    }
  }
  if (!FUSED) return;
  if (!is_last && threadIdx.x == 0) bn_wait_generation(&gen[blockIdx.x], gen0);      // the tile's statistics are final
  __syncthreads();
  if (cv * kVec < C) bn_apply_rows<T>(x, residual, y, mask, scale, shift, C, cv, r0, r1, tyi, ty, relu);
}

template <typename T>
__device__ __forceinline__ void bn_apply_rows(const T* __restrict__ x, const T* __restrict__ residual, T* __restrict__ y,
                                              unsigned char* __restrict__ mask, const float* __restrict__ scale,
                                              const float* __restrict__ shift, int C, int cv, int r0, int r1, int tyi, int ty, int relu) {
  float sc[kVec], sh[kVec];                       // per-channel constants stay in registers for the whole row loop
  bn_load8<float>(scale + cv * kVec, sc);
  bn_load8<float>(shift + cv * kVec, sh);
  const size_t col = (size_t)cv * kVec;
  int r = r0 + tyi;
  for (; r + 3 * ty < r1; r += 4 * ty) {
    float f[4][kVec], rs[4][kVec];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      bn_load8<T>(x + (size_t)(r + u * ty) * C + col, f[u]);
      if (residual != nullptr) bn_load8<T>(residual + (size_t)(r + u * ty) * C + col, rs[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      unsigned int bits = 0;
#pragma unroll
      for (int i = 0; i < kVec; ++i) {
        float v = fmaf(f[u][i], sc[i], sh[i]);
        if (residual != nullptr) v += rs[u][i];
        bits |= (v > 0.f ? 1u : 0u) << i;
        f[u][i] = relu ? fmaxf(v, 0.f) : v;
      }
      bn_store8<T>(y + (size_t)(r + u * ty) * C + col, f[u]);
      if (mask != nullptr) mask[(size_t)(r + u * ty) * (C / kVec) + cv] = (unsigned char)bits;
    }
  }
  for (; r < r1; r += ty) {
    float f[kVec], rs[kVec];
    bn_load8<T>(x + (size_t)r * C + col, f);
    if (residual != nullptr) bn_load8<T>(residual + (size_t)r * C + col, rs);
    unsigned int bits = 0;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      float v = fmaf(f[i], sc[i], sh[i]);
      if (residual != nullptr) v += rs[i];
      bits |= (v > 0.f ? 1u : 0u) << i;
      f[i] = relu ? fmaxf(v, 0.f) : v;
    }
    bn_store8<T>(y + (size_t)r * C + col, f);
    if (mask != nullptr) mask[(size_t)r * (C / kVec) + cv] = (unsigned char)bits;
  }
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_apply_kernel(const T* __restrict__ x, const T* __restrict__ residual, T* __restrict__ y,
                                                             unsigned char* __restrict__ mask, const float* __restrict__ scale,
                                                             const float* __restrict__ shift, int R, int C, int cvb, int ty, int relu) {
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  if (cv * kVec >= C) return;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  bn_apply_rows<T>(x, residual, y, mask, scale, shift, C, cv, r0, r1, tyi, ty, relu);
}

// same body, launched as a programmatic dependent of bn_stats_kernel<.., PDL = true>
template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_apply_pdl_kernel(const T* __restrict__ x, const T* __restrict__ residual, T* __restrict__ y,
                                                                 unsigned char* __restrict__ mask, const float* __restrict__ scale,
                                                                 const float* __restrict__ shift, int R, int C, int cvb, int ty, int relu) {
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  bn_wait_producer();                               // scale / shift are written by the producer's last block
  if (cv * kVec >= C) return;
  bn_apply_rows<T>(x, residual, y, mask, scale, shift, C, cv, r0, r1, tyi, ty, relu);
}

template <typename T>
__device__ __forceinline__ void bn_bwd_apply_rows(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                  T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ save_mean,
                                                  const float* __restrict__ save_rstd, const float* __restrict__ gamma,
                                                  const float* __restrict__ coef, int C, int cv, int r0, int r1, int tyi, int ty, int relu);
template <typename T>
__device__ __forceinline__ void bn_bwd_apply_rows_coef(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                       T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ save_mean,
                                                       const float* __restrict__ save_rstd, const float* __restrict__ gamma,
                                                       const float* c1p, const float* c2p, int C, int cv, int r0, int r1, int tyi, int ty, int relu);

// ------------------------------------------------------------------------------------------------------
template <typename T, bool FUSED, bool PDL = false>
__global__ void __launch_bounds__(kBnThreads, 2) bn_bwd_reduce_kernel(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                                     int R, int C, int cvb, int ty, int relu, const float* __restrict__ save_mean,
                                                                     const float* __restrict__ save_rstd, float* __restrict__ partial,
                                                                     unsigned int* __restrict__ counters, float* __restrict__ dgamma,
                                                                     float* __restrict__ dbeta, float* __restrict__ coef /*[2][C]*/,
                                                                     const float* __restrict__ gamma, T* __restrict__ dx, T* __restrict__ dres) {
  extern __shared__ float smem[];
  __shared__ bool is_last;
  unsigned int* gen = counters + gridDim.x;
  unsigned int gen0 = 0;
  if (FUSED && threadIdx.x == 0) gen0 = *reinterpret_cast<volatile unsigned int*>(&gen[blockIdx.x]);
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  float acc[2][kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  if (cv * kVec < C) {
    float mean[kVec], rstd[kVec];
    bn_load8<float>(save_mean + cv * kVec, mean);
    bn_load8<float>(save_rstd + cv * kVec, rstd);
    const size_t col = (size_t)cv * kVec;
    int r = r0 + tyi;
    for (; r + ty < r1; r += 2 * ty) {                  // 2 rows x 3 streams = 6 independent 16-byte loads in flight
      float g[2][kVec], xv[2][kVec];
      unsigned int mk[2] = {0xffu, 0xffu};
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const size_t off = (size_t)(r + u * ty) * C + col;
        bn_load8<T>(dy + off, g[u]);
        bn_load8<T>(x + off, xv[u]);
        if (relu) mk[u] = y[(size_t)(r + u * ty) * (C / kVec) + cv];
      }
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int i = 0; i < kVec; ++i) {
          const float gm = ((mk[u] >> i) & 1u) ? g[u][i] : 0.f;
          acc[0][i] += gm;
          acc[1][i] = fmaf(gm, (xv[u][i] - mean[i]) * rstd[i], acc[1][i]);
        }
    }
    for (; r < r1; r += ty) {
      float g[kVec], xv[kVec];
      const size_t off = (size_t)r * C + col;
      bn_load8<T>(dy + off, g);
      bn_load8<T>(x + off, xv);
      const unsigned int mk = relu ? y[(size_t)r * (C / kVec) + cv] : 0xffu;
#pragma unroll
      for (int i = 0; i < kVec; ++i) {
        const float gm = ((mk >> i) & 1u) ? g[i] : 0.f;
        acc[0][i] += gm;
        acc[1][i] = fmaf(gm, (xv[i] - mean[i]) * rstd[i], acc[1][i]);
      }
    }
  }
  if constexpr (PDL) bn_launch_dependents();       // the apply kernel may start scheduling; it still waits for this whole grid
  reduce_rows<2>(acc, smem, tx, tyi, cvb, ty);
  const int width = cvb * kVec;
  const int c0 = blockIdx.x * width;
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    if (c0 + c < C) {
      partial[(size_t)(0 * S + blockIdx.y) * C + c0 + c] = smem[c];
      partial[(size_t)(1 * S + blockIdx.y) * C + c0 + c] = smem[ty * width + c];
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(&counters[blockIdx.x], 1u);
    is_last = (ticket == (unsigned int)S - 1);
  }
  __syncthreads();
  if (!FUSED && !is_last) return;
  if (is_last) {
    __threadfence();
    const float inv_r = 1.f / (float)R;
    // finish: `lanes` threads per channel each sum a strided subset of the S partials (independent loads in flight),
    // then a fixed-order combine through shared memory
    const int lanes = max(1, (int)blockDim.x / width);
    {
      const int c = threadIdx.x % width, l = threadIdx.x / width;
      float ps = 0.f, pq = 0.f;
      if (l < lanes && c0 + c < C) {
  #pragma unroll 4
        for (int k = l; k < S; k += lanes) { ps += __ldcg(&partial[(size_t)(0 * S + k) * C + c0 + c]); pq += __ldcg(&partial[(size_t)(1 * S + k) * C + c0 + c]); }
      }
      __syncthreads();
      if (l < lanes) { smem[l * width + c] = ps; smem[(lanes + l) * width + c] = pq; }
      __syncthreads();
    }
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      const int ch = c0 + c;
      if (ch >= C) continue;
      float s = 0.f, q = 0.f;
      for (int l = 0; l < lanes; ++l) { s += smem[l * width + c]; q += smem[(lanes + l) * width + c]; }
      dbeta[ch] = s;
      dgamma[ch] = q;
      coef[ch] = s * inv_r;            // mean(dy*)
      coef[C + ch] = q * inv_r;        // mean(dy* xhat)
    }

    __syncthreads();
    if (threadIdx.x == 0) {
      counters[blockIdx.x] = 0u;
      if (FUSED) { __threadfence(); bn_st_release(&gen[blockIdx.x], gen0 + 1u); }
    }
  }
  if (!FUSED) return;
  if (!is_last && threadIdx.x == 0) bn_wait_generation(&gen[blockIdx.x], gen0);
  __syncthreads();
  if (cv * kVec < C) bn_bwd_apply_rows<T>(dy, x, y, dx, dres, save_mean, save_rstd, gamma, coef, C, cv, r0, r1, tyi, ty, relu);
}

// c1p / c2p point at THIS thread's 8 coefficients (global coef rows or a block's shared-memory copy)
template <typename T>
__device__ __forceinline__ void bn_bwd_apply_rows_coef(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                       T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ save_mean,
                                                       const float* __restrict__ save_rstd, const float* __restrict__ gamma,
                                                       const float* c1p, const float* c2p, int C, int cv, int r0, int r1, int tyi, int ty, int relu) {
  // dx = a*dy* + b*x + c  with per-channel a = gamma*rstd, b = -a*rstd*c2, c = -a*(c1 - mean*rstd*c2)
  float ka[kVec], kb[kVec], kc[kVec];
  {
    float mean[kVec], rstd[kVec], gam[kVec], c1[kVec], c2[kVec];
    bn_load8<float>(save_mean + cv * kVec, mean);
    bn_load8<float>(save_rstd + cv * kVec, rstd);
    bn_load8<float>(gamma + cv * kVec, gam);
    bn_load8<float>(c1p, c1);
    bn_load8<float>(c2p, c2);
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      ka[i] = gam[i] * rstd[i];
      kb[i] = -ka[i] * rstd[i] * c2[i];
      kc[i] = -ka[i] * (c1[i] - mean[i] * rstd[i] * c2[i]);
    }
  }
  const size_t col = (size_t)cv * kVec;
  int r = r0 + tyi;
  for (; r + ty < r1; r += 2 * ty) {                    // 2 rows x 3 streams in flight
    float g[2][kVec], xv[2][kVec];
    unsigned int mk[2] = {0xffu, 0xffu};
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t off = (size_t)(r + u * ty) * C + col;
      bn_load8<T>(dy + off, g[u]);
      bn_load8<T>(x + off, xv[u]);
      if (relu) mk[u] = y[(size_t)(r + u * ty) * (C / kVec) + cv];
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const size_t off = (size_t)(r + u * ty) * C + col;
      float o[kVec];
#pragma unroll
      for (int i = 0; i < kVec; ++i) {
        if (!((mk[u] >> i) & 1u)) g[u][i] = 0.f;
        o[i] = fmaf(ka[i], g[u][i], fmaf(kb[i], xv[u][i], kc[i]));
      }
      if (dres != nullptr) bn_store8<T>(dres + off, g[u]);          // gradient of the residual branch = masked dy
      bn_store8<T>(dx + off, o);
    }
  }
  for (; r < r1; r += ty) {
    const size_t off = (size_t)r * C + col;
    float g[kVec], xv[kVec], o[kVec];
    bn_load8<T>(dy + off, g);
    bn_load8<T>(x + off, xv);
    const unsigned int mk = relu ? y[(size_t)r * (C / kVec) + cv] : 0xffu;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      if (!((mk >> i) & 1u)) g[i] = 0.f;
      o[i] = fmaf(ka[i], g[i], fmaf(kb[i], xv[i], kc[i]));
    }
    if (dres != nullptr) bn_store8<T>(dres + off, g);
    bn_store8<T>(dx + off, o);
  }
}

template <typename T>
__device__ __forceinline__ void bn_bwd_apply_rows(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                  T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ save_mean,
                                                  const float* __restrict__ save_rstd, const float* __restrict__ gamma,
                                                  const float* __restrict__ coef, int C, int cv, int r0, int r1, int tyi, int ty, int relu) {
  bn_bwd_apply_rows_coef<T>(dy, x, y, dx, dres, save_mean, save_rstd, gamma, coef + cv * kVec, coef + C + cv * kVec, C, cv, r0, r1, tyi, ty, relu);
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                                 T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ save_mean,
                                                                 const float* __restrict__ save_rstd, const float* __restrict__ gamma,
                                                                 const float* __restrict__ coef, int R, int C, int cvb, int ty, int relu) {
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  if (cv * kVec >= C) return;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  bn_bwd_apply_rows<T>(dy, x, y, dx, dres, save_mean, save_rstd, gamma, coef, C, cv, r0, r1, tyi, ty, relu);
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_apply_pdl_kernel(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                                     T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ save_mean,
                                                                     const float* __restrict__ save_rstd, const float* __restrict__ gamma,
                                                                     const float* __restrict__ coef, int R, int C, int cvb, int ty, int relu) {
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  bn_wait_producer();                               // coef / dgamma / dbeta come from the producer's last block
  if (cv * kVec >= C) return;
  bn_bwd_apply_rows<T>(dy, x, y, dx, dres, save_mean, save_rstd, gamma, coef, C, cv, r0, r1, tyi, ty, relu);
}

// B200DDP_PDL=1: stats -> apply and bwd_reduce -> bwd_apply become programmatic dependent launches
int g_bn_pdl = -1;     // -1: read B200DDP_PDL on first use
bool bn_pdl_enabled() {
  if (g_bn_pdl < 0) { const char* e = getenv("B200DDP_PDL"); g_bn_pdl = (e && atoi(e) != 0) ? 1 : 0; }
  return g_bn_pdl > 0;
}

template <typename... KArgs, typename... Args>
void launch_dependent(void (*kernel)(KArgs...), dim3 grid, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(kBnThreads);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
}

Tile pick_tile(int R, int C) {
  Tile t;
  const int cv = C / kVec;
  t.cvb = cv < 8 ? cv : 8;                            // <= 64 channels per tile: 128-byte row segments, and the
  while (kBnThreads % t.cvb != 0) --t.cvb;            //    finishing block has >= 4 lanes per channel
  t.ty = kBnThreads / t.cvb;
  t.grid_x = (cv + t.cvb - 1) / t.cvb;
  // enough row splits to put ~4 blocks on every SM, but keep >= 4 row iterations per block
  int want = (4 * kNumSMs + t.grid_x - 1) / t.grid_x;
  int max_by_rows = R / (t.ty * 4);
  if (max_by_rows < 1) max_by_rows = 1;
  t.grid_y = want < max_by_rows ? want : max_by_rows;
  if (t.grid_y > 256) t.grid_y = 256;
  return t;
}

// apply kernels: same channel tiling, row splits sized so each thread sees >= 4 rows but the grid still fills the GPU
dim3 apply_grid(const Tile& t, int R) {
  int want = (8 * kNumSMs + t.grid_x - 1) / t.grid_x;
  int max_by_rows = R / (t.ty * 4);
  if (max_by_rows < 1) max_by_rows = 1;
  int gy = want < max_by_rows ? want : max_by_rows;
  return dim3(t.grid_x, gy);
}

// Fused (single-launch) variants need every block of a channel tile resident at once: cap the grid at 2 blocks per SM.
bool fused_tile(int R, int C, Tile* t) {
  static int enabled = -1;
  // one launch per direction caps the grid at what can be co-resident, which costs what the saved launch gains, so the
  // two-launch form stays the default; opt in with =1
  if (enabled < 0) { const char* e = getenv("B200DDP_BN_FUSED"); enabled = (e && atoi(e) == 1) ? 1 : 0; }
  *t = pick_tile(R, C);
  if (!enabled || t->grid_x > 2 * kNumSMs) return false;
  int cap = (2 * kNumSMs) / t->grid_x;
  if (cap < 1) cap = 1;
  if (t->grid_y > cap) t->grid_y = cap;
  return true;
}

// ---- resident (single-read) kernels ---------------------------------------------------------------------------------
constexpr int kResThreads = 256;     // 8 channel vectors x 32 row lanes
constexpr int kResTile = 64;         // channels per tile: a 128-byte bf16 row segment, one TMA box row
constexpr int kResMaxBox = 256;      // TMA box height limit
constexpr int kResMaxBoxes = 16;     // boxes (and mbarriers) per CTA and stream
constexpr int kResWarps = kResThreads / 32;
static_assert(kResMaxBox <= 8 * (kResThreads / 8), "the forward apply gives each of the 32 row lanes 8 rows of a box");
// Waves per launch.  A shape needing up to kResMaxLaunches * kResMaxWaves waves runs as that many launches over disjoint
// ranges of channel tiles (the backward of [100352, 256]: 4 waves, two launches).
constexpr int kResMaxWaves = 2;
constexpr int kResMaxLaunches = 2;
constexpr int kResMaxPartialLoads = 17;   // ceil(132 SMs / 8 warps): partial rows each thread of a tile reduction loads
// shared memory behind the slabs: mbarriers, [warps][2][64] reduction scratch, [2][64] totals, [3][64] coefficients
constexpr int kResFixedSmem = kResMaxBoxes * 8 + (kResWarps * 2 + 2 + 3) * kResTile * 4;

// set when a tile barrier wait times out (a co-residency failure): read by bn_resident_error(), never cleared by a kernel
__device__ unsigned int g_bn_resident_error = 0;

struct ResGeom {
  int R, C;
  int T;          // channel tiles per wave
  int P;          // CTAs per tile (row slabs); grid = T * P
  int box_rows;   // rows per TMA box
  int nbox;       // boxes per CTA: a CTA's slab is nbox * box_rows rows
  int waves;      // waves of this launch
  int tile0;      // first channel tile of this launch: wave w, slot s runs tile tile0 + w * T + s
  int tile_end;   // one past the last channel tile of this launch
};

// Barrier of the P CTAs of one channel tile on that tile slot's two workspace words {arrivals, generation}: a tile
// depends only on its own partials, so tiles of a wave proceed independently.  Co-residency is guaranteed by the
// cooperative launch, and the wait is still bounded (2 s) so that a failure surfaces as an error word instead of a hung GPU.
__device__ __forceinline__ void res_tile_sync(unsigned int* bar, unsigned int nblocks) {
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int* gen = bar + 1;
    const unsigned int g0 = bn_ld_acquire(gen);
    // acq_rel: releases this CTA's partial row (ordered before it by the bar.sync above), acquires the earlier arrivals'
    unsigned int old;
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(old) : "l"(bar) : "memory");
    if (old == nblocks - 1) {
      asm volatile("st.relaxed.gpu.global.u32 [%0], 0;" ::"l"(bar) : "memory");   // ready for the next wave / launch
      bn_st_release(gen, g0 + 1u);
    } else {
      unsigned long long t0;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      while (bn_ld_acquire(gen) == g0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (t - t0 > 2000000000ull) { atomicExch(&g_bn_resident_error, 1u); break; }
      }
    }
  }
  __syncthreads();
}

// Sum the 8 channels' two accumulators over the 4 row lanes of a warp, then over the warps in a fixed order, and write this
// CTA's [2][64] partial row to partial[(a * P + p) * C + c0 + c].
__device__ __forceinline__ void res_write_partials(float (&acc)[2][kVec], float* red, float* __restrict__ partial, int P, int p, int C,
                                                   int c0) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cv = threadIdx.x & 7;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      float v = acc[a][i];
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane < 8) red[(warp * 2 + a) * kResTile + cv * kVec + i] = v;
    }
  __syncthreads();
  if (threadIdx.x < 2 * kResTile) {
    const int a = threadIdx.x / kResTile, c = threadIdx.x % kResTile;
    float s = 0.f;
    for (int w = 0; w < kResWarps; ++w) s += red[(w * 2 + a) * kResTile + c];
    if (c0 + c < C) partial[((size_t)a * P + p) * C + c0 + c] = s;
  }
}

// After the tile barrier: the tile's P partial rows, summed in a fixed order (identical in every CTA of the tile).
// On return red[a * 64 + c] (a = 0: sum, 1: second moment) holds the totals of channel c0 + c.
__device__ __forceinline__ void res_reduce_partials(float* red, const float* __restrict__ partial, int P, int C, int c0) {
  const int q = threadIdx.x & 31, l = threadIdx.x >> 5;       // 2 x 16 float4 columns x 8 lanes
  const int a = q >> 4, c4 = (q & 15) * 4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c0 + c4 < C) {
    // every load of the thread is issued before the first add: one L2 round trip on the critical path instead of P / 32
    const float* base = partial + (size_t)a * P * C + c0 + c4;
    float4 v[kResMaxPartialLoads];
#pragma unroll
    for (int j = 0; j < kResMaxPartialLoads; ++j)
      if (l + j * kResWarps < P) v[j] = __ldcg(reinterpret_cast<const float4*>(base + (size_t)(l + j * kResWarps) * C));
#pragma unroll
    for (int j = 0; j < kResMaxPartialLoads; ++j)
      if (l + j * kResWarps < P) { s.x += v[j].x; s.y += v[j].y; s.z += v[j].z; s.w += v[j].w; }
  }
  __syncthreads();                                           // red may still be read by res_write_partials' tail
  *reinterpret_cast<float4*>(red + (l * 2 + a) * kResTile + c4) = s;
  __syncthreads();
  if (threadIdx.x < 2 * kResTile) {
    const int aa = threadIdx.x / kResTile, c = threadIdx.x % kResTile;
    float t = 0.f;
    for (int w = 0; w < kResWarps; ++w) t += red[(w * 2 + aa) * kResTile + c];
    red[kResWarps * 2 * kResTile + aa * kResTile + c] = t;    // staged behind the scratch: other threads may still read it
  }
  __syncthreads();
}

__device__ __forceinline__ void res_ld8(const unsigned char* s, float* f) { unpack8(*reinterpret_cast<const Bf16x8*>(s), f); }
__device__ __forceinline__ void res_st8(unsigned char* s, const float* f) { *reinterpret_cast<Bf16x8*>(s) = pack8(f); }

// Forward: statistics, running statistics, y = relu(x*scale + shift (+ residual)) and the ReLU bitmask, x read once.
__global__ void __launch_bounds__(kResThreads, 1)
bn_resident_fwd_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                       const __grid_constant__ CUtensorMap map_res, const __nv_bfloat16* __restrict__ residual, unsigned char* __restrict__ mask, const float* __restrict__ gamma,
                       const float* __restrict__ beta, float* __restrict__ running_mean, float* __restrict__ running_var,
                       long long* __restrict__ num_batches, float* __restrict__ save_mean, float* __restrict__ save_rstd,
                       float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ partial, unsigned int* __restrict__ bar,
                       float eps, float momentum, int relu, const ResGeom g) {
  extern __shared__ __align__(128) unsigned char res_smem[];
  const int slab_rows = g.nbox * g.box_rows;
  const uint32_t box_bytes = (uint32_t)g.box_rows * kResTile * 2;
  unsigned char* data = res_smem;
  uint64_t* mbar = reinterpret_cast<uint64_t*>(res_smem + (size_t)slab_rows * kResTile * 2);
  float* red = reinterpret_cast<float*>(mbar + kResMaxBoxes);       // [warps][2][64], then [2][64] totals
  float* coef = red + kResWarps * 2 * kResTile + 2 * kResTile;        // [2][64] scale, shift
  const int cv = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int cvs = g.C / kVec;
  const int slot = blockIdx.x / g.P, p = blockIdx.x % g.P;
  const int r0 = p * slab_rows;
  const int nlive = r0 >= g.R ? 0 : min(g.nbox, (g.R - r0 + g.box_rows - 1) / g.box_rows);
  bar += 2 * slot;
  // box b of the slab of tile t (the first wave's loads here; later waves' loads are issued box by box during the
  // previous wave's apply, as soon as the box's store has read it)
  auto load_box = [&](int b, int t) {
    tc::mbar_expect_tx(&mbar[b], box_bytes);
    tc::tma_load_2d(&map_x, &mbar[b], data + (size_t)b * box_bytes, t * kResTile, r0 + b * g.box_rows);
  };
  if (threadIdx.x == 0) {
    for (int b = 0; b < g.nbox; ++b) tc::mbar_init(&mbar[b], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tc::tma_prefetch_desc(&map_x);
    tc::tma_prefetch_desc(&map_y);
    if (blockIdx.x == 0 && g.tile0 == 0 && num_batches != nullptr) *num_batches += 1;
    if (g.tile0 + slot < g.tile_end)
      for (int b = 0; b < nlive; ++b) load_box(b, g.tile0 + slot);
  }
  __syncthreads();
  for (int w = 0; w < g.waves; ++w) {
    const int t = g.tile0 + w * g.T + slot;
    if (t >= g.tile_end) break;                                       // the whole tile slot is done: no later wave either
    const bool next = t + g.T < g.tile_end;
    const int c0 = t * kResTile;
    const int cvg = t * (kResTile / kVec) + cv;                       // global channel vector of this thread
    // per-channel inputs of the coefficients, read before the barrier so that their latency is off the critical path
    float gm = 0.f, bt = 0.f, rmean = 0.f, rvar = 0.f;
    if (threadIdx.x < kResTile && c0 + (int)threadIdx.x < g.C) {
      const int ch = c0 + threadIdx.x;
      gm = gamma[ch];
      bt = beta[ch];
      if (p == 0 && running_mean != nullptr) { rmean = running_mean[ch]; rvar = running_var[ch]; }
    }
    float acc[2][kVec];
#pragma unroll
    for (int i = 0; i < kVec; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    {
      for (int b = 0; b < nlive; ++b) {
        tc::mbar_wait(&mbar[b], (uint32_t)(w & 1));
        const unsigned char* box = data + (size_t)b * box_bytes + cv * 16;
        for (int rr = rl; rr < g.box_rows; rr += 4 * 32) {            // rows past R and channels past C are zero-filled
          float f[4][kVec];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (rr + u * 32 < g.box_rows) res_ld8(box + (size_t)(rr + u * 32) * (kResTile * 2), f[u]);
            else
#pragma unroll
              for (int i = 0; i < kVec; ++i) f[u][i] = 0.f;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int i = 0; i < kVec; ++i) { acc[0][i] += f[u][i]; acc[1][i] = fmaf(f[u][i], f[u][i], acc[1][i]); }
        }
      }
      if (residual != nullptr && threadIdx.x == 0) {
        // the residual slab is read right after the barrier: stage it in L2 while the grid synchronises
        for (int b = 0; b < nlive; ++b)
          asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];"
                       ::"l"(reinterpret_cast<uint64_t>(&map_res)), "r"(c0), "r"(r0 + b * g.box_rows) : "memory");
      }
      res_write_partials(acc, red, partial, g.P, p, g.C, c0);
    }
    // the residual rows of box b this thread adds: a box has at most 8 * 32 rows, row lane rl owns rows rl + 32 u
    const bool live_cv = cvg < cvs;
    auto load_res = [&](int b, Bf16x8 (&d)[8]) {
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int q = rl + u * 32, r = r0 + b * g.box_rows + q;
        if (residual != nullptr && q < g.box_rows && r < g.R && live_cv)
          d[u] = *reinterpret_cast<const Bf16x8*>(residual + (size_t)r * g.C + (size_t)cvg * kVec);
      }
    };
    Bf16x8 rv[8];
    if (nlive > 0) load_res(0, rv);                                   // box 0's residual: in flight across the barrier
    res_tile_sync(bar, g.P);
    res_reduce_partials(red, partial, g.P, g.C, c0);
    if (threadIdx.x < kResTile) {
      const float* tot = red + kResWarps * 2 * kResTile;
      const int c = threadIdx.x, ch = c0 + c;
      if (ch < g.C) {
        const float inv_r = 1.f / (float)g.R;
        const float mean = tot[c] * inv_r;
        const float var = fmaxf(tot[kResTile + c] * inv_r - mean * mean, 0.f);     // biased variance (normalisation)
        const float rstd = rsqrtf(var + eps);
        const float sc = gm * rstd;
        const float sh = bt - mean * sc;
        coef[c] = sc;
        coef[kResTile + c] = sh;
        if (p == 0) {
          save_mean[ch] = mean;
          save_rstd[ch] = rstd;
          scale[ch] = sc;
          shift[ch] = sh;
          if (running_mean != nullptr) {
            const float unbiased = g.R > 1 ? var * ((float)g.R / (float)(g.R - 1)) : var;
            running_mean[ch] = (1.f - momentum) * rmean + momentum * mean;
            running_var[ch] = (1.f - momentum) * rvar + momentum * unbiased;
          }
        }
      } else {
        coef[c] = 0.f;
        coef[kResTile + c] = 0.f;
      }
    }
    __syncthreads();
    float sc[kVec], sh[kVec];
#pragma unroll
    for (int i = 0; i < kVec; ++i) { sc[i] = coef[cv * kVec + i]; sh[i] = coef[kResTile + cv * kVec + i]; }
    for (int b = 0; b < nlive; ++b) {
      unsigned char* box = data + (size_t)b * box_bytes + cv * 16;
      const int rb = r0 + b * g.box_rows;
      Bf16x8 rn[8];
      if (b + 1 < nlive) load_res(b + 1, rn);                         // in flight while this box is normalised
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int q = rl + u * 32, r = rb + q;
        if (!(q < g.box_rows && r < g.R && live_cv)) continue;
        float f[kVec], rs[kVec];
        res_ld8(box + (size_t)q * (kResTile * 2), f);
        if (residual != nullptr) unpack8(rv[u], rs);
        unsigned int bits = 0;
#pragma unroll
        for (int i = 0; i < kVec; ++i) {
          float v = fmaf(f[i], sc[i], sh[i]);
          if (residual != nullptr) v += rs[i];
          bits |= (v > 0.f ? 1u : 0u) << i;
          f[i] = relu ? fmaxf(v, 0.f) : v;
        }
        res_st8(box + (size_t)q * (kResTile * 2), f);
        if (mask != nullptr) mask[(size_t)r * cvs + cvg] = (unsigned char)bits;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) rv[u] = rn[u];
      tc::fence_async_smem();
      __syncthreads();
      if (threadIdx.x == 0) {
        tc::tma_store_2d(&map_y, data + (size_t)b * box_bytes, c0, rb);
        tc::bulk_commit();
        // the next wave's load into the previous box, once that box's store has read it: HBM streams the next wave's
        // x while this wave's y drains
        if (next && b > 0) { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); load_box(b - 1, t + g.T); }
      }
    }
    if (threadIdx.x == 0) {
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      if (next && nlive > 0) load_box(nlive - 1, t + g.T);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) tc::bulk_wait_all();
}

// Backward: S1 = sum dy*, S2 = sum dy* xhat (dy* = dy masked by the forward ReLU), dgamma / dbeta, then
// dx = a*dy* + b*x + c and the residual branch's gradient dy*, with dy and x read once.
__global__ void __launch_bounds__(kResThreads, 1)
bn_resident_bwd_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x,
                       const __grid_constant__ CUtensorMap map_dx, const __grid_constant__ CUtensorMap map_dres,
                       const unsigned char* __restrict__ mask, const float* __restrict__ save_mean, const float* __restrict__ save_rstd,
                       const float* __restrict__ gamma, float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ coef_out,
                       float* __restrict__ partial, unsigned int* __restrict__ bar, int relu, int want_dres, const ResGeom g) {
  extern __shared__ __align__(128) unsigned char res_smem[];
  const int slab_rows = g.nbox * g.box_rows;
  const uint32_t box_bytes = (uint32_t)g.box_rows * kResTile * 2;
  unsigned char* dyd = res_smem;                                      // dy slab, then dy* (the residual gradient)
  unsigned char* xd = res_smem + (size_t)slab_rows * kResTile * 2;    // x slab, then dx
  uint64_t* mbar = reinterpret_cast<uint64_t*>(res_smem + (size_t)2 * slab_rows * kResTile * 2);
  float* red = reinterpret_cast<float*>(mbar + kResMaxBoxes);
  float* coef = red + kResWarps * 2 * kResTile + 2 * kResTile;        // [3][64] a, b, c
  unsigned char* smask = reinterpret_cast<unsigned char*>(coef + 3 * kResTile);   // [slab rows][8] ReLU mask bytes of the tile
  const int cv = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int cvs = g.C / kVec;
  const int slot = blockIdx.x / g.P, p = blockIdx.x % g.P;
  const int r0 = p * slab_rows;
  const int nlive = r0 >= g.R ? 0 : min(g.nbox, (g.R - r0 + g.box_rows - 1) / g.box_rows);
  // whole tiles of channels and an 8-byte aligned mask: a row's 8 mask bytes of a tile are one aligned 8-byte word
  const bool mask_words = g.C % kResTile == 0 && (reinterpret_cast<uintptr_t>(mask) & 7u) == 0;
  bar += 2 * slot;
  // box b of the dy and x slabs of tile t (the first wave's loads here; later waves' loads are issued box by box during
  // the previous wave's apply, as soon as the box's stores have read it)
  auto load_box = [&](int b, int t) {
    tc::mbar_expect_tx(&mbar[b], 2 * box_bytes);
    tc::tma_load_2d(&map_dy, &mbar[b], dyd + (size_t)b * box_bytes, t * kResTile, r0 + b * g.box_rows);
    tc::tma_load_2d(&map_x, &mbar[b], xd + (size_t)b * box_bytes, t * kResTile, r0 + b * g.box_rows);
  };
  if (threadIdx.x == 0) {
    for (int b = 0; b < g.nbox; ++b) tc::mbar_init(&mbar[b], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tc::tma_prefetch_desc(&map_dy);
    tc::tma_prefetch_desc(&map_x);
    if (g.tile0 + slot < g.tile_end)
      for (int b = 0; b < nlive; ++b) load_box(b, g.tile0 + slot);
  }
  __syncthreads();
  for (int w = 0; w < g.waves; ++w) {
    const int t = g.tile0 + w * g.T + slot;
    if (t >= g.tile_end) break;                                       // the whole tile slot is done: no later wave either
    const bool next = t + g.T < g.tile_end;
    const int c0 = t * kResTile;
    const int cvg = t * (kResTile / kVec) + cv;
    const bool live_cv = cvg < cvs;
    // per-channel inputs of the coefficients, read before the barrier so that their latency is off the critical path
    float gam = 0.f, smean = 0.f, srstd = 0.f;
    if (threadIdx.x < kResTile && c0 + (int)threadIdx.x < g.C) {
      const int ch = c0 + threadIdx.x;
      gam = gamma[ch];
      smean = save_mean[ch];
      srstd = save_rstd[ch];
    }
    if (relu) {
      // the slab's mask bytes (1/16 of its dy bytes), used by both passes: independent loads, overlapped with the TMA loads
      const int rows = min(slab_rows, g.R - r0);
      if (mask_words) {
#pragma unroll 4
        for (int i = threadIdx.x; i < rows; i += kResThreads)
          reinterpret_cast<unsigned long long*>(smask)[i] =
              *reinterpret_cast<const unsigned long long*>(mask + (size_t)(r0 + i) * cvs + t * (kResTile / kVec));
      } else {
#pragma unroll 8
        for (int i = threadIdx.x; i < rows * 8; i += kResThreads) {
          const int cg = t * (kResTile / kVec) + (i & 7);
          smask[i] = cg < cvs ? mask[(size_t)(r0 + (i >> 3)) * cvs + cg] : 0u;
        }
      }
      __syncthreads();
    }
    float acc[2][kVec];
#pragma unroll
    for (int i = 0; i < kVec; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    {
      float mean[kVec], rstd[kVec];
#pragma unroll
      for (int i = 0; i < kVec; ++i) { mean[i] = 0.f; rstd[i] = 0.f; }
      if (live_cv) { bn_load8<float>(save_mean + cvg * kVec, mean); bn_load8<float>(save_rstd + cvg * kVec, rstd); }
      for (int b = 0; b < nlive; ++b) {
        tc::mbar_wait(&mbar[b], (uint32_t)(w & 1));
        // rows past R and channels past C hold zero dy (TMA zero fill): they add nothing whatever their mask byte says
        for (int rr = rl; rr < g.box_rows; rr += 2 * 32) {
          float gv[2][kVec], xv[2][kVec];
          unsigned int mk[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int q = min(rr + u * 32, g.box_rows - 1);           // a clamped duplicate row is masked out below
            res_ld8(dyd + (size_t)b * box_bytes + (size_t)q * (kResTile * 2) + cv * 16, gv[u]);
            res_ld8(xd + (size_t)b * box_bytes + (size_t)q * (kResTile * 2) + cv * 16, xv[u]);
            mk[u] = rr + u * 32 < g.box_rows ? (relu ? smask[(b * g.box_rows + q) * 8 + cv] : 0xffu) : 0u;
          }
#pragma unroll
          for (int u = 0; u < 2; ++u)
#pragma unroll
            for (int i = 0; i < kVec; ++i) {
              const float gm = ((mk[u] >> i) & 1u) ? gv[u][i] : 0.f;
              acc[0][i] += gm;
              acc[1][i] = fmaf(gm, (xv[u][i] - mean[i]) * rstd[i], acc[1][i]);
            }
        }
      }
      res_write_partials(acc, red, partial, g.P, p, g.C, c0);
    }
    res_tile_sync(bar, g.P);
    res_reduce_partials(red, partial, g.P, g.C, c0);
    if (threadIdx.x < kResTile) {
      const float* tot = red + kResWarps * 2 * kResTile;
      const int c = threadIdx.x, ch = c0 + c;
      float ka = 0.f, kb = 0.f, kc = 0.f;
      if (ch < g.C) {
        const float inv_r = 1.f / (float)g.R;
        const float s1 = tot[c], s2 = tot[kResTile + c];
        const float c1 = s1 * inv_r, c2 = s2 * inv_r;                 // mean(dy*), mean(dy* xhat)
        const float mean = smean, rstd = srstd;
        ka = gam * rstd;
        kb = -ka * rstd * c2;
        kc = -ka * (c1 - mean * rstd * c2);
        if (p == 0) {
          dbeta[ch] = s1;
          dgamma[ch] = s2;
          coef_out[ch] = c1;
          coef_out[g.C + ch] = c2;
        }
      }
      coef[c] = ka;
      coef[kResTile + c] = kb;
      coef[2 * kResTile + c] = kc;
    }
    __syncthreads();
    float ka[kVec], kb[kVec], kc[kVec];
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      ka[i] = coef[cv * kVec + i];
      kb[i] = coef[kResTile + cv * kVec + i];
      kc[i] = coef[2 * kResTile + cv * kVec + i];
    }
    for (int b = 0; b < nlive; ++b) {
      const int rb = r0 + b * g.box_rows;
      unsigned char* gbox = dyd + (size_t)b * box_bytes + cv * 16;
      unsigned char* xbox = xd + (size_t)b * box_bytes + cv * 16;
      for (int rr = rl; rr < g.box_rows; rr += 2 * 32) {
        float gv[2][kVec], xv[2][kVec];
        unsigned int mk[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int q = min(rr + u * 32, g.box_rows - 1);
          res_ld8(gbox + (size_t)q * (kResTile * 2), gv[u]);
          res_ld8(xbox + (size_t)q * (kResTile * 2), xv[u]);
          mk[u] = relu ? smask[(b * g.box_rows + q) * 8 + cv] : 0xffu;
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          if (rr + u * 32 >= g.box_rows) continue;
          const size_t off = (size_t)(rr + u * 32) * (kResTile * 2);
          float o[kVec];
#pragma unroll
          for (int i = 0; i < kVec; ++i) {
            if (!((mk[u] >> i) & 1u)) gv[u][i] = 0.f;
            o[i] = fmaf(ka[i], gv[u][i], fmaf(kb[i], xv[u][i], kc[i]));
          }
          if (want_dres) res_st8(gbox + off, gv[u]);
          res_st8(xbox + off, o);
        }
      }
      tc::fence_async_smem();
      __syncthreads();
      if (threadIdx.x == 0) {
        tc::tma_store_2d(&map_dx, xd + (size_t)b * box_bytes, c0, rb);
        if (want_dres) tc::tma_store_2d(&map_dres, dyd + (size_t)b * box_bytes, c0, rb);
        tc::bulk_commit();
        // the next wave's loads into the previous box, once that box's stores have read it: HBM streams the next wave's
        // dy and x while this wave's dx (and dres) drain
        if (next && b > 0) { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); load_box(b - 1, t + g.T); }
      }
    }
    if (threadIdx.x == 0) {
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      if (next && nlive > 0) load_box(nlive - 1, t + g.T);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) tc::bulk_wait_all();
}

int g_bn_two_pass = 0;     // 1: the resident kernels are never selected (comparisons, benchmarks)

bool resident_allowed() {
  static int fused_env = -1;
  if (fused_env < 0) { const char* e = getenv("B200DDP_BN_FUSED"); fused_env = (e && atoi(e) == 1) ? 1 : 0; }
  return !g_bn_two_pass && !fused_env && !bn_pdl_enabled();
}

struct ResPlan {
  bool ok = false;
  ResGeom g{};        // geometry of the first launch; launch k runs tiles [k * T * waves, (k + 1) * T * waves)
  int launches = 0;
  int grid = 0;
  int smem = 0;
};

// Largest wave (channel tiles per wave) whose slabs fit in the co-resident CTAs' shared memory.  streams = 1 (forward: x) or
// 2 (backward: dy and x).  Computed once per (device, R, C, streams).
ResPlan resident_plan(int R, int C, int streams) {
  static std::mutex mu;
  static std::map<std::pair<int, std::pair<long long, int>>, ResPlan> cache;
  int dev = 0;
  B200_CUDA_CHECK(cudaGetDevice(&dev));
  const auto key = std::make_pair(dev, std::make_pair(((long long)R << 20) | (long long)C, streams));
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  ResPlan plan;
  int sms = 0, optin = 0;
  B200_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B200_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const long long budget = (long long)optin - kResFixedSmem - 1024;     // slabs; 1 KB for the runtime's static reservation
  const int ntiles = (C + kResTile - 1) / kResTile;
  const long long row_bytes = (long long)kResTile * 2 * streams + (streams == 2 ? 8 : 0);   // backward: + the mask bytes
  for (int T = ntiles; T >= 1 && R > 0; --T) {
    int P = std::min(sms / T, kResMaxPartialLoads * kResWarps);
    if (P < 1) continue;
    P = std::min(P, std::max(1, (R + 31) / 32));                        // >= 32 rows per CTA
    const int need = (R + P - 1) / P;
    const int nbox = (need + kResMaxBox - 1) / kResMaxBox;
    if (nbox > kResMaxBoxes) continue;
    const int box_rows = (need + nbox - 1) / nbox;
    const long long slab = (long long)nbox * box_rows * row_bytes;
    if (slab > budget) continue;
    const int waves = (ntiles + T - 1) / T;
    if (waves > kResMaxLaunches * kResMaxWaves) break;                  // fewer tiles per wave only adds waves
    plan.launches = (waves + kResMaxWaves - 1) / kResMaxWaves;
    const int per_launch = (waves + plan.launches - 1) / plan.launches;
    plan.g = ResGeom{R, C, T, (R + nbox * box_rows - 1) / (nbox * box_rows), box_rows, nbox, per_launch, 0, std::min(ntiles, T * per_launch)};
    plan.grid = plan.g.T * plan.g.P;
    plan.smem = (int)slab + kResFixedSmem;
    plan.ok = true;
    break;
  }
  cache.emplace(key, plan);
  return plan;
}

// Geometry of launch k of a plan: the k-th contiguous range of T * waves channel tiles.
ResGeom res_launch(const ResPlan& plan, int k) {
  ResGeom g = plan.g;
  g.tile0 = k * g.T * g.waves;
  g.tile_end = std::min((g.C + kResTile - 1) / kResTile, g.tile0 + g.T * g.waves);
  return g;
}

// [R, C] bf16, row-major, 64-channel x box_rows boxes, no swizzle; out-of-range rows / channels read as zero, stores clip.
CUtensorMap res_map(const void* ptr, int R, int C, int box_rows) {
  auto& drv = Driver::get();
  if (!drv.TensorMapEncodeTiled) throw std::runtime_error("batch norm: cuTensorMapEncodeTiled unavailable");
  CUtensorMap map;
  cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)R};
  cuuint64_t strides[1] = {(cuuint64_t)C * 2};
  cuuint32_t box[2] = {(cuuint32_t)kResTile, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  B200_DRV_CHECK(drv.TensorMapEncodeTiled(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
  return map;
}

int res_smem_limit() {
  int dev = 0, optin = 0;
  B200_CUDA_CHECK(cudaGetDevice(&dev));
  B200_CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  return optin;
}

bool res_aligned(const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <typename... KArgs, typename... Args>
void launch_cooperative(void (*kernel)(KArgs...), const ResPlan& plan, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(plan.grid);
  cfg.blockDim = dim3(kResThreads);
  cfg.dynamicSmemBytes = plan.smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
}

}  // namespace

// ------------------------------------------------------------------------------------------------------
// Statistics from the producing convolution's epilogue (csrc/conv_wgmma.cu): partial = [2][G][C] per-CTA column sums and
// sums of squares, G <= 132.  NO separate finishing launch: every block of the normalisation kernel first reduces the G
// rows of ITS <= 64 channels (a few tens of KB out of L2, fixed order -> deterministic), then normalises its rows; the
// blocks of the first row split also publish mean / rstd (for the backward pass) and update the running statistics.
template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_apply_partials_kernel(const T* __restrict__ x, const T* __restrict__ residual, T* __restrict__ y,
                                                                      unsigned char* __restrict__ mask, const float* __restrict__ partial, int G,
                                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                      float* __restrict__ running_mean, float* __restrict__ running_var,
                                                                      long long* __restrict__ num_batches, float* __restrict__ save_mean,
                                                                      float* __restrict__ save_rstd, float eps, float momentum, int R, int C,
                                                                      int cvb, int ty, int relu) {
  extern __shared__ float bn_smem[];                 // [2][ty][cvb*8] reduction scratch, then [2][cvb*8] scale / shift
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  const bool live = cv * kVec < C;
  float acc[2][kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  if (live) {
    for (int g = tyi; g < G; g += ty) {
      float a[kVec], b[kVec];
      bn_load8<float>(partial + (size_t)g * C + cv * kVec, a);
      bn_load8<float>(partial + ((size_t)G + g) * C + cv * kVec, b);
#pragma unroll
      for (int i = 0; i < kVec; ++i) { acc[0][i] += a[i]; acc[1][i] += b[i]; }
    }
  }
  reduce_rows<2>(acc, bn_smem, tx, tyi, cvb, ty);
  const int width = cvb * kVec;
  float* sc_s = bn_smem + 2 * ty * width;            // scale / shift of this block's channels
  float* sh_s = sc_s + width;
  if (tyi == 0 && live) {
    const float inv_r = 1.f / (float)R;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int ch = cv * kVec + i;
      const float sum = bn_smem[tx * kVec + i], sq = bn_smem[ty * width + tx * kVec + i];
      const float mean = sum * inv_r;
      const float var = fmaxf(sq * inv_r - mean * mean, 0.f);
      const float rstd = rsqrtf(var + eps);
      const float sc = gamma[ch] * rstd;
      sc_s[tx * kVec + i] = sc;
      sh_s[tx * kVec + i] = beta[ch] - mean * sc;
      if (blockIdx.y == 0) {
        save_mean[ch] = mean;
        save_rstd[ch] = rstd;
        if (running_mean != nullptr) {
          const float unbiased = R > 1 ? var * ((float)R / (float)(R - 1)) : var;
          running_mean[ch] = (1.f - momentum) * running_mean[ch] + momentum * mean;
          running_var[ch] = (1.f - momentum) * running_var[ch] + momentum * unbiased;
        }
      }
    }
  }
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && num_batches != nullptr) *num_batches += 1;
  __syncthreads();
  if (!live) return;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  // bn_apply_rows indexes scale / shift by the global channel vector: hand it pointers rebased to this block's tile
  bn_apply_rows<T>(x, residual, y, mask, sc_s - (size_t)blockIdx.x * width, sh_s - (size_t)blockIdx.x * width, C, cv, r0, r1, tyi, ty, relu);
}

// Backward twin: partial = [2][G][C] with S1 = sum dy*m and S2 = sum dy*m*xhat from the data-gradient epilogue of the convolution
// that consumes this BatchNorm's output.  Every block reduces its channels' G rows, forms c1 = S1/R, c2 = S2/R, applies
// dx = gamma*rstd*(dy*m - c1 - xhat*c2); the first row split also writes dgamma = S2, dbeta = S1.
template <typename T>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_apply_partials_kernel(const T* __restrict__ dy, const T* __restrict__ x, const unsigned char* __restrict__ y,
                                                                          T* __restrict__ dx, T* __restrict__ dres, const float* __restrict__ partial, int G,
                                                                          const float* __restrict__ save_mean, const float* __restrict__ save_rstd,
                                                                          const float* __restrict__ gamma, float* __restrict__ dgamma,
                                                                          float* __restrict__ dbeta, int R, int C, int cvb, int ty, int relu) {
  extern __shared__ float bn_smem[];                 // [2][ty][cvb*8] reduction scratch, then [2][cvb*8] coefficients
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  const bool live = cv * kVec < C;
  float acc[2][kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  if (live) {
    for (int g = tyi; g < G; g += ty) {
      float a[kVec], b[kVec];
      bn_load8<float>(partial + (size_t)g * C + cv * kVec, a);
      bn_load8<float>(partial + ((size_t)G + g) * C + cv * kVec, b);
#pragma unroll
      for (int i = 0; i < kVec; ++i) { acc[0][i] += a[i]; acc[1][i] += b[i]; }
    }
  }
  reduce_rows<2>(acc, bn_smem, tx, tyi, cvb, ty);
  const int width = cvb * kVec;
  float* c1_s = bn_smem + 2 * ty * width;            // coef layout expected by bn_bwd_apply_rows: c1 at [0, C), c2 at [C, 2C)
  float* c2_s = c1_s + width;
  if (tyi == 0 && live) {
    const float inv_r = 1.f / (float)R;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int ch = cv * kVec + i;
      const float s1 = bn_smem[tx * kVec + i], s2 = bn_smem[ty * width + tx * kVec + i];
      c1_s[tx * kVec + i] = s1 * inv_r;
      c2_s[tx * kVec + i] = s2 * inv_r;
      if (blockIdx.y == 0) { dgamma[ch] = s2; dbeta[ch] = s1; }
    }
  }
  __syncthreads();
  if (!live) return;
  const int S = gridDim.y;
  const int rows_per = (R + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  // bn_bwd_apply_rows reads coef[cv*8 + i] and coef[C + cv*8 + i]: rebase so that both land in this block's two smem rows
  // (c2 row sits `width` floats after c1: a fake "C" of `width` would break the global indexing of the other operands, so the
  // coefficients are passed through a two-pointer variant)
  bn_bwd_apply_rows_coef<T>(dy, x, y, dx, dres, save_mean, save_rstd, gamma, c1_s + tx * kVec, c2_s + tx * kVec, C, cv, r0, r1, tyi, ty, relu);
}

void set_bn_pdl(int on) { g_bn_pdl = on; }

void set_bn_two_pass(int on) { g_bn_two_pass = on ? 1 : 0; }

unsigned int bn_resident_error() {
  unsigned int v = 0;
  B200_CUDA_CHECK(cudaMemcpyFromSymbol(&v, g_bn_resident_error, sizeof(v)));
  return v;
}

// Sizes the workspace of both paths and plans the resident kernels of this shape (cached for the launches).
void bn_workspace_sizes(int R, int C, size_t* partial_floats, size_t* counters) {
  const Tile t = pick_tile(R, C);
  const ResPlan fwd = resident_plan(R, C, 1), bwd = resident_plan(R, C, 2);
  const int p = std::max(fwd.ok ? fwd.g.P : 0, bwd.ok ? bwd.g.P : 0);
  *partial_floats = (size_t)2 * std::max(t.grid_y, p) * C;
  // tickets + generation words of the two-pass kernels, then one {arrivals, generation} pair per resident tile slot
  *counters = (size_t)2 * t.grid_x + 2 * (size_t)((C + kResTile - 1) / kResTile);
}

void launch_bn_forward(const void* x, const void* residual, void* y, unsigned char* mask, DType dt, int R, int C, const float* gamma, const float* beta,
                       float* running_mean, float* running_var, long long* num_batches, float* save_mean, float* save_rstd,
                       float* scale, float* shift, float* partial, unsigned int* counters, float eps, float momentum, bool relu,
                       cudaStream_t s) {
  if (C % kVec != 0) throw std::runtime_error("fused batch norm: channel count must be a multiple of 8");
  const int r = relu ? 1 : 0;
  if (dt == DType::BF16 && resident_allowed() && res_aligned(x) && res_aligned(residual) && res_aligned(y)) {
    const ResPlan plan = resident_plan(R, C, 1);
    if (plan.ok) {
      static std::atomic<unsigned long long> smem_done{0};
      ensure_max_dynamic_smem(bn_resident_fwd_kernel, res_smem_limit(), smem_done);    // raised once: every plan fits below it
      const CUtensorMap mx = res_map(x, R, C, plan.g.box_rows), my = res_map(y, R, C, plan.g.box_rows);
      const CUtensorMap mres = residual != nullptr ? res_map(residual, R, C, plan.g.box_rows) : mx;
      for (int k = 0; k < plan.launches; ++k)
        launch_cooperative(bn_resident_fwd_kernel, plan, s, mx, my, mres, (const __nv_bfloat16*)residual, mask, gamma, beta, running_mean,
                           running_var, num_batches, save_mean, save_rstd, scale, shift, partial, counters + 2 * pick_tile(R, C).grid_x, eps,
                           momentum, r, res_launch(plan, k));
      B200_COUNT_LAUNCH(plan.launches);
      return;
    }
  }
  Tile t;
  const bool fused = fused_tile(R, C, &t);
  const size_t smem = (size_t)2 * t.ty * t.cvb * kVec * sizeof(float);
  const dim3 grid(t.grid_x, t.grid_y);
  if (!fused && bn_pdl_enabled()) {
    // opt-in: producer with an early launch_dependents, apply kernel as its programmatic dependent
#define B200_BN_FWD_PDL(T)                                                                                                                  \
    bn_stats_kernel<T, false, true><<<grid, kBnThreads, smem, s>>>((const T*)x, R, C, t.cvb, t.ty, partial, counters, gamma, beta, running_mean, \
                                                                   running_var, num_batches, save_mean, save_rstd, scale, shift, eps, momentum,  \
                                                                   (const T*)residual, (T*)y, mask, r);                                          \
    B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);                                                                                   \
    launch_dependent(bn_apply_pdl_kernel<T>, apply_grid(t, R), s, (const T*)x, (const T*)residual, (T*)y, mask, (const float*)scale,              \
                     (const float*)shift, R, C, t.cvb, t.ty, r);                                                                                  \
    B200_COUNT_LAUNCH(1)
    if (dt == DType::BF16) { B200_BN_FWD_PDL(__nv_bfloat16); } else { B200_BN_FWD_PDL(float); }
#undef B200_BN_FWD_PDL
    return;
  }
#define B200_BN_FWD(T, F)                                                                                                            \
  bn_stats_kernel<T, F><<<grid, kBnThreads, smem, s>>>((const T*)x, R, C, t.cvb, t.ty, partial, counters, gamma, beta, running_mean, \
                                                       running_var, num_batches, save_mean, save_rstd, scale, shift, eps, momentum, \
                                                       (const T*)residual, (T*)y, mask, r)
  if (dt == DType::BF16) { if (fused) B200_BN_FWD(__nv_bfloat16, true); else B200_BN_FWD(__nv_bfloat16, false); }
  else { if (fused) B200_BN_FWD(float, true); else B200_BN_FWD(float, false); }
#undef B200_BN_FWD
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  if (fused) return;
  if (dt == DType::BF16)
    bn_apply_kernel<__nv_bfloat16><<<apply_grid(t, R), kBnThreads, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)residual,
                                                                           (__nv_bfloat16*)y, mask, scale, shift, R, C, t.cvb, t.ty, r);
  else
    bn_apply_kernel<float><<<apply_grid(t, R), kBnThreads, 0, s>>>((const float*)x, (const float*)residual, (float*)y, mask, scale, shift, R, C,
                                                                   t.cvb, t.ty, r);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_bn_forward_from_partials(const void* x, const void* residual, void* y, unsigned char* mask, DType dt, int R, int C,
                                     const float* gamma, const float* beta, float* running_mean, float* running_var,
                                     long long* num_batches, float* save_mean, float* save_rstd, float* scale, float* shift,
                                     const float* partial, int groups, float eps, float momentum, bool relu, cudaStream_t s) {
  (void)scale; (void)shift;                          // each block derives them for its own channels (see bn_apply_partials_kernel)
  if (C % kVec != 0) throw std::runtime_error("fused batch norm: channel count must be a multiple of 8");
  if (groups < 1) throw std::runtime_error("fused batch norm: empty partial statistics");
  const Tile t = pick_tile(R, C);
  const int r = relu ? 1 : 0;
  const size_t smem = (size_t)(2 * t.ty + 2) * t.cvb * kVec * sizeof(float);
  if (dt == DType::BF16)
    bn_apply_partials_kernel<__nv_bfloat16><<<apply_grid(t, R), kBnThreads, smem, s>>>(
        (const __nv_bfloat16*)x, (const __nv_bfloat16*)residual, (__nv_bfloat16*)y, mask, partial, groups, gamma, beta, running_mean, running_var,
        num_batches, save_mean, save_rstd, eps, momentum, R, C, t.cvb, t.ty, r);
  else
    bn_apply_partials_kernel<float><<<apply_grid(t, R), kBnThreads, smem, s>>>(
        (const float*)x, (const float*)residual, (float*)y, mask, partial, groups, gamma, beta, running_mean, running_var, num_batches, save_mean,
        save_rstd, eps, momentum, R, C, t.cvb, t.ty, r);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_bn_backward_from_partials(const void* dy, const void* x, const void* y, void* dx, void* dres, DType dt, int R, int C, const float* gamma,
                                      const float* save_mean, const float* save_rstd, float* dgamma, float* dbeta, const float* partial, int groups,
                                      bool relu, cudaStream_t s) {
  if (C % kVec != 0) throw std::runtime_error("fused batch norm: channel count must be a multiple of 8");
  if (groups < 1) throw std::runtime_error("fused batch norm: empty partial sums");
  const Tile t = pick_tile(R, C);
  const int r = relu ? 1 : 0;
  const size_t smem = (size_t)(2 * t.ty + 2) * t.cvb * kVec * sizeof(float);
  if (dt == DType::BF16)
    bn_bwd_apply_partials_kernel<__nv_bfloat16><<<apply_grid(t, R), kBnThreads, smem, s>>>(
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const unsigned char*)y, (__nv_bfloat16*)dx, (__nv_bfloat16*)dres, partial, groups, save_mean,
        save_rstd, gamma, dgamma, dbeta, R, C, t.cvb, t.ty, r);
  else
    bn_bwd_apply_partials_kernel<float><<<apply_grid(t, R), kBnThreads, smem, s>>>(
        (const float*)dy, (const float*)x, (const unsigned char*)y, (float*)dx, (float*)dres, partial, groups, save_mean, save_rstd, gamma, dgamma, dbeta,
        R, C, t.cvb, t.ty, r);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_bn_backward(const void* dy, const void* x, const void* y, void* dx, void* dres, DType dt, int R, int C, const float* gamma,
                        const float* save_mean, const float* save_rstd, float* dgamma, float* dbeta, float* coef, float* partial,
                        unsigned int* counters, bool relu, cudaStream_t s) {
  if (C % kVec != 0) throw std::runtime_error("fused batch norm: channel count must be a multiple of 8");
  const int r = relu ? 1 : 0;
  if (dt == DType::BF16 && resident_allowed() && res_aligned(dy) && res_aligned(x) && res_aligned(dx) && res_aligned(dres)) {
    const ResPlan plan = resident_plan(R, C, 2);
    if (plan.ok) {
      static std::atomic<unsigned long long> smem_done{0};
      ensure_max_dynamic_smem(bn_resident_bwd_kernel, res_smem_limit(), smem_done);    // raised once: every plan fits below it
      const int br = plan.g.box_rows;
      const CUtensorMap mdy = res_map(dy, R, C, br), mx = res_map(x, R, C, br), mdx = res_map(dx, R, C, br);
      const CUtensorMap mdres = dres != nullptr ? res_map(dres, R, C, br) : mdx;
      for (int k = 0; k < plan.launches; ++k)
        launch_cooperative(bn_resident_bwd_kernel, plan, s, mdy, mx, mdx, mdres, (const unsigned char*)y, save_mean, save_rstd, gamma, dgamma,
                           dbeta, coef, partial, counters + 2 * pick_tile(R, C).grid_x, r, dres != nullptr ? 1 : 0, res_launch(plan, k));
      B200_COUNT_LAUNCH(plan.launches);
      return;
    }
  }
  Tile t;
  const bool fused = fused_tile(R, C, &t);
  const size_t smem = (size_t)2 * t.ty * t.cvb * kVec * sizeof(float);
  const dim3 grid(t.grid_x, t.grid_y);
  if (!fused && bn_pdl_enabled()) {
#define B200_BN_BWD_PDL(T)                                                                                                                   \
    bn_bwd_reduce_kernel<T, false, true><<<grid, kBnThreads, smem, s>>>((const T*)dy, (const T*)x, (const unsigned char*)y, R, C, t.cvb, t.ty, r,  \
                                                                        save_mean, save_rstd, partial, counters, dgamma, dbeta, coef, gamma,      \
                                                                        (T*)dx, (T*)dres);                                                        \
    B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);                                                                                     \
    launch_dependent(bn_bwd_apply_pdl_kernel<T>, apply_grid(t, R), s, (const T*)dy, (const T*)x, (const unsigned char*)y, (T*)dx, (T*)dres,         \
                     save_mean, save_rstd, gamma, (const float*)coef, R, C, t.cvb, t.ty, r);                                                        \
    B200_COUNT_LAUNCH(1)
    if (dt == DType::BF16) { B200_BN_BWD_PDL(__nv_bfloat16); } else { B200_BN_BWD_PDL(float); }
#undef B200_BN_BWD_PDL
    return;
  }
#define B200_BN_BWD(T, F)                                                                                                              \
  bn_bwd_reduce_kernel<T, F><<<grid, kBnThreads, smem, s>>>((const T*)dy, (const T*)x, (const unsigned char*)y, R, C, t.cvb, t.ty, r,  \
                                                            save_mean, save_rstd, partial, counters, dgamma, dbeta, coef, gamma,      \
                                                            (T*)dx, (T*)dres)
  if (dt == DType::BF16) { if (fused) B200_BN_BWD(__nv_bfloat16, true); else B200_BN_BWD(__nv_bfloat16, false); }
  else { if (fused) B200_BN_BWD(float, true); else B200_BN_BWD(float, false); }
#undef B200_BN_BWD
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  if (fused) return;
  if (dt == DType::BF16)
    bn_bwd_apply_kernel<__nv_bfloat16><<<apply_grid(t, R), kBnThreads, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const unsigned char*)y,
                                                                               (__nv_bfloat16*)dx, (__nv_bfloat16*)dres, save_mean, save_rstd, gamma, coef,
                                                                               R, C, t.cvb, t.ty, r);
  else
    bn_bwd_apply_kernel<float><<<apply_grid(t, R), kBnThreads, 0, s>>>((const float*)dy, (const float*)x, (const unsigned char*)y, (float*)dx,
                                                                       (float*)dres, save_mean, save_rstd, gamma, coef, R, C, t.cvb, t.ty, r);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
