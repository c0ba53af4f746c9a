// LayerNorm forward / backward (needed by the BERT
// config).  One warp per row, 16-byte vector loads, fp32 statistics; backward produces dx in the same
// pass as per-CTA partial dgamma/dbeta, finished by a small column-reduce kernel (no atomics, so the
// result is deterministic).
#include "ops.h"

namespace b200 {
namespace {

constexpr int kLnThreads = 256;            // 8 warps = 8 rows per CTA iteration
constexpr int kLnMaxPerLane = 32;          // supports cols <= 32*32 = 1024 in registers; larger cols re-read

template <typename T>
__global__ void __launch_bounds__(kLnThreads) layernorm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ gamma, const T* __restrict__ beta,
                                                                   int rows, int cols, float eps, T* __restrict__ y,
                                                                   float* __restrict__ mean, float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  for (int row = blockIdx.x * warps + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps) {
    const T* xr = x + (size_t)row * cols;
    float s = 0.f;
    for (int i = lane; i < cols; i += 32) s += to_f32<T>(xr[i]);
    const float mu = warp_sum(s) / (float)cols;
    float v = 0.f;
    for (int i = lane; i < cols; i += 32) { const float d = to_f32<T>(xr[i]) - mu; v += d * d; }
    const float rs = rsqrtf(warp_sum(v) / (float)cols + eps);
    T* yr = y + (size_t)row * cols;
    for (int i = lane; i < cols; i += 32) {
      const float xn = (to_f32<T>(xr[i]) - mu) * rs;
      yr[i] = from_f32<T>(xn * to_f32<T>(gamma[i]) + to_f32<T>(beta[i]));
    }
    if (lane == 0) { mean[row] = mu; rstd[row] = rs; }
  }
}

// Each CTA owns a contiguous stripe of rows.  Warps compute dx for their rows and accumulate
// dgamma/dbeta for the columns they touch into registers -> shared -> one partial row per CTA.
template <typename T>
__global__ void __launch_bounds__(kLnThreads) layernorm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ gamma,
                                                                   const float* __restrict__ mean, const float* __restrict__ rstd, int rows, int cols,
                                                                   T* __restrict__ dx, float* __restrict__ dgamma_partial,
                                                                   float* __restrict__ dbeta_partial) {
  extern __shared__ float smem[];            // [2][cols] per-CTA column accumulators
  float* sg = smem;
  float* sb = smem + cols;
  for (int i = threadIdx.x; i < 2 * cols; i += blockDim.x) smem[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const int rows_per_cta = (rows + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(rows, r0 + rows_per_cta);
  for (int row = r0 + warp; row < r1; row += warps) {
    const T* xr = x + (size_t)row * cols;
    const T* dyr = dy + (size_t)row * cols;
    const float mu = mean[row], rs = rstd[row];
    float s1 = 0.f, s2 = 0.f;
    for (int i = lane; i < cols; i += 32) {
      const float xn = (to_f32<T>(xr[i]) - mu) * rs;
      const float dg = to_f32<T>(dyr[i]) * to_f32<T>(gamma[i]);
      s1 += dg;
      s2 += dg * xn;
    }
    s1 = warp_sum(s1) / (float)cols;
    s2 = warp_sum(s2) / (float)cols;
    T* dxr = dx + (size_t)row * cols;
    for (int i = lane; i < cols; i += 32) {
      const float xn = (to_f32<T>(xr[i]) - mu) * rs;
      const float dyv = to_f32<T>(dyr[i]);
      const float dg = dyv * to_f32<T>(gamma[i]);
      dxr[i] = from_f32<T>(rs * (dg - s1 - xn * s2));
      // column i is only ever touched by lane (i % 32) of each warp: shared atomics across warps
      atomicAdd(&sg[i], dyv * xn);
      atomicAdd(&sb[i], dyv);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cols; i += blockDim.x) {
    dgamma_partial[(size_t)blockIdx.x * cols + i] = sg[i];
    dbeta_partial[(size_t)blockIdx.x * cols + i] = sb[i];
  }
}


// ---- fast path: cols % 8 == 0 and cols <= 1024 (BERT hidden 768/1024) ----------------------------------
// A lane owns up to 4 chunks of 8 consecutive columns (chunk c covers columns [8*(lane+32c), +8)): one
// 16-byte load per chunk, the row lives in registers, statistics need no second pass over memory.
// kRms (RMSNorm, y = x * rsqrt(mean(x^2) + eps) * gamma): no mean (mu = 0, `mean` is not written or read), no beta;
// dx = rs * (dy*gamma - xn * mean(dy*gamma*xn)) and dgamma = sum dy * xn from the same column reduction.
constexpr int kLnChunks = 4;

template <typename T> __device__ __forceinline__ void ln_load8(const T* p, float* f);
template <> __device__ __forceinline__ void ln_load8<float>(const float* p, float* f) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <> __device__ __forceinline__ void ln_load8<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
  unpack8(*reinterpret_cast<const Bf16x8*>(p), f);
}
template <typename T> __device__ __forceinline__ void ln_store8(T* p, const float* f);
template <> __device__ __forceinline__ void ln_store8<float>(float* p, const float* f) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}
template <> __device__ __forceinline__ void ln_store8<__nv_bfloat16>(__nv_bfloat16* p, const float* f) {
  *reinterpret_cast<Bf16x8*>(p) = pack8(f);
}

template <typename T, bool kRms = false>
__global__ void __launch_bounds__(kLnThreads) layernorm_fwd_fast_kernel(const T* __restrict__ x, const T* __restrict__ gamma,
                                                                        const T* __restrict__ beta, int rows, int cols, float eps,
                                                                        T* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  const int nchunk = cols >> 3;
  float g[kLnChunks][8], b[kLnChunks][8];
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c) {
    const int ch = lane + 32 * c;
    if (ch < nchunk) {
      ln_load8<T>(gamma + 8 * ch, g[c]);
      if constexpr (kRms) {
#pragma unroll
        for (int j = 0; j < 8; ++j) b[c][j] = 0.f;
      } else {
        ln_load8<T>(beta + 8 * ch, b[c]);
      }
    }
  }
  const float inv = 1.f / (float)cols;
  for (int row = blockIdx.x * warps + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps) {
    const T* xr = x + (size_t)row * cols;
    float v[kLnChunks][8];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int ch = lane + 32 * c;
      if (ch < nchunk) {
        ln_load8<T>(xr + 8 * ch, v[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[c][j];
      }
    }
    const float mu = kRms ? 0.f : warp_sum(s) * inv;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      if (lane + 32 * c < nchunk) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[c][j] - mu; q += d * d; }
      }
    }
    const float rs = rsqrtf(warp_sum(q) * inv + eps);
    T* yr = y + (size_t)row * cols;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int ch = lane + 32 * c;
      if (ch < nchunk) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = kRms ? v[c][j] * rs * g[c][j] : (v[c][j] - mu) * rs * g[c][j] + b[c][j];
        ln_store8<T>(yr + 8 * ch, o);
      }
    }
    if (lane == 0) {
      if constexpr (!kRms) mean[row] = mu;
      rstd[row] = rs;
    }
  }
}

// dx only: rows live in registers, no cross-row state -> light enough for 2 CTAs per SM.
template <typename T, bool kRms = false>
__global__ void __launch_bounds__(kLnThreads, 2) layernorm_bwd_dx_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ gamma,
                                                                         const float* __restrict__ mean, const float* __restrict__ rstd, int rows,
                                                                         int cols, T* __restrict__ dx) {
  const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  const int nchunk = cols >> 3;
  float g[kLnChunks][8];
#pragma unroll
  for (int c = 0; c < kLnChunks; ++c) {
    const int ch = lane + 32 * c;
    if (ch < nchunk) ln_load8<T>(gamma + 8 * ch, g[c]);
  }
  const float inv = 1.f / (float)cols;
  for (int row = blockIdx.x * warps + (threadIdx.x >> 5); row < rows; row += gridDim.x * warps) {
    const T* xr = x + (size_t)row * cols;
    const T* dyr = dy + (size_t)row * cols;
    const float mu = kRms ? 0.f : mean[row], rs = rstd[row];
    float xn[kLnChunks][8], d[kLnChunks][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int ch = lane + 32 * c;
      if (ch < nchunk) {
        ln_load8<T>(xr + 8 * ch, xn[c]);
        ln_load8<T>(dyr + 8 * ch, d[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xn[c][j] = (xn[c][j] - mu) * rs;
          d[c][j] *= g[c][j];
          s1 += d[c][j];
          s2 = fmaf(d[c][j], xn[c][j], s2);
        }
      }
    }
    s1 = kRms ? 0.f : warp_sum(s1) * inv;
    s2 = warp_sum(s2) * inv;
    T* dxr = dx + (size_t)row * cols;
#pragma unroll
    for (int c = 0; c < kLnChunks; ++c) {
      const int ch = lane + 32 * c;
      if (ch < nchunk) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (d[c][j] - s1 - xn[c][j] * s2);
        ln_store8<T>(dxr + 8 * ch, o);
      }
    }
  }
}

// dgamma / dbeta: column reduction over rows (same scheme as the BatchNorm reductions): threads own 8 columns,
// rows are strided over the block and over gridDim.y splits, the last block of a column tile sums the partials
// in a fixed order.  Re-reads dy and x, which are L2-resident right after the dx kernel.
template <typename T, bool kRms = false>
__global__ void __launch_bounds__(kLnThreads) layernorm_param_grad_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                          const float* __restrict__ mean, const float* __restrict__ rstd, int rows,
                                                                          int cols, int cvb, int ty, float* __restrict__ partial,
                                                                          unsigned int* __restrict__ counters, T* __restrict__ dgamma,
                                                                          T* __restrict__ dbeta) {
  extern __shared__ float smem[];
  __shared__ bool is_last;
  const int tx = threadIdx.x % cvb, tyi = threadIdx.x / cvb;
  const int cv = blockIdx.x * cvb + tx;
  const int S = gridDim.y;
  const int rows_per = (rows + S - 1) / S;
  const int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  float ag[8], ab[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { ag[i] = 0.f; ab[i] = 0.f; }
  if (cv * 8 < cols) {
    const size_t col = (size_t)cv * 8;
    int r = r0 + tyi;
    for (; r + ty < r1; r += 2 * ty) {
      float d0[8], x0[8], d1[8], x1[8];
      ln_load8<T>(dy + (size_t)r * cols + col, d0);
      ln_load8<T>(x + (size_t)r * cols + col, x0);
      ln_load8<T>(dy + (size_t)(r + ty) * cols + col, d1);
      ln_load8<T>(x + (size_t)(r + ty) * cols + col, x1);
      const float m0 = kRms ? 0.f : mean[r], s0 = rstd[r], m1 = kRms ? 0.f : mean[r + ty], s1 = rstd[r + ty];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        ab[i] += d0[i] + d1[i];
        ag[i] = fmaf(d0[i], (x0[i] - m0) * s0, ag[i]);
        ag[i] = fmaf(d1[i], (x1[i] - m1) * s1, ag[i]);
      }
    }
    for (; r < r1; r += ty) {
      float d0[8], x0[8];
      ln_load8<T>(dy + (size_t)r * cols + col, d0);
      ln_load8<T>(x + (size_t)r * cols + col, x0);
      const float m0 = kRms ? 0.f : mean[r], s0 = rstd[r];
#pragma unroll
      for (int i = 0; i < 8; ++i) { ab[i] += d0[i]; ag[i] = fmaf(d0[i], (x0[i] - m0) * s0, ag[i]); }
    }
  }
  const int width = cvb * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) { smem[(0 * ty + tyi) * width + tx * 8 + i] = ag[i]; smem[(1 * ty + tyi) * width + tx * 8 + i] = ab[i]; }
  __syncthreads();
  for (int idx = threadIdx.x; idx < 2 * width; idx += blockDim.x) {
    const int a = idx / width, c = idx % width;
    float sum = 0.f;
    for (int rr = 0; rr < ty; ++rr) sum += smem[(a * ty + rr) * width + c];
    const int ch = blockIdx.x * width + c;
    if (ch < cols) partial[(size_t)(a * S + blockIdx.y) * cols + ch] = sum;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(&counters[blockIdx.x], 1u);
    is_last = (ticket == (unsigned int)S - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    const int ch = blockIdx.x * width + c;
    if (ch >= cols) continue;
    float sg = 0.f, sb = 0.f;
    for (int k = 0; k < S; ++k) { sg += __ldcg(&partial[(size_t)(0 * S + k) * cols + ch]); sb += __ldcg(&partial[(size_t)(1 * S + k) * cols + ch]); }
    dgamma[ch] = from_f32<T>(sg);
    if constexpr (!kRms) dbeta[ch] = from_f32<T>(sb);
  }
  if (threadIdx.x == 0) counters[blockIdx.x] = 0u;
}

// ---- wide RMSNorm: cols % 8 == 0 and 1024 < cols <= 4096 (1B-class Llama hidden sizes 1536 - 4096) -------------------
// One 128-thread CTA per row (grid-stride over rows): thread t owns chunks t + 128 c (c < 4) of 8 columns, so the row stays
// in registers as on the fast path, and the row sums go through shared memory.  dgamma comes from the fast path's column
// reduction (layernorm_param_grad_kernel), which does not depend on the width.
constexpr int kRmsWideThreads = 128;
constexpr int kRmsWideChunks = 4;

// Sum over the CTA of v; red: kRmsWideThreads / 32 floats of shared memory, free again when this returns
__device__ __forceinline__ float rms_wide_block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  const float r = (red[0] + red[1]) + (red[2] + red[3]);
  __syncthreads();
  return r;
}

template <typename T>
__global__ void __launch_bounds__(kRmsWideThreads) rmsnorm_wide_fwd_kernel(const T* __restrict__ x, const T* __restrict__ gamma, int rows,
                                                                          int cols, float eps, T* __restrict__ y, float* __restrict__ rstd) {
  __shared__ float red[kRmsWideThreads / 32];
  const int nchunk = cols >> 3;
  float g[kRmsWideChunks][8];
#pragma unroll
  for (int c = 0; c < kRmsWideChunks; ++c) {
    const int ch = threadIdx.x + kRmsWideThreads * c;
    if (ch < nchunk) ln_load8<T>(gamma + 8 * ch, g[c]);
  }
  const float inv = 1.f / (float)cols;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const T* xr = x + (size_t)row * cols;
    float v[kRmsWideChunks][8];
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < kRmsWideChunks; ++c) {
      const int ch = threadIdx.x + kRmsWideThreads * c;
      if (ch < nchunk) {
        ln_load8<T>(xr + 8 * ch, v[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) q += v[c][j] * v[c][j];
      }
    }
    const float rs = rsqrtf(rms_wide_block_sum(q, red) * inv + eps);
    T* yr = y + (size_t)row * cols;
#pragma unroll
    for (int c = 0; c < kRmsWideChunks; ++c) {
      const int ch = threadIdx.x + kRmsWideThreads * c;
      if (ch < nchunk) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = v[c][j] * rs * g[c][j];
        ln_store8<T>(yr + 8 * ch, o);
      }
    }
    if (threadIdx.x == 0) rstd[row] = rs;
  }
}

// dx = rs * (dy*gamma - xn * mean(dy*gamma*xn)), xn = x * rs
template <typename T>
__global__ void __launch_bounds__(kRmsWideThreads) rmsnorm_wide_bwd_dx_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                             const T* __restrict__ gamma, const float* __restrict__ rstd,
                                                                             int rows, int cols, T* __restrict__ dx) {
  __shared__ float red[kRmsWideThreads / 32];
  const int nchunk = cols >> 3;
  float g[kRmsWideChunks][8];
#pragma unroll
  for (int c = 0; c < kRmsWideChunks; ++c) {
    const int ch = threadIdx.x + kRmsWideThreads * c;
    if (ch < nchunk) ln_load8<T>(gamma + 8 * ch, g[c]);
  }
  const float inv = 1.f / (float)cols;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const T* xr = x + (size_t)row * cols;
    const T* dyr = dy + (size_t)row * cols;
    const float rs = rstd[row];
    float xn[kRmsWideChunks][8], d[kRmsWideChunks][8];
    float s2 = 0.f;
#pragma unroll
    for (int c = 0; c < kRmsWideChunks; ++c) {
      const int ch = threadIdx.x + kRmsWideThreads * c;
      if (ch < nchunk) {
        ln_load8<T>(xr + 8 * ch, xn[c]);
        ln_load8<T>(dyr + 8 * ch, d[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xn[c][j] *= rs;
          d[c][j] *= g[c][j];
          s2 = fmaf(d[c][j], xn[c][j], s2);
        }
      }
    }
    s2 = rms_wide_block_sum(s2, red) * inv;
    T* dxr = dx + (size_t)row * cols;
#pragma unroll
    for (int c = 0; c < kRmsWideChunks; ++c) {
      const int ch = threadIdx.x + kRmsWideThreads * c;
      if (ch < nchunk) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (d[c][j] - xn[c][j] * s2);
        ln_store8<T>(dxr + 8 * ch, o);
      }
    }
  }
}

int rmsnorm_wide_blocks(int rows) { return rows < 16 * kNumSMs ? (rows < 1 ? 1 : rows) : 16 * kNumSMs; }

template <typename T>
__global__ void layernorm_bwd_finish_kernel(const float* __restrict__ dgamma_partial, const float* __restrict__ dbeta_partial, int parts,
                                            int cols, T* __restrict__ dgamma, T* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float g = 0.f, b = 0.f;
  for (int p = 0; p < parts; ++p) { g += dgamma_partial[(size_t)p * cols + c]; b += dbeta_partial[(size_t)p * cols + c]; }
  dgamma[c] = from_f32<T>(g);
  dbeta[c] = from_f32<T>(b);
}

}  // namespace

// Launch geometry of the fast path's backward (dx kernel + column-reduce kernel), shared by LayerNorm and RMSNorm:
// cvb 8-column vectors x ty rows per reduce block, a gx x gy reduce grid (gy <= max_gy row splits), dx_blocks dx CTAs.
struct LnBwdGeometry {
  int cvb, ty, gx, gy, dx_blocks;
  size_t psmem;
};
LnBwdGeometry ln_bwd_geometry(int rows, int cols, int max_gy) {
  LnBwdGeometry g;
  const int cv = cols / 8;
  g.cvb = cv < 32 ? cv : 32;
  while (kLnThreads % g.cvb != 0) --g.cvb;
  g.ty = kLnThreads / g.cvb;
  g.gx = (cv + g.cvb - 1) / g.cvb;
  g.gy = (4 * kNumSMs + g.gx - 1) / g.gx;
  const int by_rows = rows / (g.ty * 4) < 1 ? 1 : rows / (g.ty * 4);
  if (g.gy > by_rows) g.gy = by_rows;
  if (g.gy > max_gy) g.gy = max_gy < 1 ? 1 : max_gy;               // capacity of the partial buffer
  g.dx_blocks = (rows + 7) / 8;
  if (g.dx_blocks > 16 * kNumSMs) g.dx_blocks = 16 * kNumSMs;
  g.psmem = (size_t)2 * kLnThreads * 8 * sizeof(float);
  return g;
}

int layernorm_partial_rows(int rows) {
  int p = (rows + 63) / 64;
  if (p > 2 * kNumSMs) p = 2 * kNumSMs;
  if (p < 2) p = 2;          // the column-reduce path stores [2][splits][cols] partials in this buffer
  return p;
}

void launch_layernorm_fwd(const void* x, const void* gamma, const void* beta, DType dt, int rows, int cols, float eps, void* y,
                          float* mean, float* rstd, cudaStream_t s) {
  int blocks = (rows + 7) / 8;
  if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
  if (blocks < 1) blocks = 1;
  const bool fast = (cols % 8 == 0) && cols <= 8 * 32 * kLnChunks &&
                    ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(gamma) |
                      reinterpret_cast<uintptr_t>(beta)) & 31u) == 0;
  if (fast && dt == DType::BF16)
    layernorm_fwd_fast_kernel<__nv_bfloat16><<<blocks, kLnThreads, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma,
                                                                         (const __nv_bfloat16*)beta, rows, cols, eps, (__nv_bfloat16*)y, mean, rstd);
  else if (fast)
    layernorm_fwd_fast_kernel<float><<<blocks, kLnThreads, 0, s>>>((const float*)x, (const float*)gamma, (const float*)beta, rows, cols, eps,
                                                                 (float*)y, mean, rstd);
  else if (dt == DType::BF16)
    layernorm_fwd_kernel<__nv_bfloat16><<<blocks, kLnThreads, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma,
                                                                    (const __nv_bfloat16*)beta, rows, cols, eps, (__nv_bfloat16*)y, mean, rstd);
  else
    layernorm_fwd_kernel<float><<<blocks, kLnThreads, 0, s>>>((const float*)x, (const float*)gamma, (const float*)beta, rows, cols, eps,
                                                            (float*)y, mean, rstd);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd, DType dt, int rows,
                          int cols, void* dx, float* dgamma_partial, float* dbeta_partial, int partial_rows, void* dgamma,
                          void* dbeta, cudaStream_t s) {
  const size_t smem = 2 * (size_t)cols * sizeof(float);
  const bool fast = (cols % 8 == 0) && cols <= 8 * 32 * kLnChunks &&
                    ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx) |
                      reinterpret_cast<uintptr_t>(gamma)) & 31u) == 0;
  if (fast) {
    // workspace carved from the caller's partial buffers: dgamma_partial = [2][S][cols] partial sums, dbeta_partial = counters
    const LnBwdGeometry geo = ln_bwd_geometry(rows, cols, partial_rows / 2);
    const int cvb = geo.cvb, ty = geo.ty, gx = geo.gx, gy = geo.gy, blocks = geo.dx_blocks;
    const size_t psmem = geo.psmem;
    unsigned int* counters = reinterpret_cast<unsigned int*>(dbeta_partial);
    B200_CUDA_CHECK(cudaMemsetAsync(counters, 0, sizeof(unsigned int) * gx, s));   // fresh scratch from the caller
    if (dt == DType::BF16) {
      layernorm_bwd_dx_kernel<__nv_bfloat16><<<blocks, kLnThreads, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma,
                                                                           mean, rstd, rows, cols, (__nv_bfloat16*)dx);
      layernorm_param_grad_kernel<__nv_bfloat16><<<dim3(gx, gy), kLnThreads, psmem, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, mean, rstd,
                                                                                         rows, cols, cvb, ty, dgamma_partial, counters,
                                                                                         (__nv_bfloat16*)dgamma, (__nv_bfloat16*)dbeta);
    } else {
      layernorm_bwd_dx_kernel<float><<<blocks, kLnThreads, 0, s>>>((const float*)dy, (const float*)x, (const float*)gamma, mean, rstd, rows, cols,
                                                                   (float*)dx);
      layernorm_param_grad_kernel<float><<<dim3(gx, gy), kLnThreads, psmem, s>>>((const float*)dy, (const float*)x, mean, rstd, rows, cols, cvb, ty,
                                                                                 dgamma_partial, counters, (float*)dgamma, (float*)dbeta);
    }
  } else if (dt == DType::BF16) {
    layernorm_bwd_kernel<__nv_bfloat16><<<partial_rows, kLnThreads, smem, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                                             (const __nv_bfloat16*)gamma, mean, rstd, rows, cols,
                                                                             (__nv_bfloat16*)dx, dgamma_partial, dbeta_partial);
    layernorm_bwd_finish_kernel<__nv_bfloat16><<<(cols + 255) / 256, 256, 0, s>>>(dgamma_partial, dbeta_partial, partial_rows, cols,
                                                                                (__nv_bfloat16*)dgamma, (__nv_bfloat16*)dbeta);
  } else {
    layernorm_bwd_kernel<float><<<partial_rows, kLnThreads, smem, s>>>((const float*)dy, (const float*)x, (const float*)gamma, mean, rstd,
                                                                     rows, cols, (float*)dx, dgamma_partial, dbeta_partial);
    layernorm_bwd_finish_kernel<float><<<(cols + 255) / 256, 256, 0, s>>>(dgamma_partial, dbeta_partial, partial_rows, cols,
                                                                        (float*)dgamma, (float*)dbeta);
  }
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

bool rmsnorm_supported(int cols) { return cols % 8 == 0 && cols >= 8 && cols <= 8 * kRmsWideThreads * kRmsWideChunks; }
static bool rmsnorm_wide(int cols) { return cols > 8 * 32 * kLnChunks; }

// RMSNorm on the LayerNorm fast path up to 1024 columns, on the wide kernels above that: x, y, gamma 32-byte aligned,
// rstd [rows]
void launch_rmsnorm_fwd(const void* x, const void* gamma, DType dt, int rows, int cols, float eps, void* y, float* rstd,
                        cudaStream_t s) {
  if (!rmsnorm_supported(cols) ||
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(gamma)) & 31u) != 0)
    throw std::runtime_error("rmsnorm_fwd: needs cols % 8 == 0, cols <= 4096 and 32-byte aligned tensors (cols=" +
                             std::to_string(cols) + ")");
  if (rmsnorm_wide(cols)) {
    if (dt == DType::BF16)
      rmsnorm_wide_fwd_kernel<__nv_bfloat16><<<rmsnorm_wide_blocks(rows), kRmsWideThreads, 0, s>>>(
          (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, rows, cols, eps, (__nv_bfloat16*)y, rstd);
    else
      rmsnorm_wide_fwd_kernel<float><<<rmsnorm_wide_blocks(rows), kRmsWideThreads, 0, s>>>((const float*)x, (const float*)gamma, rows,
                                                                                          cols, eps, (float*)y, rstd);
    B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
    return;
  }
  int blocks = (rows + 7) / 8;
  if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
  if (blocks < 1) blocks = 1;
  if (dt == DType::BF16)
    layernorm_fwd_fast_kernel<__nv_bfloat16, true><<<blocks, kLnThreads, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma,
                                                                               nullptr, rows, cols, eps, (__nv_bfloat16*)y, nullptr, rstd);
  else
    layernorm_fwd_fast_kernel<float, true><<<blocks, kLnThreads, 0, s>>>((const float*)x, (const float*)gamma, nullptr, rows, cols, eps,
                                                                       (float*)y, nullptr, rstd);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

// partial: fp32 [2 * partial_rows, cols] workspace, counters: uint32 [>= cols / 8] workspace (zeroed here)
void launch_rmsnorm_bwd(const void* dy, const void* x, const void* gamma, const float* rstd, DType dt, int rows, int cols, void* dx,
                        float* partial, unsigned int* counters, int partial_rows, void* dgamma, cudaStream_t s) {
  if (!rmsnorm_supported(cols) ||
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx) |
        reinterpret_cast<uintptr_t>(gamma)) & 31u) != 0)
    throw std::runtime_error("rmsnorm_bwd: needs cols % 8 == 0, cols <= 4096 and 32-byte aligned tensors (cols=" +
                             std::to_string(cols) + ")");
  const LnBwdGeometry geo = ln_bwd_geometry(rows, cols, partial_rows);
  const int cvb = geo.cvb, ty = geo.ty, gx = geo.gx, gy = geo.gy, blocks = geo.dx_blocks < 1 ? 1 : geo.dx_blocks;
  const size_t psmem = geo.psmem;
  B200_CUDA_CHECK(cudaMemsetAsync(counters, 0, sizeof(unsigned int) * gx, s));
  if (dt == DType::BF16) {
    if (rmsnorm_wide(cols))
      rmsnorm_wide_bwd_dx_kernel<__nv_bfloat16><<<rmsnorm_wide_blocks(rows), kRmsWideThreads, 0, s>>>(
          (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, rstd, rows, cols, (__nv_bfloat16*)dx);
    else
      layernorm_bwd_dx_kernel<__nv_bfloat16, true><<<blocks, kLnThreads, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                                               (const __nv_bfloat16*)gamma, nullptr, rstd, rows, cols,
                                                                               (__nv_bfloat16*)dx);
    layernorm_param_grad_kernel<__nv_bfloat16, true><<<dim3(gx, gy), kLnThreads, psmem, s>>>(
        (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, nullptr, rstd, rows, cols, cvb, ty, partial, counters,
        (__nv_bfloat16*)dgamma, nullptr);
  } else {
    if (rmsnorm_wide(cols))
      rmsnorm_wide_bwd_dx_kernel<float><<<rmsnorm_wide_blocks(rows), kRmsWideThreads, 0, s>>>((const float*)dy, (const float*)x,
                                                                                             (const float*)gamma, rstd, rows, cols,
                                                                                             (float*)dx);
    else
      layernorm_bwd_dx_kernel<float, true><<<blocks, kLnThreads, 0, s>>>((const float*)dy, (const float*)x, (const float*)gamma, nullptr,
                                                                       rstd, rows, cols, (float*)dx);
    layernorm_param_grad_kernel<float, true><<<dim3(gx, gy), kLnThreads, psmem, s>>>((const float*)dy, (const float*)x, nullptr, rstd,
                                                                                   rows, cols, cvb, ty, partial, counters,
                                                                                   (float*)dgamma, nullptr);
  }
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
