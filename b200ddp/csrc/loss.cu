// Fused loss forward+backward kernels: the stock path runs sub / pow / mean-reduce and a
// separate mse_loss_backward; cross-entropy is log_softmax + nll_loss + their two backwards.
// Each loss here is one launch that emits the scalar loss AND the gradient w.r.t. its input, so the
// autograd Function's backward is just "return the saved tensor (x upstream scale)".
#include "ops.h"

namespace b200 {
namespace {

constexpr int kLossThreads = 256;

template <typename T> __device__ __forceinline__ void loss_load8(const T* p, float* f);
template <> __device__ __forceinline__ void loss_load8<__nv_bfloat16>(const __nv_bfloat16* p, float* f) { unpack8(*reinterpret_cast<const Bf16x8*>(p), f); }
template <> __device__ __forceinline__ void loss_load8<float>(const float* p, float* f) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <typename T> __device__ __forceinline__ void loss_store8(T* p, const float* f);
template <> __device__ __forceinline__ void loss_store8<__nv_bfloat16>(__nv_bfloat16* p, const float* f) { *reinterpret_cast<Bf16x8*>(p) = pack8(f); }
template <> __device__ __forceinline__ void loss_store8<float>(float* p, const float* f) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}

template <typename T>
__global__ void __launch_bounds__(kLossThreads) mse_fwd_bwd_kernel(const T* __restrict__ out, const T* __restrict__ tgt, size_t n,
                                                                   float gscale, float* __restrict__ loss, T* __restrict__ dout,
                                                                   float* __restrict__ scratch) {
  __shared__ float red[33];
  __shared__ bool last;
  const float inv_n = 1.f / (float)n;
  const float k = 2.f * inv_n * gscale;
  float acc = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(tgt) | reinterpret_cast<uintptr_t>(dout)) & 31u) == 0;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = n / 8;
    size_t v = tid;
    for (; v + stride < nvec; v += 2 * stride) {            // two independent vector pairs in flight
      float a0[8], b0[8], a1[8], b1[8];
      loss_load8<T>(out + v * 8, a0); loss_load8<T>(tgt + v * 8, b0);
      loss_load8<T>(out + (v + stride) * 8, a1); loss_load8<T>(tgt + (v + stride) * 8, b1);
#pragma unroll
      for (int i = 0; i < 8; ++i) { a0[i] -= b0[i]; acc = fmaf(a0[i], a0[i], acc); a0[i] *= k; a1[i] -= b1[i]; acc = fmaf(a1[i], a1[i], acc); a1[i] *= k; }
      loss_store8<T>(dout + v * 8, a0);
      loss_store8<T>(dout + (v + stride) * 8, a1);
    }
    for (; v < nvec; v += stride) {
      float a0[8], b0[8];
      loss_load8<T>(out + v * 8, a0); loss_load8<T>(tgt + v * 8, b0);
#pragma unroll
      for (int i = 0; i < 8; ++i) { a0[i] -= b0[i]; acc = fmaf(a0[i], a0[i], acc); a0[i] *= k; }
      loss_store8<T>(dout + v * 8, a0);
    }
    done = nvec * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    const float d = to_f32<T>(out[i]) - to_f32<T>(tgt[i]);
    acc += d * d;
    dout[i] = from_f32<T>(k * d);
  }
  const float total = block_sum(acc, red);
  // deterministic two-stage reduction: the last block to arrive sums the partials in index order
  unsigned int* counter = reinterpret_cast<unsigned int*>(scratch + gridDim.x);
  if (threadIdx.x == 0) {
    scratch[blockIdx.x] = total;
    __threadfence();
    const unsigned int ticket = atomicAdd(counter, 1u);
    last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    float s = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) s += __ldcg(scratch + i);
    s = block_sum(s, red);
    if (threadIdx.x == 0) { *loss = s * inv_n; *counter = 0u; }
  }
}

// One block per row; the row is read once into registers/smem-free streaming form twice (second read
// hits L1/L2: a 30522-wide bf16 row is 61 KB).
template <typename T>
__global__ void __launch_bounds__(kLossThreads) xent_fwd_bwd_kernel(const T* __restrict__ logits, const long long* __restrict__ targets,
                                                                    int rows, int cols, long long ignore_index, float gscale,
                                                                    float* __restrict__ row_loss, T* __restrict__ dlogits) {
  __shared__ float red[33];
  const int row = blockIdx.x;
  const T* x = logits + (size_t)row * cols;
  T* dx = dlogits + (size_t)row * cols;
  const long long t = targets[row];
  const bool ignored = (t == ignore_index) || t < 0 || t >= cols;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) m = fmaxf(m, to_f32<T>(x[i]));
  m = block_max(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) s += __expf(to_f32<T>(x[i]) - m);
  s = block_sum(s, red);
  const float lse = m + __logf(s);
  const float inv_s = 1.f / s;
  if (threadIdx.x == 0) row_loss[row] = ignored ? 0.f : lse - to_f32<T>(x[t]);
  const float valid = row_loss[rows];   // written by count_valid_kernel (mean is over non-ignored rows)
  const float g = (ignored || valid <= 0.f) ? 0.f : gscale / valid;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) {
    float p = __expf(to_f32<T>(x[i]) - m) * inv_s;
    if (i == t) p -= 1.f;
    dx[i] = from_f32<T>(p * g);
  }
}

// Row lives in shared memory: ONE global read of the logits, softmax statistics and the gradient come from smem,
// ONE global write of dlogits; 16-byte accesses with a peeled head/tail (rows of a 30522-wide matrix are only
// 4-byte aligned).  smem index = column + pad so shared and global addresses share their 16-byte phase.
template <typename T>
__global__ void __launch_bounds__(kLossThreads) xent_fwd_bwd_smem_kernel(const T* __restrict__ logits, const long long* __restrict__ targets,
                                                                         int rows, int cols, long long ignore_index, float gscale,
                                                                         float* __restrict__ row_loss, T* __restrict__ dlogits) {
  extern __shared__ __align__(16) unsigned char xsmem[];
  __shared__ float red[33];
  constexpr int EPV = 16 / sizeof(T);                   // elements per 16-byte vector
  const int row = blockIdx.x;
  const T* x = logits + (size_t)row * cols;
  T* dx = dlogits + (size_t)row * cols;
  const int pad = (int)((reinterpret_cast<uintptr_t>(x) & 15u) / sizeof(T));
  T* sx = reinterpret_cast<T*>(xsmem);                   // sx[pad + i] = x[i]
  const int head = min(cols, (EPV - pad) % EPV);         // scalars until the first aligned vector
  const int nvec = (cols - head) / EPV;
  const int tail0 = head + nvec * EPV;
  const long long t = targets[row];
  const bool ignored = (t == ignore_index) || t < 0 || t >= cols;

  float m = -INFINITY;
  for (int i = threadIdx.x; i < head; i += blockDim.x) { const T v = x[i]; sx[pad + i] = v; m = fmaxf(m, to_f32<T>(v)); }
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint4 raw = *reinterpret_cast<const uint4*>(x + head + v * EPV);
    *reinterpret_cast<uint4*>(sx + pad + head + v * EPV) = raw;
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < EPV; ++j) m = fmaxf(m, to_f32<T>(e[j]));
  }
  for (int i = tail0 + threadIdx.x; i < cols; i += blockDim.x) { const T v = x[i]; sx[pad + i] = v; m = fmaxf(m, to_f32<T>(v)); }
  m = block_max(m, red);                                 // (contains the __syncthreads that publishes smem)
  float s = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) s += __expf(to_f32<T>(sx[pad + i]) - m);
  s = block_sum(s, red);
  const float lse = m + __logf(s);
  const float valid = row_loss[rows];
  if (threadIdx.x == 0) row_loss[row] = ignored ? 0.f : lse - to_f32<T>(sx[pad + (int)t]);
  const float g = (ignored || valid <= 0.f) ? 0.f : gscale / valid;
  const float coef = g / s;
  const int ti = ignored ? -1 : (int)t;
  for (int i = threadIdx.x; i < head; i += blockDim.x) {
    float p = __expf(to_f32<T>(sx[pad + i]) - m) * coef;
    if (i == ti) p -= g;
    dx[i] = from_f32<T>(p);
  }
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const int base = head + v * EPV;
    const uint4 raw = *reinterpret_cast<const uint4*>(sx + pad + base);
    const T* e = reinterpret_cast<const T*>(&raw);
    uint4 outv;
    T* o = reinterpret_cast<T*>(&outv);
#pragma unroll
    for (int j = 0; j < EPV; ++j) {
      float p = __expf(to_f32<T>(e[j]) - m) * coef;
      if (base + j == ti) p -= g;
      o[j] = from_f32<T>(p);
    }
    *reinterpret_cast<uint4*>(dx + base) = outv;
  }
  for (int i = tail0 + threadIdx.x; i < cols; i += blockDim.x) {
    float p = __expf(to_f32<T>(sx[pad + i]) - m) * coef;
    if (i == ti) p -= g;
    dx[i] = from_f32<T>(p);
  }
}

__global__ void __launch_bounds__(1024) xent_finish_kernel(const float* __restrict__ row_loss, const long long* __restrict__ targets,
                                                           int rows, int cols, long long ignore_index, float* __restrict__ loss) {
  __shared__ float red[33];
  float s = 0.f, cnt = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    const long long t = targets[i];
    if (t != ignore_index && t >= 0 && t < cols) { s += row_loss[i]; cnt += 1.f; }
  }
  s = block_sum(s, red);
  cnt = block_sum(cnt, red);
  if (threadIdx.x == 0) *loss = cnt > 0.f ? s / cnt : 0.f;
}

__global__ void __launch_bounds__(1024) count_valid_kernel(const long long* __restrict__ targets, int rows, int cols,
                                                           long long ignore_index, float* __restrict__ out) {
  __shared__ float red[33];
  float cnt = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    const long long t = targets[i];
    if (t != ignore_index && t >= 0 && t < cols) cnt += 1.f;
  }
  cnt = block_sum(cnt, red);
  if (threadIdx.x == 0) *out = cnt;
}

}  // namespace

int mse_blocks(size_t n) {
  size_t b = (n + kLossThreads * 16 - 1) / (kLossThreads * 16);
  if (b < 1) b = 1;
  if (b > 8 * kNumSMs) b = 8 * kNumSMs;
  return (int)b;
}

void launch_mse_fwd_bwd(const void* out, const void* target, DType dt, size_t n, float gscale, float* loss, void* dout,
                        float* scratch, int blocks, cudaStream_t s) {
  if (dt == DType::BF16)
    mse_fwd_bwd_kernel<__nv_bfloat16><<<blocks, kLossThreads, 0, s>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)target, n,
                                                                     gscale, loss, (__nv_bfloat16*)dout, scratch);
  else
    mse_fwd_bwd_kernel<float><<<blocks, kLossThreads, 0, s>>>((const float*)out, (const float*)target, n, gscale, loss,
                                                             (float*)dout, scratch);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_xent_fwd_bwd(const void* logits, const long long* targets, DType dt, int rows, int cols, long long ignore_index,
                         float gscale, float* row_loss, float* loss, void* dlogits, cudaStream_t s) {
  // mean over non-ignored rows: count them on device first (row_loss has rows+1 floats; the last
  // one carries the count) so no host round trip is needed.
  const float g = gscale;
  count_valid_kernel<<<1, 1024, 0, s>>>(targets, rows, cols, ignore_index, row_loss + rows);
  const size_t esz = dt == DType::BF16 ? 2 : 4;
  const size_t smem = ((size_t)cols + 16) * esz;
  if (smem <= 200 * 1024 && ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(dlogits)) % esz) == 0 &&
      (reinterpret_cast<uintptr_t>(logits) & 15u) == (reinterpret_cast<uintptr_t>(dlogits) & 15u)) {
    // dlogits rows must share the 16-byte phase of the logits rows (both come from the same allocator: they do)
    static std::atomic<unsigned long long> configured_bf16{0}, configured_f32{0};
    ensure_max_dynamic_smem(xent_fwd_bwd_smem_kernel<__nv_bfloat16>, 200 * 1024, configured_bf16);
    ensure_max_dynamic_smem(xent_fwd_bwd_smem_kernel<float>, 200 * 1024, configured_f32);
    if (dt == DType::BF16)
      xent_fwd_bwd_smem_kernel<__nv_bfloat16><<<rows, kLossThreads, smem, s>>>((const __nv_bfloat16*)logits, targets, rows, cols, ignore_index, g,
                                                                             row_loss, (__nv_bfloat16*)dlogits);
    else
      xent_fwd_bwd_smem_kernel<float><<<rows, kLossThreads, smem, s>>>((const float*)logits, targets, rows, cols, ignore_index, g, row_loss,
                                                                     (float*)dlogits);
  } else if (dt == DType::BF16)
    xent_fwd_bwd_kernel<__nv_bfloat16><<<rows, kLossThreads, 0, s>>>((const __nv_bfloat16*)logits, targets, rows, cols, ignore_index, g,
                                                                   row_loss, (__nv_bfloat16*)dlogits);
  else
    xent_fwd_bwd_kernel<float><<<rows, kLossThreads, 0, s>>>((const float*)logits, targets, rows, cols, ignore_index, g, row_loss,
                                                           (float*)dlogits);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  xent_finish_kernel<<<1, 1024, 0, s>>>(row_loss, targets, rows, cols, ignore_index, loss);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------------------
// GELU (erf form) forward and backward as single vectorised passes.  The stock autograd formula for the backward
// (cast to fp32, erf, exp, three multiplies, cast back) is ~8 launches over a [tokens, 3072] tensor per BERT layer.
namespace b200 {
namespace {

__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad_f(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

template <typename T, bool BWD>
__global__ void __launch_bounds__(kLossThreads) gelu_kernel(const T* __restrict__ pre, const T* __restrict__ dy, T* __restrict__ out, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(out) | (BWD ? reinterpret_cast<uintptr_t>(dy) : 0)) & 31u) == 0;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = n / 8;
    for (size_t v = tid; v < nvec; v += stride) {
      float a[8], g[8];
      loss_load8<T>(pre + v * 8, a);
      if (BWD) loss_load8<T>(dy + v * 8, g);
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = BWD ? g[i] * gelu_grad_f(a[i]) : gelu_f(a[i]);
      loss_store8<T>(out + v * 8, a);
    }
    done = nvec * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    const float x = to_f32<T>(pre[i]);
    out[i] = from_f32<T>(BWD ? to_f32<T>(dy[i]) * gelu_grad_f(x) : gelu_f(x));
  }
}

}  // namespace

void launch_gelu(const void* pre, const void* dy, void* out, DType dt, size_t n, bool backward, cudaStream_t s) {
  size_t b = (n / 8 + kLossThreads - 1) / kLossThreads;
  if (b < 1) b = 1;
  if (b > (size_t)16 * kNumSMs) b = (size_t)16 * kNumSMs;
  const int blocks = (int)b;
  if (dt == DType::BF16) {
    if (backward) gelu_kernel<__nv_bfloat16, true><<<blocks, kLossThreads, 0, s>>>((const __nv_bfloat16*)pre, (const __nv_bfloat16*)dy, (__nv_bfloat16*)out, n);
    else gelu_kernel<__nv_bfloat16, false><<<blocks, kLossThreads, 0, s>>>((const __nv_bfloat16*)pre, nullptr, (__nv_bfloat16*)out, n);
  } else {
    if (backward) gelu_kernel<float, true><<<blocks, kLossThreads, 0, s>>>((const float*)pre, (const float*)dy, (float*)out, n);
    else gelu_kernel<float, false><<<blocks, kLossThreads, 0, s>>>((const float*)pre, nullptr, (float*)out, n);
  }
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
