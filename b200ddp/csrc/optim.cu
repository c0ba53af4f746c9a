// Multi-tensor fused optimizer path: the stock stack runs
// `_foreach_norm` -> stack -> `vector_norm` -> clamp -> `_foreach_mul_` -> `_foreach_add_` (>= 6
// launches + a fresh grad allocation per step).  Here: [sum of squares partials come from the
// allreduce epilogue, or from multi_sqnorm on one GPU] -> clip_coef (1 tiny block) -> multi_sgd,
// which applies clip * lr * g (+ weight decay, momentum, nesterov), maintains fp32 master weights
// for bf16 parameters, and can zero the gradient in the same pass.  multi_adamw is the same pass for AdamW, with the
// two moments in flat fp32 buffers beside the masters.
#include "ops.h"

namespace b200 {

namespace {

constexpr int kOptThreads = 256;

__device__ __forceinline__ int find_tensor(const uint32_t* blk0, int count, uint32_t b) {
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (blk0[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// load8 that copies a bf16 vector into registers before unpacking it, where common.h's load8 unpacks through the pointer.
// nvcc compiles the two to different code in these kernels, so the optimizer keeps the form it was measured with.
template <typename T> __device__ __forceinline__ void load8_copy(const T* p, float* f) { load8<T>(p, f); }
template <> __device__ __forceinline__ void load8_copy<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
  const Bf16x8 v = *reinterpret_cast<const Bf16x8*>(p);
  unpack8(v, f);
}

template <typename GT>
__global__ void __launch_bounds__(kOptThreads) multi_sqnorm_kernel(const __grid_constant__ OptTable tab, float* __restrict__ partials) {
  __shared__ uint32_t blk0[kMaxOptTensors];
  __shared__ float red[33];
  for (int i = threadIdx.x; i < tab.count; i += blockDim.x) blk0[i] = tab.t[i].blk0;
  __syncthreads();
  const int k = find_tensor(blk0, tab.count, blockIdx.x);
  const OptSlot& s = tab.t[k];
  const uint32_t begin = (blockIdx.x - s.blk0) * kOptChunk;
  const uint32_t end = min(begin + (uint32_t)kOptChunk, s.numel);
  const GT* g = reinterpret_cast<const GT*>(s.g);
  float acc = 0.f;
  if (g != nullptr) {
    uint32_t i = begin + threadIdx.x;
    if ((reinterpret_cast<uintptr_t>(g) & (sizeof(GT) == 4 ? 31u : 15u)) == 0) {
      const uint32_t vend = begin + ((end - begin) & ~7u);
      for (uint32_t v = begin + threadIdx.x * 8; v < vend; v += blockDim.x * 8) {
        float f[8];
        load8_copy<GT>(g + v, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += f[j] * f[j];
      }
      i = vend + threadIdx.x;
    }
    for (; i < end; i += blockDim.x) {
      const float v = to_f32<GT>(g[i]);
      acc += v * v;
    }
  }
  const float total = block_sum(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) clip_coef_kernel(const float* __restrict__ partials, int n, float max_norm,
                                                         float grad_scale, float* __restrict__ coef_out,
                                                         float* __restrict__ norm_out) {
  __shared__ float red[33];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partials[i];   // fixed order -> deterministic
  const float total = block_sum(acc, red);
  if (threadIdx.x == 0) {
    const float norm = sqrtf(total) * grad_scale;
    if (norm_out) *norm_out = norm;
    // torch.nn.utils.clip_grad_norm_: coef = clamp(max_norm / (norm + 1e-6), max=1)
    float coef = max_norm / (norm + 1e-6f);
    *coef_out = (max_norm > 0.f) ? fminf(coef, 1.f) : 1.f;
  }
}

struct SgdScalars { float lr, coef, momentum, dampening, weight_decay; bool first, nesterov; };

__device__ __forceinline__ float sgd_update(float w, float g, float* m, const SgdScalars& c, bool has_mom) {
  float d = g * c.coef;
  if (c.weight_decay != 0.f) d += c.weight_decay * w;
  if (has_mom) {
    const float mm = c.first ? d : c.momentum * (*m) + (1.f - c.dampening) * d;
    *m = mm;
    d = c.nesterov ? d + c.momentum * mm : mm;
  }
  return w - c.lr * d;
}

template <typename PT, typename GT>
__global__ void __launch_bounds__(kOptThreads) multi_sgd_kernel(const __grid_constant__ OptTable tab, const __grid_constant__ SgdHyper h) {
  __shared__ uint32_t blk0[kMaxOptTensors];
  for (int i = threadIdx.x; i < tab.count; i += blockDim.x) blk0[i] = tab.t[i].blk0;
  __syncthreads();
  const int k = find_tensor(blk0, tab.count, blockIdx.x);
  const OptSlot& s = tab.t[k];
  if (s.g == nullptr) return;   // parameter without a gradient: untouched, like torch
  const uint32_t begin = (blockIdx.x - s.blk0) * kOptChunk;
  const uint32_t end = min(begin + (uint32_t)kOptChunk, s.numel);
  PT* p = reinterpret_cast<PT*>(s.p);
  GT* g = reinterpret_cast<GT*>(const_cast<void*>(s.g));
  float* master = h.master ? h.master + s.flat_off : nullptr;
  float* mom = h.momentum_buf ? h.momentum_buf + s.flat_off : nullptr;
  SgdScalars c;
  c.lr = *h.lr;
  c.coef = (h.clip_coef ? *h.clip_coef : 1.f) * h.grad_scale;
  c.momentum = h.momentum; c.dampening = h.dampening; c.weight_decay = h.weight_decay;
  c.first = h.step_count ? (*h.step_count == 0) : false;
  c.nesterov = h.nesterov != 0;
  const bool has_mom = mom != nullptr;

  // vector path: chunk starts are multiples of 8 elements; only the base pointers need checking
  const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15u) == 0 &&
                       (!master || (reinterpret_cast<uintptr_t>(master) & 31u) == 0) &&
                       (!mom || (reinterpret_cast<uintptr_t>(mom) & 31u) == 0) &&
                       (sizeof(PT) == 2 || (reinterpret_cast<uintptr_t>(p) & 31u) == 0) &&
                       (sizeof(GT) == 2 || (reinterpret_cast<uintptr_t>(g) & 31u) == 0);
  uint32_t i = begin;
  if (aligned) {
    const uint32_t vend = begin + ((end - begin) & ~7u);
    for (i = begin + threadIdx.x * 8; i < vend; i += blockDim.x * 8) {
      float w[8], gr[8], m[8];
      load8_copy<GT>(g + i, gr);
      if (master) load8<float>(master + i, w); else load8_copy<PT>(p + i, w);
      if (has_mom) load8<float>(mom + i, m);
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = sgd_update(w[j], gr[j], &m[j], c, has_mom);
      if (master) store8<float>(master + i, w);
      store8<PT>(p + i, w);
      if (has_mom) store8<float>(mom + i, m);
      if (h.zero_grad) {
        float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        store8<GT>(g + i, z);
      }
    }
    i = vend + threadIdx.x;
  } else {
    i = begin + threadIdx.x;
  }
  for (; i < end; i += blockDim.x) {     // unaligned tensors and the (< 8 element) tail
    float w = master ? master[i] : to_f32<PT>(p[i]);
    float m = has_mom ? mom[i] : 0.f;
    w = sgd_update(w, to_f32<GT>(g[i]), &m, c, has_mom);
    if (master) master[i] = w;
    p[i] = from_f32<PT>(w);
    if (has_mom) mom[i] = m;
    if (h.zero_grad) g[i] = from_f32<GT>(0.f);
  }
}

struct AdamScalars { float coef, beta1, beta2, eps, decay, step_size, bc2_sqrt; };

// torch.optim.AdamW's update, in its operation order: decoupled decay, lerp / addcmul moments, eps outside the
// bias-corrected sqrt
__device__ __forceinline__ float adamw_update(float w, float g, float* m, float* v, const AdamScalars& c) {
  g *= c.coef;
  w *= c.decay;
  const float mm = *m + (1.f - c.beta1) * (g - *m);
  const float vv = c.beta2 * (*v) + (1.f - c.beta2) * g * g;
  *m = mm;
  *v = vv;
  const float denom = sqrtf(vv) / c.bc2_sqrt + c.eps;
  return w - c.step_size * (mm / denom);
}

template <typename PT, typename GT>
__global__ void __launch_bounds__(kOptThreads) multi_adamw_kernel(const __grid_constant__ OptTable tab, const __grid_constant__ AdamHyper h) {
  __shared__ uint32_t blk0[kMaxOptTensors];
  __shared__ float s_step_size, s_bc2_sqrt, s_decay;
  for (int i = threadIdx.x; i < tab.count; i += blockDim.x) blk0[i] = tab.t[i].blk0;
  if (threadIdx.x == 0) {
    // read on the device, so every replay of a captured step advances the bias correction
    const double t = (double)(*h.step_count + 1);
    const float lr = *h.lr;
    s_step_size = (float)((double)lr / (1.0 - pow((double)h.beta1, t)));
    s_bc2_sqrt = (float)sqrt(1.0 - pow((double)h.beta2, t));
    s_decay = 1.f - lr * h.weight_decay;
  }
  __syncthreads();
  const int k = find_tensor(blk0, tab.count, blockIdx.x);
  const OptSlot& s = tab.t[k];
  if (s.g == nullptr) return;   // parameter without a gradient: weights and moments untouched, like torch
  const uint32_t begin = (blockIdx.x - s.blk0) * kOptChunk;
  const uint32_t end = min(begin + (uint32_t)kOptChunk, s.numel);
  PT* p = reinterpret_cast<PT*>(s.p);
  GT* g = reinterpret_cast<GT*>(const_cast<void*>(s.g));
  float* master = h.master ? h.master + s.flat_off : nullptr;
  float* m1 = h.exp_avg + s.flat_off;
  float* m2 = h.exp_avg_sq + s.flat_off;
  AdamScalars c;
  c.coef = (h.clip_coef ? *h.clip_coef : 1.f) * h.grad_scale;
  c.beta1 = h.beta1; c.beta2 = h.beta2; c.eps = h.eps;
  c.decay = s_decay; c.step_size = s_step_size; c.bc2_sqrt = s_bc2_sqrt;

  // vector path: chunk starts are multiples of 8 elements; only the base pointers need checking
  const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15u) == 0 &&
                       (!master || (reinterpret_cast<uintptr_t>(master) & 31u) == 0) &&
                       ((reinterpret_cast<uintptr_t>(m1) | reinterpret_cast<uintptr_t>(m2)) & 31u) == 0 &&
                       (sizeof(PT) == 2 || (reinterpret_cast<uintptr_t>(p) & 31u) == 0) &&
                       (sizeof(GT) == 2 || (reinterpret_cast<uintptr_t>(g) & 31u) == 0);
  uint32_t i = begin;
  if (aligned) {
    const uint32_t vend = begin + ((end - begin) & ~7u);
    for (i = begin + threadIdx.x * 8; i < vend; i += blockDim.x * 8) {
      float w[8], gr[8], m[8], v[8];
      load8_copy<GT>(g + i, gr);
      if (master) load8<float>(master + i, w); else load8_copy<PT>(p + i, w);
      load8<float>(m1 + i, m);
      load8<float>(m2 + i, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = adamw_update(w[j], gr[j], &m[j], &v[j], c);
      if (master) store8<float>(master + i, w);
      store8<PT>(p + i, w);
      store8<float>(m1 + i, m);
      store8<float>(m2 + i, v);
      if (h.zero_grad) {
        float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        store8<GT>(g + i, z);
      }
    }
    i = vend + threadIdx.x;
  } else {
    i = begin + threadIdx.x;
  }
  for (; i < end; i += blockDim.x) {     // unaligned tensors and the (< 8 element) tail
    float w = master ? master[i] : to_f32<PT>(p[i]);
    float m = m1[i], v = m2[i];
    w = adamw_update(w, to_f32<GT>(g[i]), &m, &v, c);
    if (master) master[i] = w;
    p[i] = from_f32<PT>(w);
    m1[i] = m;
    m2[i] = v;
    if (h.zero_grad) g[i] = from_f32<GT>(0.f);
  }
}

__global__ void scale_inplace_kernel(float* x, size_t n, const float* scalar) {
  const float s = *scalar;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) x[i] *= s;
}

}  // namespace

void launch_multi_sqnorm(const OptTable& tab, DType g_dtype, float* partials, cudaStream_t s) {
  if (tab.total_blocks <= 0) return;
  if (g_dtype == DType::BF16) multi_sqnorm_kernel<__nv_bfloat16><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, partials);
  else multi_sqnorm_kernel<float><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, partials);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_clip_coef(const float* partials, int n, float max_norm, float grad_scale, float* coef_out, float* norm_out,
                      cudaStream_t s) {
  clip_coef_kernel<<<1, 1024, 0, s>>>(partials, n, max_norm, grad_scale, coef_out, norm_out);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_multi_sgd(const OptTable& tab, DType p_dtype, DType g_dtype, const SgdHyper& h, cudaStream_t s) {
  if (tab.total_blocks <= 0) return;
  const bool pb = p_dtype == DType::BF16, gb = g_dtype == DType::BF16;
  if (pb && gb) multi_sgd_kernel<__nv_bfloat16, __nv_bfloat16><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  else if (pb) multi_sgd_kernel<__nv_bfloat16, float><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  else if (gb) multi_sgd_kernel<float, __nv_bfloat16><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  else multi_sgd_kernel<float, float><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_multi_adamw(const OptTable& tab, DType p_dtype, DType g_dtype, const AdamHyper& h, cudaStream_t s) {
  if (tab.total_blocks <= 0) return;
  const bool pb = p_dtype == DType::BF16, gb = g_dtype == DType::BF16;
  if (pb && gb) multi_adamw_kernel<__nv_bfloat16, __nv_bfloat16><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  else if (pb) multi_adamw_kernel<__nv_bfloat16, float><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  else if (gb) multi_adamw_kernel<float, __nv_bfloat16><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  else multi_adamw_kernel<float, float><<<tab.total_blocks, kOptThreads, 0, s>>>(tab, h);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_scale_inplace(float* x, size_t n, const float* scalar, cudaStream_t s) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  if (blocks < 1) blocks = 1;
  scale_inplace_kernel<<<blocks, 256, 0, s>>>(x, n, scalar);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
