// Shared helpers for the sm_90a extension.  Nothing here includes torch headers: kernels take raw
// pointers + cudaStream_t so each .cu compiles in seconds; only bindings.cpp sees torch/extension.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

#define B200_CUDA_CHECK(expr)                                                                      \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      throw std::runtime_error(std::string("CUDA error ") + cudaGetErrorString(_e) + " at " +      \
                               __FILE__ + ":" + std::to_string(__LINE__) + " in " #expr);          \
    }                                                                                              \
  } while (0)

#include <atomic>

namespace b200 {

// every kernel launch issued by this extension is counted (bench.py reports it as gpu_launches)
inline std::atomic<long long>& launch_counter() {
  static std::atomic<long long> c{0};
  return c;
}
#define B200_COUNT_LAUNCH(n) ::b200::launch_counter().fetch_add((n), std::memory_order_relaxed)

// Function attributes are per DEVICE: a process that drives several GPUs (the single-process DataParallel mode) must raise the
// dynamic shared-memory limit of a kernel once on each of them.  `done` is a per-call-site bit mask over device ordinals.
template <typename Kernel>
inline void ensure_max_dynamic_smem(Kernel kernel, int bytes, std::atomic<unsigned long long>& done) {
  int dev = 0;
  B200_CUDA_CHECK(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.fetch_or(bit, std::memory_order_release);
}

constexpr int kNumSMs = 132;  // H100 SXM
constexpr int kWarp = 32;

enum class DType : int { F32 = 0, BF16 = 1, U8 = 2, I64 = 3 };

inline size_t dtype_size(DType d) {
  switch (d) {
    case DType::F32: return 4;
    case DType::BF16: return 2;
    case DType::U8: return 1;
    case DType::I64: return 8;
  }
  return 0;
}

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Block-wide sum; every thread gets the result.  `scratch` holds >= 33 floats.
__device__ __forceinline__ float block_sum(float v, float* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  if (warp == 0) {
    float t = lane < nwarp ? scratch[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) scratch[32] = t;
  }
  __syncthreads();
  return scratch[32];
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  if (warp == 0) {
    float t = lane < nwarp ? scratch[lane] : -INFINITY;
    t = warp_max(t);
    if (lane == 0) scratch[32] = t;
  }
  __syncthreads();
  return scratch[32];
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// 16-byte vector of 8 bf16 <-> 8 floats
struct alignas(16) Bf16x8 { __nv_bfloat162 h[4]; };
__device__ __forceinline__ void unpack8(const Bf16x8& v, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(v.h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ Bf16x8 pack8(const float* f) {
  Bf16x8 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) v.h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}
// 8 consecutive elements <-> registers (16-byte / 32-byte vector accesses)
template <typename T> __device__ __forceinline__ void load8(const T* p, float* f);
template <> __device__ __forceinline__ void load8<float>(const float* p, float* f) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
  unpack8(*reinterpret_cast<const Bf16x8*>(p), f);
}
template <typename T> __device__ __forceinline__ void store8(T* p, const float* f);
template <> __device__ __forceinline__ void store8<float>(float* p, const float* f) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float* f) {
  *reinterpret_cast<Bf16x8*>(p) = pack8(f);
}
#endif

}  // namespace b200
