// 3x3 / stride-2 / pad-1 max pooling for channels_last activations (the ResNet stem), forward + backward.
// ATen's max_pool_backward_nhwc is far from the copy rate for its ~64 MB of traffic at batch 32; both
// directions here are single-pass, 16-byte-vector kernels.  Forward stores the arg-max window slot (0..8) per
// element in one byte, so backward is a pure gather: every input pixel looks at the <= 4 output windows that
// cover it and sums the gradients whose recorded slot points back at it - no atomics, deterministic.
#include "ops.h"

namespace b200 {
namespace {

constexpr int kPoolThreads = 256;

template <typename T> __device__ __forceinline__ void pl_load8(const T* p, float* f);
template <> __device__ __forceinline__ void pl_load8<__nv_bfloat16>(const __nv_bfloat16* p, float* f) { unpack8(*reinterpret_cast<const Bf16x8*>(p), f); }
template <> __device__ __forceinline__ void pl_load8<float>(const float* p, float* f) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
template <typename T> __device__ __forceinline__ void pl_store8(T* p, const float* f);
template <> __device__ __forceinline__ void pl_store8<__nv_bfloat16>(__nv_bfloat16* p, const float* f) { *reinterpret_cast<Bf16x8*>(p) = pack8(f); }
template <> __device__ __forceinline__ void pl_store8<float>(float* p, const float* f) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}

// x [N,H,W,C] -> y [N,OH,OW,C], idx [N,OH,OW,C] (uint8 slot = ky*3+kx)
template <typename T>
__global__ void __launch_bounds__(kPoolThreads) maxpool3x3s2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, unsigned char* __restrict__ idx,
                                                                       int N, int H, int W, int C, int OH, int OW) {
  const int cvn = C / 8;
  const size_t total = (size_t)N * OH * OW * cvn;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(v % cvn);
    size_t p = v / cvn;
    const int ow = (int)(p % OW); p /= OW;
    const int oh = (int)(p % OH);
    const int n = (int)(p / OH);
    float best[8];
    unsigned int slot[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { best[i] = -INFINITY; slot[i] = 0; }
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int ih = oh * 2 - 1 + ky;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int iw = ow * 2 - 1 + kx;
        if (iw < 0 || iw >= W) continue;
        float f[8];
        pl_load8<T>(x + (((size_t)n * H + ih) * W + iw) * C + cv * 8, f);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (f[i] > best[i] || (f[i] != f[i])) { best[i] = f[i]; slot[i] = ky * 3 + kx; }     // first max wins, NaN propagates (torch semantics)
      }
    }
    const size_t o = (((size_t)n * OH + oh) * OW + ow) * C + cv * 8;
    pl_store8<T>(y + o, best);
    uint2 packed;
    packed.x = slot[0] | (slot[1] << 8) | (slot[2] << 16) | (slot[3] << 24);
    packed.y = slot[4] | (slot[5] << 8) | (slot[6] << 16) | (slot[7] << 24);
    *reinterpret_cast<uint2*>(idx + o) = packed;
  }
}

template <typename T>
__global__ void __launch_bounds__(kPoolThreads) maxpool3x3s2_bwd_kernel(const T* __restrict__ dy, const unsigned char* __restrict__ idx, T* __restrict__ dx,
                                                                       int N, int H, int W, int C, int OH, int OW) {
  const int cvn = C / 8;
  const size_t total = (size_t)N * H * W * cvn;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(v % cvn);
    size_t p = v / cvn;
    const int iw = (int)(p % W); p /= W;
    const int ih = (int)(p % H);
    const int n = (int)(p / H);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    // output windows covering (ih, iw): oh in {floor((ih+1)/2) - 1 .. floor((ih+1)/2)} intersected with ih - (2*oh-1) in [0,3)
    const int oh_hi = min((ih + 1) / 2, OH - 1), ow_hi = min((iw + 1) / 2, OW - 1);
    for (int oh = max(0, (ih + 1) / 2 - 1); oh <= oh_hi; ++oh) {
      const int ky = ih - (oh * 2 - 1);
      if (ky < 0 || ky > 2) continue;
      for (int ow = max(0, (iw + 1) / 2 - 1); ow <= ow_hi; ++ow) {
        const int kx = iw - (ow * 2 - 1);
        if (kx < 0 || kx > 2) continue;
        const size_t o = (((size_t)n * OH + oh) * OW + ow) * C + cv * 8;
        const uint2 packed = *reinterpret_cast<const uint2*>(idx + o);
        float g[8];
        pl_load8<T>(dy + o, g);
        const unsigned int want = ky * 3 + kx;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const unsigned int s = ((i < 4 ? packed.x : packed.y) >> (8 * (i & 3))) & 0xffu;
          if (s == want) acc[i] += g[i];
        }
      }
    }
    pl_store8<T>(dx + (((size_t)n * H + ih) * W + iw) * C + cv * 8, acc);
  }
}

int pool_blocks(size_t total) {
  size_t b = (total + kPoolThreads - 1) / kPoolThreads;
  if (b > (size_t)kNumSMs * 16) b = (size_t)kNumSMs * 16;
  return (int)(b < 1 ? 1 : b);
}

}  // namespace

void launch_maxpool3x3s2_fwd(const void* x, void* y, unsigned char* idx, DType dt, int N, int H, int W, int C, cudaStream_t s) {
  if (C % 8 != 0) throw std::runtime_error("maxpool3x3s2: channels must be a multiple of 8");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const size_t total = (size_t)N * OH * OW * (C / 8);
  if (dt == DType::BF16) maxpool3x3s2_fwd_kernel<__nv_bfloat16><<<pool_blocks(total), kPoolThreads, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, idx, N, H, W, C, OH, OW);
  else maxpool3x3s2_fwd_kernel<float><<<pool_blocks(total), kPoolThreads, 0, s>>>((const float*)x, (float*)y, idx, N, H, W, C, OH, OW);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_maxpool3x3s2_bwd(const void* dy, const unsigned char* idx, void* dx, DType dt, int N, int H, int W, int C, cudaStream_t s) {
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const size_t total = (size_t)N * H * W * (C / 8);
  if (dt == DType::BF16) maxpool3x3s2_bwd_kernel<__nv_bfloat16><<<pool_blocks(total), kPoolThreads, 0, s>>>((const __nv_bfloat16*)dy, idx, (__nv_bfloat16*)dx, N, H, W, C, OH, OW);
  else maxpool3x3s2_bwd_kernel<float><<<pool_blocks(total), kPoolThreads, 0, s>>>((const float*)dy, idx, (float*)dx, N, H, W, C, OH, OW);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
