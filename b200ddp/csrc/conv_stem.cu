// Operand packing for the strided 7x7 stem convolution (conv.h: launch_stem_conv_fprop / launch_stem_conv_wgrad).
// Reference hot path replaced: the first convolution of the model's forward / backward (the reference ddp.py:221,231), which
// the library runs as a padded-to-8-channels kernel (bench/stem_bench.py times both).
#include "conv.h"

#include <cuda_bf16.h>

namespace b200 {
namespace {

__device__ __forceinline__ uint2 stem_load_pixel(const __nv_bfloat16* x, int n, int h, int w, int H, int W) {
  uint2 out = make_uint2(0u, 0u);
  if (h >= 0 && h < H && w >= 0 && w < W) {
    const unsigned short* src = reinterpret_cast<const unsigned short*>(x) + (((long long)n * H + h) * W + w) * 3;
    const unsigned int c0 = __ldg(src), c1 = __ldg(src + 1), c2 = __ldg(src + 2);
    out.x = c0 | (c1 << 16);
    out.y = c2;
  }
  return out;
}

// xp[n, i, wp, 0..7] = { x[n, 2i - 3, wp - 4, 0..2], 0, x[n, 2i - 2, wp - 4, 0..2], 0 }, zero outside the image.
// One thread per packed pixel (16-byte store).
__global__ void __launch_bounds__(256) stem_pack_input_kernel(const __nv_bfloat16* __restrict__ x, uint4* __restrict__ xp, int N, int H, int W,
                                                              int Hp2, int Wp) {
  const long long total = (long long)N * Hp2 * Wp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wp = (int)(i % Wp);
    const long long t = i / Wp;
    const int ip = (int)(t % Hp2), n = (int)(t / Hp2);
    const int w = wp - 4, h0 = 2 * ip - 3;
    const uint2 a = stem_load_pixel(x, n, h0, w, H, W), b = stem_load_pixel(x, n, h0 + 1, w, H, W);
    xp[i] = make_uint4(a.x, a.y, b.x, b.y);
  }
}

// packed filter index -> (r, s, c) of the 7x7x3 filter, or false where the packed element is structural zero
__device__ __forceinline__ bool stem_k_to_rsc(int k, int* r, int* s, int* c) {
  const int j = k & 7, p = (k >> 3) & 7, t = k >> 6;          // k = t * 64 + p * 8 + j
  *r = 2 * t + (j >> 2); *c = j & 3; *s = p - 1;
  return *c < 3 && *r < 7 && p >= 1;
}

// w2[co, k] = w[co, r, s, c]   (w is [Cout,7,7,3])
__global__ void __launch_bounds__(256) stem_pack_weight_kernel(const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ w2, int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = i % kStemK, co = i / kStemK;
  int r, s, c;
  __nv_bfloat16 v = __float2bfloat16(0.f);
  if (stem_k_to_rsc(k, &r, &s, &c)) v = w[((co * 7 + r) * 7 + s) * 3 + c];
  w2[i] = v;
}

// dw[co, r, s, c] = dw2[co, k(r, s, c)]  (or dw2[k, co] when transposed)
__global__ void __launch_bounds__(256) stem_unpack_wgrad_kernel(const __nv_bfloat16* __restrict__ dw2, __nv_bfloat16* __restrict__ dw, int total, int Cout,
                                                                int transposed) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = i % 3;
  int t = i / 3;
  const int s = t % 7; t /= 7;
  const int r = t % 7, co = t / 7;
  const int k = (r >> 1) * 64 + (s + 1) * 8 + (r & 1) * 4 + c;
  dw[i] = transposed ? dw2[(size_t)k * Cout + co] : dw2[(size_t)co * kStemK + k];
}

}  // namespace

void launch_stem_pack_input(const void* x_nhwc3, void* xp, int N, int H, int W, cudaStream_t stream) {
  StemGeom g;
  if (!stem_geom(H, W, &g)) throw std::runtime_error("stem conv: unsupported image size");
  const long long total = (long long)N * g.Hp2 * g.Wp;
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)kNumSMs * 32);
  stem_pack_input_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(x_nhwc3), reinterpret_cast<uint4*>(xp), N, H, W, g.Hp2, g.Wp);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_stem_pack_weight(const void* w_krsc3, void* w2, int Cout, cudaStream_t stream) {
  const int total = Cout * kStemK;
  stem_pack_weight_kernel<<<(total + 255) / 256, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(w_krsc3), reinterpret_cast<__nv_bfloat16*>(w2), total);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_stem_unpack_wgrad(const void* dw2, void* dw_krsc3, int Cout, bool transposed, cudaStream_t stream) {
  const int total = Cout * 7 * 7 * 3;
  stem_unpack_wgrad_kernel<<<(total + 255) / 256, 256, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(dw2), reinterpret_cast<__nv_bfloat16*>(dw_krsc3), total,
                                                                   Cout, transposed ? 1 : 0);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
