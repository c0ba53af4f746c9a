// Vision Transformer patch embedding.  A batch of B images becomes one token stream of T = round_up(B (N + 1), 128) rows:
// image b owns rows [b (N + 1), (b + 1) (N + 1)), its class token first and its N patches after it in raster order; the
// rows past B (N + 1) are padding.  The attention kernels' document bounds then keep every image to itself
// (``ops.image_token_bounds``), and every linear runs on all T rows.
//   patchify   image (bf16, NCHW or channels_last) -> patch matrix [T, C p p] in token order, the K order of the flattened
//              [D, C, p, p] convolution weight (c, ky, kx); class and padding rows are zero
//   assemble   GEMM output [T, D] -> tokens: class_token + pos[0] at class rows, patch + pos[1 + i] at patch rows (fp32 add,
//              one bf16 rounding), exact zeros at padding rows
//   backward   dy [T, D] -> the patch rows' gradient for the weight-gradient GEMM (dy at patch rows, zero elsewhere) and
//              d pos [N + 1, D] = sum over the B images of dy at each image's row, a fixed-order fp32 sum (no atomics),
//              and d class_token = d pos[0]
#include "ops.h"

namespace b200 {
namespace {

// one thread per 8 consecutive k of one token row: (c, ky, kx..kx+7) with p % 8 == 0, so the 8 pixels lie on one image row
template <bool kChannelsLast>
__global__ void __launch_bounds__(256) patchify_kernel(const __nv_bfloat16* __restrict__ img, __nv_bfloat16* __restrict__ out, int B,
                                                       int C, int H, int W, int p, int T) {
  const int gw = W / p, n = (H / p) * gw, per = n + 1, k8 = C * p * p / 8;
  const size_t total = (size_t)T * k8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / k8), k = (int)(i % k8) * 8;
    const int b = t / per, j = t % per;
    Bf16x8 v;
    if (b >= B || j == 0) {
      v.h[0] = v.h[1] = v.h[2] = v.h[3] = __floats2bfloat162_rn(0.f, 0.f);
    } else {
      const int q = j - 1, c = k / (p * p), r = k % (p * p);
      const int y = (q / gw) * p + r / p, x = (q % gw) * p + r % p;
      if (kChannelsLast) {
        const __nv_bfloat16* s = img + (((size_t)b * H + y) * W + x) * C + c;
        __nv_bfloat16 e[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) e[u] = s[(size_t)u * C];
#pragma unroll
        for (int u = 0; u < 4; ++u) v.h[u] = __halves2bfloat162(e[2 * u], e[2 * u + 1]);
      } else {
        v = *reinterpret_cast<const Bf16x8*>(img + (((size_t)b * C + c) * H + y) * W + x);
      }
    }
    *reinterpret_cast<Bf16x8*>(out + (size_t)t * (C * p * p) + k) = v;
  }
}

__global__ void __launch_bounds__(256) patch_assemble_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ cls,
                                                             const __nv_bfloat16* __restrict__ pos, __nv_bfloat16* __restrict__ out,
                                                             int B, int per, int D, int T) {
  const int d8 = D / 8;
  const size_t total = (size_t)T * d8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / d8), d = (int)(i % d8) * 8;
    const int b = t / per, j = t % per;
    float f[8], g[8];
    if (b >= B) {
#pragma unroll
      for (int u = 0; u < 8; ++u) f[u] = 0.f;
    } else {
      load8(j == 0 ? cls + d : y + (size_t)t * D + d, f);
      load8(pos + (size_t)j * D + d, g);
#pragma unroll
      for (int u = 0; u < 8; ++u) f[u] += g[u];
    }
    store8(out + (size_t)t * D + d, f);
  }
}

// Items [0, per * D/8): one (image row j, 8 columns) each, summing dy over the B images in order b = 0..B-1 and writing
// the patch-row gradient of those B rows on the way.  Items past that: 8 columns of one padding row, zeroed.
__global__ void __launch_bounds__(256) patch_embed_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dpatch,
                                                              __nv_bfloat16* __restrict__ dpos, __nv_bfloat16* __restrict__ dcls, int B,
                                                              int per, int D, int T) {
  const int d8 = D / 8;
  const size_t sums = (size_t)per * d8, total = sums + (size_t)(T - B * per) * d8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float zero[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) zero[u] = 0.f;
    if (i >= sums) {
      const size_t z = i - sums;
      const int t = B * per + (int)(z / d8), d = (int)(z % d8) * 8;
      store8(dpatch + (size_t)t * D + d, zero);
      continue;
    }
    const int j = (int)(i / d8), d = (int)(i % d8) * 8;
    float acc[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] = 0.f;
#pragma unroll 4
    for (int b = 0; b < B; ++b) {
      const size_t off = ((size_t)b * per + j) * D + d;
      float f[8];
      load8(dy + off, f);
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] += f[u];
      if (j == 0) store8(dpatch + off, zero);
      else *reinterpret_cast<Bf16x8*>(dpatch + off) = *reinterpret_cast<const Bf16x8*>(dy + off);
    }
    store8(dpos + (size_t)j * D + d, acc);
    if (j == 0) store8(dcls + d, acc);           // the class token enters where pos[0] does
  }
}

int grid_for(size_t items) {
  size_t blocks = (items + 255) / 256;
  if (blocks > (size_t)16 * kNumSMs) blocks = (size_t)16 * kNumSMs;
  return blocks < 1 ? 1 : (int)blocks;
}

}  // namespace

void launch_patchify(const void* img, bool channels_last, int B, int C, int H, int W, int p, int T, void* out, cudaStream_t s) {
  const int blocks = grid_for((size_t)T * (C * p * p / 8));
  if (channels_last)
    patchify_kernel<true><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)img, (__nv_bfloat16*)out, B, C, H, W, p, T);
  else
    patchify_kernel<false><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)img, (__nv_bfloat16*)out, B, C, H, W, p, T);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_patch_assemble(const void* y, const void* cls, const void* pos, int B, int per, int D, int T, void* out, cudaStream_t s) {
  patch_assemble_kernel<<<grid_for((size_t)T * (D / 8)), 256, 0, s>>>((const __nv_bfloat16*)y, (const __nv_bfloat16*)cls,
                                                                     (const __nv_bfloat16*)pos, (__nv_bfloat16*)out, B, per, D, T);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_patch_embed_bwd(const void* dy, int B, int per, int D, int T, void* dpatch, void* dpos, void* dcls, cudaStream_t s) {
  patch_embed_bwd_kernel<<<grid_for((size_t)(per + T - B * per) * (D / 8)), 256, 0, s>>>(
      (const __nv_bfloat16*)dy, (__nv_bfloat16*)dpatch, (__nv_bfloat16*)dpos, (__nv_bfloat16*)dcls, B, per, D, T);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
