// CLIP's contrastive loss (Radford et al., 2021).  A rank holds B image-caption pairs; the loss contrasts each of its
// images against the N = world B captions of the global batch and each of its captions against the N images.
//   l2norm      x bf16 [B, D] -> u = x / ||x|| (fp32, one bf16 rounding), rnorm = 1 / ||x|| fp32 [B]; no eps, as
//               transformers' CLIPModel.  Backward: dx = rnorm (du - u <u, du>), u recomputed in fp32 from x.
//   contrastive z_img = u_img U_txt^T and z_txt = u_txt U_img^T (fp32 [B, N], the wgmma GEMM's), s = exp(logit_scale):
//               per row r of either matrix, with label l = offset + r, the log-sum-exp of s z in fp32, the loss term
//               lse - s z[l], dz = s (softmax - onehot) / (2B) in bf16 and the row's part of
//               d logit_scale = sum_j (softmax - onehot)_j s z_j / (2B).  A second one-block kernel sums the 2B loss terms
//               and d logit_scale parts in a fixed order (no atomics): the results are bitwise repeatable.
// Nothing is read back to the host; logit_scale stays on the device.
#include "ops.h"

namespace b200 {
namespace {

constexpr int kNormThreads = 256;     // 8 warps, one row each
constexpr int kXentThreads = 256;

__global__ void __launch_bounds__(kNormThreads) l2norm_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ u,
                                                                  float* __restrict__ rnorm, int B, int D) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (kNormThreads / 32) + (threadIdx.x >> 5);
  if (r >= B) return;
  const __nv_bfloat16* xr = x + (size_t)r * D;
  float ss = 0.f;
  for (int d = lane * 8; d < D; d += 32 * 8) {
    float f[8];
    load8(xr + d, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  }
  ss = warp_sum(ss);
  const float rn = 1.f / sqrtf(ss);
  for (int d = lane * 8; d < D; d += 32 * 8) {
    float f[8];
    load8(xr + d, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] *= rn;
    store8(u + (size_t)r * D + d, f);
  }
  if (lane == 0) rnorm[r] = rn;
}

__global__ void __launch_bounds__(kNormThreads) l2norm_bwd_kernel(const __nv_bfloat16* __restrict__ du, const __nv_bfloat16* __restrict__ x,
                                                                  const float* __restrict__ rnorm, __nv_bfloat16* __restrict__ dx, int B, int D) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (kNormThreads / 32) + (threadIdx.x >> 5);
  if (r >= B) return;
  const size_t off = (size_t)r * D;
  const float rn = rnorm[r];
  float dot = 0.f;
  for (int d = lane * 8; d < D; d += 32 * 8) {
    float f[8], g[8];
    load8(x + off + d, f);
    load8(du + off + d, g);
#pragma unroll
    for (int i = 0; i < 8; ++i) dot += f[i] * rn * g[i];
  }
  dot = warp_sum(dot);
  for (int d = lane * 8; d < D; d += 32 * 8) {
    float f[8], g[8];
    load8(x + off + d, f);
    load8(du + off + d, g);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = rn * (g[i] - f[i] * rn * dot);
    store8(dx + off + d, g);
  }
}

// One block per row: blockIdx.y = 0 reads z_img, 1 reads z_txt.  Three passes over the row (it stays in L1 / L2): the
// maximum of s z, the sums of e = exp(s z - max) and of e z, then dz.
__global__ void __launch_bounds__(kXentThreads) contrastive_xent_kernel(const float* __restrict__ z_img, const float* __restrict__ z_txt,
                                                                        const float* __restrict__ logit_scale, int B, int N, int offset,
                                                                        __nv_bfloat16* __restrict__ dz_img, __nv_bfloat16* __restrict__ dz_txt,
                                                                        float* __restrict__ row_loss, float* __restrict__ row_dscale) {
  __shared__ float scratch[33];
  const int r = blockIdx.x, which = blockIdx.y;
  const float* z = (which ? z_txt : z_img) + (size_t)r * N;
  __nv_bfloat16* dz = (which ? dz_txt : dz_img) + (size_t)r * N;
  const float s = expf(*logit_scale);
  const int label = offset + r;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < N; j += kXentThreads) m = fmaxf(m, s * z[j]);
  m = block_max(m, scratch);
  float se = 0.f, sez = 0.f;
  for (int j = threadIdx.x; j < N; j += kXentThreads) {
    const float zj = z[j], e = expf(s * zj - m);
    se += e;
    sez += e * zj;
  }
  se = block_sum(se, scratch);
  sez = block_sum(sez, scratch);
  const float inv = 1.f / se, scale = s / (2.f * (float)B);
  for (int j = threadIdx.x; j < N; j += kXentThreads) {
    const float p = expf(s * z[j] - m) * inv;
    dz[j] = __float2bfloat16_rn(scale * (p - (j == label ? 1.f : 0.f)));
  }
  if (threadIdx.x == 0) {
    const float zl = z[label];
    row_loss[which * B + r] = m + logf(se) - s * zl;
    row_dscale[which * B + r] = scale * (sez * inv - zl);
  }
}

// loss = sum of the 2B loss terms / (2B), d logit_scale = sum of the 2B parts; each thread sums a fixed stride, then a
// fixed tree
__global__ void __launch_bounds__(kXentThreads) contrastive_finish_kernel(const float* __restrict__ row_loss, const float* __restrict__ row_dscale,
                                                                          int rows, float* __restrict__ loss, float* __restrict__ dscale) {
  __shared__ float scratch[33];
  float a = 0.f, b = 0.f;
  for (int i = threadIdx.x; i < rows; i += kXentThreads) {
    a += row_loss[i];
    b += row_dscale[i];
  }
  a = block_sum(a, scratch);
  b = block_sum(b, scratch);
  if (threadIdx.x == 0) {
    loss[0] = a / (float)rows;
    dscale[0] = b;
  }
}

}  // namespace

void launch_l2norm_fwd(const void* x, int B, int D, void* u, float* rnorm, cudaStream_t s) {
  l2norm_fwd_kernel<<<ceil_div(B, kNormThreads / 32), kNormThreads, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)u, rnorm, B, D);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_l2norm_bwd(const void* du, const void* x, const float* rnorm, int B, int D, void* dx, cudaStream_t s) {
  l2norm_bwd_kernel<<<ceil_div(B, kNormThreads / 32), kNormThreads, 0, s>>>((const __nv_bfloat16*)du, (const __nv_bfloat16*)x, rnorm,
                                                                            (__nv_bfloat16*)dx, B, D);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_contrastive_xent(const float* z_img, const float* z_txt, const float* logit_scale, int B, int N, int offset, void* dz_img,
                             void* dz_txt, float* row_partials, float* loss, float* dscale, cudaStream_t s) {
  contrastive_xent_kernel<<<dim3(B, 2), kXentThreads, 0, s>>>(z_img, z_txt, logit_scale, B, N, offset, (__nv_bfloat16*)dz_img,
                                                              (__nv_bfloat16*)dz_txt, row_partials, row_partials + 2 * B);
  B200_CUDA_CHECK(cudaGetLastError());
  contrastive_finish_kernel<<<1, kXentThreads, 0, s>>>(row_partials, row_partials + 2 * B, 2 * B, loss, dscale);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

}  // namespace b200
