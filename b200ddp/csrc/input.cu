// Input pipeline kernel (reference: the blocking `x, y = x.to(args.device), y.to(args.device)` at ddp.py:220 moves fp32
// tensors as they are).  Here the host ships raw NCHW batches (uint8 pixels or fp32) from pinned memory;
// this kernel does scale/mean/std normalisation, the cast to the compute dtype and the NCHW ->
// channels_last permutation in one pass (the stock path would be .float(), sub_, div_, .to(bf16),
// .contiguous(channels_last) = 5 launches and 5 round trips through HBM).
#include "ops.h"

namespace b200 {
namespace {

template <typename SrcT, typename DstT>
__global__ void __launch_bounds__(256) normalize_cl_kernel(const SrcT* __restrict__ src, DstT* __restrict__ dst, int n, int c, int c_out, int h, int w,
                                                           const float* __restrict__ mean, const float* __restrict__ inv_std, float in_scale) {
  // thread per output pixel position (n, y, x): reads C planes (coalesced across x), writes C_out contiguous values
  // (channels [c, c_out) are zero: a 3-channel image padded to 8 gives the stem convolution a 16-byte-aligned
  // NHWC operand, which is what the bf16 tensor-core convolution kernels need)
  const size_t hw = (size_t)h * w;
  const size_t total = (size_t)n * hw;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t img = i / hw, pix = i % hw;
    const SrcT* s = src + img * c * hw + pix;
    DstT* d = dst + i * c_out;
    for (int ch = 0; ch < c; ++ch) {
      float v = (float)s[(size_t)ch * hw] * in_scale;
      v = (v - mean[ch]) * inv_std[ch];
      d[ch] = from_f32<DstT>(v);
    }
    for (int ch = c; ch < c_out; ++ch) d[ch] = from_f32<DstT>(0.f);
  }
}

}  // namespace

void launch_normalize_to_channels_last(const void* src, DType src_dt, void* dst, DType dst_dt, int n, int c, int c_out, int h, int w,
                                       const float* mean, const float* inv_std, float in_scale, cudaStream_t s) {
  const size_t total = (size_t)n * h * w;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 16 * kNumSMs) blocks = 16 * kNumSMs;
  if (blocks < 1) blocks = 1;
  const bool su8 = src_dt == DType::U8, dbf = dst_dt == DType::BF16;
  if (su8 && dbf) normalize_cl_kernel<unsigned char, __nv_bfloat16><<<blocks, 256, 0, s>>>((const unsigned char*)src, (__nv_bfloat16*)dst, n, c, c_out, h, w, mean, inv_std, in_scale);
  else if (su8) normalize_cl_kernel<unsigned char, float><<<blocks, 256, 0, s>>>((const unsigned char*)src, (float*)dst, n, c, c_out, h, w, mean, inv_std, in_scale);
  else if (dbf) normalize_cl_kernel<float, __nv_bfloat16><<<blocks, 256, 0, s>>>((const float*)src, (__nv_bfloat16*)dst, n, c, c_out, h, w, mean, inv_std, in_scale);
  else normalize_cl_kernel<float, float><<<blocks, 256, 0, s>>>((const float*)src, (float*)dst, n, c, c_out, h, w, mean, inv_std, in_scale);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
