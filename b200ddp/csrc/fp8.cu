// FP8 quantisation for the FP8 linears: current per-tensor scaling with power-of-two scales.
//
//   amax = max|t|,   s = 2^e with e the largest integer such that amax * 2^e <= fmax (clamped to [-126, 127]; amax = 0
//   gives s = 1),   q = cvt.rn.satfinite(t * s),   dequantisation factor 1/s (exact).
//
// Two passes.  fp8_amax_kernel reduces max|t| over many CTAs with an atomicMax on the float bits (max is order
// independent, so the result is deterministic).  fp8_cast_transpose_kernel reads amax from device memory, derives s, and
// writes q and, optionally, q^T through a shared-memory tile with 16-byte stores: FP8 wgmma takes K-major operands only,
// so the backward GEMMs need the transposed copies.  For a gradient it can also produce the fp32 column sums (the bias
// gradient) in the same pass: per-tile partial sums in a fixed order plus a finishing kernel, no atomics.  Running the
// amax pass first leaves a tensor of up to a few tens of MB in L2 for the cast pass.
#include <cuda_fp8.h>

#include "common.h"
#include "ops.h"

namespace b200 {
namespace {

constexpr int kAmaxThreads = 256;
constexpr int kTile = 64;              // cast tile: 64 rows x 64 columns; thread t owns 16 consecutive columns of one row
constexpr int kCastThreads = 256;
constexpr int kTileTPitch = kTile + 16;   // bytes per row of the transposed tile (16-byte aligned rows)

__device__ __forceinline__ int fp8_scale_exponent(float amax, float fmax) {
  if (!(amax > 0.f) || !isfinite(amax)) return 0;            // all zeros (or a non-finite tensor): s = 1
  int ea, ef;
  const float ma = frexpf(amax, &ea), mf = frexpf(fmax, &ef);  // amax = ma 2^ea, fmax = mf 2^ef, mantissas in [0.5, 1)
  int e = ef - ea - (ma > mf ? 1 : 0);
  return e < -126 ? -126 : (e > 127 ? 127 : e);
}

__global__ void __launch_bounds__(kAmaxThreads) fp8_amax_kernel(const __nv_bfloat16* __restrict__ x, size_t n, float* amax) {
  __shared__ float scratch[33];
  float m = 0.f;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const size_t n8 = n / 8;
  for (size_t i = tid; i < n8; i += stride) {
    const Bf16x8 v = *reinterpret_cast<const Bf16x8*>(x + 8 * i);
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) m = fmaxf(m, fabsf(f[j]));
  }
  for (size_t i = 8 * n8 + tid; i < n; i += stride) m = fmaxf(m, fabsf(__bfloat162float(x[i])));
  m = block_max(m, scratch);
  // non-negative floats order like their bit patterns
  if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int*>(amax), __float_as_uint(m));
}

template <bool E5M2>
__global__ void __launch_bounds__(kCastThreads)
fp8_cast_transpose_kernel(const __nv_bfloat16* __restrict__ x, int rows, int cols, const float* __restrict__ amax,
                          uint8_t* __restrict__ q, uint8_t* __restrict__ qt, float* __restrict__ colsum_partial,
                          float* __restrict__ scale_inv) {
  constexpr float kFmax = E5M2 ? 57344.f : 448.f;
  constexpr __nv_fp8_interpretation_t kFmt = E5M2 ? __NV_E5M2 : __NV_E4M3;
  __shared__ alignas(16) uint8_t tile_t[kTile][kTileTPitch];      // [column][row]
  __shared__ float col_part[kCastThreads / 32][kTile];
  const int r0 = blockIdx.y * kTile, c0 = blockIdx.x * kTile;
  const int tid = threadIdx.x, lr = tid >> 2, lc = (tid & 3) * 16;
  const int e = fp8_scale_exponent(*amax, kFmax);
  const float s = ldexpf(1.f, e);
  if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0) *scale_inv = ldexpf(1.f, -e);

  const int r = r0 + lr, c = c0 + lc;
  const bool live = r < rows && c < cols;                          // cols % 16 == 0: a chunk is wholly in or out
  float f[16];
  if (live) {
    const Bf16x8* src = reinterpret_cast<const Bf16x8*>(x + (size_t)r * cols + c);
    unpack8(src[0], f);
    unpack8(src[1], f + 8);
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) f[i] = 0.f;
  }
  alignas(16) __nv_fp8x2_storage_t packed[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) packed[i] = __nv_cvt_float2_to_fp8x2(make_float2(f[2 * i] * s, f[2 * i + 1] * s), __NV_SATFINITE, kFmt);
  if (live) *reinterpret_cast<uint4*>(q + (size_t)r * cols + c) = *reinterpret_cast<const uint4*>(packed);

  if (qt != nullptr) {
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(packed);
#pragma unroll
    for (int i = 0; i < 16; ++i) tile_t[lc + i][lr] = bytes[i];
  }
  if (colsum_partial != nullptr) {
    // sum the 8 rows of this warp (lane bits 2..4), then the 8 warps in a fixed order
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
#pragma unroll
      for (int i = 0; i < 16; ++i) f[i] += __shfl_xor_sync(0xffffffffu, f[i], off);
    }
    if ((tid & 31) < 4) {
#pragma unroll
      for (int i = 0; i < 16; ++i) col_part[tid >> 5][lc + i] = f[i];
    }
  }
  __syncthreads();
  if (qt != nullptr) {
    const int tc = tid >> 2, tr = (tid & 3) * 16;                  // column of the tile, first of 16 rows
    if (c0 + tc < cols && r0 + tr < rows)                          // rows % 16 == 0: a chunk is wholly in or out
      *reinterpret_cast<uint4*>(qt + (size_t)(c0 + tc) * rows + r0 + tr) = *reinterpret_cast<const uint4*>(&tile_t[tc][tr]);
  }
  if (colsum_partial != nullptr && tid < kTile && c0 + tid < cols) {
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < kCastThreads / 32; ++w) acc += col_part[w][tid];
    colsum_partial[(size_t)blockIdx.y * cols + c0 + tid] = acc;
  }
}

__global__ void fp8_colsum_finish_kernel(const float* __restrict__ partial, int parts, int cols, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float acc = 0.f;
  for (int p = 0; p < parts; ++p) acc += partial[(size_t)p * cols + c];
  out[c] = acc;
}

}  // namespace

int fp8_colsum_parts(int rows) { return ceil_div(rows, kTile); }

void launch_fp8_amax(const void* x, size_t n, float* amax, cudaStream_t s) {
  if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) throw std::runtime_error("fp8_amax: input must be 16-byte aligned");
  B200_CUDA_CHECK(cudaMemsetAsync(amax, 0, sizeof(float), s));
  size_t blocks = (n / 8 + kAmaxThreads - 1) / kAmaxThreads;
  if (blocks < 1) blocks = 1;
  if (blocks > (size_t)8 * kNumSMs) blocks = (size_t)8 * kNumSMs;
  fp8_amax_kernel<<<(unsigned)blocks, kAmaxThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), n, amax);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_fp8_cast_transpose(const void* x, int rows, int cols, const float* amax, bool e5m2, void* q, void* qt,
                               float* colsum_partial, float* colsum, float* scale_inv, cudaStream_t s) {
  if (rows < 1 || cols < 1) throw std::runtime_error("fp8_cast_transpose: empty tensor");
  if (cols % 16 != 0) throw std::runtime_error("fp8_cast_transpose: columns (" + std::to_string(cols) + ") must be a multiple of 16");
  if (qt != nullptr && rows % 16 != 0)
    throw std::runtime_error("fp8_cast_transpose: the transposed copy needs rows (" + std::to_string(rows) + ") % 16 == 0");
  if ((reinterpret_cast<uintptr_t>(x) & 15) != 0) throw std::runtime_error("fp8_cast_transpose: input must be 16-byte aligned");
  if ((colsum_partial == nullptr) != (colsum == nullptr)) throw std::runtime_error("fp8_cast_transpose: column sums need both buffers");
  const dim3 grid(ceil_div(cols, kTile), ceil_div(rows, kTile));
  auto* xb = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* qb = reinterpret_cast<uint8_t*>(q);
  auto* qtb = reinterpret_cast<uint8_t*>(qt);
  if (e5m2) fp8_cast_transpose_kernel<true><<<grid, kCastThreads, 0, s>>>(xb, rows, cols, amax, qb, qtb, colsum_partial, scale_inv);
  else fp8_cast_transpose_kernel<false><<<grid, kCastThreads, 0, s>>>(xb, rows, cols, amax, qb, qtb, colsum_partial, scale_inv);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  if (colsum != nullptr) {
    fp8_colsum_finish_kernel<<<ceil_div(cols, 256), 256, 0, s>>>(colsum_partial, (int)grid.y, cols, colsum);
    B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  }
}

}  // namespace b200
