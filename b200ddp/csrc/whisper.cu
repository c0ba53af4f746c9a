// Whisper's audio side: the log-mel front end and the gathers of the two-convolution stem.
//
// Log-mel (WhisperFeatureExtractor's torch path, 400-point Hann STFT, hop 160, 80 mels): int16 waveforms [B, 480000] ->
// [B, 80, 3000].  All arithmetic is fp32:
//   x_f[n]  = s[160 f - 200 + n] / 32768 * (0.5 - 0.5 cos(2 pi n / 400)), n in [0, 400), indices reflected at both ends
//             without repeating the edge sample (torch.stft(center=True, pad_mode="reflect"))
//   P_f[k]  = |sum_n x_f[n] e^{-2 pi i k n / 400}|^2 for k in [0, 200], twiddles from a table built in fp64 and indexed by
//             (k n) mod 400, so no phase error accumulates
//   L[m, f] = log10(max(sum_k filters[k, m] P_f[k], 1e-10))
//   out     = (max(L, M - 8) + 4) / 4 with M the clip's maximum of L
// The frame kernel writes L (into the fp32 output, or an fp32 scratch for bf16 output) and each CTA's maximum; the finish
// kernel takes every clip's maximum from those partials and applies the clamp.  Every sum runs in a fixed order, nothing
// uses atomics, and nothing is read back to the host.
//
// Stem gathers (bf16, 16-byte vectors):
//   mel_patches    P1[b F + t, j 80 + c] = features[b, c, t + j - 1] (zero outside [0, F))
//   frame_patches  P2[b S + l, j d + e] = h1[b F + 2 l + j - 1, e] for l < F / 2 (zero at 2 l + j - 1 = -1); zero rows l >= F / 2
//   its backward   dh1[b F + s, e] = sum over the taps j = 0, 1, 2 (in that order) with 2 l + j - 1 = s and l < F / 2 of
//                  dP2[b S + l, j d + e], in fp32 with one bf16 rounding; the padding rows of dP2 are never read
#include "ops.h"

namespace b200 {
namespace {

constexpr int kSamples = 480000, kFrames = 3000, kNfft = 400, kHop = 160, kBins = 201, kMels = 80;
constexpr int kFrameTile = 16;                           // frames per CTA of the frame kernel
constexpr int kFrameThreads = 224;                       // one thread per frequency bin (201 of 224 busy in the DFT)
constexpr int kFrameCtas = (kFrames + kFrameTile - 1) / kFrameTile;
constexpr int kFinishThreads = 256;

__device__ __forceinline__ int reflect(int i) { return i < 0 ? -i : (i >= kSamples ? 2 * (kSamples - 1) - i : i); }

// CTA (frame tile blockIdx.x, clip blockIdx.y): L[b, m, f] for the tile's frames and the tile's maximum of L
__global__ void __launch_bounds__(kFrameThreads) log_mel_frames_kernel(const short* __restrict__ wave, const float* __restrict__ filters,
                                                                       float* __restrict__ logmel, float* __restrict__ part_max) {
  __shared__ float2 tw[kNfft];                                           // (cos, sin)(2 pi m / 400)
  __shared__ __align__(16) float xs[kNfft * kFrameTile];                 // windowed frames [n][frame]; later the powers [frame][bin]
  __shared__ float red[kFrameThreads / 32];
  const int b = blockIdx.y, f0 = blockIdx.x * kFrameTile;
  for (int m = threadIdx.x; m < kNfft; m += blockDim.x) {
    const double a = 2.0 * m / kNfft;
    tw[m] = make_float2((float)cospi(a), (float)sinpi(a));
  }
  __syncthreads();
  const short* w = wave + (size_t)b * kSamples;
  for (int i = threadIdx.x; i < kNfft * kFrameTile; i += blockDim.x) {
    const int n = i / kFrameTile, fr = i % kFrameTile;
    const float hann = 0.5f - 0.5f * tw[n].x;
    xs[i] = (float)w[reflect((f0 + fr) * kHop - kNfft / 2 + n)] * (1.f / 32768.f) * hann;
  }
  __syncthreads();

  const int k = threadIdx.x;
  float re[kFrameTile], im[kFrameTile];
#pragma unroll
  for (int fr = 0; fr < kFrameTile; ++fr) re[fr] = im[fr] = 0.f;
  if (k < kBins) {
    int idx = 0;                                                         // (k n) mod 400
#pragma unroll 2
    for (int n = 0; n < kNfft; ++n) {
      const float2 t = tw[idx];
      const float4* xv = reinterpret_cast<const float4*>(xs + n * kFrameTile);
#pragma unroll
      for (int q = 0; q < kFrameTile / 4; ++q) {
        const float4 v = xv[q];
        re[4 * q + 0] = fmaf(v.x, t.x, re[4 * q + 0]); im[4 * q + 0] = fmaf(v.x, t.y, im[4 * q + 0]);
        re[4 * q + 1] = fmaf(v.y, t.x, re[4 * q + 1]); im[4 * q + 1] = fmaf(v.y, t.y, im[4 * q + 1]);
        re[4 * q + 2] = fmaf(v.z, t.x, re[4 * q + 2]); im[4 * q + 2] = fmaf(v.z, t.y, im[4 * q + 2]);
        re[4 * q + 3] = fmaf(v.w, t.x, re[4 * q + 3]); im[4 * q + 3] = fmaf(v.w, t.y, im[4 * q + 3]);
      }
      idx += k;
      if (idx >= kNfft) idx -= kNfft;
    }
  }
  __syncthreads();                                                       // the frames are dead: xs holds the powers now
  float* pw = xs;                                                        // [frame][201]
  if (k < kBins) {
#pragma unroll
    for (int fr = 0; fr < kFrameTile; ++fr) pw[fr * kBins + k] = fmaf(re[fr], re[fr], im[fr] * im[fr]);
  }
  __syncthreads();

  // (mel m, frame fr) per item, frames fastest so a warp's stores run along f
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < kMels * kFrameTile; i += blockDim.x) {
    const int m = i / kFrameTile, fr = i % kFrameTile, f = f0 + fr;
    if (f >= kFrames) continue;
    const float* p = pw + fr * kBins;
    float mel = 0.f;
    for (int kk = 0; kk < kBins; ++kk) mel = fmaf(__ldg(filters + kk * kMels + m), p[kk], mel);
    const float L = log10f(fmaxf(mel, 1e-10f));
    logmel[((size_t)b * kMels + m) * kFrames + f] = L;
    mx = fmaxf(mx, L);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
#pragma unroll
    for (int j = 1; j < kFrameThreads / 32; ++j) m = fmaxf(m, red[j]);
    part_max[b * kFrameCtas + blockIdx.x] = m;
  }
}

// CTA (chunk blockIdx.x, clip blockIdx.y): the clip's maximum from the frame kernel's partials, then the clamp and scale
template <typename OutT>
__global__ void __launch_bounds__(kFinishThreads) log_mel_finish_kernel(const float* __restrict__ logmel, const float* __restrict__ part_max,
                                                                        OutT* __restrict__ out) {
  __shared__ float clip_max;
  const int b = blockIdx.y;
  if (threadIdx.x < 32) {
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < kFrameCtas; i += 32) mx = fmaxf(mx, part_max[b * kFrameCtas + i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (threadIdx.x == 0) clip_max = mx;
  }
  __syncthreads();
  const float floor_ = clip_max - 8.f;
  const size_t base = (size_t)b * kMels * kFrames;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kMels * kFrames; i += gridDim.x * blockDim.x)
    out[base + i] = from_f32<OutT>((fmaxf(logmel[base + i], floor_) + 4.f) * 0.25f);
}

// one thread per 8 output columns of one P1 row: P1[b F + t, j 80 + c .. c + 7] = features[b, c .. c + 7, t + j - 1].
// Items run along t fastest, so a warp's loads of one feature row are coalesced.
__global__ void __launch_bounds__(256) mel_patches_kernel(const __nv_bfloat16* __restrict__ feat, int B, int F, __nv_bfloat16* __restrict__ p1) {
  constexpr int kVecs = 3 * kMels / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * F * kVecs) return;
  const int t = (int)(i % F);
  const long long bv = i / F;
  const int v = (int)(bv % kVecs), b = (int)(bv / kVecs);
  const long long row = (long long)b * F + t;
  const int j = v / (kMels / 8), c0 = (v % (kMels / 8)) * 8, s = t + j - 1;
  Bf16x8 out;
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(&out);
  const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
#pragma unroll
  for (int u = 0; u < 8; ++u) o[u] = (s >= 0 && s < F) ? feat[((size_t)b * kMels + c0 + u) * F + s] : zero;
  *reinterpret_cast<Bf16x8*>(p1 + row * (3 * kMels) + v * 8) = out;
}

// one thread per 8 columns of one P2 row
__global__ void __launch_bounds__(256) frame_patches_kernel(const __nv_bfloat16* __restrict__ h1, int B, int F, int S, int d,
                                                            __nv_bfloat16* __restrict__ p2) {
  const int vecs = 3 * d / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * S * vecs) return;
  const int v = (int)(i % vecs);
  const long long row = i / vecs;
  const int l = (int)(row % S), b = (int)(row / S);
  const int j = v * 8 / d, e = v * 8 - j * d, s = 2 * l + j - 1;
  Bf16x8 out;
  if (l < F / 2 && s >= 0) {
    out = *reinterpret_cast<const Bf16x8*>(h1 + ((size_t)b * F + s) * d + e);
  } else {
    out.h[0] = out.h[1] = out.h[2] = out.h[3] = __floats2bfloat162_rn(0.f, 0.f);
  }
  *reinterpret_cast<Bf16x8*>(p2 + row * 3 * d + v * 8) = out;
}

// one thread per 8 columns of one dh1 row
__global__ void __launch_bounds__(256) frame_patches_bwd_kernel(const __nv_bfloat16* __restrict__ dp2, int B, int F, int S, int d,
                                                                __nv_bfloat16* __restrict__ dh1) {
  const int vecs = d / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * F * vecs) return;
  const int e = (int)(i % vecs) * 8;
  const long long row = i / vecs;
  const int s = (int)(row % F), b = (int)(row / F);
  float acc[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) acc[u] = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int l2 = s + 1 - j;                                            // 2 l
    if (l2 < 0 || (l2 & 1) || l2 / 2 >= F / 2) continue;
    float g[8];
    load8(dp2 + ((size_t)b * S + l2 / 2) * 3 * d + j * d + e, g);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] += g[u];
  }
  store8(dh1 + row * d + e, acc);
}

}  // namespace

int log_mel_partials() { return kFrameCtas; }

void launch_log_mel(const void* wave, const float* filters, int B, bool bf16_out, float* logmel, float* part_max, void* out, cudaStream_t s) {
  log_mel_frames_kernel<<<dim3(kFrameCtas, B), kFrameThreads, 0, s>>>((const short*)wave, filters, logmel, part_max);
  B200_CUDA_CHECK(cudaGetLastError());
  const dim3 grid(ceil_div(kMels * kFrames, kFinishThreads * 8), B);
  if (bf16_out)
    log_mel_finish_kernel<__nv_bfloat16><<<grid, kFinishThreads, 0, s>>>(logmel, part_max, (__nv_bfloat16*)out);
  else
    log_mel_finish_kernel<float><<<grid, kFinishThreads, 0, s>>>(logmel, part_max, (float*)out);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

void launch_mel_patches(const void* features, int B, int F, void* p1, cudaStream_t s) {
  const long long n = (long long)B * F * (3 * kMels / 8);
  mel_patches_kernel<<<ceil_div(n, 256), 256, 0, s>>>((const __nv_bfloat16*)features, B, F, (__nv_bfloat16*)p1);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_frame_patches(const void* h1, int B, int F, int S, int d, void* p2, cudaStream_t s) {
  const long long n = (long long)B * S * (3 * d / 8);
  frame_patches_kernel<<<ceil_div(n, 256), 256, 0, s>>>((const __nv_bfloat16*)h1, B, F, S, d, (__nv_bfloat16*)p2);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_frame_patches_bwd(const void* dp2, int B, int F, int S, int d, void* dh1, cudaStream_t s) {
  const long long n = (long long)B * F * (d / 8);
  frame_patches_bwd_kernel<<<ceil_div(n, 256), 256, 0, s>>>((const __nv_bfloat16*)dp2, B, F, S, d, (__nv_bfloat16*)dh1);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
