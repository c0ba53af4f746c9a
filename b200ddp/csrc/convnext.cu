// ConvNeXt's depthwise 7x7 convolution (stride 1, padding 3) on NHWC bf16 activations x [B, H, W, C], C % 8 == 0, with
// the weight read as [C, 49] (the memory of a contiguous or channels_last [C, 1, 7, 7]).  All sums are fp32 in a fixed
// order, with one bf16 rounding at the end; nothing uses atomics, so every result is bitwise repeatable.
//   forward    y[n,h,w,c] = b[c] + sum_{i,j} x[n, h+i-3, w+j-3, c] W[c,i,j], taps in (i, j) raster order
//   data grad  the forward on dy with the kernel flipped (W[c, 6-i, 6-j]) and no bias
//   wgrad      dW[c,i,j] = sum_{n,h,w} dy[n,h,w,c] x[n, h+i-3, w+j-3, c] and db[c] = sum dy: each CTA writes the fp32 sums of
//              its (image, spatial tile, channel chunk) to its own partial slot, and a finish kernel adds the slots in order
// Each CTA stages a zero-filled halo tile of 32 channels in shared memory with 16-byte loads, so positions outside the
// image count as zero, and the output gradient is read at real pixels only.
#include <algorithm>

#include "ops.h"

namespace b200 {
namespace {

constexpr int kK = 7, kTaps = 49, kPad = 3;
constexpr int kCC = 32;                 // channels per CTA
constexpr int kCV = kCC / 8;            // 16-byte vectors per staged pixel
constexpr int kStrip = 4;               // forward: outputs along W per thread
constexpr int kSlotSums = kTaps + 1;    // wgrad partial slot: 49 taps and the bias, each [C]
constexpr int kWgradThreads = 2 * (kCC / 2) * kK;   // two row groups x 16 channel pairs x 7 tap rows

// An odd pixel pitch puts neighbouring tile rows 64 bytes apart modulo 128, so the 8 lanes of a 16-byte shared load
// (4 channel vectors of two rows) hit disjoint banks.
__host__ __device__ constexpr int tile_pitch(int cols) { return cols | 1; }

// tile[r][q][0..31] = src[n, h_org + r, w_org + q, c0..c0+31] for r < rows, q < cols; zero outside the image and past C
__device__ __forceinline__ void stage_tile(const __nv_bfloat16* __restrict__ src, Bf16x8* tile, int n, int H, int W, int C, int h_org,
                                           int w_org, int c0, int rows, int cols, int pitch) {
  const int items = rows * cols * kCV;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int v = i % kCV, p = i / kCV, r = p / cols, q = p % cols;
    const int h = h_org + r, w = w_org + q, c = c0 + v * 8;
    Bf16x8 val;
    if (h >= 0 && h < H && w >= 0 && w < W && c < C)
      val = *reinterpret_cast<const Bf16x8*>(src + (((size_t)n * H + h) * W + w) * C + c);
    else
      val.h[0] = val.h[1] = val.h[2] = val.h[3] = __floats2bfloat162_rn(0.f, 0.f);
    tile[(r * pitch + q) * kCV + v] = val;
  }
}

// CTA (spatial tile blockIdx.x, channel chunk blockIdx.y, image blockIdx.z) of TH x TW outputs; thread = (channel vector,
// tile row, strip of 4 outputs along W) with the channel vector fastest, then the row.  Each thread slides its strip's
// window along the 10 staged pixels of every kernel row.
template <bool kFlip>
__global__ void __launch_bounds__(256) dwconv_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                     const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int H, int W,
                                                     int C, int TH, int TW, int tiles_w) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* ws = reinterpret_cast<float*>(smem);                          // [49][32] fp32 taps
  Bf16x8* tile = reinterpret_cast<Bf16x8*>(ws + kTaps * kCC);          // [TH + 6][pitch][4]
  const int n = blockIdx.z, c0 = blockIdx.y * kCC;
  const int h0 = (blockIdx.x / tiles_w) * TH, w0 = (blockIdx.x % tiles_w) * TW;
  const int pitch = tile_pitch(TW + 2 * kPad);
  for (int i = threadIdx.x; i < kTaps * kCC; i += blockDim.x) {
    const int t = i / kCC, c = c0 + i % kCC;
    ws[i] = c < C ? __bfloat162float(w[(size_t)c * kTaps + (kFlip ? kTaps - 1 - t : t)]) : 0.f;
  }
  stage_tile(x, tile, n, H, W, C, h0 - kPad, w0 - kPad, c0, TH + 2 * kPad, TW + 2 * kPad, pitch);
  __syncthreads();

  const int v = threadIdx.x % kCV, r = (threadIdx.x / kCV) % TH, sx = threadIdx.x / (kCV * TH);
  const int h = h0 + r, wb = w0 + sx * kStrip, c = c0 + v * 8;
  if (h >= H || wb >= W || c >= C) return;
  float acc[kStrip][8];
#pragma unroll
  for (int s = 0; s < kStrip; ++s)
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[s][u] = 0.f;
#pragma unroll 1
  for (int i = 0; i < kK; ++i) {
    float wr[kK][8];
#pragma unroll
    for (int j = 0; j < kK; ++j) {
      const float4* p = reinterpret_cast<const float4*>(ws + (i * kK + j) * kCC + v * 8);
      const float4 a = p[0], b = p[1];
      wr[j][0] = a.x; wr[j][1] = a.y; wr[j][2] = a.z; wr[j][3] = a.w; wr[j][4] = b.x; wr[j][5] = b.y; wr[j][6] = b.z; wr[j][7] = b.w;
    }
    const Bf16x8* row = tile + ((r + i) * pitch + sx * kStrip) * kCV + v;
#pragma unroll
    for (int p = 0; p < kStrip + kK - 1; ++p) {
      float xv[8];
      unpack8(row[p * kCV], xv);
#pragma unroll
      for (int s = 0; s < kStrip; ++s) {
        const int j = p - s;                                           // output s meets this pixel at tap (i, j)
        if (j >= 0 && j < kK) {
#pragma unroll
          for (int u = 0; u < 8; ++u) acc[s][u] = fmaf(xv[u], wr[j][u], acc[s][u]);
        }
      }
    }
  }
  float b[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) b[u] = bias ? __bfloat162float(bias[c + u]) : 0.f;
#pragma unroll
  for (int s = 0; s < kStrip; ++s) {
    if (wb + s >= W) break;
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[s][u] += b[u];
    store8(y + (((size_t)n * H + h) * W + wb + s) * C + c, acc[s]);
  }
}

// CTA (spatial tile blockIdx.x, channel chunk blockIdx.y, image blockIdx.z) of TH x TW output pixels.  Thread = (channel
// pair, tap row i, row group g): it walks the pixels of its half of the tile's rows in raster order, sliding a 7-pixel
// window of x along W in registers, and keeps the 14 sums dW[c..c+1, i, 0..6] (and, for i = 0, db[c..c+1]).  Group 1
// hands its sums to group 0 through shared memory, which adds them after its own and writes the CTA's partial slot.
__global__ void __launch_bounds__(kWgradThreads) dwconv_wgrad_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                                     float* __restrict__ part, int H, int W, int C, int TH, int TW, int tiles_w) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int xpitch = tile_pitch(TW + 2 * kPad);
  Bf16x8* xt = reinterpret_cast<Bf16x8*>(smem);                          // [TH + 6][xpitch][4]
  Bf16x8* dt = xt + (TH + 2 * kPad) * xpitch * kCV;                     // [TH][TW][4]
  const int n = blockIdx.z, c0 = blockIdx.y * kCC;
  const int h0 = (blockIdx.x / tiles_w) * TH, w0 = (blockIdx.x % tiles_w) * TW;
  stage_tile(x, xt, n, H, W, C, h0 - kPad, w0 - kPad, c0, TH + 2 * kPad, TW + 2 * kPad, xpitch);
  stage_tile(dy, dt, n, H, W, C, h0, w0, c0, TH, TW, TW);
  __syncthreads();

  const int cp = threadIdx.x % (kCC / 2), i = (threadIdx.x / (kCC / 2)) % kK, g = threadIdx.x / (kCC / 2 * kK);
  const int half = (TH + 1) / 2, r_end = min(min(TH, H - h0), (g + 1) * half), cols = min(TW, W - w0);
  const __nv_bfloat162* xs = reinterpret_cast<const __nv_bfloat162*>(xt) + cp;
  const __nv_bfloat162* ds = reinterpret_cast<const __nv_bfloat162*>(dt) + cp;
  constexpr int kPix = kCC / 2;                                          // bf16 pairs per staged pixel
  float2 acc[kK], db = make_float2(0.f, 0.f);
#pragma unroll
  for (int j = 0; j < kK; ++j) acc[j] = make_float2(0.f, 0.f);
  for (int r = g * half; r < r_end; ++r) {
    const __nv_bfloat162* xrow = xs + (r + i) * xpitch * kPix;
    const __nv_bfloat162* drow = ds + r * TW * kPix;
    float2 win[kK];                                                      // win[(q + j) % 7] = x at column q + j
#pragma unroll
    for (int j = 0; j < kK - 1; ++j) win[j] = __bfloat1622float2(xrow[j * kPix]);
    for (int q0 = 0; q0 < cols; q0 += kK) {
#pragma unroll
      for (int k = 0; k < kK; ++k) {
        const int q = q0 + k;
        if (q >= cols) break;
        win[(k + kK - 1) % kK] = __bfloat1622float2(xrow[(q + kK - 1) * kPix]);
        const float2 d = __bfloat1622float2(drow[q * kPix]);
        db.x += d.x; db.y += d.y;
#pragma unroll
        for (int j = 0; j < kK; ++j) {
          acc[j].x = fmaf(d.x, win[(k + j) % kK].x, acc[j].x);
          acc[j].y = fmaf(d.y, win[(k + j) % kK].y, acc[j].y);
        }
      }
    }
  }
  __syncthreads();                                                       // the tiles are dead: reuse them for group 1's sums
  float2* hand = reinterpret_cast<float2*>(smem) + (threadIdx.x % (kCC / 2 * kK)) * (kK + 1);
  if (g == 1) {
#pragma unroll
    for (int j = 0; j < kK; ++j) hand[j] = acc[j];
    hand[kK] = db;
  }
  __syncthreads();
  const int c = c0 + 2 * cp;
  if (g == 1 || c >= C) return;
#pragma unroll
  for (int j = 0; j < kK; ++j) { const float2 o = hand[j]; acc[j].x += o.x; acc[j].y += o.y; }
  db.x += hand[kK].x; db.y += hand[kK].y;
  const size_t slot = ((size_t)n * gridDim.x + blockIdx.x) * kSlotSums;
#pragma unroll
  for (int j = 0; j < kK; ++j) *reinterpret_cast<float2*>(part + (slot + i * kK + j) * C + c) = acc[j];
  if (i == 0) *reinterpret_cast<float2*>(part + (slot + kTaps) * C + c) = db;
}

// (tap or bias t, channel c) per item: the sum of the slots in order, rounded once to bf16
__global__ void __launch_bounds__(256) dwconv_wgrad_finish_kernel(const float* __restrict__ part, int slots, int C, __nv_bfloat16* __restrict__ dw,
                                                                  __nv_bfloat16* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kSlotSums * C) return;
  const int t = i / C, c = i % C;
  const float* p = part + (size_t)t * C + c;
  float sum = 0.f;
#pragma unroll 8
  for (int s = 0; s < slots; ++s) sum += p[(size_t)s * kSlotSums * C];
  if (t < kTaps) dw[(size_t)c * kTaps + t] = __float2bfloat16_rn(sum);
  else db[c] = __float2bfloat16_rn(sum);
}

struct FwdTiles { int th, tw, tiles_w, tiles, threads, smem; };

FwdTiles fwd_tiles(int H, int W) {
  FwdTiles t;
  t.tw = std::min(16, (W + kStrip - 1) / kStrip * kStrip);
  t.th = std::min(H, 16);
  t.tiles_w = ceil_div(W, t.tw);
  t.tiles = ceil_div(H, t.th) * t.tiles_w;
  t.threads = t.th * (t.tw / kStrip) * kCV;
  t.smem = kTaps * kCC * 4 + (t.th + 2 * kPad) * tile_pitch(t.tw + 2 * kPad) * kCC * 2;
  return t;
}

struct WgradTiles { int th, tw, tiles_w, tiles, smem; };

// the staged x halo and dy tile; at least the hand-off of group 1's sums
constexpr int wgrad_smem(int th, int tw) {
  return std::max(((th + 2 * kPad) * tile_pitch(tw + 2 * kPad) + th * tw) * kCC * 2, kWgradThreads / 2 * (kK + 1) * 8);
}
// the largest tiles wgrad_tiles picks: 8 x 56 and 16 x 28
constexpr int kWgradSmemMax = std::max(wgrad_smem(8, 56), wgrad_smem(16, 28));

WgradTiles wgrad_tiles(int H, int W) {
  WgradTiles t;
  t.tw = std::min(W, 56);
  t.th = std::min(H, t.tw <= 28 ? 16 : 8);
  t.tiles_w = ceil_div(W, t.tw);
  t.tiles = ceil_div(H, t.th) * t.tiles_w;
  t.smem = wgrad_smem(t.th, t.tw);
  return t;
}

template <bool kFlip>
void launch_dwconv(const void* x, const void* w, const void* bias, int B, int H, int W, int C, void* y, cudaStream_t s) {
  const FwdTiles t = fwd_tiles(H, W);
  const dim3 grid(t.tiles, ceil_div(C, kCC), B);
  dwconv_kernel<kFlip><<<grid, t.threads, t.smem, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)bias,
                                                       (__nv_bfloat16*)y, H, W, C, t.th, t.tw, t.tiles_w);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace

int dwconv_wgrad_slots(int B, int H, int W) { return B * wgrad_tiles(H, W).tiles; }

void launch_dwconv_fwd(const void* x, const void* w, const void* bias, int B, int H, int W, int C, void* y, cudaStream_t s) {
  launch_dwconv<false>(x, w, bias, B, H, W, C, y, s);
}

void launch_dwconv_dgrad(const void* dy, const void* w, int B, int H, int W, int C, void* dx, cudaStream_t s) {
  launch_dwconv<true>(dy, w, nullptr, B, H, W, C, dx, s);
}

void launch_dwconv_wgrad(const void* dy, const void* x, int B, int H, int W, int C, float* part, void* dw, void* db, cudaStream_t s) {
  static std::atomic<unsigned long long> smem_set{0};
  ensure_max_dynamic_smem(dwconv_wgrad_kernel, kWgradSmemMax, smem_set);
  const WgradTiles t = wgrad_tiles(H, W);
  const dim3 grid(t.tiles, ceil_div(C, kCC), B);
  dwconv_wgrad_kernel<<<grid, kWgradThreads, t.smem, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, part, H, W, C, t.th, t.tw,
                                                          t.tiles_w);
  B200_CUDA_CHECK(cudaGetLastError());
  dwconv_wgrad_finish_kernel<<<ceil_div(kSlotSums * C, 256), 256, 0, s>>>(part, B * t.tiles, C, (__nv_bfloat16*)dw, (__nv_bfloat16*)db);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

}  // namespace b200
