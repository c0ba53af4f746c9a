// Rotary position embedding (RoPE) on the fused qkv projection, Hugging Face convention (rotate_half, non-interleaved):
// within each head of width d (64 or 128), element i pairs with i + d/2 (i < d/2) and, at position p with angle
// a = p * theta^(-2i/d),
//   forward:  out_i = x_i cos a - x_{i+d/2} sin a,   out_{i+d/2} = x_{i+d/2} cos a + x_i sin a
//   backward: the transpose rotation (sin a -> -sin a).
// qkv bf16 [rows, (H + 2*Hkv)*d] (query | key | value column blocks): the H + Hkv query and key heads are rotated, the
// value heads are copied, so the op is out of place.  Positions are int32 [rows] (restarting in every packed document),
// clamped to [0, max_pos).  cos / sin come from an fp32 table [max_pos, 2, d/2] (cos a_i, then sin a_i) built on the host
// in fp64: the kernel evaluates no trigonometric function, so its error does not grow with the position.
#include "ops.h"

#include <cmath>

namespace b200 {
namespace {

constexpr int kRopeThreads = 256;

// One thread per (row, head, 8 pairs): columns [8 c, 8 c + 8) and [8 c + kHalf, 8 c + kHalf + 8) of the head, c < kHalf / 8
// (head dim 2 kHalf).
// kScaleQ: the first q_heads heads (the query heads) are also multiplied by q_scale, a power of two (exact in bf16), in
// both directions.
template <bool kBwd, int kHalf, bool kScaleQ = false>
__global__ void __launch_bounds__(kRopeThreads) rotary_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ pos,
                                                              const float* __restrict__ table, int max_pos, size_t rows, int rot_heads,
                                                              int heads, __nv_bfloat16* __restrict__ y, int q_heads = 0,
                                                              float q_scale = 1.f) {
  constexpr int kParts = kHalf / 8, kShift = kParts == 4 ? 2 : 3;
  static_assert(kParts == 1 << kShift, "kHalf is 32 or 64");
  const size_t n = rows * (size_t)heads * kParts;
  const int pitch = heads * 2 * kHalf;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    const size_t r = t / ((size_t)heads * kParts);
    const int rest = (int)(t - r * heads * kParts), hh = rest >> kShift, c = (rest & (kParts - 1)) * 8;
    const size_t off = r * pitch + hh * 2 * kHalf + c;
    const Bf16x8 lo_raw = *reinterpret_cast<const Bf16x8*>(x + off);
    const Bf16x8 hi_raw = *reinterpret_cast<const Bf16x8*>(x + off + kHalf);
    if (hh >= rot_heads) {                                      // value head: copied
      *reinterpret_cast<Bf16x8*>(y + off) = lo_raw;
      *reinterpret_cast<Bf16x8*>(y + off + kHalf) = hi_raw;
      continue;
    }
    const int p = min(max(__ldg(pos + r), 0), max_pos - 1);
    const float4* cs = reinterpret_cast<const float4*>(table + (size_t)p * 2 * kHalf + c);
    const float4 c0 = __ldg(cs), c1 = __ldg(cs + 1), s0 = __ldg(cs + kHalf / 4), s1 = __ldg(cs + kHalf / 4 + 1);
    const float cv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    float lo[8], hi[8], olo[8], ohi[8];
    unpack8(lo_raw, lo);
    unpack8(hi_raw, hi);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float sn = kBwd ? -sv[i] : sv[i];
      olo[i] = lo[i] * cv[i] - hi[i] * sn;
      ohi[i] = hi[i] * cv[i] + lo[i] * sn;
    }
    if constexpr (kScaleQ) {
      if (hh < q_heads) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { olo[i] *= q_scale; ohi[i] *= q_scale; }
      }
    }
    *reinterpret_cast<Bf16x8*>(y + off) = pack8(olo);
    *reinterpret_cast<Bf16x8*>(y + off + kHalf) = pack8(ohi);
  }
}

template <int kHalf>
void rotary_launch(const __nv_bfloat16* x, const int* pos, const float* table, int max_pos, size_t rows, int heads, int kv_heads,
                   __nv_bfloat16* y, bool backward, float q_scale, cudaStream_t s) {
  const int all = heads + 2 * kv_heads;
  size_t b = (rows * all * (kHalf / 8) + kRopeThreads - 1) / kRopeThreads;
  if (b < 1) b = 1;
  if (b > (size_t)16 * kNumSMs) b = (size_t)16 * kNumSMs;
  if (q_scale != 1.f) {
    if (backward)
      rotary_kernel<true, kHalf, true><<<(int)b, kRopeThreads, 0, s>>>(x, pos, table, max_pos, rows, heads + kv_heads, all, y, heads, q_scale);
    else
      rotary_kernel<false, kHalf, true><<<(int)b, kRopeThreads, 0, s>>>(x, pos, table, max_pos, rows, heads + kv_heads, all, y, heads, q_scale);
  } else if (backward)
    rotary_kernel<true, kHalf><<<(int)b, kRopeThreads, 0, s>>>(x, pos, table, max_pos, rows, heads + kv_heads, all, y);
  else
    rotary_kernel<false, kHalf><<<(int)b, kRopeThreads, 0, s>>>(x, pos, table, max_pos, rows, heads + kv_heads, all, y);
}

// ---- per-head q / k RMSNorm fused with rotary (Qwen3), head dim 128 --------------------------------------------------
// Forward, per query head (weight wq) and key head (wk) of a row: y = rope(x * rstd * w), rstd = rsqrt(mean(x^2) + eps)
// over the head's 128 elements, all in fp32 with one rounding to bf16; value heads are copied; rstd fp32 [rows, H + Hkv].
// Backward: g = rope^-1(dy), xn = x * rstd, dx = rstd * (g w - xn mean(g w xn)), dw = sum over rows and heads of g xn.
// rotary_kernel's thread mapping (one thread per (row, head, 8 pairs)): the 8 threads of a head are 8 adjacent,
// 8-aligned lanes, so a head's sums are three xor shuffles among them.
constexpr int kQkHalf = 64, kQkParts = kQkHalf / 8;

__device__ __forceinline__ float qk_head_sum(float v) {
  const unsigned mask = 0xffu << (threadIdx.x & 24);
  v += __shfl_xor_sync(mask, v, 1);
  v += __shfl_xor_sync(mask, v, 2);
  v += __shfl_xor_sync(mask, v, 4);
  return v;
}

// cos / sin of the 8 pairs [c, c + 8) of the head at row position p
__device__ __forceinline__ void qk_rope_table(const float* __restrict__ table, int p, int c, float* cv, float* sv) {
  const float4* cs = reinterpret_cast<const float4*>(table + (size_t)p * 2 * kQkHalf + c);
  const float4 c0 = __ldg(cs), c1 = __ldg(cs + 1), s0 = __ldg(cs + kQkHalf / 4), s1 = __ldg(cs + kQkHalf / 4 + 1);
  cv[0] = c0.x; cv[1] = c0.y; cv[2] = c0.z; cv[3] = c0.w; cv[4] = c1.x; cv[5] = c1.y; cv[6] = c1.z; cv[7] = c1.w;
  sv[0] = s0.x; sv[1] = s0.y; sv[2] = s0.z; sv[3] = s0.w; sv[4] = s1.x; sv[5] = s1.y; sv[6] = s1.z; sv[7] = s1.w;
}

__global__ void __launch_bounds__(kRopeThreads) qk_norm_rotary_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ wq,
                                                                          const __nv_bfloat16* __restrict__ wk, const int* __restrict__ pos,
                                                                          const float* __restrict__ table, int max_pos, size_t rows, int heads,
                                                                          int kv_heads, float eps, __nv_bfloat16* __restrict__ y,
                                                                          float* __restrict__ rstd) {
  const int all = heads + 2 * kv_heads, normed = heads + kv_heads;
  const size_t n = rows * (size_t)all * kQkParts;
  const int pitch = all * 2 * kQkHalf;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    const size_t r = t / ((size_t)all * kQkParts);
    const int rest = (int)(t - r * all * kQkParts), hh = rest / kQkParts, c = (rest % kQkParts) * 8;
    const size_t off = r * pitch + hh * 2 * kQkHalf + c;
    const Bf16x8 lo_raw = *reinterpret_cast<const Bf16x8*>(x + off);
    const Bf16x8 hi_raw = *reinterpret_cast<const Bf16x8*>(x + off + kQkHalf);
    if (hh >= normed) {                                         // value head: copied
      *reinterpret_cast<Bf16x8*>(y + off) = lo_raw;
      *reinterpret_cast<Bf16x8*>(y + off + kQkHalf) = hi_raw;
      continue;
    }
    float lo[8], hi[8], wl[8], wh[8], cv[8], sv[8], olo[8], ohi[8];
    unpack8(lo_raw, lo);
    unpack8(hi_raw, hi);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) q = fmaf(hi[i], hi[i], fmaf(lo[i], lo[i], q));
    const float rs = rsqrtf(qk_head_sum(q) * (1.f / (2 * kQkHalf)) + eps);
    const __nv_bfloat16* w = hh < heads ? wq : wk;
    unpack8(*reinterpret_cast<const Bf16x8*>(w + c), wl);
    unpack8(*reinterpret_cast<const Bf16x8*>(w + c + kQkHalf), wh);
    qk_rope_table(table, min(max(__ldg(pos + r), 0), max_pos - 1), c, cv, sv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a = lo[i] * rs * wl[i], b = hi[i] * rs * wh[i];
      olo[i] = a * cv[i] - b * sv[i];
      ohi[i] = b * cv[i] + a * sv[i];
    }
    *reinterpret_cast<Bf16x8*>(y + off) = pack8(olo);
    *reinterpret_cast<Bf16x8*>(y + off + kQkHalf) = pack8(ohi);
    if (c == 0) rstd[r * normed + hh] = rs;
  }
}

// partial: fp32 [2][gridDim.x][128], this CTA's column sums of g xn over its query heads (0) and key heads (1), each
// summed in a fixed order (per thread over its grid-stride items, then over lanes, then over warps)
__global__ void __launch_bounds__(kRopeThreads, 2) qk_norm_rotary_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                                             const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ wq,
                                                                             const __nv_bfloat16* __restrict__ wk, const int* __restrict__ pos,
                                                                             const float* __restrict__ table, int max_pos, size_t rows,
                                                                             int heads, int kv_heads, __nv_bfloat16* __restrict__ dx,
                                                                             float* __restrict__ partial) {
  __shared__ float red[kRopeThreads / 32][2][2 * kQkHalf];
  const int all = heads + 2 * kv_heads, normed = heads + kv_heads;
  const size_t n = rows * (size_t)all * kQkParts;
  const int pitch = all * 2 * kQkHalf;
  const int c = (threadIdx.x % kQkParts) * 8;                   // fixed per thread: the grid stride is a multiple of kQkParts
  float aq[16], ak[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { aq[i] = 0.f; ak[i] = 0.f; }
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x) {
    const size_t r = t / ((size_t)all * kQkParts);
    const int hh = (int)(t - r * all * kQkParts) / kQkParts;
    const size_t off = r * pitch + hh * 2 * kQkHalf + c;
    const Bf16x8 dlo_raw = *reinterpret_cast<const Bf16x8*>(dy + off);
    const Bf16x8 dhi_raw = *reinterpret_cast<const Bf16x8*>(dy + off + kQkHalf);
    if (hh >= normed) {                                         // value head: the gradient passes through
      *reinterpret_cast<Bf16x8*>(dx + off) = dlo_raw;
      *reinterpret_cast<Bf16x8*>(dx + off + kQkHalf) = dhi_raw;
      continue;
    }
    float dlo[8], dhi[8], xlo[8], xhi[8], wl[8], wh[8], cv[8], sv[8];
    unpack8(dlo_raw, dlo);
    unpack8(dhi_raw, dhi);
    unpack8(*reinterpret_cast<const Bf16x8*>(x + off), xlo);
    unpack8(*reinterpret_cast<const Bf16x8*>(x + off + kQkHalf), xhi);
    const bool is_q = hh < heads;
    const __nv_bfloat16* w = is_q ? wq : wk;
    unpack8(*reinterpret_cast<const Bf16x8*>(w + c), wl);
    unpack8(*reinterpret_cast<const Bf16x8*>(w + c + kQkHalf), wh);
    qk_rope_table(table, min(max(__ldg(pos + r), 0), max_pos - 1), c, cv, sv);
    const float rs = __ldg(rstd + r * normed + hh);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float glo = dlo[i] * cv[i] + dhi[i] * sv[i], ghi = dhi[i] * cv[i] - dlo[i] * sv[i];   // rope^-1(dy)
      xlo[i] *= rs;
      xhi[i] *= rs;
      dlo[i] = glo;                                             // dlo / dhi hold g from here on
      dhi[i] = ghi;
      s = fmaf(glo * wl[i], xlo[i], s);
      s = fmaf(ghi * wh[i], xhi[i], s);
    }
    s = qk_head_sum(s) * (1.f / (2 * kQkHalf));
    float olo[8], ohi[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      olo[i] = rs * (dlo[i] * wl[i] - xlo[i] * s);
      ohi[i] = rs * (dhi[i] * wh[i] - xhi[i] * s);
    }
    *reinterpret_cast<Bf16x8*>(dx + off) = pack8(olo);
    *reinterpret_cast<Bf16x8*>(dx + off + kQkHalf) = pack8(ohi);
    if (is_q) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { aq[i] = fmaf(dlo[i], xlo[i], aq[i]); aq[8 + i] = fmaf(dhi[i], xhi[i], aq[8 + i]); }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) { ak[i] = fmaf(dlo[i], xlo[i], ak[i]); ak[8 + i] = fmaf(dhi[i], xhi[i], ak[8 + i]); }
    }
  }
  // lanes l, l ^ 8, l ^ 16, l ^ 24 own the same columns
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    aq[i] += __shfl_xor_sync(0xffffffffu, aq[i], 8);
    ak[i] += __shfl_xor_sync(0xffffffffu, ak[i], 8);
    aq[i] += __shfl_xor_sync(0xffffffffu, aq[i], 16);
    ak[i] += __shfl_xor_sync(0xffffffffu, ak[i], 16);
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) < kQkParts) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      red[warp][0][c + i] = aq[i];
      red[warp][0][kQkHalf + c + i] = aq[8 + i];
      red[warp][1][c + i] = ak[i];
      red[warp][1][kQkHalf + c + i] = ak[8 + i];
    }
  }
  __syncthreads();
  const int which = threadIdx.x / (2 * kQkHalf), col = threadIdx.x % (2 * kQkHalf);   // kRopeThreads == 2 * 128
  float sum = 0.f;
#pragma unroll
  for (int w = 0; w < kRopeThreads / 32; ++w) sum += red[w][which][col];
  partial[((size_t)which * gridDim.x + blockIdx.x) * (2 * kQkHalf) + col] = sum;
}

void qk_norm_rotary_check(const void* a, const void* b, const void* wq, const void* wk, const float* table, int max_pos, int heads,
                          int kv_heads, int head_dim) {
  if (max_pos < 1 || heads < 1 || kv_heads < 1 || head_dim != 2 * kQkHalf ||
      ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(wq) |
        reinterpret_cast<uintptr_t>(wk) | reinterpret_cast<uintptr_t>(table)) & 15u) != 0)
    throw std::runtime_error("qk_norm_rotary: needs heads, kv_heads, max_pos >= 1, head dim 128, 16-byte aligned qkv / out, "
                             "weights and table");
}

}  // namespace

int qk_norm_rotary_partials(size_t rows) {
  const size_t b = (rows + 7) / 8;
  return b < 1 ? 1 : b > (size_t)2 * kNumSMs ? 2 * kNumSMs : (int)b;
}

void launch_qk_norm_rotary_fwd(const void* x, const void* wq, const void* wk, const int* pos, const float* table, int max_pos, size_t rows,
                               int heads, int kv_heads, int head_dim, float eps, void* y, float* rstd, cudaStream_t s) {
  qk_norm_rotary_check(x, y, wq, wk, table, max_pos, heads, kv_heads, head_dim);
  if (!(eps > 0.f)) throw std::runtime_error("qk_norm_rotary: eps must be > 0, got " + std::to_string(eps));
  size_t b = (rows * (heads + 2 * kv_heads) * kQkParts + kRopeThreads - 1) / kRopeThreads;
  if (b < 1) b = 1;
  if (b > (size_t)16 * kNumSMs) b = (size_t)16 * kNumSMs;
  qk_norm_rotary_fwd_kernel<<<(int)b, kRopeThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(wq),
                                                           reinterpret_cast<const __nv_bfloat16*>(wk), pos, table, max_pos, rows, heads,
                                                           kv_heads, eps, reinterpret_cast<__nv_bfloat16*>(y), rstd);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_qk_norm_rotary_bwd(const void* dy, const void* x, const float* rstd, const void* wq, const void* wk, const int* pos,
                               const float* table, int max_pos, size_t rows, int heads, int kv_heads, int head_dim, void* dx,
                               float* partial, void* dwq, void* dwk, cudaStream_t s) {
  qk_norm_rotary_check(dy, dx, wq, wk, table, max_pos, heads, kv_heads, head_dim);
  if ((reinterpret_cast<uintptr_t>(x) & 15u) != 0) throw std::runtime_error("qk_norm_rotary: needs 16-byte aligned qkv");
  const int parts = qk_norm_rotary_partials(rows);
  qk_norm_rotary_bwd_kernel<<<parts, kRopeThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(x),
                                                          rstd, reinterpret_cast<const __nv_bfloat16*>(wq),
                                                          reinterpret_cast<const __nv_bfloat16*>(wk), pos, table, max_pos, rows, heads,
                                                          kv_heads, reinterpret_cast<__nv_bfloat16*>(dx), partial);
  B200_CUDA_CHECK(cudaGetLastError());
  launch_column_sum_pair_bf16(partial, partial + (size_t)parts * 2 * kQkHalf, parts, 2 * kQkHalf, dwq, dwk, s);
  B200_COUNT_LAUNCH(2);
}

void launch_rotary(const void* x, const int* pos, const float* table, int max_pos, size_t rows, int heads, int kv_heads, int head_dim,
                   void* y, bool backward, cudaStream_t s, float q_scale) {
  if (max_pos < 1 || heads < 1 || kv_heads < 1 || (head_dim != 64 && head_dim != 128) ||
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) != 0 || (reinterpret_cast<uintptr_t>(table) & 15u) != 0)
    throw std::runtime_error("rotary: needs heads, kv_heads, max_pos >= 1, head dim 64 or 128, 16-byte aligned qkv / out and table");
  int e2 = 0;
  if (!(q_scale > 0.f) || std::frexp(q_scale, &e2) != 0.5f)
    throw std::runtime_error("rotary: the query scale must be a positive power of two (exact in bf16), got " + std::to_string(q_scale));
  const auto* xi = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* yo = reinterpret_cast<__nv_bfloat16*>(y);
  if (head_dim == 64) rotary_launch<32>(xi, pos, table, max_pos, rows, heads, kv_heads, yo, backward, q_scale, s);
  else rotary_launch<64>(xi, pos, table, max_pos, rows, heads, kv_heads, yo, backward, q_scale, s);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
