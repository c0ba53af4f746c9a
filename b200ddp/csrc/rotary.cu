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

namespace b200 {
namespace {

constexpr int kRopeThreads = 256;

// One thread per (row, head, 8 pairs): columns [8 c, 8 c + 8) and [8 c + kHalf, 8 c + kHalf + 8) of the head, c < kHalf / 8
// (head dim 2 kHalf).
template <bool kBwd, int kHalf>
__global__ void __launch_bounds__(kRopeThreads) rotary_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ pos,
                                                              const float* __restrict__ table, int max_pos, size_t rows, int rot_heads,
                                                              int heads, __nv_bfloat16* __restrict__ y) {
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
    *reinterpret_cast<Bf16x8*>(y + off) = pack8(olo);
    *reinterpret_cast<Bf16x8*>(y + off + kHalf) = pack8(ohi);
  }
}

template <int kHalf>
void rotary_launch(const __nv_bfloat16* x, const int* pos, const float* table, int max_pos, size_t rows, int heads, int kv_heads,
                   __nv_bfloat16* y, bool backward, cudaStream_t s) {
  const int all = heads + 2 * kv_heads;
  size_t b = (rows * all * (kHalf / 8) + kRopeThreads - 1) / kRopeThreads;
  if (b < 1) b = 1;
  if (b > (size_t)16 * kNumSMs) b = (size_t)16 * kNumSMs;
  if (backward)
    rotary_kernel<true, kHalf><<<(int)b, kRopeThreads, 0, s>>>(x, pos, table, max_pos, rows, heads + kv_heads, all, y);
  else
    rotary_kernel<false, kHalf><<<(int)b, kRopeThreads, 0, s>>>(x, pos, table, max_pos, rows, heads + kv_heads, all, y);
}

}  // namespace

void launch_rotary(const void* x, const int* pos, const float* table, int max_pos, size_t rows, int heads, int kv_heads, int head_dim,
                   void* y, bool backward, cudaStream_t s) {
  if (max_pos < 1 || heads < 1 || kv_heads < 1 || (head_dim != 64 && head_dim != 128) ||
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) != 0 || (reinterpret_cast<uintptr_t>(table) & 15u) != 0)
    throw std::runtime_error("rotary: needs heads, kv_heads, max_pos >= 1, head dim 64 or 128, 16-byte aligned qkv / out and table");
  const auto* xi = reinterpret_cast<const __nv_bfloat16*>(x);
  auto* yo = reinterpret_cast<__nv_bfloat16*>(y);
  if (head_dim == 64) rotary_launch<32>(xi, pos, table, max_pos, rows, heads, kv_heads, yo, backward, s);
  else rotary_launch<64>(xi, pos, table, max_pos, rows, heads, kv_heads, yo, backward, s);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
