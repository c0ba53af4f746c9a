// Masked-autoencoder pretraining (He et al., 2021) on bf16 token streams: the batch's images are documents of one stream, as
// in vit.cu, but the encoder sees only each image's `keep` kept patches and the decoder all N of them again.
//
//   shuffle     noise fp32 [B, N] -> ids_keep int32 [B, keep] and ids_restore int32 [B, N]: one CTA per image ranks each
//               patch by counting, rank_i = #{j : n_j < n_i, or n_j == n_i and j < i} (a stable argsort; NaN ranks last)
//   patchify    the kept patches' rows of the patch matrix, image b's kept patch j (ids_keep[b, j]) at stream row
//               b (keep + 1) + 1 + j, in the convolution weight's (c, ky, kx) K order; class and padding rows zero
//   assemble    GEMM output -> encoder tokens: cls + pos[0] at class rows, patch + pos[1 + ids_keep] at patch rows (fp32 add,
//               one bf16 rounding), zero padding rows; its backward passes dy at patch rows to the weight-gradient GEMM and
//               sums d cls over the class rows in image order (pos is a frozen table: no d pos)
//   unshuffle   decoder_embed's output [Te, E] -> decoder stream [Td, E], Td rows of B images of N + 1 rows: the class row,
//               then patch i = the encoder row of rank ids_restore[b, i] if that is below keep, else mask_token; plus pos.
//               Backward: each encoder row gathers its one decoder row's gradient (through ids_keep), and d mask_token is a
//               fixed-order fp32 sum over the masked rows: per-CTA partials and an in-order finish
//   attention   per-image attention at head dim 32 over up to 256 rows (the decoder's 197): one CTA per (image, head) with
//               the image's q / k / v rows of that head in shared memory, m16n8k16 MMAs over 64-key chunks, online fp32
//               softmax.  Backward: key-tile warps form dK and dV, query-tile warps dQ, each recomputing P from lse; plain
//               stores, since every row belongs to one image
//   loss        mean over the masked patches of the per-patch mean of (pred - target)^2, the target read from the bf16
//               image in (ky, kx, c) order and optionally normalised per patch; per-patch losses and an in-order finish
// No atomics, so two runs give bitwise-equal results; nothing is read back to the host.
#include "ops.h"
#include "warp_mma.cuh"

namespace b200 {
namespace {

constexpr int kHd = 32, kPitch = kHd + 8;          // bf16 pitch of a staged row: 80 bytes, conflict-free fragments and ldmatrix
constexpr int kMaxTok = 256, kChunk = 64, kWarps = 8, kAttnThreads = kWarps * 32;
constexpr float kScale = 0.17677669529663687f;    // 32^-0.5
constexpr float kLog2e = 1.4426950408889634f;
constexpr int kMaxGroups = 3;                      // 8-wide groups per lane of a loss row: C p^2 <= 768
constexpr int kFinishThreads = 1024;

int grid_for(size_t items) {
  size_t blocks = (items + 255) / 256;
  if (blocks > (size_t)16 * kNumSMs) blocks = (size_t)16 * kNumSMs;
  return blocks < 1 ? 1 : (int)blocks;
}

// ---- shuffle ----------------------------------------------------------------------------------------------------------
// an unsigned key in the order of the floats: -0 and +0 equal, every NaN above +inf
__device__ __forceinline__ uint32_t order_key(float f) {
  if (f != f) return 0xffffffffu;
  if (f == 0.f) return 0x80000000u;
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(256) mae_shuffle_kernel(const float* __restrict__ noise, int N, int keep, int* __restrict__ ids_keep,
                                                          int* __restrict__ ids_restore) {
  __shared__ uint32_t key[1024];
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < N; i += blockDim.x) key[i] = order_key(noise[(size_t)b * N + i]);
  __syncthreads();
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const uint32_t ki = key[i];
    int r = 0;
    for (int j = 0; j < N; ++j) {
      const uint32_t kj = key[j];
      r += (kj < ki) | ((kj == ki) & (j < i));
    }
    ids_restore[(size_t)b * N + i] = r;
    if (r < keep) ids_keep[(size_t)b * keep + r] = i;
  }
}

// ---- masked patch embedding -------------------------------------------------------------------------------------------
// one thread per 8 consecutive k of one token row: (c, ky, kx..kx+7) with p % 8 == 0, so the 8 pixels lie on one image row
template <bool kChannelsLast>
__global__ void __launch_bounds__(256) mae_patchify_kernel(const __nv_bfloat16* __restrict__ img, const int* __restrict__ ids_keep,
                                                           __nv_bfloat16* __restrict__ out, int B, int C, int H, int W, int p, int keep,
                                                           int T) {
  const int gw = W / p, per = keep + 1, k8 = C * p * p / 8;
  const size_t total = (size_t)T * k8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / k8), k = (int)(i % k8) * 8;
    const int b = t / per, j = t % per;
    Bf16x8 v;
    if (b >= B || j == 0) {
      v.h[0] = v.h[1] = v.h[2] = v.h[3] = __floats2bfloat162_rn(0.f, 0.f);
    } else {
      const int q = ids_keep[(size_t)b * keep + j - 1], c = k / (p * p), r = k % (p * p);
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

__global__ void __launch_bounds__(256) mae_patch_assemble_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ cls,
                                                                 const __nv_bfloat16* __restrict__ pos, const int* __restrict__ ids_keep,
                                                                 __nv_bfloat16* __restrict__ out, int B, int keep, int D, int T) {
  const int d8 = D / 8, per = keep + 1;
  const size_t total = (size_t)T * d8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / d8), d = (int)(i % d8) * 8;
    const int b = t / per, j = t % per;
    float f[8], g[8];
    if (b >= B) {
#pragma unroll
      for (int u = 0; u < 8; ++u) f[u] = 0.f;
    } else {
      const int prow = j == 0 ? 0 : 1 + ids_keep[(size_t)b * keep + j - 1];
      load8(j == 0 ? cls + d : y + (size_t)t * D + d, f);
      load8(pos + (size_t)prow * D + d, g);
#pragma unroll
      for (int u = 0; u < 8; ++u) f[u] += g[u];
    }
    store8(out + (size_t)t * D + d, f);
  }
}

// Items [0, T D/8): 8 columns of one row of dpatch (dy at patch rows, zero at class and padding rows).  Items past that: 8
// columns of d cls, the class rows' dy summed in image order.
__global__ void __launch_bounds__(256) mae_patch_embed_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dpatch,
                                                                  __nv_bfloat16* __restrict__ dcls, int B, int per, int D, int T) {
  const int d8 = D / 8;
  const size_t rows = (size_t)T * d8, total = rows + d8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    if (i >= rows) {
      const int d = (int)(i - rows) * 8;
      float acc[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = 0.f;
#pragma unroll 4
      for (int b = 0; b < B; ++b) {
        float f[8];
        load8(dy + (size_t)b * per * D + d, f);
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] += f[u];
      }
      store8(dcls + d, acc);
      continue;
    }
    const int t = (int)(i / d8), d = (int)(i % d8) * 8;
    const int b = t / per, j = t % per;
    const size_t off = (size_t)t * D + d;
    if (b < B && j > 0) {
      *reinterpret_cast<Bf16x8*>(dpatch + off) = *reinterpret_cast<const Bf16x8*>(dy + off);
    } else {
      float zero[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) zero[u] = 0.f;
      store8(dpatch + off, zero);
    }
  }
}

// ---- unshuffle --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mae_unshuffle_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ mask,
                                                            const __nv_bfloat16* __restrict__ pos, const int* __restrict__ ids_restore,
                                                            __nv_bfloat16* __restrict__ z, int B, int N, int keep, int E, int Td) {
  const int e8 = E / 8, per = keep + 1, dper = N + 1;
  const size_t total = (size_t)Td * e8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / e8), d = (int)(i % e8) * 8;
    const int b = t / dper, j = t % dper;
    float f[8], g[8];
    if (b >= B) {
#pragma unroll
      for (int u = 0; u < 8; ++u) f[u] = 0.f;
    } else {
      const __nv_bfloat16* src = y + (size_t)b * per * E;
      if (j > 0) {
        const int r = ids_restore[(size_t)b * N + j - 1];
        src = r < keep ? src + (size_t)(1 + r) * E : mask;
      }
      load8(src + d, f);
      load8(pos + (size_t)j * E + d, g);
#pragma unroll
      for (int u = 0; u < 8; ++u) f[u] += g[u];
    }
    store8(z + (size_t)t * E + d, f);
  }
}

int mask_chunks(int B) { return B < 2 * kNumSMs ? B : 2 * kNumSMs; }

// CTA c owns images [c B / chunks, (c + 1) B / chunks): it gathers their encoder rows' gradient, and its thread groups add
// the masked decoder rows' gradient in a fixed interleave, combined in group order into part[c]; the last CTA also zeroes
// the encoder's padding rows.
__global__ void __launch_bounds__(256) mae_unshuffle_bwd_kernel(const __nv_bfloat16* __restrict__ dz, const int* __restrict__ ids_keep,
                                                                const int* __restrict__ ids_restore, int B, int N, int keep, int E, int Te,
                                                                __nv_bfloat16* __restrict__ dy, float* __restrict__ part) {
  __shared__ float red[256 * 8];
  const int chunks = gridDim.x, c = blockIdx.x, e8 = E / 8, per = keep + 1, dper = N + 1;
  const int b0 = (int)((long long)c * B / chunks), b1 = (int)((long long)(c + 1) * B / chunks);
  const size_t rows = (size_t)(b1 - b0) * per * e8;
  for (size_t i = threadIdx.x; i < rows; i += blockDim.x) {
    const int t = b0 * per + (int)(i / e8), d = (int)(i % e8) * 8;
    const int b = t / per, j = t % per;
    const int src = b * dper + (j == 0 ? 0 : 1 + ids_keep[(size_t)b * keep + j - 1]);
    *reinterpret_cast<Bf16x8*>(dy + (size_t)t * E + d) = *reinterpret_cast<const Bf16x8*>(dz + (size_t)src * E + d);
  }
  if (c == chunks - 1) {
    float zero[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) zero[u] = 0.f;
    for (size_t i = threadIdx.x; i < (size_t)(Te - B * per) * e8; i += blockDim.x)
      store8(dy + (size_t)(B * per) * E + i * 8, zero);
  }
  const int groups = blockDim.x / e8, grp = threadIdx.x / e8, col = (threadIdx.x % e8) * 8;
  if (grp < groups) {
    float acc[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] = 0.f;
    const int n = (b1 - b0) * N;
    for (int m = grp; m < n; m += groups) {
      const int b = b0 + m / N, i = m % N;
      if (ids_restore[(size_t)b * N + i] < keep) continue;
      float f[8];
      load8(dz + ((size_t)b * dper + 1 + i) * E + col, f);
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] += f[u];
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) red[grp * E + col + u] = acc[u];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    float s = 0.f;
    for (int g = 0; g < groups; ++g) s += red[g * E + e];
    part[(size_t)c * E + e] = s;
  }
}

__global__ void __launch_bounds__(256) mae_mask_grad_finish_kernel(const float* __restrict__ part, int chunks, int E,
                                                                   __nv_bfloat16* __restrict__ dmask) {
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += part[(size_t)c * E + e];
    dmask[e] = __float2bfloat16_rn(s);
  }
}

// ---- per-image attention, head dim 32 ---------------------------------------------------------------------------------
// rows [0, np) of one head's 32 columns into dst with pitch kPitch; rows past n are zero
__device__ __forceinline__ void stage(const __nv_bfloat16* __restrict__ src, size_t pitch, int n, int np, __nv_bfloat16* dst) {
  for (int it = threadIdx.x; it < np * 4; it += blockDim.x) {
    const int r = it >> 2, ch = it & 3;
    Bf16x8 v;
    if (r < n) {
      v = *reinterpret_cast<const Bf16x8*>(src + (size_t)r * pitch + ch * 8);
    } else {
      v.h[0] = v.h[1] = v.h[2] = v.h[3] = __floats2bfloat162_rn(0.f, 0.f);
    }
    *reinterpret_cast<Bf16x8*>(dst + r * kPitch + ch * 8) = v;
  }
}

// the A fragments of rows [m0, m0 + 16) x 32 columns of a staged tile
__device__ __forceinline__ void load_a(uint32_t (&a)[2][4], const __nv_bfloat16* A, int m0, int g, int t) {
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
    const __nv_bfloat16* lo = A + (m0 + g) * kPitch + 16 * kk + 2 * t;
    a[kk][0] = ld32(lo);
    a[kk][1] = ld32(lo + 8 * kPitch);
    a[kk][2] = ld32(lo + 8);
    a[kk][3] = ld32(lo + 8 * kPitch + 8);
  }
}

// c[16 x 64] = A-tile B[c0 .. c0 + 64, 0 .. 32)^T
__device__ __forceinline__ void mma_abt(float (&c)[8][4], const uint32_t (&a)[2][4], const __nv_bfloat16* B, int g, int t) {
#pragma unroll
  for (int j = 0; j < 8; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __nv_bfloat16* b = B + (8 * j + g) * kPitch + 16 * kk + 2 * t;
      mma16816(c[j], a[kk], ld32(b), ld32(b + 8));
    }
  }
}

// c[16 x 32] += P[16 x 64] B[0 .. 64, 0 .. 32): P an m16 x n64 fp32 accumulator fragment rounded to bf16 as the A operand
__device__ __forceinline__ void mma_pb(float (&c)[4][4], const float (&p)[8][4], const __nv_bfloat16* B, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack2(p[2 * kk][0], p[2 * kk][1]), pack2(p[2 * kk][2], p[2 * kk][3]),
                           pack2(p[2 * kk + 1][0], p[2 * kk + 1][1]), pack2(p[2 * kk + 1][2], p[2 * kk + 1][3])};
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b[4];
      ldsm_x4_t(b, B + (16 * kk + (lane & 7) + ((lane >> 3) & 1) * 8) * kPitch + 16 * np + (lane >> 4) * 8);
      mma16816(c[2 * np], a, b[0], b[1]);
      mma16816(c[2 * np + 1], a, b[2], b[3]);
    }
  }
}

// rows m0 + g + 8 r (r = 0, 1) of a 16 x 32 fragment, times `scale`, to dst + row * pitch
__device__ __forceinline__ void store_rows(const float (&c)[4][4], __nv_bfloat16* dst, size_t pitch, int m0, int n, int g, int t, float scale) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    if (i >= n) continue;
    __nv_bfloat16* d = dst + (size_t)i * pitch + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(d + 8 * j) = pack2(c[j][2 * r] * scale, c[j][2 * r + 1] * scale);
  }
}

struct AttnFwdSmem {
  __nv_bfloat16 q[kMaxTok * kPitch], k[kMaxTok * kPitch], v[kMaxTok * kPitch];
};

__global__ void __launch_bounds__(kAttnThreads) image_attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, int n, int heads,
                                                                      __nv_bfloat16* __restrict__ o, float* __restrict__ lse) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AttnFwdSmem& sm = *reinterpret_cast<AttnFwdSmem*>(smem_raw);
  const int b = blockIdx.x, h = blockIdx.y, C = heads * kHd, np = (n + kChunk - 1) / kChunk * kChunk;
  const size_t row0 = (size_t)b * n, pitch = (size_t)3 * C;
  stage(qkv + row0 * pitch + h * kHd, pitch, n, np, sm.q);
  stage(qkv + row0 * pitch + C + h * kHd, pitch, n, np, sm.k);
  stage(qkv + row0 * pitch + 2 * C + h * kHd, pitch, n, np, sm.v);
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  for (int m0 = 16 * warp; m0 < n; m0 += 16 * kWarps) {
    uint32_t qa[2][4];
    load_a(qa, sm.q, m0, g, t);
    float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int c0 = 0; c0 < n; c0 += kChunk) {
      float s[8][4];
      mma_abt(s, qa, sm.k + c0 * kPitch, g, t);
      float cm[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          s[j][e] = c0 + 8 * j + 2 * t + (e & 1) < n ? s[j][e] * kScale : -INFINITY;
          cm[e >> 1] = fmaxf(cm[e >> 1], s[j][e]);
        }
      }
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        cm[r] = fmaxf(cm[r], __shfl_xor_sync(0xffffffffu, cm[r], 1));
        cm[r] = fmaxf(cm[r], __shfl_xor_sync(0xffffffffu, cm[r], 2));
        const float m = fmaxf(mx[r], cm[r]);                 // finite: key c0 < n is always real
        alpha[r] = exp2f((mx[r] - m) * kLog2e);
        mx[r] = m;
        l[r] *= alpha[r];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          s[j][e] = exp2f((s[j][e] - mx[e >> 1]) * kLog2e);
          l[e >> 1] += s[j][e];
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] *= alpha[e >> 1];
      mma_pb(acc, s, sm.v + c0 * kPitch, lane);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = m0 + g + 8 * r;
      if (i >= n) continue;
      const float inv = 1.f / l[r];
      __nv_bfloat16* dst = o + (row0 + i) * C + h * kHd + 2 * t;
#pragma unroll
      for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
      if (t == 0) lse[(row0 + i) * heads + h] = mx[r] + logf(l[r]);
    }
  }
}

struct AttnBwdSmem {
  __nv_bfloat16 q[kMaxTok * kPitch], k[kMaxTok * kPitch], v[kMaxTok * kPitch], dout[kMaxTok * kPitch];
  float D[kMaxTok], lse[kMaxTok];
};

__global__ void __launch_bounds__(kAttnThreads) image_attn_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ qkv,
                                                                      const __nv_bfloat16* __restrict__ o, const float* __restrict__ lse,
                                                                      int n, int heads, __nv_bfloat16* __restrict__ dqkv) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AttnBwdSmem& sm = *reinterpret_cast<AttnBwdSmem*>(smem_raw);
  const int b = blockIdx.x, h = blockIdx.y, C = heads * kHd, np = (n + kChunk - 1) / kChunk * kChunk;
  const size_t row0 = (size_t)b * n, pitch = (size_t)3 * C;
  stage(qkv + row0 * pitch + h * kHd, pitch, n, np, sm.q);
  stage(qkv + row0 * pitch + C + h * kHd, pitch, n, np, sm.k);
  stage(qkv + row0 * pitch + 2 * C + h * kHd, pitch, n, np, sm.v);
  stage(dout + row0 * C + h * kHd, C, n, np, sm.dout);
  // D = rowsum(dO o O) from O in HBM; rows past n get D = 0 and lse = +inf, so their P is zero
  for (int r = threadIdx.x; r < np; r += blockDim.x) {
    float d = 0.f, lr = INFINITY;
    if (r < n) {
      const __nv_bfloat16* orow = o + (row0 + r) * C + h * kHd;
      const __nv_bfloat16* drow = dout + (row0 + r) * C + h * kHd;
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        float a[8], c[8];
        load8(orow + 8 * ch, a);
        load8(drow + 8 * ch, c);
#pragma unroll
        for (int u = 0; u < 8; ++u) d = fmaf(a[u], c[u], d);
      }
      lr = lse[(row0 + r) * heads + h];
    }
    sm.D[r] = d;
    sm.lse[r] = lr;
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  __nv_bfloat16* dq = dqkv + row0 * pitch + h * kHd;
  // key tiles: dV = P^T dO and dK = scale dS^T Q over every query chunk
  for (int m0 = 16 * warp; m0 < n; m0 += 16 * kWarps) {
    uint32_t ka[2][4], va[2][4];
    load_a(ka, sm.k, m0, g, t);
    load_a(va, sm.v, m0, g, t);
    float dv[4][4], dk[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
      dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = 0.f;
    }
    for (int c0 = 0; c0 < n; c0 += kChunk) {
      float st[8][4], dpt[8][4];
      mma_abt(st, ka, sm.q + c0 * kPitch, g, t);                    // S^T: keys x queries
      mma_abt(dpt, va, sm.dout + c0 * kPitch, g, t);                // dP^T = V dO^T
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = c0 + 8 * j + 2 * t + (e & 1);
          const float p = exp2f((st[j][e] * kScale - sm.lse[qi]) * kLog2e);
          st[j][e] = p;
          dpt[j][e] = p * (dpt[j][e] - sm.D[qi]);
        }
      }
      mma_pb(dv, st, sm.dout + c0 * kPitch, lane);
      mma_pb(dk, dpt, sm.q + c0 * kPitch, lane);
    }
    store_rows(dk, dq + C, pitch, m0, n, g, t, kScale);
    store_rows(dv, dq + 2 * C, pitch, m0, n, g, t, 1.f);
  }
  // query tiles: dQ = scale dS K over every key chunk
  for (int m0 = 16 * warp; m0 < n; m0 += 16 * kWarps) {
    uint32_t qa[2][4], da[2][4];
    load_a(qa, sm.q, m0, g, t);
    load_a(da, sm.dout, m0, g, t);
    const float lr[2] = {sm.lse[m0 + g], sm.lse[m0 + g + 8]}, Dr[2] = {sm.D[m0 + g], sm.D[m0 + g + 8]};
    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int c0 = 0; c0 < n; c0 += kChunk) {
      float s[8][4], dp[8][4];
      mma_abt(s, qa, sm.k + c0 * kPitch, g, t);
      mma_abt(dp, da, sm.v + c0 * kPitch, g, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = e >> 1;
          const float p = c0 + 8 * j + 2 * t + (e & 1) < n ? exp2f((s[j][e] * kScale - lr[r]) * kLog2e) : 0.f;
          dp[j][e] = p * (dp[j][e] - Dr[r]);
        }
      }
      mma_pb(acc, dp, sm.k + c0 * kPitch, lane);
    }
    store_rows(acc, dq, pitch, m0, n, g, t, kScale);
  }
}

// ---- reconstruction loss ----------------------------------------------------------------------------------------------
// The target of image b's patch i in pred's (ky, kx, c) order, in 8-wide groups: lane holds groups lane, lane + 32, lane + 64
// (of G = C p^2 / 8); normalised by the patch's mean and unbiased variance when norm_pix.
template <bool kChannelsLast>
__device__ __forceinline__ void load_target(float (&x)[kMaxGroups][8], const __nv_bfloat16* __restrict__ img, int b, int i, int C, int H,
                                            int W, int p, bool norm_pix, int lane) {
  const int gw = W / p, y0 = (i / gw) * p, x0 = (i % gw) * p, row = p * C, G = row * p / 8;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    const int gi = lane + 32 * k;
    if (gi >= G) continue;
    const int e = 8 * gi, ky = e / row, r = e % row;
    if (kChannelsLast) {
      load8(img + (((size_t)b * H + y0 + ky) * W + x0) * C + r, x[k]);
    } else {
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int kx = (r + u) / C, c = (r + u) % C;
        x[k][u] = __bfloat162float(img[(((size_t)b * C + c) * H + y0 + ky) * W + x0 + kx]);
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) s += x[k][u];
  }
  if (!norm_pix) return;
  const float P = (float)(8 * G);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / P;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    if (lane + 32 * k >= G) continue;
#pragma unroll
    for (int u = 0; u < 8; ++u) ss += (x[k][u] - mean) * (x[k][u] - mean);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float sd = sqrtf(ss / (P - 1.f) + 1e-6f);
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k)
#pragma unroll
    for (int u = 0; u < 8; ++u) x[k][u] = (x[k][u] - mean) / sd;
}

// one warp per patch (b, i): rowloss[b N + i] = mean over the patch of (pred - target)^2 if it is masked, else 0
template <bool kChannelsLast>
__global__ void __launch_bounds__(256) mae_loss_fwd_kernel(const __nv_bfloat16* __restrict__ pred, const __nv_bfloat16* __restrict__ img,
                                                           const int* __restrict__ ids_restore, int B, int C, int H, int W, int p, int keep,
                                                           bool norm_pix, float* __restrict__ rowloss) {
  const int N = (H / p) * (W / p), w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= B * N) return;
  const int b = w / N, i = w % N, P = C * p * p, G = P / 8;
  if (ids_restore[w] < keep) {
    if (lane == 0) rowloss[w] = 0.f;
    return;
  }
  float x[kMaxGroups][8];
  load_target<kChannelsLast>(x, img, b, i, C, H, W, p, norm_pix, lane);
  const __nv_bfloat16* pr = pred + ((size_t)b * (N + 1) + 1 + i) * P;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    const int gi = lane + 32 * k;
    if (gi >= G) continue;
    float f[8];
    load8(pr + 8 * gi, f);
#pragma unroll
    for (int u = 0; u < 8; ++u) s += (f[u] - x[k][u]) * (f[u] - x[k][u]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) rowloss[w] = s / (float)P;
}

// loss = the rowloss entries summed in a fixed order (thread k adds k, k + 1024, ...; then a fixed tree), over B (N - keep)
__global__ void __launch_bounds__(kFinishThreads) mae_loss_finish_kernel(const float* __restrict__ rowloss, int n, float count,
                                                                         float* __restrict__ loss) {
  __shared__ float red[kFinishThreads];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += kFinishThreads) s += rowloss[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = kFinishThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = red[0] / count;
}

// one warp per decoder row: dpred = 2 (pred - target) dloss / (P B (N - keep)) at masked patch rows, zero elsewhere
template <bool kChannelsLast>
__global__ void __launch_bounds__(256) mae_loss_bwd_kernel(const float* __restrict__ dloss, const __nv_bfloat16* __restrict__ pred,
                                                           const __nv_bfloat16* __restrict__ img, const int* __restrict__ ids_restore, int B,
                                                           int C, int H, int W, int p, int keep, bool norm_pix, int Td,
                                                           __nv_bfloat16* __restrict__ dpred) {
  const int N = (H / p) * (W / p), t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= Td) return;
  const int b = t / (N + 1), j = t % (N + 1), P = C * p * p, G = P / 8;
  __nv_bfloat16* out = dpred + (size_t)t * P;
  if (b >= B || j == 0 || ids_restore[(size_t)b * N + j - 1] < keep) {
    float zero[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) zero[u] = 0.f;
    for (int gi = lane; gi < G; gi += 32) store8(out + 8 * gi, zero);
    return;
  }
  float x[kMaxGroups][8];
  load_target<kChannelsLast>(x, img, b, j - 1, C, H, W, p, norm_pix, lane);
  const float coef = 2.f * dloss[0] / ((float)P * (float)((long long)B * (N - keep)));
  const __nv_bfloat16* pr = pred + (size_t)t * P;
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    const int gi = lane + 32 * k;
    if (gi >= G) continue;
    float f[8];
    load8(pr + 8 * gi, f);
#pragma unroll
    for (int u = 0; u < 8; ++u) f[u] = (f[u] - x[k][u]) * coef;
    store8(out + 8 * gi, f);
  }
}

}  // namespace

void launch_mae_shuffle(const float* noise, int B, int N, int keep, int* ids_keep, int* ids_restore, cudaStream_t s) {
  mae_shuffle_kernel<<<B, 256, 0, s>>>(noise, N, keep, ids_keep, ids_restore);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mae_patchify(const void* img, bool channels_last, const int* ids_keep, int B, int C, int H, int W, int p, int keep, int T,
                         void* out, cudaStream_t s) {
  const int blocks = grid_for((size_t)T * (C * p * p / 8));
  if (channels_last)
    mae_patchify_kernel<true><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)img, ids_keep, (__nv_bfloat16*)out, B, C, H, W, p, keep, T);
  else
    mae_patchify_kernel<false><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)img, ids_keep, (__nv_bfloat16*)out, B, C, H, W, p, keep, T);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mae_patch_assemble(const void* y, const void* cls, const void* pos, const int* ids_keep, int B, int keep, int D, int T, void* out,
                               cudaStream_t s) {
  mae_patch_assemble_kernel<<<grid_for((size_t)T * (D / 8)), 256, 0, s>>>((const __nv_bfloat16*)y, (const __nv_bfloat16*)cls,
                                                                         (const __nv_bfloat16*)pos, ids_keep, (__nv_bfloat16*)out, B, keep,
                                                                         D, T);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mae_patch_embed_bwd(const void* dy, int B, int per, int D, int T, void* dpatch, void* dcls, cudaStream_t s) {
  mae_patch_embed_bwd_kernel<<<grid_for((size_t)(T + 1) * (D / 8)), 256, 0, s>>>((const __nv_bfloat16*)dy, (__nv_bfloat16*)dpatch,
                                                                                 (__nv_bfloat16*)dcls, B, per, D, T);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mae_unshuffle(const void* y, const void* mask_token, const void* pos, const int* ids_restore, int B, int N, int keep, int E,
                          int Td, void* z, cudaStream_t s) {
  mae_unshuffle_kernel<<<grid_for((size_t)Td * (E / 8)), 256, 0, s>>>((const __nv_bfloat16*)y, (const __nv_bfloat16*)mask_token,
                                                                     (const __nv_bfloat16*)pos, ids_restore, (__nv_bfloat16*)z, B, N, keep,
                                                                     E, Td);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

int mae_mask_partials(int B) { return mask_chunks(B); }

void launch_mae_unshuffle_bwd(const void* dz, const int* ids_keep, const int* ids_restore, int B, int N, int keep, int E, int Te, void* dy,
                              float* part, void* dmask, cudaStream_t s) {
  const int chunks = mask_chunks(B);
  mae_unshuffle_bwd_kernel<<<chunks, 256, 0, s>>>((const __nv_bfloat16*)dz, ids_keep, ids_restore, B, N, keep, E, Te, (__nv_bfloat16*)dy,
                                                  part);
  B200_CUDA_CHECK(cudaGetLastError());
  mae_mask_grad_finish_kernel<<<1, 256, 0, s>>>(part, chunks, E, (__nv_bfloat16*)dmask);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

void launch_image_attention_fwd(const void* qkv, int B, int tokens, int heads, int T, void* o, float* lse, cudaStream_t s) {
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(image_attn_fwd_kernel, (int)sizeof(AttnFwdSmem), configured);
  const size_t real = (size_t)B * tokens, pad = (size_t)T - real, C = (size_t)heads * kHd;
  if (pad) {
    B200_CUDA_CHECK(cudaMemsetAsync((__nv_bfloat16*)o + real * C, 0, pad * C * sizeof(__nv_bfloat16), s));
    B200_CUDA_CHECK(cudaMemsetAsync(lse + real * heads, 0, pad * heads * sizeof(float), s));
  }
  image_attn_fwd_kernel<<<dim3(B, heads), kAttnThreads, sizeof(AttnFwdSmem), s>>>((const __nv_bfloat16*)qkv, tokens, heads,
                                                                                  (__nv_bfloat16*)o, lse);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_image_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, int B, int tokens, int heads, int T,
                                void* dqkv, cudaStream_t s) {
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(image_attn_bwd_kernel, (int)sizeof(AttnBwdSmem), configured);
  const size_t real = (size_t)B * tokens, pad = (size_t)T - real, C = (size_t)heads * kHd;
  if (pad) B200_CUDA_CHECK(cudaMemsetAsync((__nv_bfloat16*)dqkv + real * 3 * C, 0, pad * 3 * C * sizeof(__nv_bfloat16), s));
  image_attn_bwd_kernel<<<dim3(B, heads), kAttnThreads, sizeof(AttnBwdSmem), s>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)qkv,
                                                                                  (const __nv_bfloat16*)o, lse, tokens, heads,
                                                                                  (__nv_bfloat16*)dqkv);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mae_loss_fwd(const void* pred, const void* img, bool channels_last, const int* ids_restore, int B, int C, int H, int W, int p,
                         int keep, bool norm_pix, float* rowloss, float* loss, cudaStream_t s) {
  const int N = (H / p) * (W / p), blocks = ceil_div((long long)B * N, 8);
  if (channels_last)
    mae_loss_fwd_kernel<true><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)pred, (const __nv_bfloat16*)img, ids_restore, B, C, H, W, p, keep,
                                                     norm_pix, rowloss);
  else
    mae_loss_fwd_kernel<false><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)pred, (const __nv_bfloat16*)img, ids_restore, B, C, H, W, p, keep,
                                                      norm_pix, rowloss);
  B200_CUDA_CHECK(cudaGetLastError());
  mae_loss_finish_kernel<<<1, kFinishThreads, 0, s>>>(rowloss, B * N, (float)((long long)B * (N - keep)), loss);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

void launch_mae_loss_bwd(const float* dloss, const void* pred, const void* img, bool channels_last, const int* ids_restore, int B, int C,
                         int H, int W, int p, int keep, bool norm_pix, int Td, void* dpred, cudaStream_t s) {
  const int blocks = ceil_div(Td, 8);
  if (channels_last)
    mae_loss_bwd_kernel<true><<<blocks, 256, 0, s>>>(dloss, (const __nv_bfloat16*)pred, (const __nv_bfloat16*)img, ids_restore, B, C, H, W, p,
                                                     keep, norm_pix, Td, (__nv_bfloat16*)dpred);
  else
    mae_loss_bwd_kernel<false><<<blocks, 256, 0, s>>>(dloss, (const __nv_bfloat16*)pred, (const __nv_bfloat16*)img, ids_restore, B, C, H, W,
                                                      p, keep, norm_pix, Td, (__nv_bfloat16*)dpred);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
