// Mamba-1's causal depthwise conv1d + SiLU and selective scan on bf16 token rows, with the state reset at every document
// start of `bounds` (int32 [B, S, 2], ops.document_bounds) and padding rows (start == end) giving zeros.
//
//   xz    bf16 [T, 2E]        in_proj's output, x | z (T = B S rows)
//   u     bf16 [T, E]         silu(conv(x) + bias)
//   draw  bf16 [T, E]         dt_proj's bias-free output
//   xbc   bf16 [T, R + 2N]    x_proj's output dt | B | C (N = 16)
//   y     bf16 [T, E]         (C_t . h_t + D u_t) silu(z_t)
//
// Conv: one thread per (row, 8 channels), four fp32 taps in order after the bias, one bf16 rounding.  Its backward walks a
// block of 32 rows per thread with the pre-activation recomputed, writes dx into the x half of a [T, 2E] buffer and fp32
// weight / bias partials per block, which a finish kernel adds in block order.
//
// Scan: one thread per (channel e, state n), 16 channels per 256-thread CTA, sequence chunks of 128 rows.
//   fwd  local scan of each chunk from h = 0 -> end state and sum of delta (+inf when the chunk resets), an in-order
//        combine over the chunks that leaves each chunk's true start state in place (kept for the backward), and a
//        rescan from those states that writes y.
//   bwd  the mirror: a local reverse scan of dh from 0 -> gradient into the state before each chunk, an in-order reverse
//        combine -> the gradient carried into each chunk's end, then the gradient pass.  It recomputes the chunk's states
//        from the saved start state (checkpoints every 16 rows in shared memory, 16 states in registers), and writes du,
//        d draw (through the softplus) and dz (into the z half of the [T, 2E] buffer).  dB and dC are summed over the
//        CTA's 128-channel group in a fixed order into fp32 partials, A_log / D / dt_bias as partials per (row, chunk);
//        finish kernels add them in order.
// No atomics, so two runs give bitwise-equal results; every buffer size is known on the host, nothing is read back.
#include "ops.h"

namespace b200 {
namespace {

constexpr int kN = 16, kK = 4, kChunk = 128, kSub = 16, kCh = 16, kThreads = 256, kGroup = 128;
constexpr int kConvBlock = 32, kConvThreads = 256;
constexpr float kSoftplusThreshold = 20.f;

__device__ __forceinline__ float softplus(float v) { return v > kSoftplusThreshold ? v : log1pf(expf(v)); }
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }
__device__ __forceinline__ float bf(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// sum over the 16 lanes of a half warp (the 16 states of one channel)
__device__ __forceinline__ float sum16(float v) {
#pragma unroll
  for (int o = 8; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------- causal depthwise conv1d + SiLU ----------------------------------------------------------------------
// The bodies take the input rows through a pitch policy: Mamba-1 reads the x half of xz [T, 2E] (XzRows), Mamba-2 the xBC
// column window of zxbcdt [T, W] (PitchRows, x already offset to the window).  E is the channel count; u and du are
// [T, E] contiguous.
struct XzRows {
  int E;
  __device__ __forceinline__ size_t in(size_t r) const { return r * 2 * E; }
  __device__ __forceinline__ size_t out(size_t r) const { return r * 2 * E; }
};
struct PitchRows {
  size_t in_pitch, out_pitch;
  __device__ __forceinline__ size_t in(size_t r) const { return r * in_pitch; }
  __device__ __forceinline__ size_t out(size_t r) const { return r * out_pitch; }
};

template <class Rows>
__device__ __forceinline__ void conv_fwd_body(const __nv_bfloat16* __restrict__ xz, const float* __restrict__ w, const float* __restrict__ bias,
                                              const int2* __restrict__ bounds, int T, int S, int E, Rows rows, __nv_bfloat16* __restrict__ u) {
  const int groups = E / 8;
  const long long idx = (long long)blockIdx.x * kConvThreads + threadIdx.x;
  if (idx >= (long long)T * groups) return;
  const int t = (int)(idx / groups), e0 = (int)(idx % groups) * 8, s = t % S;
  const int2 bd = bounds[t];
  float acc[8];
  if (bd.x >= bd.y) {
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    store8(u + (size_t)t * E + e0, acc);
    return;
  }
  float wv[8][kK];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float4 q = reinterpret_cast<const float4*>(w)[e0 + c];
    wv[c][0] = q.x; wv[c][1] = q.y; wv[c][2] = q.z; wv[c][3] = q.w;
    acc[c] = bias[e0 + c];
  }
#pragma unroll
  for (int j = 0; j < kK; ++j) {
    const int p = s - (kK - 1) + j;
    if (p < max(bd.x, 0)) continue;
    float xv[8];
    load8(xz + rows.in((size_t)(t - (kK - 1) + j)) + e0, xv);
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = fmaf(wv[c][j], xv[c], acc[c]);
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = acc[c] * sigmoidf_(acc[c]);
  store8(u + (size_t)t * E + e0, acc);
}

__global__ void __launch_bounds__(kConvThreads) mamba_conv_fwd_kernel(const __nv_bfloat16* __restrict__ xz, const float* __restrict__ w,
                                                                      const float* __restrict__ bias, const int2* __restrict__ bounds,
                                                                      int T, int S, int E, __nv_bfloat16* __restrict__ u) {
  conv_fwd_body(xz, w, bias, bounds, T, S, E, XzRows{E}, u);
}

__global__ void __launch_bounds__(kConvThreads) mamba2_conv_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w,
                                                                       const float* __restrict__ bias, const int2* __restrict__ bounds,
                                                                       int T, int S, int E, PitchRows rows, __nv_bfloat16* __restrict__ u) {
  conv_fwd_body(x, w, bias, bounds, T, S, E, rows, u);
}

// thread = (row b, block of kConvBlock positions, 8 channels); part fp32 [B * blocks, 5, E] (4 taps, bias)
template <class Rows>
__device__ __forceinline__ void conv_bwd_body(const __nv_bfloat16* __restrict__ du, const __nv_bfloat16* __restrict__ xz,
                                              const float* __restrict__ w, const float* __restrict__ bias, const int2* __restrict__ bounds,
                                              int B, int S, int E, Rows rows, __nv_bfloat16* __restrict__ dxz, float* __restrict__ part) {
  const int groups = E / 8, blocks = (S + kConvBlock - 1) / kConvBlock;
  const long long idx = (long long)blockIdx.x * kConvThreads + threadIdx.x;
  if (idx >= (long long)B * blocks * groups) return;
  const int e0 = (int)(idx % groups) * 8, blk = (int)(idx / groups), b = blk / blocks, s0 = (blk % blocks) * kConvBlock;
  const int s1 = min(s0 + kConvBlock, S);
  float wv[8][kK], bv[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float4 q = reinterpret_cast<const float4*>(w)[e0 + c];
    wv[c][0] = q.x; wv[c][1] = q.y; wv[c][2] = q.z; wv[c][3] = q.w;
    bv[c] = bias[e0 + c];
  }
  float xr[kK][8], dr[kK][8], dw[kK][8], db[8];
  int st[kK];
#pragma unroll
  for (int j = 0; j < kK; ++j) {
    st[j] = INT_MAX;
#pragma unroll
    for (int c = 0; c < 8; ++c) xr[j][c] = dr[j][c] = dw[j][c] = 0.f;
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) db[c] = 0.f;
  const size_t row0 = (size_t)b * S;
  for (int s = s0 - (kK - 1); s < s1 + kK - 1; ++s) {
    // shift the rings: index kK - 1 is position s
#pragma unroll
    for (int j = 0; j < kK - 1; ++j) {
      st[j] = st[j + 1];
#pragma unroll
      for (int c = 0; c < 8; ++c) { xr[j][c] = xr[j + 1][c]; dr[j][c] = dr[j + 1][c]; }
    }
    st[kK - 1] = INT_MAX;
#pragma unroll
    for (int c = 0; c < 8; ++c) { xr[kK - 1][c] = 0.f; dr[kK - 1][c] = 0.f; }
    if (s >= 0 && s < S) load8(xz + rows.in(row0 + s) + e0, xr[kK - 1]);
    if (s >= s0 && s < S) {
      const int2 bd = bounds[row0 + s];
      if (bd.x < bd.y) {
        const int lo = max(bd.x, 0);
        float g[8], pre[8];
        load8(du + (row0 + s) * E + e0, g);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          pre[c] = bv[c];
#pragma unroll
          for (int j = 0; j < kK; ++j)
            if (s - (kK - 1) + j >= lo) pre[c] = fmaf(wv[c][j], xr[j][c], pre[c]);
          const float sg = sigmoidf_(pre[c]);
          dr[kK - 1][c] = g[c] * sg * (1.f + pre[c] * (1.f - sg));
        }
        st[kK - 1] = lo;
        if (s < s1) {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            db[c] += dr[kK - 1][c];
#pragma unroll
            for (int j = 0; j < kK; ++j)
              if (s - (kK - 1) + j >= lo) dw[j][c] = fmaf(dr[kK - 1][c], xr[j][c], dw[j][c]);
          }
        }
      }
    }
    const int t = s - (kK - 1);
    if (t >= s0 && t < s1) {
      // dx[t] = sum_j w_j dpre[t + 3 - j] over the positions t + 3 - j whose document reaches back to t
      float dx[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) dx[c] = 0.f;
#pragma unroll
      for (int j = 0; j < kK; ++j) {
        const int r = kK - 1 - j;                 // ring slot of position t + 3 - j
        if (st[r] <= t) {
#pragma unroll
          for (int c = 0; c < 8; ++c) dx[c] = fmaf(wv[c][j], dr[r][c], dx[c]);
        }
      }
      store8(dxz + rows.out(row0 + t) + e0, dx);
    }
  }
  float* p = part + (size_t)blk * 5 * E + e0;
#pragma unroll
  for (int j = 0; j < kK; ++j) store8(p + (size_t)j * E, dw[j]);
  store8(p + (size_t)kK * E, db);
}

__global__ void __launch_bounds__(kConvThreads) mamba_conv_bwd_kernel(const __nv_bfloat16* __restrict__ du, const __nv_bfloat16* __restrict__ xz,
                                                                      const float* __restrict__ w, const float* __restrict__ bias,
                                                                      const int2* __restrict__ bounds, int B, int S, int E,
                                                                      __nv_bfloat16* __restrict__ dxz, float* __restrict__ part) {
  conv_bwd_body(du, xz, w, bias, bounds, B, S, E, XzRows{E}, dxz, part);
}

__global__ void __launch_bounds__(kConvThreads) mamba2_conv_bwd_kernel(const __nv_bfloat16* __restrict__ du, const __nv_bfloat16* __restrict__ x,
                                                                       const float* __restrict__ w, const float* __restrict__ bias,
                                                                       const int2* __restrict__ bounds, int B, int S, int E, PitchRows rows,
                                                                       __nv_bfloat16* __restrict__ dx, float* __restrict__ part) {
  conv_bwd_body(du, x, w, bias, bounds, B, S, E, rows, dx, part);
}

// dw fp32 [E, 4], db fp32 [E]: the block partials added in block order
__global__ void __launch_bounds__(kConvThreads) mamba_conv_finish_kernel(const float* __restrict__ part, int nblk, int E, float* __restrict__ dw,
                                                                         float* __restrict__ db) {
  const int idx = blockIdx.x * kConvThreads + threadIdx.x;
  if (idx >= 5 * E) return;
  const int j = idx / E, e = idx % E;
  float sum = 0.f;
  for (int k = 0; k < nblk; ++k) sum += part[((size_t)k * 5 + j) * E + e];
  if (j < kK) dw[e * kK + j] = sum;
  else db[e] = sum;
}

// ---------------- selective scan ----------------------------------------------------------------------------------------
// position flags of one chunk: 0 continue, 1 document start (no state carried in), 2 padding or past the row
__device__ __forceinline__ void load_flags(int* flags, const int2* __restrict__ bounds, int b, int c, int S) {
  if (threadIdx.x < kChunk) {
    const int s = c * kChunk + threadIdx.x;
    int f = 2;
    if (s < S) {
      const int2 bd = bounds[(size_t)b * S + s];
      f = bd.x >= bd.y ? 2 : (s == 0 || bd.x >= s) ? 1 : 0;
    }
    flags[threadIdx.x] = f;
  }
  __syncthreads();
}

struct ScanArgs {
  const __nv_bfloat16 *u, *draw, *xbc, *xz;
  const float *A_log, *D, *dt_bias;
  const int2* bounds;
  int B, S, E, pitch, boff, nc;   // pitch of xbc, boff = R (B at R, C at R + 16)
};

struct Lane {
  int b, c, e, n;
  bool active;
  float A, bias;
  __device__ Lane(const ScanArgs& a, int cb) {
    c = blockIdx.x; b = blockIdx.y;
    e = cb + threadIdx.x / kN; n = threadIdx.x % kN;
    active = e < a.E;
    const int ec = active ? e : 0;
    A = -expf(a.A_log[ec * kN + n]);
    bias = a.dt_bias[ec];
  }
};

// one step of the recurrence at row t: returns the new state, sets delta, the decay a and v = draw + dt_bias
__device__ __forceinline__ float step(const ScanArgs& a, const Lane& l, size_t t, int f, float h, float& d, float& decay, float& v, float& uu,
                                      float& Bn) {
  if (f == 2 || !l.active) { d = decay = v = uu = Bn = 0.f; return 0.f; }
  v = bf(a.draw + t * a.E + l.e) + l.bias;
  d = softplus(v);
  uu = bf(a.u + t * a.E + l.e);
  Bn = bf(a.xbc + t * a.pitch + a.boff + l.n);
  decay = f == 1 ? 0.f : expf(d * l.A);
  return fmaf(decay, h, d * Bn * uu);
}

// hst fp32 [B, nc, E, 16] end state of each chunk scanned from 0; sumd fp32 [B, nc, E] (+inf when the chunk resets)
__global__ void __launch_bounds__(kThreads) mamba_scan_local_fwd_kernel(ScanArgs a, float* __restrict__ hst, float* __restrict__ sumd) {
  __shared__ int flags[kChunk];
  const Lane l(a, blockIdx.z * kCh);
  load_flags(flags, a.bounds, l.b, l.c, a.S);
  float h = 0.f, sd = 0.f;
  const int len = min(kChunk, a.S - l.c * kChunk);
  for (int i = 0; i < len; ++i) {
    const size_t t = (size_t)l.b * a.S + l.c * kChunk + i;
    float d, decay, v, uu, Bn;
    h = step(a, l, t, flags[i], h, d, decay, v, uu, Bn);
    sd = flags[i] ? INFINITY : sd + d;
  }
  if (!l.active) return;
  const size_t cell = ((size_t)l.b * a.nc + l.c) * a.E + l.e;
  hst[cell * kN + l.n] = h;
  if (l.n == 0) sumd[cell] = sd;
}

// in place: hst's chunk end states become each chunk's start state (forward), or dq's chunk gradients become the gradient
// carried into each chunk's end (backward, reverse order)
__global__ void __launch_bounds__(kThreads) mamba_scan_combine_kernel(const float* __restrict__ A_log, const float* __restrict__ sumd, int B,
                                                                      int E, int nc, bool reverse, float* __restrict__ st) {
  const long long idx = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= (long long)B * E * kN) return;
  const int n = (int)(idx % kN), e = (int)(idx / kN % E), b = (int)(idx / ((long long)kN * E));
  const float A = -expf(A_log[e * kN + n]);
  float h = 0.f;
  for (int k = 0; k < nc; ++k) {
    const int c = reverse ? nc - 1 - k : k;
    const size_t cell = ((size_t)b * nc + c) * E + e;
    const float local = st[cell * kN + n];
    st[cell * kN + n] = h;
    h = fmaf(expf(A * sumd[cell]), h, local);
  }
}

// y from each chunk's start state
__global__ void __launch_bounds__(kThreads) mamba_scan_out_fwd_kernel(ScanArgs a, const float* __restrict__ hst, __nv_bfloat16* __restrict__ y) {
  __shared__ int flags[kChunk];
  const Lane l(a, blockIdx.z * kCh);
  load_flags(flags, a.bounds, l.b, l.c, a.S);
  const size_t cell = ((size_t)l.b * a.nc + l.c) * a.E + l.e;
  float h = l.active ? hst[cell * kN + l.n] : 0.f;
  const float Dv = l.active ? a.D[l.e] : 0.f;
  const int len = min(kChunk, a.S - l.c * kChunk);
  for (int i = 0; i < len; ++i) {
    const size_t t = (size_t)l.b * a.S + l.c * kChunk + i;
    float d, decay, v, uu, Bn;
    h = step(a, l, t, flags[i], h, d, decay, v, uu, Bn);
    const float Cn = l.active && flags[i] != 2 ? bf(a.xbc + t * a.pitch + a.boff + kN + l.n) : 0.f;
    const float s = sum16(Cn * h);
    if (l.n == 0 && l.active) {
      float out = 0.f;
      if (flags[i] != 2) {
        const float z = bf(a.xz + t * 2 * a.E + a.E + l.e);
        out = (s + Dv * uu) * (z * sigmoidf_(z));
      }
      y[t * a.E + l.e] = __float2bfloat16_rn(out);
    }
  }
}

// dq fp32 [B, nc, E, 16]: the gradient into the state before each chunk from that chunk alone (dh from 0 at its end)
__global__ void __launch_bounds__(kThreads) mamba_scan_local_bwd_kernel(ScanArgs a, const __nv_bfloat16* __restrict__ dy, float* __restrict__ dq) {
  __shared__ int flags[kChunk];
  const Lane l(a, blockIdx.z * kCh);
  load_flags(flags, a.bounds, l.b, l.c, a.S);
  float g = 0.f;
  const int len = min(kChunk, a.S - l.c * kChunk);
  for (int i = len - 1; i >= 0; --i) {
    const int f = flags[i];
    if (f == 2 || !l.active) { g = 0.f; continue; }
    const size_t t = (size_t)l.b * a.S + l.c * kChunk + i;
    const float z = bf(a.xz + t * 2 * a.E + a.E + l.e);
    const float ds = bf(dy + t * a.E + l.e) * (z * sigmoidf_(z));
    const float dh = fmaf(ds, bf(a.xbc + t * a.pitch + a.boff + kN + l.n), g);
    const float d = softplus(bf(a.draw + t * a.E + l.e) + l.bias);
    g = f == 1 ? 0.f : expf(d * l.A) * dh;
  }
  if (!l.active) return;
  dq[(((size_t)l.b * a.nc + l.c) * a.E + l.e) * kN + l.n] = g;
}

struct GradOut {
  __nv_bfloat16 *du, *ddraw, *dxz;
  float *dbc_part, *dA_part, *dD_part, *dbias_part;   // [T, groups, 32], [B nc, E, 16], [B nc, E], [B nc, E]
  int groups;
};

struct GradSmem {
  float ck[kChunk / kSub][kThreads];       // the state before each 16-row sub-chunk
  float red[kSub][kThreads / 32][2 * kN];  // per warp (two channels) dB | dC of the sub-chunk's rows
  float acc[kChunk][2 * kN];               // dB | dC of the chunk's rows, summed over the CTA's channel group
  int flags[kChunk];
};

// grid (nc, B, groups): the CTA walks its group's 128 channels in blocks of 16
__global__ void __launch_bounds__(kThreads) mamba_scan_grad_kernel(ScanArgs a, const __nv_bfloat16* __restrict__ dy, const float* __restrict__ hst,
                                                                   const float* __restrict__ dq, GradOut o) {
  __shared__ __align__(16) GradSmem sm;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  load_flags(sm.flags, a.bounds, blockIdx.y, blockIdx.x, a.S);
  for (int i = threadIdx.x; i < kChunk * 2 * kN; i += kThreads) (&sm.acc[0][0])[i] = 0.f;
  const int len = min(kChunk, a.S - (int)blockIdx.x * kChunk);
  for (int cb = blockIdx.z * kGroup; cb < blockIdx.z * kGroup + kGroup; cb += kCh) {
    const Lane l(a, cb);
    const size_t cell = ((size_t)l.b * a.nc + l.c) * a.E + l.e;
    const float Dv = l.active ? a.D[l.e] : 0.f;
    float h = l.active ? hst[cell * kN + l.n] : 0.f;
    float G = l.active ? dq[cell * kN + l.n] : 0.f;
    const size_t t0 = (size_t)l.b * a.S + l.c * kChunk;
    for (int k = 0; k < kChunk / kSub; ++k) {
      sm.ck[k][threadIdx.x] = h;
#pragma unroll
      for (int i = 0; i < kSub; ++i) {
        const int r = k * kSub + i;
        float d, decay, v, uu, Bn;
        if (r < len) h = step(a, l, t0 + r, sm.flags[r], h, d, decay, v, uu, Bn);
      }
    }
    float dA = 0.f, dD = 0.f, dbias = 0.f;
    for (int k = kChunk / kSub - 1; k >= 0; --k) {
      if (k * kSub >= len) continue;                                 // uniform across the CTA
      float hs[kSub], dec[kSub], dl[kSub], ul[kSub], bl[kSub], vl[kSub];
      const float hk = sm.ck[k][threadIdx.x];
      h = hk;
#pragma unroll
      for (int i = 0; i < kSub; ++i) {
        const int r = k * kSub + i;
        dec[i] = dl[i] = ul[i] = bl[i] = vl[i] = 0.f;
        if (r < len) h = step(a, l, t0 + r, sm.flags[r], h, dl[i], dec[i], vl[i], ul[i], bl[i]);
        else h = 0.f;
        hs[i] = h;
      }
#pragma unroll
      for (int i = kSub - 1; i >= 0; --i) {
        const int r = k * kSub + i;
        const int f = r < len ? sm.flags[r] : 2;
        float dBc = 0.f, dCc = 0.f;
        if (f == 2) {
          G = 0.f;
          if (r < len && l.n == 0 && l.active) {
            const size_t t = t0 + r;
            const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
            o.du[t * a.E + l.e] = zero;
            o.ddraw[t * a.E + l.e] = zero;
            o.dxz[t * 2 * a.E + a.E + l.e] = zero;
          }
        } else {
          const size_t t = t0 + r;
          const float hp = i > 0 ? hs[i - 1] : hk;
          float dyv = 0.f, z = 0.f, Cn = 0.f;
          if (l.active) {
            dyv = bf(dy + t * a.E + l.e);
            z = bf(a.xz + t * 2 * a.E + a.E + l.e);
            Cn = bf(a.xbc + t * a.pitch + a.boff + kN + l.n);
          }
          const float sg = sigmoidf_(z);
          const float s = sum16(Cn * hs[i]);
          const float ds = dyv * (z * sg);
          const float dz = dyv * fmaf(Dv, ul[i], s) * (sg * (1.f + z * (1.f - sg)));
          const float dh = fmaf(ds, Cn, G);
          const float ddl = sum16(dh * fmaf(l.A * dec[i], hp, bl[i] * ul[i]));
          const float dul = sum16(dh * dl[i] * bl[i]);
          dA = fmaf(dh * dl[i] * dec[i], hp, dA);
          dBc = dh * dl[i] * ul[i];
          dCc = ds * hs[i];
          G = dec[i] * dh;
          if (l.n == 0 && l.active) {
            const float ddraw = vl[i] > kSoftplusThreshold ? ddl : ddl * sigmoidf_(vl[i]);
            o.du[t * a.E + l.e] = __float2bfloat16_rn(fmaf(ds, Dv, dul));
            o.ddraw[t * a.E + l.e] = __float2bfloat16_rn(ddraw);
            o.dxz[t * 2 * a.E + a.E + l.e] = __float2bfloat16_rn(dz);
            dD = fmaf(ds, ul[i], dD);
            dbias += ddraw;
          }
        }
        // the warp's two channels, then lanes 0-15 keep dB and lanes 16-31 dC
        dBc += __shfl_xor_sync(0xffffffffu, dBc, 16);
        dCc += __shfl_xor_sync(0xffffffffu, dCc, 16);
        sm.red[i][warp][lane] = lane < kN ? dBc : dCc;
      }
      __syncthreads();
      for (int q = threadIdx.x; q < kSub * 2 * kN; q += kThreads) {
        const int i = q / (2 * kN), j = q % (2 * kN);
        float sum = 0.f;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) sum += sm.red[i][w][j];
        sm.acc[k * kSub + i][j] += sum;
      }
      __syncthreads();
    }
    if (l.active) {
      o.dA_part[cell * kN + l.n] = dA;
      if (l.n == 0) {
        o.dD_part[cell] = dD;
        o.dbias_part[cell] = dbias;
      }
    }
  }
  __syncthreads();
  for (int q = threadIdx.x; q < len * 2 * kN; q += kThreads) {
    const int r = q / (2 * kN), j = q % (2 * kN);
    const size_t t = (size_t)blockIdx.y * a.S + blockIdx.x * kChunk + r;
    o.dbc_part[(t * o.groups + blockIdx.z) * 2 * kN + j] = sm.acc[r][j];
  }
}

// dxbc bf16 [T, R + 32]: zeros in the dt columns, dB | dC = the group partials added in group order
__global__ void __launch_bounds__(kThreads) mamba_dbc_finish_kernel(const float* __restrict__ part, int T, int R, int groups,
                                                                    __nv_bfloat16* __restrict__ dxbc) {
  const int width = R + 2 * kN;
  const long long idx = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= (long long)T * width) return;
  const size_t t = idx / width;
  const int col = (int)(idx % width);
  float sum = 0.f;
  if (col >= R)
    for (int g = 0; g < groups; ++g) sum += part[(t * groups + g) * 2 * kN + col - R];
  dxbc[idx] = __float2bfloat16_rn(sum);
}

// dA_log [E, 16] = A * (sum of the (row, chunk) partials in order), dD [E], ddt_bias [E]
__global__ void __launch_bounds__(kThreads) mamba_param_finish_kernel(const float* __restrict__ A_log, const float* __restrict__ dA_part,
                                                                      const float* __restrict__ dD_part, const float* __restrict__ dbias_part,
                                                                      int P, int E, float* __restrict__ dA_log, float* __restrict__ dD,
                                                                      float* __restrict__ dbias) {
  const int idx = blockIdx.x * kThreads + threadIdx.x;
  if (idx < E * kN) {
    float sum = 0.f;
    for (int p = 0; p < P; ++p) sum += dA_part[(size_t)p * E * kN + idx];
    dA_log[idx] = -expf(A_log[idx]) * sum;
  } else if (idx < E * kN + 2 * E) {
    const bool isD = idx < E * kN + E;
    const int e = isD ? idx - E * kN : idx - E * kN - E;
    const float* part = isD ? dD_part : dbias_part;
    float sum = 0.f;
    for (int p = 0; p < P; ++p) sum += part[(size_t)p * E + e];
    (isD ? dD : dbias)[e] = sum;
  }
}

void check_mamba_shape(const char* who, int B, int S, int E) {
  if (B < 1 || S < 1 || E < 8 || E % 8 || B > 65535)
    throw std::runtime_error(std::string(who) + ": needs B, S >= 1 and E a positive multiple of 8 (got B=" + std::to_string(B) +
                             ", S=" + std::to_string(S) + ", E=" + std::to_string(E) + ")");
  if ((long long)B * S * 2 * E >= (1ll << 31)) throw std::runtime_error(std::string(who) + ": problem too large");
}

ScanArgs scan_args(const void* u, const void* draw, const void* xbc, const void* xz, const float* A_log, const float* D, const float* dt_bias,
                   const int* bounds, int B, int S, int E, int R) {
  ScanArgs a;
  a.u = (const __nv_bfloat16*)u; a.draw = (const __nv_bfloat16*)draw; a.xbc = (const __nv_bfloat16*)xbc; a.xz = (const __nv_bfloat16*)xz;
  a.A_log = A_log; a.D = D; a.dt_bias = dt_bias; a.bounds = (const int2*)bounds;
  a.B = B; a.S = S; a.E = E; a.pitch = R + 2 * kN; a.boff = R; a.nc = mamba_chunks(S);
  return a;
}

}  // namespace

int mamba_conv_blocks(int B, int S) { return B * ceil_div(S, kConvBlock); }
int mamba_chunks(int S) { return ceil_div(S, kChunk); }
int mamba_groups(int E) { return ceil_div(E, kGroup); }

void launch_mamba_conv_fwd(const void* xz, const float* w, const float* bias, const int* bounds, int B, int S, int E, void* u, cudaStream_t s) {
  check_mamba_shape("mamba_conv_fwd", B, S, E);
  const long long n = (long long)B * S * (E / 8);
  mamba_conv_fwd_kernel<<<ceil_div(n, kConvThreads), kConvThreads, 0, s>>>((const __nv_bfloat16*)xz, w, bias, (const int2*)bounds, B * S, S, E,
                                                                          (__nv_bfloat16*)u);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mamba_conv_bwd(const void* du, const void* xz, const float* w, const float* bias, const int* bounds, int B, int S, int E, void* dxz,
                           float* part, float* dw, float* db, cudaStream_t s) {
  check_mamba_shape("mamba_conv_bwd", B, S, E);
  const int nblk = mamba_conv_blocks(B, S);
  mamba_conv_bwd_kernel<<<ceil_div((long long)nblk * (E / 8), kConvThreads), kConvThreads, 0, s>>>(
      (const __nv_bfloat16*)du, (const __nv_bfloat16*)xz, w, bias, (const int2*)bounds, B, S, E, (__nv_bfloat16*)dxz, part);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_conv_finish_kernel<<<ceil_div(5 * E, kConvThreads), kConvThreads, 0, s>>>(part, nblk, E, dw, db);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

void launch_mamba2_conv_fwd(const void* x, long long x_pitch, const float* w, const float* bias, const int* bounds, int B, int S, int E,
                            void* u, cudaStream_t s) {
  check_mamba_shape("mamba2_conv_fwd", B, S, E);
  const long long n = (long long)B * S * (E / 8);
  mamba2_conv_fwd_kernel<<<ceil_div(n, kConvThreads), kConvThreads, 0, s>>>((const __nv_bfloat16*)x, w, bias, (const int2*)bounds, B * S, S, E,
                                                                           PitchRows{(size_t)x_pitch, (size_t)x_pitch}, (__nv_bfloat16*)u);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_mamba2_conv_bwd(const void* du, const void* x, long long x_pitch, const float* w, const float* bias, const int* bounds, int B, int S,
                            int E, void* dx, long long dx_pitch, float* part, float* dw, float* db, cudaStream_t s) {
  check_mamba_shape("mamba2_conv_bwd", B, S, E);
  const int nblk = mamba_conv_blocks(B, S);
  mamba2_conv_bwd_kernel<<<ceil_div((long long)nblk * (E / 8), kConvThreads), kConvThreads, 0, s>>>(
      (const __nv_bfloat16*)du, (const __nv_bfloat16*)x, w, bias, (const int2*)bounds, B, S, E, PitchRows{(size_t)x_pitch, (size_t)dx_pitch},
      (__nv_bfloat16*)dx, part);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_conv_finish_kernel<<<ceil_div(5 * E, kConvThreads), kConvThreads, 0, s>>>(part, nblk, E, dw, db);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

void launch_mamba_scan_fwd(const void* u, const void* draw, const void* xbc, const void* xz, const float* A_log, const float* D,
                           const float* dt_bias, const int* bounds, int B, int S, int E, int R, void* y, float* hst, float* sumd,
                           cudaStream_t s) {
  check_mamba_shape("mamba_scan_fwd", B, S, E);
  const ScanArgs a = scan_args(u, draw, xbc, xz, A_log, D, dt_bias, bounds, B, S, E, R);
  const dim3 grid(a.nc, B, ceil_div(E, kCh));
  mamba_scan_local_fwd_kernel<<<grid, kThreads, 0, s>>>(a, hst, sumd);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_scan_combine_kernel<<<ceil_div((long long)B * E * kN, kThreads), kThreads, 0, s>>>(A_log, sumd, B, E, a.nc, false, hst);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_scan_out_fwd_kernel<<<grid, kThreads, 0, s>>>(a, hst, (__nv_bfloat16*)y);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(3);
}

void launch_mamba_scan_bwd(const void* dy, const void* u, const void* draw, const void* xbc, const void* xz, const float* A_log, const float* D,
                           const float* dt_bias, const int* bounds, const float* hst, const float* sumd, int B, int S, int E, int R,
                           float* dq, float* dbc_part, float* dA_part, float* dD_part, float* dbias_part, void* du, void* ddraw, void* dxbc,
                           void* dxz, float* dA_log, float* dD, float* dbias, cudaStream_t s) {
  check_mamba_shape("mamba_scan_bwd", B, S, E);
  const ScanArgs a = scan_args(u, draw, xbc, xz, A_log, D, dt_bias, bounds, B, S, E, R);
  mamba_scan_local_bwd_kernel<<<dim3(a.nc, B, ceil_div(E, kCh)), kThreads, 0, s>>>(a, (const __nv_bfloat16*)dy, dq);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_scan_combine_kernel<<<ceil_div((long long)B * E * kN, kThreads), kThreads, 0, s>>>(A_log, sumd, B, E, a.nc, true, dq);
  B200_CUDA_CHECK(cudaGetLastError());
  GradOut o;
  o.du = (__nv_bfloat16*)du; o.ddraw = (__nv_bfloat16*)ddraw; o.dxz = (__nv_bfloat16*)dxz;
  o.dbc_part = dbc_part; o.dA_part = dA_part; o.dD_part = dD_part; o.dbias_part = dbias_part; o.groups = mamba_groups(E);
  mamba_scan_grad_kernel<<<dim3(a.nc, B, o.groups), kThreads, 0, s>>>(a, (const __nv_bfloat16*)dy, hst, dq, o);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_dbc_finish_kernel<<<ceil_div((long long)B * S * (R + 2 * kN), kThreads), kThreads, 0, s>>>(dbc_part, B * S, R, o.groups,
                                                                                                  (__nv_bfloat16*)dxbc);
  B200_CUDA_CHECK(cudaGetLastError());
  mamba_param_finish_kernel<<<ceil_div(E * kN + 2 * E, kThreads), kThreads, 0, s>>>(A_log, dA_part, dD_part, dbias_part, B * a.nc, E, dA_log,
                                                                                   dD, dbias);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(5);
}

}  // namespace b200
