// Mamba-2's chunked state-space scan (SSD, "Transformers are SSMs", Dao & Gu 2024) on bf16 token rows, one group
// (n_groups = 1), head dim P = 64, state N = 128, with the state reset at every document start of `bounds` (int32 [B, S, 2],
// ops.document_bounds) and padding rows (start == end) giving zeros.
//
//   xbc   bf16 [T, E + 2N]     silu(conv(xBC)) = x | B | C (T = B S rows, E = H P)
//   dt    bf16 [T, H] view     in_proj's dt columns, read through their row pitch; dt = softplus(dt + dt_bias) (threshold 20)
//   y     bf16 [T, E]          per head h: y = Y_diag + Y_off + D x, one rounding
//
// The sequence is cut into chunks of L = 64 rows.  Per (chunk, head), with cum_i = sum_{k <= i} A dt_k inside the chunk:
//   Y_diag = (C B^T o M) X,  M_ij = exp(cum_i - cum_j) dt_j for start_i <= j <= i, else 0
//   Y_off  = exp(cum_i) C_i h_in for rows whose document began before the chunk
//   S_c    = B^T diag(exp(cum_last - cum_j) dt_j) X over the rows j of the chunk's last document, [N, P]
//   h_in(c + 1) = dec_c h_in(c) + S_c, dec_c = exp(cum_last) when that document began before the chunk, else 0
// exp is only ever taken of a difference cum_i - cum_j (j <= i) or of cum_i itself, so it never exceeds 1.
//
// Kernels (grid (chunks, B) for the per-chunk ones; 256 threads = 8 warps of mma.sync m16n8k16, bf16 operands, fp32 sums):
//   state    S_c per head into fp32 [B, chunks, H, N, P], dec_c; in the backward the same kernel on (C, dy) gives the
//            gradient into each chunk's incoming state from that chunk alone
//   pass     in place, in chunk order per (b, h, n, p): S_c becomes h_in(c) (forward), or, in reverse order, the local
//            gradients become the gradient into each chunk's outgoing state
//   out      C B^T once per chunk (shared by all heads), then y per head
//   grad     per chunk, the heads in order: dx, and dB / dC summed over the heads in registers (fixed order), d dt_raw
//            through the softplus into the dt columns of in_proj's gradient, and (b, chunk, head) partials of dA_log, dD,
//            d dt_bias, which a finish kernel adds in order
// Operands that are fp32 sums rather than bf16 inputs enter the products as two bf16 parts, hi + lo (~16 mantissa bits):
// the chunk states and their gradients everywhere, and (C B^T o M) and M o (dY X^T) in the backward, whose row sums cancel
// over terms much larger than the result.  (C B^T o M) in the forward is one bf16 rounding.
// The backward recomputes the chunk states (state + pass) instead of keeping them from the forward.  No atomics, so two
// runs give bitwise-equal results; every buffer size is known on the host, nothing is read back.
#include "ops.h"

namespace b200 {
namespace {

constexpr int kP = 64, kN = 128, kL = 64, kThreads = 256;
constexpr int kLd = kP + 8;        // bf16 row stride of the [*, 64] tiles
constexpr int kLdN = kN + 8;       // bf16 row stride of the [64, 128] B and C tiles
constexpr int kLdF = kL + 4;       // fp32 row stride of the [64, 64] tiles
constexpr float kSoftplusThreshold = 20.f;

__device__ __forceinline__ float softplus(float v) { return v > kSoftplusThreshold ? v : log1pf(expf(v)); }
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// d (+)= a b, m16n8k16, bf16 x bf16 -> fp32
__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 lo, __nv_bfloat16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// Operand accessors of shared-memory bf16 tiles: a(r, k) gives the pair (r, k), (r, k + 1) of A; b(k, n) gives (k, n), (k + 1, n)
// of B.  Row: element (r, c) at p[r * ld + c], read along c; Col: element (r, c) at p[c * ld + r], read along r.
struct RowPair {   // A(r, k) = p[r][k], or B(k, n) = p[n][k]
  const __nv_bfloat16* p; int ld;
  __device__ __forceinline__ uint32_t operator()(int r, int k) const { return *reinterpret_cast<const uint32_t*>(p + r * ld + k); }
};
struct ColPair {   // A(r, k) = p[k][r], or B(k, n) = p[k][n]
  const __nv_bfloat16* p; int ld;
  __device__ __forceinline__ uint32_t operator()(int r, int k) const { return pack2(p[k * ld + r], p[(k + 1) * ld + r]); }
};

// acc[t] (+)= A B over rows [m0, m0 + 16) and columns [n0 + 8 t, n0 + 8 t + 8) of the warp's tile, K a multiple of 16.
// fb is called as fb(n, k) for Row (B(k, n) = p[n][k]) and as fb(n, k) for Col (B(k, n) = p[k][n]): both take (n, k).
template <int NT, class FA, class FB>
__device__ __forceinline__ void warp_mma(float (&acc)[NT][4], int m0, int n0, int K, FA fa, FB fb) {
  const int g = (threadIdx.x & 31) >> 2, q = threadIdx.x & 3;
#pragma unroll 2
  for (int k0 = 0; k0 < K; k0 += 16) {
    const uint32_t a0 = fa(m0 + g, k0 + 2 * q), a1 = fa(m0 + g + 8, k0 + 2 * q), a2 = fa(m0 + g, k0 + 2 * q + 8),
                   a3 = fa(m0 + g + 8, k0 + 2 * q + 8);
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int n = n0 + 8 * t + g;
      mma16816(acc[t], a0, a1, a2, a3, fb(n, k0 + 2 * q), fb(n, k0 + 2 * q + 8));
    }
  }
}

template <int NT>
__device__ __forceinline__ void zero(float (&acc)[NT][4]) {
#pragma unroll
  for (int t = 0; t < NT; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
}

struct SsdArgs {
  const __nv_bfloat16* xbc;   // [T, E + 2N]
  const __nv_bfloat16* dt;    // [T, *] with row pitch dtp
  const float *A_log, *D, *dt_bias;
  const int2* bounds;
  int B, S, H, nc;
  long long dtp;
  __device__ __forceinline__ int E() const { return H * kP; }
  __device__ __forceinline__ int pitch() const { return H * kP + 2 * kN; }
};

// The rows of one chunk: real (start < end and inside the sequence), the document start, and per head dt and cum.
struct ChunkRows {
  float dt[kL], cum[kL], v[kL];
  int st[kL];
  int real[kL];
  int len, last;       // rows in the chunk; index of its last row
  float dec;           // exp(cum_last) when the last row's document began before the chunk, else 0
  int carry;
};

__device__ __forceinline__ void load_rows(ChunkRows& r, const SsdArgs& a, int b, int c) {
  const int c0 = c * kL;
  if (threadIdx.x < kL) {
    const int s = c0 + threadIdx.x;
    int real = 0, st = 0;
    if (s < a.S) {
      const int2 bd = a.bounds[(size_t)b * a.S + s];
      real = bd.x < bd.y;
      st = max(bd.x, 0);
    }
    r.real[threadIdx.x] = real;
    r.st[threadIdx.x] = st;
  }
  if (threadIdx.x == 0) {
    r.len = min(kL, a.S - c0);
    r.last = r.len - 1;
  }
}

// dt, cum and dec of head h; the caller syncs before and after
__device__ __forceinline__ void head_rows(ChunkRows& r, const SsdArgs& a, int b, int c, int h, float A) {
  if (threadIdx.x < kL) {
    const int i = threadIdx.x;
    float dt = 0.f, v = 0.f;
    if (r.real[i]) {
      v = __bfloat162float(a.dt[((size_t)b * a.S + c * kL + i) * a.dtp + h]) + a.dt_bias[h];
      dt = softplus(v);
    }
    r.dt[i] = dt;
    r.v[i] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float cum = 0.f;
    for (int i = 0; i < kL; ++i) {
      cum += A * r.dt[i];
      r.cum[i] = cum;
    }
    const int l = r.last;
    r.carry = r.real[l] && r.st[l] < c * kL;
    r.dec = r.carry ? expf(r.cum[l]) : 0.f;
  }
}

// weight of row j in the chunk's outgoing state: exp(cum_last - cum_j) for the rows of the last document, else 0
__device__ __forceinline__ float state_decay(const ChunkRows& r, int j) {
  const int l = r.last;
  return r.real[l] && r.real[j] && j <= l && r.st[j] == r.st[l] ? expf(r.cum[l] - r.cum[j]) : 0.f;
}

// copy rows [c0, c0 + 64) of a bf16 matrix (row pitch `pitch`, 64 or 128 columns from col) into a smem tile, zero for rows
// that are not real
template <int kCols>
__device__ __forceinline__ void load_tile(__nv_bfloat16* dst, int ld, const __nv_bfloat16* src, size_t pitch, size_t row0, const ChunkRows& r) {
  constexpr int kVec = kCols / 8;
  for (int q = threadIdx.x; q < kL * kVec; q += kThreads) {
    const int i = q / kVec, v = q % kVec;
    Bf16x8 val;
    if (r.real[i]) val = *reinterpret_cast<const Bf16x8*>(src + (row0 + i) * pitch + 8 * v);
    else val.h[0] = val.h[1] = val.h[2] = val.h[3] = __floats2bfloat162_rn(0.f, 0.f);
    *reinterpret_cast<Bf16x8*>(dst + i * ld + 8 * v) = val;
  }
}

// fp32 [N, P] state -> two bf16 smem tiles [N][kLd], hi = bf16(st) and lo = bf16(st - hi), so that a product with hi + lo
// keeps ~16 mantissa bits of the state (a long document's state and its gradient grow large next to the per-row terms);
// returns this thread's share of sum(st * other) when other != nullptr
__device__ __forceinline__ float load_state(__nv_bfloat16* hi, __nv_bfloat16* lo, const float* __restrict__ st, const float* __restrict__ other) {
  float dot = 0.f;
  for (int q = threadIdx.x; q < kN * kP / 4; q += kThreads) {
    const int n = q / (kP / 4), p = 4 * (q % (kP / 4));
    const float4 v = reinterpret_cast<const float4*>(st)[q];
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y), h1 = __floats2bfloat162_rn(v.z, v.w);
    *reinterpret_cast<__nv_bfloat162*>(hi + n * kLd + p) = h0;
    *reinterpret_cast<__nv_bfloat162*>(hi + n * kLd + p + 2) = h1;
    *reinterpret_cast<__nv_bfloat162*>(lo + n * kLd + p) = __floats2bfloat162_rn(v.x - __low2float(h0), v.y - __high2float(h0));
    *reinterpret_cast<__nv_bfloat162*>(lo + n * kLd + p + 2) = __floats2bfloat162_rn(v.z - __low2float(h1), v.w - __high2float(h1));
    if (other) {
      const float4 o = reinterpret_cast<const float4*>(other)[q];
      dot = fmaf(v.x, o.x, dot); dot = fmaf(v.y, o.y, dot); dot = fmaf(v.z, o.z, dot); dot = fmaf(v.w, o.w, dot);
    }
  }
  return dot;
}

// ---------------- chunk states ------------------------------------------------------------------------------------------
struct StateSmem {
  __nv_bfloat16 R[kL * kLdN];    // B (forward) or C (backward) rows
  __nv_bfloat16 V[kL * kLd];     // weighted x (forward) or dy (backward) rows
  ChunkRows rows;
};

// kGrad = false: out = S_c = B^T diag(exp(cum_last - cum_j) dt_j) X, dec = dec_c.
// kGrad = true:  out = C^T diag(exp(cum_i) [document began before the chunk]) dY, the gradient into h_in(c) from chunk c.
template <bool kGrad>
__global__ void __launch_bounds__(kThreads) ssd_state_kernel(SsdArgs a, const __nv_bfloat16* __restrict__ dy, float* __restrict__ out,
                                                             float* __restrict__ dec) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  StateSmem& sm = *reinterpret_cast<StateSmem*>(smem_raw);
  const int c = blockIdx.x, b = blockIdx.y, warp = threadIdx.x / 32;
  const int E = a.E(), pitch = a.pitch();
  const size_t row0 = (size_t)b * a.S + (size_t)c * kL;
  load_rows(sm.rows, a, b, c);
  __syncthreads();
  load_tile<kN>(sm.R, kLdN, a.xbc + E + (kGrad ? kN : 0), pitch, row0, sm.rows);
  for (int h = 0; h < a.H; ++h) {
    __syncthreads();
    head_rows(sm.rows, a, b, c, h, -expf(a.A_log[h]));
    __syncthreads();
    const ChunkRows& r = sm.rows;
    for (int q = threadIdx.x; q < kL * kP / 2; q += kThreads) {
      const int j = q / (kP / 2), p = 2 * (q % (kP / 2));
      float w = 0.f, v0 = 0.f, v1 = 0.f;
      if (r.real[j]) {
        const __nv_bfloat162 x = kGrad ? *reinterpret_cast<const __nv_bfloat162*>(dy + (row0 + j) * E + h * kP + p)
                                       : *reinterpret_cast<const __nv_bfloat162*>(a.xbc + (row0 + j) * pitch + h * kP + p);
        v0 = __low2float(x); v1 = __high2float(x);
        w = kGrad ? (r.st[j] < c * kL ? expf(r.cum[j]) : 0.f) : state_decay(r, j) * r.dt[j];
      }
      *reinterpret_cast<__nv_bfloat162*>(sm.V + j * kLd + p) = __floats2bfloat162_rn(w * v0, w * v1);
    }
    __syncthreads();
    // out[n][p] = sum_j R[j][n] V[j][p]: warp w owns rows n in [16 w, 16 w + 16), all 64 columns p
    float acc[8][4];
    zero(acc);
    warp_mma(acc, 16 * warp, 0, kL, ColPair{sm.R, kLdN}, ColPair{sm.V, kLd});
    float* o = out + (((size_t)b * a.nc + c) * a.H + h) * kN * kP;
    const int g = (threadIdx.x & 31) >> 2, qd = threadIdx.x & 3;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int n = 16 * warp + g, p = 8 * t + 2 * qd;
      *reinterpret_cast<float2*>(o + n * kP + p) = make_float2(acc[t][0], acc[t][1]);
      *reinterpret_cast<float2*>(o + (n + 8) * kP + p) = make_float2(acc[t][2], acc[t][3]);
    }
    if (!kGrad && threadIdx.x == 0) dec[((size_t)b * a.nc + c) * a.H + h] = r.dec;
  }
}

// in place over the chunks of (b, h, element): st[c] <- the value carried into chunk c, carried = dec_c carried + st[c]
__global__ void __launch_bounds__(kThreads) ssd_pass_kernel(const float* __restrict__ dec, int B, int H, int nc, bool reverse,
                                                            float* __restrict__ st) {
  const long long idx = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= (long long)B * H * kN * kP) return;
  const int e = (int)(idx % (kN * kP)), h = (int)(idx / (kN * kP) % H), b = (int)(idx / ((long long)kN * kP * H));
  float carried = 0.f;
  for (int k = 0; k < nc; ++k) {
    const int c = reverse ? nc - 1 - k : k;
    const size_t cell = ((size_t)b * nc + c) * H + h;
    const float local = st[cell * kN * kP + e];
    st[cell * kN * kP + e] = carried;
    carried = fmaf(dec[cell], carried, local);
  }
}

// ---------------- forward output ----------------------------------------------------------------------------------------
struct OutSmem {
  __nv_bfloat16 C[kL * kLdN], B[kL * kLdN];
  float CB[kL * kLdF];
  __nv_bfloat16 X[kL * kLd], M[kL * kLd], Hs[kN * kLd], Hl[kN * kLd];
  ChunkRows rows;
};

__device__ __forceinline__ bool in_doc(const ChunkRows& r, int i, int j, int c0) {
  return j <= i && r.real[i] && r.real[j] && c0 + j >= r.st[i];
}

__global__ void __launch_bounds__(kThreads) ssd_out_kernel(SsdArgs a, const float* __restrict__ hin, __nv_bfloat16* __restrict__ y) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  OutSmem& sm = *reinterpret_cast<OutSmem*>(smem_raw);
  const int c = blockIdx.x, b = blockIdx.y, c0 = c * kL, warp = threadIdx.x / 32;
  const int E = a.E(), pitch = a.pitch();
  const int g = (threadIdx.x & 31) >> 2, qd = threadIdx.x & 3, m0 = 16 * (warp % 4), n0 = 32 * (warp / 4);
  const size_t row0 = (size_t)b * a.S + (size_t)c0;
  load_rows(sm.rows, a, b, c);
  __syncthreads();
  load_tile<kN>(sm.B, kLdN, a.xbc + E, pitch, row0, sm.rows);
  load_tile<kN>(sm.C, kLdN, a.xbc + E + kN, pitch, row0, sm.rows);
  __syncthreads();
  {  // CB[i][j] = C_i . B_j
    float acc[4][4];
    zero(acc);
    warp_mma(acc, m0, n0, kN, RowPair{sm.C, kLdN}, RowPair{sm.B, kLdN});
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int j = n0 + 8 * t + 2 * qd;
      sm.CB[(m0 + g) * kLdF + j] = acc[t][0]; sm.CB[(m0 + g) * kLdF + j + 1] = acc[t][1];
      sm.CB[(m0 + g + 8) * kLdF + j] = acc[t][2]; sm.CB[(m0 + g + 8) * kLdF + j + 1] = acc[t][3];
    }
  }
  const ChunkRows& r = sm.rows;
  for (int h = 0; h < a.H; ++h) {
    __syncthreads();
    head_rows(sm.rows, a, b, c, h, -expf(a.A_log[h]));
    load_tile<kP>(sm.X, kLd, a.xbc + h * kP, pitch, row0, r);
    load_state(sm.Hs, sm.Hl, hin + (((size_t)b * a.nc + c) * a.H + h) * kN * kP, nullptr);
    __syncthreads();
    for (int q = threadIdx.x; q < kL * kL; q += kThreads) {
      const int i = q / kL, j = q % kL;
      const float m = in_doc(r, i, j, c0) ? sm.CB[i * kLdF + j] * expf(r.cum[i] - r.cum[j]) * r.dt[j] : 0.f;
      sm.M[i * kLd + j] = __float2bfloat16_rn(m);
    }
    __syncthreads();
    float yd[4][4], yo[4][4];
    zero(yd);
    zero(yo);
    warp_mma(yd, m0, n0, kL, RowPair{sm.M, kLd}, ColPair{sm.X, kLd});
    warp_mma(yo, m0, n0, kN, RowPair{sm.C, kLdN}, ColPair{sm.Hs, kLd});
    warp_mma(yo, m0, n0, kN, RowPair{sm.C, kLdN}, ColPair{sm.Hl, kLd});
    const float Dh = a.D[h];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int i = m0 + g + 8 * half;
      if (i >= r.len) continue;
      const float off = r.real[i] && r.st[i] < c0 ? expf(r.cum[i]) : 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int p = n0 + 8 * t + 2 * qd;
        float o0 = 0.f, o1 = 0.f;
        if (r.real[i]) {
          const __nv_bfloat162 x = *reinterpret_cast<const __nv_bfloat162*>(sm.X + i * kLd + p);
          o0 = fmaf(off, yo[t][2 * half], yd[t][2 * half]) + Dh * __low2float(x);
          o1 = fmaf(off, yo[t][2 * half + 1], yd[t][2 * half + 1]) + Dh * __high2float(x);
        }
        *reinterpret_cast<__nv_bfloat162*>(y + (row0 + i) * E + h * kP + p) = __floats2bfloat162_rn(o0, o1);
      }
    }
  }
}

// ---------------- backward ----------------------------------------------------------------------------------------------
struct GradSmem {
  __nv_bfloat16 C[kL * kLdN], B[kL * kLdN];
  float CB[kL * kLdF];
  __nv_bfloat16 X[kL * kLd], DY[kL * kLd];
  __nv_bfloat16 Hs[kN * kLd], G[kN * kLd];     // h_in(c) and the gradient into the chunk's outgoing state (hi parts)
  __nv_bfloat16 Hl[kN * kLd], Gl[kN * kLd];     // their lo parts
  __nv_bfloat16 MT[kL * kLd], Pm[kL * kLd];    // MT[j][i] = (C B^T o M)_ij, Pm[i][j] = M_ij (dY X^T)_ij (hi parts)
  __nv_bfloat16 MTl[kL * kLd], Pml[kL * kLd];  // their lo parts
  float Q[kL * kLdF], R[kL * kLdF];            // dY X^T, then Q = CB M dYX^T and R = CB exp(cum_i - cum_j) dYX^T
  float rowQ[kL], colQ[kL], colR[kL], diag[kL], dcum[kL], direct[kL], draw[kL], dAdt[kL];
  float offt[2][kL], stt[2][kL];
  float red[kThreads];
  ChunkRows rows;
};

struct GradOut {
  __nv_bfloat16* dxbc;       // [T, E + 2N]
  __nv_bfloat16* ddt;        // [T, *] with row pitch ddtp
  long long ddtp;
  float *dA_part, *dD_part, *dbias_part;   // [B chunks, H]
};

__global__ void __launch_bounds__(kThreads, 1) ssd_grad_kernel(SsdArgs a, const __nv_bfloat16* __restrict__ dy, const float* __restrict__ hin,
                                                               const float* __restrict__ gout, GradOut o) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  GradSmem& sm = *reinterpret_cast<GradSmem*>(smem_raw);
  const int c = blockIdx.x, b = blockIdx.y, c0 = c * kL, warp = threadIdx.x / 32;
  const int E = a.E(), pitch = a.pitch();
  const int g = (threadIdx.x & 31) >> 2, qd = threadIdx.x & 3, m0 = 16 * (warp % 4), half_w = warp / 4;
  const size_t row0 = (size_t)b * a.S + (size_t)c0;
  load_rows(sm.rows, a, b, c);
  __syncthreads();
  load_tile<kN>(sm.B, kLdN, a.xbc + E, pitch, row0, sm.rows);
  load_tile<kN>(sm.C, kLdN, a.xbc + E + kN, pitch, row0, sm.rows);
  __syncthreads();
  {
    float acc[4][4];
    zero(acc);
    warp_mma(acc, m0, 32 * half_w, kN, RowPair{sm.C, kLdN}, RowPair{sm.B, kLdN});
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int j = 32 * half_w + 8 * t + 2 * qd;
      sm.CB[(m0 + g) * kLdF + j] = acc[t][0]; sm.CB[(m0 + g) * kLdF + j + 1] = acc[t][1];
      sm.CB[(m0 + g + 8) * kLdF + j] = acc[t][2]; sm.CB[(m0 + g + 8) * kLdF + j + 1] = acc[t][3];
    }
  }
  // dB and dC of the warp's rows [m0, m0 + 16) and state columns [64 half_w, 64 half_w + 64), summed over the heads in order
  float dBacc[8][4], dCacc[8][4];
  zero(dBacc);
  zero(dCacc);
  const ChunkRows& r = sm.rows;
  for (int h = 0; h < a.H; ++h) {
    const float A = -expf(a.A_log[h]);
    const size_t cell = ((size_t)b * a.nc + c) * a.H + h;
    __syncthreads();
    head_rows(sm.rows, a, b, c, h, A);
    load_tile<kP>(sm.X, kLd, a.xbc + h * kP, pitch, row0, r);
    load_tile<kP>(sm.DY, kLd, dy + h * kP, E, row0, r);
    sm.red[threadIdx.x] = load_state(sm.Hs, sm.Hl, hin + cell * kN * kP, gout + cell * kN * kP);
    load_state(sm.G, sm.Gl, gout + cell * kN * kP, nullptr);
    __syncthreads();
    {  // Q = dY X^T
      float acc[4][4];
      zero(acc);
      warp_mma(acc, m0, 32 * half_w, kP, RowPair{sm.DY, kLd}, RowPair{sm.X, kLd});
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int j = 32 * half_w + 8 * t + 2 * qd;
        sm.Q[(m0 + g) * kLdF + j] = acc[t][0]; sm.Q[(m0 + g) * kLdF + j + 1] = acc[t][1];
        sm.Q[(m0 + g + 8) * kLdF + j] = acc[t][2]; sm.Q[(m0 + g + 8) * kLdF + j + 1] = acc[t][3];
      }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < kL * kL; q += kThreads) {
      const int i = q / kL, j = q % kL;
      const float dyx = sm.Q[i * kLdF + j];
      if (i == j) sm.diag[i] = dyx;
      const float e = in_doc(r, i, j, c0) ? expf(r.cum[i] - r.cum[j]) : 0.f;
      const float cb = sm.CB[i * kLdF + j], l = e * r.dt[j];
      const float mt = cb * l, pm = l * dyx;
      const __nv_bfloat16 mth = __float2bfloat16_rn(mt), pmh = __float2bfloat16_rn(pm);
      sm.MT[j * kLd + i] = mth;
      sm.MTl[j * kLd + i] = __float2bfloat16_rn(mt - __bfloat162float(mth));
      sm.Pm[i * kLd + j] = pmh;
      sm.Pml[i * kLd + j] = __float2bfloat16_rn(pm - __bfloat162float(pmh));
      sm.Q[i * kLdF + j] = cb * l * dyx;
      sm.R[i * kLdF + j] = cb * e * dyx;
    }
    __syncthreads();
    if (threadIdx.x < kL) {
      float s = 0.f;
      for (int j = 0; j < kL; ++j) s += sm.Q[threadIdx.x * kLdF + j];
      sm.rowQ[threadIdx.x] = s;
    } else if (threadIdx.x < 2 * kL) {
      const int j = threadIdx.x - kL;
      float sq = 0.f, sr = 0.f;
      for (int i = 0; i < kL; ++i) { sq += sm.Q[i * kLdF + j]; sr += sm.R[i * kLdF + j]; }
      sm.colQ[j] = sq;
      sm.colR[j] = sr;
    }
    {  // dx[j][p] = sum_i MT[j][i] dY[i][p] + w_j sum_n B[j][n] G[n][p] + D dy[j][p]
      const int n0 = 32 * half_w;
      float acc[4][4], accg[4][4];
      zero(acc);
      zero(accg);
      warp_mma(acc, m0, n0, kL, RowPair{sm.MT, kLd}, ColPair{sm.DY, kLd});
      warp_mma(acc, m0, n0, kL, RowPair{sm.MTl, kLd}, ColPair{sm.DY, kLd});
      warp_mma(accg, m0, n0, kN, RowPair{sm.B, kLdN}, ColPair{sm.G, kLd});
      warp_mma(accg, m0, n0, kN, RowPair{sm.B, kLdN}, ColPair{sm.Gl, kLd});
      const float Dh = a.D[h];
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int j = m0 + g + 8 * hf;
        if (j >= r.len) continue;
        const float w = state_decay(r, j) * r.dt[j];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int p = n0 + 8 * t + 2 * qd;
          float o0 = 0.f, o1 = 0.f;
          if (r.real[j]) {
            const __nv_bfloat162 d = *reinterpret_cast<const __nv_bfloat162*>(sm.DY + j * kLd + p);
            o0 = fmaf(w, accg[t][2 * hf], acc[t][2 * hf]) + Dh * __low2float(d);
            o1 = fmaf(w, accg[t][2 * hf + 1], acc[t][2 * hf + 1]) + Dh * __high2float(d);
          }
          *reinterpret_cast<__nv_bfloat162*>(o.dxbc + (row0 + j) * pitch + h * kP + p) = __floats2bfloat162_rn(o0, o1);
        }
      }
    }
    const int n0 = 64 * half_w;
    {  // dC[i][n] += sum_j Pm[i][j] B[j][n] + off_i exp(cum_i) sum_p dY[i][p] h_in[n][p]
      warp_mma(dCacc, m0, n0, kL, RowPair{sm.Pm, kLd}, ColPair{sm.B, kLdN});
      warp_mma(dCacc, m0, n0, kL, RowPair{sm.Pml, kLd}, ColPair{sm.B, kLdN});
      float tmp[8][4];
      zero(tmp);
      warp_mma(tmp, m0, n0, kP, RowPair{sm.DY, kLd}, RowPair{sm.Hs, kLd});
      warp_mma(tmp, m0, n0, kP, RowPair{sm.DY, kLd}, RowPair{sm.Hl, kLd});
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int i = m0 + g + 8 * hf;
        const float off = r.real[i] && r.st[i] < c0 ? expf(r.cum[i]) : 0.f;
        float dot = 0.f;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int n = n0 + 8 * t + 2 * qd;
          dCacc[t][2 * hf] = fmaf(off, tmp[t][2 * hf], dCacc[t][2 * hf]);
          dCacc[t][2 * hf + 1] = fmaf(off, tmp[t][2 * hf + 1], dCacc[t][2 * hf + 1]);
          dot = fmaf(__bfloat162float(sm.C[i * kLdN + n]), tmp[t][2 * hf], dot);
          dot = fmaf(__bfloat162float(sm.C[i * kLdN + n + 1]), tmp[t][2 * hf + 1], dot);
        }
        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
        dot += __shfl_xor_sync(0xffffffffu, dot, 2);
        if (qd == 0) sm.offt[half_w][i] = off * dot;
      }
    }
    {  // dB[j][n] += sum_i Pm[i][j] C[i][n] + w_j sum_p X[j][p] G[n][p]
      warp_mma(dBacc, m0, n0, kL, ColPair{sm.Pm, kLd}, ColPair{sm.C, kLdN});
      warp_mma(dBacc, m0, n0, kL, ColPair{sm.Pml, kLd}, ColPair{sm.C, kLdN});
      float tmp[8][4];
      zero(tmp);
      warp_mma(tmp, m0, n0, kP, RowPair{sm.X, kLd}, RowPair{sm.G, kLd});
      warp_mma(tmp, m0, n0, kP, RowPair{sm.X, kLd}, RowPair{sm.Gl, kLd});
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int j = m0 + g + 8 * hf;
        const float sd = state_decay(r, j), w = sd * r.dt[j];
        float dot = 0.f;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int n = n0 + 8 * t + 2 * qd;
          dBacc[t][2 * hf] = fmaf(w, tmp[t][2 * hf], dBacc[t][2 * hf]);
          dBacc[t][2 * hf + 1] = fmaf(w, tmp[t][2 * hf + 1], dBacc[t][2 * hf + 1]);
          dot = fmaf(__bfloat162float(sm.B[j * kLdN + n]), tmp[t][2 * hf], dot);
          dot = fmaf(__bfloat162float(sm.B[j * kLdN + n + 1]), tmp[t][2 * hf + 1], dot);
        }
        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
        dot += __shfl_xor_sync(0xffffffffu, dot, 2);
        if (qd == 0) sm.stt[half_w][j] = dot;     // B_j . (G x_j)
      }
    }
    __syncthreads();
    // the gradient into cum_i, then into A dt_k = the reverse cumulative sum over the chunk
    if (threadIdx.x < kL) {
      const int i = threadIdx.x;
      const float sd = state_decay(r, i), bgx = sm.stt[0][i] + sm.stt[1][i];
      sm.dcum[i] = sm.rowQ[i] - sm.colQ[i] + (sm.offt[0][i] + sm.offt[1][i]) - sd * r.dt[i] * bgx;
      sm.direct[i] = sm.colR[i] + sd * bgx;
      sm.draw[i] = sd * r.dt[i] * bgx;          // this row's share of the outgoing state's gradient into cum_last
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float to_last = 0.f, carry = 0.f;
      for (int i = 0; i < kL; ++i) to_last += sm.draw[i];
      for (int k = 0; k < kThreads; ++k) carry += sm.red[k];
      sm.dcum[r.last] += to_last + r.dec * carry;
      float acc = 0.f;
      for (int k = kL - 1; k >= 0; --k) {
        acc += sm.dcum[k];
        sm.dAdt[k] = acc;
      }
    }
    __syncthreads();
    if (threadIdx.x < kL) {
      const int k = threadIdx.x;
      float d = 0.f;
      if (r.real[k]) {
        const float ddt = fmaf(A, sm.dAdt[k], sm.direct[k]);
        d = r.v[k] > kSoftplusThreshold ? ddt : ddt * sigmoidf_(r.v[k]);
      }
      sm.draw[k] = d;
      if (k < r.len) o.ddt[(row0 + k) * o.ddtp + h] = __float2bfloat16_rn(d);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float dA = 0.f, dD = 0.f, dbias = 0.f;
      for (int k = 0; k < kL; ++k) {
        dA = fmaf(r.dt[k], sm.dAdt[k], dA);
        dD += r.real[k] ? sm.diag[k] : 0.f;
        dbias += sm.draw[k];
      }
      o.dA_part[cell] = dA;
      o.dD_part[cell] = dD;
      o.dbias_part[cell] = dbias;
    }
  }
  // dB | dC of the chunk's rows
  const int n0 = 64 * half_w;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int i = m0 + g + 8 * hf;
    if (i >= r.len) continue;
    const bool real = r.real[i];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int n = n0 + 8 * t + 2 * qd;
      __nv_bfloat16* row = o.dxbc + (row0 + i) * pitch + E;
      *reinterpret_cast<__nv_bfloat162*>(row + n) =
          __floats2bfloat162_rn(real ? dBacc[t][2 * hf] : 0.f, real ? dBacc[t][2 * hf + 1] : 0.f);
      *reinterpret_cast<__nv_bfloat162*>(row + kN + n) =
          __floats2bfloat162_rn(real ? dCacc[t][2 * hf] : 0.f, real ? dCacc[t][2 * hf + 1] : 0.f);
    }
  }
}

// dA_log[h] = A_h (sum of the (b, chunk) partials in order), dD[h], ddt_bias[h]
__global__ void __launch_bounds__(kThreads) ssd_param_finish_kernel(const float* __restrict__ A_log, const float* __restrict__ dA_part,
                                                                    const float* __restrict__ dD_part, const float* __restrict__ dbias_part,
                                                                    int parts, int H, float* __restrict__ dA_log, float* __restrict__ dD,
                                                                    float* __restrict__ dbias) {
  const int idx = blockIdx.x * kThreads + threadIdx.x;
  if (idx >= 3 * H) return;
  const int which = idx / H, h = idx % H;
  const float* part = which == 0 ? dA_part : which == 1 ? dD_part : dbias_part;
  float sum = 0.f;
  for (int k = 0; k < parts; ++k) sum += part[(size_t)k * H + h];
  if (which == 0) dA_log[h] = -expf(A_log[h]) * sum;
  else (which == 1 ? dD : dbias)[h] = sum;
}

void check_ssd_shape(const char* who, int B, int S, int H) {
  if (B < 1 || S < 1 || H < 1 || B > 65535 || H % 8)
    throw std::runtime_error(std::string(who) + ": needs B, S >= 1 and heads a positive multiple of 8 (got B=" + std::to_string(B) +
                             ", S=" + std::to_string(S) + ", H=" + std::to_string(H) + ")");
}

SsdArgs ssd_args(const void* xbc, const void* dt, long long dtp, const float* A_log, const float* D, const float* dt_bias, const int* bounds,
                 int B, int S, int H) {
  SsdArgs a;
  a.xbc = (const __nv_bfloat16*)xbc; a.dt = (const __nv_bfloat16*)dt; a.dtp = dtp;
  a.A_log = A_log; a.D = D; a.dt_bias = dt_bias; a.bounds = (const int2*)bounds;
  a.B = B; a.S = S; a.H = H; a.nc = ssd_chunks(S);
  return a;
}

template <class K>
void set_smem(K kernel, size_t bytes) {
  B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}

void run_states(const SsdArgs& a, float* st, float* dec, cudaStream_t s) {
  set_smem(ssd_state_kernel<false>, sizeof(StateSmem));
  ssd_state_kernel<false><<<dim3(a.nc, a.B), kThreads, sizeof(StateSmem), s>>>(a, nullptr, st, dec);
  B200_CUDA_CHECK(cudaGetLastError());
  ssd_pass_kernel<<<ceil_div((long long)a.B * a.H * kN * kP, kThreads), kThreads, 0, s>>>(dec, a.B, a.H, a.nc, false, st);
  B200_CUDA_CHECK(cudaGetLastError());
}

}  // namespace

int ssd_chunks(int S) { return ceil_div(S, kL); }

void launch_ssd_fwd(const void* xbc, const void* dt, long long dt_pitch, const float* A_log, const float* D, const float* dt_bias,
                    const int* bounds, int B, int S, int H, float* states, float* dec, void* y, cudaStream_t s) {
  check_ssd_shape("ssd_fwd", B, S, H);
  const SsdArgs a = ssd_args(xbc, dt, dt_pitch, A_log, D, dt_bias, bounds, B, S, H);
  run_states(a, states, dec, s);
  set_smem(ssd_out_kernel, sizeof(OutSmem));
  ssd_out_kernel<<<dim3(a.nc, B), kThreads, sizeof(OutSmem), s>>>(a, states, (__nv_bfloat16*)y);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(3);
}

void launch_ssd_bwd(const void* dy, const void* xbc, const void* dt, long long dt_pitch, const float* A_log, const float* D,
                    const float* dt_bias, const int* bounds, int B, int S, int H, float* states, float* gstates, float* dec,
                    float* dA_part, float* dD_part, float* dbias_part, void* dxbc, void* ddt, long long ddt_pitch, float* dA_log,
                    float* dD, float* dbias, cudaStream_t s) {
  check_ssd_shape("ssd_bwd", B, S, H);
  const SsdArgs a = ssd_args(xbc, dt, dt_pitch, A_log, D, dt_bias, bounds, B, S, H);
  run_states(a, states, dec, s);
  set_smem(ssd_state_kernel<true>, sizeof(StateSmem));
  ssd_state_kernel<true><<<dim3(a.nc, B), kThreads, sizeof(StateSmem), s>>>(a, (const __nv_bfloat16*)dy, gstates, nullptr);
  B200_CUDA_CHECK(cudaGetLastError());
  ssd_pass_kernel<<<ceil_div((long long)B * H * kN * kP, kThreads), kThreads, 0, s>>>(dec, B, H, a.nc, true, gstates);
  B200_CUDA_CHECK(cudaGetLastError());
  GradOut o;
  o.dxbc = (__nv_bfloat16*)dxbc; o.ddt = (__nv_bfloat16*)ddt; o.ddtp = ddt_pitch;
  o.dA_part = dA_part; o.dD_part = dD_part; o.dbias_part = dbias_part;
  set_smem(ssd_grad_kernel, sizeof(GradSmem));
  ssd_grad_kernel<<<dim3(a.nc, B), kThreads, sizeof(GradSmem), s>>>(a, (const __nv_bfloat16*)dy, states, gstates, o);
  B200_CUDA_CHECK(cudaGetLastError());
  ssd_param_finish_kernel<<<ceil_div(3 * H, kThreads), kThreads, 0, s>>>(A_log, dA_part, dD_part, dbias_part, B * a.nc, H, dA_log, dD, dbias);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(6);
}

}  // namespace b200
