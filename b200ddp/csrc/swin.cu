// Swin Transformer's shifted-window attention (window 7, head dim 32) on bf16 token rows in raster order, with no roll,
// window partition or permute in memory, and Swin V2's cosine variant at window 8 (section at the end).
//
//   qkv   bf16 [B*H*W, 3C]   the qkv projection of the rows (b, y, x), columns [q heads | k heads | v heads], C = 32 heads
//   table fp32 [169, heads]  the learned relative position bias, entry (dy + 6) * 13 + (dx + 6)
//   o     bf16 [B*H*W, C]    each token's output on its own row
//   lse   fp32 [B*H*W, heads] natural-log row log-sum-exp of the biased, masked scores
//
// The token at (y, x) sits at shifted coordinates y' = (y - sy) mod H, x' = (x - sx) mod W, in window (y' / 7, x' / 7) at
// local index 7 (y' % 7) + x' % 7.  Its score against token j of its window is
//   s_ij = 32^-0.5 q_i . k_j + table[(yi - yj + 6) 13 + (xi - xj + 6), h] + m_ij
// with m_ij = -100 (torchvision's value) where i and j lie in different shift regions: [0, H-7), [H-7, H-sy), [H-sy, H)
// along y' when sy > 0 (one region when sy = 0), and the same along x'.
//
// One CTA of four warps per (window, head).  The 49 q, k and v rows (64 bytes each) are gathered with 16-byte loads into
// shared memory padded to 64 rows; warp w owns query rows [16 w, 16 w + 16) and runs m16n8k16 tensor-core MMAs with the
// scores and P in registers.  Padding keys get -inf, padding query rows are never stored.  The kernel moves far more
// bytes than it computes (K = 32), so warp-level MMAs keep up with HBM.
//   fwd     S = Q K^T, softmax in fp32 registers with the head's table row in shared memory, O = P V.
//   bwd     per window: P from lse, D = rowsum(dO o O), dP = dO V^T, dS = P (dP - D), dQ = scale dS K, dV = P^T dO,
//           dK = scale dS^T Q; dqkv by plain stores (each row belongs to exactly one window).  The window's fp32 dS is
//           folded into its 169 bins in a fixed order and written as one partial per CTA, and a finish kernel adds the
//           partials in window order.
// No atomics, so two runs give bitwise-equal results; nothing is read back to the host.
#include "ops.h"
#include "warp_mma.cuh"

namespace b200 {
namespace {

constexpr int kWin = 7, kTok = 49, kRows = 64, kHd = 32, kBins = 169;
constexpr int kThreads = 128;
constexpr int kPitch = kHd + 8;        // bf16 pitch of a staged row: 80 bytes, conflict-free fragment loads and ldmatrix
constexpr int kPPitch = kRows + 8;     // bf16 pitch of a staged P / dS row: 144 bytes
constexpr float kScale = 0.17677669529663687f;   // 32^-0.5
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kMask = -100.f;
constexpr int kFinishWarps = 32;

// c[16 x 64] = A[m0 .. m0 + 16, 0 .. 32) B[0 .. 64, 0 .. 32)^T, both row-major bf16 in shared memory with pitch kPitch
__device__ __forceinline__ void mma_abt(float (&c)[8][4], const __nv_bfloat16* A, const __nv_bfloat16* B, int m0, int g, int t) {
#pragma unroll
  for (int j = 0; j < 8; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < kHd / 16; ++kk) {
    const __nv_bfloat16* a_lo = A + (m0 + g) * kPitch + 16 * kk + 2 * t;
    const __nv_bfloat16* a_hi = a_lo + 8 * kPitch;
    const uint32_t a[4] = {ld32(a_lo), ld32(a_hi), ld32(a_lo + 8), ld32(a_hi + 8)};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __nv_bfloat16* b = B + (8 * j + g) * kPitch + 16 * kk + 2 * t;
      mma16816(c[j], a, ld32(b), ld32(b + 8));
    }
  }
}

// c[16 x 32] = P[16 x 64] B[0 .. 64, 0 .. 32): P is an m16 x n64 fp32 accumulator fragment, rounded to bf16 as the A
// operand; B row-major bf16 in shared memory with pitch kPitch
__device__ __forceinline__ void mma_pb(float (&c)[4][4], const float (&p)[8][4], const __nv_bfloat16* B, int lane) {
#pragma unroll
  for (int j = 0; j < 4; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < kRows / 16; ++kk) {
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

// c[16 x 32] = A^T[m0 .. m0 + 16, 0 .. 64) B[0 .. 64, 0 .. 32): A [64 x 64] row-major bf16 with pitch kPPitch (read
// transposed), B row-major bf16 with pitch kPitch
__device__ __forceinline__ void mma_atb(float (&c)[4][4], const __nv_bfloat16* A, const __nv_bfloat16* B, int m0, int lane) {
#pragma unroll
  for (int j = 0; j < 4; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
  const int i = lane >> 3, rr = lane & 7;
#pragma unroll
  for (int kk = 0; kk < kRows / 16; ++kk) {
    uint32_t a[4];
    ldsm_x4_t(a, A + (16 * kk + (i >> 1) * 8 + rr) * kPPitch + m0 + (i & 1) * 8);
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b[4];
      ldsm_x4_t(b, B + (16 * kk + rr + (i & 1) * 8) * kPitch + 16 * np + (i >> 1) * 8);
      mma16816(c[2 * np], a, b[0], b[1]);
      mma16816(c[2 * np + 1], a, b[2], b[3]);
    }
  }
}

// The geometry of a Win x Win window: the raster row of each of its tokens and, per token,
// (2 Win - 1) ly + lx | region << 8 (-1 past Win^2).
template <int Win>
struct WindowOf {
  int H, W, sy, sx;
  int b, wy, wx;
  __device__ WindowOf(int w, int H_, int W_, int sy_, int sx_) : H(H_), W(W_), sy(sy_), sx(sx_) {
    const int nwx = W / Win, per = (H / Win) * nwx;
    b = w / per;
    wy = (w % per) / nwx;
    wx = w % nwx;
  }
  __device__ int row(int i) const {
    int y = wy * Win + i / Win + sy, x = wx * Win + i % Win + sx;
    if (y >= H) y -= H;
    if (x >= W) x -= W;
    return ((b * H) + y) * W + x;
  }
  __device__ int info(int i) const {
    if (i >= Win * Win) return -1;
    const int ly = i / Win, lx = i % Win, ys = wy * Win + ly, xs = wx * Win + lx;
    const int ry = sy == 0 ? 0 : ys < H - Win ? 0 : ys < H - sy ? 1 : 2;
    const int rx = sx == 0 ? 0 : xs < W - Win ? 0 : xs < W - sx ? 1 : 2;
    return ((2 * Win - 1) * ly + lx) | ((3 * ry + rx) << 8);
  }
};
using Window = WindowOf<kWin>;

// n staged [64][kPitch] tiles: tile k holds columns [col + k step, col + k step + 32) of the rows src + rows[i] pitch and
// sits at dst + k 64 kPitch; rows past Tok are zero
template <int Tok = kTok>
__device__ __forceinline__ void stage(const __nv_bfloat16* __restrict__ src, size_t pitch, int col, int step, int n, const int* rows,
                                      __nv_bfloat16* dst) {
  for (int it = threadIdx.x; it < n * kRows * 4; it += kThreads) {
    const int ch = it & 3, r = (it >> 2) & (kRows - 1), k = it / (kRows * 4);
    Bf16x8 v;
    if (r < Tok) {
      v = *reinterpret_cast<const Bf16x8*>(src + (size_t)rows[r] * pitch + col + k * step + ch * 8);
    } else {
      v.h[0] = v.h[1] = v.h[2] = v.h[3] = __floats2bfloat162_rn(0.f, 0.f);
    }
    *reinterpret_cast<Bf16x8*>(dst + (k * kRows + r) * kPitch + ch * 8) = v;
  }
}

// the biased, masked, scaled scores of this lane's fragment: rows m0 + g (+ 8), keys 8 j + 2 t (+ 1); info codes of a
// Win x Win window
template <int Win = kWin>
__device__ __forceinline__ void bias_mask(float (&s)[8][4], const float* tbl, const int* info, int m0, int g, int t, float scale = kScale) {
  const int i0 = max(info[m0 + g], 0), i1 = max(info[m0 + g + 8], 0);   // a padding query row scores as token 0
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int qi = e < 2 ? i0 : i1, kj = info[8 * j + 2 * t + (e & 1)];
      float v = -INFINITY;
      if (kj >= 0) {
        v = s[j][e] * scale + tbl[(qi & 0xff) - (kj & 0xff) + (Win - 1) * (2 * Win - 1) + Win - 1];
        if ((qi >> 8) != (kj >> 8)) v += kMask;
      }
      s[j][e] = v;
    }
  }
}

struct FwdSmem {
  __nv_bfloat16 q[kRows * kPitch], k[kRows * kPitch], v[kRows * kPitch];
  float tbl[kBins];
  int rows[kRows], info[kRows];
};

__global__ void __launch_bounds__(kThreads) swin_attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ table,
                                                                  int H, int W, int heads, int sy, int sx, __nv_bfloat16* __restrict__ o,
                                                                  float* __restrict__ lse) {
  __shared__ __align__(16) FwdSmem sm;
  const int h = blockIdx.y, C = heads * kHd;
  const Window win(blockIdx.x, H, W, sy, sx);
  if (threadIdx.x < kRows) {
    sm.rows[threadIdx.x] = threadIdx.x < kTok ? win.row(threadIdx.x) : 0;
    sm.info[threadIdx.x] = win.info(threadIdx.x);
  }
  for (int i = threadIdx.x; i < kBins; i += kThreads) sm.tbl[i] = table[i * heads + h];
  __syncthreads();
  stage(qkv, (size_t)3 * C, h * kHd, C, 3, sm.rows, sm.q);                // q, k, v are consecutive
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, m0 = 16 * warp;
  float s[8][4];
  mma_abt(s, sm.q, sm.k, m0, g, t);
  bias_mask(s, sm.tbl, sm.info, m0, g, t);
  float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mx[0] = fmaxf(mx[0], fmaxf(s[j][0], s[j][1]));
    mx[1] = fmaxf(mx[1], fmaxf(s[j][2], s[j][3]));
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
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
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  float acc[4][4];
  mma_pb(acc, s, sm.v, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    if (i >= kTok) continue;
    const float inv = 1.f / l[r];
    __nv_bfloat16* dst = o + (size_t)sm.rows[i] * C + h * kHd + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
    if (t == 0) lse[(size_t)sm.rows[i] * heads + h] = mx[r] + logf(l[r]);
  }
}

struct BwdSmem {
  __nv_bfloat16 q[kRows * kPitch], k[kRows * kPitch], v[kRows * kPitch], dout[kRows * kPitch];
  __nv_bfloat16 p[kRows * kPPitch], ds[kRows * kPPitch];   // [query][key]; p first holds the staged O rows (pitch kPitch)
  float dsf[kTok * kTok];                                 // fp32 dS of the real tokens, for the table gradient
  float tbl[kBins];
  int rows[kRows], info[kRows];
};

__global__ void __launch_bounds__(kThreads) swin_attn_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ qkv,
                                                                  const __nv_bfloat16* __restrict__ o, const float* __restrict__ lse,
                                                                  const float* __restrict__ table, int H, int W, int heads, int sy, int sx,
                                                                  __nv_bfloat16* __restrict__ dqkv, float* __restrict__ part) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdSmem& sm = *reinterpret_cast<BwdSmem*>(smem_raw);
  const int h = blockIdx.y, C = heads * kHd;
  const Window win(blockIdx.x, H, W, sy, sx);
  if (threadIdx.x < kRows) {
    sm.rows[threadIdx.x] = threadIdx.x < kTok ? win.row(threadIdx.x) : 0;
    sm.info[threadIdx.x] = win.info(threadIdx.x);
  }
  for (int i = threadIdx.x; i < kBins; i += kThreads) sm.tbl[i] = table[i * heads + h];
  __syncthreads();
  // O goes to the P area with pitch kPitch for the row sums D; the warp that owns a query row reads it and later writes P there
  stage(qkv, (size_t)3 * C, h * kHd, C, 3, sm.rows, sm.q);                // q, k, v are consecutive
  stage(dout, C, h * kHd, 0, 1, sm.rows, sm.dout);
  stage(o, C, h * kHd, 0, 1, sm.rows, sm.p);
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, m0 = 16 * warp;
  float D[2], lr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    float a[8], b[8], sum = 0.f;
    unpack8(*reinterpret_cast<const Bf16x8*>(sm.dout + i * kPitch + 8 * t), a);
    unpack8(*reinterpret_cast<const Bf16x8*>(sm.p + i * kPitch + 8 * t), b);
#pragma unroll
    for (int u = 0; u < 8; ++u) sum = fmaf(a[u], b[u], sum);
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    D[r] = sum;
    lr[r] = i < kTok ? lse[(size_t)sm.rows[i] * heads + h] : INFINITY;   // padding query rows get P = 0
  }
  __syncthreads();                                                      // every O row is read before P overwrites them

  float s[8][4], dp[8][4];
  mma_abt(s, sm.q, sm.k, m0, g, t);
  mma_abt(dp, sm.dout, sm.v, m0, g, t);
  bias_mask(s, sm.tbl, sm.info, m0, g, t);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = e >> 1;
      const float p = exp2f((s[j][e] - lr[r]) * kLog2e);
      s[j][e] = p;
      dp[j][e] = p * (dp[j][e] - D[r]);                                 // dS
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = m0 + g + 8 * r, key = 8 * j + 2 * t;
      *reinterpret_cast<uint32_t*>(sm.p + i * kPPitch + key) = pack2(s[j][2 * r], s[j][2 * r + 1]);
      *reinterpret_cast<uint32_t*>(sm.ds + i * kPPitch + key) = pack2(dp[j][2 * r], dp[j][2 * r + 1]);
      if (i < kTok) {
        if (key < kTok) sm.dsf[i * kTok + key] = dp[j][2 * r];
        if (key + 1 < kTok) sm.dsf[i * kTok + key + 1] = dp[j][2 * r + 1];
      }
    }
  }
  const size_t pitch = (size_t)3 * C;
  float acc[4][4];
  mma_pb(acc, dp, sm.k, lane);                                          // dQ = dS K
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    if (i >= kTok) continue;
    __nv_bfloat16* dst = dqkv + (size_t)sm.rows[i] * pitch + h * kHd + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r] * kScale, acc[j][2 * r + 1] * kScale);
  }
  __syncthreads();

  // warp w now owns key rows [16 w, 16 w + 16)
  mma_atb(acc, sm.ds, sm.q, m0, lane);                                  // dK = dS^T Q
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    if (i >= kTok) continue;
    __nv_bfloat16* dst = dqkv + (size_t)sm.rows[i] * pitch + C + h * kHd + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r] * kScale, acc[j][2 * r + 1] * kScale);
  }
  mma_atb(acc, sm.p, sm.dout, m0, lane);                                // dV = P^T dO
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    if (i >= kTok) continue;
    __nv_bfloat16* dst = dqkv + (size_t)sm.rows[i] * pitch + 2 * C + h * kHd + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r], acc[j][2 * r + 1]);
  }

  // bin (dy, dx) = sum of dS_ij over the pairs with yi - yj = dy, xi - xj = dx, i in raster order
  for (int bin = threadIdx.x; bin < kBins; bin += kThreads) {
    const int dy = bin / 13 - 6, dx = bin % 13 - 6;
    float sum = 0.f;
    for (int yi = max(0, dy); yi < min(kWin, kWin + dy); ++yi)
      for (int xi = max(0, dx); xi < min(kWin, kWin + dx); ++xi)
        sum += sm.dsf[(yi * kWin + xi) * kTok + (yi - dy) * kWin + (xi - dx)];
    part[((size_t)h * gridDim.x + blockIdx.x) * kBins + bin] = sum;
  }
}

// dtable[bin, h] = the window partials part[h][w][bin] summed in window order: warp k of the CTA adds windows k, k + 32,
// ... for the 32 bins of its lanes, and warp 0 then adds the 32 warp sums in warp order
// (The body of both finish kernels: part [heads][windows][Cols] -> dtable [Cols, heads].)
template <int Cols>
__device__ __forceinline__ void table_grad_finish(const float* __restrict__ part, int windows, int heads, float* __restrict__ dtable) {
  __shared__ float red[kFinishWarps][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, h = blockIdx.y;
  const int bin = blockIdx.x * 32 + lane;
  float sum = 0.f;
  if (bin < Cols) {
    const float* p = part + (size_t)h * windows * Cols + bin;
#pragma unroll 4
    for (int w = warp; w < windows; w += kFinishWarps) sum += p[(size_t)w * Cols];
  }
  red[warp][lane] = sum;
  __syncthreads();
  if (warp != 0 || bin >= Cols) return;
  float total = 0.f;
#pragma unroll
  for (int k = 0; k < kFinishWarps; ++k) total += red[k][lane];
  dtable[bin * heads + h] = total;
}

__global__ void __launch_bounds__(kFinishWarps * 32) swin_table_grad_finish_kernel(const float* __restrict__ part, int windows, int heads,
                                                                                  float* __restrict__ dtable) {
  table_grad_finish<kBins>(part, windows, heads, dtable);
}

// ---- Swin V2: window 8, cosine scores ---------------------------------------------------------------------------------
// 64 tokens per window, exactly kRows, so no row is padded; 225 bins, entry (dy + 7) * 15 + (dx + 7).  The score is
//   s_ij = scale_h (q^_i . k^_j) + table[bin, h] + m_ij,   x^ = x / max(||x||, 1e-12) rounded once to bf16,
// with scale_h = exp(min(logit_scale_h, log 100)) and table = 16 sigmoid(cpb_mlp(...)) finished in torch.  The backward
// adds dcos = scale_h dS (rounded to bf16 for the MMAs, as V1 rounds dS), dq^ = dcos k^ and dk^ = dcos^T q^ in fp32, and
// projects them back through the normalisation: dq = (dq^ - q^ (q^ . dq^)) / max(||q||, 1e-12) (no projection below
// 1e-12, where the clamp passes no gradient to the norm).  Each CTA's partial row gains column 225, sum_ij dS_ij cos_ij,
// which the finish kernel sums in window order into d scale_h.
constexpr int kWin2 = 8, kTok2 = 64, kBins2 = 225, kCols2 = kBins2 + 1;
constexpr float kNormEps = 1e-12f;
static_assert(kTok2 == kRows && kThreads == 2 * kRows, "one V2 window fills the 64 staged rows; one thread per q / k row");

// the 64 q rows and the 64 k rows staged consecutively at qk, each divided by max(norm, 1e-12) and rounded once to bf16 in
// place; norm[r] = the fp32 norm of row r's 32 bf16 values (summed in column order), q rows first
__device__ __forceinline__ void normalize_rows(__nv_bfloat16* qk, float* norm) {
  __nv_bfloat16* row = qk + threadIdx.x * kPitch;
  float f[kHd];
#pragma unroll
  for (int c = 0; c < kHd / 8; ++c) unpack8(*reinterpret_cast<const Bf16x8*>(row + 8 * c), f + 8 * c);
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < kHd; ++c) ss = fmaf(f[c], f[c], ss);
  const float n = sqrtf(ss), d = fmaxf(n, kNormEps);
#pragma unroll
  for (int c = 0; c < kHd; ++c) f[c] = f[c] / d;
#pragma unroll
  for (int c = 0; c < kHd / 8; ++c) *reinterpret_cast<Bf16x8*>(row + 8 * c) = pack8(f + 8 * c);
  norm[threadIdx.x] = n;
}

// dx = (dx^ - x^ (x^ . dx^)) / max(||x||, 1e-12) for this lane's rows m0 + g (+ 8) of the fp32 fragment acc (columns
// 8 j + 2 t (+ 1)), x^ the staged normalised rows and norm their norms; stored as bf16 at dst + rows[i] pitch
__device__ __forceinline__ void unnormalize_store(const float (&acc)[4][4], const __nv_bfloat16* xh, const float* norm, const int* rows,
                                                  int m0, int g, int t, size_t pitch, __nv_bfloat16* __restrict__ dst) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    float x[8], dot = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(xh + i * kPitch + 8 * j + 2 * t);
      x[2 * j] = __low2float(v);
      x[2 * j + 1] = __high2float(v);
      dot = fmaf(x[2 * j], acc[j][2 * r], dot);
      dot = fmaf(x[2 * j + 1], acc[j][2 * r + 1], dot);
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    const float n = norm[i], d = fmaxf(n, kNormEps);
    if (!(n >= kNormEps)) dot = 0.f;
    __nv_bfloat16* out = dst + (size_t)rows[i] * pitch + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint32_t*>(out + 8 * j) = pack2((acc[j][2 * r] - x[2 * j] * dot) / d, (acc[j][2 * r + 1] - x[2 * j + 1] * dot) / d);
  }
}

struct V2FwdSmem {
  __nv_bfloat16 q[kRows * kPitch], k[kRows * kPitch], v[kRows * kPitch];
  float tbl[kBins2];
  float norm[2 * kRows];
  int rows[kRows], info[kRows];
};

__global__ void __launch_bounds__(kThreads) swin_v2_attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ table,
                                                                     const float* __restrict__ scale, int H, int W, int heads, int sy, int sx,
                                                                     __nv_bfloat16* __restrict__ o, float* __restrict__ lse) {
  __shared__ __align__(16) V2FwdSmem sm;
  const int h = blockIdx.y, C = heads * kHd;
  const WindowOf<kWin2> win(blockIdx.x, H, W, sy, sx);
  if (threadIdx.x < kRows) {
    sm.rows[threadIdx.x] = win.row(threadIdx.x);
    sm.info[threadIdx.x] = win.info(threadIdx.x);
  }
  for (int i = threadIdx.x; i < kBins2; i += kThreads) sm.tbl[i] = table[i * heads + h];
  const float sc = scale[h];
  __syncthreads();
  stage<kTok2>(qkv, (size_t)3 * C, h * kHd, C, 3, sm.rows, sm.q);         // q, k, v are consecutive
  __syncthreads();
  normalize_rows(sm.q, sm.norm);
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, m0 = 16 * warp;
  float s[8][4];
  mma_abt(s, sm.q, sm.k, m0, g, t);
  bias_mask<kWin2>(s, sm.tbl, sm.info, m0, g, t, sc);
  float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mx[0] = fmaxf(mx[0], fmaxf(s[j][0], s[j][1]));
    mx[1] = fmaxf(mx[1], fmaxf(s[j][2], s[j][3]));
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
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
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  float acc[4][4];
  mma_pb(acc, s, sm.v, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    const float inv = 1.f / l[r];
    __nv_bfloat16* dst = o + (size_t)sm.rows[i] * C + h * kHd + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
    if (t == 0) lse[(size_t)sm.rows[i] * heads + h] = mx[r] + logf(l[r]);
  }
}

struct V2BwdSmem {
  __nv_bfloat16 q[kRows * kPitch], k[kRows * kPitch], v[kRows * kPitch], dout[kRows * kPitch];
  __nv_bfloat16 p[kRows * kPPitch], ds[kRows * kPPitch];   // [query][key]; p first holds the staged O rows (pitch kPitch),
                                                          // ds holds bf16(dcos) = bf16(scale dS)
  float dsf[kTok2 * kTok2];                               // fp32 dS, for the table gradient
  float tbl[kBins2];
  float norm[2 * kRows];
  float cos_part[kThreads / 32];                          // each warp's sum of dS cos
  int rows[kRows], info[kRows];
};

__global__ void __launch_bounds__(kThreads) swin_v2_attn_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ qkv,
                                                                     const __nv_bfloat16* __restrict__ o, const float* __restrict__ lse,
                                                                     const float* __restrict__ table, const float* __restrict__ scale, int H,
                                                                     int W, int heads, int sy, int sx, __nv_bfloat16* __restrict__ dqkv,
                                                                     float* __restrict__ part) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  V2BwdSmem& sm = *reinterpret_cast<V2BwdSmem*>(smem_raw);
  const int h = blockIdx.y, C = heads * kHd;
  const WindowOf<kWin2> win(blockIdx.x, H, W, sy, sx);
  if (threadIdx.x < kRows) {
    sm.rows[threadIdx.x] = win.row(threadIdx.x);
    sm.info[threadIdx.x] = win.info(threadIdx.x);
  }
  for (int i = threadIdx.x; i < kBins2; i += kThreads) sm.tbl[i] = table[i * heads + h];
  const float sc = scale[h];
  __syncthreads();
  stage<kTok2>(qkv, (size_t)3 * C, h * kHd, C, 3, sm.rows, sm.q);         // q, k, v are consecutive
  stage<kTok2>(dout, C, h * kHd, 0, 1, sm.rows, sm.dout);
  stage<kTok2>(o, C, h * kHd, 0, 1, sm.rows, sm.p);
  __syncthreads();
  normalize_rows(sm.q, sm.norm);                                          // bitwise the forward's q^ and k^

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, m0 = 16 * warp;
  float D[2], lr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    float a[8], b[8], sum = 0.f;
    unpack8(*reinterpret_cast<const Bf16x8*>(sm.dout + i * kPitch + 8 * t), a);
    unpack8(*reinterpret_cast<const Bf16x8*>(sm.p + i * kPitch + 8 * t), b);
#pragma unroll
    for (int u = 0; u < 8; ++u) sum = fmaf(a[u], b[u], sum);
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    D[r] = sum;
    lr[r] = lse[(size_t)sm.rows[i] * heads + h];
  }
  __syncthreads();                                                      // q^, k^ written; every O row read before P overwrites them

  float s[8][4], dp[8][4], cs[8][4];
  mma_abt(s, sm.q, sm.k, m0, g, t);
  mma_abt(dp, sm.dout, sm.v, m0, g, t);
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) cs[j][e] = s[j][e];                     // cos = q^ . k^
  bias_mask<kWin2>(s, sm.tbl, sm.info, m0, g, t, sc);
  float dsc = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = e >> 1;
      const float p = exp2f((s[j][e] - lr[r]) * kLog2e);
      s[j][e] = p;
      dp[j][e] = p * (dp[j][e] - D[r]);                                 // dS
      dsc = fmaf(dp[j][e], cs[j][e], dsc);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = m0 + g + 8 * r, key = 8 * j + 2 * t;
      *reinterpret_cast<float2*>(sm.dsf + i * kTok2 + key) = make_float2(dp[j][2 * r], dp[j][2 * r + 1]);
      dp[j][2 * r] *= sc;                                               // dcos
      dp[j][2 * r + 1] *= sc;
      *reinterpret_cast<uint32_t*>(sm.p + i * kPPitch + key) = pack2(s[j][2 * r], s[j][2 * r + 1]);
      *reinterpret_cast<uint32_t*>(sm.ds + i * kPPitch + key) = pack2(dp[j][2 * r], dp[j][2 * r + 1]);
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) dsc += __shfl_xor_sync(0xffffffffu, dsc, m);
  if (lane == 0) sm.cos_part[warp] = dsc;
  const size_t pitch = (size_t)3 * C;
  float acc[4][4];
  mma_pb(acc, dp, sm.k, lane);                                          // dq^ = dcos k^
  unnormalize_store(acc, sm.q, sm.norm, sm.rows, m0, g, t, pitch, dqkv + h * kHd);
  __syncthreads();

  // warp w now owns key rows [16 w, 16 w + 16)
  mma_atb(acc, sm.ds, sm.q, m0, lane);                                  // dk^ = dcos^T q^
  unnormalize_store(acc, sm.k, sm.norm + kRows, sm.rows, m0, g, t, pitch, dqkv + C + h * kHd);
  mma_atb(acc, sm.p, sm.dout, m0, lane);                                // dV = P^T dO
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = m0 + g + 8 * r;
    __nv_bfloat16* dst = dqkv + (size_t)sm.rows[i] * pitch + 2 * C + h * kHd + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(acc[j][2 * r], acc[j][2 * r + 1]);
  }

  // bin (dy, dx) = sum of dS_ij over the pairs with yi - yj = dy, xi - xj = dx, i in raster order; column 225 the four warp
  // sums of dS cos in warp order
  float* out = part + ((size_t)h * gridDim.x + blockIdx.x) * kCols2;
  for (int bin = threadIdx.x; bin < kBins2; bin += kThreads) {
    const int dy = bin / 15 - 7, dx = bin % 15 - 7;
    float sum = 0.f;
    for (int yi = max(0, dy); yi < min(kWin2, kWin2 + dy); ++yi)
      for (int xi = max(0, dx); xi < min(kWin2, kWin2 + dx); ++xi)
        sum += sm.dsf[(yi * kWin2 + xi) * kTok2 + (yi - dy) * kWin2 + (xi - dx)];
    out[bin] = sum;
  }
  if (threadIdx.x == 0) out[kBins2] = ((sm.cos_part[0] + sm.cos_part[1]) + sm.cos_part[2]) + sm.cos_part[3];
}

__global__ void __launch_bounds__(kFinishWarps * 32) swin_v2_grad_finish_kernel(const float* __restrict__ part, int windows, int heads,
                                                                               float* __restrict__ dtable) {
  table_grad_finish<kCols2>(part, windows, heads, dtable);
}

template <int Win>
void check_swin_shape(const char* who, int B, int H, int W, int heads, int sy, int sx) {
  if (B < 1 || H < Win || W < Win || H % Win || W % Win || heads < 1 || heads > 65535 || sy < 0 || sy >= Win || sx < 0 || sx >= Win)
    throw std::runtime_error(std::string(who) + ": needs B, heads >= 1, H and W positive multiples of " + std::to_string(Win) +
                             " and 0 <= shift < " + std::to_string(Win) + " (got B=" +
                             std::to_string(B) + ", H=" + std::to_string(H) + ", W=" + std::to_string(W) + ", heads=" +
                             std::to_string(heads) + ", shift=(" + std::to_string(sy) + ", " + std::to_string(sx) + "))");
  if ((long long)B * H * W * 3 * heads * kHd >= (1ll << 31)) throw std::runtime_error(std::string(who) + ": problem too large");
}

}  // namespace

int swin_windows(int B, int H, int W) { return B * (H / kWin) * (W / kWin); }

void launch_swin_attention_fwd(const void* qkv, const float* table, int B, int H, int W, int heads, int sy, int sx, void* o, float* lse,
                               cudaStream_t s) {
  check_swin_shape<kWin>("swin_attention_fwd", B, H, W, heads, sy, sx);
  swin_attn_fwd_kernel<<<dim3(swin_windows(B, H, W), heads), kThreads, 0, s>>>((const __nv_bfloat16*)qkv, table, H, W, heads, sy, sx,
                                                                               (__nv_bfloat16*)o, lse);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_swin_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const float* table, int B, int H, int W,
                               int heads, int sy, int sx, void* dqkv, float* part, float* dtable, cudaStream_t s) {
  check_swin_shape<kWin>("swin_attention_bwd", B, H, W, heads, sy, sx);
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(swin_attn_bwd_kernel, (int)sizeof(BwdSmem), configured);
  const int windows = swin_windows(B, H, W);
  swin_attn_bwd_kernel<<<dim3(windows, heads), kThreads, sizeof(BwdSmem), s>>>(
      (const __nv_bfloat16*)dout, (const __nv_bfloat16*)qkv, (const __nv_bfloat16*)o, lse, table, H, W, heads, sy, sx,
      (__nv_bfloat16*)dqkv, part);
  B200_CUDA_CHECK(cudaGetLastError());
  swin_table_grad_finish_kernel<<<dim3(ceil_div(kBins, 32), heads), kFinishWarps * 32, 0, s>>>(part, windows, heads, dtable);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

int swin_v2_windows(int B, int H, int W) { return B * (H / kWin2) * (W / kWin2); }

void launch_swin_v2_attention_fwd(const void* qkv, const float* table, const float* scale, int B, int H, int W, int heads, int sy, int sx,
                                  void* o, float* lse, cudaStream_t s) {
  check_swin_shape<kWin2>("swin_v2_attention_fwd", B, H, W, heads, sy, sx);
  swin_v2_attn_fwd_kernel<<<dim3(swin_v2_windows(B, H, W), heads), kThreads, 0, s>>>((const __nv_bfloat16*)qkv, table, scale, H, W, heads,
                                                                                     sy, sx, (__nv_bfloat16*)o, lse);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_swin_v2_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const float* table, const float* scale,
                                  int B, int H, int W, int heads, int sy, int sx, void* dqkv, float* part, float* dtable, cudaStream_t s) {
  check_swin_shape<kWin2>("swin_v2_attention_bwd", B, H, W, heads, sy, sx);
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(swin_v2_attn_bwd_kernel, (int)sizeof(V2BwdSmem), configured);
  const int windows = swin_v2_windows(B, H, W);
  swin_v2_attn_bwd_kernel<<<dim3(windows, heads), kThreads, sizeof(V2BwdSmem), s>>>(
      (const __nv_bfloat16*)dout, (const __nv_bfloat16*)qkv, (const __nv_bfloat16*)o, lse, table, scale, H, W, heads, sy, sx,
      (__nv_bfloat16*)dqkv, part);
  B200_CUDA_CHECK(cudaGetLastError());
  swin_v2_grad_finish_kernel<<<dim3(ceil_div(kCols2, 32), heads), kFinishWarps * 32, 0, s>>>(part, windows, heads, dtable);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

}  // namespace b200
