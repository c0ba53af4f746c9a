// bf16 GEMM on the Hopper tensor cores (replacement for the cuBLASLt calls behind nn.Linear forward / dgrad / wgrad).
//
//   D[M,N] = epilogue( sum_k A[m,k] * B[n,k] )        fp32 accumulation in registers
//
// Hand-written for sm_90a: one TMA producer warp stages 128B-swizzled operand tiles into a ring of shared-memory stages
// (mbarrier full / empty pairs); one warpgroup (warps 4-7) issues wgmma (m64 x BLOCK_N x k16, two per k step for the
// 128-row tile) with fp32 accumulators in registers, then copies the accumulator tile to shared memory so that each
// epilogue thread owns one output row: bias / ReLU / GELU / column statistics and the bf16 or fp32 stores work on whole
// rows.  Persistent: one CTA per SM walks tiles m-fastest so CTAs running concurrently share the same B tile in L2, and
// the producer prefetches the next tile while the warpgroup runs the epilogue.
//
// Operand majorness (so backward needs no transposes):
//   A "K-major"  : A stored [M, K] row-major   (forward x, dgrad dy)
//   A "MN-major" : A stored [K, M] row-major   (wgrad: dy^T)
//   B "K-major"  : B stored [N, K] row-major   (forward W)
//   B "MN-major" : B stored [K, N] row-major   (dgrad W, wgrad x)
//
// FP8 variants (OP != 0): 8-bit operands, K-major only (the only layout FP8 wgmma accepts), 128-element k-blocks (still
// 128 bytes per row, so the swizzle, the TMA boxes in bytes and the descriptor stepping are those of bf16) and k32
// steps.  Each k-block's four k32 steps accumulate into a fresh register tile that is then added to an fp32 tile: FP8
// wgmma keeps fewer accumulator bits than fp32, and promoting every 128 products bounds the loss at large K.  The
// epilogue multiplies by the device-resident dequantisation factors 1/s_a * 1/s_b before bias / activation / store.
#include "gemm.h"

#include <cuda.h>
#include <cstdlib>

#include "tc_primitives.cuh"
#include "tensor_map.h"

namespace b200 {
namespace {
using namespace tc;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int UMMA_K = 16;
constexpr int kOpBF16 = 0, kOpE4M3 = 1, kOpE5M2 = 2;   // operand types: bf16 x bf16, e4m3 x e4m3, e5m2 x e4m3
constexpr int kNumEpilogueWarps = 4;
constexpr int kNumThreads = 128 + kNumEpilogueWarps * 32;   // warp 0: TMA producer, warps 1..3 idle; warps 4..7: MMA + epilogue

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

struct GemmParams {
  int M, N, K;
  int epilogue;           // 0 none, 1 +bias, 2 +bias,relu, 3 +bias,gelu(erf)
  int out_fp32;
  int accumulate;         // D += result (fp32 output only; gradient accumulation)
  int group_m;            // tile rasterisation, see gemm_tile_coords
  int stat_groups;        // ceil(M / 32): row groups of the column-statistics workspace
  float* col_stats;       // [2][stat_groups][N] per-32-row partial column sums / sums of squares of the stored output, or nullptr
  void* d;
  const __nv_bfloat16* bias;
  // FP8 only: device scalars 1/s_a, 1/s_b (dequantisation factors).  The row-bounded bf16 modes (kBoundRows, kBoundK)
  // never dequantise, so their device row count `bound_rows` shares scale_a's bytes.
  union { const float* scale_a; const int* bound_rows; };
  const float* scale_b;
  // fused LM-head cross-entropy (LM != kLmNone).  Appended after the fields above so that their offsets stay as they
  // were, and kept to 56 bytes: at 128 bytes or less the struct's parameter loads, and the code of every other variant,
  // compile as before.  kLmLse writes its (max, sum exp) partials to `d` (it stores no output tile).
  // The grouped expert GEMMs (GRP != kGrpNone) never run an LM-head epilogue, so their four fields (grp_*) share these bytes:
  //   grp_tile_expert  kGrpRows: [M / 128] expert of each 128-row tile of A and D, -1 = unused (skipped)
  //   grp_offsets      kGrpWgrad: [E + 1] start row of each expert's 128-aligned segment of A and B
  //   grp_rows         kGrpRows: B rows per expert (expert e's B starts at row e * grp_rows of its 2-D view);
  //                    kGrpWgrad: output rows per expert (D is [E * grp_rows, N])
  //   grp_experts      kGrpWgrad: E
  union { const long long* lm_targets; const int* grp_tile_expert; };   // [M] target column of each row (global vocabulary index)
  float* lm_target_logit;        // kLmLse: [M] the row's target logit, written by the one tile that holds it
  union { const float* lm_lse; const int* grp_offsets; };              // kLmDlogits: [M] row log-sum-exp
  const float* lm_gscale;        // kLmDlogits: device scalars, upstream gradient and number of non-ignored rows
  const float* lm_valid;
  int lm_ignore_index;           // kLmDlogits: ignore_index if it lies in [0, lm_vocab), else -1 (already ignored as out of range)
  union { int lm_col_offset; int grp_rows; };                          // kLmDlogits: global vocabulary index of this GEMM's column 0
  union { int lm_vocab; int grp_experts; };                            // full vocabulary: targets outside [0, lm_vocab) are ignored
};

constexpr int kLmNone = 0, kLmLse = 1, kLmDlogits = 2;
// Grouped (mixture-of-experts) modes.  kGrpRows: forward / data gradient, A's rows are sorted by expert in 128-aligned
// segments, so every 128-row tile multiplies one expert's B.  kGrpWgrad: D_e = A_e^T B_e per expert e, both operands
// MN-major, the k-loop running over expert e's segment only.
constexpr int kGrpNone = 0, kGrpRows = 1, kGrpWgrad = 2;
// Row-bounded modes, the same tile-schedule slot: only the first *bound_rows rows of A (a device count, so the host never
// reads it back) carry data.  kBoundRows (A K-major): the schedule walks the 128-row tiles below the count only, so no CTA
// waits on skipped tiles; D's rows in skipped tiles are not written.  kBoundK (A and B MN-major, the token dimension as K):
// the k-loop stops at the count rounded up to the k-block; an empty loop stores zeros.
constexpr int kBoundRows = 3, kBoundK = 4;

// bias / activation on 32 consecutive accumulator columns starting at `col0`
__device__ __forceinline__ void epilogue_math(const GemmParams& p, int col0, const uint32_t* r, float* v) {
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
  if (p.epilogue >= 1 && p.bias != nullptr) {
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (col0 + i < p.N) v[i] += __bfloat162float(p.bias[col0 + i]);
  }
  if (p.epilogue == 2) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
  } else if (p.epilogue == 3) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
  }
}

// Column statistics of the producing GEMM (opt-in: BatchNorm statistics of a 1x1 convolution's output without
// re-reading it).  A warp holds a 32-row x 32-column block, one row per lane.  Butterfly "transpose-reduce": in each
// of 5 steps a lane keeps half of its columns and receives the partner's partial sums for them, so after 31 shuffles
// lane l owns the sum over the 32 rows of column l.  Values are rounded to bf16 first (the statistics describe the
// tensor as stored); rows beyond M contribute zero.  Deterministic: no atomics, one writer per workspace element.
__device__ __forceinline__ float warp_column_sum(float* t, int lane) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const float keep = upper ? t[i + off] : t[i];
      const float send = upper ? t[i] : t[i + off];
      t[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return t[0];
}

__device__ __forceinline__ void column_stats_chunk(const GemmParams& p, int row, int row0, int col0, const float* v, int lane) {
  float s[32], q[32];
  const bool live = row < p.M;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float r = p.out_fp32 ? v[i] : __bfloat162float(__float2bfloat16_rn(v[i]));
    s[i] = live ? r : 0.f;
    q[i] = s[i] * s[i];
  }
  const float cs = warp_column_sum(s, lane);
  const float cq = warp_column_sum(q, lane);
  const int col = col0 + lane;
  if (col < p.N && row0 < p.M) {
    const size_t g = (size_t)(row0 >> 5);
    p.col_stats[(g) * p.N + col] = cs;
    p.col_stats[((size_t)p.stat_groups + g) * p.N + col] = cq;
  }
}

// Epilogue for one accumulator row chunk: 32 consecutive columns of row `row` starting at `col0`.
__device__ __forceinline__ void store_row_chunk(const GemmParams& p, int row, int col0, const uint32_t* r) {
  if (row < p.M && col0 < p.N) {
    float v[32];
    epilogue_math(p, col0, r, v);
    const bool full = (col0 + 32 <= p.N);
    if (p.out_fp32) {
      float* out = reinterpret_cast<float*>(p.d) + (size_t)row * p.N + col0;
      if (full && ((reinterpret_cast<uintptr_t>(out) & 15) == 0)) {
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          float4 o = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
          if (p.accumulate) { const float4 old = *reinterpret_cast<float4*>(out + i); o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w; }
          *reinterpret_cast<float4*>(out + i) = o;
        }
      } else {
        for (int i = 0; i < 32; ++i)
          if (col0 + i < p.N) out[i] = p.accumulate ? out[i] + v[i] : v[i];
      }
    } else {
      __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.d) + (size_t)row * p.N + col0;
      if (full && ((reinterpret_cast<uintptr_t>(out) & 15) == 0)) {
#pragma unroll
        for (int i = 0; i < 32; i += 8) {
          __nv_bfloat162 h[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(v[i + 2 * q], v[i + 2 * q + 1]);
          *reinterpret_cast<uint4*>(out + i) = *reinterpret_cast<uint4*>(h);
        }
      } else {
        for (int i = 0; i < 32; ++i)
          if (col0 + i < p.N) out[i] = __float2bfloat16_rn(v[i]);
      }
    }
  }
}

// ---- fused LM-head cross-entropy epilogues (128-column tiles, one thread per row) -----------------------------
// The logits are never stored.  Each value is biased and rounded to bf16 first, exactly as the unfused head GEMM
// stores it, so both paths see the same logits.  The target column is found by comparing every column index with it
// (a select per column: no dynamic register indexing).
//   kLmLse     : (max, sum exp(x - max)) of the row over the tile -> d as float2 [ceil(N / 128)][M], the target logit ->
//                lm_target_logit.
//   kLmDlogits : d = (exp(x - lse) - [col == target]) * g / valid in bf16 -> D; ignored rows get zeros.
template <int LM>
__device__ __forceinline__ void lm_epilogue_tile(const GemmParams& p, const float* arow, int row, int n0) {
  const bool live = row < p.M;
  const long long t = live ? __ldg(p.lm_targets + row) : -1;
  if constexpr (LM == kLmLse) {
    const int tcol = (t >= n0 && t < n0 + 128 && t < p.N) ? (int)(t - n0) : -1;
    float m = -INFINITY, s = 0.f, tl = 0.f;
#pragma unroll 1
    for (int c = 0; c < 128; c += 32) {
      if (n0 + c >= p.N) break;                          // warp-uniform
      uint32_t r[32];
      float v[32];
      acc_row_ld32(arow, 0, 0, c, r);
      epilogue_math(p, n0 + c, r, v);
      float cm = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float x = n0 + c + i < p.N ? __bfloat162float(__float2bfloat16_rn(v[i])) : -INFINITY;
        if (tcol == c + i) tl = x;
        v[i] = x;
        cm = fmaxf(cm, x);
      }
      const float nm = fmaxf(m, cm);
      float cs = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) cs += __expf(v[i] - nm);
      s = s * __expf(m - nm) + cs;                       // first chunk: m = -inf, s = 0
      m = nm;
    }
    if (live) {
      reinterpret_cast<float2*>(p.d)[(size_t)(n0 / 128) * p.M + row] = make_float2(m, s);
      if (tcol >= 0) p.lm_target_logit[row] = tl;
    }
  } else {
    const bool ignored = t == p.lm_ignore_index || t < 0 || t >= p.lm_vocab;
    const long long base = (long long)p.lm_col_offset + n0;
    const int tcol = (!ignored && t >= base && t < base + 128) ? (int)(t - base) : -1;
    const float valid = __ldg(p.lm_valid);
    const float coef = (ignored || valid <= 0.f) ? 0.f : __ldg(p.lm_gscale) / valid;
    const float lse = live ? p.lm_lse[row] : 0.f;
#pragma unroll 1
    for (int c = 0; c < 128; c += 32) {
      if (n0 + c >= p.N) break;                          // warp-uniform
      uint32_t r[32];
      float v[32];
      acc_row_ld32(arow, 0, 0, c, r);
      epilogue_math(p, n0 + c, r, v);
      // A row without a gradient (ignored, no valid row, or past a row-bounded count, whose lse reads 0) writes zeros
      // without its exponential: a logit above ~88.7 would make it inf, and inf * 0 = NaN.
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        float d = coef != 0.f ? __expf(__bfloat162float(__float2bfloat16_rn(v[i])) - lse) : 0.f;
        if (tcol == c + i) d -= 1.f;
        v[i] = d * coef;
      }
      if (!live) continue;
      const int col0 = n0 + c;
      __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.d) + (size_t)row * p.N + col0;
      if (col0 + 32 <= p.N && ((reinterpret_cast<uintptr_t>(out) & 15) == 0)) {
#pragma unroll
        for (int i = 0; i < 32; i += 8) {
          __nv_bfloat162 h[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(v[i + 2 * q], v[i + 2 * q + 1]);
          *reinterpret_cast<uint4*>(out + i) = *reinterpret_cast<uint4*>(h);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (col0 + i < p.N) out[i] = __float2bfloat16_rn(v[i]);
      }
    }
  }
}

// ---- opt-in epilogue through shared memory + TMA store (bf16 outputs) ---------------------------------------
// Each epilogue warp owns two 4 KB staging buffers (32 rows x 64 bf16 columns, 128B-swizzled exactly like the
// operand tiles).  A lane converts its accumulator row, writes eight 16-byte chunks at (chunk ^ (row & 7)) - bank
// conflict free - and lane 0 hands the slab to the TMA unit, which writes full 128-byte rows and clips the M / N
// edges.  The direct path instead issues 16-byte stores to 32 different rows per instruction.
constexpr int kStoreSlabBytes = 32 * 64 * 2;                       // 4 KB
constexpr int kStoreStageBytes = kNumEpilogueWarps * 2 * kStoreSlabBytes;   // 32 KB per CTA

// One warp drains its 32 accumulator rows x TILE_N columns.  `row0` = global row of lane 0, `slab` = running slab
// counter of this warp (selects the staging buffer; persists across tiles).
template <int TILE_N, bool STATS>
__device__ __forceinline__ void epilogue_tile_tma(const GemmParams& p, const CUtensorMap* map_d, uint8_t* stage, const float* arow,
                                                  int row0, int n0, int lane, uint32_t& slab) {
#pragma unroll 1
  for (int c = 0; c < TILE_N; c += 64) {
    if (n0 + c >= p.N) break;                       // warp-uniform: the rest of the tile is outside the matrix
    uint8_t* buf = stage + (slab & 1u) * kStoreSlabBytes;
    const uint32_t buf_s = smem_u32(buf);
    // the store that used this buffer two slabs ago must have finished reading it
    if (lane == 0) bulk_wait_read_le1();
    __syncwarp();
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      uint32_t r[32];
      float v[32];
      acc_row_ld32(arow, 0, 0, c + 32 * half, r);
      epilogue_math(p, n0 + c + 32 * half, r, v);
      if constexpr (STATS) column_stats_chunk(p, row0 + lane, row0, n0 + c + 32 * half, v, lane);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        __nv_bfloat162 h[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(v[8 * q + 2 * j], v[8 * q + 2 * j + 1]);
        const int chunk = half * 4 + q;              // 16-byte chunk index inside the 128-byte row
        const uint32_t* w = reinterpret_cast<const uint32_t*>(h);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                     ::"r"(buf_s + (uint32_t)(lane * 128 + ((chunk ^ (lane & 7)) << 4))), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
      }
    }
    fence_async_smem();                              // generic-proxy writes -> visible to the TMA (async proxy)
    __syncwarp();
    if (lane == 0 && row0 < p.M) {
      tma_store_2d(map_d, buf, n0 + c, row0);
      bulk_commit();
    }
    ++slab;
  }
}

// The scheduled tile's coordinates.  Grouped modes also give its expert `e`, its k-block range [kb0, kb1) and B's row
// offset; false = an unused tile of kGrpRows, which the producer and the MMA warpgroup both skip.
template <int GRP>
__device__ __forceinline__ bool grouped_tile(const GemmParams& p, int tile, int num_m, int num_n, int* mb,
                                             int* nb, int* e, int* kb0, int* kb1, int* b_off) {
  if constexpr (GRP == kGrpNone) {
    gemm_tile_coords(tile, num_m, num_n, p.group_m, mb, nb);
    return true;
  } else if constexpr (GRP == kGrpRows) {
    gemm_tile_coords(tile, num_m, num_n, 0, mb, nb);
    *e = __ldg(p.grp_tile_expert + *mb);
    *b_off = *e * p.grp_rows;
    return *e >= 0;
  } else if constexpr (GRP == kBoundRows) {                    // the live tiles are numbered first, m-fastest
    const int live_m = min(num_m, (__ldg(p.bound_rows) + BLOCK_M - 1) / BLOCK_M);
    if (tile >= live_m * num_n) return false;
    gemm_tile_coords(tile, live_m, num_n, 0, mb, nb);
    return true;
  } else if constexpr (GRP == kBoundK) {
    gemm_tile_coords(tile, num_m, num_n, 0, mb, nb);
    *kb1 = min(*kb1, (__ldg(p.bound_rows) + BLOCK_K - 1) / BLOCK_K);
    return true;
  } else {                                                     // expert-major: all tiles of expert 0, then expert 1, ...
    const int per_expert = num_m * num_n;
    *e = tile / per_expert;
    gemm_tile_coords(tile - *e * per_expert, num_m, num_n, 0, mb, nb);
    *kb0 = __ldg(p.grp_offsets + *e) / BLOCK_K;
    *kb1 = __ldg(p.grp_offsets + *e + 1) / BLOCK_K;
    return true;
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool TMA_ST>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarrierBytes = 1024;
  static constexpr int kAccStride = BLOCK_N + 8;                       // floats per accumulator row in shared memory
  static constexpr int kAccBytes = BLOCK_M * kAccStride * 4;
  static constexpr int kFixed = kBarrierBytes + (TMA_ST ? kStoreStageBytes : 0) + kAccBytes + 1024 /*alignment slack*/;
  static constexpr int kStages = (227 * 1024 - kFixed) / kStageBytes > 8 ? 8 : (227 * 1024 - kFixed) / kStageBytes;
  static constexpr int kTotal = kStages * kStageBytes + kFixed;
};

// PAIR: launched as clusters of two CTAs that compute vertically adjacent 128-row tiles of the same n-tile (a 256 x BLOCK_N
// pair tile).  Each CTA loads its own A tile and HALF of the B tile, multicast into both CTAs' shared memory, so every B
// byte leaves L2 once per pair.  A stage may be refilled only when the consumers of BOTH CTAs are done with it: the empty
// barriers count the arrivals of the local and the peer warpgroup.
template <int BLOCK_N, bool A_MN, bool B_MN, bool TMA_ST, bool STATS, bool PAIR, int OP = kOpBF16, int LM = kLmNone,
          int GRP = kGrpNone>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_d, const GemmParams p) {
  using L = SmemLayout<BLOCK_N, A_MN, B_MN, TMA_ST>;
  constexpr int kStages = L::kStages;
  constexpr bool kFP8 = OP != kOpBF16;
  static_assert(!kFP8 || (!A_MN && !B_MN && !TMA_ST && !STATS && !PAIR && BLOCK_N == 64),
                "FP8: K-major operands, direct epilogue, 128 x 64 tiles (partial + promoted accumulators fill the registers)");
  static_assert(sizeof(GemmParams) <= 128, "GemmParams: see the note on the LM-head fields");
  static_assert(LM == kLmNone || (!kFP8 && !A_MN && !B_MN && !TMA_ST && !STATS && !PAIR && BLOCK_N == 128),
                "LM-head epilogues: bf16 K-major operands, direct epilogue, single-CTA 128 x 128 tiles");
  static_assert(GRP == kGrpNone || GRP >= kBoundRows ||
                    (!kFP8 && LM == kLmNone && !TMA_ST && !STATS && !PAIR && BLOCK_N == 128 && (GRP == kGrpRows ? !A_MN : (A_MN && B_MN))),
                "grouped GEMMs: bf16, direct epilogue, single-CTA 128 x 128 tiles; A K-major (rows) or A and B MN-major (wgrad)");
  static_assert(GRP < kBoundRows || (!kFP8 && !TMA_ST && !STATS && !PAIR && BLOCK_N == 128 &&
                                     (GRP == kBoundRows ? !A_MN : (A_MN && B_MN && LM == kLmNone))),
                "row-bounded GEMMs: bf16, direct epilogue, single-CTA 128 x 128 tiles; A K-major (rows) or A and B MN-major (k)");
  constexpr int kBK = kFP8 ? 2 * BLOCK_K : BLOCK_K;            // elements per k-block: one 128-byte row either way
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* barrier_area = smem + kStages * L::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(barrier_area);
  uint64_t* empty_bar = full_bar + kStages;
  uint8_t* store_stage = barrier_area + L::kBarrierBytes;
  float* acc_smem = reinterpret_cast<float*>(store_stage + (TMA_ST ? kStoreStageBytes : 0));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kM = PAIR ? 2 * BLOCK_M : BLOCK_M;            // rows of a scheduled tile (a pair tile with PAIR)
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int first = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int stride = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const int num_m_blocks = ((GRP == kGrpWgrad ? p.grp_rows : p.M) + kM - 1) / kM;
  const int num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = num_m_blocks * num_n_blocks * (GRP == kGrpWgrad ? p.grp_experts : 1);
  const int num_k_blocks = (p.K + kBK - 1) / kBK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], (PAIR ? 2 : 1) * kNumEpilogueWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if constexpr (PAIR) cluster_sync_all();                      // the peer's barriers exist before anyone signals them

  if (warp == 0) {
    // ===================== TMA producer (one elected lane) =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = first; tile < num_tiles; tile += stride) {
        int mb, nb, e, kb0 = 0, kb1 = num_k_blocks, b_off = 0;
        if (!grouped_tile<GRP>(p, tile, num_m_blocks, num_n_blocks, &mb, &nb, &e, &kb0, &kb1, &b_off)) continue;
        const int m0 = mb * kM + (int)rank * BLOCK_M;            // rows past M arrive as zeros and are never stored
        const int n0 = nb * BLOCK_N;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes;
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          const int k0 = kb * kBK;
          if constexpr (!A_MN) {
            tma_load_2d(&map_a, &full_bar[stage], sa, k0, m0);                    // box {64 k, 128 m}
          } else {
#pragma unroll
            for (int c = 0; c < BLOCK_M / 64; ++c)                               // box {64 m, 64 k} per chunk
              tma_load_2d(&map_a, &full_bar[stage], sa + c * (64 * BLOCK_K * 2), m0 + 64 * c, k0);
          }
          if constexpr (PAIR) {
            static_assert(BLOCK_N == 128, "pair tiles are 128 wide: one 64-row half of B per CTA");
            constexpr int kHalfB = (BLOCK_N / 2) * BLOCK_K * 2;                   // 64 rows (K-major) / one 64-wide chunk (MN-major)
            if constexpr (!B_MN) tma_load_2d_multicast(&map_b, &full_bar[stage], sb + rank * kHalfB, k0, n0 + 64 * (int)rank, 0x3);
            else tma_load_2d_multicast(&map_b, &full_bar[stage], sb + rank * kHalfB, n0 + 64 * (int)rank, k0, 0x3);
          } else if constexpr (!B_MN) {
            tma_load_2d(&map_b, &full_bar[stage], sb, k0, n0 + b_off);            // box {64 k, BLOCK_N n}
          } else {
#pragma unroll
            for (int c = 0; c < BLOCK_N / 64; ++c)
              tma_load_2d(&map_b, &full_bar[stage], sb + c * (64 * BLOCK_K * 2), n0 + 64 * c, k0 + b_off);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== MMA warpgroup: wgmma -> registers -> shared memory -> epilogue =====================
    const int ew = warp - 4;                         // this warp's epilogue rows: [32*ew, 32*ew+32) of the tile
    // K-major : SBO = 8 rows * 128 B, LBO unused ; advance 32 B per k16 step
    // MN-major: SBO = 8 k-rows * 128 B, LBO = one 64-wide MN chunk (BLOCK_K rows * 128 B); advance 16 rows
    // Rows [64, 128) of A start 8 KB in, in both layouts (64 rows of 128 B, or the second 64-wide MN chunk).
    constexpr uint32_t kSbo = 1024;
    constexpr uint32_t kLboA = A_MN ? BLOCK_K * 128 : 16;
    constexpr uint32_t kLboB = B_MN ? BLOCK_K * 128 : 16;
    constexpr uint32_t kStepA = A_MN ? UMMA_K * 128 : UMMA_K * 2;
    constexpr uint32_t kStepB = B_MN ? UMMA_K * 128 : UMMA_K * 2;
    constexpr uint32_t kHalfA = 64 * 128;
    int stage = 0;
    uint32_t phase = 0;
    [[maybe_unused]] uint32_t slab = 0;
    for (int tile = first; tile < num_tiles; tile += stride) {
      int mb, nb, e, kb0 = 0, kb1 = num_k_blocks, b_off = 0;
      if (!grouped_tile<GRP>(p, tile, num_m_blocks, num_n_blocks, &mb, &nb, &e, &kb0, &kb1, &b_off)) continue;
      const int m0 = mb * kM + (int)rank * BLOCK_M;
      const int n0 = nb * BLOCK_N;
      WgAcc<BLOCK_N> acc;
      [[maybe_unused]] WgAcc<BLOCK_N> part;                    // FP8: this k-block's products before promotion
      if constexpr (kFP8 || GRP == kGrpWgrad || GRP == kBoundK) {   // an empty k-loop (no rows) runs no wgmma and stores zeros
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) { acc.h[0][i] = 0.f; acc.h[1][i] = 0.f; }
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * L::kStageBytes);
        const uint32_t b_addr = a_addr + L::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {            // 32 bytes of every row per step: k16 bf16 or k32 FP8
          const uint64_t da0 = make_smem_desc(a_addr + k * kStepA, kLboA, kSbo);
          const uint64_t da1 = make_smem_desc(a_addr + kHalfA + k * kStepA, kLboA, kSbo);
          const uint64_t db = make_smem_desc(b_addr + k * kStepB, kLboB, kSbo);
          if constexpr (kFP8) wgmma_tile_fp8<BLOCK_N, OP == kOpE5M2 ? 1 : 0>(part, da0, da1, db, k != 0 ? 1u : 0u);
          else wgmma_tile<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da0, da1, db, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) {                                        // smem slot reusable: this warp's MMAs have read it
          mbar_arrive(&empty_bar[stage]);
          if constexpr (PAIR) mbar_arrive_cluster(&empty_bar[stage], rank ^ 1u);   // the peer multicasts into it too
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
        if constexpr (kFP8) {                                   // promote into the fp32 tile
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; ++i) { acc.h[0][i] += part.h[0][i]; acc.h[1][i] += part.h[1][i]; }
        }
      }
      if constexpr (kFP8) {
        const float deq = __ldg(p.scale_a) * __ldg(p.scale_b);  // both powers of two: exact
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) { acc.h[0][i] *= deq; acc.h[1][i] *= deq; }
      }
      wg_bar_sync();                                           // the previous tile's epilogue is done reading acc_smem
      acc_to_smem<BLOCK_N>(acc, acc_smem, L::kAccStride, threadIdx.x - 128);
      wg_bar_sync();
      int row = m0 + ew * 32 + lane;
      if constexpr (GRP == kGrpWgrad) row = row < p.grp_rows ? e * p.grp_rows + row : p.M;   // expert e's rows of D; the rest unstored
      const float* arow = acc_smem + (size_t)(ew * 32 + lane) * L::kAccStride;
      if constexpr (LM != kLmNone) {
        lm_epilogue_tile<LM>(p, arow, row, n0);
      } else if constexpr (TMA_ST) {
        epilogue_tile_tma<BLOCK_N, STATS>(p, &map_d, store_stage + ew * 2 * kStoreSlabBytes, arow, m0 + ew * 32, n0, lane, slab);
      } else {
#pragma unroll 1
        for (int c = 0; c < BLOCK_N; c += 32) {
          uint32_t r[32];
          acc_row_ld32(arow, 0, 0, c, r);
          if constexpr (STATS) {
            if (n0 + c < p.N) {                                   // warp-uniform
              float v[32];
              epilogue_math(p, n0 + c, r, v);
              column_stats_chunk(p, row, m0 + ew * 32, n0 + c, v, lane);
            }
          }
          store_row_chunk(p, row, n0 + c, r);
        }
      }
    }
    if constexpr (TMA_ST) {
      if (lane == 0) bulk_wait_all();                         // staging smem must outlive the last store
    }
  }
  if constexpr (PAIR) {
    __syncthreads();
    cluster_sync_all();                      // no CTA exits while its peer may still arrive on its barriers
  }
}

// ---------------- host side ------------------------------------------------------------------------
// 2-D row-major tensor [rows, cols] of bf16 (elem_bytes 2) or 8-bit (elem_bytes 1) elements; box = [box_rows, box_cols]
// with box_cols * elem_bytes == 128 bytes.
CUtensorMap make_map(const void* ptr, int rows, int cols, int box_rows, int box_cols, int elem_bytes = 2) {
  const uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows};
  const uint64_t strides[1] = {(uint64_t)cols * elem_bytes};
  const uint32_t box[2] = {(uint32_t)box_cols, (uint32_t)box_rows};
  const CUtensorMapDataType dt = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  return encode_tensor_map(ptr, dt, CU_TENSOR_MAP_SWIZZLE_128B, 2, dims, strides, box);
}

// TMA_ST: epilogue through shared memory + TMA store (bf16 output, N % 8 == 0); the D map's box is one warp slab.
template <int BLOCK_N, bool A_MN, bool B_MN, bool TMA_ST, bool STATS = false, bool PAIR = false, int OP = kOpBF16, int LM = kLmNone,
          int GRP = kGrpNone>
void launch_variant(const void* a, const void* b, const GemmParams& p, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N, A_MN, B_MN, TMA_ST>;
  constexpr int kSmem = L::kTotal;
  static_assert(L::kStages >= 3 && kSmem <= 227 * 1024, "shared memory budget");
  // A: K-major stored [M,K] -> box {BLOCK_M rows, 64 cols};  MN-major stored [K,M] -> box {64 rows(k), 64 cols(m)}
  // FP8: K-major boxes of 128 one-byte elements (the same 128 bytes per row)
  constexpr int kEB = OP == kOpBF16 ? 2 : 1;
  constexpr int kBK = 128 / kEB;
  CUtensorMap map_a = A_MN ? make_map(a, p.K, p.M, BLOCK_K, 64) : make_map(a, p.M, p.K, BLOCK_M, kBK, kEB);
  CUtensorMap map_b = B_MN ? make_map(b, p.K, p.N, BLOCK_K, 64) : make_map(b, p.N, p.K, PAIR ? BLOCK_N / 2 : BLOCK_N, kBK, kEB);
  CUtensorMap map_d = TMA_ST ? make_map(p.d, p.M, p.N, 32, 64) : map_a;       // unused by the direct epilogue
  auto kernel = gemm_bf16_kernel<BLOCK_N, A_MN, B_MN, TMA_ST, STATS, PAIR, OP, LM, GRP>;
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(kernel, kSmem, configured);
  if constexpr (PAIR) {
    const int tiles = ceil_div(p.M, 2 * BLOCK_M) * ceil_div(p.N, BLOCK_N);
    const int pairs = tiles < kNumSMs / 2 ? tiles : kNumSMs / 2;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2 * pairs);
    cfg.blockDim = dim3(kNumThreads);
    cfg.dynamicSmemBytes = kSmem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, map_a, map_b, map_d, p));
  } else {
    const int tiles = ceil_div(p.M, BLOCK_M) * ceil_div(p.N, BLOCK_N);
    const int grid = tiles < kNumSMs ? tiles : kNumSMs;
    kernel<<<grid, kNumThreads, kSmem, stream>>>(map_a, map_b, map_d, p);
  }
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

int g_gemm_mode = -1;      // -1 = read B200DDP_GEMM_CTAS on first use: 0 auto, 1 single CTAs, 2 cluster pairs
int g_gemm_group_m = -1;   // -1 = read B200DDP_GEMM_GROUP_M on first use
int g_gemm_tma_store = -1; // -1 = read B200DDP_GEMM_TMA_STORE on first use (default 0: direct register -> global epilogue)

}  // namespace

void set_gemm_cta_mode(int mode) { g_gemm_mode = mode; }
void set_gemm_group_m(int group_m) { g_gemm_group_m = group_m; }
void set_gemm_tma_store(int on) { g_gemm_tma_store = on; }

bool gemm_shape_supported(int M, int N, int K, bool a_mn, bool b_mn) {
  if (M < 1 || N < 1 || K < 1) return false;
  // TMA: global row pitch must be a multiple of 16 bytes
  const int a_cols = a_mn ? M : K, b_cols = b_mn ? N : K;
  if (a_cols % 8 != 0 || b_cols % 8 != 0) return false;
  return true;
}

void launch_gemm_bf16(const void* a, const void* b, void* d, const void* bias, int M, int N, int K, bool a_mn, bool b_mn,
                      int epilogue, DType out_dtype, bool accumulate, cudaStream_t stream, float* col_stats) {
  if (!gemm_shape_supported(M, N, K, a_mn, b_mn)) throw std::runtime_error("gemm_bf16: shape not TMA-compatible (row pitch % 16 B)");
  if (out_dtype != DType::BF16 && out_dtype != DType::F32) throw std::runtime_error("gemm_bf16: output must be bf16 or fp32");
  if (accumulate && out_dtype != DType::F32) throw std::runtime_error("gemm_bf16: accumulate needs fp32 output");
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.epilogue = epilogue;
  p.out_fp32 = out_dtype == DType::F32 ? 1 : 0;
  p.accumulate = accumulate ? 1 : 0;
  p.d = d;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.col_stats = col_stats;
  p.stat_groups = (M + 31) / 32;
  if (g_gemm_mode == -1) {
    const char* e = getenv("B200DDP_GEMM_CTAS");
    g_gemm_mode = e ? atoi(e) : 0;
  }
  if (g_gemm_group_m == -1) {
    const char* e = getenv("B200DDP_GEMM_GROUP_M");
    g_gemm_group_m = e ? atoi(e) : 0;
  }
  p.group_m = g_gemm_group_m > 0 ? g_gemm_group_m : 0;
  if (g_gemm_tma_store == -1) {
    const char* e = getenv("B200DDP_GEMM_TMA_STORE");
    g_gemm_tma_store = e ? atoi(e) : 0;
  }
  // staged epilogue: bf16 output with a TMA-legal row pitch, 16-byte aligned base, no read-modify-write
  const bool tma_st = g_gemm_tma_store > 0 && !p.out_fp32 && !p.accumulate && N % 8 == 0 && (reinterpret_cast<uintptr_t>(d) & 15) == 0;
  // Tile shape.  128 x 64 tiles when the output is at most 64 wide (half of a 128-wide tile would be padding), 128 x 128
  // otherwise: a 128 x 128 fp32 accumulator is 128 registers per thread of the warpgroup (two m64 halves of 64), and a
  // 256-wide tile would need 256, more than a thread can hold.  Cluster pairs (256 x 128 per pair, B multicast) halve the B traffic out of L2 but, in this kernel's
  // one-stage-at-a-time pipeline, tie each CTA to its peer's pace: they are opt-in (mode 2), not the automatic choice.
  int choice;   // 0 = cluster pair 256 x 128, 1 = single 128 x 128, 2 = single 128 x 64
  if (g_gemm_mode == 2) choice = 0;
  else choice = N <= 64 ? 2 : 1;
  if (col_stats != nullptr) {
    // column statistics ride on the forward layout only (A [M,K], B [N,K]): that is where a normalisation follows
    if (a_mn || b_mn) throw std::runtime_error("gemm_bf16: column statistics need K-major operands");
    if (tma_st) {
      if (choice == 0) launch_variant<128, false, false, true, true, true>(a, b, p, stream);
      else if (choice == 1) launch_variant<128, false, false, true, true>(a, b, p, stream);
      else launch_variant<64, false, false, true, true>(a, b, p, stream);
    } else {
      if (choice == 0) launch_variant<128, false, false, false, true, true>(a, b, p, stream);
      else if (choice == 1) launch_variant<128, false, false, false, true>(a, b, p, stream);
      else launch_variant<64, false, false, false, true>(a, b, p, stream);
    }
    return;
  }
#define B200_GEMM_DISPATCH(AMN, BMN)                                                   \
  if (a_mn == AMN && b_mn == BMN) {                                                    \
    if (tma_st) {                                                                      \
      if (choice == 0) launch_variant<128, AMN, BMN, true, false, true>(a, b, p, stream);  \
      else if (choice == 1) launch_variant<128, AMN, BMN, true>(a, b, p, stream);      \
      else launch_variant<64, AMN, BMN, true>(a, b, p, stream);                        \
    } else {                                                                           \
      if (choice == 0) launch_variant<128, AMN, BMN, false, false, true>(a, b, p, stream); \
      else if (choice == 1) launch_variant<128, AMN, BMN, false>(a, b, p, stream);     \
      else launch_variant<64, AMN, BMN, false>(a, b, p, stream);                       \
    }                                                                                  \
    return;                                                                            \
  }
  B200_GEMM_DISPATCH(false, false)
  B200_GEMM_DISPATCH(false, true)
  B200_GEMM_DISPATCH(true, true)
  B200_GEMM_DISPATCH(true, false)
#undef B200_GEMM_DISPATCH
}

void launch_gemm_nt_bf16(const void* a, const void* b, void* d, const void* bias, int M, int N, int K, int epilogue,
                         DType out_dtype, cudaStream_t stream) {
  launch_gemm_bf16(a, b, d, bias, M, N, K, false, false, epilogue, out_dtype, false, stream, nullptr);
}

void launch_gemm_fp8(const void* a, const void* b, void* d, const void* bias, const float* a_scale_inv, const float* b_scale_inv,
                     int M, int N, int K, bool a_e5m2, int epilogue, cudaStream_t stream) {
  if (M < 1 || N < 1 || K < 1) throw std::runtime_error("gemm_fp8: empty problem");
  // TMA: the operands' row pitch (K one-byte elements) must be a multiple of 16 bytes
  if (K % 16 != 0) throw std::runtime_error("gemm_fp8: K = " + std::to_string(K) + " is not a multiple of 16");
  if (a_scale_inv == nullptr || b_scale_inv == nullptr) throw std::runtime_error("gemm_fp8: missing dequantisation factors");
  if (epilogue < 0 || epilogue > 3) throw std::runtime_error("gemm_fp8: bad epilogue");
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.epilogue = epilogue;
  p.d = d;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.scale_a = a_scale_inv;
  p.scale_b = b_scale_inv;
  if (g_gemm_group_m == -1) {
    const char* e = getenv("B200DDP_GEMM_GROUP_M");
    g_gemm_group_m = e ? atoi(e) : 0;
  }
  p.group_m = g_gemm_group_m > 0 ? g_gemm_group_m : 0;
  if (a_e5m2) launch_variant<64, false, false, false, false, false, kOpE5M2>(a, b, p, stream);
  else launch_variant<64, false, false, false, false, false, kOpE4M3>(a, b, p, stream);
}

namespace {
GemmParams lm_params(int M, int N, int K, const void* bias, const long long* targets) {
  if (!gemm_shape_supported(M, N, K, false, false)) throw std::runtime_error("gemm_lm: hidden size must be a multiple of 8");
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.epilogue = bias != nullptr ? 1 : 0;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.lm_targets = targets;
  return p;
}
}  // namespace

void launch_gemm_lm_lse(const void* hidden, const void* weight, const void* bias, int M, int V, int K, const long long* targets,
                        float* partial, float* target_logit, cudaStream_t stream, const int* rows) {
  GemmParams p = lm_params(M, V, K, bias, targets);
  p.d = partial;
  p.lm_target_logit = target_logit;
  p.bound_rows = rows;
  if (rows != nullptr) launch_variant<128, false, false, false, false, false, kOpBF16, kLmLse, kBoundRows>(hidden, weight, p, stream);
  else launch_variant<128, false, false, false, false, false, kOpBF16, kLmLse>(hidden, weight, p, stream);
}

void launch_gemm_lm_dlogits(const void* hidden, const void* weight, const void* bias, int M, int N, int K, int col_offset, int vocab,
                            const long long* targets, long long ignore_index, const float* lse, const float* gscale,
                            const float* valid, void* dlogits, cudaStream_t stream, const int* rows) {
  GemmParams p = lm_params(M, N, K, bias, targets);
  p.d = dlogits;
  p.lm_lse = lse;
  p.lm_gscale = gscale;
  p.lm_valid = valid;
  p.lm_ignore_index = ignore_index >= 0 && ignore_index < vocab ? (int)ignore_index : -1;
  p.lm_col_offset = col_offset;
  p.lm_vocab = vocab;
  p.bound_rows = rows;
  if (rows != nullptr) launch_variant<128, false, false, false, false, false, kOpBF16, kLmDlogits, kBoundRows>(hidden, weight, p, stream);
  else launch_variant<128, false, false, false, false, false, kOpBF16, kLmDlogits>(hidden, weight, p, stream);
}

void launch_gemm_bf16_rows(const void* a, const void* b, void* d, int M, int N, int K, bool a_mn, DType out_dtype, bool accumulate,
                           const int* rows, cudaStream_t stream) {
  if (!gemm_shape_supported(M, N, K, a_mn, true)) throw std::runtime_error("gemm_bf16_rows: shape not TMA-compatible (row pitch % 16 B)");
  if (out_dtype != DType::BF16 && out_dtype != DType::F32) throw std::runtime_error("gemm_bf16_rows: output must be bf16 or fp32");
  if (accumulate && out_dtype != DType::F32) throw std::runtime_error("gemm_bf16_rows: accumulate needs fp32 output");
  if (rows == nullptr) throw std::runtime_error("gemm_bf16_rows: missing the device row count");
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.out_fp32 = out_dtype == DType::F32 ? 1 : 0;
  p.accumulate = accumulate ? 1 : 0;
  p.d = d;
  p.bound_rows = rows;
  if (a_mn) launch_variant<128, true, true, false, false, false, kOpBF16, kLmNone, kBoundK>(a, b, p, stream);
  else launch_variant<128, false, true, false, false, false, kOpBF16, kLmNone, kBoundRows>(a, b, p, stream);
}

namespace {
template <bool A_MN, bool B_MN, int GRP>
void launch_grouped(const CUtensorMap& map_a, const CUtensorMap& map_b, const GemmParams& p, int tiles, cudaStream_t stream) {
  using L = SmemLayout<128, A_MN, B_MN, false>;
  static_assert(L::kStages >= 3 && L::kTotal <= 227 * 1024, "shared memory budget");
  auto kernel = gemm_bf16_kernel<128, A_MN, B_MN, false, false, false, kOpBF16, kLmNone, GRP>;
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(kernel, L::kTotal, configured);
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  kernel<<<grid, kNumThreads, L::kTotal, stream>>>(map_a, map_b, map_a, p);     // D map unused by the direct epilogue
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void grouped_check(int rows, int N, int K, int experts) {
  if (rows < 128 || rows % 128 != 0 || N < 64 || N % 64 != 0 || K < 64 || K % 64 != 0 || experts < 1)
    throw std::runtime_error("gemm_grouped: needs rows a positive multiple of 128, N and K positive multiples of 64 and >= 1 expert, got rows=" +
                             std::to_string(rows) + " N=" + std::to_string(N) + " K=" + std::to_string(K) + " experts=" + std::to_string(experts));
}
}  // namespace

void launch_gemm_grouped(const void* a, const void* b, void* d, int rows, int N, int K, int experts, bool b_mn, const int* tile_expert,
                         cudaStream_t stream) {
  grouped_check(rows, N, K, experts);
  GemmParams p = {};
  p.M = rows; p.N = N; p.K = K;
  p.d = d;
  p.grp_tile_expert = tile_expert;
  p.grp_rows = b_mn ? K : N;
  const CUtensorMap map_a = make_map(a, rows, K, BLOCK_M, 64);
  const int tiles = (rows / BLOCK_M) * ceil_div(N, 128);
  if (b_mn) launch_grouped<false, true, kGrpRows>(map_a, make_map(b, experts * K, N, BLOCK_K, 64), p, tiles, stream);
  else launch_grouped<false, false, kGrpRows>(map_a, make_map(b, experts * N, K, 128, 64), p, tiles, stream);
}

void launch_gemm_grouped_wgrad(const void* a, const void* b, void* d, int rows, int M, int N, int experts, const int* offsets,
                               cudaStream_t stream) {
  grouped_check(rows, N, M, experts);
  GemmParams p = {};
  p.M = experts * M; p.N = N; p.K = rows;
  p.d = d;
  p.grp_offsets = offsets;
  p.grp_rows = M;
  p.grp_experts = experts;
  const int tiles = experts * ceil_div(M, BLOCK_M) * ceil_div(N, 128);
  launch_grouped<true, true, kGrpWgrad>(make_map(a, rows, M, BLOCK_K, 64), make_map(b, rows, N, BLOCK_K, 64), p, tiles, stream);
}

}  // namespace b200
