// Multi-head attention with a key-padding mask on the Hopper tensor cores (the BERT encoder's attention for right-padded
// batches).  Head dim 64, softmax scale 1/8; the causal mode also runs at head dim 128 (last section of this file).
//
//   qkv  bf16 [B*S, 3*H*64]   the fused projection's output: column blocks query | key | value, head h at h*64 .. h*64+63
//   o    bf16 [B*S, H*64]     written in the layout the output projection reads (no transpose)
//   lse  fp32 [B, H, S]       natural-log row log-sum-exp of the scaled scores (-inf for a sequence of length 0)
//
// Three mask modes, chosen at compile time (template parameter kMode):
//   kKeyPadding  seq_lens int32 [B]: key j of sequence b is visible iff j < seq_lens[b] (clamped to [0, S] here: the host
//                cannot validate device lengths without a synchronisation).  Every query row is computed, padded ones
//                included, so every row equals softmax attention over the visible keys; a sequence of length 0 gets zero
//                output and zero gradients.
//   kSegment     bounds int32 [B*S, 2] (packed documents): query i of a sequence sees key j of the same sequence iff
//                start[i] <= j < end[i] (start clamped to [0, S], end to [start, S]).  A row with start == end (padding)
//                gets zero output, lse = -inf and zero gradients.  Each CTA visits only the tiles inside the union of its
//                128 rows' intervals; dK / dV mask with the key rows' own bounds, which is the same test as the query's for
//                a block-diagonal mask.
//   kCausal      the same bounds, causal inside each document: query i sees key j iff start[i] <= j <= i and j < end[i].
//                Both sides are still intervals: query i sees keys [start_i, min(end_i, i + 1)), key k is seen by
//                queries [max(start_k, k), end_k), so the forward and dQ stop at the diagonal tile and dK / dV start at
//                it.  Padding rows behave as in kSegment; a row inside its document always sees itself.  Tile work
//                grows with the query tile (forward, dQ) and shrinks with the key tile (dK / dV), so the grid is walked
//                heaviest tiles first.
//
// Each kernel has one TMA producer warp (warp 0; warps 1-3 idle) and two consumer warpgroups (warps 4-7, 8-11) that own
// 64 rows each.  All tiles are 64-row boxes of one 2-D tensor map over qkv (or dO), 128B-swizzled, so a head's 64
// columns are exactly one swizzle row and the same shared-memory tile serves as a K-major operand (Q K^T) or an MN-major
// one (P V).  P and dS never touch shared memory: the fp32 accumulator fragment packed to bf16x2 IS the register A
// fragment of the next wgmma (tc::wgmma_n64_rs).
//
// Forward (flash attention): CTA = (query tile of 128, head, batch); K/V tiles of 128 keys stream through a 2-stage ring;
// online softmax in fp32 registers; key tiles at or beyond the length are never loaded.
// Backward, deterministic (no atomics; every output element has one writer):
//   attn_bwd_dot  D = rowsum(dO * O)
//   attn_bwd_dkdv CTA = (key tile of 128, head, batch), loops over all query tiles: S^T = K Q^T, P^T = exp(S^T - lse),
//                 dV += P^T dO, dP^T = V dO^T, dS^T = P^T (dP^T - D), dK += dS^T Q.  Key tiles wholly beyond the length
//                 only write zeros.
//   attn_bwd_dq   CTA = (query tile of 128, head, batch), loops over the key tiles below the length: S, P, dP = dO V^T,
//                 dS, dQ += dS K.
// Recomputing P in both backward kernels costs two GEMMs more than accumulating dQ with atomics inside the dK/dV loop;
// that is the price of bit-identical gradients on every run.
//
// Grouped-query attention (kCausal only, compile-time kGqa): qkv is [B*S, (H + 2*Hkv)*64] with column blocks query (H
// heads) | key (Hkv heads) | value (Hkv heads); query head h reads K/V head h / (H / Hkv) (Hugging Face's repeat_kv
// order).  The forward and dQ keep their grid (S/128, H, B) and only read K/V at other columns.  dK/dV runs on
// (S/128, Hkv, B): its ring walks every (query head of the group, query tile) pair and accumulates the whole group's
// contribution in registers, so each dK/dV element still has one writer.
#include "attention_common.cuh"

namespace b200 {
namespace {

__device__ __forceinline__ int clamped_len(const int* lens, int b, int S) {
  const int n = __ldg(lens + b);
  return n < 0 ? 0 : (n > S ? S : n);
}
// (tile, head, batch) of this CTA.  kCausal walks the grid heaviest tiles first: every (head, batch) pair's last query
// tile (kKeySide = false: the forward and dQ, whose work grows with the tile) or first key tile (dK / dV) before any
// pair's next one, so the light tiles fill the tail of the launch.
template <int kMode, bool kKeySide>
__device__ __forceinline__ int3 tile_coords() {
  if constexpr (kMode == kCausal) {
    const int pairs = gridDim.y * gridDim.z;
    const int id = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
    const int step = id / pairs, pair = id - step * pairs;
    return make_int3(kKeySide ? step : (int)gridDim.x - 1 - step, pair % (int)gridDim.y, pair / (int)gridDim.y);
  } else {
    return make_int3(blockIdx.x, blockIdx.y, blockIdx.z);
  }
}

// Columns of query head h's key and value heads in qkv (H query heads, HD = H * 64; Hkv K/V heads when kGqa)
template <bool kGqa>
__device__ __forceinline__ int2 kv_cols(int h, int H, int HD, int Hkv) {
  if constexpr (kGqa) {
    const int hk = h / (H / Hkv);
    return make_int2(HD + hk * kHd, HD + (Hkv + hk) * kHd);
  } else {
    return make_int2(HD + h * kHd, 2 * HD + h * kHd);
  }
}

// ============================================== relative position bias ===============================================
// kBias (kSegment / kCausal, multi-head): T5's learned relative position bias.  table fp32 [H, 257] holds head h's bias
// for the clamped distance k - i in [-128, 128] at column k - i + 128; the score of a visible pair is q.k + table[h, .]
// with no 1/sqrt(d) scale, so lse, P and the gradients are those of the unscaled, biased scores.  Each CTA keeps its
// head's row in shared memory (after the 256 bytes of barriers and scratch every layout reserves), widened to the
// distances [-264, 264] so that a thread's lookups need no clamp: a thread with any distance inside (-128, 128) has all
// of them within 129 of it.
constexpr int kRelMax = 128;
constexpr int kRelCols = 2 * kRelMax + 1;                       // 257
constexpr int kRelMid = kRelMax + 136;                          // the widened row: distance d at kRelMid + d
constexpr int kBiasTable = 2304;                                // 2 kRelMid + 1 entries, then 16 floats of far-sum scratch
constexpr int kFarRed = 2 * kRelMid + 4;                        // the scratch's offset in floats
constexpr int kPartStride = 25;                                 // dQ: floats per thread in a diagonal-fold buffer (odd: no bank conflicts)
constexpr int kPartBytes = 2 * 256 * kPartStride * 4;           // dQ: two buffers of 256 consumer threads

// Copies head h's table row, widened, into shared memory; every thread calls it before the kernel's first __syncthreads.
__device__ __forceinline__ void load_bias_table(float* tbl, const float* __restrict__ table, int h) {
  for (int i = threadIdx.x; i <= 2 * kRelMid; i += blockDim.x)
    tbl[i] = __ldg(table + (size_t)h * kRelCols + min(max(i - kRelMid, -kRelMax), kRelMax) + kRelMax);
}

// Adds the bias to one thread's fragment of 4 * kJ scores.  Element (i, j, e) (s[4 j + 2 i + e]: row half i, column
// 8 j + e from the thread's first) lies at distance base + i * kDi + kSign * (8 j + e), in [base + kLo, base + kHi].  A
// thread whose distances all lie beyond +-128 on one side has a constant bias: its base is moved to where its nearest
// distance is +-128, which reads that same entry everywhere from the widened row, so one branch-free path serves both.
// rel_bias_row gives the thread's row pointer t: the bias of element (i, j, e) is t[i * kDi + kSign * (8 j + e)].
template <int kJ, int kSign, int kDi>
__device__ __forceinline__ const float* rel_bias_row(const float* tbl, int base) {
  constexpr int kSpan = 8 * (kJ - 1);
  constexpr int kLo = (kDi < 0 ? kDi : 0) - (kSign < 0 ? kSpan + 1 : 0), kHi = (kDi > 0 ? kDi : 0) + (kSign > 0 ? kSpan + 1 : 0);
  static_assert(kHi - kLo <= kRelMid - kRelMax, "the widened row must cover a thread's distances");
  return tbl + kRelMid + min(max(base, -kRelMax - kHi), kRelMax - kLo);
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
template <int kJ, int kSign, int kDi>
__device__ __forceinline__ void add_rel_bias(float (&s)[4 * kJ], const float* tbl, int base) {
  const float* t = rel_bias_row<kJ, kSign, kDi>(tbl, base);
#pragma unroll
  for (int j = 0; j < kJ; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) s[4 * j + 2 * i + e] += t[i * kDi + kSign * (8 * j + e)];
    }
  }
}

// ============================================== forward ==============================================================
// mask: seq_lens [B] (kKeyPadding) or bounds [B*S, 2] (kSegment, kCausal); Hkv: K/V heads (read only when kGqa);
// table: the relative bias (read only when kBias)
template <int kMode, bool kGqa = false, bool kBias = false>
__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap map_qkv, const int* __restrict__ mask, int S, int H,
                __nv_bfloat16* __restrict__ o, float* __restrict__ lse, int Hkv, const float* __restrict__ table) {
  static_assert(!kBias || (kMode != kKeyPadding && !kGqa), "the relative bias is a document-mode, multi-head instantiation");
  constexpr float kSc = kBias ? 1.f : kScale;                   // natural-log units per score unit
  constexpr float kSL = kSc * kLog2e;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sq = smem;                                           // 128 query rows
  uint8_t* ring = sq + 2 * kBoxBytes;                           // stage: K 128 rows, V 128 rows
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(ring + kFwdStages * 4 * kBoxBytes);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kFwdStages;
  float* tbl = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(q_bar) + 256);   // kBias

  const int3 tc = tile_coords<kMode, false>();
  const int qt = tc.x, h = tc.y, b = tc.z;
  const int HD = H * kHd;
  const size_t seq_row = (size_t)b * S;
  int len = 0, kt0 = 0, n_kt;                                   // key tiles kt0 .. kt0 + n_kt - 1
  if constexpr (kMode == kKeyPadding) {
    len = clamped_len(mask, b, S);
    n_kt = (len + 127) / 128;
  } else {
    const int2 r = cta_range<kMode, false>(mask, seq_row + qt * 128, qt * 128, S, reinterpret_cast<int*>(empty_bar + kFwdStages));
    kt0 = r.x / 128;
    n_kt = r.x < r.y ? (r.y + 127) / 128 - kt0 : 0;
  }
  float* lse_bh = lse + ((size_t)b * H + h) * S;
  if (n_kt == 0) {                                              // no visible key: zero output, empty log-sum-exp
    zero_rows(o + h * kHd, HD, seq_row + qt * 128, 128);
    if (threadIdx.x < 128) lse_bh[qt * 128 + threadIdx.x] = -INFINITY;
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) {
    mbar_init(q_bar, 1);
    for (int i = 0; i < kFwdStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerArrivals); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if constexpr (kBias) load_bias_table(tbl, table, h);
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&map_qkv);
      const int q_row = (int)seq_row + qt * 128;
      mbar_expect_tx(q_bar, 2 * kBoxBytes);
      tma_load_2d(&map_qkv, q_bar, sq, h * kHd, q_row);
      tma_load_2d(&map_qkv, q_bar, sq + kBoxBytes, h * kHd, q_row + 64);
      const int2 kv = kv_cols<kGqa>(h, H, HD, Hkv);
      int stage = 0;
      uint32_t phase = 0;
      for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sk = ring + stage * 4 * kBoxBytes;
        uint8_t* sv = sk + 2 * kBoxBytes;
        const int k_row = (int)seq_row + kt * 128;
        mbar_expect_tx(&full_bar[stage], 4 * kBoxBytes);
        tma_load_2d(&map_qkv, &full_bar[stage], sk, kv.x, k_row);
        tma_load_2d(&map_qkv, &full_bar[stage], sk + kBoxBytes, kv.x, k_row + 64);
        tma_load_2d(&map_qkv, &full_bar[stage], sv, kv.y, k_row);
        tma_load_2d(&map_qkv, &full_bar[stage], sv + kBoxBytes, kv.y, k_row + 64);
        if (++stage == kFwdStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;                             // query rows [64 wg, 64 wg + 64) of the tile
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);         // this thread's rows: r0 and r0 + 8 of the warpgroup's 64
    const int c0 = 2 * (lane & 3);
    const uint32_t q_addr = smem_u32(sq + wg * kBoxBytes);
    int2 rb0, rb1;                                              // kSegment / kCausal: the intervals of this thread's two rows
    if constexpr (kMode != kKeyPadding) {
      rb0 = mask_interval<kMode, false>(mask, seq_row + qt * 128 + wg * 64 + r0, qt * 128 + wg * 64 + r0, S);
      rb1 = mask_interval<kMode, false>(mask, seq_row + qt * 128 + wg * 64 + r0 + 8, qt * 128 + wg * 64 + r0 + 8, S);
    }
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(q_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t k_addr = smem_u32(ring + stage * 4 * kBoxBytes);
      const uint32_t v_addr = k_addr + 2 * kBoxBytes;
      float s[64];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHd / 16; ++k)
        wgmma_n128<0, 0>(s, desc_k(q_addr + k * kStepK), desc_k(k_addr + k * kStepK), k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      const int key0 = kt * 128;
      if constexpr (kBias) add_rel_bias<16, 1, -8>(s, tbl, key0 + c0 - (qt * 128 + wg * 64 + r0));
      if constexpr (kMode == kKeyPadding) {
        if (key0 + 128 > len) {                                 // partial tile: hide keys at or beyond the length
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (key0 + 8 * j + c0 + e >= len) { s[4 * j + e] = -INFINITY; s[4 * j + 2 + e] = -INFINITY; }
            }
          }
        }
      } else {
        if (key0 < max(rb0.x, rb1.x) || key0 + 128 > min(rb0.y, rb1.y)) {   // tile not wholly inside both intervals
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int key = key0 + 8 * j + c0 + e;
              if (!inside(key, rb0)) s[4 * j + e] = -INFINITY;
              if (!inside(key, rb1)) s[4 * j + 2 + e] = -INFINITY;
            }
          }
        }
      }
      // online softmax: the four threads of a quad share a row
      float mx[2] = {m[0], m[1]};
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        mx[0] = fmaxf(mx[0], fmaxf(s[4 * j], s[4 * j + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[4 * j + 2], s[4 * j + 3]));
      }
      float alpha[2], mb[2], rs[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
        mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
        if constexpr (kMode == kKeyPadding) {
          alpha[i] = exp2f((m[i] - mx[i]) * kSL);               // key 0 is visible, so mx is finite; 0 on the first tile
          m[i] = mx[i];
          mb[i] = mx[i] * kSL;
        } else {
          // a row may have seen no visible key yet (mx = -inf): subtract 0 instead, so exp2 gives 0 rather than NaN
          const float base = mx[i] == -INFINITY ? 0.f : mx[i];
          alpha[i] = exp2f((m[i] - base) * kSL);
          m[i] = mx[i];
          mb[i] = base * kSL;
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        s[4 * j] = exp2f(s[4 * j] * kSL - mb[0]);
        s[4 * j + 1] = exp2f(s[4 * j + 1] * kSL - mb[0]);
        s[4 * j + 2] = exp2f(s[4 * j + 2] * kSL - mb[1]);
        s[4 * j + 3] = exp2f(s[4 * j + 3] * kSL - mb[1]);
        rs[0] += s[4 * j] + s[4 * j + 1];
        rs[1] += s[4 * j + 2] + s[4 * j + 3];
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) l[i] = l[i] * alpha[i] + rs[i];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[4 * j] *= alpha[0]; acc[4 * j + 1] *= alpha[0];
        acc[4 * j + 2] *= alpha[1]; acc[4 * j + 3] *= alpha[1];
      }
      // O += P V: P from registers (16 keys per k16 step), V MN-major
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                               pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
        wgmma_n64_rs<1>(acc, a, desc_mn(v_addr + kk * kStepMN), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == kFwdStages) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
    }
    const int row = qt * 128 + wg * 64 + r0;                    // position in the sequence
    if constexpr (kMode == kKeyPadding) {
      store_frag(acc, 1.f / l[0], 1.f / l[1], o + (seq_row + row) * HD + h * kHd, HD, c0);
      if ((lane & 3) == 0) {
        lse_bh[row] = m[0] * kSc + logf(l[0]);
        lse_bh[row + 8] = m[1] * kSc + logf(l[1]);
      }
    } else {                                                    // a row that saw no key: zeros and -inf
      store_frag(acc, l[0] > 0.f ? 1.f / l[0] : 0.f, l[1] > 0.f ? 1.f / l[1] : 0.f, o + (seq_row + row) * HD + h * kHd, HD, c0);
      if ((lane & 3) == 0) {
        lse_bh[row] = l[0] > 0.f ? m[0] * kSc + logf(l[0]) : -INFINITY;
        lse_bh[row + 8] = l[1] > 0.f ? m[1] * kSc + logf(l[1]) : -INFINITY;
      }
    }
  }
}

// ============================================== backward =============================================================


// The ring of the GQA dK/dV kernel: for each of the `groups` query heads h0 + g, `n` stages of (Q, dO) tiles of 64 rows
// from ring_row0, at columns (h0 + g) * 64 of qkv and dO.
__device__ __forceinline__ void bwd_produce_groups(const BwdSmem& L, const CUtensorMap* map_qkv, const CUtensorMap* map_do,
                                                   int h0, int groups, int ring_row0, int n) {
  int stage = 0;
  uint32_t phase = 0;
  for (int g = 0; g < groups; ++g) {
    for (int i = 0; i < n; ++i) {
      mbar_wait(&L.empty_bar[stage], phase ^ 1);
      uint8_t* t0 = L.ring + stage * 2 * kBoxBytes;
      mbar_expect_tx(&L.full_bar[stage], 2 * kBoxBytes);
      tma_load_2d(map_qkv, &L.full_bar[stage], t0, (h0 + g) * kHd, ring_row0 + 64 * i);
      tma_load_2d(map_do, &L.full_bar[stage], t0 + kBoxBytes, (h0 + g) * kHd, ring_row0 + 64 * i);
      if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
    }
  }
}

// The consumer warpgroups of the GQA dK/dV kernel: the loop of attn_bwd_dkdv_kernel (kSegment / kCausal masks), run
// once per query head h * groups + g of K/V head h, all into the same dK / dV accumulators.  It is a copy of that loop
// rather than a shared function because factoring the loop out changes the code the multi-head instantiations compile
// to; keep the two in step.  lse and D are indexed with a 32-bit offset (B * H * S < 2^31) from the kernel parameters,
// and the output columns are computed after the loop, so the kernel fits its 168 registers without spilling.
template <int kMode>
__device__ __forceinline__ void dkdv_consume_group(const BwdSmem& L, const int* __restrict__ mask, int S, int H, int Hkv, int b,
                                                   int h, int kt, int qt0, int n_qt, const float* __restrict__ lse,
                                                   const float* __restrict__ Dsum, __nv_bfloat16* __restrict__ dqkv) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = (warp - 4) >> 2;                               // keys [64 wg, 64 wg + 64) of the tile
  const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  const int key = kt * 128 + wg * 64 + r0;
  const size_t seq_row = (size_t)b * S;
  const uint32_t k_addr = smem_u32(L.fixed0 + wg * kBoxBytes), v_addr = smem_u32(L.fixed1 + wg * kBoxBytes);
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  mbar_wait(L.fixed_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
  const int groups = H / Hkv;
  const int bh_end = (b * H + (h + 1) * groups) * S;
#pragma unroll 1
  for (int bh = (b * H + h * groups) * S; bh < bh_end; bh += S) {   // lse / D rows of query heads h * groups + g
    for (int qt = qt0; qt < qt0 + n_qt; ++qt) {
      const int2 kb0 = mask_interval<kMode, true>(mask, seq_row + key, key, S);
      const int2 kb1 = mask_interval<kMode, true>(mask, seq_row + key + 8, key + 8, S);
      const int q0 = qt * 64 + c0;
      const uint32_t vis = frag_mask16(kb0.x - q0, kb0.y - q0) | (frag_mask16(kb1.x - q0, kb1.y - q0) << 16);
      mbar_wait(&L.full_bar[stage], phase);
      const uint32_t q_addr = smem_u32(L.ring + stage * 2 * kBoxBytes), do_addr = q_addr + kBoxBytes;
      float st[32], dpt[32];
      wgmma_fence();
      mma_hd_n64(st, k_addr, q_addr);                           // S^T = K Q^T     [keys, queries]
      mma_hd_n64(dpt, v_addr, do_addr);                         // dP^T = V dO^T
      wgmma_commit();
      wgmma_wait<0>();
      uint32_t pa[16], dsa[16];
#pragma unroll
      for (int j = 0; j < 8; ++j) {                             // query columns 8 j + c0, + 1
        const int q = qt * 64 + 8 * j + c0;
        const float2 lq = *reinterpret_cast<const float2*>(lse + (bh + q));
        const float2 dq = *reinterpret_cast<const float2*>(Dsum + (bh + q));
        const float l0 = lq.x == -INFINITY ? INFINITY : lq.x * kLog2e;   // a query that saw no key gets P = 0
        const float l1 = lq.y == -INFINITY ? INFINITY : lq.y * kLog2e;
        const bool v00 = (vis >> (2 * j)) & 1u, v01 = (vis >> (2 * j + 1)) & 1u;
        const bool v10 = (vis >> (16 + 2 * j)) & 1u, v11 = (vis >> (17 + 2 * j)) & 1u;
        const float p00 = v00 ? exp2f(st[4 * j] * kScaleLog2 - l0) : 0.f;
        const float p01 = v01 ? exp2f(st[4 * j + 1] * kScaleLog2 - l1) : 0.f;
        const float p10 = v10 ? exp2f(st[4 * j + 2] * kScaleLog2 - l0) : 0.f;
        const float p11 = v11 ? exp2f(st[4 * j + 3] * kScaleLog2 - l1) : 0.f;
        pa[2 * j] = pack_bf16x2(p00, p01);
        pa[2 * j + 1] = pack_bf16x2(p10, p11);
        dsa[2 * j] = pack_bf16x2(p00 * (dpt[4 * j] - dq.x), p01 * (dpt[4 * j + 1] - dq.y));
        dsa[2 * j + 1] = pack_bf16x2(p10 * (dpt[4 * j + 2] - dq.x), p11 * (dpt[4 * j + 3] - dq.y));
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_n64_rs<1>(dv, pa + 4 * kk, desc_mn(do_addr + kk * kStepMN), 1u);   // dV += P^T dO
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_n64_rs<1>(dk, dsa + 4 * kk, desc_mn(q_addr + kk * kStepMN), 1u);  // dK += dS^T Q
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&L.empty_bar[stage]);
      if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
    }
  }
  const size_t pitch = (size_t)(H + 2 * Hkv) * kHd;
  __nv_bfloat16* krow = dqkv + (seq_row + key) * pitch + (H + h) * kHd;
  store_frag(dk, kScale, kScale, krow, pitch, c0);
  store_frag(dv, 1.f, 1.f, krow + Hkv * kHd, pitch, c0);
}

// dK, dV for one tile of 128 keys.  Fixed: K, V.  Ring: (Q, dO) tiles of 64 queries: all S / 64 of them (kKeyPadding),
// or those inside the union of the key rows' intervals (kSegment, kCausal); with kGqa, those tiles of every query head
// of the K/V head's group in turn (h is then the K/V head).  kBias: P recomputed with the relative bias.
template <int kMode, bool kGqa = false, bool kBias = false>
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap map_qkv, const __grid_constant__ CUtensorMap map_do,
                     const int* __restrict__ mask, int S, int H, const float* __restrict__ lse, const float* __restrict__ Dsum,
                     __nv_bfloat16* __restrict__ dqkv, int Hkv, const float* __restrict__ table) {
  static_assert(!kBias || (kMode != kKeyPadding && !kGqa), "the relative bias is a document-mode, multi-head instantiation");
  constexpr float kSc = kBias ? 1.f : kScale;
  constexpr float kSL = kSc * kLog2e;
  extern __shared__ uint8_t smem_raw[];
  const BwdSmem L = bwd_smem(smem_raw);
  float* tbl = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(L.fixed_bar) + 256);   // kBias
  const int3 tc = tile_coords<kMode, true>();
  const int kt = tc.x, h = tc.y, b = tc.z;
  const int HD = H * kHd;
  const size_t pitch = kGqa ? (size_t)(H + 2 * Hkv) * kHd : (size_t)3 * HD;
  const int groups = kGqa ? H / Hkv : 1;                        // query heads h * groups + g read this K/V head
  const int kcol = HD + h * kHd;                                // this K/V head's key and value columns
  const int vcol = kGqa ? HD + (Hkv + h) * kHd : 2 * HD + h * kHd;
  const size_t seq_row = (size_t)b * S;
  int len = 0, qt0 = 0, n_qt = S / 64;                          // query tiles qt0 .. qt0 + n_qt - 1
  bool hidden;
  if constexpr (kMode == kKeyPadding) {
    len = clamped_len(mask, b, S);
    hidden = kt * 128 >= len;
  } else {
    const int2 r = cta_range<kMode, true>(mask, seq_row + kt * 128, kt * 128, S, reinterpret_cast<int*>(L.empty_bar + kBwdStages));
    hidden = r.x >= r.y;
    qt0 = r.x / 64;
    n_qt = (r.y + 63) / 64 - qt0;
  }
  if (hidden) {                                                 // every key of the tile is hidden: no gradient
    if constexpr (kGqa) {
      zero_rows(dqkv + kcol, pitch, seq_row + kt * 128, 128);
      zero_rows(dqkv + vcol, pitch, seq_row + kt * 128, 128);
    } else {
      zero_rows(dqkv + HD + h * kHd, pitch, seq_row + kt * 128, 128);
      zero_rows(dqkv + 2 * HD + h * kHd, pitch, seq_row + kt * 128, 128);
    }
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) bwd_init_barriers(L);
  if constexpr (kBias) load_bias_table(tbl, table, h);
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&map_qkv);
      tma_prefetch_desc(&map_do);
      if constexpr (kGqa) {
        mbar_expect_tx(L.fixed_bar, 4 * kBoxBytes);
        tma_load_2d(&map_qkv, L.fixed_bar, L.fixed0, kcol, (int)seq_row + kt * 128);
        tma_load_2d(&map_qkv, L.fixed_bar, L.fixed0 + kBoxBytes, kcol, (int)seq_row + kt * 128 + 64);
        tma_load_2d(&map_qkv, L.fixed_bar, L.fixed1, vcol, (int)seq_row + kt * 128);
        tma_load_2d(&map_qkv, L.fixed_bar, L.fixed1 + kBoxBytes, vcol, (int)seq_row + kt * 128 + 64);
        bwd_produce_groups(L, &map_qkv, &map_do, h * groups, groups, (int)seq_row + 64 * qt0, n_qt);
      } else {
        bwd_produce(L, &map_qkv, HD + h * kHd, &map_qkv, 2 * HD + h * kHd, (int)seq_row + kt * 128,
                    &map_qkv, h * kHd, &map_do, h * kHd, (int)seq_row + 64 * qt0, n_qt);
      }
    }
  } else if (warp >= 4) {
    if constexpr (kGqa) {
      dkdv_consume_group<kMode>(L, mask, S, H, Hkv, b, h, kt, qt0, n_qt, lse, Dsum, dqkv);
      return;
    }
    const int wg = (warp - 4) >> 2;                             // keys [64 wg, 64 wg + 64) of the tile
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const int key = kt * 128 + wg * 64 + r0;
    const bool vis0 = key < len, vis1 = key + 8 < len;          // kKeyPadding
    const uint32_t k_addr = smem_u32(L.fixed0 + wg * kBoxBytes), v_addr = smem_u32(L.fixed1 + wg * kBoxBytes);
    const float* lse_bh = lse + ((size_t)b * H + h) * S;
    const float* D_bh = Dsum + ((size_t)b * H + h) * S;
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
    mbar_wait(L.fixed_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int qt = qt0; qt < qt0 + n_qt; ++qt) {
      // kSegment / kCausal: the key rows' intervals as one bit mask over this thread's 16 query columns (bits 0-15: row
      // key, 16-31: row key + 8), so the mask costs one register while the accumulators are live
      uint32_t vis = 0;
      if constexpr (kMode != kKeyPadding) {
        const size_t mrow = kBias ? (size_t)(unsigned)(b * S + key) : seq_row + key;   // kBias: a 32-bit row (no spills)
        const int2 kb0 = mask_interval<kMode, true>(mask, mrow, key, S);
        const int2 kb1 = mask_interval<kMode, true>(mask, mrow + 8, key + 8, S);
        const int q0 = qt * 64 + c0;
        vis = frag_mask16(kb0.x - q0, kb0.y - q0) | (frag_mask16(kb1.x - q0, kb1.y - q0) << 16);
      }
      mbar_wait(&L.full_bar[stage], phase);
      const uint32_t q_addr = smem_u32(L.ring + stage * 2 * kBoxBytes), do_addr = q_addr + kBoxBytes;
      float st[32], dpt[32];
      wgmma_fence();
      mma_hd_n64(st, k_addr, q_addr);                           // S^T = K Q^T     [keys, queries]
      mma_hd_n64(dpt, v_addr, do_addr);                         // dP^T = V dO^T
      wgmma_commit();
      wgmma_wait<0>();
      uint32_t bias_t = 0;                                      // kBias: a 32-bit shared address, and the bias added column
      if constexpr (kBias) bias_t = smem_u32(rel_bias_row<8, -1, 8>(tbl, key - (qt * 64 + c0)));   // by column: no spills
      uint32_t pa[16], dsa[16];
#pragma unroll
      for (int j = 0; j < 8; ++j) {                             // query columns 8 j + c0, + 1
        const int q = qt * 64 + 8 * j + c0;
        // kBias: lse and D at a 32-bit offset from the kernel parameters (B * H * S < 2^31), as in dkdv_consume_group
        const int bhq = (b * H + h) * S + q;
        const float2 lq = *reinterpret_cast<const float2*>(kBias ? lse + bhq : lse_bh + q);
        const float2 dq = *reinterpret_cast<const float2*>(kBias ? Dsum + bhq : D_bh + q);
        float l0 = lq.x * kLog2e, l1 = lq.y * kLog2e;
        if constexpr (kMode != kKeyPadding) {                   // a query that saw no key (lse = -inf) gets P = 0, even
          l0 = lq.x == -INFINITY ? INFINITY : l0;               // where malformed bounds put it inside a key's interval
          l1 = lq.y == -INFINITY ? INFINITY : l1;
        }
        bool v00, v01, v10, v11;                                // (key row, query column)
        if constexpr (kMode == kKeyPadding) {
          v00 = v01 = vis0;
          v10 = v11 = vis1;
        } else {
          v00 = (vis >> (2 * j)) & 1u; v01 = (vis >> (2 * j + 1)) & 1u;
          v10 = (vis >> (16 + 2 * j)) & 1u; v11 = (vis >> (17 + 2 * j)) & 1u;
        }
        if constexpr (kBias) {
          st[4 * j] += lds_f32(bias_t - 32 * j); st[4 * j + 1] += lds_f32(bias_t - 32 * j - 4);
          st[4 * j + 2] += lds_f32(bias_t + 32 - 32 * j); st[4 * j + 3] += lds_f32(bias_t + 28 - 32 * j);
        }
        const float p00 = v00 ? exp2f(st[4 * j] * kSL - l0) : 0.f;
        const float p01 = v01 ? exp2f(st[4 * j + 1] * kSL - l1) : 0.f;
        const float p10 = v10 ? exp2f(st[4 * j + 2] * kSL - l0) : 0.f;
        const float p11 = v11 ? exp2f(st[4 * j + 3] * kSL - l1) : 0.f;
        pa[2 * j] = pack_bf16x2(p00, p01);
        pa[2 * j + 1] = pack_bf16x2(p10, p11);
        dsa[2 * j] = pack_bf16x2(p00 * (dpt[4 * j] - dq.x), p01 * (dpt[4 * j + 1] - dq.y));
        dsa[2 * j + 1] = pack_bf16x2(p10 * (dpt[4 * j + 2] - dq.x), p11 * (dpt[4 * j + 3] - dq.y));
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_n64_rs<1>(dv, pa + 4 * kk, desc_mn(do_addr + kk * kStepMN), 1u);   // dV += P^T dO
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_n64_rs<1>(dk, dsa + 4 * kk, desc_mn(q_addr + kk * kStepMN), 1u);  // dK += dS^T Q
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&L.empty_bar[stage]);
      if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
    }
    __nv_bfloat16* krow = dqkv + (seq_row + key) * pitch + h * kHd;
    store_frag(dk, kSc, kSc, krow + HD, pitch, c0);
    store_frag(dv, 1.f, 1.f, krow + 2 * HD, pitch, c0);
  }
}

// dQ for one tile of 128 queries.  Fixed: Q, dO.  Ring: (K, V) tiles of 64 keys below the length (kKeyPadding), or
// inside the union of the query rows' intervals (kSegment, kCausal).  kGqa: K / V from the query head's K/V head.
//
// kBias: P recomputed with the relative bias, and this CTA's share of the bias gradient: dtable_part[b, qt, h, c] =
// the sum of fp32 dS over its visible pairs at clamped distance c - 128, with no atomics.  A thread's 32 dS values of a
// 128 x 64 tile lie on 18 diagonals (slot 2 m + e: distance kt * 64 + c0 - row + 8 (m - 1) + e), which it folds in
// registers.  Slots at distance beyond +-128, and whole tiles beyond it, go to two running sums per thread (columns 0
// and 256).  For the other tiles the slots go through shared memory, where the owner of column c (consumer thread c - 1)
// adds the up to 64 slots of its diagonal in a fixed order to a register.  The tiles are walked in key order, so every
// sum has one fixed order.
template <int kMode, bool kGqa = false, bool kBias = false>
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap map_qkv, const __grid_constant__ CUtensorMap map_do,
                   const int* __restrict__ mask, int S, int H, const float* __restrict__ lse, const float* __restrict__ Dsum,
                   __nv_bfloat16* __restrict__ dqkv, int Hkv, const float* __restrict__ table, float* __restrict__ dtable_part) {
  static_assert(!kBias || (kMode != kKeyPadding && !kGqa), "the relative bias is a document-mode, multi-head instantiation");
  constexpr float kSc = kBias ? 1.f : kScale;
  constexpr float kSL = kSc * kLog2e;
  extern __shared__ uint8_t smem_raw[];
  const BwdSmem L = bwd_smem(smem_raw);
  float* tbl = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(L.fixed_bar) + 256);   // kBias: table, far-sum scratch,
  float* far_red = tbl + kFarRed;                                                           // then the two fold buffers
  float* fold = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(tbl) + kBiasTable);
  const int3 tc = tile_coords<kMode, false>();
  const int qt = tc.x, h = tc.y, b = tc.z;
  const int HD = H * kHd;
  const size_t pitch = kGqa ? (size_t)(H + 2 * Hkv) * kHd : (size_t)3 * HD;
  const size_t seq_row = (size_t)b * S;
  float* part_out = kBias ? dtable_part + (((size_t)b * (S / 128) + qt) * H + h) * kRelCols : nullptr;
  int len = 0, kt0 = 0, kt_end = 0;
  bool hidden;
  if constexpr (kMode == kKeyPadding) {
    len = clamped_len(mask, b, S);
    hidden = len == 0;
  } else {
    const int2 r = cta_range<kMode, false>(mask, seq_row + qt * 128, qt * 128, S, reinterpret_cast<int*>(L.empty_bar + kBwdStages));
    hidden = r.x >= r.y;
    kt0 = r.x / 64;
    kt_end = (r.y + 63) / 64;
  }
  if (hidden) {
    zero_rows(dqkv + h * kHd, pitch, seq_row + qt * 128, 128);
    if constexpr (kBias)
      for (int i = threadIdx.x; i < kRelCols; i += blockDim.x) part_out[i] = 0.f;
    return;
  }
  const int n_kt = kMode == kKeyPadding ? (len + 63) / 64 : kt_end - kt0;   // key tiles kt0 .. kt0 + n_kt - 1
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) bwd_init_barriers(L);
  if constexpr (kBias) load_bias_table(tbl, table, h);
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&map_qkv);
      tma_prefetch_desc(&map_do);
      if constexpr (kGqa) {
        const int2 kv = kv_cols<kGqa>(h, H, HD, Hkv);
        bwd_produce(L, &map_qkv, h * kHd, &map_do, h * kHd, (int)seq_row + qt * 128,
                    &map_qkv, kv.x, &map_qkv, kv.y, (int)seq_row + 64 * kt0, n_kt);
      } else {
        bwd_produce(L, &map_qkv, h * kHd, &map_do, h * kHd, (int)seq_row + qt * 128,
                    &map_qkv, HD + h * kHd, &map_qkv, 2 * HD + h * kHd, (int)seq_row + 64 * kt0, n_kt);
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const int row = qt * 128 + wg * 64 + r0;
    int2 qb0, qb1;                                              // kSegment / kCausal: the intervals of query rows row, row + 8
    if constexpr (kMode != kKeyPadding) {
      qb0 = mask_interval<kMode, false>(mask, seq_row + row, row, S);
      qb1 = mask_interval<kMode, false>(mask, seq_row + row + 8, row + 8, S);
    }
    const uint32_t q_addr = smem_u32(L.fixed0 + wg * kBoxBytes), do_addr = smem_u32(L.fixed1 + wg * kBoxBytes);
    const size_t bh = ((size_t)b * H + h) * S;
    const float l0 = lse[bh + row] * kLog2e, l1 = lse[bh + row + 8] * kLog2e;
    const float d0 = Dsum[bh + row], d1 = Dsum[bh + row + 8];
    float dq[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] = 0.f;
    const int u = threadIdx.x - 128;                            // kBias: consumer thread index; owns column u + 1 (u < 255)
    float col_sum = 0.f, far_lo = 0.f, far_hi = 0.f;            // kBias: column u + 1, columns 0 and 256
    mbar_wait(L.fixed_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
      mbar_wait(&L.full_bar[stage], phase);
      const uint32_t k_addr = smem_u32(L.ring + stage * 2 * kBoxBytes), v_addr = k_addr + kBoxBytes;
      float s[32], dp[32];
      wgmma_fence();
      mma_hd_n64(s, q_addr, k_addr);                            // S = Q K^T
      mma_hd_n64(dp, do_addr, v_addr);                          // dP = dO V^T
      wgmma_commit();
      wgmma_wait<0>();
      const int tile_rel = kt * 64 - qt * 128;                  // distance of the tile's key 0 from its query 0
      if constexpr (kBias) add_rel_bias<8, 1, -8>(s, tbl, tile_rel + c0 - (wg * 64 + r0));
      float slot[18];
#pragma unroll
      for (int t = 0; t < 18; ++t) slot[t] = 0.f;
      uint32_t dsa[16];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k0 = kt * 64 + 8 * j + c0;
        bool v00, v01, v10, v11;                                // (query row, key column)
        if constexpr (kMode == kKeyPadding) {
          v00 = v10 = k0 < len;
          v01 = v11 = k0 + 1 < len;
        } else {
          v00 = inside(k0, qb0); v01 = inside(k0 + 1, qb0);
          v10 = inside(k0, qb1); v11 = inside(k0 + 1, qb1);
        }
        const float p00 = v00 ? exp2f(s[4 * j] * kSL - l0) : 0.f;
        const float p01 = v01 ? exp2f(s[4 * j + 1] * kSL - l0) : 0.f;
        const float p10 = v10 ? exp2f(s[4 * j + 2] * kSL - l1) : 0.f;
        const float p11 = v11 ? exp2f(s[4 * j + 3] * kSL - l1) : 0.f;
        if constexpr (kBias) {
          const float ds00 = p00 * (dp[4 * j] - d0), ds01 = p01 * (dp[4 * j + 1] - d0);
          const float ds10 = p10 * (dp[4 * j + 2] - d1), ds11 = p11 * (dp[4 * j + 3] - d1);
          dsa[2 * j] = pack_bf16x2(ds00, ds01);
          dsa[2 * j + 1] = pack_bf16x2(ds10, ds11);
          slot[2 * j + 2] += ds00; slot[2 * j + 3] += ds01;     // row r0: m = j + 1
          slot[2 * j] += ds10; slot[2 * j + 1] += ds11;         // row r0 + 8: m = j
        } else {
          dsa[2 * j] = pack_bf16x2(p00 * (dp[4 * j] - d0), p01 * (dp[4 * j + 1] - d0));
          dsa[2 * j + 1] = pack_bf16x2(p10 * (dp[4 * j + 2] - d1), p11 * (dp[4 * j + 3] - d1));
        }
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_n64_rs<1>(dq, dsa + 4 * kk, desc_mn(k_addr + kk * kStepMN), 1u);  // dQ += dS K
      wgmma_commit();
      if constexpr (kBias) {
        if (tile_rel + 63 <= -kRelMax) {                        // the whole tile lies at distance <= -128 (CTA-uniform)
#pragma unroll
          for (int t = 0; t < 18; ++t) far_lo += slot[t];
        } else if (tile_rel - 127 >= kRelMax) {                 // ... or >= 128
#pragma unroll
          for (int t = 0; t < 18; ++t) far_hi += slot[t];
        } else {
          float* buf = fold + (kt & 1) * 256 * kPartStride;
          const int d_slot0 = tile_rel + c0 - (wg * 64 + r0) - 8;
#pragma unroll
          for (int t = 0; t < 18; ++t) {
            const int d = d_slot0 + 8 * (t >> 1) + (t & 1);
            if (d <= -kRelMax) far_lo += slot[t];
            else if (d >= kRelMax) far_hi += slot[t];
            buf[u * kPartStride + t] = slot[t];
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");        // the consumer warpgroups' slots are in buf
          // Column u + 1 is tile diagonal dl = key - row (tile-local).  The thread group of warp w, quad q (rows
          // 16 w + q and 16 w + q + 8) holds it at kk = 16 w + q + dl + 8 if that lies in [0, 72): lane 4 q + (kk & 7) / 2,
          // slot 2 (kk >> 3) + (kk & 1).  Only the quads in that range are visited, in increasing (w, q).
          const int dl = u - (kRelMax - 1) - tile_rel;
          if (u < 2 * kRelMax - 1 && dl >= -127 && dl <= 63) {
            for (int w = 0; w < 8; ++w) {
              const int kk0 = 16 * w + dl + 8;
              for (int kk = max(kk0, 0); kk < min(kk0 + 8, 72); ++kk)
                col_sum += buf[(32 * w + 4 * (kk - kk0) + ((kk & 7) >> 1)) * kPartStride + 2 * (kk >> 3) + (kk & 1)];
            }
          }
        }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&L.empty_bar[stage]);
      if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
    }
    store_frag(dq, kSc, kSc, dqkv + (seq_row + row) * pitch + h * kHd, pitch, c0);
    if constexpr (kBias) {
      if (u < 2 * kRelMax - 1) part_out[u + 1] = col_sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        far_lo += __shfl_xor_sync(0xffffffffu, far_lo, o);
        far_hi += __shfl_xor_sync(0xffffffffu, far_hi, o);
      }
      if (lane == 0) { far_red[warp - 4] = far_lo; far_red[8 + warp - 4] = far_hi; }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (u == 0) {
        float lo = 0.f, hi = 0.f;
        for (int w = 0; w < 8; ++w) { lo += far_red[w]; hi += far_red[8 + w]; }
        part_out[0] = lo;
        part_out[2 * kRelMax] = hi;
      }
    }
  }
}

// ============================================== head dim 128 (kCausal, grouped-query) ================================
// The same causal-document contract, grid walk and determinism as the kernels above, at d = 128 for
// qkv [B*S, (H + 2*Hkv)*128] (Hkv == H is multi-head attention).  A TMA box row is at most one 128-byte swizzle row, so a
// tile of R rows x 128 columns is two R x 64 chunks side by side in shared memory, chunk 1 at R * 128 bytes: Q K^T walks
// eight k16 steps, four per chunk, and an N = 128 product (P V, dS K, P^T dO, dS^T Q) is one wgmma n64 per chunk into two
// 32-register accumulator halves.  The tiles are those of d = 64; the accumulators double (forward O: 64 registers,
// dQ: 64, dK + dV: 128), which does not fit the 168 registers a thread gets at 384 threads and one CTA per SM.  So the
// producer warpgroup, which needs few, gives registers back (setmaxnreg: 40) and the two consumer warpgroups take them
// (232 each: 40 * 128 + 232 * 256 = 168 * 384).
constexpr int kHd128 = 128;
constexpr float kScale128 = 0.08838834764831845f;              // 1/sqrt(128)
constexpr float kScale128Log2 = kScale128 * kLog2e;
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kFwd128Smem = 1024 + 4 * kBoxBytes + kFwdStages * 8 * kBoxBytes + 256;   // Q 128 x 128 + ring of (K, V) 128 x 128
constexpr int kBwd128Smem = 1024 + 8 * kBoxBytes + kBwdStages * 4 * kBoxBytes + 256;   // fixed 2 x (128 x 128) + ring of 2 x (64 x 128)

// S (+)= A B^T over d = 128: A and B K-major tiles of 64 rows, chunk 1 at a + a_chunk and b + b_chunk bytes
__device__ __forceinline__ void mma_hd128_n64(float (&acc)[32], uint32_t a, uint32_t a_chunk, uint32_t b, uint32_t b_chunk) {
#pragma unroll
  for (int k = 0; k < kHd128 / 16; ++k)
    wgmma_n64<0, 0>(acc, desc_k(a + (k >> 2) * a_chunk + (k & 3) * kStepK), desc_k(b + (k >> 2) * b_chunk + (k & 3) * kStepK),
                    k != 0 ? 1u : 0u);
}
// D += A B over 16 kSteps k rows, N = 128: A the register fragments a[4 kSteps], B MN-major with chunk 1 at b + b_chunk
template <int kSteps>
__device__ __forceinline__ void mma_rs_n128(float (&d0)[32], float (&d1)[32], const uint32_t* a, uint32_t b, uint32_t b_chunk) {
#pragma unroll
  for (int kk = 0; kk < kSteps; ++kk) {
    wgmma_n64_rs<1>(d0, a + 4 * kk, desc_mn(b + kk * kStepMN), 1u);
    wgmma_n64_rs<1>(d1, a + 4 * kk, desc_mn(b + b_chunk + kk * kStepMN), 1u);
  }
}
// TMA-loads `rows` (a multiple of 64) rows x 128 columns from column col, row row into two chunks at dst, dst + rows * 128
__device__ __forceinline__ void tma_load_tile128(const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int col, int row, int rows) {
  for (int c = 0; c < 2; ++c)
    for (int r = 0; r < rows; r += kBoxRows) tma_load_2d(map, bar, dst + (c * rows + r) * 128, col + c * kHd, row + r);
}
__device__ __forceinline__ void zero_rows128(__nv_bfloat16* base, size_t pitch, size_t row0, int rows) {
  zero_rows(base, pitch, row0, rows);
  zero_rows(base + kHd, pitch, row0, rows);
}

__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_d128_kernel(const __grid_constant__ CUtensorMap map_qkv, const int* __restrict__ bounds, int S, int H,
                     __nv_bfloat16* __restrict__ o, float* __restrict__ lse, int Hkv) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sq = smem;                                           // 128 query rows x 128
  uint8_t* ring = sq + 4 * kBoxBytes;                           // stage: K 128 x 128, V 128 x 128
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(ring + kFwdStages * 8 * kBoxBytes);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kFwdStages;

  const int3 tc = tile_coords<kCausal, false>();
  const int qt = tc.x, h = tc.y, b = tc.z;
  const int HD = H * kHd128;
  const size_t seq_row = (size_t)b * S;
  const int2 r = cta_range<kCausal, false>(bounds, seq_row + qt * 128, qt * 128, S, reinterpret_cast<int*>(empty_bar + kFwdStages));
  const int kt0 = r.x / 128;
  const int n_kt = r.x < r.y ? (r.y + 127) / 128 - kt0 : 0;   // key tiles kt0 .. kt0 + n_kt - 1
  float* lse_bh = lse + ((size_t)b * H + h) * S;
  if (n_kt == 0) {
    zero_rows128(o + h * kHd128, HD, seq_row + qt * 128, 128);
    if (threadIdx.x < 128) lse_bh[qt * 128 + threadIdx.x] = -INFINITY;
    return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) {
    mbar_init(q_bar, 1);
    for (int i = 0; i < kFwdStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerArrivals); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    warpgroup_reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&map_qkv);
      const int q_row = (int)seq_row + qt * 128;
      mbar_expect_tx(q_bar, 4 * kBoxBytes);
      tma_load_tile128(&map_qkv, q_bar, sq, h * kHd128, q_row, 128);
      const int hk = h / (H / Hkv);
      const int kcol = HD + hk * kHd128, vcol = HD + (Hkv + hk) * kHd128;
      int stage = 0;
      uint32_t phase = 0;
      for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sk = ring + stage * 8 * kBoxBytes;
        mbar_expect_tx(&full_bar[stage], 8 * kBoxBytes);
        tma_load_tile128(&map_qkv, &full_bar[stage], sk, kcol, (int)seq_row + kt * 128, 128);
        tma_load_tile128(&map_qkv, &full_bar[stage], sk + 4 * kBoxBytes, vcol, (int)seq_row + kt * 128, 128);
        if (++stage == kFwdStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    warpgroup_reg_alloc<kConsumerRegs>();
    const int wg = (warp - 4) >> 2;                             // query rows [64 wg, 64 wg + 64) of the tile
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const uint32_t q_addr = smem_u32(sq + wg * kBoxBytes);      // chunk 1 at + 2 * kBoxBytes
    const int row = qt * 128 + wg * 64 + r0;                    // position in the sequence
    const int2 rb0 = mask_interval<kCausal, false>(bounds, seq_row + row, row, S);
    const int2 rb1 = mask_interval<kCausal, false>(bounds, seq_row + row + 8, row + 8, S);
    float acc0[32], acc1[32];                                   // O columns 0-63, 64-127
#pragma unroll
    for (int i = 0; i < 32; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(q_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t k_addr = smem_u32(ring + stage * 8 * kBoxBytes);   // K and V: chunk 1 at + 2 * kBoxBytes
      const uint32_t v_addr = k_addr + 4 * kBoxBytes;
      float s[64];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kHd128 / 16; ++k)
        wgmma_n128<0, 0>(s, desc_k(q_addr + (k >> 2) * 2 * kBoxBytes + (k & 3) * kStepK),
                         desc_k(k_addr + (k >> 2) * 2 * kBoxBytes + (k & 3) * kStepK), k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      const int key0 = kt * 128;
      if (key0 < max(rb0.x, rb1.x) || key0 + 128 > min(rb0.y, rb1.y)) {   // tile not wholly inside both intervals
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = key0 + 8 * j + c0 + e;
            if (!inside(key, rb0)) s[4 * j + e] = -INFINITY;
            if (!inside(key, rb1)) s[4 * j + 2 + e] = -INFINITY;
          }
        }
      }
      float mx[2] = {m[0], m[1]};
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        mx[0] = fmaxf(mx[0], fmaxf(s[4 * j], s[4 * j + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(s[4 * j + 2], s[4 * j + 3]));
      }
      float alpha[2], mb[2], rs[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
        mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
        const float base = mx[i] == -INFINITY ? 0.f : mx[i];   // no visible key yet: exp2 gives 0 rather than NaN
        alpha[i] = exp2f((m[i] - base) * kScale128Log2);
        m[i] = mx[i];
        mb[i] = base * kScale128Log2;
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        s[4 * j] = exp2f(s[4 * j] * kScale128Log2 - mb[0]);
        s[4 * j + 1] = exp2f(s[4 * j + 1] * kScale128Log2 - mb[0]);
        s[4 * j + 2] = exp2f(s[4 * j + 2] * kScale128Log2 - mb[1]);
        s[4 * j + 3] = exp2f(s[4 * j + 3] * kScale128Log2 - mb[1]);
        rs[0] += s[4 * j] + s[4 * j + 1];
        rs[1] += s[4 * j + 2] + s[4 * j + 3];
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) l[i] = l[i] * alpha[i] + rs[i];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc0[4 * j] *= alpha[0]; acc0[4 * j + 1] *= alpha[0]; acc0[4 * j + 2] *= alpha[1]; acc0[4 * j + 3] *= alpha[1];
        acc1[4 * j] *= alpha[0]; acc1[4 * j + 1] *= alpha[0]; acc1[4 * j + 2] *= alpha[1]; acc1[4 * j + 3] *= alpha[1];
      }
      // O += P V: P from registers (16 keys per k16 step), V MN-major, one n64 per 64-column chunk
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                               pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
        wgmma_n64_rs<1>(acc0, a, desc_mn(v_addr + kk * kStepMN), 1u);
        wgmma_n64_rs<1>(acc1, a, desc_mn(v_addr + 2 * kBoxBytes + kk * kStepMN), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == kFwdStages) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
      l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
    }
    const float sc0 = l[0] > 0.f ? 1.f / l[0] : 0.f, sc1 = l[1] > 0.f ? 1.f / l[1] : 0.f;   // no key seen: zeros, -inf
    __nv_bfloat16* orow = o + (seq_row + row) * HD + h * kHd128;
    store_frag(acc0, sc0, sc1, orow, HD, c0);
    store_frag(acc1, sc0, sc1, orow + kHd, HD, c0);
    if ((lane & 3) == 0) {
      lse_bh[row] = l[0] > 0.f ? m[0] * kScale128 + logf(l[0]) : -INFINITY;
      lse_bh[row + 8] = l[1] > 0.f ? m[1] * kScale128 + logf(l[1]) : -INFINITY;
    }
  }
}

// D[b, h, s] = sum_d dO[b*S + s, h*128 + d] * O[b*S + s, h*128 + d]; sixteen threads per (row, head), 16 bytes each
__global__ void attn_bwd_dot_d128_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ out, int rows,
                                         int S, int H, float* __restrict__ D) {
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t item = gid >> 4;
  const int part = (int)(gid & 15);
  const bool live = item < (size_t)rows * H;
  float acc = 0.f;
  if (live) {
    const size_t off = item * kHd128 + part * 8;              // [rows, H * 128] row-major: item = row * H + head
    float a[8], c[8];
    unpack8(*reinterpret_cast<const Bf16x8*>(dout + off), a);
    unpack8(*reinterpret_cast<const Bf16x8*>(out + off), c);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc += a[i] * c[i];
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  acc += __shfl_xor_sync(0xffffffffu, acc, 8);
  if (live && part == 0) {
    const size_t row = item / H, hh = item % H;
    const size_t b = row / S, s = row % S;
    D[(b * H + hh) * S + s] = acc;
  }
}

// Shared layout of both d = 128 backward kernels: fixed0, fixed1 of 128 x 128 (4 boxes each), then a ring of two 64 x 128
// tiles (2 boxes each) per stage.
__device__ __forceinline__ BwdSmem bwd128_smem(uint8_t* raw) {
  BwdSmem L;
  L.fixed0 = align1024(raw);
  L.fixed1 = L.fixed0 + 4 * kBoxBytes;
  L.ring = L.fixed1 + 4 * kBoxBytes;
  L.fixed_bar = reinterpret_cast<uint64_t*>(L.ring + kBwdStages * 4 * kBoxBytes);
  L.full_bar = L.fixed_bar + 1;
  L.empty_bar = L.full_bar + kBwdStages;
  return L;
}

// dK, dV for one tile of 128 keys of K/V head hk.  Fixed: K, V.  Ring: (Q, dO) tiles of 64 queries inside the union of the
// key rows' intervals, for every query head of the group in turn; the whole group accumulates in registers, so each
// dK / dV element has one writer.
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_dkdv_d128_kernel(const __grid_constant__ CUtensorMap map_qkv, const __grid_constant__ CUtensorMap map_do,
                          const int* __restrict__ bounds, int S, int H, const float* __restrict__ lse, const float* __restrict__ Dsum,
                          __nv_bfloat16* __restrict__ dqkv, int Hkv) {
  extern __shared__ uint8_t smem_raw[];
  const BwdSmem L = bwd128_smem(smem_raw);
  const int3 tc = tile_coords<kCausal, true>();
  const int kt = tc.x, hk = tc.y, b = tc.z;
  const int HD = H * kHd128;
  const size_t pitch = (size_t)(H + 2 * Hkv) * kHd128;
  const int groups = H / Hkv;                                   // query heads hk * groups + g read this K/V head
  const int kcol = HD + hk * kHd128, vcol = HD + (Hkv + hk) * kHd128;
  const size_t seq_row = (size_t)b * S;
  const int2 r = cta_range<kCausal, true>(bounds, seq_row + kt * 128, kt * 128, S, reinterpret_cast<int*>(L.empty_bar + kBwdStages));
  if (r.x >= r.y) {                                             // every key of the tile is hidden: no gradient
    zero_rows128(dqkv + kcol, pitch, seq_row + kt * 128, 128);
    zero_rows128(dqkv + vcol, pitch, seq_row + kt * 128, 128);
    return;
  }
  const int qt0 = r.x / 64, n_qt = (r.y + 63) / 64 - qt0;      // query tiles qt0 .. qt0 + n_qt - 1
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) bwd_init_barriers(L);
  __syncthreads();

  if (warp < 4) {
    warpgroup_reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&map_qkv);
      tma_prefetch_desc(&map_do);
      mbar_expect_tx(L.fixed_bar, 8 * kBoxBytes);
      tma_load_tile128(&map_qkv, L.fixed_bar, L.fixed0, kcol, (int)seq_row + kt * 128, 128);
      tma_load_tile128(&map_qkv, L.fixed_bar, L.fixed1, vcol, (int)seq_row + kt * 128, 128);
      int stage = 0;
      uint32_t phase = 0;
      for (int g = 0; g < groups; ++g) {
        const int col = (hk * groups + g) * kHd128;
        for (int i = 0; i < n_qt; ++i) {
          mbar_wait(&L.empty_bar[stage], phase ^ 1);
          uint8_t* t0 = L.ring + stage * 4 * kBoxBytes;
          mbar_expect_tx(&L.full_bar[stage], 4 * kBoxBytes);
          tma_load_tile128(&map_qkv, &L.full_bar[stage], t0, col, (int)seq_row + 64 * (qt0 + i), 64);
          tma_load_tile128(&map_do, &L.full_bar[stage], t0 + 2 * kBoxBytes, col, (int)seq_row + 64 * (qt0 + i), 64);
          if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    warpgroup_reg_alloc<kConsumerRegs>();
    const int wg = (warp - 4) >> 2;                             // keys [64 wg, 64 wg + 64) of the tile
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const int key = kt * 128 + wg * 64 + r0;
    const uint32_t k_addr = smem_u32(L.fixed0 + wg * kBoxBytes), v_addr = smem_u32(L.fixed1 + wg * kBoxBytes);   // chunk 1: + 2 boxes
    float dv0[32], dv1[32], dk0[32], dk1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv0[i] = 0.f; dv1[i] = 0.f; dk0[i] = 0.f; dk1[i] = 0.f; }
    mbar_wait(L.fixed_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    // lse / D rows of query heads hk * groups + g, with a 32-bit offset (B * H * S < 2^31)
    const int bh_end = (b * H + (hk + 1) * groups) * S;
#pragma unroll 1
    for (int bh = (b * H + hk * groups) * S; bh < bh_end; bh += S) {
      for (int qt = qt0; qt < qt0 + n_qt; ++qt) {
        const int2 kb0 = mask_interval<kCausal, true>(bounds, seq_row + key, key, S);
        const int2 kb1 = mask_interval<kCausal, true>(bounds, seq_row + key + 8, key + 8, S);
        const int q0 = qt * 64 + c0;
        const uint32_t vis = frag_mask16(kb0.x - q0, kb0.y - q0) | (frag_mask16(kb1.x - q0, kb1.y - q0) << 16);
        mbar_wait(&L.full_bar[stage], phase);
        const uint32_t q_addr = smem_u32(L.ring + stage * 4 * kBoxBytes), do_addr = q_addr + 2 * kBoxBytes;   // chunk 1: + 1 box
        // two halves of 32 queries: S^T and dP^T of a whole 64-query tile (64 registers) beside the 128 of dK and dV
        // would not fit the consumers' 232
#pragma unroll 1
        for (int half = 0; half < 2; ++half) {
          const uint32_t qh = q_addr + half * 32 * 128, doh = do_addr + half * 32 * 128;
          float st[16], dpt[16];
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kHd128 / 16; ++k) {               // S^T = K Q^T, dP^T = V dO^T   [keys, 32 queries]
            const uint32_t ko = (k >> 2) * 2 * kBoxBytes + (k & 3) * kStepK, qo = (k >> 2) * kBoxBytes + (k & 3) * kStepK;
            wgmma_n32<0, 0>(st, desc_k(k_addr + ko), desc_k(qh + qo), k != 0 ? 1u : 0u);
            wgmma_n32<0, 0>(dpt, desc_k(v_addr + ko), desc_k(doh + qo), k != 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          uint32_t pa[8], dsa[8];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {                      // query columns 32 half + 8 jj + c0, + 1
            const int j = 4 * half + jj;                        // of the tile: bits 2 j, 2 j + 1 of vis
            const int q = qt * 64 + 8 * j + c0;
            const float2 lq = *reinterpret_cast<const float2*>(lse + (bh + q));
            const float2 dq = *reinterpret_cast<const float2*>(Dsum + (bh + q));
            const float l0 = lq.x == -INFINITY ? INFINITY : lq.x * kLog2e;   // a query that saw no key gets P = 0
            const float l1 = lq.y == -INFINITY ? INFINITY : lq.y * kLog2e;
            const bool v00 = (vis >> (2 * j)) & 1u, v01 = (vis >> (2 * j + 1)) & 1u;
            const bool v10 = (vis >> (16 + 2 * j)) & 1u, v11 = (vis >> (17 + 2 * j)) & 1u;
            const float p00 = v00 ? exp2f(st[4 * jj] * kScale128Log2 - l0) : 0.f;
            const float p01 = v01 ? exp2f(st[4 * jj + 1] * kScale128Log2 - l1) : 0.f;
            const float p10 = v10 ? exp2f(st[4 * jj + 2] * kScale128Log2 - l0) : 0.f;
            const float p11 = v11 ? exp2f(st[4 * jj + 3] * kScale128Log2 - l1) : 0.f;
            pa[2 * jj] = pack_bf16x2(p00, p01);
            pa[2 * jj + 1] = pack_bf16x2(p10, p11);
            dsa[2 * jj] = pack_bf16x2(p00 * (dpt[4 * jj] - dq.x), p01 * (dpt[4 * jj + 1] - dq.y));
            dsa[2 * jj + 1] = pack_bf16x2(p10 * (dpt[4 * jj + 2] - dq.x), p11 * (dpt[4 * jj + 3] - dq.y));
          }
          wgmma_fence();
          mma_rs_n128<2>(dv0, dv1, pa, doh, kBoxBytes);        // dV += P^T dO
          mma_rs_n128<2>(dk0, dk1, dsa, qh, kBoxBytes);        // dK += dS^T Q
          wgmma_commit();
          wgmma_wait<0>();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&L.empty_bar[stage]);
        if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
      }
    }
    __nv_bfloat16* krow = dqkv + (seq_row + key) * pitch + kcol;
    store_frag(dk0, kScale128, kScale128, krow, pitch, c0);
    store_frag(dk1, kScale128, kScale128, krow + kHd, pitch, c0);
    store_frag(dv0, 1.f, 1.f, krow + (vcol - kcol), pitch, c0);
    store_frag(dv1, 1.f, 1.f, krow + (vcol - kcol) + kHd, pitch, c0);
  }
}

// dQ for one tile of 128 queries.  Fixed: Q, dO.  Ring: (K, V) tiles of 64 keys of the query head's K/V head inside the
// union of the query rows' intervals.
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_dq_d128_kernel(const __grid_constant__ CUtensorMap map_qkv, const __grid_constant__ CUtensorMap map_do,
                        const int* __restrict__ bounds, int S, int H, const float* __restrict__ lse, const float* __restrict__ Dsum,
                        __nv_bfloat16* __restrict__ dqkv, int Hkv) {
  extern __shared__ uint8_t smem_raw[];
  const BwdSmem L = bwd128_smem(smem_raw);
  const int3 tc = tile_coords<kCausal, false>();
  const int qt = tc.x, h = tc.y, b = tc.z;
  const int HD = H * kHd128;
  const size_t pitch = (size_t)(H + 2 * Hkv) * kHd128;
  const size_t seq_row = (size_t)b * S;
  const int2 r = cta_range<kCausal, false>(bounds, seq_row + qt * 128, qt * 128, S, reinterpret_cast<int*>(L.empty_bar + kBwdStages));
  if (r.x >= r.y) {
    zero_rows128(dqkv + h * kHd128, pitch, seq_row + qt * 128, 128);
    return;
  }
  const int kt0 = r.x / 64, n_kt = (r.y + 63) / 64 - kt0;      // key tiles kt0 .. kt0 + n_kt - 1
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) bwd_init_barriers(L);
  __syncthreads();

  if (warp < 4) {
    warpgroup_reg_dealloc<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      tma_prefetch_desc(&map_qkv);
      tma_prefetch_desc(&map_do);
      mbar_expect_tx(L.fixed_bar, 8 * kBoxBytes);
      tma_load_tile128(&map_qkv, L.fixed_bar, L.fixed0, h * kHd128, (int)seq_row + qt * 128, 128);
      tma_load_tile128(&map_do, L.fixed_bar, L.fixed1, h * kHd128, (int)seq_row + qt * 128, 128);
      const int hk = h / (H / Hkv);
      const int kcol = HD + hk * kHd128, vcol = HD + (Hkv + hk) * kHd128;
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < n_kt; ++i) {
        mbar_wait(&L.empty_bar[stage], phase ^ 1);
        uint8_t* t0 = L.ring + stage * 4 * kBoxBytes;
        mbar_expect_tx(&L.full_bar[stage], 4 * kBoxBytes);
        tma_load_tile128(&map_qkv, &L.full_bar[stage], t0, kcol, (int)seq_row + 64 * (kt0 + i), 64);
        tma_load_tile128(&map_qkv, &L.full_bar[stage], t0 + 2 * kBoxBytes, vcol, (int)seq_row + 64 * (kt0 + i), 64);
        if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    warpgroup_reg_alloc<kConsumerRegs>();
    const int wg = (warp - 4) >> 2;
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const int row = qt * 128 + wg * 64 + r0;
    const int2 qb0 = mask_interval<kCausal, false>(bounds, seq_row + row, row, S);
    const int2 qb1 = mask_interval<kCausal, false>(bounds, seq_row + row + 8, row + 8, S);
    const uint32_t q_addr = smem_u32(L.fixed0 + wg * kBoxBytes), do_addr = smem_u32(L.fixed1 + wg * kBoxBytes);   // chunk 1: + 2 boxes
    const size_t bh = ((size_t)b * H + h) * S;
    const float l0 = lse[bh + row] * kLog2e, l1 = lse[bh + row + 8] * kLog2e;
    const float d0 = Dsum[bh + row], d1 = Dsum[bh + row + 8];
    float dq0[32], dq1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dq0[i] = 0.f; dq1[i] = 0.f; }
    mbar_wait(L.fixed_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
      mbar_wait(&L.full_bar[stage], phase);
      const uint32_t k_addr = smem_u32(L.ring + stage * 4 * kBoxBytes), v_addr = k_addr + 2 * kBoxBytes;   // chunk 1: + 1 box
      float s[32], dp[32];
      wgmma_fence();
      mma_hd128_n64(s, q_addr, 2 * kBoxBytes, k_addr, kBoxBytes);      // S = Q K^T
      mma_hd128_n64(dp, do_addr, 2 * kBoxBytes, v_addr, kBoxBytes);    // dP = dO V^T
      wgmma_commit();
      wgmma_wait<0>();
      uint32_t dsa[16];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k0 = kt * 64 + 8 * j + c0;
        const float p00 = inside(k0, qb0) ? exp2f(s[4 * j] * kScale128Log2 - l0) : 0.f;
        const float p01 = inside(k0 + 1, qb0) ? exp2f(s[4 * j + 1] * kScale128Log2 - l0) : 0.f;
        const float p10 = inside(k0, qb1) ? exp2f(s[4 * j + 2] * kScale128Log2 - l1) : 0.f;
        const float p11 = inside(k0 + 1, qb1) ? exp2f(s[4 * j + 3] * kScale128Log2 - l1) : 0.f;
        dsa[2 * j] = pack_bf16x2(p00 * (dp[4 * j] - d0), p01 * (dp[4 * j + 1] - d0));
        dsa[2 * j + 1] = pack_bf16x2(p10 * (dp[4 * j + 2] - d1), p11 * (dp[4 * j + 3] - d1));
      }
      wgmma_fence();
      mma_rs_n128<4>(dq0, dq1, dsa, k_addr, kBoxBytes);        // dQ += dS K
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&L.empty_bar[stage]);
      if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
    }
    __nv_bfloat16* qrow = dqkv + (seq_row + row) * pitch + h * kHd128;
    store_frag(dq0, kScale128, kScale128, qrow, pitch, c0);
    store_frag(dq1, kScale128, kScale128, qrow + kHd, pitch, c0);
  }
}


// heads query heads and kv_heads K/V heads (equal for multi-head attention; a divisor of heads for GQA) of width hd
void check_shape(const char* who, int B, int S, int heads, int kv_heads, int hd = kHd) {
  if (B < 1 || heads < 1 || S < 128 || S % 128 != 0)
    throw std::runtime_error(std::string(who) + ": needs B >= 1, heads >= 1 and S a positive multiple of 128 (got B=" +
                             std::to_string(B) + ", S=" + std::to_string(S) + ", heads=" + std::to_string(heads) + ")");
  if (kv_heads < 1 || heads % kv_heads != 0)
    throw std::runtime_error(std::string(who) + ": kv_heads must divide heads (got heads=" + std::to_string(heads) +
                             ", kv_heads=" + std::to_string(kv_heads) + ")");
  if (B > 65535 || (long long)B * S * (heads + 2 * kv_heads) * hd >= (1ll << 31))
    throw std::runtime_error(std::string(who) + ": problem too large");
}

template <int kMode, bool kGqa = false>
void attention_fwd(const char* who, const void* qkv, const int* mask, int B, int S, int heads, void* o, float* lse, cudaStream_t s,
                   int kv_heads) {
  check_shape(who, B, S, heads, kv_heads);
  const CUtensorMap map_qkv = rows_map(qkv, B * S, (heads + 2 * kv_heads) * kHd);
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(attn_fwd_kernel<kMode, kGqa>, kFwdSmem, configured);
  attn_fwd_kernel<kMode, kGqa><<<dim3(S / 128, heads, B), kThreads, kFwdSmem, s>>>(
      map_qkv, mask, S, heads, reinterpret_cast<__nv_bfloat16*>(o), lse, kv_heads, nullptr);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

template <int kMode, bool kGqa = false>
void attention_bwd(const char* who, const void* dout, const void* qkv, const void* o, const float* lse, const int* mask, int B,
                   int S, int heads, float* dsum, void* dqkv, cudaStream_t s, int kv_heads) {
  check_shape(who, B, S, heads, kv_heads);
  const int rows = B * S;
  const long long items = (long long)rows * heads * 8;
  attn_bwd_dot_kernel<<<ceil_div(items, 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dout),
                                                           reinterpret_cast<const __nv_bfloat16*>(o), rows, S, heads, dsum);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  const CUtensorMap map_qkv = rows_map(qkv, rows, (heads + 2 * kv_heads) * kHd);
  const CUtensorMap map_do = rows_map(dout, rows, heads * kHd);
  auto* dq = reinterpret_cast<__nv_bfloat16*>(dqkv);
  static std::atomic<unsigned long long> configured_dkdv{0}, configured_dq{0};
  ensure_max_dynamic_smem(attn_bwd_dkdv_kernel<kMode, kGqa>, kBwdSmem, configured_dkdv);
  ensure_max_dynamic_smem(attn_bwd_dq_kernel<kMode, kGqa>, kBwdSmem, configured_dq);
  // dK / dV: one CTA per (key tile, K/V head, batch)
  attn_bwd_dkdv_kernel<kMode, kGqa><<<dim3(S / 128, kGqa ? kv_heads : heads, B), kThreads, kBwdSmem, s>>>(
      map_qkv, map_do, mask, S, heads, lse, dsum, dq, kv_heads, nullptr);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  attn_bwd_dq_kernel<kMode, kGqa><<<dim3(S / 128, heads, B), kThreads, kBwdSmem, s>>>(
      map_qkv, map_do, mask, S, heads, lse, dsum, dq, kv_heads, nullptr, nullptr);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

// ---- relative position bias (T5) ----
constexpr int kRelFwdSmem = kFwdSmem + kBiasTable;
constexpr int kRelDkdvSmem = kBwdSmem + kBiasTable;
constexpr int kRelDqSmem = kBwdSmem + kBiasTable + kPartBytes;

// dtable[h, c] = sum over (b, query tile) of part[b, qt, h, c], in that order
__global__ void rel_bias_finish_kernel(const float* __restrict__ part, int n, int H, float* __restrict__ dtable) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;          // h * 257 + c
  if (i >= H * kRelCols) return;
  float acc = 0.f;
  for (int k = 0; k < n; ++k) acc += part[(size_t)k * H * kRelCols + i];
  dtable[i] = acc;
}

// table[h, c] = weight[bucket[c], h]: weight [num_buckets, H] fp32 or bf16
template <typename T>
__global__ void rel_table_gather_kernel(const T* __restrict__ weight, const int* __restrict__ bucket, int H, float* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * kRelCols) return;
  const int h = i / kRelCols, c = i - h * kRelCols;
  table[i] = static_cast<float>(weight[(size_t)__ldg(bucket + c) * H + h]);
}

// dweight[k, h] = sum of dtable[h, c] over the columns c of bucket k, in increasing c (one writer per element)
template <typename T>
__global__ void rel_table_fold_kernel(const float* __restrict__ dtable, const int* __restrict__ bucket, int num_buckets, int H,
                                      T* __restrict__ dweight) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;          // k * H + h
  if (i >= num_buckets * H) return;
  const int k = i / H, h = i - k * H;
  float acc = 0.f;
  for (int c = 0; c < kRelCols; ++c)
    if (__ldg(bucket + c) == k) acc += dtable[(size_t)h * kRelCols + c];
  dweight[i] = static_cast<T>(acc);
}

template <int kMode>
void relative_fwd(const char* who, const void* qkv, const int* bounds, const float* table, int B, int S, int heads, void* o,
                  float* lse, cudaStream_t s) {
  check_shape(who, B, S, heads, heads);
  const CUtensorMap map_qkv = rows_map(qkv, B * S, 3 * heads * kHd);
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(attn_fwd_kernel<kMode, false, true>, kRelFwdSmem, configured);
  attn_fwd_kernel<kMode, false, true><<<dim3(S / 128, heads, B), kThreads, kRelFwdSmem, s>>>(
      map_qkv, bounds, S, heads, reinterpret_cast<__nv_bfloat16*>(o), lse, heads, table);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

template <int kMode>
void relative_bwd(const char* who, const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds,
                  const float* table, int B, int S, int heads, float* dsum, float* dtable_part, void* dqkv, float* dtable,
                  cudaStream_t s) {
  check_shape(who, B, S, heads, heads);
  const int rows = B * S;
  const long long items = (long long)rows * heads * 8;
  attn_bwd_dot_kernel<<<ceil_div(items, 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dout),
                                                           reinterpret_cast<const __nv_bfloat16*>(o), rows, S, heads, dsum);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  const CUtensorMap map_qkv = rows_map(qkv, rows, 3 * heads * kHd);
  const CUtensorMap map_do = rows_map(dout, rows, heads * kHd);
  auto* dq = reinterpret_cast<__nv_bfloat16*>(dqkv);
  static std::atomic<unsigned long long> configured_dkdv{0}, configured_dq{0};
  ensure_max_dynamic_smem(attn_bwd_dkdv_kernel<kMode, false, true>, kRelDkdvSmem, configured_dkdv);
  ensure_max_dynamic_smem(attn_bwd_dq_kernel<kMode, false, true>, kRelDqSmem, configured_dq);
  attn_bwd_dkdv_kernel<kMode, false, true><<<dim3(S / 128, heads, B), kThreads, kRelDkdvSmem, s>>>(
      map_qkv, map_do, bounds, S, heads, lse, dsum, dq, heads, table);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  attn_bwd_dq_kernel<kMode, false, true><<<dim3(S / 128, heads, B), kThreads, kRelDqSmem, s>>>(
      map_qkv, map_do, bounds, S, heads, lse, dsum, dq, heads, table, dtable_part);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  rel_bias_finish_kernel<<<ceil_div((long long)heads * kRelCols, 256), 256, 0, s>>>(dtable_part, B * (S / 128), heads, dtable);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace

void launch_relative_attention_fwd(const void* qkv, const int* bounds, const float* table, int B, int S, int heads, bool causal,
                                   void* o, float* lse, cudaStream_t s) {
  if (causal) relative_fwd<kCausal>("relative_attention_fwd", qkv, bounds, table, B, S, heads, o, lse, s);
  else relative_fwd<kSegment>("relative_attention_fwd", qkv, bounds, table, B, S, heads, o, lse, s);
}

void launch_relative_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds,
                                   const float* table, int B, int S, int heads, bool causal, float* dsum, float* dtable_part,
                                   void* dqkv, float* dtable, cudaStream_t s) {
  if (causal)
    relative_bwd<kCausal>("relative_attention_bwd", dout, qkv, o, lse, bounds, table, B, S, heads, dsum, dtable_part, dqkv, dtable, s);
  else
    relative_bwd<kSegment>("relative_attention_bwd", dout, qkv, o, lse, bounds, table, B, S, heads, dsum, dtable_part, dqkv, dtable, s);
}

void launch_relative_table_fwd(const void* weight, bool bf16, const int* bucket, int heads, float* table, cudaStream_t s) {
  const int n = heads * kRelCols;
  if (bf16)
    rel_table_gather_kernel<<<ceil_div(n, 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(weight), bucket, heads, table);
  else
    rel_table_gather_kernel<<<ceil_div(n, 256), 256, 0, s>>>(reinterpret_cast<const float*>(weight), bucket, heads, table);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_relative_table_bwd(const float* dtable, const int* bucket, int num_buckets, int heads, bool bf16, void* dweight,
                               cudaStream_t s) {
  const int n = num_buckets * heads;
  if (bf16)
    rel_table_fold_kernel<<<ceil_div(n, 256), 256, 0, s>>>(dtable, bucket, num_buckets, heads, reinterpret_cast<__nv_bfloat16*>(dweight));
  else
    rel_table_fold_kernel<<<ceil_div(n, 256), 256, 0, s>>>(dtable, bucket, num_buckets, heads, reinterpret_cast<float*>(dweight));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_causal_attention_d128_fwd(const void* qkv, const int* bounds, int B, int S, int heads, int kv_heads, void* o, float* lse, cudaStream_t s) {
  check_shape("causal_attention_d128_fwd", B, S, heads, kv_heads, kHd128);
  const CUtensorMap map_qkv = rows_map(qkv, B * S, (heads + 2 * kv_heads) * kHd128);
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(attn_fwd_d128_kernel, kFwd128Smem, configured);
  attn_fwd_d128_kernel<<<dim3(S / 128, heads, B), kThreads, kFwd128Smem, s>>>(map_qkv, bounds, S, heads,
                                                                              reinterpret_cast<__nv_bfloat16*>(o), lse, kv_heads);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_causal_attention_d128_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                      int S, int heads, int kv_heads, float* dsum, void* dqkv, cudaStream_t s) {
  check_shape("causal_attention_d128_bwd", B, S, heads, kv_heads, kHd128);
  const int rows = B * S;
  const long long items = (long long)rows * heads * 16;
  attn_bwd_dot_d128_kernel<<<ceil_div(items, 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dout),
                                                                reinterpret_cast<const __nv_bfloat16*>(o), rows, S, heads, dsum);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  const CUtensorMap map_qkv = rows_map(qkv, rows, (heads + 2 * kv_heads) * kHd128);
  const CUtensorMap map_do = rows_map(dout, rows, heads * kHd128);
  auto* dq = reinterpret_cast<__nv_bfloat16*>(dqkv);
  static std::atomic<unsigned long long> configured_dkdv{0}, configured_dq{0};
  ensure_max_dynamic_smem(attn_bwd_dkdv_d128_kernel, kBwd128Smem, configured_dkdv);
  ensure_max_dynamic_smem(attn_bwd_dq_d128_kernel, kBwd128Smem, configured_dq);
  attn_bwd_dkdv_d128_kernel<<<dim3(S / 128, kv_heads, B), kThreads, kBwd128Smem, s>>>(map_qkv, map_do, bounds, S, heads, lse, dsum,
                                                                                       dq, kv_heads);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  attn_bwd_dq_d128_kernel<<<dim3(S / 128, heads, B), kThreads, kBwd128Smem, s>>>(map_qkv, map_do, bounds, S, heads, lse, dsum, dq,
                                                                                  kv_heads);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_attention_fwd(const void* qkv, const int* seq_lens, int B, int S, int heads, void* o, float* lse, cudaStream_t s) {
  attention_fwd<kKeyPadding>("attention_fwd", qkv, seq_lens, B, S, heads, o, lse, s, heads);
}

void launch_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* seq_lens, int B, int S,
                          int heads, float* dsum, void* dqkv, cudaStream_t s) {
  attention_bwd<kKeyPadding>("attention_bwd", dout, qkv, o, lse, seq_lens, B, S, heads, dsum, dqkv, s, heads);
}

void launch_packed_attention_fwd(const void* qkv, const int* bounds, int B, int S, int heads, void* o, float* lse, cudaStream_t s) {
  attention_fwd<kSegment>("packed_attention_fwd", qkv, bounds, B, S, heads, o, lse, s, heads);
}

void launch_packed_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                 int S, int heads, float* dsum, void* dqkv, cudaStream_t s) {
  attention_bwd<kSegment>("packed_attention_bwd", dout, qkv, o, lse, bounds, B, S, heads, dsum, dqkv, s, heads);
}

void launch_causal_attention_fwd(const void* qkv, const int* bounds, int B, int S, int heads, void* o, float* lse, cudaStream_t s) {
  attention_fwd<kCausal>("causal_attention_fwd", qkv, bounds, B, S, heads, o, lse, s, heads);
}

void launch_causal_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                 int S, int heads, float* dsum, void* dqkv, cudaStream_t s) {
  attention_bwd<kCausal>("causal_attention_bwd", dout, qkv, o, lse, bounds, B, S, heads, dsum, dqkv, s, heads);
}

void launch_causal_gqa_attention_fwd(const void* qkv, const int* bounds, int B, int S, int heads, int kv_heads, void* o, float* lse,
                                     cudaStream_t s) {
  attention_fwd<kCausal, true>("causal_gqa_attention_fwd", qkv, bounds, B, S, heads, o, lse, s, kv_heads);
}

void launch_causal_gqa_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                     int S, int heads, int kv_heads, float* dsum, void* dqkv, cudaStream_t s) {
  attention_bwd<kCausal, true>("causal_gqa_attention_bwd", dout, qkv, o, lse, bounds, B, S, heads, dsum, dqkv, s, kv_heads);
}

}  // namespace b200
