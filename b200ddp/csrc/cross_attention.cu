// Cross-attention on the Hopper tensor cores (an encoder-decoder's decoder queries attending to the encoder output), head
// dim 64, softmax scale 1/8, bf16.
//
//   q    bf16 [B*Sq, H*64]     the query projection's output, head h at h*64 .. h*64+63
//   kv   bf16 [B*Sk, 2*H*64]   the fused key | value projection of the other sequence: K block first, then V
//   o    bf16 [B*Sq, H*64]     written in the layout the output projection reads
//   lse  fp32 [B, H, Sq]       natural-log row log-sum-exp of the scaled scores (-inf for a query that sees no key)
//
// Sq and Sk are multiples of 128 and may differ.  The mask is two interval lists over the same block structure as the
// segment mode of attention.cu, one per side:
//   q_bounds  int32 [B*Sq, 2]  query i of row b sees key j of row b iff start <= j < end (clamped to [0, Sk])
//   kv_bounds int32 [B*Sk, 2]  key j of row b is seen by queries [start, end) of row b (clamped to [0, Sq])
// The two must describe the same mask (checking it would take a host synchronisation, so the kernels trust it).  A query
// with an empty interval gets o = 0, lse = -inf and dQ = 0; a key no query sees gets dK = dV = 0.
//
// The kernels are those of attention.cu's segment mode with Q, K / V and dO read through separate tensor maps and the
// two sides indexed by their own lengths.  Each CTA visits only the tiles inside the union of its 128 rows' intervals.
//   cross_fwd   CTA = (query tile of 128, head, row); K / V tiles of 128 keys through a 2-stage ring, online softmax in
//               fp32 registers, P kept in registers as the A operand of P V.
//   attn_bwd_dot (attention_common.cuh) D = rowsum(dO * O) over [B*Sq, H*64].
//   cross_dkdv  CTA = (key tile of 128, head, row); ring of (Q, dO) tiles of 64 queries inside the keys' kv_bounds union,
//               masked with the key rows' own intervals.
//   cross_dq    CTA = (query tile of 128, head, row); ring of (K, V) tiles of 64 keys inside the queries' q_bounds union.
// No atomics: every output element has one writer, so two runs give bitwise-equal gradients.  Nothing is read back to
// the host.
#include "attention_common.cuh"

namespace b200 {
namespace {

// ============================================== forward ==============================================================
__global__ void __launch_bounds__(kThreads, 1)
cross_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv, const int* __restrict__ q_bounds,
                 int Sq, int Sk, int H, __nv_bfloat16* __restrict__ o, float* __restrict__ lse) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sq = smem;                                           // 128 query rows
  uint8_t* ring = sq + 2 * kBoxBytes;                           // stage: K 128 rows, V 128 rows
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(ring + kFwdStages * 4 * kBoxBytes);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kFwdStages;

  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int HD = H * kHd;
  const size_t q_seq = (size_t)b * Sq, k_seq = (size_t)b * Sk;
  const int2 r = cta_range<kSegment, false>(q_bounds, q_seq + qt * 128, qt * 128, Sk, reinterpret_cast<int*>(empty_bar + kFwdStages));
  const int kt0 = r.x / 128;
  const int n_kt = r.x < r.y ? (r.y + 127) / 128 - kt0 : 0;   // key tiles kt0 .. kt0 + n_kt - 1
  float* lse_bh = lse + ((size_t)b * H + h) * Sq;
  if (n_kt == 0) {                                              // no visible key: zero output, empty log-sum-exp
    zero_rows(o + h * kHd, HD, q_seq + qt * 128, 128);
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

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&map_q);
      tma_prefetch_desc(&map_kv);
      const int q_row = (int)q_seq + qt * 128;
      mbar_expect_tx(q_bar, 2 * kBoxBytes);
      tma_load_2d(&map_q, q_bar, sq, h * kHd, q_row);
      tma_load_2d(&map_q, q_bar, sq + kBoxBytes, h * kHd, q_row + 64);
      int stage = 0;
      uint32_t phase = 0;
      for (int kt = kt0; kt < kt0 + n_kt; ++kt) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sk = ring + stage * 4 * kBoxBytes;
        uint8_t* sv = sk + 2 * kBoxBytes;
        const int k_row = (int)k_seq + kt * 128;
        mbar_expect_tx(&full_bar[stage], 4 * kBoxBytes);
        tma_load_2d(&map_kv, &full_bar[stage], sk, h * kHd, k_row);
        tma_load_2d(&map_kv, &full_bar[stage], sk + kBoxBytes, h * kHd, k_row + 64);
        tma_load_2d(&map_kv, &full_bar[stage], sv, HD + h * kHd, k_row);
        tma_load_2d(&map_kv, &full_bar[stage], sv + kBoxBytes, HD + h * kHd, k_row + 64);
        if (++stage == kFwdStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;                             // query rows [64 wg, 64 wg + 64) of the tile
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);         // this thread's rows: r0 and r0 + 8 of the warpgroup's 64
    const int c0 = 2 * (lane & 3);
    const uint32_t q_addr = smem_u32(sq + wg * kBoxBytes);
    const int row = qt * 128 + wg * 64 + r0;                    // query position
    const int2 rb0 = row_bounds(q_bounds, q_seq + row, Sk), rb1 = row_bounds(q_bounds, q_seq + row + 8, Sk);
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
        // a row may have seen no visible key yet (mx = -inf): subtract 0 instead, so exp2 gives 0 rather than NaN
        const float base = mx[i] == -INFINITY ? 0.f : mx[i];
        alpha[i] = exp2f((m[i] - base) * kScaleLog2);
        m[i] = mx[i];
        mb[i] = base * kScaleLog2;
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        s[4 * j] = exp2f(s[4 * j] * kScaleLog2 - mb[0]);
        s[4 * j + 1] = exp2f(s[4 * j + 1] * kScaleLog2 - mb[0]);
        s[4 * j + 2] = exp2f(s[4 * j + 2] * kScaleLog2 - mb[1]);
        s[4 * j + 3] = exp2f(s[4 * j + 3] * kScaleLog2 - mb[1]);
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
    // a row that saw no key: zeros and -inf
    store_frag(acc, l[0] > 0.f ? 1.f / l[0] : 0.f, l[1] > 0.f ? 1.f / l[1] : 0.f, o + (q_seq + row) * HD + h * kHd, HD, c0);
    if ((lane & 3) == 0) {
      lse_bh[row] = l[0] > 0.f ? m[0] * kScale + logf(l[0]) : -INFINITY;
      lse_bh[row + 8] = l[1] > 0.f ? m[1] * kScale + logf(l[1]) : -INFINITY;
    }
  }
}

// ============================================== backward =============================================================
// dK, dV for one tile of 128 keys.  Fixed: K, V.  Ring: (Q, dO) tiles of 64 queries inside the union of the key rows'
// kv_bounds intervals.
__global__ void __launch_bounds__(kThreads, 1)
cross_dkdv_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                  const __grid_constant__ CUtensorMap map_do, const int* __restrict__ kv_bounds, int Sq, int Sk, int H,
                  const float* __restrict__ lse, const float* __restrict__ Dsum, __nv_bfloat16* __restrict__ dkv) {
  extern __shared__ uint8_t smem_raw[];
  const BwdSmem L = bwd_smem(smem_raw);
  const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int HD = H * kHd;
  const size_t pitch = (size_t)2 * HD;
  const size_t q_seq = (size_t)b * Sq, k_seq = (size_t)b * Sk;
  const int2 r = cta_range<kSegment, true>(kv_bounds, k_seq + kt * 128, kt * 128, Sq, reinterpret_cast<int*>(L.empty_bar + kBwdStages));
  if (r.x >= r.y) {                                             // no query sees a key of the tile: no gradient
    zero_rows(dkv + h * kHd, pitch, k_seq + kt * 128, 128);
    zero_rows(dkv + HD + h * kHd, pitch, k_seq + kt * 128, 128);
    return;
  }
  const int qt0 = r.x / 64, n_qt = (r.y + 63) / 64 - qt0;      // query tiles qt0 .. qt0 + n_qt - 1
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) bwd_init_barriers(L);
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&map_q);
      tma_prefetch_desc(&map_kv);
      tma_prefetch_desc(&map_do);
      bwd_produce(L, &map_kv, h * kHd, &map_kv, HD + h * kHd, (int)k_seq + kt * 128,
                  &map_q, h * kHd, &map_do, h * kHd, (int)q_seq + 64 * qt0, n_qt);
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;                             // keys [64 wg, 64 wg + 64) of the tile
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const int key = kt * 128 + wg * 64 + r0;
    const uint32_t k_addr = smem_u32(L.fixed0 + wg * kBoxBytes), v_addr = smem_u32(L.fixed1 + wg * kBoxBytes);
    const float* lse_bh = lse + ((size_t)b * H + h) * Sq;
    const float* D_bh = Dsum + ((size_t)b * H + h) * Sq;
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
    mbar_wait(L.fixed_bar, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int qt = qt0; qt < qt0 + n_qt; ++qt) {
      // the key rows' intervals as one bit mask over this thread's 16 query columns (bits 0-15: row key, 16-31: key + 8)
      const int2 kb0 = row_bounds(kv_bounds, k_seq + key, Sq), kb1 = row_bounds(kv_bounds, k_seq + key + 8, Sq);
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
        const float2 lq = *reinterpret_cast<const float2*>(lse_bh + q);
        const float2 dq = *reinterpret_cast<const float2*>(D_bh + q);
        // a query that saw no key (lse = -inf) gets P = 0, even where malformed bounds put it inside a key's interval
        const float l0 = lq.x == -INFINITY ? INFINITY : lq.x * kLog2e;
        const float l1 = lq.y == -INFINITY ? INFINITY : lq.y * kLog2e;
        const bool v00 = (vis >> (2 * j)) & 1u, v01 = (vis >> (2 * j + 1)) & 1u;   // (key row, query column)
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
    __nv_bfloat16* krow = dkv + (k_seq + key) * pitch + h * kHd;
    store_frag(dk, kScale, kScale, krow, pitch, c0);
    store_frag(dv, 1.f, 1.f, krow + HD, pitch, c0);
  }
}

// dQ for one tile of 128 queries.  Fixed: Q, dO.  Ring: (K, V) tiles of 64 keys inside the union of the query rows'
// q_bounds intervals.
__global__ void __launch_bounds__(kThreads, 1)
cross_dq_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                const __grid_constant__ CUtensorMap map_do, const int* __restrict__ q_bounds, int Sq, int Sk, int H,
                const float* __restrict__ lse, const float* __restrict__ Dsum, __nv_bfloat16* __restrict__ dq_out) {
  extern __shared__ uint8_t smem_raw[];
  const BwdSmem L = bwd_smem(smem_raw);
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int HD = H * kHd;
  const size_t q_seq = (size_t)b * Sq, k_seq = (size_t)b * Sk;
  const int2 r = cta_range<kSegment, false>(q_bounds, q_seq + qt * 128, qt * 128, Sk, reinterpret_cast<int*>(L.empty_bar + kBwdStages));
  if (r.x >= r.y) {
    zero_rows(dq_out + h * kHd, HD, q_seq + qt * 128, 128);
    return;
  }
  const int kt0 = r.x / 64, n_kt = (r.y + 63) / 64 - kt0;      // key tiles kt0 .. kt0 + n_kt - 1
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1 && lane == 0) bwd_init_barriers(L);
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&map_q);
      tma_prefetch_desc(&map_kv);
      tma_prefetch_desc(&map_do);
      bwd_produce(L, &map_q, h * kHd, &map_do, h * kHd, (int)q_seq + qt * 128,
                  &map_kv, h * kHd, &map_kv, HD + h * kHd, (int)k_seq + 64 * kt0, n_kt);
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;
    const int r0 = 16 * ((warp - 4) & 3) + (lane >> 2);
    const int c0 = 2 * (lane & 3);
    const int row = qt * 128 + wg * 64 + r0;
    const int2 qb0 = row_bounds(q_bounds, q_seq + row, Sk), qb1 = row_bounds(q_bounds, q_seq + row + 8, Sk);
    const uint32_t q_addr = smem_u32(L.fixed0 + wg * kBoxBytes), do_addr = smem_u32(L.fixed1 + wg * kBoxBytes);
    const size_t bh = ((size_t)b * H + h) * Sq;
    const float l0 = lse[bh + row] * kLog2e, l1 = lse[bh + row + 8] * kLog2e;
    const float d0 = Dsum[bh + row], d1 = Dsum[bh + row + 8];
    float dq[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] = 0.f;
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
      uint32_t dsa[16];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k0 = kt * 64 + 8 * j + c0;
        const bool v00 = inside(k0, qb0), v01 = inside(k0 + 1, qb0);   // (query row, key column)
        const bool v10 = inside(k0, qb1), v11 = inside(k0 + 1, qb1);
        const float p00 = v00 ? exp2f(s[4 * j] * kScaleLog2 - l0) : 0.f;
        const float p01 = v01 ? exp2f(s[4 * j + 1] * kScaleLog2 - l0) : 0.f;
        const float p10 = v10 ? exp2f(s[4 * j + 2] * kScaleLog2 - l1) : 0.f;
        const float p11 = v11 ? exp2f(s[4 * j + 3] * kScaleLog2 - l1) : 0.f;
        dsa[2 * j] = pack_bf16x2(p00 * (dp[4 * j] - d0), p01 * (dp[4 * j + 1] - d0));
        dsa[2 * j + 1] = pack_bf16x2(p10 * (dp[4 * j + 2] - d1), p11 * (dp[4 * j + 3] - d1));
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_n64_rs<1>(dq, dsa + 4 * kk, desc_mn(k_addr + kk * kStepMN), 1u);  // dQ += dS K
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&L.empty_bar[stage]);
      if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
    }
    store_frag(dq, kScale, kScale, dq_out + (q_seq + row) * HD + h * kHd, HD, c0);
  }
}

void check_cross_shape(const char* who, int B, int Sq, int Sk, int heads) {
  if (B < 1 || heads < 1 || Sq < 128 || Sq % 128 != 0 || Sk < 128 || Sk % 128 != 0)
    throw std::runtime_error(std::string(who) + ": needs B >= 1, heads >= 1 and Sq, Sk positive multiples of 128 (got B=" +
                             std::to_string(B) + ", Sq=" + std::to_string(Sq) + ", Sk=" + std::to_string(Sk) + ", heads=" +
                             std::to_string(heads) + ")");
  if (B > 65535 || heads > 65535 || (long long)B * std::max(Sq, 2 * Sk) * heads * kHd >= (1ll << 31))
    throw std::runtime_error(std::string(who) + ": problem too large");
}

}  // namespace

void launch_cross_attention_fwd(const void* q, const void* kv, const int* q_bounds, int B, int Sq, int Sk, int heads, void* o, float* lse,
                                cudaStream_t s) {
  check_cross_shape("cross_attention_fwd", B, Sq, Sk, heads);
  const CUtensorMap map_q = rows_map(q, B * Sq, heads * kHd);
  const CUtensorMap map_kv = rows_map(kv, B * Sk, 2 * heads * kHd);
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(cross_fwd_kernel, kFwdSmem, configured);
  cross_fwd_kernel<<<dim3(Sq / 128, heads, B), kThreads, kFwdSmem, s>>>(map_q, map_kv, q_bounds, Sq, Sk, heads,
                                                                       reinterpret_cast<__nv_bfloat16*>(o), lse);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_cross_attention_bwd(const void* dout, const void* q, const void* kv, const void* o, const float* lse, const int* q_bounds,
                                const int* kv_bounds, int B, int Sq, int Sk, int heads, float* dsum, void* dq, void* dkv, cudaStream_t s) {
  check_cross_shape("cross_attention_bwd", B, Sq, Sk, heads);
  const int rows = B * Sq;
  const long long items = (long long)rows * heads * 8;
  attn_bwd_dot_kernel<<<ceil_div(items, 256), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dout),
                                                           reinterpret_cast<const __nv_bfloat16*>(o), rows, Sq, heads, dsum);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  const CUtensorMap map_q = rows_map(q, rows, heads * kHd);
  const CUtensorMap map_kv = rows_map(kv, B * Sk, 2 * heads * kHd);
  const CUtensorMap map_do = rows_map(dout, rows, heads * kHd);
  static std::atomic<unsigned long long> configured_dkdv{0}, configured_dq{0};
  ensure_max_dynamic_smem(cross_dkdv_kernel, kBwdSmem, configured_dkdv);
  ensure_max_dynamic_smem(cross_dq_kernel, kBwdSmem, configured_dq);
  cross_dkdv_kernel<<<dim3(Sk / 128, heads, B), kThreads, kBwdSmem, s>>>(map_q, map_kv, map_do, kv_bounds, Sq, Sk, heads, lse, dsum,
                                                                         reinterpret_cast<__nv_bfloat16*>(dkv));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  cross_dq_kernel<<<dim3(Sq / 128, heads, B), kThreads, kBwdSmem, s>>>(map_q, map_kv, map_do, q_bounds, Sq, Sk, heads, lse, dsum,
                                                                       reinterpret_cast<__nv_bfloat16*>(dq));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
