// wgmma / TMA / mbarrier building blocks shared by the sm_90a tensor-core kernels (inline PTX wrappers only: no state, no
// policy).  Used by the GEMM and convolution kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace b200 {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
#ifndef B200_MBAR_SPIN
#define B200_MBAR_SPIN 0
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if B200_MBAR_SPIN
  // Non-suspending poll.  mbarrier.try_wait parks the thread for a system-dependent time slice when the phase is not
  // complete yet; a consumer that is FASTER than its producer (small-K convolutions: the issuer catches up with the TMA
  // stream on every k-block) then pays that slice per k-block instead of the actual remaining latency.
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
#endif
}

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// ---- thread-block clusters: CTA pairs that share operand tiles through TMA multicast ---------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// the box lands at the same offset in every CTA of `cta_mask` and signals complete_tx on each one's barrier at `bar`'s offset
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask) : "memory");
}

// ---- warpgroup MMA (wgmma): one aligned warpgroup of 128 threads issues every instruction together ----------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor, 128B swizzle (layout type 1 in bits [62,64)).  K-major: SBO = 8 rows * 128 B, LBO unused.
// MN-major: LBO = distance between 64-wide MN chunks, SBO = 8 k-rows * 128 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);            // [0,14)  start address >> 4
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;        // [16,30) leading byte offset >> 4
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;        // [32,46) stride byte offset >> 4
  d |= (uint64_t)1 << 62;                                  // SWIZZLE_128B
  return d;
}

// D (+)= A[smem desc] * B[smem desc], m64 x N x k16, bf16 x bf16 -> fp32 in registers.  TA / TB: 1 = operand is MN-major.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB));
}

// A 128 x BN fp32 accumulator tile held by one warpgroup: rows [0, 64) in h[0], rows [64, 128) in h[1].  Thread t of the
// warpgroup holds, per half, rows 16 * (t / 32) + (t % 32) / 4 (+ 8) and column pairs 8 j + 2 (t % 4) of every 8-column group.
template <int BN>
struct WgAcc {
  static_assert(BN == 64 || BN == 128, "accumulator width");
  float h[2][BN / 2];
};

// acc (+)= A * B for one k16 step; da0 / da1 address A rows [0, 64) / [64, 128)
template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(WgAcc<BN>& acc, uint64_t da0, uint64_t da1, uint64_t db, uint32_t accumulate) {
  if constexpr (BN == 64) {
    wgmma_n64<TA, TB>(acc.h[0], da0, db, accumulate);
    wgmma_n64<TA, TB>(acc.h[1], da1, db, accumulate);
  } else {
    wgmma_n128<TA, TB>(acc.h[0], da0, db, accumulate);
    wgmma_n128<TA, TB>(acc.h[1], da1, db, accumulate);
  }
}

// The accumulator tile as fp32 rows of `stride` floats in shared memory (stride % 32 == 8: conflict-free 8-byte stores), so
// that an epilogue thread can read one whole row: the register layout of wgmma spreads a row over four threads.
template <int BN>
__device__ __forceinline__ void acc_to_smem(const WgAcc<BN>& acc, float* dst, int stride, int wg_thread) {
  const int warp = wg_thread >> 5, lane = wg_thread & 31;
  const int r0 = warp * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float* p = dst + (size_t)(half * 64 + r0) * stride + 8 * j + c0;
      *reinterpret_cast<float2*>(p) = make_float2(acc.h[half][4 * j], acc.h[half][4 * j + 1]);
      *reinterpret_cast<float2*>(p + 8 * stride) = make_float2(acc.h[half][4 * j + 2], acc.h[half][4 * j + 3]);
    }
  }
}
// 32 consecutive fp32 accumulator values of one row, from the shared-memory copy written by acc_to_smem
__device__ __forceinline__ void acc_row_ld32(const float* src, int stride, int row, int col, uint32_t* r) {
  const float4* p = reinterpret_cast<const float4*>(src + (size_t)row * stride + col);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 v = p[q];
    r[4 * q] = __float_as_uint(v.x); r[4 * q + 1] = __float_as_uint(v.y); r[4 * q + 2] = __float_as_uint(v.z); r[4 * q + 3] = __float_as_uint(v.w);
  }
}
// bar.sync over the 128 threads of the MMA / epilogue warpgroup (named barrier 1)
__device__ __forceinline__ void wg_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }


// ---- TMA store (shared -> global), bulk-group completion -----------------------------------------------------------
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(smem)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_le1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }


}  // namespace tc
}  // namespace b200
