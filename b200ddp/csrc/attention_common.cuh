// Device pieces shared by the head-dim-64 attention kernels of attention.cu (one fused qkv) and cross_attention.cu (queries
// and keys / values from two tensors): tile geometry and constants, interval masks, wgmma descriptors and products,
// fragment stores, the rowsum(dO * O) kernel, the backward kernels' shared-memory layout and TMA producer, and the tensor
// map over a row-major bf16 matrix.  Everything sits in an anonymous namespace, so each including file compiles its own
// copy of the one definition here.
#pragma once
#include <cuda.h>

#include "common.h"
#include "ops.h"
#include "tc_primitives.cuh"
#include "tensor_map.h"

namespace b200 {
namespace {
using namespace tc;


constexpr int kHd = 64;                        // head dim: 128 bytes, one swizzle row
constexpr int kBoxRows = 64;
constexpr int kBoxBytes = kBoxRows * kHd * 2;  // 8 KB
constexpr int kThreads = 384;
constexpr int kConsumerArrivals = 8;           // lane 0 of each consumer warp releases a ring stage
constexpr float kScale = 0.125f;               // 1/sqrt(64)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kScaleLog2 = kScale * kLog2e;
constexpr uint32_t kSbo = 1024;                // 8 rows x 128 B
constexpr uint32_t kLboMN = kBoxRows * 128;    // MN-major: distance between 64-wide chunks (only one chunk is used)
constexpr uint32_t kStepK = 32;                // K-major: 16 bf16 columns
constexpr uint32_t kStepMN = 16 * 128;         // MN-major: 16 rows

constexpr int kFwdStages = 2;
constexpr int kFwdSmem = 1024 + 2 * kBoxBytes + kFwdStages * 4 * kBoxBytes + 256;   // Q 128 rows + ring of (K, V) 128 rows
constexpr int kBwdStages = 4;
constexpr int kBwdSmem = 1024 + 4 * kBoxBytes + kBwdStages * 2 * kBoxBytes + 256;   // fixed 2 x 128 rows + ring of 2 x 64 rows

constexpr int kKeyPadding = 0;
constexpr int kSegment = 1;
constexpr int kCausal = 2;

// (start, end) of global row `row` of bounds [B*S, 2], clamped to 0 <= start <= end <= S
__device__ __forceinline__ int2 row_bounds(const int* bounds, size_t row, int S) {
  const int2 v = __ldg(reinterpret_cast<const int2*>(bounds) + row);
  const int s = min(max(v.x, 0), S);
  return make_int2(s, min(max(v.y, s), S));
}
// The interval of global row `row` (position `pos` in its sequence) as a query (the keys it sees, kKeySide = false) or as
// a key (the queries that see it, kKeySide = true).  kSegment: the row's bounds either way.  kCausal: the query side
// stops after `pos`, the key side starts at `pos`; both stay non-empty-or-(x == y) so `inside` and the masks hold.
template <int kMode, bool kKeySide>
__device__ __forceinline__ int2 mask_interval(const int* bounds, size_t row, int pos, int S) {
  int2 r = row_bounds(bounds, row, S);
  if constexpr (kMode == kCausal) {
    if constexpr (kKeySide) r.x = min(max(r.x, pos), r.y);
    else r.y = max(min(r.y, pos + 1), r.x);
  }
  return r;
}
__device__ __forceinline__ bool inside(int j, int2 r) { return (unsigned)(j - r.x) < (unsigned)(r.y - r.x); }
// A fragment thread owns columns 8 j + e (j < 8, e < 2) of a 64-wide tile, counted from its first column.  Bit 2 j + e
// is set where that column lies in [lo, hi).  The columns are increasing in the bit index, so the set bits are the range
// [#columns below lo, #columns below hi).
__device__ __forceinline__ uint32_t frag_mask16(int lo, int hi) {
  lo = min(max(lo, 0), 64);
  hi = min(max(hi, lo), 64);
  const int nlo = 2 * (lo >> 3) + min(lo & 7, 2), nhi = 2 * (hi >> 3) + min(hi & 7, 2);
  return ((1u << nhi) - 1u) & ~((1u << nlo) - 1u);
}
// [lo, hi): the union of the intervals (mask_interval) of rows row0 .. row0 + 127, at positions pos0 .. pos0 + 127 (lo >= hi
// when all are empty).  Every thread of the block calls it (it holds a __syncthreads); scratch is 8 ints of shared memory.
template <int kMode, bool kKeySide>
__device__ __forceinline__ int2 cta_range(const int* bounds, size_t row0, int pos0, int S, int* scratch) {
  const int t = threadIdx.x;
  if (t < 128) {
    const int2 r = mask_interval<kMode, kKeySide>(bounds, row0 + t, pos0 + t, S);
    const bool empty = r.x >= r.y;
    const int lo = __reduce_min_sync(0xffffffffu, empty ? S : r.x);
    const int hi = __reduce_max_sync(0xffffffffu, empty ? 0 : r.y);
    if ((t & 31) == 0) { scratch[t >> 5] = lo; scratch[4 + (t >> 5)] = hi; }
  }
  __syncthreads();
  return make_int2(min(min(scratch[0], scratch[1]), min(scratch[2], scratch[3])),
                   max(max(scratch[4], scratch[5]), max(scratch[6], scratch[7])));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}
__device__ __forceinline__ uint64_t desc_k(uint32_t addr) { return make_smem_desc(addr, 16, kSbo); }
__device__ __forceinline__ uint64_t desc_mn(uint32_t addr) { return make_smem_desc(addr, kLboMN, kSbo); }

// S (+)= A B^T over the 64-wide head dim (four k16 steps), both operands K-major 64-row tiles (B: 64 or 128 rows)
__device__ __forceinline__ void mma_hd_n64(float (&acc)[32], uint32_t a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < kHd / 16; ++k) wgmma_n64<0, 0>(acc, desc_k(a + k * kStepK), desc_k(b + k * kStepK), k != 0 ? 1u : 0u);
}

// Zero rows [row0, row0 + rows) of one head's 64 columns in a row-major bf16 matrix with `pitch` elements per row
__device__ __forceinline__ void zero_rows(__nv_bfloat16* base, size_t pitch, size_t row0, int rows) {
  for (int i = threadIdx.x; i < rows * 32; i += blockDim.x)
    *reinterpret_cast<uint32_t*>(base + (row0 + (i >> 5)) * pitch + 2 * (i & 31)) = 0u;
}

// Stores one warpgroup's m64 x 64 fp32 fragment (times `scale`) as bf16: rows r0 / r0 + 8, column pairs 8 j + c0.
__device__ __forceinline__ void store_frag(const float (&acc)[32], float scale0, float scale1, __nv_bfloat16* row0_ptr,
                                           size_t pitch, int c0) {
  __nv_bfloat16* row1_ptr = row0_ptr + 8 * pitch;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    *reinterpret_cast<uint32_t*>(row0_ptr + 8 * j + c0) = pack_bf16x2(acc[4 * j] * scale0, acc[4 * j + 1] * scale0);
    *reinterpret_cast<uint32_t*>(row1_ptr + 8 * j + c0) = pack_bf16x2(acc[4 * j + 2] * scale1, acc[4 * j + 3] * scale1);
  }
}

// D[b, h, s] = sum_d dO[b*S + s, h*64 + d] * O[b*S + s, h*64 + d]; eight threads per (row, head), 16 bytes each
__global__ void attn_bwd_dot_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ out, int rows,
                                    int S, int H, float* __restrict__ D) {
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t item = gid >> 3;
  const int part = (int)(gid & 7);
  const bool live = item < (size_t)rows * H;
  float acc = 0.f;
  size_t row = 0;
  int hh = 0;
  if (live) {
    row = item / H;
    hh = (int)(item % H);
    const size_t off = row * (size_t)H * kHd + hh * kHd + part * 8;
    float a[8], c[8];
    unpack8(*reinterpret_cast<const Bf16x8*>(dout + off), a);
    unpack8(*reinterpret_cast<const Bf16x8*>(out + off), c);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc += a[i] * c[i];
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (live && part == 0) {
    const size_t b = row / S, s = row % S;
    D[(b * H + hh) * S + s] = acc;
  }
}

// Shared layout of both backward kernels: two fixed 128-row tiles (loaded once), then a ring of two 64-row tiles.
struct BwdSmem {
  uint8_t* fixed0;      // 128 rows
  uint8_t* fixed1;      // 128 rows
  uint8_t* ring;        // stage: tile0 64 rows, tile1 64 rows
  uint64_t* fixed_bar;
  uint64_t* full_bar;
  uint64_t* empty_bar;
};
__device__ __forceinline__ BwdSmem bwd_smem(uint8_t* raw) {
  BwdSmem L;
  L.fixed0 = align1024(raw);
  L.fixed1 = L.fixed0 + 2 * kBoxBytes;
  L.ring = L.fixed1 + 2 * kBoxBytes;
  L.fixed_bar = reinterpret_cast<uint64_t*>(L.ring + kBwdStages * 2 * kBoxBytes);
  L.full_bar = L.fixed_bar + 1;
  L.empty_bar = L.full_bar + kBwdStages;
  return L;
}
__device__ __forceinline__ void bwd_init_barriers(const BwdSmem& L) {
  mbar_init(L.fixed_bar, 1);
  for (int i = 0; i < kBwdStages; ++i) { mbar_init(&L.full_bar[i], 1); mbar_init(&L.empty_bar[i], kConsumerArrivals); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// Producer: fixed tiles (map0 at column col0f, map1 at col1f, rows fixed_row .. + 127), then `n` ring stages of
// (map0r at col0r, map1r at col1r, rows ring_row0 + 64 i .. + 63).
__device__ __forceinline__ void bwd_produce(const BwdSmem& L, const CUtensorMap* map0, int col0f, const CUtensorMap* map1, int col1f,
                                            int fixed_row, const CUtensorMap* map0r, int col0r, const CUtensorMap* map1r, int col1r,
                                            int ring_row0, int n) {
  mbar_expect_tx(L.fixed_bar, 4 * kBoxBytes);
  tma_load_2d(map0, L.fixed_bar, L.fixed0, col0f, fixed_row);
  tma_load_2d(map0, L.fixed_bar, L.fixed0 + kBoxBytes, col0f, fixed_row + 64);
  tma_load_2d(map1, L.fixed_bar, L.fixed1, col1f, fixed_row);
  tma_load_2d(map1, L.fixed_bar, L.fixed1 + kBoxBytes, col1f, fixed_row + 64);
  int stage = 0;
  uint32_t phase = 0;
  for (int i = 0; i < n; ++i) {
    mbar_wait(&L.empty_bar[stage], phase ^ 1);
    uint8_t* t0 = L.ring + stage * 2 * kBoxBytes;
    mbar_expect_tx(&L.full_bar[stage], 2 * kBoxBytes);
    tma_load_2d(map0r, &L.full_bar[stage], t0, col0r, ring_row0 + 64 * i);
    tma_load_2d(map1r, &L.full_bar[stage], t0 + kBoxBytes, col1r, ring_row0 + 64 * i);
    if (++stage == kBwdStages) { stage = 0; phase ^= 1; }
  }
}

CUtensorMap rows_map(const void* ptr, int rows, int cols) {
  const uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows};
  const uint64_t strides[1] = {(uint64_t)cols * 2};
  const uint32_t box[2] = {(uint32_t)kHd, (uint32_t)kBoxRows};
  return encode_tensor_map(ptr, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 2, dims, strides, box);
}

}  // namespace
}  // namespace b200
