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
#include "gemm.h"

#include <cuda.h>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "drv.h"
#include "tc_primitives.cuh"

namespace b200 {
namespace {
using namespace tc;

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int UMMA_K = 16;
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
};

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
template <int BLOCK_N, bool A_MN, bool B_MN, bool TMA_ST, bool STATS, bool PAIR>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_d, const GemmParams p) {
  using L = SmemLayout<BLOCK_N, A_MN, B_MN, TMA_ST>;
  constexpr int kStages = L::kStages;
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
  const int num_m_blocks = (p.M + kM - 1) / kM;
  const int num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = num_m_blocks * num_n_blocks;
  const int num_k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;

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
        int mb, nb;
        gemm_tile_coords(tile, num_m_blocks, num_n_blocks, p.group_m, &mb, &nb);
        const int m0 = mb * kM + (int)rank * BLOCK_M;            // rows past M arrive as zeros and are never stored
        const int n0 = nb * BLOCK_N;
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::kStageBytes;
          uint8_t* sb = sa + L::kABytes;
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          const int k0 = kb * BLOCK_K;
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
            tma_load_2d(&map_b, &full_bar[stage], sb, k0, n0);                    // box {64 k, BLOCK_N n}
          } else {
#pragma unroll
            for (int c = 0; c < BLOCK_N / 64; ++c)
              tma_load_2d(&map_b, &full_bar[stage], sb + c * (64 * BLOCK_K * 2), n0 + 64 * c, k0);
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
      int mb, nb;
      gemm_tile_coords(tile, num_m_blocks, num_n_blocks, p.group_m, &mb, &nb);
      const int m0 = mb * kM + (int)rank * BLOCK_M;
      const int n0 = nb * BLOCK_N;
      WgAcc<BLOCK_N> acc;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * L::kStageBytes);
        const uint32_t b_addr = a_addr + L::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
          const uint64_t da0 = make_smem_desc(a_addr + k * kStepA, kLboA, kSbo);
          const uint64_t da1 = make_smem_desc(a_addr + kHalfA + k * kStepA, kLboA, kSbo);
          const uint64_t db = make_smem_desc(b_addr + k * kStepB, kLboB, kSbo);
          wgmma_tile<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da0, da1, db, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) {                                        // smem slot reusable: this warp's MMAs have read it
          mbar_arrive(&empty_bar[stage]);
          if constexpr (PAIR) mbar_arrive_cluster(&empty_bar[stage], rank ^ 1u);   // the peer multicasts into it too
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wg_bar_sync();                                           // the previous tile's epilogue is done reading acc_smem
      acc_to_smem<BLOCK_N>(acc, acc_smem, L::kAccStride, threadIdx.x - 128);
      wg_bar_sync();
      const int row = m0 + ew * 32 + lane;
      const float* arow = acc_smem + (size_t)(ew * 32 + lane) * L::kAccStride;
      if constexpr (TMA_ST) {
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
struct MapKey {
  const void* ptr; int rows, cols, box_rows, box_cols;
  bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows && box_cols == o.box_cols; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    for (int v : {k.rows, k.cols, k.box_rows, k.box_cols}) h = h * 1000003u ^ (size_t)v;
    return h;
  }
};

// 2-D row-major bf16 tensor [rows, cols]; box = [box_rows, box_cols] with box_cols * 2 == 128 bytes.
CUtensorMap make_map(const void* ptr, int rows, int cols, int box_rows, int box_cols) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  MapKey key{ptr, rows, cols, box_rows, box_cols};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
  }
  auto& drv = Driver::get();
  if (!drv.TensorMapEncodeTiled) throw std::runtime_error("gemm: cuTensorMapEncodeTiled unavailable");
  // driver-API calls need a current context; autograd worker threads only get one lazily from the runtime
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { B200_CUDA_CHECK(cudaFree(nullptr)); ctx_bound = true; }
  CUtensorMap map;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t elem_strides[2] = {1, 1};
  B200_DRV_CHECK(drv.TensorMapEncodeTiled(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box,
                                          elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
  std::lock_guard<std::mutex> g(mu);
  if (cache.size() > 4096) cache.clear();
  cache.emplace(key, map);
  return map;
}

// TMA_ST: epilogue through shared memory + TMA store (bf16 output, N % 8 == 0); the D map's box is one warp slab.
template <int BLOCK_N, bool A_MN, bool B_MN, bool TMA_ST, bool STATS = false, bool PAIR = false>
void launch_variant(const void* a, const void* b, const GemmParams& p, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N, A_MN, B_MN, TMA_ST>;
  constexpr int kSmem = L::kTotal;
  static_assert(L::kStages >= 3 && kSmem <= 227 * 1024, "shared memory budget");
  // A: K-major stored [M,K] -> box {BLOCK_M rows, 64 cols};  MN-major stored [K,M] -> box {64 rows(k), 64 cols(m)}
  CUtensorMap map_a = A_MN ? make_map(a, p.K, p.M, BLOCK_K, 64) : make_map(a, p.M, p.K, BLOCK_M, BLOCK_K);
  CUtensorMap map_b = B_MN ? make_map(b, p.K, p.N, BLOCK_K, 64) : make_map(b, p.N, p.K, PAIR ? BLOCK_N / 2 : BLOCK_N, BLOCK_K);
  CUtensorMap map_d = TMA_ST ? make_map(p.d, p.M, p.N, 32, 64) : map_a;       // unused by the direct epilogue
  auto kernel = gemm_bf16_kernel<BLOCK_N, A_MN, B_MN, TMA_ST, STATS, PAIR>;
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

}  // namespace b200
