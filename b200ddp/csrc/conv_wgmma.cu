// Convolution forward / data-gradient for channels_last bf16 activations as an implicit GEMM on the Hopper tensor cores
// (replaces the cuDNN implicit-GEMM kernels behind the model's forward / backward when selected, see ops/functional.py).
//
//   D[pixel, n] = sum_{tap (r,s)} sum_{c} A[pixel shifted by the tap, c] * B_tap[n, c]          fp32 accumulation in registers
//
// No im2col buffer and no im2col-mode descriptors.  One kernel, three tilings of the output grid (conv.h: ConvTilePlan):
//   flat  (1x1)  the NHWC tensor *is* the row-major [N*H*W, C] operand; a tile is 128 consecutive pixels.
//   patch (3x3)  every tap re-fetches its shifted patch with a rank-4 TMA box {64 ch, W, BH, BI}; coordinates outside
//                the image are zero-filled by the TMA unit - that is the padding.
//   halo  (3x3)  the (BH+2) x (W+2) halo of the tile is fetched ONCE per 64-channel block; tap (r,s) is the same
//                shared-memory tile read through a descriptor whose start address is advanced by r*(W+2)+s rows (the tile
//                is K-major with 128-byte rows, so a pixel shift is a whole-row offset).  9x less operand traffic from L2
//                than "patch".
// Filter: [Cout][R][S][Cin] (a channels_last nn.Conv2d weight) is the K-major matrix [Cout, R*S*Cin] for the forward
// pass and, read MN-major (rows = Cout = reduction, columns = Cin), the B operand of the data gradient with mirrored taps -
// no transposed / flipped copy of the weights is ever materialised.
//
// Roles (256 threads): warp 0 = activation TMA producer, warp 3 = filter TMA producer (two rings: activation slots and filter
// slots), warps 4-7 = one warpgroup that issues wgmma (two m64 halves of the 128-row tile, accumulators in registers), copies
// the accumulator tile to shared memory and runs the epilogue one output row per thread (bf16 -> 128B-swizzled staging tile
// -> one TMA store per 64 output channels; optional per-CTA column sums / sums of squares for the BatchNorm that follows).
// Persistent over tiles; the producers run ahead into the next tile while the warpgroup drains the current one.
#include "conv.h"

#include <cuda.h>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "drv.h"
#include "tc_primitives.cuh"

namespace b200 {
namespace {
using namespace tc;

constexpr int BLOCK_K = 64;
constexpr int UMMA_K = 16;
constexpr int kThreads = 256;
constexpr int kMmaWarps = 4;                   // warps 4-7: the MMA / epilogue warpgroup
constexpr int kMaxRing = 12;
constexpr int kSlabBytes = 128 * 128;          // one dense staging tile: 128 rows x 64 bf16
constexpr int kStagingBytes = 2 * kSlabBytes;
constexpr int kBarrierBytes = 1024;
constexpr int kTrStride = 36;                       // floats per row of the per-warp 32 x 32 transpose scratch (conflict-free v4 stores / column loads)
constexpr int kStatsScratchBytes = 4 * 32 * kTrStride * 4;   // epilogue statistics scratch: one 32 x 36 fp32 tile per epilogue warp
// the fp32 accumulator tile in shared memory, 128 rows of BLOCK_N + 8 floats
__host__ __device__ constexpr int acc_stride(int block_n) { return block_n + 8; }
__host__ __device__ constexpr int acc_bytes(int block_n) { return 128 * acc_stride(block_n) * 4; }

struct TapGemmParams {
  int M_total, Kc, Nc;      // output pixels, reduction channels per tap, output channels
  int R, S, pad;
  int mirror;               // data gradient: input offset of tap r is pad - r (forward: r - pad)
  int mode;                 // 0 flat, 1 patch, 2 halo
  int H, W;
  int BH, BI, tiles_h, Wp;
  int num_m_tiles, num_n_tiles;
  int dense_rows;
  int a_chunk_bytes;        // bytes reserved per activation chunk (flat / patch) or per halo tile
  int KC, TB;               // k chunks per ring-S stage (flat / patch); filter taps per ring-B slot (halo)
  int s_stage_bytes, s_stages, b_slot_bytes, b_stages;
  uint32_t a_tx_bytes;
  int set_base_offset;
  int b_tap_stride;         // column distance between taps in the filter matrix (Cin of the filter tensor)
  int row_mul;              // patch tiling: input row of output row h and tap r is row_mul * h + r - pad
  int b_resident;           // flat / patch tilings with one n-tile: all filter chunks of a tile are loaded ONCE per CTA into ring B
  int chunk_stride;         // bytes between consecutive k chunks of a ring-S stage (activation chunk [+ filter chunk])
  float* col_stats;         // [2][G][Nc] or nullptr (EPI 1: sum / sum of squares of the output; EPI 2: S1 / S2 of the BatchNorm backward)
  const __nv_bfloat16* addend;   // EPI 2: [M_total, Nc] added to the output (shortcut gradient) or nullptr
  const __nv_bfloat16* bn_x;     // EPI 2: [M_total, Nc] input of the BatchNorm whose backward consumes the output, or nullptr
  const uint8_t* bn_mask;        // EPI 2: [M_total, Nc / 8] ReLU bit mask of that BatchNorm's output, or nullptr (no ReLU)
  const float* bn_mean;          // EPI 2: [Nc]
  const float* bn_rstd;          // EPI 2: [Nc]
  long long* dbg;           // optional [16] cycle counters of CTA 0's roles (diagnostics)
};

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// 128B-swizzle K-major descriptor whose start address may sit on any 128-byte row of the tile
__device__ __forceinline__ uint64_t make_desc_rowoff(uint32_t addr, uint32_t lbo, uint32_t sbo, int set_base_offset) {
  uint64_t d = make_smem_desc(addr, lbo, sbo);
  if (set_base_offset) d |= (uint64_t)((addr >> 7) & 7u) << 49;
  return d;
}

// accumulator row i of a tile -> row inside the dense staging / output tile; false if the row holds nothing
__device__ __forceinline__ bool acc_row_to_dense(const TapGemmParams& p, int i, int* dense) {
  if (p.mode == 2) {
    const int h = i / p.Wp, w = i - h * p.Wp;
    *dense = h * p.W + w;
    return h < p.BH && w < p.W;
  }
  *dense = i;
  return i < p.dense_rows;
}

// Column sums of a 32-row x 32-column block held one row per lane: the block goes through a per-warp shared-memory tile
// (row stride 36 floats: the eight 16-byte stores of a row and the 32 column reads are bank-conflict free) and lane l adds up
// column l.  ~1.7x fewer instructions than a shuffle butterfly, which made small-K layers epilogue-bound.
__device__ __forceinline__ float warp_column_sum32(const float* v, float* tr, int lane) {
#pragma unroll
  for (int q = 0; q < 8; ++q)
    *reinterpret_cast<float4*>(tr + lane * kTrStride + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  __syncwarp();
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < 32; ++r) s += tr[r * kTrStride + lane];
  __syncwarp();
  return s;
}

// exactly one lane of a converged warp; code guarded by it is known single-threaded to the compiler, which keeps
// descriptors / addresses in uniform registers and issues the TMA instructions directly (a plain `lane == 0` branch makes
// every such instruction a per-lane loop with register -> uniform-register moves)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}

// EPI: 0 plain store; 1 forward + column statistics of the output (BatchNorm forward); 2 data gradient + optional addend
// (shortcut gradient) + optional partial sums of the BatchNorm backward that consumes this gradient
template <int BLOCK_N, bool B_MN, int EPI>
__global__ void __launch_bounds__(kThreads, 1)
conv_tap_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                     const __grid_constant__ CUtensorMap map_d, const TapGemmParams p) {
  constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  constexpr int kAccStride = acc_stride(BLOCK_N);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // ring S: flat / patch: KC x (activation chunk + filter chunk) per stage;  halo: the activation halo of one channel block
  // ring B (halo only): TB filter taps per slot
  uint8_t* s_ring = smem;
  uint8_t* b_ring = s_ring + p.s_stages * p.s_stage_bytes;
  uint8_t* staging = b_ring + p.b_stages * p.b_slot_bytes;
  [[maybe_unused]] float* stats_scratch = reinterpret_cast<float*>(staging + kStagingBytes);
  float* acc_smem = reinterpret_cast<float*>(staging + kStagingBytes + (EPI != 0 ? kStatsScratchBytes : 0));
  uint64_t* s_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_smem) + acc_bytes(BLOCK_N));
  uint64_t* s_empty = s_full + kMaxRing;
  uint64_t* b_full = s_empty + kMaxRing;
  uint64_t* b_empty = b_full + kMaxRing;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long t_begin = clock64();
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int cblocks = p.Kc / BLOCK_K;
  const int taps = p.R * p.S;
  const int chunks_per_tile = cblocks * taps;              // flat / patch: 64-deep k chunks of one tile

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&map_a); tma_prefetch_desc(&map_b); tma_prefetch_desc(&map_d); }
  if (warp == 1) {                                     // one lane per ring slot: the ~50 barrier inits are off the serial path
    if (lane < kMaxRing) {   // empty slots: one arrival per MMA warp once its wgmma reads of the slot are complete
      mbar_init(&s_full[lane], (p.mode == 2 || p.b_resident) ? 1 : 2); mbar_init(&s_empty[lane], kMmaWarps);
      mbar_init(&b_full[lane], 1); mbar_init(&b_empty[lane], kMmaWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
#define B200_T0 if (dbg) t = clock64();
#define B200_T1(acc) if (dbg) acc += clock64() - t;

  if (warp == 0 || warp == 3) {
    // ===================== TMA producers: warp 0 streams activations, warp 3 streams filter tiles =====================
    // (the two operands get a warp each so that neither stream waits behind the other's TMA issue; the whole warp walks the
    // loop, one elected lane issues)
    const bool is_a = (warp == 0);
    int ss = 0, bs = 0;
    uint32_t sph = 0, bph = 0;
    long long d_w = 0, d_i = 0, t = 0;
    const bool dbg = p.dbg != nullptr && blockIdx.x == 0;
    if constexpr (!B_MN) {
      if (!is_a && p.b_resident) {                         // the whole (small) filter of the single n-tile: once per CTA
        if (elect_one()) {
          mbar_expect_tx(&b_full[0], (uint32_t)chunks_per_tile * kBBytes);
          int cb_i = 0, r_i = 0, s_i = 0;
          for (int q = 0; q < chunks_per_tile; ++q) {
            tma_load_2d(&map_b, &b_full[0], b_ring + q * kBBytes, (r_i * p.S + s_i) * p.b_tap_stride + cb_i * BLOCK_K, 0);
            if (++s_i == p.S) { s_i = 0; if (++r_i == p.R) { r_i = 0; ++cb_i; } }
          }
        }
        __syncwarp();
      }
    }
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;     // n-tiles of one patch run on neighbouring CTAs
      const int n0 = nt * BLOCK_N;
      int img0 = 0, h0 = 0;
      if (p.mode != 0) { img0 = (mt / p.tiles_h) * p.BI; h0 = (mt % p.tiles_h) * p.BH; }
      if (p.mode != 2) {
        if (!is_a && p.b_resident) continue;               // nothing to stream for this warp
        int cb = 0, r = 0, sx = 0;                           // chunk q = (cb, tap (r, sx)), taps fastest
        for (int q0 = 0; q0 < chunks_per_tile; q0 += p.KC) {
          B200_T0 mbar_wait(&s_empty[ss], sph ^ 1); B200_T1(d_w)
          B200_T0
          if (elect_one()) {
            uint8_t* dst = s_ring + ss * p.s_stage_bytes;
            int cb_i = cb, r_i = r, s_i = sx;
            if (is_a) {
              mbar_expect_tx(&s_full[ss], (uint32_t)p.KC * p.a_tx_bytes);
              for (int j = 0; j < p.KC; ++j) {
                if (p.mode == 0) {
                  tma_load_4d(&map_a, &s_full[ss], dst, cb_i * BLOCK_K, mt * 128, 0, 0);
                } else {
                  const int dh = p.mirror ? p.pad - r_i : r_i - p.pad, dw = p.mirror ? p.pad - s_i : s_i - p.pad;
                  tma_load_4d(&map_a, &s_full[ss], dst, cb_i * BLOCK_K, dw, h0 * p.row_mul + dh, img0);  // out-of-image rows / columns arrive as zeros
                }
                dst += p.chunk_stride;
                if (++s_i == p.S) { s_i = 0; if (++r_i == p.R) { r_i = 0; ++cb_i; } }
              }
            } else {
              mbar_expect_tx(&s_full[ss], (uint32_t)p.KC * kBBytes);
              for (int j = 0; j < p.KC; ++j) {
                uint8_t* sb = dst + p.a_chunk_bytes;
                const int bcol = (r_i * p.S + s_i) * p.b_tap_stride;
                if constexpr (!B_MN) {
                  tma_load_2d(&map_b, &s_full[ss], sb, bcol + cb_i * BLOCK_K, n0);            // box {64 k, BLOCK_N n}
                } else {
#pragma unroll
                  for (int c = 0; c < BLOCK_N / 64; ++c)                                      // box {64 n, 64 k} per chunk
                    tma_load_2d(&map_b, &s_full[ss], sb + c * (64 * BLOCK_K * 2), bcol + n0 + 64 * c, cb_i * BLOCK_K);
                }
                dst += p.chunk_stride;
                if (++s_i == p.S) { s_i = 0; if (++r_i == p.R) { r_i = 0; ++cb_i; } }
              }
            }
          }
          __syncwarp();
          for (int j = 0; j < p.KC; ++j) { if (++sx == p.S) { sx = 0; if (++r == p.R) { r = 0; ++cb; } } }
          if (++ss == p.s_stages) { ss = 0; sph ^= 1; }
          B200_T1(d_i)
        }
      } else if (is_a) {
        for (int cb = 0; cb < cblocks; ++cb) {
          B200_T0 mbar_wait(&s_empty[ss], sph ^ 1); B200_T1(d_w)
          B200_T0
          if (elect_one()) {
            mbar_expect_tx(&s_full[ss], p.a_tx_bytes);
            tma_load_4d(&map_a, &s_full[ss], s_ring + ss * p.s_stage_bytes, cb * BLOCK_K, -p.pad, h0 - p.pad, img0);
          }
          __syncwarp();
          if (++ss == p.s_stages) { ss = 0; sph ^= 1; }
          B200_T1(d_i)
        }
      } else {
        for (int cb = 0; cb < cblocks; ++cb) {
          for (int tap0 = 0; tap0 < taps; tap0 += p.TB) {
            B200_T0 mbar_wait(&b_empty[bs], bph ^ 1); B200_T1(d_w)
            B200_T0
            if (elect_one()) {
              mbar_expect_tx(&b_full[bs], (uint32_t)p.TB * kBBytes);
              for (int j = 0; j < p.TB; ++j) {
                uint8_t* sb = b_ring + bs * p.b_slot_bytes + j * kBBytes;
                const int bcol = (tap0 + j) * p.b_tap_stride;
                if constexpr (!B_MN) {
                  tma_load_2d(&map_b, &b_full[bs], sb, bcol + cb * BLOCK_K, n0);
                } else {
#pragma unroll
                  for (int c = 0; c < BLOCK_N / 64; ++c)
                    tma_load_2d(&map_b, &b_full[bs], sb + c * (64 * BLOCK_K * 2), bcol + n0 + 64 * c, cb * BLOCK_K);
                }
              }
            }
            __syncwarp();
            if (++bs == p.b_stages) { bs = 0; bph ^= 1; }
            B200_T1(d_i)
          }
        }
      }
    }
    if (dbg && lane == 0) { p.dbg[is_a ? 0 : 2] = d_w; p.dbg[is_a ? 1 : 3] = d_i; }
  } else if (warp >= 4) {
    // ===================== MMA warpgroup: wgmma -> registers -> shared memory -> epilogue =====================
    constexpr int kTB = B_MN ? 1 : 0;
    constexpr uint32_t kLboB = B_MN ? BLOCK_K * 128 : 16;
    constexpr uint32_t kStepB = B_MN ? UMMA_K * 128 : UMMA_K * 2;
    constexpr uint64_t kHalfA = (64 * 128) >> 4;             // rows [64, 128) of an activation tile (K-major, 128-byte rows)
    // descriptors = constant high part + (address >> 4) in the low 14 bits: one 64-bit add per operand and MMA
    const uint64_t a_desc0 = make_smem_desc(smem_u32(s_ring), 16, 1024);
    const uint64_t b_desc_s0 = make_smem_desc(smem_u32(s_ring), kLboB, 1024);      // filter chunks inside ring S (flat / patch)
    const uint64_t b_desc_b0 = make_smem_desc(smem_u32(b_ring), kLboB, 1024);      // filter slots of ring B (halo)
    const int ew = warp - 4;                         // this warp's epilogue rows: [32*ew, 32*ew + 32) of the tile
    const bool t0 = (ew == 0 && lane == 0);
    int ss = 0, bs = 0;
    uint32_t sph = 0, bph = 0, slab = 0;
    long long d_wf = 0, d_mma = 0, d_ep = 0, t = 0;
    const bool dbg = p.dbg != nullptr && blockIdx.x == 0 && t0;
    // STATS: the grid is a multiple of num_n_tiles, so every tile of this CTA has the same n-tile; after the transpose a lane
    // owns column `lane` of each 32-column chunk and keeps its running sum / sum of squares in registers across tiles
    [[maybe_unused]] float st_s[BLOCK_N / 32], st_q[BLOCK_N / 32];
    constexpr bool STATS = (EPI != 0);
    [[maybe_unused]] float* tr = stats_scratch + ew * (32 * kTrStride);
    if constexpr (STATS) {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 32; ++i) { st_s[i] = 0.f; st_q[i] = 0.f; }
    }
    if (p.b_resident) mbar_wait(&b_full[0], 0);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      WgAcc<BLOCK_N> acc;
      uint32_t acc_on = 0;                                   // 0 for the very first MMA of the tile
      if (p.mode != 2) {
        for (int q0 = 0; q0 < chunks_per_tile; q0 += p.KC) {
          B200_T0 mbar_wait(&s_full[ss], sph); B200_T1(d_wf)
          B200_T0
          wgmma_fence();
          uint32_t off = (uint32_t)(ss * p.s_stage_bytes);
          for (int j = 0; j < p.KC; ++j) {
            const uint64_t da = a_desc0 + (uint64_t)(off >> 4);
            const uint64_t db = p.b_resident ? b_desc_b0 + (uint64_t)(((uint32_t)(q0 + j) * (uint32_t)kBBytes) >> 4)
                                             : b_desc_s0 + (uint64_t)((off + p.a_chunk_bytes) >> 4);
#pragma unroll
            for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
              const uint64_t dak = da + (uint64_t)(k * ((UMMA_K * 2) >> 4));
              wgmma_tile<BLOCK_N, 0, kTB>(acc, dak, dak + kHalfA, db + (uint64_t)(k * (kStepB >> 4)), acc_on);
              acc_on = 1;
            }
            off += (uint32_t)p.chunk_stride;
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&s_empty[ss]);
          if (++ss == p.s_stages) { ss = 0; sph ^= 1; }
          B200_T1(d_mma)
        }
      } else {
        for (int cb = 0; cb < cblocks; ++cb) {
          B200_T0 mbar_wait(&s_full[ss], sph); B200_T1(d_wf)
          const uint32_t a_off = (uint32_t)(ss * p.s_stage_bytes);
          for (int tap0 = 0; tap0 < taps; tap0 += p.TB) {
            B200_T0 mbar_wait(&b_full[bs], bph); B200_T1(d_wf)
            B200_T0
            wgmma_fence();
            int r = tap0 / p.S, sx = tap0 - r * p.S;
            for (int j = 0; j < p.TB; ++j) {
              const int rr = p.mirror ? (p.R - 1 - r) : r, sc = p.mirror ? (p.S - 1 - sx) : sx;
              const uint64_t da = make_desc_rowoff(smem_u32(s_ring) + a_off + (uint32_t)(rr * p.Wp + sc) * 128u, 16, 1024, p.set_base_offset);
              const uint64_t db = b_desc_b0 + (uint64_t)((uint32_t)(bs * p.b_slot_bytes + j * kBBytes) >> 4);
#pragma unroll
              for (int k = 0; k < BLOCK_K / UMMA_K; ++k) {
                const uint64_t dak = da + (uint64_t)(k * ((UMMA_K * 2) >> 4));
                wgmma_tile<BLOCK_N, 0, kTB>(acc, dak, dak + kHalfA, db + (uint64_t)(k * (kStepB >> 4)), acc_on);
                acc_on = 1;
              }
              if (++sx == p.S) { sx = 0; ++r; }
            }
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(&b_empty[bs]);
              if (tap0 + p.TB >= taps) mbar_arrive(&s_empty[ss]);
            }
            if (++bs == p.b_stages) { bs = 0; bph ^= 1; }
            B200_T1(d_mma)
          }
          if (++ss == p.s_stages) { ss = 0; sph ^= 1; }
        }
      }
      B200_T0
      // ---- epilogue ----
      const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
      const int n0 = nt * BLOCK_N;
      int row0;
      if (p.mode == 0) row0 = mt * 128;
      else row0 = (((mt / p.tiles_h) * p.BI) * p.H + (mt % p.tiles_h) * p.BH) * p.W;
      int dense;
      bool valid = acc_row_to_dense(p, ew * 32 + lane, &dense);
      valid = valid && (row0 + dense < p.M_total);
      wg_bar_sync();                                         // the previous tile's epilogue is done reading acc_smem
      acc_to_smem<BLOCK_N>(acc, acc_smem, kAccStride, threadIdx.x - 128);
      wg_bar_sync();
#pragma unroll
      for (int c = 0; c < BLOCK_N; c += 64) {
        if (n0 + c >= p.Nc) break;                   // uniform over the CTA
        uint8_t* buf = staging + (slab & 1u) * kSlabBytes;
        const uint32_t buf_s = smem_u32(buf);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          uint32_t rr[32];
          acc_row_ld32(acc_smem, kAccStride, ew * 32 + lane, c + 32 * half, rr);
          if constexpr (EPI == 1) {
            float sv[32], qv[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const float v = __bfloat162float(__float2bfloat16_rn(__uint_as_float(rr[i])));   // the statistics describe the tensor as stored
              sv[i] = valid ? v : 0.f;
              qv[i] = sv[i] * sv[i];
            }
            const float cs = warp_column_sum32(sv, tr, lane);
            const float cq = warp_column_sum32(qv, tr, lane);
            const int ci = (c >> 5) + half;                 // 32-column chunk index inside the tile (compile-time after unrolling)
#pragma unroll
            for (int i = 0; i < BLOCK_N / 32; ++i)
              if (i == ci) { st_s[i] += cs; st_q[i] += cq; }
          }
          if constexpr (EPI == 2) {
            // data-gradient epilogue: (+ shortcut gradient) -> round to bf16 as stored -> partial sums of the BatchNorm backward that
            // consumes this tensor: S1 = sum dy*m, S2 = sum dy*m*xhat  (m = ReLU mask of that BatchNorm's output, xhat from its input)
            const int col0 = n0 + c + 32 * half;
            const size_t grow = (size_t)(row0 + dense);
            float v[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(rr[i]);
            if (p.addend != nullptr && valid) {
              const uint4* ap = reinterpret_cast<const uint4*>(p.addend + grow * p.Nc + col0);
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const uint4 raw = __ldg(ap + q);
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
                for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); v[8 * q + 2 * j] += f.x; v[8 * q + 2 * j + 1] += f.y; }
              }
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) { v[i] = __bfloat162float(__float2bfloat16_rn(v[i])); rr[i] = __float_as_uint(v[i]); }
            if (p.bn_x != nullptr) {
              float sv[32], qv[32];
              uint32_t mk = 0xffffffffu;
              float xv[32];
              if (valid) {
                const uint4* xp = reinterpret_cast<const uint4*>(p.bn_x + grow * p.Nc + col0);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const uint4 raw = __ldg(xp + q);
                  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
                  for (int j = 0; j < 4; ++j) { const float2 f = __bfloat1622float2(h[j]); xv[8 * q + 2 * j] = f.x; xv[8 * q + 2 * j + 1] = f.y; }
                }
                if (p.bn_mask != nullptr) mk = __ldg(reinterpret_cast<const uint32_t*>(p.bn_mask + grow * (size_t)(p.Nc >> 3) + (col0 >> 3)));
              } else {
                mk = 0u;
#pragma unroll
                for (int i = 0; i < 32; ++i) xv[i] = 0.f;
              }
              const float my_mean = (col0 + lane < p.Nc) ? __ldg(p.bn_mean + col0 + lane) : 0.f;
              const float my_rstd = (col0 + lane < p.Nc) ? __ldg(p.bn_rstd + col0 + lane) : 0.f;
#pragma unroll
              for (int i = 0; i < 32; ++i) {
                const float mean_i = __shfl_sync(0xffffffffu, my_mean, i), rstd_i = __shfl_sync(0xffffffffu, my_rstd, i);
                const float dyp = ((mk >> i) & 1u) ? v[i] : 0.f;
                sv[i] = dyp;
                qv[i] = dyp * (xv[i] - mean_i) * rstd_i;
              }
              const float cs = warp_column_sum32(sv, tr, lane);
              const float cq = warp_column_sum32(qv, tr, lane);
              const int ci = (c >> 5) + half;
#pragma unroll
              for (int i = 0; i < BLOCK_N / 32; ++i)
                if (i == ci) { st_s[i] += cs; st_q[i] += cq; }
            }
          }
          if (valid) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              __nv_bfloat162 h[4];
#pragma unroll
              for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(__uint_as_float(rr[8 * q + 2 * j]), __uint_as_float(rr[8 * q + 2 * j + 1]));
              const int chunk = half * 4 + q;              // 16-byte chunk inside the 128-byte staging row
              const uint32_t* w = reinterpret_cast<const uint32_t*>(h);
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                           ::"r"(buf_s + (uint32_t)(dense * 128 + ((chunk ^ (dense & 7)) << 4))), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
            }
          }
        }
        fence_async_smem();                          // generic-proxy writes -> visible to the TMA unit
        if (t0) bulk_wait_read_all();                // the store that read the OTHER staging tile has drained it
        epi_bar_sync();
        if (t0) { tma_store_2d(&map_d, buf, n0 + c, row0); bulk_commit(); }
        ++slab;
      }
      B200_T1(d_ep)
    }
    if (dbg) { p.dbg[5] = d_wf; p.dbg[6] = d_mma; p.dbg[9] = d_ep; }
    if (STATS && p.col_stats != nullptr) {
      // the four epilogue warps' sums are combined through shared memory (fixed order), then ONE row of the workspace per CTA:
      // [2][G = gridDim / num_n_tiles][Nc], row = blockIdx / num_n_tiles, columns of this CTA's n-tile
      float* comb = stats_scratch;                       // [4][2][BLOCK_N]
      epi_bar_sync();                                    // everyone is done with the transpose scratch
#pragma unroll
      for (int i = 0; i < BLOCK_N / 32; ++i) {
        comb[(ew * 2 + 0) * BLOCK_N + 32 * i + lane] = st_s[i];
        comb[(ew * 2 + 1) * BLOCK_N + 32 * i + lane] = st_q[i];
      }
      epi_bar_sync();
      const int nt = blockIdx.x % p.num_n_tiles;
      const size_t g = (size_t)(blockIdx.x / p.num_n_tiles), G = (size_t)(gridDim.x / p.num_n_tiles);
      for (int j = ew * 32 + lane; j < 2 * BLOCK_N; j += 128) {
        const int which = j / BLOCK_N, cc = j - which * BLOCK_N;
        const int col = nt * BLOCK_N + cc;
        if (col < p.Nc) {
          const float v = ((comb[(0 * 2 + which) * BLOCK_N + cc] + comb[(1 * 2 + which) * BLOCK_N + cc]) + comb[(2 * 2 + which) * BLOCK_N + cc]) +
                          comb[(3 * 2 + which) * BLOCK_N + cc];
          p.col_stats[((size_t)which * G + g) * p.Nc + col] = v;
        }
      }
    }
    if (t0) bulk_wait_all();                         // staging memory must outlive the last store
  }

  __syncthreads();
  if (p.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) p.dbg[10] = clock64() - t_begin;
}
#undef B200_T0
#undef B200_T1

// ---------------- host side ------------------------------------------------------------------------
struct MapKey {
  const void* ptr; uint64_t d[4]; uint64_t s[3]; uint32_t b[4]; int rank;
  bool operator==(const MapKey& o) const {
    if (ptr != o.ptr || rank != o.rank) return false;
    for (int i = 0; i < 4; ++i) if (d[i] != o.d[i] || b[i] != o.b[i]) return false;
    for (int i = 0; i < 3; ++i) if (s[i] != o.s[i]) return false;
    return true;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr) ^ (size_t)k.rank;
    for (int i = 0; i < 4; ++i) h = (h * 1000003u) ^ (size_t)k.d[i] ^ ((size_t)k.b[i] << 20);
    for (int i = 0; i < 3; ++i) h = (h * 1000003u) ^ (size_t)k.s[i];
    return h;
  }
};

}  // namespace

// bf16 tiled tensor map, 128B swizzle, rank <= 4 (dims / box innermost first; strides in bytes for dims 1..rank-1).  Cached:
// encoding costs a few microseconds on the host and the same (pointer, shape) recurs every step.
CUtensorMap conv_encode_map(const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides, const uint32_t* box) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  MapKey key{};
  key.ptr = ptr; key.rank = rank;
  for (int i = 0; i < rank; ++i) { key.d[i] = dims[i]; key.b[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) key.s[i] = strides[i];
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
  }
  auto& drv = Driver::get();
  if (!drv.TensorMapEncodeTiled) throw std::runtime_error("conv: cuTensorMapEncodeTiled unavailable");
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { B200_CUDA_CHECK(cudaFree(nullptr)); ctx_bound = true; }
  CUtensorMap map;
  cuuint64_t d[4], s[3];
  cuuint32_t b[4], es[4] = {1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) s[i] = strides[i];
  B200_DRV_CHECK(drv.TensorMapEncodeTiled(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), d, s, b, es,
                                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
  std::lock_guard<std::mutex> g(mu);
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, map);
  return map;
}

bool conv_tile_plan(int N, int H, int W, int R, int S, int want_mode, ConvTilePlan* plan) {
  ConvTilePlan pl;
  const int taps = R * S;
  if (taps == 1) {
    if (want_mode > 0) return false;
    pl.mode = 0;
    pl.num_m_tiles = ceil_div((long long)N * H * W, 128);
    pl.dense_rows = 128; pl.acc_rows = 128; pl.a_rows = 128;
    *plan = pl;
    return true;
  }
  if (R != 3 || S != 3) return false;
  auto halo = [&]() {
    const int Wp = W + 2;
    int bh = 0;
    for (int d = 1; d <= H; ++d)
      if (H % d == 0 && d * Wp <= 128 && (d + 2) * Wp <= 256 * 1) bh = d;      // box dims <= 256 each; rows checked below
    if (bh == 0 || Wp > 256 || bh + 2 > 256) return false;
    pl.mode = 2; pl.BH = bh; pl.BI = 1; pl.tiles_h = H / bh; pl.Wp = Wp;
    pl.num_m_tiles = N * pl.tiles_h;
    pl.dense_rows = bh * W; pl.acc_rows = bh * Wp; pl.a_rows = (bh + 2) * Wp;
    return true;
  };
  auto patch = [&]() {
    if (W > 128) return false;
    int bh = 0;
    for (int d = 1; d <= H; ++d)
      if (H % d == 0 && W * d <= 128) bh = d;
    if (bh == 0) return false;
    int bi = 1;
    if (bh == H)
      for (int d = 1; d <= N; ++d)
        if (N % d == 0 && W * H * d <= 128) bi = d;
    pl.mode = 1; pl.BH = bh; pl.BI = bi; pl.tiles_h = H / bh; pl.Wp = W;
    pl.num_m_tiles = (N / bi) * pl.tiles_h;
    pl.dense_rows = W * bh * bi; pl.acc_rows = pl.dense_rows; pl.a_rows = pl.dense_rows;
    return true;
  };
  bool ok;
  if (want_mode == 1) ok = patch();
  else if (want_mode == 2) ok = halo();
  else ok = halo() || patch();
  if (!ok) return false;
  *plan = pl;
  return true;
}

// persistent grid: one CTA per SM; with column statistics it is a multiple of num_n_tiles so that a CTA only sees one n-tile
int conv_grid_size(int num_m_tiles, int num_n_tiles, bool stats) {
  const long long tiles = (long long)num_m_tiles * num_n_tiles;
  int grid = tiles < kNumSMs ? (int)tiles : kNumSMs;
  if (stats && num_n_tiles > 1) {
    grid = (grid / num_n_tiles) * num_n_tiles;
    if (grid < num_n_tiles) grid = num_n_tiles;
  }
  return grid;
}

// A 128 x 128 fp32 accumulator is 128 registers per thread of the MMA warpgroup (two m64 halves of 64); a 256-wide tile would
// need 256, more than a thread can hold, so a requested 256-wide tile runs as two 128-wide n-tiles.
int conv_pick_block_n(int Nc, int num_m_tiles, int want) {
  (void)num_m_tiles;
  if (want == 256) return 128;
  if (want != 0) return want;
  return Nc % 128 != 0 ? 64 : 128;
}

int conv_stat_groups(int N, int H, int W, int Cin, int Cout, int R, int S, const ConvLaunchCfg& cfg) {
  ConvTilePlan pl;
  int mode = cfg.mode;
  if (mode < 0 && R == 3) mode = (Cin == 64) ? 2 : 1;
  if (!conv_tile_plan(N, H, W, R, S, mode, &pl)) return 0;
  const int bn = conv_pick_block_n(Cout, pl.num_m_tiles, cfg.block_n);
  const int nn = ceil_div(Cout, bn);
  return conv_grid_size(pl.num_m_tiles, nn, true) / nn;
}

namespace {

template <int BLOCK_N, bool B_MN, int EPI>
void launch_variant(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& md, TapGemmParams p, int want_kc, cudaStream_t stream) {
  constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  // All shared memory that is not the epilogue staging or the accumulator tile is ring depth.
  const int budget = 227 * 1024 - kStagingBytes - kBarrierBytes - 1024 - (EPI != 0 ? kStatsScratchBytes : 0) - acc_bytes(BLOCK_N);
  const int taps = p.R * p.S;
  if (p.mode != 2) {
    // ring S stage = KC x (activation chunk + filter chunk): one barrier wait + one wgmma group per KC * 4 k16 steps
    const int chunks_per_tile = (p.Kc / BLOCK_K) * taps;
    if (p.b_resident && (B_MN || p.num_n_tiles != 1)) throw std::runtime_error("conv: a resident filter needs a K-major filter and one n-tile");
    p.chunk_stride = p.a_chunk_bytes + (p.b_resident ? 0 : kBBytes);
    p.b_slot_bytes = p.b_resident ? chunks_per_tile * kBBytes : 0;
    p.b_stages = p.b_resident ? 1 : 0;
    const int chunk = p.chunk_stride;
    const int ring_budget = budget - p.b_stages * p.b_slot_bytes;
    int kc = want_kc > 0 ? want_kc : 2;
    while (kc > 1 && (chunks_per_tile % kc != 0 || ring_budget / (kc * chunk) < 3)) --kc;
    p.KC = kc; p.TB = 1;
    p.s_stage_bytes = kc * chunk;
    p.s_stages = ring_budget / p.s_stage_bytes;
    if (p.s_stages > kMaxRing) p.s_stages = kMaxRing;
    if (p.s_stages < 2) throw std::runtime_error("conv: shared memory budget exceeded");
  } else {
    // ring S = activation halo per channel block; ring B = TB filter taps per slot (a filter row when it fits)
    p.KC = 1; p.chunk_stride = 0; p.b_resident = 0;
    p.s_stage_bytes = p.a_chunk_bytes;
    int s_st = 0, b_st = 0;
    for (int tb = 3; tb >= 1; tb -= 2) {                   // one filter tap per slot when three leave too few slots
      if (tb == 3 && (3 * kBBytes > 48 * 1024 || taps % 3 != 0)) continue;
      p.TB = tb;
      p.b_slot_bytes = p.TB * kBBytes;
      const int groups = taps / p.TB;
      s_st = budget / (p.s_stage_bytes + groups * p.b_slot_bytes);
      if (s_st < 2) s_st = 2;
      if (s_st > kMaxRing) s_st = kMaxRing;
      b_st = (budget - s_st * p.s_stage_bytes) / p.b_slot_bytes;
      if (b_st > kMaxRing) b_st = kMaxRing;
      if (b_st >= 2) break;
    }
    if (b_st < 2) throw std::runtime_error("conv: shared memory budget exceeded");
    p.s_stages = s_st; p.b_stages = b_st;
  }
  const int smem = p.s_stages * p.s_stage_bytes + p.b_stages * p.b_slot_bytes + kStagingBytes + kBarrierBytes + 1024 + (EPI != 0 ? kStatsScratchBytes : 0) +
                   acc_bytes(BLOCK_N);
  auto kernel = conv_tap_gemm_kernel<BLOCK_N, B_MN, EPI>;
  static std::atomic<unsigned long long> configured{0};
  ensure_max_dynamic_smem(kernel, 227 * 1024, configured);
  const int grid = conv_grid_size(p.num_m_tiles, p.num_n_tiles, EPI != 0);
  kernel<<<grid, kThreads, smem, stream>>>(ma, mb, md, p);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace

void launch_conv_tap_gemm(const void* a, const void* w, void* d, int N, int H, int W, int Cin, int Cout, int R, int S, bool dgrad,
                          const ConvLaunchCfg& cfg, float* col_stats, cudaStream_t stream, const ConvBwdFusion* fuse) {
  const int Kc = dgrad ? Cout : Cin, Nc = dgrad ? Cin : Cout;
  if (Kc % BLOCK_K != 0 || Nc % 64 != 0) throw std::runtime_error("conv: channel counts must be multiples of 64");
  if (R != S || (R != 1 && R != 3)) throw std::runtime_error("conv: 1x1 or 3x3 filters");
  if (dgrad && fuse == nullptr && col_stats != nullptr) throw std::runtime_error("conv: column statistics ride on the forward pass only");
  if (fuse != nullptr && !dgrad) throw std::runtime_error("conv: the BatchNorm-backward fusion rides on the data gradient");
  if (fuse != nullptr && fuse->bn_x != nullptr && col_stats == nullptr) throw std::runtime_error("conv: fused BatchNorm backward needs the partial-sum workspace");
  ConvTilePlan pl;
  int mode = cfg.mode;
  // 3x3 tilings: the halo tiling when a tile's filter taps are small (64 reduction channels: layer1), where re-fetching the
  // patch for every tap would dominate; the patch tiling otherwise (its operand tiles start 1024-byte aligned)
  if (mode < 0 && R == 3) mode = (Kc == 64) ? 2 : 1;
  if (!conv_tile_plan(N, H, W, R, S, mode, &pl)) throw std::runtime_error("conv: no tile plan for this geometry");
  const long long M_total = (long long)N * H * W;
  TapGemmParams p{};
  p.M_total = (int)M_total; p.Kc = Kc; p.Nc = Nc;
  p.R = R; p.S = S; p.pad = (R - 1) / 2;
  p.mirror = dgrad ? 1 : 0;
  p.mode = pl.mode;
  p.H = H; p.W = W; p.BH = pl.BH; p.BI = pl.BI; p.tiles_h = pl.tiles_h; p.Wp = pl.Wp;
  p.num_m_tiles = pl.num_m_tiles;
  p.dense_rows = pl.dense_rows;
  p.a_tx_bytes = (uint32_t)(pl.a_rows * 128);
  p.a_chunk_bytes = ((pl.a_rows * 128 + 1023) / 1024) * 1024;
  if (p.a_chunk_bytes < 128 * 128) p.a_chunk_bytes = 128 * 128;   // the MMA reads 128 rows from the chunk start
  p.set_base_offset = cfg.set_base_offset;
  p.b_tap_stride = Cin;
  p.row_mul = 1;
  p.b_resident = 0;
  p.col_stats = col_stats;
  p.addend = fuse ? reinterpret_cast<const __nv_bfloat16*>(fuse->addend) : nullptr;
  p.bn_x = fuse ? reinterpret_cast<const __nv_bfloat16*>(fuse->bn_x) : nullptr;
  p.bn_mask = fuse ? reinterpret_cast<const uint8_t*>(fuse->bn_mask) : nullptr;
  p.bn_mean = fuse ? fuse->bn_mean : nullptr;
  p.bn_rstd = fuse ? fuse->bn_rstd : nullptr;
  p.dbg = reinterpret_cast<long long*>(cfg.debug_counters);
  const int block_n = conv_pick_block_n(Nc, pl.num_m_tiles, cfg.block_n);
  if (block_n != 64 && block_n != 128) throw std::runtime_error("conv: block_n must be 0 (auto), 64, 128 or 256 (runs as two 128-wide n-tiles)");
  p.num_n_tiles = ceil_div(Nc, block_n);

  // activation map
  CUtensorMap ma;
  if (pl.mode == 0) {
    uint64_t dm[4] = {(uint64_t)Kc, (uint64_t)M_total, 1, 1};
    uint64_t st[3] = {(uint64_t)Kc * 2, (uint64_t)Kc * 2 * (uint64_t)M_total, (uint64_t)Kc * 2 * (uint64_t)M_total};
    uint32_t bx[4] = {64, 128, 1, 1};
    ma = conv_encode_map(a, 4, dm, st, bx);
  } else {
    uint64_t dm[4] = {(uint64_t)Kc, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t st[3] = {(uint64_t)Kc * 2, (uint64_t)W * Kc * 2, (uint64_t)H * W * Kc * 2};
    uint32_t bx[4] = {64, (uint32_t)(pl.mode == 2 ? pl.Wp : W), (uint32_t)(pl.mode == 2 ? pl.BH + 2 : pl.BH), (uint32_t)pl.BI};
    ma = conv_encode_map(a, 4, dm, st, bx);
  }
  // filter map: [Cout, R*S*Cin] row-major
  CUtensorMap mb;
  {
    uint64_t dm[2] = {(uint64_t)R * S * Cin, (uint64_t)Cout};
    uint64_t st[1] = {(uint64_t)R * S * Cin * 2};
    uint32_t bx[2] = {64, (uint32_t)(dgrad ? 64 : block_n)};
    mb = conv_encode_map(w, 2, dm, st, bx);
  }
  // output map: [M_total, Nc] row-major, one dense tile per store
  CUtensorMap md;
  {
    uint64_t dm[2] = {(uint64_t)Nc, (uint64_t)M_total};
    uint64_t st[1] = {(uint64_t)Nc * 2};
    uint32_t bx[2] = {64, (uint32_t)pl.dense_rows};
    md = conv_encode_map(d, 2, dm, st, bx);
  }
#define B200_CONV_DISPATCH(BN)                                                                         \
  if (block_n == BN) {                                                                                 \
    if (dgrad && fuse != nullptr) launch_variant<BN, true, 2>(ma, mb, md, p, cfg.kc, stream);          \
    else if (dgrad) launch_variant<BN, true, 0>(ma, mb, md, p, cfg.kc, stream);                        \
    else if (col_stats != nullptr) launch_variant<BN, false, 1>(ma, mb, md, p, cfg.kc, stream);        \
    else launch_variant<BN, false, 0>(ma, mb, md, p, cfg.kc, stream);                                  \
    return;                                                                                            \
  }
  B200_CONV_DISPATCH(64)
  B200_CONV_DISPATCH(128)
#undef B200_CONV_DISPATCH
}

// ---- strided 7x7 stem: the same kernel, patch tiling with one output row per tile and four taps of 64 over the row-pair image ----
int stem_stat_groups(int N, int H, int W) {
  StemGeom g;
  if (!stem_geom(H, W, &g)) return 0;
  return conv_grid_size(N * g.Ho, 1, true);
}

void launch_stem_conv_fprop(const void* xp, const void* w2, void* y, int N, int H, int W, int Cout, float* col_stats, bool resident_filter,
                            void* debug_counters, cudaStream_t stream) {
  StemGeom g;
  if (!stem_geom(H, W, &g)) throw std::runtime_error("stem conv: unsupported image size");
  if (Cout != 64) throw std::runtime_error("stem conv: 64 output channels");
  const long long M_total = (long long)N * g.Ho * g.Wo;
  TapGemmParams p{};
  p.M_total = (int)M_total; p.Kc = 64; p.Nc = Cout;
  p.R = kStemTaps; p.S = 1; p.pad = 0; p.mirror = 0;
  p.mode = 1;
  p.H = g.Ho; p.W = g.Wo; p.BH = 1; p.BI = 1; p.tiles_h = g.Ho; p.Wp = g.Wo;
  p.num_m_tiles = N * g.Ho;
  p.num_n_tiles = 1;
  p.dense_rows = g.Wo;
  p.a_tx_bytes = (uint32_t)(g.Wo * 128);
  p.a_chunk_bytes = 128 * 128;
  p.b_tap_stride = 64;
  p.row_mul = 1;                                     // pair row of output row oh and tap t: oh + t
  p.b_resident = resident_filter ? 1 : 0;
  p.col_stats = col_stats;
  p.dbg = reinterpret_cast<long long*>(debug_counters);
  const uint64_t row_pitch = (uint64_t)g.Wp * 16;
  CUtensorMap ma, mb, md;
  {   // overlapping windows: 64 elements (8 sixteen-byte pixels) every 32 bytes
    uint64_t dm[4] = {64, (uint64_t)g.Wo, (uint64_t)g.Hp2, (uint64_t)N};
    uint64_t st[3] = {32, row_pitch, row_pitch * (uint64_t)g.Hp2};
    uint32_t bx[4] = {64, (uint32_t)g.Wo, 1, 1};
    ma = conv_encode_map(xp, 4, dm, st, bx);
  }
  {
    uint64_t dm[2] = {(uint64_t)kStemK, (uint64_t)Cout};
    uint64_t st[1] = {(uint64_t)kStemK * 2};
    uint32_t bx[2] = {64, 64};
    mb = conv_encode_map(w2, 2, dm, st, bx);
  }
  {
    uint64_t dm[2] = {(uint64_t)Cout, (uint64_t)M_total};
    uint64_t st[1] = {(uint64_t)Cout * 2};
    uint32_t bx[2] = {64, (uint32_t)g.Wo};
    md = conv_encode_map(y, 2, dm, st, bx);
  }
  if (col_stats != nullptr) launch_variant<64, false, 1>(ma, mb, md, p, 0, stream);
  else launch_variant<64, false, 0>(ma, mb, md, p, 0, stream);
}

}  // namespace b200
