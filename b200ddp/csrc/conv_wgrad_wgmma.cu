// Convolution weight gradient for channels_last bf16 activations on the Hopper tensor cores (replaces cuDNN's wgrad kernels
// when selected, see ops/functional.py).
//
//   dw[co, (r,s), ci] = sum over pixels p of dy[p, co] * x[p shifted by the tap, ci]
//
// As a GEMM the reduction runs over PIXELS, so both operands are "MN-major": dy is stored [pixels, Cout], x is stored
// [pixels, Cin] - exactly the 128-byte-row shared-memory layout wgmma reads MN-major operands from, no transposes.
// The reduction is long (up to 100 352 pixels) and the output small, so the pixel range is SPLIT across all SMs:
//   unit = (block of 128 output channels, tile of input channels, filter tap, pixel range)
// Each CTA keeps one 128 x tile_n fp32 accumulator in the registers of its MMA warpgroup and writes an fp32 partial; a second
// kernel sums the partials in a fixed order (deterministic, no atomics) and emits bf16.  3x3 taps re-fetch the shifted x
// patch with a rank-4 TMA box; rows / columns outside the image arrive as zeros (the padding).
#include "conv.h"

#include <cuda.h>

#include "tc_primitives.cuh"
#include "tensor_map.h"

namespace b200 {
namespace {
using namespace tc;

constexpr int UMMA_K = 16;
constexpr int kThreads = 256;                  // warp 0: dy producer, warp 3: x producer, warps 4-7: MMA warpgroup
constexpr int kMmaWarps = 4;
constexpr int kMaxRing = 12;
constexpr int kBarrierBytes = 1024;

struct WgradParams {
  int Cout, Cin, R, S, pad;
  int mode;                 // 0 flat (1x1): pixel block = KB consecutive pixels; 1 patch: pixel block = BI images x BH rows x W columns
  int H, W, BH, BI, tiles_h;
  int row_mul;              // patch mode: x row of pixel-block row h and tap r is row_mul * h + r - pad (2 for the strided stem)
  int KB;                   // pixels (shared-memory rows) per pixel block, multiple of 16
  int num_kblocks;          // pixel blocks in the whole tensor
  int MB, TG, tile_n;       // Cout blocks of 128 per CTA (1), taps per CTA (1), input channels per CTA (64 or 128)
  int m_groups, n_tiles, tap_groups, split;
  int a_slot_bytes, b_slot_bytes, a_stages, b_stages;
  float* partial;           // [split][Cout][R*S*Cin]
};

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

__device__ __forceinline__ bool elect_one() {     // one lane of a converged warp (see conv_wgmma.cu)
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}

// One m64 accumulator half as fp32 rows of a row-major matrix: thread t holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) of the half
// and column pairs 8 j + 2 (t % 4).  Rows >= rows_valid / columns >= cols_valid are not stored; zero = no pixels were summed.
template <int N>
__device__ __forceinline__ void store_half_rows(const float (&h)[N / 2], float* out, size_t ld, int rows_valid, int cols_valid, bool zero, int wg_thread) {
  const int r0 = (wg_thread >> 5) * 16 + ((wg_thread & 31) >> 2), c0 = 2 * (wg_thread & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int hi = 0; hi < 2; ++hi) {
      const int r = r0 + 8 * hi, c = 8 * j + c0;
      if (r < rows_valid && c < cols_valid)
        *reinterpret_cast<float2*>(out + (size_t)r * ld + c) = zero ? make_float2(0.f, 0.f) : make_float2(h[4 * j + 2 * hi], h[4 * j + 2 * hi + 1]);
    }
  }
}

template <int TILE_N>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x, const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = a_ring + p.a_stages * p.a_slot_bytes;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(b_ring + p.b_stages * p.b_slot_bytes);
  uint64_t* a_empty = a_full + kMaxRing;
  uint64_t* b_full = a_empty + kMaxRing;
  uint64_t* b_empty = b_full + kMaxRing;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // unit -> (output tile group, pixel range)
  const int unit = blockIdx.x;
  const int grp = unit / p.split, sp = unit - grp * p.split;
  const int tg = grp % p.tap_groups;
  const int nt = (grp / p.tap_groups) % p.n_tiles;
  const int mg = grp / (p.tap_groups * p.n_tiles);
  const int taps = p.R * p.S;
  const int tap0 = tg * p.TG;
  const int ntaps = min(p.TG, taps - tap0);
  const int co0 = mg * p.MB * 128;
  const int ci0 = nt * p.tile_n;
  const int kb0 = (int)(((long long)p.num_kblocks * sp) / p.split);
  const int kb1 = (int)(((long long)p.num_kblocks * (sp + 1)) / p.split);
  const int chunk_bytes = p.KB * 128;                       // one 64-channel chunk of a pixel block
  const int a_chunks = p.MB * 2, b_chunks = p.tile_n / 64;

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&map_dy); tma_prefetch_desc(&map_x); }
  if (warp == 1) {
    if (lane < kMaxRing) { mbar_init(&a_full[lane], 1); mbar_init(&a_empty[lane], kMmaWarps); mbar_init(&b_full[lane], 1); mbar_init(&b_empty[lane], kMmaWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer for dy (converged warp, one elected lane issues) =====================
    int as = 0;
    uint32_t aph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      int c1 = 0, c2 = 0, c3 = 0;                          // coordinates of the pixel block (dims 1..3 of the maps)
      if (p.mode == 0) c1 = kb * p.KB;
      else { c3 = (kb / p.tiles_h) * p.BI; c2 = (kb % p.tiles_h) * p.BH; }
      mbar_wait(&a_empty[as], aph ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&a_full[as], (uint32_t)(a_chunks * chunk_bytes));
        for (int j = 0; j < a_chunks; ++j)                  // channels beyond Cout arrive as zeros
          tma_load_4d(&map_dy, &a_full[as], a_ring + as * p.a_slot_bytes + j * chunk_bytes, co0 + 64 * j, c1, c2, c3);
      }
      __syncwarp();
      if (++as == p.a_stages) { as = 0; aph ^= 1; }
    }
  } else if (warp == 3) {
    // ===================== TMA producer for the (shifted) x tiles =====================
    int bs = 0;
    uint32_t bph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      int c1 = 0, c2 = 0, c3 = 0;
      if (p.mode == 0) c1 = kb * p.KB;
      else { c3 = (kb / p.tiles_h) * p.BI; c2 = (kb % p.tiles_h) * p.BH; }
      int r = tap0 / p.S, sx = tap0 - r * p.S;
      for (int t = 0; t < ntaps; ++t) {
        mbar_wait(&b_empty[bs], bph ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&b_full[bs], (uint32_t)(b_chunks * chunk_bytes));
          for (int j = 0; j < b_chunks; ++j)
            tma_load_4d(&map_x, &b_full[bs], b_ring + bs * p.b_slot_bytes + j * chunk_bytes, ci0 + 64 * j,
                        p.mode == 0 ? c1 : sx - p.pad, p.mode == 0 ? 0 : c2 * p.row_mul + r - p.pad, c3);
        }
        __syncwarp();
        if (++sx == p.S) { sx = 0; ++r; }
        if (++bs == p.b_stages) { bs = 0; bph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================== MMA warpgroup: wgmma into registers, then the fp32 partial =====================
    const uint32_t lbo = (uint32_t)chunk_bytes;             // next 64-wide MN chunk
    const int ksteps = p.KB / UMMA_K;
    const uint64_t a_desc0 = make_smem_desc(smem_u32(a_ring), lbo, 1024);
    const uint64_t b_desc0 = make_smem_desc(smem_u32(b_ring), lbo, 1024);
    const uint64_t half_a = (uint64_t)(chunk_bytes >> 4);   // Cout rows [64, 128): the second 64-wide chunk of the dy slot
    WgAcc<TILE_N> acc;
    int as = 0, bs = 0;
    uint32_t aph = 0, bph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&a_full[as], aph);
      for (int t = 0; t < ntaps; ++t) {
        mbar_wait(&b_full[bs], bph);
        wgmma_fence();
        const uint64_t da0 = a_desc0 + (uint64_t)((uint32_t)(as * p.a_slot_bytes) >> 4);
        const uint64_t db0 = b_desc0 + (uint64_t)((uint32_t)(bs * p.b_slot_bytes) >> 4);
        for (int k = 0; k < ksteps; ++k) {
          const uint64_t step = (uint64_t)(k * ((UMMA_K * 128) >> 4));
          wgmma_tile<TILE_N, 1, 1>(acc, da0 + step, da0 + half_a + step, db0 + step, (kb != kb0 || k != 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&b_empty[bs]);
          if (t == ntaps - 1) mbar_arrive(&a_empty[as]);
        }
        if (++bs == p.b_stages) { bs = 0; bph ^= 1; }
      }
      if (++as == p.a_stages) { as = 0; aph ^= 1; }
    }
    const int row_len = taps * p.Cin;
    float* out = p.partial + (size_t)sp * p.Cout * row_len + (size_t)co0 * row_len + (size_t)tap0 * p.Cin + ci0;
#pragma unroll
    for (int half = 0; half < 2; ++half)
      store_half_rows<TILE_N>(acc.h[half], out + (size_t)(64 * half) * row_len, (size_t)row_len, p.Cout - co0 - 64 * half, p.Cin - ci0,
                              kb1 <= kb0, threadIdx.x - 128);
  }
}

// out[e] = bf16( sum_s partial[s][e] ).  Block = 32 element-vectors (8 floats each) x 8 split lanes: lane j sums splits j, j+8, ...
// in order, the 8 lane sums are combined in order through shared memory -> a fixed summation tree (deterministic, no atomics)
// with 8x the memory-level parallelism of a serial loop over `split` (up to 132) partials.
__global__ void __launch_bounds__(256) conv_wgrad_reduce_kernel(const float* __restrict__ partial, __nv_bfloat16* __restrict__ out, size_t n, int split) {
  __shared__ float sm[8][32][9];
  const int v = threadIdx.x & 31, sl = threadIdx.x >> 5;
  const size_t e = ((size_t)blockIdx.x * 32 + v) * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (e < n) {
#pragma unroll 2
    for (int s = sl; s < split; s += 8) {
      const float4 lo = __ldcg(reinterpret_cast<const float4*>(partial + (size_t)s * n + e));
      const float4 hi = __ldcg(reinterpret_cast<const float4*>(partial + (size_t)s * n + e + 4));
      acc[0] += lo.x; acc[1] += lo.y; acc[2] += lo.z; acc[3] += lo.w;
      acc[4] += hi.x; acc[5] += hi.y; acc[6] += hi.z; acc[7] += hi.w;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sm[sl][v][i] = acc[i];
  __syncthreads();
  if (sl == 0 && e < n) {
#pragma unroll
    for (int j = 1; j < 8; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += sm[j][v][i];
    *reinterpret_cast<Bf16x8*>(out + e) = pack8(acc);
  }
}

struct WgradPlan {
  WgradParams p;
  int smem;
  int grid;
};

bool wgrad_plan(int N, int H, int W, int Cin, int Cout, int R, int S, const WgradCfg& cfg, WgradPlan* out) {
  if (Cin % 64 != 0 || Cout % 64 != 0 || R != S || (R != 1 && R != 3)) return false;
  WgradParams p{};
  p.Cout = Cout; p.Cin = Cin; p.R = R; p.S = S; p.pad = (R - 1) / 2;
  p.H = H; p.W = W; p.row_mul = 1;
  const int taps = R * S;
  if (taps == 1) {
    p.mode = 0; p.KB = 64;
    p.num_kblocks = ceil_div((long long)N * H * W, p.KB);
    p.BH = p.BI = p.tiles_h = 0;
  } else {
    // pixel block = whole rows; the row count is rounded up so that KB is a multiple of 16 - rows beyond the image are
    // zero-filled by the TMA unit in BOTH operands and contribute nothing
    p.mode = 1;
    int bh = 0, bi = 1;
    for (int d = 1; d <= 16 && bh == 0; ++d) {              // smallest patch with >= 96 rows, KB % 16 == 0, KB <= 128
      for (int i = 1; i <= (d >= H ? 4 : 1); ++i) {
        const int kb = W * d * i;
        if (kb % 16 == 0 && kb >= 96 && kb <= 128) { bh = d; bi = i; break; }
      }
    }
    if (bh == 0) {                                          // fall back: any multiple of 16 up to 128
      for (int d = 1; d <= H + 15 && bh == 0; ++d)
        if ((W * d) % 16 == 0 && W * d <= 128) bh = d;
      if (bh == 0) return false;
    }
    if (bi > 1 && N % bi != 0) return false;
    p.BH = bh; p.BI = bi; p.tiles_h = ceil_div(H, bh);
    p.KB = W * bh * bi;
    p.num_kblocks = (N / bi) * p.tiles_h;
  }
  // output tiling
  // One 128 x tile_n accumulator per CTA (128 registers per thread of the MMA warpgroup at tile_n = 128): one Cout block of 128,
  // one filter tap, 64 or 128 input channels.
  const int MB = 1, TG = 1;
  int tile_n = Cin < 128 ? Cin : 128;
  if (cfg.tile_m > 0 && cfg.tile_m != 128) return false;
  if (cfg.tile_n > 0) tile_n = cfg.tile_n;
  if ((tile_n != 64 && tile_n != 128) || tile_n > Cin) return false;
  p.MB = MB; p.TG = TG; p.tile_n = tile_n;
  p.m_groups = ceil_div(Cout, 128 * MB);
  p.n_tiles = ceil_div(Cin, tile_n);
  p.tap_groups = ceil_div(taps, TG);
  const int groups = p.m_groups * p.n_tiles * p.tap_groups;
  int split = cfg.split > 0 ? cfg.split : kNumSMs / groups;
  if (split < 1) split = 1;
  if (split > p.num_kblocks) split = p.num_kblocks;
  p.split = split;
  const int chunk = p.KB * 128;
  p.a_slot_bytes = MB * 2 * chunk;
  p.b_slot_bytes = (tile_n / 64) * chunk;
  // all of shared memory is prefetch depth (the pixel stream comes from HBM: bytes in flight / latency bounds a CTA);
  const int budget = 227 * 1024 - kBarrierBytes - 1024;
  int ast = budget / (p.a_slot_bytes + TG * p.b_slot_bytes);
  if (ast < 1) ast = 1;
  if (ast > kMaxRing) ast = kMaxRing;
  int bst = (budget - ast * p.a_slot_bytes) / p.b_slot_bytes;
  if (bst > kMaxRing) bst = kMaxRing;
  if (bst < 1) return false;
  p.a_stages = ast;
  p.b_stages = bst;
  out->p = p;
  out->smem = p.a_stages * p.a_slot_bytes + p.b_stages * p.b_slot_bytes + kBarrierBytes + 1024;
  out->grid = groups * split;
  return true;
}

void launch_wgrad_kernel(const CUtensorMap& mdy, const CUtensorMap& mx, const WgradPlan& pl, cudaStream_t stream) {
  if (pl.p.tile_n == 64) {
    static std::atomic<unsigned long long> configured{0};
    ensure_max_dynamic_smem(conv_wgrad_kernel<64>, 227 * 1024, configured);
    conv_wgrad_kernel<64><<<pl.grid, kThreads, pl.smem, stream>>>(mdy, mx, pl.p);
  } else {
    static std::atomic<unsigned long long> configured{0};
    ensure_max_dynamic_smem(conv_wgrad_kernel<128>, 227 * 1024, configured);
    conv_wgrad_kernel<128><<<pl.grid, kThreads, pl.smem, stream>>>(mdy, mx, pl.p);
  }
}

}  // namespace

size_t conv_wgrad_workspace_floats(int N, int H, int W, int Cin, int Cout, int R, int S, const WgradCfg& cfg) {
  WgradPlan pl;
  if (!wgrad_plan(N, H, W, Cin, Cout, R, S, cfg, &pl)) return 0;
  return (size_t)pl.p.split * Cout * R * S * Cin;
}

void launch_conv_wgrad(const void* dy, const void* x, void* dw, int N, int H, int W, int Cin, int Cout, int R, int S,
                       const WgradCfg& cfg, float* workspace, cudaStream_t stream) {
  WgradPlan pl;
  if (!wgrad_plan(N, H, W, Cin, Cout, R, S, cfg, &pl)) throw std::runtime_error("conv wgrad: unsupported geometry / tiling");
  WgradParams& p = pl.p;
  p.partial = workspace;
  const long long M_total = (long long)N * H * W;
  CUtensorMap mdy, mx;
  if (p.mode == 0) {
    uint64_t dd[4] = {(uint64_t)Cout, (uint64_t)M_total, 1, 1};
    uint64_t ds[3] = {(uint64_t)Cout * 2, (uint64_t)Cout * 2 * (uint64_t)M_total, (uint64_t)Cout * 2 * (uint64_t)M_total};
    uint32_t bx[4] = {64, (uint32_t)p.KB, 1, 1};
    mdy = encode_tensor_map(dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 4, dd, ds, bx);
    uint64_t xd[4] = {(uint64_t)Cin, (uint64_t)M_total, 1, 1};
    uint64_t xs[3] = {(uint64_t)Cin * 2, (uint64_t)Cin * 2 * (uint64_t)M_total, (uint64_t)Cin * 2 * (uint64_t)M_total};
    mx = encode_tensor_map(x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 4, xd, xs, bx);
  } else {
    uint32_t bx[4] = {64, (uint32_t)W, (uint32_t)p.BH, (uint32_t)p.BI};
    uint64_t dd[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t ds[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
    mdy = encode_tensor_map(dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 4, dd, ds, bx);
    uint64_t xd[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t xs[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
    mx = encode_tensor_map(x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 4, xd, xs, bx);
  }
  launch_wgrad_kernel(mdy, mx, pl, stream);
  B200_CUDA_CHECK(cudaGetLastError());
  const size_t n = (size_t)Cout * R * S * Cin;
  conv_wgrad_reduce_kernel<<<(unsigned)((n / 8 + 31) / 32), 256, 0, stream>>>(workspace, reinterpret_cast<__nv_bfloat16*>(dw), n, p.split);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

// ---- strided 7x7 stem (conv.h): the x operand is the overlapping-window tensor map over the row-pair image --------------------
// Dedicated kernel (variant 0).  The generic kernel above puts Cout on the accumulator rows, which for Cout = 64 wastes half of
// every MMA and needs one MMA group per tap.  Here the WINDOW ELEMENTS are the rows: one 128-row operand = two taps side by side
// (two 64-wide MN-major chunks, LBO apart), the 64 output channels are the columns:
//   D_g[(tap 2g + c) * 64 + e, co] += sum over the pixels of one output row of  window_{2g+c}[pixel, e] * dy[pixel, co],   g = 0, 1
// -> two MMA groups per output row instead of four (seven before the row-pair packing), every dy row loaded once and never
// zero-padded.  Pixel range split over all SMs, fp32 partials [split][256][Cout], reduced by conv_wgrad_reduce_kernel.
namespace {

struct StemWgradParams {
  int KB;                   // pixels per block = Wo
  int Ho, num_kblocks, split, Cout;
  int chunk_bytes, a_stages, b_stages;
  float* partial;           // [split][kStemK][Cout]
};
constexpr int kStemGroups = kStemTaps / 2;

__global__ void __launch_bounds__(kThreads, 1)
stem_wgrad_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_dy, const StemWgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int a_slot_bytes = 2 * p.chunk_bytes;
  uint8_t* a_ring = smem;                                    // window pairs
  uint8_t* b_ring = a_ring + p.a_stages * a_slot_bytes;      // dy rows
  uint64_t* a_full = reinterpret_cast<uint64_t*>(b_ring + p.b_stages * p.chunk_bytes);
  uint64_t* a_empty = a_full + kMaxRing;
  uint64_t* b_full = a_empty + kMaxRing;
  uint64_t* b_empty = b_full + kMaxRing;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sp = blockIdx.x;
  const int kb0 = (int)(((long long)p.num_kblocks * sp) / p.split);
  const int kb1 = (int)(((long long)p.num_kblocks * (sp + 1)) / p.split);

  if (warp == 0 && lane == 0) { tma_prefetch_desc(&map_x); tma_prefetch_desc(&map_dy); }
  if (warp == 1) {
    if (lane < kMaxRing) { mbar_init(&a_full[lane], 1); mbar_init(&a_empty[lane], kMmaWarps); mbar_init(&b_full[lane], 1); mbar_init(&b_empty[lane], kMmaWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== window producer: two taps (pair rows oh + 2g, oh + 2g + 1) per slot =====================
    int as = 0;
    uint32_t aph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      const int img = kb / p.Ho, oh = kb - img * p.Ho;
      for (int g = 0; g < kStemGroups; ++g) {
        mbar_wait(&a_empty[as], aph ^ 1);
        if (elect_one()) {
          uint8_t* dst = a_ring + as * a_slot_bytes;
          mbar_expect_tx(&a_full[as], (uint32_t)(2 * p.chunk_bytes));
          tma_load_4d(&map_x, &a_full[as], dst, 0, 0, oh + 2 * g, img);
          tma_load_4d(&map_x, &a_full[as], dst + p.chunk_bytes, 0, 0, oh + 2 * g + 1, img);
        }
        __syncwarp();
        if (++as == p.a_stages) { as = 0; aph ^= 1; }
      }
    }
  } else if (warp == 3) {
    // ===================== dy producer: one output row of gradients per slot =====================
    int bs = 0;
    uint32_t bph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      const int img = kb / p.Ho, oh = kb - img * p.Ho;
      mbar_wait(&b_empty[bs], bph ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&b_full[bs], (uint32_t)p.chunk_bytes);
        tma_load_4d(&map_dy, &b_full[bs], b_ring + bs * p.chunk_bytes, 0, 0, oh, img);
      }
      __syncwarp();
      if (++bs == p.b_stages) { bs = 0; bph ^= 1; }
    }
  } else if (warp >= 4) {
    // ===================== MMA warpgroup: one 128 x 64 accumulator per tap pair =====================
    const int ksteps = p.KB / UMMA_K;
    const uint64_t a_desc0 = make_smem_desc(smem_u32(a_ring), (uint32_t)p.chunk_bytes, 1024);
    const uint64_t b_desc0 = make_smem_desc(smem_u32(b_ring), (uint32_t)p.chunk_bytes, 1024);
    const uint64_t half_a = (uint64_t)(p.chunk_bytes >> 4);   // window rows [64, 128): the second tap of the pair
    WgAcc<64> acc[kStemGroups];
    int as = 0, bs = 0;
    uint32_t aph = 0, bph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&b_full[bs], bph);
#pragma unroll
      for (int g = 0; g < kStemGroups; ++g) {
        mbar_wait(&a_full[as], aph);
        wgmma_fence();
        const uint64_t da0 = a_desc0 + (uint64_t)((uint32_t)(as * a_slot_bytes) >> 4);
        const uint64_t db0 = b_desc0 + (uint64_t)((uint32_t)(bs * p.chunk_bytes) >> 4);
        for (int k = 0; k < ksteps; ++k) {
          const uint64_t step = (uint64_t)(k * ((UMMA_K * 128) >> 4));
          wgmma_tile<64, 1, 1>(acc[g], da0 + step, da0 + half_a + step, db0 + step, (kb != kb0 || k != 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&a_empty[as]);
          if (g == kStemGroups - 1) mbar_arrive(&b_empty[bs]);
        }
        if (++as == p.a_stages) { as = 0; aph ^= 1; }
      }
      if (++bs == p.b_stages) { bs = 0; bph ^= 1; }
    }
    // fp32 partial [kStemK][Cout] of this split: row = packed filter index (tap pair g, window element)
    float* base = p.partial + (size_t)sp * kStemK * p.Cout;
#pragma unroll
    for (int g = 0; g < kStemGroups; ++g)
#pragma unroll
      for (int half = 0; half < 2; ++half)
        store_half_rows<64>(acc[g].h[half], base + (size_t)(g * 128 + 64 * half) * p.Cout, (size_t)p.Cout, 64, p.Cout, kb1 <= kb0, threadIdx.x - 128);
  }
}

bool stem_generic_plan(int N, int H, int W, int Cout, WgradPlan* out) {      // variant 1: generic kernel, four taps
  StemGeom g;
  if (!stem_geom(H, W, &g) || Cout != 64) return false;
  WgradParams p{};
  p.Cout = Cout; p.Cin = 64; p.R = kStemTaps; p.S = 1; p.pad = 0;
  p.mode = 1; p.H = g.Ho; p.W = g.Wo; p.BH = 1; p.BI = 1; p.tiles_h = g.Ho; p.row_mul = 1;
  p.KB = g.Wo;
  p.num_kblocks = N * g.Ho;
  p.MB = 1; p.TG = 1; p.tile_n = 64;
  p.m_groups = 1; p.n_tiles = 1; p.tap_groups = kStemTaps;
  p.split = kNumSMs / kStemTaps;
  if (p.split > p.num_kblocks) p.split = p.num_kblocks;
  const int chunk = p.KB * 128;
  p.a_slot_bytes = 2 * chunk;
  p.b_slot_bytes = chunk;
  const int budget = 227 * 1024 - kBarrierBytes - 1024;
  p.a_stages = 3;
  int bst = (budget - p.a_stages * p.a_slot_bytes) / p.b_slot_bytes;
  if (bst > kMaxRing) bst = kMaxRing;
  if (bst < 2) return false;
  p.b_stages = bst;
  out->p = p;
  out->smem = p.a_stages * p.a_slot_bytes + p.b_stages * p.b_slot_bytes + kBarrierBytes + 1024;
  out->grid = p.tap_groups * p.split;
  return true;
}

bool stem_dedicated_plan(int N, int H, int W, int Cout, StemWgradParams* out, int* smem) {
  StemGeom g;
  if (!stem_geom(H, W, &g) || Cout != 64) return false;
  StemWgradParams p{};
  p.KB = g.Wo; p.Ho = g.Ho; p.Cout = Cout;
  p.num_kblocks = N * g.Ho;
  p.split = p.num_kblocks < kNumSMs ? p.num_kblocks : kNumSMs;
  p.chunk_bytes = p.KB * 128;
  const int budget = 227 * 1024 - kBarrierBytes - 1024;
  p.b_stages = 3;
  int ast = (budget - p.b_stages * p.chunk_bytes) / (2 * p.chunk_bytes);
  if (ast > kMaxRing) ast = kMaxRing;
  if (ast < 2) return false;
  p.a_stages = ast;
  *out = p;
  *smem = p.a_stages * 2 * p.chunk_bytes + p.b_stages * p.chunk_bytes + kBarrierBytes + 1024;
  return true;
}
}  // namespace

size_t stem_wgrad_workspace_floats(int N, int H, int W, int Cout, int variant) {
  if (variant == 1) {
    WgradPlan pl;
    if (!stem_generic_plan(N, H, W, Cout, &pl)) return 0;
    return (size_t)pl.p.split * Cout * kStemK;
  }
  StemWgradParams p; int smem;
  if (!stem_dedicated_plan(N, H, W, Cout, &p, &smem)) return 0;
  return (size_t)p.split * Cout * kStemK;
}

void launch_stem_conv_wgrad(const void* dy, const void* xp, void* dw2, int N, int H, int W, int Cout, int variant, float* workspace,
                            cudaStream_t stream) {
  StemGeom g;
  if (!stem_geom(H, W, &g)) throw std::runtime_error("stem wgrad: unsupported geometry");
  CUtensorMap mdy, mx;
  uint32_t bx[4] = {64, (uint32_t)g.Wo, 1, 1};
  {
    uint64_t dd[4] = {(uint64_t)Cout, (uint64_t)g.Wo, (uint64_t)g.Ho, (uint64_t)N};
    uint64_t ds[3] = {(uint64_t)Cout * 2, (uint64_t)g.Wo * Cout * 2, (uint64_t)g.Ho * g.Wo * Cout * 2};
    mdy = encode_tensor_map(dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 4, dd, ds, bx);
  }
  {
    const uint64_t row_pitch = (uint64_t)g.Wp * 16;
    uint64_t xd[4] = {64, (uint64_t)g.Wo, (uint64_t)g.Hp2, (uint64_t)N};
    uint64_t xs[3] = {32, row_pitch, row_pitch * (uint64_t)g.Hp2};
    mx = encode_tensor_map(xp, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B, 4, xd, xs, bx);
  }
  const size_t n = (size_t)Cout * kStemK;
  int split = 0;
  if (variant == 1) {
    WgradPlan pl;
    if (!stem_generic_plan(N, H, W, Cout, &pl)) throw std::runtime_error("stem wgrad: unsupported geometry");
    pl.p.partial = workspace;
    launch_wgrad_kernel(mdy, mx, pl, stream);
    split = pl.p.split;
  } else {
    StemWgradParams p; int smem;
    if (!stem_dedicated_plan(N, H, W, Cout, &p, &smem)) throw std::runtime_error("stem wgrad: unsupported geometry");
    p.partial = workspace;
    static std::atomic<unsigned long long> configured{0};
    ensure_max_dynamic_smem(stem_wgrad_kernel, 227 * 1024, configured);
    stem_wgrad_kernel<<<p.split, kThreads, smem, stream>>>(mx, mdy, p);
    split = p.split;
  }
  B200_CUDA_CHECK(cudaGetLastError());
  conv_wgrad_reduce_kernel<<<(unsigned)((n / 8 + 31) / 32), 256, 0, stream>>>(workspace, reinterpret_cast<__nv_bfloat16*>(dw2), n, split);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

}  // namespace b200
