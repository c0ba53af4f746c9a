// Mixture-of-experts routing, token permutation and combine (sm_90a).  The expert GEMMs themselves are the grouped mode of
// the wgmma GEMM (gemm_wgmma.cu); everything here is memory-bound and works one warp per token or per permuted row.
//
//   router   : top-k of each token's E logits (ties to the lower expert), softmax over the k chosen logits in fp32 rounded
//              to bf16 once, and optionally each expert's sum over tokens of the full softmax (the load-balancing loss),
//              reduced per 64-token block and then over blocks, both in a fixed order.
//   permute  : a stable counting sort of the T*k (token, slot) assignments by expert into segments that start at
//              multiples of 128, so that each 128-row tile of the permuted rows belongs to one expert.  Three launches
//              (per-chunk histograms, a single-block scan, a scatter that re-derives each assignment's rank with
//              __match_any_sync), no atomics, and every size follows from (T, E, k): nothing is read back to the host.
//   gather / combine : the permuted rows are gathered from the tokens, and each token's k expert outputs are gathered
//              back and summed in slot order; the backward passes are gathers as well, with one writer per element.
#include "ops.h"

#include <cmath>

namespace b200 {
namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kRouterTokensPerWarp = 8;
constexpr int kRouterTokens = kWarps * kRouterTokensPerWarp;   // tokens per router block (one partial row of the aux sums)
constexpr int kChunk = 1024;                                   // assignments per permutation block: 8 warps x 4 rounds of 32

__device__ __forceinline__ bool better(float v1, int i1, float v2, int i2) { return v1 > v2 || (v1 == v2 && i1 < i2); }

// Warp-wide best (value, expert) over every lane's candidate; every lane gets the result.
__device__ __forceinline__ void warp_best(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (better(ov, oi, v, i)) { v = ov; i = oi; }
  }
}

// Lane l holds the logits of experts l and l + 32 (-inf beyond E).  Returns the k chosen experts and their logits (in
// every lane), in descending order with ties to the lower expert.
__device__ __forceinline__ void top_k(float v0, float v1, int E, int k, int lane, int* sid, float* sel) {
  uint64_t taken = 0;
#pragma unroll
  for (int j = 0; j < kMoeMaxTopK; ++j) {
    if (j >= k) break;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    if (lane < E && !((taken >> lane) & 1)) { bv = v0; bi = lane; }
    if (lane + 32 < E && !((taken >> (lane + 32)) & 1) && better(v1, lane + 32, bv, bi)) { bv = v1; bi = lane + 32; }
    warp_best(bv, bi);
    sid[j] = bi;
    sel[j] = bv;
    taken |= 1ull << bi;
  }
}

__global__ void __launch_bounds__(kThreads) moe_router_fwd_kernel(const __nv_bfloat16* __restrict__ logits, int T, int E, int k,
                                                                  int* __restrict__ ids, __nv_bfloat16* __restrict__ gates,
                                                                  float* __restrict__ partial) {
  __shared__ float part[kWarps][kMoeMaxExperts];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc0 = 0.f, acc1 = 0.f;                                // this warp's full-softmax sums of experts lane, lane + 32
  for (int i = 0; i < kRouterTokensPerWarp; ++i) {
    const int t = blockIdx.x * kRouterTokens + warp * kRouterTokensPerWarp + i;
    if (t >= T) break;                                         // warp-uniform
    const __nv_bfloat16* row = logits + (size_t)t * E;
    const float v0 = lane < E ? __bfloat162float(row[lane]) : -INFINITY;
    const float v1 = lane + 32 < E ? __bfloat162float(row[lane + 32]) : -INFINITY;
    int sid[kMoeMaxTopK];
    float sel[kMoeMaxTopK];
    top_k(v0, v1, E, k, lane, sid, sel);
    const float m = sel[0];
    float s = 0.f, mine = 0.f;
    int my_id = 0;
#pragma unroll
    for (int j = 0; j < kMoeMaxTopK; ++j) {
      if (j >= k) break;
      const float ex = expf(sel[j] - m);
      s += ex;
      if (lane == j) { mine = ex; my_id = sid[j]; }
    }
    if (lane < k) {
      ids[(size_t)t * k + lane] = my_id;
      gates[(size_t)t * k + lane] = __float2bfloat16_rn(mine / s);
    }
    if (partial != nullptr) {
      const float e0 = lane < E ? expf(v0 - m) : 0.f, e1 = lane + 32 < E ? expf(v1 - m) : 0.f;
      const float z = warp_sum(e0 + e1);
      acc0 += e0 / z;
      acc1 += e1 / z;
    }
  }
  if (partial == nullptr) return;
  part[warp][lane] = acc0;
  part[warp][lane + 32] = acc1;
  __syncthreads();
  if (threadIdx.x < E) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) s += part[w][threadIdx.x];
    partial[(size_t)blockIdx.x * E + threadIdx.x] = s;
  }
}

__global__ void moe_probsum_kernel(const float* __restrict__ partial, int blocks, int E, float* __restrict__ probsum) {
  const int e = threadIdx.x;
  if (e >= E) return;
  float s = 0.f;
  for (int b = 0; b < blocks; ++b) s += partial[(size_t)b * E + e];
  probsum[e] = s;
}

__global__ void __launch_bounds__(kThreads) moe_router_bwd_kernel(const __nv_bfloat16* __restrict__ logits, int T, int E, int k,
                                                                  const int* __restrict__ ids, const float* __restrict__ dgates,
                                                                  const float* __restrict__ dprobsum, __nv_bfloat16* __restrict__ dlogits) {
  const int lane = threadIdx.x & 31;
  const float dp0 = dprobsum != nullptr && lane < E ? __ldg(dprobsum + lane) : 0.f;
  const float dp1 = dprobsum != nullptr && lane + 32 < E ? __ldg(dprobsum + lane + 32) : 0.f;
  for (int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < T; t += (gridDim.x * blockDim.x) >> 5) {
    const __nv_bfloat16* row = logits + (size_t)t * E;
    const float v0 = lane < E ? __bfloat162float(row[lane]) : -INFINITY;
    const float v1 = lane + 32 < E ? __bfloat162float(row[lane + 32]) : -INFINITY;
    const int my_id = lane < k ? __ldg(ids + (size_t)t * k + lane) : 0;
    const float my_dg = lane < k ? __ldg(dgates + (size_t)t * k + lane) : 0.f;
    // the chosen logits, by shuffling from the lane that holds each
    const float s0 = __shfl_sync(0xffffffffu, v0, my_id & 31), s1 = __shfl_sync(0xffffffffu, v1, my_id & 31);
    const float my_sel = (my_id & 32) ? s1 : s0;
    const float m = warp_max(lane < k ? my_sel : -INFINITY);
    const float ex = lane < k ? expf(my_sel - m) : 0.f;
    const float g = ex / warp_sum(ex);                         // fp32 gate of slot `lane` (lanes >= k: 0)
    const float dot = warp_sum(g * my_dg);
    const float dsel = g * (my_dg - dot);                      // d logit of expert my_id through the top-k softmax
    float d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int j = 0; j < kMoeMaxTopK; ++j) {
      if (j >= k) break;
      const int id = __shfl_sync(0xffffffffu, my_id, j);
      const float dj = __shfl_sync(0xffffffffu, dsel, j);
      if (id == lane) d0 += dj;
      if (id == lane + 32) d1 += dj;
    }
    if (dprobsum != nullptr) {
      const float mm = warp_max(fmaxf(v0, v1));
      const float e0 = lane < E ? expf(v0 - mm) : 0.f, e1 = lane + 32 < E ? expf(v1 - mm) : 0.f;
      const float z = warp_sum(e0 + e1);
      const float p0 = e0 / z, p1 = e1 / z;
      const float pdot = warp_sum(p0 * dp0 + p1 * dp1);
      d0 += p0 * (dp0 - pdot);
      d1 += p1 * (dp1 - pdot);
    }
    __nv_bfloat16* out = dlogits + (size_t)t * E;
    if (lane < E) out[lane] = __float2bfloat16_rn(d0);
    if (lane + 32 < E) out[lane + 32] = __float2bfloat16_rn(d1);
  }
}

// Per-warp expert histogram of a chunk's assignments into hist[warp][*] (zeroed by the caller).  Round r of warp w covers
// assignments chunk * 1024 + w * 128 + r * 32 + lane; in each round the lowest lane of every group of equal ids adds the
// group's size, so each counter has one writer per round.
__device__ __forceinline__ void chunk_histogram(const int* __restrict__ ids, int n, int chunk, int warp, int lane, int (*hist)[kMoeMaxExperts]) {
#pragma unroll
  for (int r = 0; r < kChunk / kThreads; ++r) {
    const int a = chunk * kChunk + warp * (kChunk / kWarps) + r * 32 + lane;
    const int id = a < n ? __ldg(ids + a) : -1;
    const unsigned match = __match_any_sync(0xffffffffu, id);
    if (id >= 0 && (__ffs(match) - 1) == lane) hist[warp][id] += __popc(match);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kThreads) moe_count_kernel(const int* __restrict__ ids, int n, int E, int* __restrict__ chunk_counts) {
  __shared__ int hist[kWarps][kMoeMaxExperts];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kWarps * kMoeMaxExperts; i += kThreads) (&hist[0][0])[i] = 0;
  __syncthreads();
  chunk_histogram(ids, n, blockIdx.x, warp, lane, hist);
  __syncthreads();
  if (threadIdx.x < E) {
    int c = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) c += hist[w][threadIdx.x];
    chunk_counts[(size_t)blockIdx.x * E + threadIdx.x] = c;
  }
}

// One block of 128 threads (at least E + 1): each expert's total and its rows' start in every chunk (chunk_base = the expert's padded offset + the rows of
// earlier chunks), the padded offsets and the tile table.
__global__ void __launch_bounds__(2 * kMoeMaxExperts) moe_offsets_kernel(const int* __restrict__ chunk_counts, int chunks, int E, int tiles,
                                                                     int* __restrict__ chunk_base, int* __restrict__ counts,
                                                                     int* __restrict__ offsets, int* __restrict__ tile_expert) {
  __shared__ int off[kMoeMaxExperts + 1];
  const int e = threadIdx.x;
  int total = 0;
  if (e < E) {
    for (int c = 0; c < chunks; ++c) {
      chunk_base[(size_t)c * E + e] = total;
      total += chunk_counts[(size_t)c * E + e];
    }
    counts[e] = total;
    off[e + 1] = (total + kMoeAlign - 1) / kMoeAlign * kMoeAlign;
  }
  __syncthreads();
  if (e == 0) {
    off[0] = 0;
    for (int i = 1; i <= E; ++i) off[i] += off[i - 1];
  }
  __syncthreads();
  if (e <= E) offsets[e] = off[e];
  if (e < E)
    for (int c = 0; c < chunks; ++c) chunk_base[(size_t)c * E + e] += off[e];
  for (int i = e; i < tiles; i += blockDim.x) {
    const int r = i * kMoeAlign;
    int owner = -1;
    for (int x = 0; x < E; ++x)
      if (off[x] <= r && r < off[x + 1]) owner = x;
    tile_expert[i] = owner;
  }
}

__global__ void __launch_bounds__(kThreads) moe_scatter_kernel(const int* __restrict__ ids, int n, int E, const int* __restrict__ chunk_base,
                                                               int* __restrict__ fwd_map, int* __restrict__ inv_map) {
  __shared__ int hist[kWarps][kMoeMaxExperts];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kWarps * kMoeMaxExperts; i += kThreads) (&hist[0][0])[i] = 0;
  __syncthreads();
  chunk_histogram(ids, n, blockIdx.x, warp, lane, hist);
  __syncthreads();
  if (threadIdx.x < E) {                                       // hist[w][e] <- first row of warp w's expert-e assignments
    int run = chunk_base[(size_t)blockIdx.x * E + threadIdx.x];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const int c = hist[w][threadIdx.x];
      hist[w][threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < kChunk / kThreads; ++r) {
    const int a = blockIdx.x * kChunk + warp * (kChunk / kWarps) + r * 32 + lane;
    const int id = a < n ? __ldg(ids + a) : -1;
    const unsigned match = __match_any_sync(0xffffffffu, id);
    const int row = id >= 0 ? hist[warp][id] + __popc(match & lt) : 0;
    __syncwarp();
    if (id >= 0) {
      fwd_map[row] = a;
      inv_map[a] = row;
      if ((__ffs(match) - 1) == lane) hist[warp][id] += __popc(match);
    }
    __syncwarp();
  }
}

int warp_grid(long long items) {
  const long long b = (items + kWarps - 1) / kWarps;
  return (int)(b < 1 ? 1 : (b > 16LL * kNumSMs ? 16LL * kNumSMs : b));
}

__global__ void __launch_bounds__(kThreads) moe_gather_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ fwd_map, int rows,
                                                              int H, int k, __nv_bfloat16* __restrict__ x_perm) {
  const int lane = threadIdx.x & 31, vecs = H / 8;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
    const int a = __ldg(fwd_map + r);
    Bf16x8* out = reinterpret_cast<Bf16x8*>(x_perm + (size_t)r * H);
    if (a < 0) {
      const Bf16x8 z = {};
      for (int v = lane; v < vecs; v += 32) out[v] = z;
    } else {
      const Bf16x8* in = reinterpret_cast<const Bf16x8*>(x + (size_t)(a / k) * H);
      for (int v = lane; v < vecs; v += 32) out[v] = in[v];
    }
  }
}

__global__ void __launch_bounds__(kThreads) moe_combine_kernel(const __nv_bfloat16* __restrict__ y_perm, const int* __restrict__ inv_map,
                                                               const __nv_bfloat16* __restrict__ gates, int T, int H, int k,
                                                               __nv_bfloat16* __restrict__ out) {
  const int lane = threadIdx.x & 31, vecs = H / 8;
  for (int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < T; t += (gridDim.x * blockDim.x) >> 5) {
    for (int v = lane; v < vecs; v += 32) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < k; ++j) {
        const int row = __ldg(inv_map + (size_t)t * k + j);
        const float g = gates != nullptr ? __bfloat162float(gates[(size_t)t * k + j]) : 1.f;
        float y[8];
        unpack8(reinterpret_cast<const Bf16x8*>(y_perm + (size_t)row * H)[v], y);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += g * y[i];
      }
      reinterpret_cast<Bf16x8*>(out + (size_t)t * H)[v] = pack8(acc);
    }
  }
}

__global__ void __launch_bounds__(kThreads) moe_combine_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ y_perm,
                                                                   const int* __restrict__ fwd_map, const __nv_bfloat16* __restrict__ gates,
                                                                   int rows, int H, int k, __nv_bfloat16* __restrict__ dy_perm,
                                                                   float* __restrict__ dgates) {
  const int lane = threadIdx.x & 31, vecs = H / 8;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
    const int a = __ldg(fwd_map + r);
    Bf16x8* out = reinterpret_cast<Bf16x8*>(dy_perm + (size_t)r * H);
    if (a < 0) {
      const Bf16x8 z = {};
      for (int v = lane; v < vecs; v += 32) out[v] = z;
      continue;
    }
    const float g = __bfloat162float(gates[a]);
    const Bf16x8* d_in = reinterpret_cast<const Bf16x8*>(dout + (size_t)(a / k) * H);
    const Bf16x8* y_in = reinterpret_cast<const Bf16x8*>(y_perm + (size_t)r * H);
    float dot = 0.f;
    for (int v = lane; v < vecs; v += 32) {
      float d[8], y[8], o[8];
      unpack8(d_in[v], d);
      unpack8(y_in[v], y);
#pragma unroll
      for (int i = 0; i < 8; ++i) { o[i] = g * d[i]; dot += d[i] * y[i]; }
      out[v] = pack8(o);
    }
    dot = warp_sum(dot);
    if (lane == 0) dgates[a] = dot;
  }
}

void moe_check(int T, int E, int k) {
  if (T < 1 || E < 1 || E > kMoeMaxExperts || k < 1 || k > kMoeMaxTopK || k > E)
    throw std::runtime_error("moe: needs T >= 1, 1 <= E <= 64 and 1 <= k <= min(E, 8), got T=" + std::to_string(T) + " E=" +
                             std::to_string(E) + " k=" + std::to_string(k));
}

void hidden_check(int H, const void* a, const void* b) {
  if (H < 64 || H % 64 != 0 || ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15u) != 0)
    throw std::runtime_error("moe: needs the hidden size a positive multiple of 64 and 16-byte aligned rows, got H=" + std::to_string(H));
}

}  // namespace

void launch_moe_router_fwd(const void* logits, int T, int E, int k, int* ids, void* gates, float* partial, float* probsum, cudaStream_t s) {
  moe_check(T, E, k);
  const int blocks = ceil_div(T, kRouterTokens);
  moe_router_fwd_kernel<<<blocks, kThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(logits), T, E, k, ids,
                                                    reinterpret_cast<__nv_bfloat16*>(gates), probsum != nullptr ? partial : nullptr);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  if (probsum != nullptr) {
    moe_probsum_kernel<<<1, kMoeMaxExperts, 0, s>>>(partial, blocks, E, probsum);
    B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  }
}

void launch_moe_router_bwd(const void* logits, int T, int E, int k, const int* ids, const float* dgates, const float* dprobsum,
                           void* dlogits, cudaStream_t s) {
  moe_check(T, E, k);
  moe_router_bwd_kernel<<<warp_grid(T), kThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(logits), T, E, k, ids, dgates, dprobsum,
                                                          reinterpret_cast<__nv_bfloat16*>(dlogits));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_moe_permute(const int* ids, int T, int E, int k, int* chunk_counts, int* counts, int* offsets, int* fwd_map, int* inv_map,
                        int* tile_expert, cudaStream_t s) {
  moe_check(T, E, k);
  const int n = T * k, chunks = moe_chunks(T, k), capacity = moe_capacity(T, E, k);
  int* chunk_base = chunk_counts + (size_t)chunks * E;
  B200_CUDA_CHECK(cudaMemsetAsync(fwd_map, 0xff, (size_t)capacity * sizeof(int), s));   // -1: padding rows
  moe_count_kernel<<<chunks, kThreads, 0, s>>>(ids, n, E, chunk_counts);
  B200_CUDA_CHECK(cudaGetLastError());
  moe_offsets_kernel<<<1, 2 * kMoeMaxExperts, 0, s>>>(chunk_counts, chunks, E, capacity / kMoeAlign, chunk_base, counts, offsets, tile_expert);
  B200_CUDA_CHECK(cudaGetLastError());
  moe_scatter_kernel<<<chunks, kThreads, 0, s>>>(ids, n, E, chunk_base, fwd_map, inv_map);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(3);
}

void launch_moe_gather(const void* x, const int* fwd_map, int capacity, int H, int k, void* x_perm, cudaStream_t s) {
  hidden_check(H, x, x_perm);
  moe_gather_kernel<<<warp_grid(capacity), kThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), fwd_map, capacity, H, k,
                                                             reinterpret_cast<__nv_bfloat16*>(x_perm));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_moe_combine(const void* y_perm, const int* inv_map, const void* gates, int T, int H, int k, void* out, cudaStream_t s) {
  hidden_check(H, y_perm, out);
  moe_combine_kernel<<<warp_grid(T), kThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(y_perm), inv_map,
                                                       reinterpret_cast<const __nv_bfloat16*>(gates), T, H, k,
                                                       reinterpret_cast<__nv_bfloat16*>(out));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_moe_combine_bwd(const void* dout, const void* y_perm, const int* fwd_map, const void* gates, int capacity, int H, int k,
                            void* dy_perm, float* dgates, cudaStream_t s) {
  hidden_check(H, dout, y_perm);
  hidden_check(H, dy_perm, dy_perm);
  moe_combine_bwd_kernel<<<warp_grid(capacity), kThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dout),
                                                                  reinterpret_cast<const __nv_bfloat16*>(y_perm), fwd_map,
                                                                  reinterpret_cast<const __nv_bfloat16*>(gates), capacity, H, k,
                                                                  reinterpret_cast<__nv_bfloat16*>(dy_perm), dgates);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
