// Rank-`src` -> everyone broadcast of a list of tensors through peer memory
// (replaces `_sync_module_states` -> ncclBroadcast + flatten/unflatten copies).
//
// One launch moves one chunk (<= staging size, <= kMaxBucketTensors tensors):
//   src rank : gather its tensors (bytes) into staging - its own arena, or, with NVLS, a
//              multimem.st that lands in every rank's arena at once
//   [peer barrier]
//   others   : pull 16-byte vectors from the source arena over NVLink (or read their local copy
//              after a multicast) and scatter straight into their own tensors - no flat temp
//   [peer barrier] so the next chunk may reuse the staging region
#include <cstdlib>
#include "comm_kernels.cuh"
#include "comm.h"

namespace b200 {

struct BcArgs {
  CommCtx ctx;
  size_t stage_off;
  int src_rank;
  int use_mc;
  BucketTable tab;   // numel/off are BYTES here
};

__global__ void __launch_bounds__(kCommThreads, kCommMinCtasPerSm) peer_broadcast_kernel(const __grid_constant__ BcArgs a) {
  __shared__ TensorSlot slots[kMaxBucketTensors];
  __shared__ uint32_t offs[kMaxBucketTensors + 1];
  const CommCtx& c = a.ctx;
  const int count = a.tab.count;
  if (a.src_rank < 0) return;                          // diagnostics (B200DDP_DEBUG_BCAST_NOOP): same node, no work
  for (int i = threadIdx.x; i < count; i += blockDim.x) { slots[i] = a.tab.t[i]; offs[i] = a.tab.t[i].off; }
  if (threadIdx.x == 0) offs[count] = a.tab.data_elems;
  __shared__ uint32_t s_epoch;
  const uint32_t epoch = comm_begin(c, &s_epoch);

  const uint32_t V = a.tab.total_elems / 16;   // 16-byte vectors
  const uint32_t step = gridDim.x * blockDim.x;
  const uint32_t first = blockIdx.x * blockDim.x + threadIdx.x;
  const bool is_src = c.rank == a.src_rank;

  if (is_src) {
    char* stage = (a.use_mc ? c.mc_base : c.base + (size_t)c.rank * c.stride) + a.stage_off;
    for (uint32_t v = first; v < V; v += step) {
      const uint32_t b0 = v * 16;
      const int k = find_slot(offs, count, b0);
      const uint32_t idx = b0 - offs[k];
      const uint32_t n = slots[k].numel;
      const char* src = reinterpret_cast<const char*>(slots[k].ptr) + idx;
      Vec16 x;
      if (idx + 16 <= n && (reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
        x = *reinterpret_cast<const Vec16*>(src);
      } else {
        unsigned char tmp[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) tmp[i] = (idx + i < n) ? (unsigned char)src[i] : 0;
        x = *reinterpret_cast<Vec16*>(tmp);
      }
      if (a.use_mc) multimem_st(stage + (size_t)v * 16, x);
      else *reinterpret_cast<Vec16*>(stage + (size_t)v * 16) = x;
    }
  }
  peer_block_barrier<kFlagReady>(c, epoch);
  if (!is_src) {
    const char* stage = c.base + (size_t)(a.use_mc ? c.rank : a.src_rank) * c.stride + a.stage_off;
    for (uint32_t v = first; v < V; v += step) {
      const uint32_t b0 = v * 16;
      const int k = find_slot(offs, count, b0);
      const uint32_t idx = b0 - offs[k];
      const uint32_t n = slots[k].numel;
      if (idx >= n) continue;
      const Vec16 x = a.use_mc ? ld_cg(stage + (size_t)v * 16) : ld_sys(stage + (size_t)v * 16);
      char* dst = reinterpret_cast<char*>(slots[k].ptr) + idx;
      if (idx + 16 <= n && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
        *reinterpret_cast<Vec16*>(dst) = x;
      } else {
        const unsigned char* tmp = reinterpret_cast<const unsigned char*>(&x);
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (idx + i < n) dst[i] = (char)tmp[i];
      }
    }
  }
  comm_signal_done(c, epoch);   // the next chunk may reuse the staging region once every peer has pulled
}

void launch_peer_broadcast(const CommCtx& ctx, const BucketTable& tab, size_t stage_off, int src_rank,
                           bool use_multicast, int blocks, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxCommBlocks) throw std::runtime_error("peer_broadcast: bad block count");
  if (tab.total_elems % 16 != 0) throw std::runtime_error("peer_broadcast: chunk not padded to 16 bytes");
  BcArgs args;
  args.ctx = ctx;
  args.stage_off = stage_off;
  static const bool noop = [] { const char* e = getenv("B200DDP_DEBUG_BCAST_NOOP"); return e && atoi(e) != 0; }();
  args.src_rank = noop ? -1 : src_rank;
  args.use_mc = (use_multicast && ctx.mc_base != nullptr) ? 1 : 0;
  args.tab = tab;
  peer_broadcast_kernel<<<blocks, kCommThreads, 0, stream>>>(args);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

// ---- link probes --------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCommThreads) peer_pull_kernel(const char* __restrict__ src, char* __restrict__ dst, size_t vecs) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  // 4 independent 16-byte requests in flight per thread
  for (; v + 3 * step < vecs; v += 4 * step) {
    Vec16 x0 = ld_sys(src + v * 16), x1 = ld_sys(src + (v + step) * 16), x2 = ld_sys(src + (v + 2 * step) * 16),
          x3 = ld_sys(src + (v + 3 * step) * 16);
    *reinterpret_cast<Vec16*>(dst + v * 16) = x0;
    *reinterpret_cast<Vec16*>(dst + (v + step) * 16) = x1;
    *reinterpret_cast<Vec16*>(dst + (v + 2 * step) * 16) = x2;
    *reinterpret_cast<Vec16*>(dst + (v + 3 * step) * 16) = x3;
  }
  for (; v < vecs; v += step) *reinterpret_cast<Vec16*>(dst + v * 16) = ld_sys(src + v * 16);
}

__global__ void __launch_bounds__(kCommThreads) peer_push_kernel(const char* __restrict__ src, char* __restrict__ dst, size_t vecs) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < vecs; v += step)
    st_sys(dst + v * 16, *reinterpret_cast<const Vec16*>(src + v * 16));
}

__global__ void __launch_bounds__(kCommThreads) peer_barrier_kernel(const __grid_constant__ CommCtx c) {
  __shared__ uint32_t s_epoch;
  const uint32_t epoch = comm_begin(c, &s_epoch);
  peer_block_barrier<kFlagReady>(c, epoch);
  comm_signal_done(c, epoch);
}

void launch_peer_pull(const CommCtx& ctx, int peer, size_t src_off, void* dst, size_t bytes, int blocks, cudaStream_t stream) {
  peer_pull_kernel<<<blocks, kCommThreads, 0, stream>>>(ctx.base + (size_t)peer * ctx.stride + src_off, (char*)dst, bytes / 16);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}
void launch_peer_push(const CommCtx& ctx, int peer, size_t dst_off, const void* src, size_t bytes, int blocks, cudaStream_t stream) {
  peer_push_kernel<<<blocks, kCommThreads, 0, stream>>>((const char*)src, ctx.base + (size_t)peer * ctx.stride + dst_off, bytes / 16);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}
void launch_peer_barrier(const CommCtx& ctx, int blocks, cudaStream_t stream) {
  peer_barrier_kernel<<<blocks, kCommThreads, 0, stream>>>(ctx);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
