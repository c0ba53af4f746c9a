// Device-side building blocks for the peer-memory collectives: system-scope signal primitives,
// the block-wise cross-GPU barrier, multimem (NVLS) accessors and the bucket tensor table.
// (the transport the reference gets from ProcessGroupNCCL, `init_process_group("nccl")` at ddp.py:103.)
#pragma once
#include "common.h"
#include "peer_mem.h"

namespace b200 {

constexpr int kMaxBucketTensors = 192;      // keeps the whole launch argument block under 4 KB
// Comm CTAs are deliberately light (256 threads, <= 85 registers/thread -> a third of an SM's register
// file): they must slot in beside the CTAs of the backward kernels they overlap with instead of
// evicting them (a 512-thread / 118-register CTA monopolises an SM and turns persistent cuDNN kernels
// into two waves, which exposes the whole communication time).
constexpr int kCommThreads = 256;
constexpr int kCommMinCtasPerSm = 3;

// One gradient (or parameter) participating in a flat bucket.
struct TensorSlot {
  void* ptr;            // device pointer (nullptr = no gradient this iteration)
  uint32_t numel;       // elements
  uint32_t off;         // element offset of the slot in the flat bucket (multiple of 8)
};

struct BucketTable {
  int count;
  uint32_t data_elems;  // end of the padded data region == start of the "used" flags
  uint32_t total_elems; // data + flags, multiple of 8
  uint32_t _pad;
  TensorSlot t[kMaxBucketTensors];
};

// Signal-pad set: one per staging region (bucket / generic scratch).  All words start at 0.
//   ready [block][rank] : "rank's block has packed its staging for epoch e"
//   second[block][rank] : second rendezvous of the same launch (two-shot: results delivered)
//   done  [block][rank] : "rank's block no longer reads my staging of epoch e" (checked lazily by the NEXT launch)
//   epoch [block]       : local launch counter (device-resident, so a captured CUDA graph never bakes it)
struct PadSet {
  uint32_t ready[kMaxCommBlocks][kMaxRanks];
  uint32_t second[kMaxCommBlocks][kMaxRanks];
  uint32_t done[kMaxCommBlocks][kMaxRanks];
  uint32_t epoch[kMaxCommBlocks];
};
static_assert(sizeof(PadSet) <= kPadSetBytes, "pad set does not fit its slot");

struct CommCtx {
  char* base;           // VA of rank 0's arena; rank r at base + r*stride
  char* mc_base;        // multicast VA of the arena (nullptr if NVLS unavailable)
  size_t stride;
  size_t pad_off;       // byte offset of this communicator's PadSet inside the arena
  int* error_word;      // host-mapped; non-zero after a barrier timeout
  unsigned long long timeout_ns;
  int rank, world;
};

#ifdef __CUDACC__

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// One-way flags: the sender posts a monotonically increasing epoch with a release store straight into the
// receiver's memory (fire and forget - no round trip), the receiver polls its OWN memory with acquire loads.
__device__ __forceinline__ void st_release_sys(uint32_t* addr, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}

__device__ __forceinline__ PadSet* pad_of(const CommCtx& c, int rank) {
  return reinterpret_cast<PadSet*>(c.base + (size_t)rank * c.stride + c.pad_off);
}

// wait until *addr >= epoch (wrap-safe), bounded by the timeout
__device__ __forceinline__ bool wait_epoch(const uint32_t* addr, uint32_t epoch, const CommCtx& c, int code) {
  const unsigned long long t0 = globaltimer_ns();
  while ((int32_t)(ld_acquire_sys(addr) - epoch) < 0) {
    if (globaltimer_ns() - t0 > c.timeout_ns) { *c.error_word = code + c.rank; return false; }
  }
  return true;
}

// Every launch starts here: fetch + bump this block's epoch, then make sure every peer finished reading
// the staging region of the PREVIOUS launch on this pad set (it did long ago - this is off the critical path).
__device__ __forceinline__ uint32_t comm_begin(const CommCtx& c, uint32_t* smem_epoch) {
  PadSet* mine = pad_of(c, c.rank);
  if (threadIdx.x == 0) {
    const uint32_t e = mine->epoch[blockIdx.x] + 1;
    mine->epoch[blockIdx.x] = e;
    *smem_epoch = e;
  }
  __syncthreads();
  const uint32_t e = *smem_epoch;
  if ((int)threadIdx.x < c.world) wait_epoch(&mine->done[blockIdx.x][threadIdx.x], e - 1, c, 300);
  __syncthreads();
  return e;
}

enum : int { kFlagReady = 0, kFlagSecond = 1 };

// Rendezvous of block `blockIdx.x` of every rank.  Writes made by any thread of this block before the call
// are visible to the peer blocks after their call returns (bar.sync -> st.release.sys ... ld.acquire.sys -> bar.sync).
template <int WHICH>
__device__ __forceinline__ void peer_block_barrier(const CommCtx& c, uint32_t epoch) {
  __syncthreads();
  if ((int)threadIdx.x < c.world) {
    const int peer = threadIdx.x;
    PadSet* theirs = pad_of(c, peer);
    PadSet* mine = pad_of(c, c.rank);
    if (WHICH == kFlagReady) {
      st_release_sys(&theirs->ready[blockIdx.x][c.rank], epoch);
      wait_epoch(&mine->ready[blockIdx.x][peer], epoch, c, 100);
    } else {
      st_release_sys(&theirs->second[blockIdx.x][c.rank], epoch);
      wait_epoch(&mine->second[blockIdx.x][peer], epoch, c, 200);
    }
  }
  __syncthreads();
}

// "I will not read your staging of this epoch any more" - posted, never waited for in this launch.
__device__ __forceinline__ void comm_signal_done(const CommCtx& c, uint32_t epoch) {
  __syncthreads();
  if ((int)threadIdx.x < c.world) st_release_sys(&pad_of(c, threadIdx.x)->done[blockIdx.x][c.rank], epoch);
}

// ---- 16-byte accessors -----------------------------------------------------------------------
struct alignas(16) Vec16 { uint32_t w[4]; };

__device__ __forceinline__ Vec16 ld_sys(const void* p) {   // coherent load (peer memory)
  Vec16 v;
  asm volatile("ld.relaxed.sys.global.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_sys(void* p, const Vec16& v) {
  asm volatile("st.relaxed.sys.global.v4.b32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.w[0]), "r"(v.w[1]), "r"(v.w[2]), "r"(v.w[3]) : "memory");
}
__device__ __forceinline__ Vec16 ld_cg(const void* p) {    // local load, L1 bypass
  Vec16 v;
  asm volatile("ld.global.cg.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(p) : "memory");
  return v;
}

// NVLS: in-switch reduction of the same offset in every rank's arena, and broadcast store.
__device__ __forceinline__ Vec16 multimem_ld_reduce_bf16(const void* mc) {
  Vec16 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ Vec16 multimem_ld_reduce_f32(const void* mc) {
  Vec16 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3]) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st(void* mc, const Vec16& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "r"(v.w[0]), "r"(v.w[1]), "r"(v.w[2]), "r"(v.w[3]) : "memory");
}

// Wire-format traits: how many elements ride in one 16-byte vector.
template <typename WireT> struct Wire;
template <> struct Wire<__nv_bfloat16> {
  static constexpr int VE = 8;
  __device__ static void unpack(const Vec16& v, float* f) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&v.w[i]);
      float2 t = __bfloat1622float2(h);
      f[2 * i] = t.x; f[2 * i + 1] = t.y;
    }
  }
  __device__ static Vec16 pack(const float* f) {
    Vec16 v;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      v.w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return v;
  }
  __device__ static Vec16 mc_reduce(const void* mc) { return multimem_ld_reduce_bf16(mc); }
};
template <> struct Wire<float> {
  static constexpr int VE = 4;
  __device__ static void unpack(const Vec16& v, float* f) {
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = __uint_as_float(v.w[i]);
  }
  __device__ static Vec16 pack(const float* f) {
    Vec16 v;
#pragma unroll
    for (int i = 0; i < 4; ++i) v.w[i] = __float_as_uint(f[i]);
    return v;
  }
  __device__ static Vec16 mc_reduce(const void* mc) { return multimem_ld_reduce_f32(mc); }
};

// Which slot of the (shared-memory) offset array contains element e?  offs[count] == data_elems.
__device__ __forceinline__ int find_slot(const uint32_t* offs, int count, uint32_t e) {
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (offs[mid] <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

#endif  // __CUDACC__

}  // namespace b200
