// Fused gradient-bucket allreduce over NVSwitch peer memory (replaces NCCL's allreduce on the DDP hot path).
//
// ONE launch per bucket does, tile by tile:
//   gather (flatten scattered .grad tensors) -> x scale (1/world) -> cast to wire dtype -> local
//   symmetric staging -> [peer barrier] -> reduce-scatter (P2P loads from every peer, fp32
//   accumulate; or multimem.ld_reduce in the switch) -> all-gather (P2P stores to every peer; or
//   multimem.st) -> [peer barrier] -> cast back -> scatter into .grad / the flat bucket view,
//   + per-block sum of squares (for clip_grad_norm) + the reduced "parameter used" flags.
// No NCCL call and no separate elementwise kernel exists on this path.
//
// Work ownership is block-local across all phases (block b of every rank touches the same vector
// set), so only block<->block barriers between GPUs are needed, never a grid-wide one.
#include "comm_kernels.cuh"
#include "comm.h"

namespace b200 {

struct ArArgs {
  CommCtx ctx;
  size_t stage_off;     // byte offset (in every arena) of this bucket's wire staging region
  void* flat_out;       // flat bucket in grad dtype (gradient_as_bucket_view) or nullptr
  float* sq_partials;   // [gridDim.x] or nullptr
  float* flags_out;     // [count] host-mapped, or nullptr
  float scale;
  int scatter;          // write reduced values back into each tensor's own storage
  int direct;           // the staging region IS the (symmetric) user buffer: no pack / unpack phases
  BucketTable tab;
};

template <typename InT, int VE>
__device__ __forceinline__ void gather_vec(const TensorSlot* slots, const uint32_t* offs, int count,
                                           uint32_t data_elems, uint32_t e0, float scale, float* f, int& hint) {
  if (e0 >= data_elems) {  // "used" flags ride behind the data
#pragma unroll
    for (int i = 0; i < VE; ++i) {
      const uint32_t k = e0 - data_elems + i;
      f[i] = (k < (uint32_t)count && slots[k].ptr != nullptr) ? 1.f : 0.f;
    }
    return;
  }
  int k = hint;
  if (!(offs[k] <= e0 && e0 < offs[k + 1])) k = find_slot(offs, count, e0);
  hint = k;
  const uint32_t idx = e0 - offs[k];
  const uint32_t n = slots[k].numel;
  const InT* src = reinterpret_cast<const InT*>(slots[k].ptr);
  if (src == nullptr || idx >= n) {
#pragma unroll
    for (int i = 0; i < VE; ++i) f[i] = 0.f;
    return;
  }
  src += idx;
  if (idx + VE <= n && (reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
    if constexpr (sizeof(InT) == 4) {
#pragma unroll
      for (int q = 0; q < VE / 4; ++q) {
        float4 t = __ldg(reinterpret_cast<const float4*>(src) + q);
        f[4 * q] = t.x * scale; f[4 * q + 1] = t.y * scale; f[4 * q + 2] = t.z * scale; f[4 * q + 3] = t.w * scale;
      }
    } else {
      if constexpr (VE == 8) {
        uint4 raw = __ldg(reinterpret_cast<const uint4*>(src));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int q = 0; q < 4; ++q) { float2 t = __bfloat1622float2(h[q]); f[2 * q] = t.x * scale; f[2 * q + 1] = t.y * scale; }
      } else {
        uint2 raw = __ldg(reinterpret_cast<const uint2*>(src));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int q = 0; q < 2; ++q) { float2 t = __bfloat1622float2(h[q]); f[2 * q] = t.x * scale; f[2 * q + 1] = t.y * scale; }
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < VE; ++i) f[i] = (idx + i < n) ? to_f32<InT>(src[i]) * scale : 0.f;
  }
}

template <typename InT, int VE>
__device__ __forceinline__ float deliver_vec(const ArArgs& a, const TensorSlot* slots, const uint32_t* offs,
                                             uint32_t e0, const float* f, int& hint) {
  const int count = a.tab.count;
  if (e0 >= a.tab.data_elems) {
    if (a.flags_out != nullptr) {
#pragma unroll
      for (int i = 0; i < VE; ++i) {
        const uint32_t k = e0 - a.tab.data_elems + i;
        if (k < (uint32_t)count) a.flags_out[k] = f[i];
      }
    }
    return 0.f;
  }
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VE; ++i) sq += f[i] * f[i];
  if (a.flat_out != nullptr) {
    InT* dst = reinterpret_cast<InT*>(a.flat_out) + e0;   // slots are 8-element aligned: always vectorisable
    if constexpr (sizeof(InT) == 4) {
#pragma unroll
      for (int q = 0; q < VE / 4; ++q)
        reinterpret_cast<float4*>(dst)[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
    } else {
      __nv_bfloat162 h[VE / 2];
#pragma unroll
      for (int q = 0; q < VE / 2; ++q) h[q] = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
      if constexpr (VE == 8) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<uint4*>(h);
      else *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<uint2*>(h);
    }
  }
  if (a.scatter) {
    int k = hint;
    if (!(offs[k] <= e0 && e0 < offs[k + 1])) k = find_slot(offs, count, e0);
    hint = k;
    const uint32_t idx = e0 - offs[k];
    const uint32_t n = slots[k].numel;
    InT* dst = reinterpret_cast<InT*>(slots[k].ptr);
    if (dst != nullptr && idx < n) {
      dst += idx;
      if (idx + VE <= n && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
        if constexpr (sizeof(InT) == 4) {
#pragma unroll
          for (int q = 0; q < VE / 4; ++q)
            reinterpret_cast<float4*>(dst)[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
        } else {
          __nv_bfloat162 h[VE / 2];
#pragma unroll
          for (int q = 0; q < VE / 2; ++q) h[q] = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
          if constexpr (VE == 8) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<uint4*>(h);
          else *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<uint2*>(h);
        }
      } else {
#pragma unroll
        for (int i = 0; i < VE; ++i)
          if (idx + i < n) dst[i] = from_f32<InT>(f[i]);
      }
    }
  }
  return sq;
}


// Sum the same 16-byte vector over all ranks' staging regions (P2P loads).  PW = compile-time rank count so that
// 8 / PW vectors x PW peers = 8 independent 16-byte NVLink requests are in flight per thread whatever the world size.
template <typename W, int PW, int UV>
__device__ __forceinline__ void pull_and_sum(const CommCtx& c, size_t stage_off, const uint32_t* v_idx, const bool* valid,
                                             float (*acc)[W::VE]) {
  Vec16 x[UV][PW];
#pragma unroll
  for (int u = 0; u < UV; ++u)
#pragma unroll
    for (int p = 0; p < PW; ++p)
      if (valid[u] && p < c.world) x[u][p] = ld_sys(c.base + (size_t)p * c.stride + stage_off + (size_t)v_idx[u] * 16);
#pragma unroll
  for (int u = 0; u < UV; ++u) {
#pragma unroll
    for (int i = 0; i < W::VE; ++i) acc[u][i] = 0.f;
    if (!valid[u]) continue;
#pragma unroll
    for (int p = 0; p < PW; ++p)
      if (p < c.world) {
        float f[W::VE];
        W::unpack(x[u][p], f);
#pragma unroll
        for (int i = 0; i < W::VE; ++i) acc[u][i] += f[i];
      }
  }
}

template <typename InT, typename W, int PW>
__device__ __forceinline__ float one_shot_body(const ArArgs& a, const TensorSlot* slots, const uint32_t* offs, uint32_t V,
                                               uint32_t first, uint32_t step) {
  constexpr int UV = 8 / PW, VE = W::VE;
  const CommCtx& c = a.ctx;
  float sq = 0.f;
  int hint = 0;
  for (uint32_t v = first; v < V; v += UV * step) {
    uint32_t idx[UV];
    bool valid[UV];
    float acc[UV][VE];
#pragma unroll
    for (int u = 0; u < UV; ++u) { idx[u] = v + u * step; valid[u] = idx[u] < V; }
    pull_and_sum<W, PW, UV>(c, a.stage_off, idx, valid, acc);
#pragma unroll
    for (int u = 0; u < UV; ++u) {
      if (!valid[u]) continue;
      // round through the wire format so every algorithm yields the same values
      Vec16 packed = W::pack(acc[u]);
      W::unpack(packed, acc[u]);
      sq += deliver_vec<InT, VE>(a, slots, offs, idx[u] * VE, acc[u], hint);
    }
  }
  return sq;
}

template <typename W, int PW>
__device__ __forceinline__ void two_shot_exchange_body(const ArArgs& a, uint32_t base_v, uint32_t lim, uint32_t first, uint32_t step) {
  constexpr int UV = 8 / PW, VE = W::VE;
  const CommCtx& c = a.ctx;
  for (uint32_t j = first; j < lim; j += UV * step) {
    uint32_t idx[UV];
    bool valid[UV];
    float acc[UV][VE];
#pragma unroll
    for (int u = 0; u < UV; ++u) { valid[u] = j + u * step < lim; idx[u] = base_v + j + u * step; }
    pull_and_sum<W, PW, UV>(c, a.stage_off, idx, valid, acc);
#pragma unroll
    for (int u = 0; u < UV; ++u) {
      if (!valid[u]) continue;
      if (a.direct && a.scale != 1.f) {
#pragma unroll
        for (int i = 0; i < VE; ++i) acc[u][i] *= a.scale;
      }
      const Vec16 out = W::pack(acc[u]);
      const size_t byte_off = a.stage_off + (size_t)idx[u] * 16;
#pragma unroll
      for (int p = 0; p < PW; ++p)
        if (p < c.world) st_sys(c.base + (size_t)p * c.stride + byte_off, out);
    }
  }
}

template <typename InT, typename WireT, int ALGO>
__global__ void __launch_bounds__(kCommThreads, kCommMinCtasPerSm) bucket_allreduce_kernel(const __grid_constant__ ArArgs a) {
  using W = Wire<WireT>;
  constexpr int VE = W::VE;
  __shared__ TensorSlot slots[kMaxBucketTensors];
  __shared__ uint32_t offs[kMaxBucketTensors + 1];
  __shared__ float red[33];
  __shared__ uint32_t s_epoch;

  const CommCtx& c = a.ctx;
  const int P = c.world, r = c.rank, count = a.tab.count;
  for (int i = threadIdx.x; i < count; i += blockDim.x) { slots[i] = a.tab.t[i]; offs[i] = a.tab.t[i].off; }
  if (threadIdx.x == 0) offs[count] = a.tab.data_elems;
  const uint32_t epoch = comm_begin(c, &s_epoch);   // also the __syncthreads that publishes slots/offs

  const uint32_t V = a.tab.total_elems / VE;
  const uint32_t Vs = (V + P - 1) / P;
  const uint32_t step = gridDim.x * blockDim.x;
  const uint32_t first = blockIdx.x * blockDim.x + threadIdx.x;
  char* const my_stage = c.base + (size_t)r * c.stride + a.stage_off;
  float sq = 0.f;
  int hint = 0;
  constexpr int U = (sizeof(InT) == 4 && VE == 8) ? 2 : 4;    // independent vector requests in flight per thread and trip

  // ---- phase 1: gather + scale + cast into local symmetric staging.
  // Block ownership of a vector must be identical in every phase (the only cross-GPU synchronisation is block b <-> block b):
  // the two-shot algorithms index every phase as slice_base + first + m * step, so they pack slice by slice; the one-shot
  // algorithms read flat (first + m * step over [0, V)), so they pack flat too.
  constexpr bool kFlat = (ALGO == kAlgoOneShot || ALGO == kAlgoNvlsOneShot);
  const int pack_slices = a.direct ? 0 : (kFlat ? 1 : P);
  for (int s = 0; s < pack_slices; ++s) {
    const uint32_t base_v = kFlat ? 0u : (uint32_t)s * Vs;
    const uint32_t lim = kFlat ? V : min(Vs, V > base_v ? V - base_v : 0u);     // vectors of this slice that exist
    for (uint32_t j = first; j < lim; j += U * step) {
      float f[U][VE];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t jj = j + u * step;
        if (jj < lim) gather_vec<InT, VE>(slots, offs, count, a.tab.data_elems, (base_v + jj) * VE, a.scale, f[u], hint);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t jj = j + u * step;
        if (jj < lim) *reinterpret_cast<Vec16*>(my_stage + (size_t)(base_v + jj) * 16) = W::pack(f[u]);
      }
    }
  }
  peer_block_barrier<kFlagReady>(c, epoch);

  if constexpr (ALGO == kAlgoNvlsOneShot) {
    // ---- every rank lets the switch reduce the whole bucket for it: one multimem.ld_reduce per vector,
    //      no second exchange phase (lowest latency for small buckets)
    hint = 0;
    for (uint32_t v = first; v < V; v += U * step) {
      Vec16 x[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (v + u * step < V) x[u] = W::mc_reduce(c.mc_base + a.stage_off + (size_t)(v + u * step) * 16);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (v + u * step >= V) continue;
        float f[VE];
        W::unpack(x[u], f);
        sq += deliver_vec<InT, VE>(a, slots, offs, (v + u * step) * VE, f, hint);
      }
    }
  } else if constexpr (ALGO == kAlgoOneShot) {
    // ---- every rank pulls every vector from every peer and reduces locally
    if (P <= 2) sq += one_shot_body<InT, W, 2>(a, slots, offs, V, first, step);
    else if (P <= 4) sq += one_shot_body<InT, W, 4>(a, slots, offs, V, first, step);
    else sq += one_shot_body<InT, W, 8>(a, slots, offs, V, first, step);
  } else {
    // ---- phase 2: reduce-scatter my slice, then all-gather it to every peer
    const uint32_t base_v = (uint32_t)r * Vs;
    const uint32_t lim = min(Vs, V > base_v ? V - base_v : 0u);
    if constexpr (ALGO == kAlgoNvls) {
      for (uint32_t j = first; j < lim; j += U * step) {
        Vec16 red16[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (j + u * step < lim) red16[u] = W::mc_reduce(c.mc_base + a.stage_off + (size_t)(base_v + j + u * step) * 16);
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (j + u * step < lim) {
            if (a.direct && a.scale != 1.f) {       // in-place symmetric mode: the scale was not applied by a pack phase
              float f[VE];
              W::unpack(red16[u], f);
#pragma unroll
              for (int i = 0; i < VE; ++i) f[i] *= a.scale;
              red16[u] = W::pack(f);
            }
            multimem_st(c.mc_base + a.stage_off + (size_t)(base_v + j + u * step) * 16, red16[u]);
          }
      }
    } else {
      if (P <= 2) two_shot_exchange_body<W, 2>(a, base_v, lim, first, step);
      else if (P <= 4) two_shot_exchange_body<W, 4>(a, base_v, lim, first, step);
      else two_shot_exchange_body<W, 8>(a, base_v, lim, first, step);
    }
    peer_block_barrier<kFlagSecond>(c, epoch);
    // ---- phase 3: cast back + scatter from local staging
    hint = 0;
    for (int s = 0; s < (a.direct ? 0 : P); ++s) {
      const uint32_t bv = (uint32_t)s * Vs;
      const uint32_t ls = min(Vs, V > bv ? V - bv : 0u);
      for (uint32_t j = first; j < ls; j += U * step) {
        Vec16 x[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (j + u * step < ls) x[u] = ld_cg(my_stage + (size_t)(bv + j + u * step) * 16);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (j + u * step >= ls) continue;
          float f[VE];
          W::unpack(x[u], f);
          sq += deliver_vec<InT, VE>(a, slots, offs, (bv + j + u * step) * VE, f, hint);
        }
      }
    }
  }

  // tell every peer this block is finished with their staging; the NEXT launch on this pad set checks it
  comm_signal_done(c, epoch);

  if (a.sq_partials != nullptr) {
    const float total = block_sum(sq, red);
    if (threadIdx.x == 0) a.sq_partials[blockIdx.x] = total;
  }
}

template <typename InT, typename WireT>
static void launch_typed(const ArArgs& args, int algo, int blocks, cudaStream_t stream) {
  switch (algo) {
    case kAlgoOneShot: bucket_allreduce_kernel<InT, WireT, kAlgoOneShot><<<blocks, kCommThreads, 0, stream>>>(args); break;
    case kAlgoTwoShot: bucket_allreduce_kernel<InT, WireT, kAlgoTwoShot><<<blocks, kCommThreads, 0, stream>>>(args); break;
    case kAlgoNvls:    bucket_allreduce_kernel<InT, WireT, kAlgoNvls><<<blocks, kCommThreads, 0, stream>>>(args); break;
    case kAlgoNvlsOneShot: bucket_allreduce_kernel<InT, WireT, kAlgoNvlsOneShot><<<blocks, kCommThreads, 0, stream>>>(args); break;
    default: throw std::runtime_error("bucket_allreduce: unknown algorithm");
  }
}

void launch_symmetric_allreduce(const CommCtx& ctx, size_t buf_off, size_t numel, DType dtype, int algo, int blocks, float scale,
                                cudaStream_t stream) {
  if (algo != kAlgoTwoShot && algo != kAlgoNvls) throw std::runtime_error("symmetric allreduce: two_shot or nvls");
  const size_t ve = dtype == DType::BF16 ? 8 : 4;
  if (numel % ve != 0 || buf_off % 16 != 0) throw std::runtime_error("symmetric allreduce: buffer must be 16-byte granular");
  if (numel > 0xFFFFFFF0ull) throw std::runtime_error("symmetric allreduce: more than 2^32 elements in one call (element offsets are 32-bit)");
  if (blocks < 1 || blocks > kMaxCommBlocks) throw std::runtime_error("symmetric allreduce: bad block count");
  if (algo == kAlgoNvls && ctx.mc_base == nullptr) throw std::runtime_error("symmetric allreduce: NVLS requested without multicast");
  BucketTable tab;
  tab.count = 0;
  tab.data_elems = (uint32_t)numel;
  tab.total_elems = (uint32_t)numel;
  tab._pad = 0;
  ArArgs args;
  args.ctx = ctx;
  args.stage_off = buf_off;
  args.flat_out = nullptr;
  args.sq_partials = nullptr;
  args.flags_out = nullptr;
  args.scale = scale;
  args.scatter = 0;
  args.direct = 1;
  args.tab = tab;
  if (dtype == DType::BF16) launch_typed<__nv_bfloat16, __nv_bfloat16>(args, algo, blocks, stream);
  else if (dtype == DType::F32) launch_typed<float, float>(args, algo, blocks, stream);
  else throw std::runtime_error("symmetric allreduce: fp32 or bf16");
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_bucket_allreduce(const CommCtx& ctx, const BucketTable& tab, size_t stage_off, DType in_dtype,
                             DType wire_dtype, int algo, int blocks, void* flat_out, float* sq_partials,
                             float* flags_out, float scale, bool scatter, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxCommBlocks) throw std::runtime_error("bucket_allreduce: bad block count");
  if ((algo == kAlgoNvls || algo == kAlgoNvlsOneShot) && ctx.mc_base == nullptr) throw std::runtime_error("bucket_allreduce: NVLS requested without multicast");
  if (tab.total_elems % 8 != 0) throw std::runtime_error("bucket_allreduce: bucket not padded to 8 elements");
  if (tab.count < 1) throw std::runtime_error("bucket_allreduce: empty bucket");
  ArArgs args;
  args.ctx = ctx;
  args.stage_off = stage_off;
  args.flat_out = flat_out;
  args.sq_partials = sq_partials;
  args.flags_out = flags_out;
  args.scale = scale;
  args.scatter = scatter ? 1 : 0;
  args.direct = 0;
  args.tab = tab;
  const bool in_bf16 = in_dtype == DType::BF16, wire_bf16 = wire_dtype == DType::BF16;
  if (in_dtype != DType::BF16 && in_dtype != DType::F32) throw std::runtime_error("bucket_allreduce: grads must be fp32 or bf16");
  if (in_bf16 && wire_bf16) launch_typed<__nv_bfloat16, __nv_bfloat16>(args, algo, blocks, stream);
  else if (in_bf16) launch_typed<__nv_bfloat16, float>(args, algo, blocks, stream);
  else if (wire_bf16) launch_typed<float, __nv_bfloat16>(args, algo, blocks, stream);
  else launch_typed<float, float>(args, algo, blocks, stream);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200
