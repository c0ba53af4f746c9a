// Host-callable entry points of the peer-memory collectives: what replaces the NCCL calls torch DDP issues for the
// reference (init broadcast at wrap time, ddp.py:192-196; per-bucket allreduce during backward, ddp.py:230-232).
#pragma once
#include <cuda_runtime.h>
#include "common.h"
#include "peer_mem.h"

namespace b200 {

struct CommCtx;
struct BucketTable;

enum : int { kAlgoAuto = -1, kAlgoOneShot = 0, kAlgoTwoShot = 1, kAlgoNvls = 2, kAlgoNvlsOneShot = 3 };

// allreduce.cu
void launch_bucket_allreduce(const CommCtx& ctx, const BucketTable& tab, size_t stage_off, DType in_dtype,
                             DType wire_dtype, int algo, int blocks, void* flat_out, float* sq_partials,
                             float* flags_out, float scale, bool scatter, cudaStream_t stream);

// in-place allreduce of a buffer that already lives at the same offset in every rank's arena (symmetric memory)
void launch_symmetric_allreduce(const CommCtx& ctx, size_t buf_off, size_t numel, DType dtype, int algo, int blocks, float scale,
                                cudaStream_t stream);

// broadcast.cu : `tab` slots are byte ranges (numel/off in BYTES, off multiple of 16)
void launch_peer_broadcast(const CommCtx& ctx, const BucketTable& tab, size_t stage_off, int src_rank,
                           bool use_multicast, int blocks, cudaStream_t stream);

// link probes (broadcast.cu)
void launch_peer_pull(const CommCtx& ctx, int peer, size_t src_off, void* dst, size_t bytes, int blocks,
                      cudaStream_t stream);
void launch_peer_push(const CommCtx& ctx, int peer, size_t dst_off, const void* src, size_t bytes, int blocks,
                      cudaStream_t stream);
void launch_peer_barrier(const CommCtx& ctx, int blocks, cudaStream_t stream);

}  // namespace b200
