// Native gradient reducer (replacement for c10d::Reducer).
//
// Host-side state machine only - all data movement happens inside the fused kernel it launches:
//   mark_ready(param, grad_ptr, compute_stream)  called from the parameter's post-accumulate hook;
//       stores the gradient's device pointer in the bucket's tensor table and decrements the
//       bucket's pending count.  When a bucket completes AND every earlier bucket has launched
//       (strict plan order on every rank -> no cross-rank launch-order deadlock), it records an
//       event on the compute stream, makes the high-priority comm stream wait on it, and launches
//       ONE bucket_allreduce kernel there.
//   finalize(compute_stream)  end of backward: launches what is left (parameters that never
//       fired contribute zeros and a cleared "used" flag), then makes the compute stream wait for
//       the comm stream.  Works unchanged under CUDA-graph capture (only event record/wait and
//       kernel launches are issued).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "comm.h"
#include "comm_kernels.cuh"

namespace b200 {

// Greedy size-capped bucket assignment (same algorithm as parallel/buckets.py::assign_by_size).
std::vector<std::vector<int>> assign_by_size(const std::vector<long long>& nbytes, const std::vector<int>& keys,
                                             const std::vector<long long>& limits, int max_tensors);

struct BucketPlan {
  std::vector<int> param_indices;
  std::vector<uint32_t> numels;
  std::vector<uint32_t> offsets;
  uint32_t data_elems = 0;
  uint32_t total_elems = 0;
  int grad_dtype = 0;   // DType of this bucket's gradients (buckets are planned per dtype)
  int wire_dtype = 0;   // DType on the wire
  bool tail = false;    // finishes at the end of backward: gets the wide (tail_blocks) grid
};

struct ReducerOptions {
  int algo = kAlgoAuto;
  int max_blocks = 24;        // CTAs for buckets that overlap with the rest of backward (light: see comm_kernels.cuh)
  int tail_blocks = 96;       // CTAs for the last bucket of the plan: nothing is left to overlap with, latency is exposed
  long long one_shot_max_bytes = 256 * 1024;
  long long tail_one_shot_max_bytes = 8ll << 20;   // tail bucket: single-rendezvous algorithm up to this wire size
  bool as_view = false;
  bool find_unused = false;
  float extra_scale = 1.0f;
  double timeout_s = 30.0;
  // Where the bucket kernels run.  -1 (default): launches recorded into a CUDA graph fork onto the comm stream (they overlap the
  // rest of backward when the graph replays); launches issued eagerly follow set_eager_inline(): on the comm stream for an
  // eager training loop, IN LINE on the compute stream for the few eager warm-up steps of a graph-captured loop.  Reason,
  // once a THIRD stream of the process has executed work, every later graph replay pays extra at each of its ~430 kernel
  // boundaries; default stream + capture stream are two.  0 / 1 force comm stream / in line everywhere.
  int serial = -1;
  int wide_blocks = 264;
};

class Reducer {
 public:
  Reducer(PeerArena* arena, std::vector<BucketPlan> plans, int num_params, ReducerOptions opt);
  ~Reducer();

  int num_buckets() const { return (int)plans_.size(); }
  int bucket_blocks(int b) const { return buckets_[b].blocks; }
  int bucket_algo(int b) const { return buckets_[b].algo; }
  // python-owned device buffers
  void set_flat_out(int b, uintptr_t ptr) { buckets_[b].flat_out = reinterpret_cast<void*>(ptr); }
  void set_sq_partials(uintptr_t ptr, int stride) { sq_partials_ = reinterpret_cast<float*>(ptr); sq_stride_ = stride; }

  void reset();
  void mark_ready(int param_index, uintptr_t grad_ptr, uintptr_t compute_stream);
  int finalize(uintptr_t compute_stream);      // returns #params that never fired
  std::vector<float> read_used_flags(int b);   // syncs the comm stream; only for the unused-param path
  void synchronize();
  uintptr_t comm_stream() const { return reinterpret_cast<uintptr_t>(comm_stream_); }
  // true if bucket kernels launched from `compute_stream` right now would run in line (see ReducerOptions::serial)
  bool runs_inline(uintptr_t compute_stream) const;
  void note_comm_stream_used() { used_comm_stream_ = true; }
  void set_eager_inline(bool on) { eager_inline_ = on; }
  int error_code() const { return arena_->check_error(); }

  long long launches = 0, bytes_on_wire = 0, iterations = 0;
  std::vector<int> ready_order;  // observed in the first iteration

 private:
  struct BucketState {
    BucketTable table;
    size_t stage_off = 0;
    void* flat_out = nullptr;
    float* flags_host = nullptr;  // pinned, mapped
    float* flags_dev = nullptr;
    int pending = 0, blocks = 1, blocks_wide = 1, algo = kAlgoTwoShot;
    bool launched = false;
    cudaEvent_t ready_event = nullptr;
  };
  void launch_in_order(cudaStream_t compute);
  void launch_bucket(int b, cudaStream_t compute);

  PeerArena* arena_;
  std::vector<BucketPlan> plans_;
  std::vector<BucketState> buckets_;
  std::vector<std::pair<int, int>> where_;   // param -> (bucket, slot)
  std::vector<char> fired_;
  ReducerOptions opt_;
  CommCtx ctx_;
  cudaStream_t comm_stream_ = nullptr;
  cudaEvent_t done_event_ = nullptr;
  float* sq_partials_ = nullptr;
  int sq_stride_ = 0;
  int next_bucket_ = 0;
  bool active_ = false;
  bool first_iter_ = true;
  bool eager_inline_ = false;       // see ReducerOptions::serial
  bool used_comm_stream_ = false;   // this backward pass forked onto the comm stream: finalize must join it
};

}  // namespace b200
