// Host side of the gradient reducer (see reducer.h).  Reference behaviour being replaced: the c10d Reducer that
// `DistributedDataParallel(model, ..., find_unused_parameters=True)` (reference ddp.py:192-196) builds at wrap time and
// drives from autograd hooks on every `loss.backward()` (reference ddp.py:230-232).
#include "reducer.h"

#include <algorithm>
#include <cstdlib>
#include <map>

#include <nvtx3/nvToolsExt.h>   // header-only; a no-op unless a tool injected itself

namespace b200 {

std::vector<std::vector<int>> assign_by_size(const std::vector<long long>& nbytes, const std::vector<int>& keys,
                                             const std::vector<long long>& limits, int max_tensors) {
  if (limits.empty()) throw std::runtime_error("assign_by_size: need at least one limit");
  struct Open { std::vector<int> members; long long total = 0; };
  std::map<int, Open> open;
  std::map<int, size_t> cursor;
  std::vector<std::vector<int>> closed;
  for (size_t i = 0; i < nbytes.size(); ++i) {
    const int key = keys.empty() ? 0 : keys[i];
    Open& o = open[key];
    o.members.push_back((int)i);
    o.total += nbytes[i];
    size_t& pos = cursor[key];
    const bool by_size = o.total >= limits[pos];
    const bool by_count = max_tensors > 0 && (int)o.members.size() >= max_tensors;
    if (by_size || by_count) {
      closed.push_back(std::move(o.members));
      open.erase(key);
      if (by_size && pos + 1 < limits.size()) ++pos;
    }
  }
  for (auto& kv : open)
    if (!kv.second.members.empty()) closed.push_back(std::move(kv.second.members));
  std::sort(closed.begin(), closed.end(), [](const std::vector<int>& a, const std::vector<int>& b) {
    return *std::min_element(a.begin(), a.end()) < *std::min_element(b.begin(), b.end());
  });
  return closed;
}

Reducer::Reducer(PeerArena* arena, std::vector<BucketPlan> plans, int num_params, ReducerOptions opt)
    : arena_(arena), plans_(std::move(plans)), opt_(opt) {
  B200_CUDA_CHECK(cudaSetDevice(arena_->device()));
  int lo = 0, hi = 0;
  B200_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  B200_CUDA_CHECK(cudaStreamCreateWithPriority(&comm_stream_, cudaStreamNonBlocking, hi));
  B200_CUDA_CHECK(cudaEventCreateWithFlags(&done_event_, cudaEventDisableTiming));

  ctx_.base = arena_->base();
  ctx_.mc_base = arena_->mc_base();
  ctx_.stride = arena_->stride();
  ctx_.pad_off = 0;   // per bucket: pad set 2 + bucket index (sets 0/1 belong to the generic collectives)
  ctx_.error_word = arena_->error_word_dev();
  ctx_.timeout_ns = (unsigned long long)(opt_.timeout_s * 1e9);
  ctx_.rank = arena_->rank();
  ctx_.world = arena_->world();

  where_.assign(num_params, {-1, -1});
  fired_.assign(num_params, 0);
  buckets_.resize(plans_.size());
  for (size_t b = 0; b < plans_.size(); ++b) {
    const BucketPlan& p = plans_[b];
    BucketState& s = buckets_[b];
    if ((2 + b + 1) * kPadSetBytes > kSignalBytes) throw std::runtime_error("Reducer: too many buckets for the signal-pad area");
    if ((int)p.param_indices.size() > kMaxBucketTensors)
      throw std::runtime_error("Reducer: bucket has more tensors than one launch can carry");
    if (p.total_elems % 8 != 0) throw std::runtime_error("Reducer: bucket not padded to 8 elements");
    s.table.count = (int)p.param_indices.size();
    s.table.data_elems = p.data_elems;
    s.table.total_elems = p.total_elems;
    s.table._pad = 0;
    for (int k = 0; k < s.table.count; ++k) {
      s.table.t[k].ptr = nullptr;
      s.table.t[k].numel = p.numels[k];
      s.table.t[k].off = p.offsets[k];
      where_.at(p.param_indices[k]) = {(int)b, k};
    }
    const size_t wire_bytes = (size_t)p.total_elems * dtype_size((DType)p.wire_dtype);
    s.stage_off = arena_->alloc(wire_bytes, 4096);
    // algorithm + grid per bucket (static, so every rank picks the same)
    int algo = opt_.algo;
    if (algo == kAlgoAuto) {
      const bool mc = arena_->has_multicast();
      // The bucket that completes at the very end of backward is pure exposed latency: with in-switch reduction every rank
      // simply multimem.ld_reduce's the whole (<= tail_one_shot_max_bytes) bucket - one rendezvous, no second exchange phase.
      const bool is_tail = p.tail || b + 1 == plans_.size();
      if ((long long)wire_bytes <= opt_.one_shot_max_bytes) algo = mc ? kAlgoNvlsOneShot : kAlgoOneShot;
      else if (is_tail && mc && (long long)wire_bytes <= opt_.tail_one_shot_max_bytes) algo = kAlgoNvlsOneShot;
      else if (is_tail && !mc && ctx_.world == 2 && (long long)wire_bytes <= opt_.tail_one_shot_max_bytes) algo = kAlgoOneShot;
      else algo = mc ? kAlgoNvls : kAlgoTwoShot;
    }
    if (algo == kAlgoNvls && !arena_->has_multicast()) algo = kAlgoTwoShot;
    if (algo == kAlgoNvlsOneShot && !arena_->has_multicast()) algo = kAlgoOneShot;
    s.algo = algo;
    const long long vecs = (long long)(wire_bytes / 16);
    const long long per_rank = (algo == kAlgoOneShot || algo == kAlgoNvlsOneShot) ? vecs : (vecs + ctx_.world - 1) / ctx_.world;
    long long blocks = (per_rank + kCommThreads * 8 - 1) / (kCommThreads * 8);
    const int cap = (p.tail || b + 1 == plans_.size()) ? opt_.tail_blocks : opt_.max_blocks;
    s.blocks = (int)std::max(1LL, std::min<long long>(blocks, std::min(cap, kMaxCommBlocks)));
    const long long wide = (per_rank + kCommThreads * 2 - 1) / (kCommThreads * 2);
    s.blocks_wide = (int)std::max(1LL, std::min<long long>(wide, std::min(opt_.wide_blocks, kMaxCommBlocks)));
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&s.ready_event, cudaEventDisableTiming));
    B200_CUDA_CHECK(cudaHostAlloc((void**)&s.flags_host, sizeof(float) * kMaxBucketTensors, cudaHostAllocMapped));
    B200_CUDA_CHECK(cudaHostGetDevicePointer((void**)&s.flags_dev, s.flags_host, 0));
    std::fill(s.flags_host, s.flags_host + kMaxBucketTensors, 0.f);
  }
  for (auto& w : where_)
    if (w.first < 0) throw std::runtime_error("Reducer: a parameter is missing from the bucket plan");
}

Reducer::~Reducer() {
  if (comm_stream_) cudaStreamSynchronize(comm_stream_);
  for (auto& s : buckets_) {
    if (s.ready_event) cudaEventDestroy(s.ready_event);
    if (s.flags_host) cudaFreeHost(s.flags_host);
  }
  if (done_event_) cudaEventDestroy(done_event_);
  if (comm_stream_) cudaStreamDestroy(comm_stream_);
}

void Reducer::reset() {
  for (size_t b = 0; b < buckets_.size(); ++b) {
    BucketState& s = buckets_[b];
    s.pending = s.table.count;
    s.launched = false;
    for (int k = 0; k < s.table.count; ++k) s.table.t[k].ptr = nullptr;
  }
  std::fill(fired_.begin(), fired_.end(), 0);
  next_bucket_ = 0;
  active_ = true;
}

void Reducer::mark_ready(int param_index, uintptr_t grad_ptr, uintptr_t compute_stream) {
  if (!active_) reset();
  if (fired_.at(param_index))
    throw std::runtime_error("Reducer: parameter #" + std::to_string(param_index) +
                             " produced a gradient twice in one backward pass");
  fired_[param_index] = 1;
  const auto [b, k] = where_[param_index];
  BucketState& s = buckets_[b];
  s.table.t[k].ptr = reinterpret_cast<void*>(grad_ptr);
  if (first_iter_) ready_order.push_back(param_index);
  if (--s.pending == 0) launch_in_order(reinterpret_cast<cudaStream_t>(compute_stream));
}

void Reducer::launch_in_order(cudaStream_t compute) {
  while (next_bucket_ < (int)buckets_.size() && buckets_[next_bucket_].pending == 0) {
    launch_bucket(next_bucket_, compute);
    ++next_bucket_;
  }
}

namespace {
// B200DDP_NVTX=1: one range per bucket launch ("b200ddp.bucket<k> <bytes>B algo<a> x<blocks>") for timeline tools.
bool nvtx_enabled() {
  static const bool on = [] { const char* e = std::getenv("B200DDP_NVTX"); return e && std::atoi(e) != 0; }();
  return on;
}
}  // namespace

bool Reducer::runs_inline(uintptr_t compute_stream) const {
  if (opt_.serial == 0 || opt_.serial == 1) return opt_.serial != 0;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(reinterpret_cast<cudaStream_t>(compute_stream), &st) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  const bool capturing = st == cudaStreamCaptureStatusActive;
  if (opt_.serial == 3) return capturing;                 // diagnostics: the opposite assignment
  return capturing ? false : eager_inline_;               // captured launches fork onto the comm stream; eager ones as configured
}

void Reducer::launch_bucket(int b, cudaStream_t compute) {
  BucketState& s = buckets_[b];
  const bool inline_run = runs_inline(reinterpret_cast<uintptr_t>(compute));
  cudaStream_t where = inline_run ? compute : comm_stream_;
  const int blocks = inline_run ? s.blocks_wide : s.blocks;
  const bool mark = nvtx_enabled();
  if (mark) {
    const std::string label = "b200ddp.bucket" + std::to_string(b) + " " +
                              std::to_string((long long)s.table.total_elems * (long long)dtype_size((DType)plans_[b].wire_dtype)) +
                              "B algo" + std::to_string(s.algo) + " x" + std::to_string(s.blocks);
    nvtxRangePushA(label.c_str());
  }
  if (!inline_run) {
    B200_CUDA_CHECK(cudaEventRecord(s.ready_event, compute));
    B200_CUDA_CHECK(cudaStreamWaitEvent(comm_stream_, s.ready_event, 0));
    used_comm_stream_ = true;
  }
  float* sq = sq_partials_ ? sq_partials_ + (size_t)b * sq_stride_ : nullptr;
  const float scale = opt_.extra_scale / (float)ctx_.world;
  const bool scatter = !opt_.as_view;
  CommCtx ctx = ctx_;
  ctx.pad_off = (size_t)(2 + b) * kPadSetBytes;
  static const int debug_mode = [] { const char* e = std::getenv("B200DDP_DEBUG_BUCKET"); return e ? std::atoi(e) : 0; }();
  if (debug_mode == 1) { s.launched = true; ++launches; if (mark) nvtxRangePop(); return; }                 // diagnostics: bookkeeping only
  launch_bucket_allreduce(ctx, s.table, s.stage_off, (DType)plans_[b].grad_dtype, (DType)plans_[b].wire_dtype, s.algo, blocks,
                          (opt_.as_view || opt_.find_unused) ? s.flat_out : nullptr, sq,
                          opt_.find_unused ? s.flags_dev : nullptr, scale, scatter, where);
  if (mark) nvtxRangePop();
  s.launched = true;
  ++launches;
  bytes_on_wire += (long long)s.table.total_elems * (long long)dtype_size((DType)plans_[b].wire_dtype);
}

int Reducer::finalize(uintptr_t compute_stream) {
  if (!active_) return 0;
  active_ = false;
  cudaStream_t compute = reinterpret_cast<cudaStream_t>(compute_stream);
  int missing = 0;
  for (char f : fired_) missing += f ? 0 : 1;
  if (missing && !opt_.find_unused) {
    std::string which;
    for (size_t i = 0, shown = 0; i < fired_.size() && shown < 8; ++i)
      if (!fired_[i]) { which += std::to_string(i) + " "; ++shown; }
    throw std::runtime_error(std::to_string(missing) + " parameter(s) (indices " + which +
                             "...) received no gradient in this backward pass; construct "
                             "DistributedDataParallel(find_unused_parameters=True) if that is expected");
  }
  for (auto& s : buckets_)
    if (!s.launched) s.pending = 0;   // missing tensors keep ptr == nullptr: zeros + cleared flag
  launch_in_order(compute);
  if (used_comm_stream_) {
    B200_CUDA_CHECK(cudaEventRecord(done_event_, comm_stream_));
    B200_CUDA_CHECK(cudaStreamWaitEvent(compute, done_event_, 0));
    used_comm_stream_ = false;
  }
  first_iter_ = false;
  ++iterations;
  return missing;
}

std::vector<float> Reducer::read_used_flags(int b) {
  B200_CUDA_CHECK(cudaStreamSynchronize(comm_stream_));
  BucketState& s = buckets_.at(b);
  return std::vector<float>(s.flags_host, s.flags_host + s.table.count);
}

void Reducer::synchronize() { B200_CUDA_CHECK(cudaStreamSynchronize(comm_stream_)); }

}  // namespace b200
