// Python bindings.  The only translation unit that sees torch headers.  Which reference call site each op stands in for is
// documented on the Python side (b200ddp/ops/functional.py, parallel/peer.py, optim/).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include "comm.h"
#include "comm_kernels.cuh"
#include "conv.h"
#include "gemm.h"
#include "ops.h"
#include "peer_mem.h"
#include "reducer.h"
#include "tensor_map.h"

namespace py = pybind11;
using namespace b200;

namespace {

DType dtype_of(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return DType::F32;
    case at::kBFloat16: return DType::BF16;
    case at::kByte: return DType::U8;
    case at::kLong: return DType::I64;
    default: throw std::runtime_error("b200ddp: unsupported dtype " + std::string(c10::toString(t.scalar_type())));
  }
}

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

void check_cuda(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.is_contiguous() || t.is_non_overlapping_and_dense(), name, " must be dense");
}

CommCtx make_ctx(PeerArena& a, size_t pad_off, double timeout_s) {
  CommCtx c;
  c.base = a.base();
  c.mc_base = a.mc_base();
  c.stride = a.stride();
  c.pad_off = pad_off;
  c.error_word = a.error_word_dev();
  c.timeout_ns = (unsigned long long)(timeout_s * 1e9);
  c.rank = a.rank();
  c.world = a.world();
  return c;
}

// Standalone fused allreduce of a list of tensors treated as one flat bucket (tests, sweeps,
// PeerCollectives.allreduce_).  Slots are padded to 8 elements, a flags tail is appended.
void allreduce_tensors(PeerArena& arena, const std::vector<at::Tensor>& tensors, const std::string& wire, int algo,
                       int blocks, size_t stage_off, size_t stage_bytes, double scale, int pad_set, double timeout_s,
                       c10::optional<at::Tensor> sq_partials) {
  TORCH_CHECK(!tensors.empty() && (int)tensors.size() <= kMaxBucketTensors, "allreduce_tensors: 1..", kMaxBucketTensors, " tensors");
  const DType in_dt = dtype_of(tensors[0]);
  const DType wire_dt = wire == "fp32" ? DType::F32 : DType::BF16;
  BucketTable tab;
  uint32_t off = 0;
  tab.count = (int)tensors.size();
  for (int k = 0; k < tab.count; ++k) {
    const at::Tensor& t = tensors[k];
    check_cuda(t, "tensor");
    TORCH_CHECK(dtype_of(t) == in_dt, "allreduce_tensors: mixed dtypes in one bucket");
    tab.t[k].ptr = t.data_ptr();
    tab.t[k].numel = (uint32_t)t.numel();
    tab.t[k].off = off;
    off += (uint32_t)((t.numel() + 7) / 8 * 8);
  }
  tab.data_elems = off;
  tab.total_elems = off + (uint32_t)((tab.count + 7) / 8 * 8);
  tab._pad = 0;
  TORCH_CHECK((size_t)tab.total_elems * dtype_size(wire_dt) <= stage_bytes, "allreduce_tensors: staging region too small");
  CommCtx ctx = make_ctx(arena, (size_t)pad_set * kPadSetBytes, timeout_s);
  if (algo == kAlgoAuto) algo = arena.has_multicast() ? kAlgoNvls : kAlgoTwoShot;
  float* sq = sq_partials.has_value() ? sq_partials->data_ptr<float>() : nullptr;
  launch_bucket_allreduce(ctx, tab, stage_off, in_dt, wire_dt, algo, blocks, nullptr, sq, nullptr, (float)scale,
                          /*scatter=*/true, cur_stream());
}

// Broadcast arbitrary tensors from `src`; chunked through the staging region.
int broadcast_tensors(PeerArena& arena, const std::vector<at::Tensor>& tensors, int src, size_t stage_off,
                      size_t stage_bytes, bool use_mc, int blocks, int pad_set, double timeout_s) {
  CommCtx ctx = make_ctx(arena, (size_t)pad_set * kPadSetBytes, timeout_s);
  int launches = 0;
  size_t i = 0;
  const size_t n = tensors.size();
  // a tensor larger than the staging region is sent in pieces
  size_t piece_off = 0;
  while (i < n) {
    BucketTable tab;
    tab.count = 0;
    uint32_t off = 0;
    while (i < n && tab.count < kMaxBucketTensors) {
      const at::Tensor& t = tensors[i];
      check_cuda(t, "tensor");
      const size_t nbytes = (size_t)t.numel() * t.element_size() - piece_off;
      const size_t room = stage_bytes - off;
      if (room < 16) break;
      size_t take = nbytes <= room ? nbytes : (room / 16) * 16;
      if (take == 0) break;
      tab.t[tab.count].ptr = static_cast<char*>(t.data_ptr()) + piece_off;
      tab.t[tab.count].numel = (uint32_t)take;
      tab.t[tab.count].off = off;
      ++tab.count;
      off += (uint32_t)((take + 15) / 16 * 16);
      if (take == nbytes) { ++i; piece_off = 0; } else { piece_off += take; break; }
    }
    if (tab.count == 0) throw std::runtime_error("broadcast_tensors: staging region too small");
    tab.data_elems = off;
    tab.total_elems = off;
    tab._pad = 0;
    launch_peer_broadcast(ctx, tab, stage_off, src, use_mc, blocks, cur_stream());
    ++launches;
  }
  return launches;
}

// ---- optimizer ---------------------------------------------------------------------------------
struct OptPlan {
  std::vector<uintptr_t> params;
  std::vector<long long> numels, flat_offs;
  DType p_dtype, g_dtype;
  int total_blocks = 0;
  OptPlan(std::vector<uintptr_t> p, std::vector<long long> n, std::vector<long long> fo, int pd, int gd)
      : params(std::move(p)), numels(std::move(n)), flat_offs(std::move(fo)), p_dtype((DType)pd), g_dtype((DType)gd) {
    for (auto v : numels) total_blocks += ceil_div(v, kOptChunk);
  }
  template <typename F>
  void for_each_table(const std::vector<uintptr_t>& grads, F&& fn) const {
    size_t i = 0;
    int block_base = 0;
    while (i < params.size()) {
      OptTable tab;
      tab.count = 0;
      tab.total_blocks = 0;
      while (i < params.size() && tab.count < kMaxOptTensors) {
        OptSlot& s = tab.t[tab.count++];
        s.p = reinterpret_cast<void*>(params[i]);
        s.g = reinterpret_cast<const void*>(grads[i]);
        s.flat_off = (unsigned long long)flat_offs[i];
        s.numel = (uint32_t)numels[i];
        s.blk0 = (uint32_t)tab.total_blocks;
        tab.total_blocks += ceil_div(numels[i], kOptChunk);
        ++i;
      }
      fn(tab, block_base);
      block_base += tab.total_blocks;
    }
  }
  int sqnorm(const std::vector<uintptr_t>& grads, uintptr_t partials, uintptr_t stream) const {
    TORCH_CHECK(grads.size() == params.size(), "OptPlan: gradient list length mismatch");
    for_each_table(grads, [&](const OptTable& tab, int base) {
      launch_multi_sqnorm(tab, g_dtype, reinterpret_cast<float*>(partials) + base, reinterpret_cast<cudaStream_t>(stream));
    });
    return total_blocks;
  }
  void step(const std::vector<uintptr_t>& grads, uintptr_t lr, uintptr_t clip_coef, uintptr_t master, uintptr_t mom,
            uintptr_t step_count, double momentum, double dampening, double weight_decay, double grad_scale, bool nesterov,
            bool zero_grad, uintptr_t stream) const {
    TORCH_CHECK(grads.size() == params.size(), "OptPlan: gradient list length mismatch");
    SgdHyper h;
    h.lr = reinterpret_cast<const float*>(lr);
    h.clip_coef = reinterpret_cast<const float*>(clip_coef);
    h.master = reinterpret_cast<float*>(master);
    h.momentum_buf = reinterpret_cast<float*>(mom);
    h.step_count = reinterpret_cast<const int*>(step_count);
    h.momentum = (float)momentum;
    h.dampening = (float)dampening;
    h.weight_decay = (float)weight_decay;
    h.grad_scale = (float)grad_scale;
    h.nesterov = nesterov ? 1 : 0;
    h.zero_grad = zero_grad ? 1 : 0;
    for_each_table(grads, [&](const OptTable& tab, int) {
      launch_multi_sgd(tab, p_dtype, g_dtype, h, reinterpret_cast<cudaStream_t>(stream));
    });
  }
  void adamw(const std::vector<uintptr_t>& grads, uintptr_t lr, uintptr_t clip_coef, uintptr_t master, uintptr_t exp_avg,
             uintptr_t exp_avg_sq, uintptr_t step_count, double beta1, double beta2, double eps, double weight_decay,
             double grad_scale, bool zero_grad, uintptr_t stream) const {
    TORCH_CHECK(grads.size() == params.size(), "OptPlan: gradient list length mismatch");
    TORCH_CHECK(lr && exp_avg && exp_avg_sq && step_count, "OptPlan.adamw: lr, moments and step count are required");
    AdamHyper h;
    h.lr = reinterpret_cast<const float*>(lr);
    h.clip_coef = reinterpret_cast<const float*>(clip_coef);
    h.master = reinterpret_cast<float*>(master);
    h.exp_avg = reinterpret_cast<float*>(exp_avg);
    h.exp_avg_sq = reinterpret_cast<float*>(exp_avg_sq);
    h.step_count = reinterpret_cast<const int*>(step_count);
    h.beta1 = (float)beta1;
    h.beta2 = (float)beta2;
    h.eps = (float)eps;
    h.weight_decay = (float)weight_decay;
    h.grad_scale = (float)grad_scale;
    h.zero_grad = zero_grad ? 1 : 0;
    for_each_table(grads, [&](const OptTable& tab, int) {
      launch_multi_adamw(tab, p_dtype, g_dtype, h, reinterpret_cast<cudaStream_t>(stream));
    });
  }
};

// grouped-query causal documents: qkv [B*S, (heads + 2*kv_heads)*hd] with head dim hd = 64 (causal_gqa_attention_*) or
// 128 (causal_attention_d128_*, kv_heads == heads included); the same bounds as the packed pair
int gqa_check(const at::Tensor& qkv, const at::Tensor& bounds, int heads, int kv_heads, int hd, const char* who) {
  check_cuda(qkv, "qkv");
  TORCH_CHECK(qkv.scalar_type() == at::kBFloat16 && qkv.dim() == 2 && qkv.is_contiguous(), who,
              ": qkv must be contiguous bf16 [B*S, (heads + 2*kv_heads)*", hd, "]");
  TORCH_CHECK(heads >= 1 && kv_heads >= 1 && heads % kv_heads == 0, who, ": kv_heads (", kv_heads, ") must divide heads (", heads, ")");
  TORCH_CHECK(qkv.size(1) == (int64_t)(heads + 2 * kv_heads) * hd, who, ": qkv has ", qkv.size(1),
              " columns, expected (heads + 2 * kv_heads) * ", hd, " with heads = ", heads, ", kv_heads = ", kv_heads);
  check_cuda(bounds, "bounds");
  TORCH_CHECK(bounds.scalar_type() == at::kInt && bounds.dim() == 3 && bounds.size(2) == 2 && bounds.is_contiguous() && bounds.numel() >= 2,
              who, ": bounds must be contiguous int32 [B, S, 2]");
  TORCH_CHECK(qkv.size(0) == bounds.size(0) * bounds.size(1), who, ": qkv rows (", qkv.size(0), ") are not B * S for bounds [",
              bounds.size(0), ", ", bounds.size(1), ", 2]");
  TORCH_CHECK(bounds.device() == qkv.device(), who, ": bounds must be on qkv's device");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(qkv.data_ptr()) & 15) == 0 && (reinterpret_cast<uintptr_t>(bounds.data_ptr()) & 7) == 0,
              who, ": qkv must be 16-byte and bounds 8-byte aligned");
  return (int)bounds.size(0);
}

using GqaFwd = void (*)(const void*, const int*, int, int, int, int, void*, float*, cudaStream_t);
using GqaBwd = void (*)(const void*, const void*, const void*, const float*, const int*, int, int, int, int, float*, void*, cudaStream_t);

std::tuple<at::Tensor, at::Tensor> gqa_fwd(GqaFwd launch, int hd, const char* who, const at::Tensor& qkv, const at::Tensor& bounds,
                                           int heads, int kv_heads, c10::optional<at::Tensor> o_out, c10::optional<at::Tensor> lse_out) {
  const int B = gqa_check(qkv, bounds, heads, kv_heads, hd, who);
  c10::cuda::CUDAGuard guard(qkv.device());
  const int S = (int)(qkv.size(0) / B);
  at::Tensor o = o_out.has_value() ? *o_out : at::empty({qkv.size(0), (int64_t)heads * hd}, qkv.options());
  at::Tensor lse = lse_out.has_value() ? *lse_out : at::empty({B, heads, S}, qkv.options().dtype(at::kFloat));
  TORCH_CHECK(o.is_cuda() && o.scalar_type() == at::kBFloat16 && o.is_contiguous() && o.numel() == qkv.size(0) * heads * hd, who, ": bad o");
  TORCH_CHECK(lse.is_cuda() && lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == (int64_t)B * heads * S, who, ": bad lse");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(o.data_ptr()) & 15) == 0 && (reinterpret_cast<uintptr_t>(lse.data_ptr()) & 7) == 0,
              who, ": o must be 16-byte and lse 8-byte aligned");
  launch(qkv.data_ptr(), bounds.data_ptr<int>(), B, S, heads, kv_heads, o.data_ptr(), lse.data_ptr<float>(), cur_stream());
  return std::make_tuple(o, lse);
}

at::Tensor gqa_bwd(GqaBwd launch, int hd, const char* who, const at::Tensor& dout, const at::Tensor& qkv, const at::Tensor& o,
                   const at::Tensor& lse, const at::Tensor& bounds, int heads, int kv_heads, c10::optional<at::Tensor> dqkv_out) {
  const int B = gqa_check(qkv, bounds, heads, kv_heads, hd, who);
  c10::cuda::CUDAGuard guard(qkv.device());
  const int S = (int)(qkv.size(0) / B);
  for (const at::Tensor* t : {&dout, &o}) {
    check_cuda(*t, "dout / o");
    TORCH_CHECK(t->scalar_type() == at::kBFloat16 && t->is_contiguous() && t->numel() == qkv.size(0) * heads * hd &&
                (reinterpret_cast<uintptr_t>(t->data_ptr()) & 15) == 0, who, ": dout and o must be 16-byte aligned contiguous bf16 [B*S, heads*",
                hd, "]");
  }
  TORCH_CHECK(lse.is_cuda() && lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == (int64_t)B * heads * S &&
              (reinterpret_cast<uintptr_t>(lse.data_ptr()) & 7) == 0, who, ": lse must be 8-byte aligned contiguous fp32 [B, heads, S]");
  at::Tensor dqkv = dqkv_out.has_value() ? *dqkv_out : at::empty_like(qkv);
  TORCH_CHECK(dqkv.is_cuda() && dqkv.scalar_type() == at::kBFloat16 && dqkv.is_contiguous() && dqkv.numel() == qkv.numel() &&
              (reinterpret_cast<uintptr_t>(dqkv.data_ptr()) & 3) == 0, who, ": bad dqkv");
  at::Tensor dsum = at::empty({B, heads, S}, qkv.options().dtype(at::kFloat));
  launch(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), bounds.data_ptr<int>(), B, S, heads, kv_heads,
         dsum.data_ptr<float>(), dqkv.data_ptr(), cur_stream());
  return dqkv;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "b200ddp native extension (sm_90a)";
  m.attr("MAX_BUCKET_TENSORS") = kMaxBucketTensors;
  m.attr("MAX_COMM_BLOCKS") = kMaxCommBlocks;
  m.attr("SIGNAL_BYTES") = (long long)kSignalBytes;
  m.attr("ALGO_AUTO") = (int)kAlgoAuto;
  m.attr("ALGO_ONE_SHOT") = (int)kAlgoOneShot;
  m.attr("ALGO_TWO_SHOT") = (int)kAlgoTwoShot;
  m.attr("ALGO_NVLS") = (int)kAlgoNvls;
  m.attr("ALGO_NVLS_ONE_SHOT") = (int)kAlgoNvlsOneShot;

  m.def("launch_count", []() { return (long long)launch_counter().load(); });
  m.def("assign_by_size", &assign_by_size, py::arg("nbytes"), py::arg("keys"), py::arg("limits"), py::arg("max_tensors") = 0);
  // the 128 bytes of the tensor map the kernels would get for this geometry (tests compare them with recorded ones)
  m.def("_tensor_map_bytes", [](uintptr_t ptr, int dtype, int swizzle, const std::vector<uint64_t>& dims, const std::vector<uint64_t>& strides,
                                const std::vector<uint32_t>& box) {
    TORCH_CHECK(!dims.empty() && dims.size() <= 4 && box.size() == dims.size() && strides.size() + 1 == dims.size(), "tensor map: bad rank");
    const CUtensorMap map = encode_tensor_map(reinterpret_cast<const void*>(ptr), (CUtensorMapDataType)dtype, (CUtensorMapSwizzle)swizzle,
                                              (int)dims.size(), dims.data(), strides.data(), box.data());
    return py::bytes(reinterpret_cast<const char*>(&map), sizeof(map));
  });

  py::class_<PeerArena>(m, "PeerArena")
      .def(py::init<int, int, int, size_t, const std::string&>())
      .def("bind_socket", &PeerArena::bind_socket)
      .def("exchange", &PeerArena::exchange, py::call_guard<py::gil_scoped_release>())
      .def("multicast_supported", &PeerArena::multicast_supported)
      .def("multicast_create", &PeerArena::multicast_create, py::call_guard<py::gil_scoped_release>())
      .def("multicast_add_device", &PeerArena::multicast_add_device)
      .def("multicast_bind", &PeerArena::multicast_bind)
      .def("disable_multicast", &PeerArena::disable_multicast)
      .def("has_multicast", &PeerArena::has_multicast)
      .def("alloc", &PeerArena::alloc, py::arg("nbytes"), py::arg("align") = 256)
      .def("used", &PeerArena::used)
      .def("rewind", &PeerArena::rewind)
      .def("bytes", &PeerArena::bytes)
      .def("rank", &PeerArena::rank)
      .def("world", &PeerArena::world)
      .def("local_ptr", [](PeerArena& a) { return (uintptr_t)a.local(); })
      .def("peer_ptr", [](PeerArena& a, int r) { return (uintptr_t)a.peer(r); })
      .def("mc_ptr", [](PeerArena& a) { return (uintptr_t)a.mc_base(); })
      .def("check_error", &PeerArena::check_error)
      .def("clear_error", &PeerArena::clear_error)
      .def("close", &PeerArena::close);

  m.def("allreduce_tensors", &allreduce_tensors, py::arg("arena"), py::arg("tensors"), py::arg("wire") = "bf16",
        py::arg("algo") = (int)kAlgoAuto, py::arg("blocks") = 32, py::arg("stage_off"), py::arg("stage_bytes"),
        py::arg("scale") = 1.0, py::arg("pad_set") = 1, py::arg("timeout_s") = 30.0, py::arg("sq_partials") = py::none());
  m.def("arena_tensor", [](PeerArena& a, size_t offset, int64_t numel, int dtype_code) {
    auto dt = dtype_code == 1 ? at::kBFloat16 : dtype_code == 2 ? at::kByte : at::kFloat;
    auto opts = at::TensorOptions().dtype(dt).device(at::kCUDA, a.device());
    return at::from_blob(a.local() + offset, {numel}, [](void*) {}, opts);
  });
  m.def("allreduce_symmetric", [](PeerArena& a, size_t buf_off, int64_t numel, int dtype_code, int algo, int blocks, double scale,
                                  int pad_set, double timeout_s) {
    CommCtx ctx = make_ctx(a, (size_t)pad_set * kPadSetBytes, timeout_s);
    if (algo == kAlgoAuto) algo = a.has_multicast() ? kAlgoNvls : kAlgoTwoShot;
    launch_symmetric_allreduce(ctx, buf_off, (size_t)numel, (DType)dtype_code, algo, blocks, (float)scale, cur_stream());
  });
  m.def("broadcast_tensors", &broadcast_tensors, py::arg("arena"), py::arg("tensors"), py::arg("src") = 0, py::arg("stage_off"),
        py::arg("stage_bytes"), py::arg("use_mc") = false, py::arg("blocks") = 32, py::arg("pad_set") = 1,
        py::arg("timeout_s") = 30.0);
  m.def("peer_pull", [](PeerArena& a, int peer, size_t src_off, at::Tensor dst, size_t bytes, int blocks) {
    launch_peer_pull(make_ctx(a, 0, 30.0), peer, src_off, dst.data_ptr(), bytes, blocks, cur_stream());
  });
  m.def("peer_push", [](PeerArena& a, int peer, size_t dst_off, at::Tensor src, size_t bytes, int blocks) {
    launch_peer_push(make_ctx(a, 0, 30.0), peer, dst_off, src.data_ptr(), bytes, blocks, cur_stream());
  });
  m.def("peer_barrier", [](PeerArena& a, int blocks, int pad_set, double timeout_s) {
    launch_peer_barrier(make_ctx(a, (size_t)pad_set * kPadSetBytes, timeout_s), blocks, cur_stream());
  }, py::arg("arena"), py::arg("blocks") = 1, py::arg("pad_set") = 1, py::arg("timeout_s") = 30.0);

  py::class_<BucketPlan>(m, "BucketPlan")
      .def(py::init<>())
      .def_readwrite("param_indices", &BucketPlan::param_indices)
      .def_readwrite("numels", &BucketPlan::numels)
      .def_readwrite("offsets", &BucketPlan::offsets)
      .def_readwrite("data_elems", &BucketPlan::data_elems)
      .def_readwrite("total_elems", &BucketPlan::total_elems)
      .def_readwrite("grad_dtype", &BucketPlan::grad_dtype)
      .def_readwrite("wire_dtype", &BucketPlan::wire_dtype)
      .def_readwrite("tail", &BucketPlan::tail);

  py::class_<Reducer>(m, "Reducer")
      .def(py::init([](PeerArena& arena, std::vector<BucketPlan> plans, int num_params, int algo,
                       int max_blocks, int tail_blocks, long long one_shot_max_bytes, bool as_view, bool find_unused, double extra_scale,
                       double timeout_s, int serial, int wide_blocks, long long tail_one_shot_max_bytes) {
             ReducerOptions o;
             o.algo = algo;
             o.max_blocks = max_blocks;
             o.tail_blocks = tail_blocks;
             o.one_shot_max_bytes = one_shot_max_bytes;
             o.as_view = as_view;
             o.find_unused = find_unused;
             o.extra_scale = (float)extra_scale;
             o.timeout_s = timeout_s;
             o.serial = serial;
             o.wide_blocks = wide_blocks;
             o.tail_one_shot_max_bytes = tail_one_shot_max_bytes;
             return std::make_unique<Reducer>(&arena, std::move(plans), num_params, o);
           }),
           py::keep_alive<1, 2>())
      .def("num_buckets", &Reducer::num_buckets)
      .def("bucket_blocks", &Reducer::bucket_blocks)
      .def("bucket_algo", &Reducer::bucket_algo)
      .def("set_flat_out", &Reducer::set_flat_out)
      .def("set_sq_partials", &Reducer::set_sq_partials)
      .def("reset", &Reducer::reset)
      .def("mark_ready", &Reducer::mark_ready)
      .def("finalize", &Reducer::finalize)
      .def("read_used_flags", &Reducer::read_used_flags)
      .def("synchronize", &Reducer::synchronize)
      .def("comm_stream", &Reducer::comm_stream)
      .def("runs_inline", &Reducer::runs_inline)
      .def("note_comm_stream_used", &Reducer::note_comm_stream_used)
      .def("set_eager_inline", &Reducer::set_eager_inline)
      .def("error_code", &Reducer::error_code)
      .def_readonly("launches", &Reducer::launches)
      .def_readonly("bytes_on_wire", &Reducer::bytes_on_wire)
      .def_readonly("iterations", &Reducer::iterations)
      .def_readonly("ready_order", &Reducer::ready_order);

  py::class_<OptPlan>(m, "OptPlan")
      .def(py::init<std::vector<uintptr_t>, std::vector<long long>, std::vector<long long>, int, int>())
      .def_readonly("total_blocks", &OptPlan::total_blocks)
      .def("sqnorm", &OptPlan::sqnorm)
      .def("step", &OptPlan::step)
      .def("adamw", &OptPlan::adamw);
  m.def("clip_coef", [](at::Tensor partials, int n, double max_norm, double grad_scale, at::Tensor coef, at::Tensor norm) {
    launch_clip_coef(partials.data_ptr<float>(), n, (float)max_norm, (float)grad_scale, coef.data_ptr<float>(),
                     norm.data_ptr<float>(), cur_stream());
  });

  // ---- losses -----------------------------------------------------------------------------------
  m.def("mse_fwd_bwd", [](at::Tensor out, at::Tensor target, double gscale) {
    check_cuda(out, "out"); check_cuda(target, "target");
    TORCH_CHECK(out.is_contiguous() && target.is_contiguous() && out.sizes() == target.sizes() && out.dtype() == target.dtype(),
                "mse_fwd_bwd: out/target must be contiguous with equal shape and dtype");
    c10::cuda::CUDAGuard guard(out.device());
    const size_t n = (size_t)out.numel();
    const int blocks = mse_blocks(n);
    at::Tensor loss = at::empty({}, out.options().dtype(at::kFloat));
    at::Tensor dout = at::empty_like(out);
    at::Tensor scratch = at::zeros({blocks + 1}, out.options().dtype(at::kFloat));
    launch_mse_fwd_bwd(out.data_ptr(), target.data_ptr(), dtype_of(out), n, (float)gscale, loss.data_ptr<float>(), dout.data_ptr(),
                       scratch.data_ptr<float>(), blocks, cur_stream());
    return std::make_tuple(loss, dout);
  });
  m.def("xent_fwd_bwd", [](at::Tensor logits, at::Tensor targets, long long ignore_index, double gscale) {
    check_cuda(logits, "logits"); check_cuda(targets, "targets");
    TORCH_CHECK(logits.dim() == 2 && logits.is_contiguous() && targets.is_contiguous() && targets.scalar_type() == at::kLong &&
                targets.numel() == logits.size(0), "xent_fwd_bwd: logits [rows, cols] contiguous, targets int64 [rows]");
    c10::cuda::CUDAGuard guard(logits.device());
    const int rows = (int)logits.size(0), cols = (int)logits.size(1);
    at::Tensor loss = at::empty({}, logits.options().dtype(at::kFloat));
    at::Tensor row_loss = at::empty({rows + 1}, logits.options().dtype(at::kFloat));
    at::Tensor dlogits = at::empty_like(logits);
    launch_xent_fwd_bwd(logits.data_ptr(), targets.data_ptr<int64_t>() ? (const long long*)targets.data_ptr<int64_t>() : nullptr,
                        dtype_of(logits), rows, cols, ignore_index, (float)gscale, row_loss.data_ptr<float>(), loss.data_ptr<float>(),
                        dlogits.data_ptr(), cur_stream());
    return std::make_tuple(loss, dlogits);
  });
  // Fused LM-head cross-entropy: mean over non-ignored rows of cross_entropy(hidden [N,H] . weight [V,H]^T + bias [V]) without
  // the [N, V] logits.  Forward -> (loss fp32 [], lse fp32 [N], row_loss fp32 [N+1], row_loss[N] = non-ignored rows).
  auto lm_check = [](const at::Tensor& hidden, const at::Tensor& weight, const at::Tensor& targets, const c10::optional<at::Tensor>& bias) {
    check_cuda(hidden, "hidden"); check_cuda(weight, "weight"); check_cuda(targets, "targets");
    TORCH_CHECK(hidden.scalar_type() == at::kBFloat16 && weight.scalar_type() == at::kBFloat16 && hidden.dim() == 2 && weight.dim() == 2 &&
                hidden.is_contiguous() && weight.is_contiguous() && hidden.size(1) == weight.size(1),
                "lm_loss: hidden [N,H] and weight [V,H], bf16 contiguous");
    TORCH_CHECK(hidden.size(1) % 8 == 0 && weight.size(0) % 8 == 0, "lm_loss: H and V must be multiples of 8 (16-byte rows), got H=",
                hidden.size(1), ", V=", weight.size(0));
    TORCH_CHECK(hidden.size(0) >= 1, "lm_loss: no rows");
    TORCH_CHECK(targets.scalar_type() == at::kLong && targets.is_contiguous() && targets.numel() == hidden.size(0), "lm_loss: targets int64 [N]");
    if (bias.has_value())
      TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() && bias->numel() == weight.size(0), "lm_loss: bias bf16 [V]");
  };
  auto lm_out = [](const c10::optional<at::Tensor>& given, at::IntArrayRef sizes, const at::TensorOptions& opt, const char* name) {
    if (!given.has_value()) return at::empty(sizes, opt);
    TORCH_CHECK(given->is_contiguous() && given->sizes() == sizes && given->scalar_type() == opt.dtype().toScalarType(),
                "lm_loss: bad ", name, " output");
    return *given;
  };
  // rows (optional): int32 [1] device count of the leading rows that carry labels (compact_rows' count).  Only the 128-row tiles
  // below it are computed; the rows at or past it must be ignored ones, and get lse = row_loss = 0 (dh: zeros).
  auto rows_ptr = [](const c10::optional<at::Tensor>& rows, const at::Tensor& hidden) -> const int* {
    if (!rows.has_value()) return nullptr;
    check_cuda(*rows, "rows");
    TORCH_CHECK(rows->scalar_type() == at::kInt && rows->numel() == 1 && rows->device() == hidden.device(),
                "lm_loss: rows must be an int32 [1] tensor on the hidden states' device");
    return rows->data_ptr<int>();
  };
  m.def("lm_loss_fwd", [lm_check, lm_out, rows_ptr](at::Tensor hidden, at::Tensor weight, at::Tensor targets, c10::optional<at::Tensor> bias,
                                                    long long ignore_index, c10::optional<at::Tensor> lse_out, c10::optional<at::Tensor> row_loss_out,
                                                    c10::optional<at::Tensor> rows) {
    lm_check(hidden, weight, targets, bias);
    const int* bound = rows_ptr(rows, hidden);
    c10::cuda::CUDAGuard guard(hidden.device());
    const int N = (int)hidden.size(0), H = (int)hidden.size(1), V = (int)weight.size(0), tiles = (V + 127) / 128;
    const auto f32 = hidden.options().dtype(at::kFloat);
    at::Tensor loss = at::empty({}, f32);
    at::Tensor lse = lm_out(lse_out, {N}, f32, "lse");
    at::Tensor row_loss = lm_out(row_loss_out, {N + 1}, f32, "row_loss");
    at::Tensor partial = at::empty({tiles, N, 2}, f32);
    at::Tensor target_logit = at::empty({N}, f32);
    const auto* t = (const long long*)targets.data_ptr<int64_t>();
    launch_gemm_lm_lse(hidden.data_ptr(), weight.data_ptr(), bias.has_value() ? bias->data_ptr() : nullptr, N, V, H, t,
                       partial.data_ptr<float>(), target_logit.data_ptr<float>(), cur_stream(), bound);
    launch_lm_loss_combine(partial.data_ptr<float>(), target_logit.data_ptr<float>(), t, N, tiles, V, ignore_index, lse.data_ptr<float>(),
                           row_loss.data_ptr<float>(), loss.data_ptr<float>(), cur_stream(), bound);
    return std::make_tuple(loss, lse, row_loss);
  }, py::arg("hidden"), py::arg("weight"), py::arg("targets"), py::arg("bias") = py::none(), py::arg("ignore_index") = -100,
     py::arg("lse_out") = py::none(), py::arg("row_loss_out") = py::none(), py::arg("rows") = py::none());
  // Backward, `slice` vocabulary columns at a time: recompute the slice's logits into its bf16 gradient (one GEMM), then
  // dh += dlogits . weight[slice] (fp32, cast to bf16 once at the end), dweight[slice] = dlogits^T . hidden and, with
  // need_dbias, dbias[slice] = the column sums of dlogits (fixed order).  gscale: fp32 device scalar (the upstream
  // gradient).  rows: as for lm_loss_fwd.  Returns (dh bf16 [N,H], dweight bf16 [V,H], dbias bf16 [V]; each None when not asked for).
  m.def("lm_loss_bwd", [lm_check, lm_out, rows_ptr](at::Tensor hidden, at::Tensor weight, at::Tensor targets, c10::optional<at::Tensor> bias,
                                                    at::Tensor lse, at::Tensor row_loss, at::Tensor gscale, long long ignore_index, int slice,
                                                    bool need_dh, bool need_dweight, c10::optional<at::Tensor> dh_out,
                                                    c10::optional<at::Tensor> dweight_out, c10::optional<at::Tensor> rows, bool need_dbias) {
    lm_check(hidden, weight, targets, bias);
    TORCH_CHECK(!need_dbias || bias.has_value(), "lm_loss_bwd: need_dbias needs the bias");
    const int* bound = rows_ptr(rows, hidden);
    const int N = (int)hidden.size(0), H = (int)hidden.size(1), V = (int)weight.size(0);
    TORCH_CHECK(slice >= 128 && slice % 128 == 0, "lm_loss_bwd: slice must be a positive multiple of 128, got ", slice);
    for (const at::Tensor* t : {&lse, &row_loss, &gscale}) {
      check_cuda(*t, "lse / row_loss / gscale");
      TORCH_CHECK(t->scalar_type() == at::kFloat && t->is_contiguous(), "lm_loss_bwd: lse, row_loss and gscale are contiguous fp32");
    }
    TORCH_CHECK(lse.numel() == N && row_loss.numel() == N + 1 && gscale.numel() == 1, "lm_loss_bwd: lse [N], row_loss [N+1], gscale [1]");
    c10::cuda::CUDAGuard guard(hidden.device());
    const auto bf16 = hidden.options();
    at::Tensor dh, dweight, dbias, dh32, colsum;
    if (need_dh) {
      dh = lm_out(dh_out, {N, H}, bf16, "dh");
      // row-bounded: the data-gradient GEMM skips the tiles past the count, whose rows must read as zeros
      dh32 = bound != nullptr ? at::zeros({N, H}, bf16.dtype(at::kFloat)) : at::empty({N, H}, bf16.dtype(at::kFloat));
    }
    if (need_dweight) dweight = lm_out(dweight_out, {V, H}, bf16, "dweight");
    if (need_dbias) dbias = at::empty({V}, bf16);
    if (!need_dh && !need_dweight && !need_dbias) return std::make_tuple(dh, dweight, dbias);
    const int width = slice < V ? slice : V;
    at::Tensor dlogits = at::empty({(int64_t)N * width}, bf16);
    if (need_dbias) colsum = at::empty({(int64_t)column_sum_workspace(N, width)}, bf16.dtype(at::kFloat));
    const auto* t = (const long long*)targets.data_ptr<int64_t>();
    const auto* w = reinterpret_cast<const __nv_bfloat16*>(weight.data_ptr());
    const auto* b = bias.has_value() ? reinterpret_cast<const __nv_bfloat16*>(bias->data_ptr()) : nullptr;
    for (int v0 = 0; v0 < V; v0 += width) {
      const int vs = V - v0 < width ? V - v0 : width;
      launch_gemm_lm_dlogits(hidden.data_ptr(), w + (size_t)v0 * H, b ? b + v0 : nullptr, N, vs, H, v0, V, t, ignore_index,
                             lse.data_ptr<float>(), gscale.data_ptr<float>(), row_loss.data_ptr<float>() + N, dlogits.data_ptr(), cur_stream(),
                             bound);
      // dh [N,H] (+)= dlogits [N,vs] . weight[v0:v0+vs] (stored [vs,H]: MN-major B)
      if (need_dh && bound != nullptr)
        launch_gemm_bf16_rows(dlogits.data_ptr(), w + (size_t)v0 * H, dh32.data_ptr(), N, H, vs, false, DType::F32, v0 > 0, bound, cur_stream());
      else if (need_dh)
        launch_gemm_bf16(dlogits.data_ptr(), w + (size_t)v0 * H, dh32.data_ptr(), nullptr, N, H, vs, false, true, 0, DType::F32, v0 > 0,
                         cur_stream());
      // dweight[v0:v0+vs] [vs,H] = dlogits^T (stored [N,vs]: MN-major A) . hidden (stored [N,H]: MN-major B)
      auto* dw = need_dweight ? reinterpret_cast<__nv_bfloat16*>(dweight.data_ptr()) + (size_t)v0 * H : nullptr;
      if (need_dweight && bound != nullptr)
        launch_gemm_bf16_rows(dlogits.data_ptr(), hidden.data_ptr(), dw, vs, H, N, true, DType::BF16, false, bound, cur_stream());
      else if (need_dweight)
        launch_gemm_bf16(dlogits.data_ptr(), hidden.data_ptr(), dw, nullptr, vs, H, N, true, true, 0, DType::BF16, false, cur_stream());
      if (need_dbias)
        launch_column_sum(dlogits.data_ptr(), N, vs, bound, colsum.data_ptr<float>(),
                          reinterpret_cast<__nv_bfloat16*>(dbias.data_ptr()) + v0, cur_stream());
    }
    if (need_dh) dh.copy_(dh32);
    return std::make_tuple(dh, dweight, dbias);
  }, py::arg("hidden"), py::arg("weight"), py::arg("targets"), py::arg("bias"), py::arg("lse"), py::arg("row_loss"), py::arg("gscale"),
     py::arg("ignore_index"), py::arg("slice"), py::arg("need_dh") = true, py::arg("need_dweight") = true, py::arg("dh_out") = py::none(),
     py::arg("dweight_out") = py::none(), py::arg("rows") = py::none(), py::arg("need_dbias") = false);
  // Sparse prediction: compact_rows(targets int64 [T], ignore_index, vocab) -> (index int32 [T], count int32 [1], targets int64
  // [T]): a stable partition of the rows, those whose target is not ignore_index and lies in [0, vocab) first; the compacted
  // targets hold ignore_index from count on.  No host synchronisation.
  m.def("compact_rows", [](at::Tensor targets, long long ignore_index, long long vocab) {
    check_cuda(targets, "targets");
    TORCH_CHECK(targets.scalar_type() == at::kLong && targets.dim() == 1 && targets.is_contiguous() && targets.numel() >= 1 &&
                targets.numel() < (1LL << 31), "compact_rows: targets int64 [T], contiguous, 1 <= T < 2^31");
    TORCH_CHECK(vocab >= 1, "compact_rows: vocab must be positive, got ", vocab);
    c10::cuda::CUDAGuard guard(targets.device());
    const int T = (int)targets.numel();
    const auto i32 = targets.options().dtype(at::kInt);
    at::Tensor index = at::empty({T}, i32), count = at::empty({1}, i32), out = at::empty_like(targets);
    at::Tensor work = at::empty({2 * compact_chunks(T)}, i32);
    launch_compact_rows((const long long*)targets.data_ptr<int64_t>(), T, ignore_index, vocab, work.data_ptr<int>(), index.data_ptr<int>(),
                        count.data_ptr<int>(), (long long*)out.data_ptr<int64_t>(), cur_stream());
    return std::make_tuple(index, count, out);
  }, py::arg("targets"), py::arg("ignore_index"), py::arg("vocab"));
  auto rows_check = [](const at::Tensor& x, const at::Tensor& index, const at::Tensor& count, const char* name) {
    check_cuda(x, name); check_cuda(index, "index"); check_cuda(count, "count");
    TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous() && x.size(1) % 8 == 0,
                name, ": bf16 [T, H] contiguous with H % 8 == 0");
    TORCH_CHECK(index.scalar_type() == at::kInt && index.is_contiguous() && index.numel() == x.size(0) &&
                count.scalar_type() == at::kInt && count.numel() == 1, name, ": index int32 [T] and count int32 [1] (compact_rows)");
    TORCH_CHECK(index.device() == x.device() && count.device() == x.device(), name, ": tensors on different devices");
  };
  // gather_rows(x [T, H], index, count): out[r] = x[index[r]] for r < count, zero rows from count on
  m.def("gather_rows", [rows_check](at::Tensor x, at::Tensor index, at::Tensor count) {
    rows_check(x, index, count, "gather_rows");
    c10::cuda::CUDAGuard guard(x.device());
    at::Tensor out = at::empty_like(x);
    launch_gather_rows(x.data_ptr(), index.data_ptr<int>(), count.data_ptr<int>(), (int)x.size(0), (int)x.size(1), out.data_ptr(), cur_stream());
    return out;
  }, py::arg("x"), py::arg("index"), py::arg("count"));
  // scatter_rows(dy [T, H], index, count): dx[index[r]] = dy[r] for r < count, every other row of dx zero
  m.def("scatter_rows", [rows_check](at::Tensor dy, at::Tensor index, at::Tensor count) {
    rows_check(dy, index, count, "scatter_rows");
    c10::cuda::CUDAGuard guard(dy.device());
    at::Tensor dx = at::empty_like(dy);
    launch_scatter_rows(dy.data_ptr(), index.data_ptr<int>(), count.data_ptr<int>(), (int)dy.size(0), (int)dy.size(1), dx.data_ptr(),
                        cur_stream());
    return dx;
  }, py::arg("dy"), py::arg("index"), py::arg("count"));

  // tanh = false: the erf form; true: the tanh approximation
  m.def("gelu_fwd", [](at::Tensor pre, bool tanh) {
    check_cuda(pre, "pre");
    TORCH_CHECK(pre.is_contiguous(), "gelu_fwd: contiguous input");
    c10::cuda::CUDAGuard guard(pre.device());
    at::Tensor out = at::empty_like(pre);
    launch_gelu(pre.data_ptr(), nullptr, out.data_ptr(), dtype_of(pre), (size_t)pre.numel(), false, cur_stream(), tanh);
    return out;
  }, py::arg("pre"), py::arg("tanh") = false);
  m.def("gelu_bwd", [](at::Tensor dy, at::Tensor pre, bool tanh) {
    check_cuda(pre, "pre");
    TORCH_CHECK(pre.is_contiguous() && dy.is_contiguous() && dy.dtype() == pre.dtype() && dy.numel() == pre.numel(), "gelu_bwd: matching contiguous tensors");
    c10::cuda::CUDAGuard guard(pre.device());
    at::Tensor out = at::empty_like(pre);
    launch_gelu(pre.data_ptr(), dy.data_ptr(), out.data_ptr(), dtype_of(pre), (size_t)pre.numel(), true, cur_stream(), tanh);
    return out;
  }, py::arg("dy"), py::arg("pre"), py::arg("tanh") = false);

  // ---- layer norm -------------------------------------------------------------------------------
  m.def("layernorm_fwd", [](at::Tensor x, at::Tensor gamma, at::Tensor beta, double eps) {
    check_cuda(x, "x");
    TORCH_CHECK(x.is_contiguous() && gamma.is_contiguous() && beta.is_contiguous(), "layernorm_fwd: contiguous inputs");
    TORCH_CHECK(gamma.dtype() == x.dtype() && beta.dtype() == x.dtype(), "layernorm_fwd: gamma/beta dtype must match x");
    c10::cuda::CUDAGuard guard(x.device());
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    at::Tensor y = at::empty_like(x);
    at::Tensor mean = at::empty({rows}, x.options().dtype(at::kFloat));
    at::Tensor rstd = at::empty({rows}, x.options().dtype(at::kFloat));
    launch_layernorm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), dtype_of(x), rows, cols, (float)eps, y.data_ptr(),
                         mean.data_ptr<float>(), rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, mean, rstd);
  });
  m.def("layernorm_bwd", [](at::Tensor dy, at::Tensor x, at::Tensor gamma, at::Tensor mean, at::Tensor rstd) {
    check_cuda(dy, "dy");
    TORCH_CHECK(dy.is_contiguous() && x.is_contiguous(), "layernorm_bwd: contiguous inputs");
    c10::cuda::CUDAGuard guard(x.device());
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    const int parts = layernorm_partial_rows(rows);
    at::Tensor dx = at::empty_like(x);
    at::Tensor dgp = at::empty({parts, cols}, x.options().dtype(at::kFloat));
    at::Tensor dbp = at::empty({parts, cols}, x.options().dtype(at::kFloat));
    at::Tensor dgamma = at::empty_like(gamma);
    at::Tensor dbeta = at::empty_like(gamma);
    launch_layernorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(), dtype_of(x),
                         rows, cols, dx.data_ptr(), dgp.data_ptr<float>(), dbp.data_ptr<float>(), parts, dgamma.data_ptr(),
                         dbeta.data_ptr(), cur_stream());
    return std::make_tuple(dx, dgamma, dbeta);
  });

  // ---- linears ----------------------------------------------------------------------------------
  m.def("small_linear_fwd", [](at::Tensor x, at::Tensor w, c10::optional<at::Tensor> b, bool relu) {
    check_cuda(x, "x");
    TORCH_CHECK(x.scalar_type() == at::kFloat && w.scalar_type() == at::kFloat && x.is_contiguous() && w.is_contiguous(),
                "small_linear_fwd: fp32 contiguous");
    c10::cuda::CUDAGuard guard(x.device());
    const int K = (int)x.size(-1), N = (int)w.size(0);
    const int M = (int)(x.numel() / K);
    auto sizes = x.sizes().vec();
    sizes.back() = N;
    at::Tensor y = at::empty(sizes, x.options());
    launch_small_linear_fwd(x.data_ptr<float>(), w.data_ptr<float>(), b.has_value() ? b->data_ptr<float>() : nullptr,
                            y.data_ptr<float>(), M, N, K, relu ? 1 : 0, cur_stream());
    return y;
  });
  m.def("small_linear_bwd", [](at::Tensor dy, at::Tensor x, at::Tensor w, at::Tensor y, bool relu, bool need_dx, bool has_bias) {
    check_cuda(dy, "dy");
    c10::cuda::CUDAGuard guard(x.device());
    const int K = (int)x.size(-1), N = (int)w.size(0);
    const int M = (int)(x.numel() / K);
    at::Tensor dyc = dy.contiguous();
    at::Tensor dx = need_dx ? at::empty_like(x) : at::Tensor();
    at::Tensor dw = at::empty_like(w);
    at::Tensor db = has_bias ? at::empty({N}, w.options()) : at::Tensor();
    launch_small_linear_bwd(dyc.data_ptr<float>(), x.data_ptr<float>(), w.data_ptr<float>(), y.data_ptr<float>(),
                            need_dx ? dx.data_ptr<float>() : nullptr, dw.data_ptr<float>(), has_bias ? db.data_ptr<float>() : nullptr,
                            M, N, K, relu ? 1 : 0, 0, cur_stream());
    return std::make_tuple(dx, dw, db);
  });

  // wgmma GEMM: D[M,N] = act(A[M,K] @ B[N,K]^T + bias) ; all bf16 row-major, fp32 accumulate in registers
  m.def("gemm_nt", [](at::Tensor a, at::Tensor b, c10::optional<at::Tensor> bias, int epilogue, c10::optional<at::Tensor> out) {
    check_cuda(a, "a"); check_cuda(b, "b");
    TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm_nt: bf16 operands");
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.size(1) == b.size(1) && a.is_contiguous() && b.is_contiguous(),
                "gemm_nt: A [M,K], B [N,K], both K-major contiguous");
    c10::cuda::CUDAGuard guard(a.device());
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    at::Tensor d = out.has_value() ? *out : at::empty({M, N}, a.options());
    TORCH_CHECK(d.is_contiguous() && d.size(0) == M && d.size(1) == N, "gemm_nt: bad output");
    const void* bias_ptr = nullptr;
    if (bias.has_value()) {
      TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N, "gemm_nt: bias bf16 [N]");
      bias_ptr = bias->data_ptr();
    }
    launch_gemm_nt_bf16(a.data_ptr(), b.data_ptr(), d.data_ptr(), bias_ptr, M, N, K, epilogue, dtype_of(d), cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("epilogue") = 0, py::arg("out") = py::none());
  // general form: a_mn=false -> a is [M,K]; true -> a is stored [K,M].  b_mn=false -> b is [N,K]; true -> stored [K,N].
  m.def("gemm", [](at::Tensor a, at::Tensor b, c10::optional<at::Tensor> bias, bool a_mn, bool b_mn, int epilogue, bool out_fp32,
                   c10::optional<at::Tensor> out) {
    check_cuda(a, "a"); check_cuda(b, "b");
    TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm: bf16 operands");
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous(), "gemm: 2-D contiguous operands");
    c10::cuda::CUDAGuard guard(a.device());
    const int M = (int)(a_mn ? a.size(1) : a.size(0)), K = (int)(a_mn ? a.size(0) : a.size(1));
    const int N = (int)(b_mn ? b.size(1) : b.size(0)), Kb = (int)(b_mn ? b.size(0) : b.size(1));
    TORCH_CHECK(K == Kb, "gemm: reduction dims differ (", K, " vs ", Kb, ")");
    bool accumulate = false;
    at::Tensor d;
    if (out.has_value()) { d = *out; accumulate = d.scalar_type() == at::kFloat && out_fp32; }
    else d = at::empty({M, N}, a.options().dtype(out_fp32 ? at::kFloat : at::kBFloat16));
    TORCH_CHECK(d.is_contiguous() && d.size(0) == M && d.size(1) == N, "gemm: bad output");
    const void* bias_ptr = nullptr;
    if (bias.has_value()) {
      TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N, "gemm: bias bf16 [N]");
      bias_ptr = bias->data_ptr();
    }
    launch_gemm_bf16(a.data_ptr(), b.data_ptr(), d.data_ptr(), bias_ptr, M, N, K, a_mn, b_mn, epilogue, dtype_of(d), accumulate,
                     cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("a_mn") = false, py::arg("b_mn") = false,
     py::arg("epilogue") = 0, py::arg("out_fp32") = false, py::arg("out") = py::none());
  // forward GEMM (a [M,K], b [N,K]) that also returns per-32-row partial column statistics of its output: [2][ceil(M/32)][N]
  m.def("gemm_stats", [](at::Tensor a, at::Tensor b) {
    check_cuda(a, "a"); check_cuda(b, "b");
    TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm_stats: bf16 operands");
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous() && a.size(1) == b.size(1), "gemm_stats: [M,K] x [N,K]");
    c10::cuda::CUDAGuard guard(a.device());
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    at::Tensor d = at::empty({M, N}, a.options());
    at::Tensor stats = at::empty({2, (M + 31) / 32, N}, a.options().dtype(at::kFloat));
    launch_gemm_bf16(a.data_ptr(), b.data_ptr(), d.data_ptr(), nullptr, M, N, K, false, false, 0, DType::BF16, false, cur_stream(),
                     stats.data_ptr<float>());
    return std::make_tuple(d, stats);
  });
  // ---- FP8 (fp8.cu, gemm_wgmma.cu): E4M3 activations / weights, E5M2 gradients, power-of-two per-tensor scales ------------
  m.def("fp8_amax", [](at::Tensor t) {
    check_cuda(t, "t");
    TORCH_CHECK(t.scalar_type() == at::kBFloat16 && t.is_contiguous(), "fp8_amax: contiguous bf16 tensor");
    c10::cuda::CUDAGuard guard(t.device());
    if ((reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) != 0) t = t.clone();
    at::Tensor amax = at::empty({1}, t.options().dtype(at::kFloat));
    launch_fp8_amax(t.data_ptr(), (size_t)t.numel(), amax.data_ptr<float>(), cur_stream());
    return amax;
  });
  // q (t's shape), q^T [cols, rows] or None, scale_inv [1] (= 1/s), fp32 column sums [cols] or None; s comes from `amax`
  auto fp8_cast = [](at::Tensor t, at::Tensor amax, const std::string& fmt, bool want_transpose, bool want_colsum) {
    TORCH_CHECK(fmt == "e4m3" || fmt == "e5m2", "fp8: format must be 'e4m3' or 'e5m2', got '", fmt, "'");
    TORCH_CHECK(amax.is_cuda() && amax.scalar_type() == at::kFloat && amax.numel() == 1, "fp8: amax must be a 1-element fp32 CUDA tensor");
    const bool e5m2 = fmt == "e5m2";
    const int cols = (int)t.size(-1);
    const int rows = (int)(t.numel() / cols);
    at::Tensor q = at::empty(t.sizes(), t.options().dtype(e5m2 ? at::kFloat8_e5m2 : at::kFloat8_e4m3fn));
    at::Tensor qt = want_transpose ? at::empty({cols, rows}, q.options()) : at::Tensor();
    at::Tensor scale_inv = at::empty({1}, t.options().dtype(at::kFloat));
    at::Tensor colsum, partial;
    if (want_colsum) {
      colsum = at::empty({cols}, t.options().dtype(at::kFloat));
      partial = at::empty({fp8_colsum_parts(rows), cols}, t.options().dtype(at::kFloat));
    }
    launch_fp8_cast_transpose(t.data_ptr(), rows, cols, amax.data_ptr<float>(), e5m2, q.data_ptr(),
                              want_transpose ? qt.data_ptr() : nullptr, want_colsum ? partial.data_ptr<float>() : nullptr,
                              want_colsum ? colsum.data_ptr<float>() : nullptr, scale_inv.data_ptr<float>(), cur_stream());
    return py::make_tuple(q, want_transpose ? py::cast(qt) : py::none(), scale_inv, want_colsum ? py::cast(colsum) : py::none());
  };
  auto fp8_input = [](at::Tensor t) {
    check_cuda(t, "t");
    TORCH_CHECK(t.scalar_type() == at::kBFloat16 && t.is_contiguous() && t.dim() >= 1, "fp8: contiguous bf16 tensor");
    return (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) != 0 ? t.clone() : t;
  };
  m.def("fp8_cast_transpose", [fp8_cast, fp8_input](at::Tensor t, at::Tensor amax, const std::string& fmt, bool want_transpose, bool want_colsum) {
    t = fp8_input(t);
    c10::cuda::CUDAGuard guard(t.device());
    return fp8_cast(t, amax, fmt, want_transpose, want_colsum);
  }, py::arg("t"), py::arg("amax"), py::arg("fmt"), py::arg("want_transpose") = false, py::arg("want_colsum") = false);
  m.def("fp8_quantize", [fp8_cast, fp8_input](at::Tensor t, const std::string& fmt, bool want_transpose, bool want_colsum) {
    t = fp8_input(t);
    c10::cuda::CUDAGuard guard(t.device());
    at::Tensor amax = at::empty({1}, t.options().dtype(at::kFloat));
    launch_fp8_amax(t.data_ptr(), (size_t)t.numel(), amax.data_ptr<float>(), cur_stream());
    return fp8_cast(t, amax, fmt, want_transpose, want_colsum);
  }, py::arg("t"), py::arg("fmt"), py::arg("want_transpose") = false, py::arg("want_colsum") = false);
  // D[M,N] bf16 = epi(a_scale_inv * b_scale_inv * A[M,K] @ B[N,K]^T + bias): A e4m3 or e5m2, B e4m3, both K-major
  m.def("gemm_fp8", [](at::Tensor a, at::Tensor b, at::Tensor a_scale_inv, at::Tensor b_scale_inv, c10::optional<at::Tensor> bias,
                       int epilogue) {
    check_cuda(a, "a"); check_cuda(b, "b");
    TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn || a.scalar_type() == at::kFloat8_e5m2, "gemm_fp8: A must be float8_e4m3fn or float8_e5m2");
    TORCH_CHECK(b.scalar_type() == at::kFloat8_e4m3fn, "gemm_fp8: B must be float8_e4m3fn");
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.is_contiguous() && b.is_contiguous() && a.size(1) == b.size(1),
                "gemm_fp8: A [M,K], B [N,K], both K-major contiguous");
    for (const at::Tensor* s : {&a_scale_inv, &b_scale_inv})
      TORCH_CHECK(s->is_cuda() && s->scalar_type() == at::kFloat && s->numel() == 1, "gemm_fp8: scale factors are 1-element fp32 CUDA tensors");
    c10::cuda::CUDAGuard guard(a.device());
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    TORCH_CHECK(K % 16 == 0, "gemm_fp8: K = ", K, " must be a multiple of 16 (row pitch of the 8-bit operands)");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(a.data_ptr()) & 15) == 0 && (reinterpret_cast<uintptr_t>(b.data_ptr()) & 15) == 0,
                "gemm_fp8: operands must be 16-byte aligned");
    at::Tensor d = at::empty({M, N}, a.options().dtype(at::kBFloat16));
    const void* bias_ptr = nullptr;
    if (bias.has_value()) {
      TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == N && bias->is_contiguous(), "gemm_fp8: bias bf16 [N]");
      bias_ptr = bias->data_ptr();
    }
    launch_gemm_fp8(a.data_ptr(), b.data_ptr(), d.data_ptr(), bias_ptr, a_scale_inv.data_ptr<float>(), b_scale_inv.data_ptr<float>(),
                    M, N, K, a.scalar_type() == at::kFloat8_e5m2, epilogue, cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("a_scale_inv"), py::arg("b_scale_inv"), py::arg("bias") = py::none(), py::arg("epilogue") = 0);
  // ---- attention (attention.cu): head dim 64, S % 128 == 0, masks on the device ----------------------------------------
  auto attn_qkv_check = [](const at::Tensor& qkv, int heads, const char* who) {
    check_cuda(qkv, "qkv");
    TORCH_CHECK(qkv.scalar_type() == at::kBFloat16 && qkv.dim() == 2 && qkv.is_contiguous(), who, ": qkv must be contiguous bf16 [B*S, 3*heads*64]");
    TORCH_CHECK(heads >= 1 && qkv.size(1) == 3LL * heads * 64, who, ": qkv has ", qkv.size(1), " columns, expected 3 * heads * 64 with heads = ", heads);
  };
  // key padding: seq_lens int32 [B]; returns B
  auto attn_check = [attn_qkv_check](const at::Tensor& qkv, const at::Tensor& seq_lens, int heads, const char* who) {
    attn_qkv_check(qkv, heads, who);
    check_cuda(seq_lens, "seq_lens");
    TORCH_CHECK(seq_lens.scalar_type() == at::kInt && seq_lens.dim() == 1 && seq_lens.is_contiguous() && seq_lens.numel() >= 1, who, ": seq_lens must be int32 [B]");
    TORCH_CHECK(qkv.size(0) % seq_lens.numel() == 0, who, ": qkv rows (", qkv.size(0), ") are not B * S for B = ", seq_lens.numel());
    TORCH_CHECK(seq_lens.device() == qkv.device(), who, ": seq_lens must be on qkv's device");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(qkv.data_ptr()) & 15) == 0, who, ": qkv must be 16-byte aligned");
    return (int)seq_lens.numel();
  };
  // packed documents: bounds int32 [B, S, 2] (contiguous, so [B*S, 2] rows of (start, end)); returns B
  auto packed_check = [attn_qkv_check](const at::Tensor& qkv, const at::Tensor& bounds, int heads, const char* who) {
    attn_qkv_check(qkv, heads, who);
    check_cuda(bounds, "bounds");
    TORCH_CHECK(bounds.scalar_type() == at::kInt && bounds.dim() == 3 && bounds.size(2) == 2 && bounds.is_contiguous() && bounds.numel() >= 2,
                who, ": bounds must be contiguous int32 [B, S, 2]");
    TORCH_CHECK(qkv.size(0) == bounds.size(0) * bounds.size(1), who, ": qkv rows (", qkv.size(0), ") are not B * S for bounds [",
                bounds.size(0), ", ", bounds.size(1), ", 2]");
    TORCH_CHECK(bounds.device() == qkv.device(), who, ": bounds must be on qkv's device");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(qkv.data_ptr()) & 15) == 0 && (reinterpret_cast<uintptr_t>(bounds.data_ptr()) & 7) == 0,
                who, ": qkv must be 16-byte and bounds 8-byte aligned");
    return (int)bounds.size(0);
  };
  using AttnFwd = void (*)(const void*, const int*, int, int, int, void*, float*, cudaStream_t);
  using AttnBwd = void (*)(const void*, const void*, const void*, const float*, const int*, int, int, int, float*, void*, cudaStream_t);
  // (o [B*S, heads*64] bf16, lse [B, heads, S] fp32); optional caller-owned outputs
  auto attn_fwd = [](AttnFwd launch, const char* who, const at::Tensor& qkv, const at::Tensor& mask, int B, int heads,
                     c10::optional<at::Tensor> o_out, c10::optional<at::Tensor> lse_out) {
    c10::cuda::CUDAGuard guard(qkv.device());
    const int S = (int)(qkv.size(0) / B);
    at::Tensor o = o_out.has_value() ? *o_out : at::empty({qkv.size(0), (int64_t)heads * 64}, qkv.options());
    at::Tensor lse = lse_out.has_value() ? *lse_out : at::empty({B, heads, S}, qkv.options().dtype(at::kFloat));
    TORCH_CHECK(o.is_cuda() && o.scalar_type() == at::kBFloat16 && o.is_contiguous() && o.numel() == qkv.numel() / 3, who, ": bad o");
    TORCH_CHECK(lse.is_cuda() && lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == (int64_t)B * heads * S, who, ": bad lse");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(o.data_ptr()) & 15) == 0 && (reinterpret_cast<uintptr_t>(lse.data_ptr()) & 7) == 0,
                who, ": o must be 16-byte and lse 8-byte aligned");
    launch(qkv.data_ptr(), mask.data_ptr<int>(), B, S, heads, o.data_ptr(), lse.data_ptr<float>(), cur_stream());
    return std::make_tuple(o, lse);
  };
  // dqkv [B*S, 3*heads*64] bf16: the query / key / value column blocks hold dQ / dK / dV
  auto attn_bwd = [](AttnBwd launch, const char* who, const at::Tensor& dout, const at::Tensor& qkv, const at::Tensor& o,
                     const at::Tensor& lse, const at::Tensor& mask, int B, int heads, c10::optional<at::Tensor> dqkv_out) {
    c10::cuda::CUDAGuard guard(qkv.device());
    const int S = (int)(qkv.size(0) / B);
    for (const at::Tensor* t : {&dout, &o}) {
      check_cuda(*t, "dout / o");
      TORCH_CHECK(t->scalar_type() == at::kBFloat16 && t->is_contiguous() && t->numel() == qkv.numel() / 3 &&
                  (reinterpret_cast<uintptr_t>(t->data_ptr()) & 15) == 0, who, ": dout and o must be 16-byte aligned contiguous bf16 [B*S, heads*64]");
    }
    TORCH_CHECK(lse.is_cuda() && lse.scalar_type() == at::kFloat && lse.is_contiguous() && lse.numel() == (int64_t)B * heads * S &&
                (reinterpret_cast<uintptr_t>(lse.data_ptr()) & 7) == 0, who, ": lse must be 8-byte aligned contiguous fp32 [B, heads, S]");
    at::Tensor dqkv = dqkv_out.has_value() ? *dqkv_out : at::empty_like(qkv);
    TORCH_CHECK(dqkv.is_cuda() && dqkv.scalar_type() == at::kBFloat16 && dqkv.is_contiguous() && dqkv.numel() == qkv.numel() &&
                (reinterpret_cast<uintptr_t>(dqkv.data_ptr()) & 3) == 0, who, ": bad dqkv");
    at::Tensor dsum = at::empty({B, heads, S}, qkv.options().dtype(at::kFloat));
    launch(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), mask.data_ptr<int>(), B, S, heads,
           dsum.data_ptr<float>(), dqkv.data_ptr(), cur_stream());
    return dqkv;
  };
  m.def("attention_fwd", [attn_check, attn_fwd](at::Tensor qkv, at::Tensor seq_lens, int heads, c10::optional<at::Tensor> o_out,
                                                c10::optional<at::Tensor> lse_out) {
    const int B = attn_check(qkv, seq_lens, heads, "attention_fwd");
    return attn_fwd(&launch_attention_fwd, "attention_fwd", qkv, seq_lens, B, heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("seq_lens"), py::arg("heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("attention_bwd", [attn_check, attn_bwd](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor seq_lens,
                                                int heads, c10::optional<at::Tensor> dqkv_out) {
    const int B = attn_check(qkv, seq_lens, heads, "attention_bwd");
    return attn_bwd(&launch_attention_bwd, "attention_bwd", dout, qkv, o, lse, seq_lens, B, heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("seq_lens"), py::arg("heads"), py::arg("dqkv") = py::none());
  m.def("packed_attention_fwd", [packed_check, attn_fwd](at::Tensor qkv, at::Tensor bounds, int heads, c10::optional<at::Tensor> o_out,
                                                         c10::optional<at::Tensor> lse_out) {
    const int B = packed_check(qkv, bounds, heads, "packed_attention_fwd");
    return attn_fwd(&launch_packed_attention_fwd, "packed_attention_fwd", qkv, bounds, B, heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("packed_attention_bwd", [packed_check, attn_bwd](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds,
                                                         int heads, c10::optional<at::Tensor> dqkv_out) {
    const int B = packed_check(qkv, bounds, heads, "packed_attention_bwd");
    return attn_bwd(&launch_packed_attention_bwd, "packed_attention_bwd", dout, qkv, o, lse, bounds, B, heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("dqkv") = py::none());
  // causal documents: the same bounds and checks as the packed pair
  m.def("causal_attention_fwd", [packed_check, attn_fwd](at::Tensor qkv, at::Tensor bounds, int heads, c10::optional<at::Tensor> o_out,
                                                         c10::optional<at::Tensor> lse_out) {
    const int B = packed_check(qkv, bounds, heads, "causal_attention_fwd");
    return attn_fwd(&launch_causal_attention_fwd, "causal_attention_fwd", qkv, bounds, B, heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("causal_attention_bwd", [packed_check, attn_bwd](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds,
                                                         int heads, c10::optional<at::Tensor> dqkv_out) {
    const int B = packed_check(qkv, bounds, heads, "causal_attention_bwd");
    return attn_bwd(&launch_causal_attention_bwd, "causal_attention_bwd", dout, qkv, o, lse, bounds, B, heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("dqkv") = py::none());
  m.def("causal_gqa_attention_fwd", [](at::Tensor qkv, at::Tensor bounds, int heads, int kv_heads, c10::optional<at::Tensor> o_out,
                                              c10::optional<at::Tensor> lse_out) {
    return gqa_fwd(&launch_causal_gqa_attention_fwd, 64, "causal_gqa_attention_fwd", qkv, bounds, heads, kv_heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("causal_gqa_attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds, int heads,
                                              int kv_heads, c10::optional<at::Tensor> dqkv_out) {
    return gqa_bwd(&launch_causal_gqa_attention_bwd, 64, "causal_gqa_attention_bwd", dout, qkv, o, lse, bounds, heads, kv_heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"),
     py::arg("dqkv") = py::none());
  m.def("causal_attention_d128_fwd", [](at::Tensor qkv, at::Tensor bounds, int heads, int kv_heads, c10::optional<at::Tensor> o_out,
                                               c10::optional<at::Tensor> lse_out) {
    return gqa_fwd(&launch_causal_attention_d128_fwd, 128, "causal_attention_d128_fwd", qkv, bounds, heads, kv_heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("causal_attention_d128_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds, int heads,
                                               int kv_heads, c10::optional<at::Tensor> dqkv_out) {
    return gqa_bwd(&launch_causal_attention_d128_bwd, 128, "causal_attention_d128_bwd", dout, qkv, o, lse, bounds, heads, kv_heads,
                   dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"),
     py::arg("dqkv") = py::none());

  // ---- Llama building blocks: rotary embedding (rotary.cu), RMSNorm (layernorm.cu), SwiGLU (loss.cu) --------------------
  // y = rope(qkv) (backward: the transpose rotation); qkv bf16 [rows, (heads + 2*kv_heads)*d] with d = 64 or 128, positions
  // int32 [rows], table fp32 [max_pos, 2, d/2]
  m.def("rotary", [](at::Tensor x, at::Tensor pos, at::Tensor table, int heads, int kv_heads, bool backward, double q_scale) {
    check_cuda(x, "x"); check_cuda(pos, "position_ids"); check_cuda(table, "cos_sin");
    TORCH_CHECK(table.scalar_type() == at::kFloat && table.is_contiguous() && table.dim() == 3 && table.size(1) == 2 &&
                (table.size(2) == 32 || table.size(2) == 64), "rotary: cos_sin must be contiguous fp32 [max_position, 2, d/2], d = 64 or 128");
    const int d = (int)table.size(2) * 2;
    TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous() && heads >= 1 && kv_heads >= 1 &&
                x.size(1) == (int64_t)(heads + 2 * kv_heads) * d, "rotary: x must be contiguous bf16 [rows, (heads + 2*kv_heads)*d] for the "
                "table's head dim d = ", d);
    TORCH_CHECK(pos.scalar_type() == at::kInt && pos.is_contiguous() && pos.numel() == x.size(0), "rotary: position_ids must be int32 [rows]");
    c10::cuda::CUDAGuard guard(x.device());
    if ((reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) != 0) x = x.clone();
    at::Tensor y = at::empty_like(x);
    launch_rotary(x.data_ptr(), pos.data_ptr<int>(), table.data_ptr<float>(), (int)table.size(0), (size_t)x.size(0), heads, kv_heads, d,
                  y.data_ptr(), backward, cur_stream(), (float)q_scale);
    return y;
  }, py::arg("x"), py::arg("position_ids"), py::arg("cos_sin"), py::arg("heads"), py::arg("kv_heads"), py::arg("backward") = false,
     py::arg("q_scale") = 1.0);
  // Qwen3's per-head q / k RMSNorm + rotary, d = 128: (y, rstd fp32 [rows, heads + kv_heads]) = fwd(qkv, wq, wk, ...);
  // (dqkv, dwq, dwk) = bwd(dy, qkv, rstd, wq, wk, ...) with qkv the forward's input
  auto qk_norm_check = [](const char* name, at::Tensor x, at::Tensor wq, at::Tensor wk, at::Tensor pos, at::Tensor table, int heads,
                          int kv_heads) {
    check_cuda(x, "x"); check_cuda(wq, "q_weight"); check_cuda(wk, "k_weight"); check_cuda(pos, "position_ids"); check_cuda(table, "cos_sin");
    TORCH_CHECK(table.scalar_type() == at::kFloat && table.is_contiguous() && table.dim() == 3 && table.size(1) == 2 && table.size(2) == 64,
                name, ": cos_sin must be contiguous fp32 [max_position, 2, 64]");
    TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous() && heads >= 1 && kv_heads >= 1 &&
                x.size(1) == (int64_t)(heads + 2 * kv_heads) * 128, name, ": x must be contiguous bf16 [rows, (heads + 2*kv_heads)*128]");
    for (const at::Tensor& w : {wq, wk})
      TORCH_CHECK(w.scalar_type() == at::kBFloat16 && w.is_contiguous() && w.numel() == 128 && w.device() == x.device(), name,
                  ": q_weight and k_weight must be contiguous bf16 [128] on x's device");
    TORCH_CHECK(pos.scalar_type() == at::kInt && pos.is_contiguous() && pos.numel() == x.size(0), name, ": position_ids must be int32 [rows]");
  };
  m.def("qk_norm_rotary_fwd", [qk_norm_check](at::Tensor x, at::Tensor wq, at::Tensor wk, at::Tensor pos, at::Tensor table, int heads,
                                              int kv_heads, double eps) {
    qk_norm_check("qk_norm_rotary_fwd", x, wq, wk, pos, table, heads, kv_heads);
    c10::cuda::CUDAGuard guard(x.device());
    at::Tensor y = at::empty_like(x);
    at::Tensor rstd = at::empty({x.size(0), heads + kv_heads}, x.options().dtype(at::kFloat));
    launch_qk_norm_rotary_fwd(x.data_ptr(), wq.data_ptr(), wk.data_ptr(), pos.data_ptr<int>(), table.data_ptr<float>(), (int)table.size(0),
                              (size_t)x.size(0), heads, kv_heads, 128, (float)eps, y.data_ptr(), rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, rstd);
  }, py::arg("x"), py::arg("q_weight"), py::arg("k_weight"), py::arg("position_ids"), py::arg("cos_sin"), py::arg("heads"),
     py::arg("kv_heads"), py::arg("eps"));
  m.def("qk_norm_rotary_bwd", [qk_norm_check](at::Tensor dy, at::Tensor x, at::Tensor rstd, at::Tensor wq, at::Tensor wk, at::Tensor pos,
                                              at::Tensor table, int heads, int kv_heads) {
    qk_norm_check("qk_norm_rotary_bwd", x, wq, wk, pos, table, heads, kv_heads);
    check_cuda(dy, "dy"); check_cuda(rstd, "rstd");
    TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && dy.is_contiguous() && dy.sizes() == x.sizes() && dy.device() == x.device(),
                "qk_norm_rotary_bwd: dy must be contiguous bf16 shaped like x");
    TORCH_CHECK(rstd.scalar_type() == at::kFloat && rstd.is_contiguous() && rstd.device() == x.device() &&
                rstd.numel() == x.size(0) * (int64_t)(heads + kv_heads), "qk_norm_rotary_bwd: rstd must be fp32 [rows, heads + kv_heads]");
    c10::cuda::CUDAGuard guard(x.device());
    const int parts = qk_norm_rotary_partials((size_t)x.size(0));
    at::Tensor dx = at::empty_like(x);
    at::Tensor partial = at::empty({2, parts, 128}, x.options().dtype(at::kFloat));
    at::Tensor dwq = at::empty_like(wq), dwk = at::empty_like(wk);
    launch_qk_norm_rotary_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr<float>(), wq.data_ptr(), wk.data_ptr(), pos.data_ptr<int>(),
                              table.data_ptr<float>(), (int)table.size(0), (size_t)x.size(0), heads, kv_heads, 128, dx.data_ptr(),
                              partial.data_ptr<float>(), dwq.data_ptr(), dwk.data_ptr(), cur_stream());
    return std::make_tuple(dx, dwq, dwk);
  }, py::arg("dy"), py::arg("x"), py::arg("rstd"), py::arg("q_weight"), py::arg("k_weight"), py::arg("position_ids"), py::arg("cos_sin"),
     py::arg("heads"), py::arg("kv_heads"));
  auto aligned32 = [](at::Tensor t) { return (reinterpret_cast<uintptr_t>(t.data_ptr()) & 31) != 0 ? t.clone() : t; };
  m.def("rmsnorm_fwd", [aligned32](at::Tensor x, at::Tensor gamma, double eps) {
    check_cuda(x, "x"); check_cuda(gamma, "gamma");
    TORCH_CHECK(gamma.device() == x.device(), "rmsnorm_fwd: gamma must be on x's device");
    TORCH_CHECK(x.is_contiguous() && gamma.is_contiguous() && gamma.dtype() == x.dtype() && gamma.numel() == x.size(-1),
                "rmsnorm_fwd: contiguous x [..., cols] and gamma [cols] of one dtype");
    c10::cuda::CUDAGuard guard(x.device());
    x = aligned32(x); gamma = aligned32(gamma);
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    at::Tensor y = at::empty_like(x);
    at::Tensor rstd = at::empty({rows}, x.options().dtype(at::kFloat));
    launch_rmsnorm_fwd(x.data_ptr(), gamma.data_ptr(), dtype_of(x), rows, cols, (float)eps, y.data_ptr(), rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, rstd);
  });
  m.def("rmsnorm_bwd", [aligned32](at::Tensor dy, at::Tensor x, at::Tensor gamma, at::Tensor rstd) {
    check_cuda(dy, "dy"); check_cuda(x, "x"); check_cuda(gamma, "gamma"); check_cuda(rstd, "rstd");
    TORCH_CHECK(gamma.device() == x.device() && dy.device() == x.device() && rstd.device() == x.device() &&
                rstd.scalar_type() == at::kFloat && rstd.numel() == x.numel() / x.size(-1), "rmsnorm_bwd: dy, gamma and fp32 rstd [rows] on x's device");
    TORCH_CHECK(dy.is_contiguous() && x.is_contiguous() && dy.sizes() == x.sizes() && dy.dtype() == x.dtype(), "rmsnorm_bwd: matching contiguous inputs");
    c10::cuda::CUDAGuard guard(x.device());
    dy = aligned32(dy); x = aligned32(x); gamma = aligned32(gamma.contiguous());
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    const int parts = layernorm_partial_rows(rows);
    at::Tensor dx = at::empty_like(x);
    at::Tensor partial = at::empty({2 * parts, cols}, x.options().dtype(at::kFloat));
    at::Tensor counters = at::empty({(cols + 7) / 8}, x.options().dtype(at::kInt));
    at::Tensor dgamma = at::empty_like(gamma);
    launch_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), rstd.data_ptr<float>(), dtype_of(x), rows, cols, dx.data_ptr(),
                       partial.data_ptr<float>(), reinterpret_cast<unsigned int*>(counters.data_ptr<int>()), parts, dgamma.data_ptr(),
                       cur_stream());
    return std::make_tuple(dx, dgamma);
  });
  // Gated linear units on one projection [M, 2I]: SwiGLU (gate | up, out = silu(gate) * up) and GeGLU (input | gate,
  // out = gelu(input) * gate).  Forward: out [M, I]; backward: the gradient of both column blocks [M, 2I] from dy [M, I].
  using GluLaunch = void (*)(const void*, const void*, void*, size_t, int, bool, cudaStream_t);
  auto glu_fwd = [](at::Tensor gate_up, GluLaunch launch, const char* name) {
    check_cuda(gate_up, "gate_up");
    TORCH_CHECK(gate_up.scalar_type() == at::kBFloat16 && gate_up.is_contiguous() && gate_up.size(-1) % 16 == 0,
                name, "_fwd: contiguous bf16 [..., 2I] with I % 8 == 0");
    c10::cuda::CUDAGuard guard(gate_up.device());
    if ((reinterpret_cast<uintptr_t>(gate_up.data_ptr()) & 15) != 0) gate_up = gate_up.clone();
    auto sizes = gate_up.sizes().vec();
    const int inter = (int)(sizes.back() / 2);
    sizes.back() = inter;
    at::Tensor out = at::empty(sizes, gate_up.options());
    launch(gate_up.data_ptr(), nullptr, out.data_ptr(), (size_t)(gate_up.numel() / (2 * inter)), inter, false, cur_stream());
    return out;
  };
  auto glu_bwd = [](at::Tensor dy, at::Tensor gate_up, GluLaunch launch, const char* name) {
    check_cuda(dy, "dy"); check_cuda(gate_up, "gate_up");
    TORCH_CHECK(gate_up.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16 && gate_up.is_contiguous() &&
                dy.is_contiguous() && gate_up.size(-1) % 16 == 0 && dy.numel() * 2 == gate_up.numel() && dy.size(-1) * 2 == gate_up.size(-1),
                name, "_bwd: contiguous bf16 dy [..., I] and gate_up [..., 2I]");
    c10::cuda::CUDAGuard guard(gate_up.device());
    if ((reinterpret_cast<uintptr_t>(gate_up.data_ptr()) & 15) != 0) gate_up = gate_up.clone();
    if ((reinterpret_cast<uintptr_t>(dy.data_ptr()) & 15) != 0) dy = dy.clone();
    const int inter = (int)dy.size(-1);
    at::Tensor out = at::empty_like(gate_up);
    launch(gate_up.data_ptr(), dy.data_ptr(), out.data_ptr(), (size_t)(dy.numel() / inter), inter, true, cur_stream());
    return out;
  };
  m.def("swiglu_fwd", [glu_fwd](at::Tensor gate_up) { return glu_fwd(gate_up, launch_swiglu, "swiglu"); });
  m.def("swiglu_bwd", [glu_bwd](at::Tensor dy, at::Tensor gate_up) { return glu_bwd(dy, gate_up, launch_swiglu, "swiglu"); });
  m.def("geglu_fwd", [glu_fwd](at::Tensor input_gate) { return glu_fwd(input_gate, launch_geglu, "geglu"); });
  m.def("geglu_bwd", [glu_bwd](at::Tensor dy, at::Tensor input_gate) { return glu_bwd(dy, input_gate, launch_geglu, "geglu"); });

  // ---- mixture of experts (moe.cu, grouped GEMMs in gemm_wgmma.cu) -------------------------------------------------
  auto moe_tensor = [](const at::Tensor& t, at::ScalarType st, int64_t numel, const char* what) {
    check_cuda(t, what);
    TORCH_CHECK(t.scalar_type() == st && t.is_contiguous() && t.numel() == numel, "moe: ", what, " must be a contiguous ",
                c10::toString(st), " tensor of ", numel, " elements, got ", c10::toString(t.scalar_type()), " ", t.sizes());
  };
  // logits bf16 [T, E] -> (ids int32 [T, k], gates bf16 [T, k], probsum fp32 [E] (aux) or None)
  m.def("moe_route", [moe_tensor](at::Tensor logits, int k, bool aux) {
    TORCH_CHECK(logits.dim() == 2, "moe_route: logits [T, E]");
    const int T = (int)logits.size(0), E = (int)logits.size(1);
    moe_tensor(logits, at::kBFloat16, (int64_t)T * E, "logits");
    c10::cuda::CUDAGuard guard(logits.device());
    at::Tensor ids = at::empty({T, k}, logits.options().dtype(at::kInt));
    at::Tensor gates = at::empty({T, k}, logits.options());
    c10::optional<at::Tensor> probsum;
    at::Tensor partial;
    if (aux) {
      probsum = at::empty({E}, logits.options().dtype(at::kFloat));
      partial = at::empty({(T + 63) / 64, E}, logits.options().dtype(at::kFloat));
    }
    launch_moe_router_fwd(logits.data_ptr(), T, E, k, ids.data_ptr<int>(), gates.data_ptr(), aux ? partial.data_ptr<float>() : nullptr,
                          aux ? probsum->data_ptr<float>() : nullptr, cur_stream());
    return std::make_tuple(ids, gates, probsum);
  });
  // dlogits bf16 [T, E] from d(gates) fp32 [T, k] and d(probsum) fp32 [E] (or None)
  m.def("moe_router_bwd", [moe_tensor](at::Tensor logits, at::Tensor ids, at::Tensor dgates, c10::optional<at::Tensor> dprobsum) {
    TORCH_CHECK(logits.dim() == 2 && ids.dim() == 2 && ids.size(0) == logits.size(0), "moe_router_bwd: logits [T, E], ids [T, k]");
    const int T = (int)logits.size(0), E = (int)logits.size(1), k = (int)ids.size(1);
    moe_tensor(logits, at::kBFloat16, (int64_t)T * E, "logits");
    moe_tensor(ids, at::kInt, (int64_t)T * k, "ids");
    moe_tensor(dgates, at::kFloat, (int64_t)T * k, "dgates");
    if (dprobsum.has_value()) moe_tensor(*dprobsum, at::kFloat, E, "dprobsum");
    c10::cuda::CUDAGuard guard(logits.device());
    at::Tensor dlogits = at::empty_like(logits);
    launch_moe_router_bwd(logits.data_ptr(), T, E, k, ids.data_ptr<int>(), dgates.data_ptr<float>(),
                          dprobsum.has_value() ? dprobsum->data_ptr<float>() : nullptr, dlogits.data_ptr(), cur_stream());
    return dlogits;
  });
  // ids int32 [T, k] -> (counts [E], offsets [E + 1], fwd_map [capacity], inv_map [T, k], tile_expert [capacity / 128]), int32
  m.def("moe_permute", [moe_tensor](at::Tensor ids, int E) {
    TORCH_CHECK(ids.dim() == 2, "moe_permute: ids [T, k]");
    const int T = (int)ids.size(0), k = (int)ids.size(1);
    moe_tensor(ids, at::kInt, (int64_t)T * k, "ids");
    TORCH_CHECK(T >= 1 && E >= 1 && E <= kMoeMaxExperts && k >= 1 && k <= kMoeMaxTopK && k <= E,
                "moe_permute: needs T >= 1, 1 <= E <= 64, 1 <= k <= min(E, 8), got T=", T, " E=", E, " k=", k);
    c10::cuda::CUDAGuard guard(ids.device());
    const int cap = moe_capacity(T, E, k), chunks = moe_chunks(T, k);
    auto opt = ids.options();
    at::Tensor work = at::empty({2, chunks, E}, opt), counts = at::empty({E}, opt), offsets = at::empty({E + 1}, opt);
    at::Tensor fwd = at::empty({cap}, opt), inv = at::empty({T, k}, opt), tiles = at::empty({cap / kMoeAlign}, opt);
    launch_moe_permute(ids.data_ptr<int>(), T, E, k, work.data_ptr<int>(), counts.data_ptr<int>(), offsets.data_ptr<int>(),
                       fwd.data_ptr<int>(), inv.data_ptr<int>(), tiles.data_ptr<int>(), cur_stream());
    return std::make_tuple(counts, offsets, fwd, inv, tiles);
  });
  m.def("moe_capacity", [](int T, int E, int k) { return moe_capacity(T, E, k); });
  // x bf16 [T, H] -> x_perm [capacity, H]
  m.def("moe_gather", [moe_tensor](at::Tensor x, at::Tensor fwd_map, int k) {
    TORCH_CHECK(x.dim() == 2 && fwd_map.dim() == 1, "moe_gather: x [T, H], fwd_map [capacity]");
    moe_tensor(x, at::kBFloat16, x.numel(), "x");
    moe_tensor(fwd_map, at::kInt, fwd_map.numel(), "fwd_map");
    c10::cuda::CUDAGuard guard(x.device());
    const int H = (int)x.size(1), cap = (int)fwd_map.numel();
    at::Tensor out = at::empty({cap, H}, x.options());
    launch_moe_gather(x.data_ptr(), fwd_map.data_ptr<int>(), cap, H, k, out.data_ptr(), cur_stream());
    return out;
  });
  // forward: a [capacity, K] . w_e^T with w [E, N, K] -> [capacity, N]; dgrad: a [capacity, K] . w_e with w [E, K, N] -> [capacity, N]
  m.def("moe_gemm", [moe_tensor](at::Tensor a, at::Tensor w, at::Tensor tile_expert, bool dgrad, c10::optional<at::Tensor> out) {
    TORCH_CHECK(a.dim() == 2 && w.dim() == 3, "moe_gemm: a [rows, K], w [E, *, *]");
    const int rows = (int)a.size(0), E = (int)w.size(0);
    const int K = (int)(dgrad ? w.size(1) : w.size(2)), N = (int)(dgrad ? w.size(2) : w.size(1));
    TORCH_CHECK(a.size(1) == K, "moe_gemm: a has ", a.size(1), " columns, the weight's reduction dim is ", K);
    moe_tensor(a, at::kBFloat16, a.numel(), "a");
    moe_tensor(w, at::kBFloat16, w.numel(), "w");
    moe_tensor(tile_expert, at::kInt, rows / kMoeAlign, "tile_expert");
    c10::cuda::CUDAGuard guard(a.device());
    at::Tensor d = out.has_value() ? *out : at::empty({rows, N}, a.options());
    if (out.has_value()) moe_tensor(d, at::kBFloat16, (int64_t)rows * N, "out");
    launch_gemm_grouped(a.data_ptr(), w.data_ptr(), d.data_ptr(), rows, N, K, E, dgrad, tile_expert.data_ptr<int>(), cur_stream());
    return d;
  }, py::arg("a"), py::arg("w"), py::arg("tile_expert"), py::arg("dgrad"), py::arg("out") = py::none());
  // weight gradient: dw [E, M, N] (bf16), dw_e = a[s_e]^T . b[s_e] over expert e's segment of a [capacity, M] and b [capacity, N]
  m.def("moe_gemm_wgrad", [moe_tensor](at::Tensor a, at::Tensor b, at::Tensor offsets, c10::optional<at::Tensor> out) {
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.size(0) == b.size(0) && offsets.dim() == 1, "moe_gemm_wgrad: a [rows, M], b [rows, N], offsets [E + 1]");
    moe_tensor(a, at::kBFloat16, a.numel(), "a");
    moe_tensor(b, at::kBFloat16, b.numel(), "b");
    moe_tensor(offsets, at::kInt, offsets.numel(), "offsets");
    c10::cuda::CUDAGuard guard(a.device());
    const int rows = (int)a.size(0), M = (int)a.size(1), N = (int)b.size(1), E = (int)offsets.numel() - 1;
    at::Tensor d = out.has_value() ? *out : at::empty({E, M, N}, a.options());
    if (out.has_value()) moe_tensor(d, at::kBFloat16, (int64_t)E * M * N, "out");
    launch_gemm_grouped_wgrad(a.data_ptr(), b.data_ptr(), d.data_ptr(), rows, M, N, E, offsets.data_ptr<int>(), cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("offsets"), py::arg("out") = py::none());
  // out [T, H] = sum_j gate[t, j] * y_perm[inv[t, j]] (gates None: weight 1)
  m.def("moe_combine", [moe_tensor](at::Tensor y_perm, at::Tensor inv_map, c10::optional<at::Tensor> gates) {
    TORCH_CHECK(y_perm.dim() == 2 && inv_map.dim() == 2, "moe_combine: y_perm [capacity, H], inv_map [T, k]");
    const int T = (int)inv_map.size(0), k = (int)inv_map.size(1), H = (int)y_perm.size(1);
    moe_tensor(y_perm, at::kBFloat16, y_perm.numel(), "y_perm");
    moe_tensor(inv_map, at::kInt, (int64_t)T * k, "inv_map");
    if (gates.has_value()) moe_tensor(*gates, at::kBFloat16, (int64_t)T * k, "gates");
    c10::cuda::CUDAGuard guard(y_perm.device());
    at::Tensor out = at::empty({T, H}, y_perm.options());
    launch_moe_combine(y_perm.data_ptr(), inv_map.data_ptr<int>(), gates.has_value() ? gates->data_ptr() : nullptr, T, H, k, out.data_ptr(),
                       cur_stream());
    return out;
  });
  // (dy_perm bf16 [capacity, H], dgates fp32 [T, k]) from dout bf16 [T, H]
  m.def("moe_combine_bwd", [moe_tensor](at::Tensor dout, at::Tensor y_perm, at::Tensor fwd_map, at::Tensor gates) {
    TORCH_CHECK(dout.dim() == 2 && y_perm.dim() == 2 && gates.dim() == 2 && dout.size(1) == y_perm.size(1) && gates.size(0) == dout.size(0),
                "moe_combine_bwd: dout [T, H], y_perm [capacity, H], gates [T, k]");
    const int T = (int)dout.size(0), H = (int)dout.size(1), k = (int)gates.size(1), cap = (int)y_perm.size(0);
    moe_tensor(dout, at::kBFloat16, dout.numel(), "dout");
    moe_tensor(y_perm, at::kBFloat16, y_perm.numel(), "y_perm");
    moe_tensor(fwd_map, at::kInt, cap, "fwd_map");
    moe_tensor(gates, at::kBFloat16, (int64_t)T * k, "gates");
    c10::cuda::CUDAGuard guard(dout.device());
    at::Tensor dy = at::empty_like(y_perm);
    at::Tensor dgates = at::empty({T, k}, dout.options().dtype(at::kFloat));
    launch_moe_combine_bwd(dout.data_ptr(), y_perm.data_ptr(), fwd_map.data_ptr<int>(), gates.data_ptr(), cap, H, k, dy.data_ptr(),
                           dgates.data_ptr<float>(), cur_stream());
    return std::make_tuple(dy, dgates);
  });
  m.def("gemm_supported", &gemm_shape_supported);
  m.def("set_gemm_cta_mode", &set_gemm_cta_mode);
  m.def("set_gemm_group_m", &set_gemm_group_m);
  m.def("set_gemm_tma_store", &set_gemm_tma_store);
  m.def("gemm_tile_order", [](int num_m, int num_n, int group_m) {
    // host mirror of the device rasterisation: tile id -> (m block, n block)
    std::vector<std::pair<int, int>> out((size_t)num_m * num_n);
    for (int t = 0; t < num_m * num_n; ++t) gemm_tile_coords(t, num_m, num_n, group_m, &out[t].first, &out[t].second);
    return out;
  });

  // ---- convolutions on wgmma (conv_wgmma.cu / conv_wgrad_wgmma.cu): channels_last bf16, stride 1, 1x1 or 3x3 ------
  m.def("conv_fprop", [](at::Tensor x, at::Tensor w, int stride, int pad, int mode, int block_n, int base_offset, bool stats,
                         c10::optional<at::Tensor> debug, int kc) {
    check_cuda(x, "x"); check_cuda(w, "w");
    TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16, "conv_fprop: bf16 tensors");
    TORCH_CHECK(x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast), "conv_fprop: x must be 4-D channels_last");
    TORCH_CHECK(w.dim() == 4 && w.size(1) == x.size(1) && w.is_contiguous(at::MemoryFormat::ChannelsLast), "conv_fprop: filter must be [K, C, R, S] channels_last");
    const int R = (int)w.size(2), S = (int)w.size(3);
    TORCH_CHECK(stride == 1 && R == S && pad == (R - 1) / 2, "conv_fprop: stride 1, 'same' padding");
    c10::cuda::CUDAGuard guard(x.device());
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), K = (int)w.size(0);
    at::Tensor y = at::empty({N, K, H, W}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    ConvLaunchCfg cfg; cfg.mode = mode; cfg.block_n = block_n; cfg.set_base_offset = base_offset; cfg.kc = kc;
    if (debug.has_value()) { TORCH_CHECK(debug->scalar_type() == at::kLong && debug->numel() >= 16 && debug->is_cuda(), "debug: int64[16] cuda"); cfg.debug_counters = debug->data_ptr(); }
    at::Tensor st;
    float* stp = nullptr;
    if (stats) {
      const int groups = conv_stat_groups(N, H, W, C, K, R, S, cfg);
      TORCH_CHECK(groups > 0, "conv_fprop: no tile plan");
      st = at::empty({2, groups, K}, x.options().dtype(at::kFloat));
      stp = st.data_ptr<float>();
    }
    launch_conv_tap_gemm(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, C, K, R, S, false, cfg, stp, cur_stream());
    return std::make_tuple(y, st);
  }, py::arg("x"), py::arg("w"), py::arg("stride") = 1, py::arg("pad") = 0, py::arg("mode") = -1, py::arg("block_n") = 0,
     py::arg("base_offset") = 0, py::arg("stats") = false, py::arg("debug") = py::none(), py::arg("kc") = 0);
  // optional epilogue fusion: addend [N,C,H,W] is added to dx; (bn_x, bn_mask, bn_stats) make the epilogue also emit the partial
  // sums of the BatchNorm backward that consumes dx (returned as the second tensor, [2, G, C]; empty otherwise)
  m.def("conv_dgrad", [](at::Tensor dy, at::Tensor w, int stride, int pad, int mode, int block_n, int base_offset, int kc,
                         c10::optional<at::Tensor> addend, c10::optional<at::Tensor> bn_x, c10::optional<at::Tensor> bn_mask,
                         c10::optional<at::Tensor> bn_stats) {
    check_cuda(dy, "dy"); check_cuda(w, "w");
    TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16, "conv_dgrad: bf16 tensors");
    TORCH_CHECK(dy.dim() == 4 && dy.is_contiguous(at::MemoryFormat::ChannelsLast), "conv_dgrad: dy must be 4-D channels_last");
    TORCH_CHECK(w.dim() == 4 && w.size(0) == dy.size(1) && w.is_contiguous(at::MemoryFormat::ChannelsLast), "conv_dgrad: filter must be [K, C, R, S] channels_last");
    const int R = (int)w.size(2), S = (int)w.size(3);
    TORCH_CHECK(stride == 1 && R == S && pad == (R - 1) / 2, "conv_dgrad: stride 1, 'same' padding");
    c10::cuda::CUDAGuard guard(dy.device());
    const int N = (int)dy.size(0), K = (int)dy.size(1), H = (int)dy.size(2), W = (int)dy.size(3), C = (int)w.size(1);
    at::Tensor dx = at::empty({N, C, H, W}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
    ConvLaunchCfg cfg; cfg.mode = mode; cfg.block_n = block_n; cfg.set_base_offset = base_offset; cfg.kc = kc;
    ConvBwdFusion fuse;
    bool any = false;
    at::Tensor part;
    float* pp = nullptr;
    if (addend.has_value()) {
      TORCH_CHECK(addend->sizes() == dx.sizes() && addend->scalar_type() == at::kBFloat16 && addend->is_contiguous(at::MemoryFormat::ChannelsLast),
                  "conv_dgrad: addend must match dx (bf16, channels_last)");
      fuse.addend = addend->data_ptr(); any = true;
    }
    if (bn_x.has_value()) {
      TORCH_CHECK(bn_stats.has_value() && bn_stats->scalar_type() == at::kFloat && bn_stats->dim() == 2 && bn_stats->size(1) == C && bn_stats->size(0) >= 2,
                  "conv_dgrad: bn_stats must be fp32 [>=2, C] (rows: mean, rstd)");
      TORCH_CHECK(bn_x->sizes() == dx.sizes() && bn_x->scalar_type() == at::kBFloat16 && bn_x->is_contiguous(at::MemoryFormat::ChannelsLast),
                  "conv_dgrad: bn_x must match dx (bf16, channels_last)");
      fuse.bn_x = bn_x->data_ptr();
      if (bn_mask.has_value()) {
        TORCH_CHECK(bn_mask->scalar_type() == at::kByte && bn_mask->numel() == (int64_t)N * H * W * (C / 8), "conv_dgrad: bn_mask must be uint8 [N*H*W, C/8]");
        fuse.bn_mask = bn_mask->data_ptr();
      }
      fuse.bn_mean = bn_stats->data_ptr<float>();
      fuse.bn_rstd = bn_stats->data_ptr<float>() + C;
      // the statistics workspace of the data gradient has one row per CTA of an n-tile over the Cin columns
      const int groups = conv_stat_groups(N, H, W, K, C, R, S, cfg);
      TORCH_CHECK(groups > 0, "conv_dgrad: no tile plan");
      part = at::empty({2, groups, C}, dy.options().dtype(at::kFloat));
      pp = part.data_ptr<float>();
      any = true;
    }
    launch_conv_tap_gemm(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), N, H, W, C, K, R, S, true, cfg, pp, cur_stream(), any ? &fuse : nullptr);
    return std::make_tuple(dx, part);
  }, py::arg("dy"), py::arg("w"), py::arg("stride") = 1, py::arg("pad") = 0, py::arg("mode") = -1, py::arg("block_n") = 0,
     py::arg("base_offset") = 0, py::arg("kc") = 0, py::arg("addend") = py::none(), py::arg("bn_x") = py::none(),
     py::arg("bn_mask") = py::none(), py::arg("bn_stats") = py::none());
  m.def("conv_wgrad", [](at::Tensor dy, at::Tensor x, int ksize, int stride, int pad, int split, int tile_m, int tile_n) {
    check_cuda(dy, "dy"); check_cuda(x, "x");
    TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && x.scalar_type() == at::kBFloat16, "conv_wgrad: bf16 tensors");
    TORCH_CHECK(dy.dim() == 4 && dy.is_contiguous(at::MemoryFormat::ChannelsLast) && x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast),
                "conv_wgrad: channels_last 4-D tensors");
    TORCH_CHECK(stride == 1 && pad == (ksize - 1) / 2 && dy.size(0) == x.size(0) && dy.size(2) == x.size(2) && dy.size(3) == x.size(3),
                "conv_wgrad: stride 1, 'same' padding");
    c10::cuda::CUDAGuard guard(dy.device());
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), K = (int)dy.size(1);
    WgradCfg cfg; cfg.split = split; cfg.tile_m = tile_m; cfg.tile_n = tile_n;
    const size_t ws = conv_wgrad_workspace_floats(N, H, W, C, K, ksize, ksize, cfg);
    TORCH_CHECK(ws > 0, "conv_wgrad: unsupported geometry / tiling");
    at::Tensor work = at::empty({(int64_t)ws}, x.options().dtype(at::kFloat));
    at::Tensor dw = at::empty({K, C, ksize, ksize}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    launch_conv_wgrad(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), N, H, W, C, K, ksize, ksize, cfg, work.data_ptr<float>(), cur_stream());
    return dw;
  }, py::arg("dy"), py::arg("x"), py::arg("ksize"), py::arg("stride") = 1, py::arg("pad") = 0, py::arg("split") = 0,
     py::arg("tile_m") = 0, py::arg("tile_n") = 0);
  // strided 7x7 stem (3 -> 64 channels, stride 2, padding 3) on the wgmma tap-GEMM through an overlapping-window tensor map
  m.def("stem_conv_supported", [](int H, int W) { StemGeom g; return stem_geom(H, W, &g); });
  m.def("stem_pack_input", [](at::Tensor x) {
    check_cuda(x, "x");
    TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 4 && x.size(1) == 3 && x.is_contiguous(at::MemoryFormat::ChannelsLast),
                "stem_pack_input: x must be bf16 [N,3,H,W] channels_last");
    c10::cuda::CUDAGuard guard(x.device());
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g), "stem_pack_input: unsupported image size ", H, "x", W);
    at::Tensor xp = at::empty({N, g.Hp2, g.Wp, 8}, x.options());
    launch_stem_pack_input(x.data_ptr(), xp.data_ptr(), N, H, W, cur_stream());
    return xp;
  });
  m.def("stem_pack_weight", [](at::Tensor w) {
    check_cuda(w, "w");
    TORCH_CHECK(w.scalar_type() == at::kBFloat16 && w.dim() == 4 && w.size(0) == 64 && w.size(1) == 3 && w.size(2) == 7 && w.size(3) == 7 &&
                w.is_contiguous(at::MemoryFormat::ChannelsLast), "stem_pack_weight: w must be bf16 [64,3,7,7] channels_last");
    c10::cuda::CUDAGuard guard(w.device());
    at::Tensor w2 = at::empty({w.size(0), (int64_t)kStemK}, w.options().memory_format(at::MemoryFormat::Contiguous));
    launch_stem_pack_weight(w.data_ptr(), w2.data_ptr(), (int)w.size(0), cur_stream());
    return w2;
  });
  m.def("stem_conv_fprop_packed", [](at::Tensor xp, at::Tensor w2, int H, int W, bool stats, bool resident, bool debug) {
    check_cuda(xp, "xp"); check_cuda(w2, "w2");
    c10::cuda::CUDAGuard guard(xp.device());
    StemGeom g;
    const int N = (int)xp.size(0), K = (int)w2.size(0);
    TORCH_CHECK(stem_geom(H, W, &g) && xp.dim() == 4 && xp.size(1) == g.Hp2 && xp.size(2) == g.Wp && xp.size(3) == 8 && xp.is_contiguous() &&
                w2.dim() == 2 && w2.size(1) == kStemK && w2.is_contiguous() && xp.scalar_type() == at::kBFloat16 && w2.scalar_type() == at::kBFloat16,
                "stem_conv_fprop_packed: operands do not match the packed layout");
    at::Tensor y = at::empty({N, K, g.Ho, g.Wo}, xp.options().memory_format(at::MemoryFormat::ChannelsLast));
    at::Tensor part, dbg;
    float* sp = nullptr;
    if (stats) { part = at::empty({2, stem_stat_groups(N, H, W), K}, xp.options().dtype(at::kFloat)); sp = part.data_ptr<float>(); }
    if (debug) dbg = at::zeros({16}, xp.options().dtype(at::kLong));
    launch_stem_conv_fprop(xp.data_ptr(), w2.data_ptr(), y.data_ptr(), N, H, W, K, sp, resident, debug ? dbg.data_ptr() : nullptr, cur_stream());
    return std::make_tuple(y, part, dbg);
  }, py::arg("xp"), py::arg("w2"), py::arg("H"), py::arg("W"), py::arg("stats") = false, py::arg("resident") = true, py::arg("debug") = false);
  m.def("stem_conv_fprop", [](at::Tensor x, at::Tensor w, bool stats, bool resident) {
    check_cuda(x, "x"); check_cuda(w, "w");
    TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16, "stem_conv_fprop: bf16 tensors");
    TORCH_CHECK(x.dim() == 4 && x.size(1) == 3 && x.is_contiguous(at::MemoryFormat::ChannelsLast), "stem_conv_fprop: x must be [N,3,H,W] channels_last");
    TORCH_CHECK(w.dim() == 4 && w.size(0) == 64 && w.size(1) == 3 && w.size(2) == 7 && w.size(3) == 7 && w.is_contiguous(at::MemoryFormat::ChannelsLast),
                "stem_conv_fprop: w must be [64,3,7,7] channels_last");
    c10::cuda::CUDAGuard guard(x.device());
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3), K = (int)w.size(0);
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g), "stem_conv_fprop: unsupported image size ", H, "x", W);
    at::Tensor xp = at::empty({N, g.Hp2, g.Wp, 8}, x.options().memory_format(at::MemoryFormat::Contiguous));
    at::Tensor w2 = at::empty({K, (int64_t)kStemK}, x.options().memory_format(at::MemoryFormat::Contiguous));
    at::Tensor y = at::empty({N, K, g.Ho, g.Wo}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    at::Tensor part;
    float* sp = nullptr;
    if (stats) { part = at::empty({2, stem_stat_groups(N, H, W), K}, x.options().dtype(at::kFloat).memory_format(at::MemoryFormat::Contiguous)); sp = part.data_ptr<float>(); }
    cudaStream_t st = cur_stream();
    launch_stem_pack_input(x.data_ptr(), xp.data_ptr(), N, H, W, st);
    launch_stem_pack_weight(w.data_ptr(), w2.data_ptr(), K, st);
    launch_stem_conv_fprop(xp.data_ptr(), w2.data_ptr(), y.data_ptr(), N, H, W, K, sp, resident, nullptr, st);
    return std::make_tuple(y, part, xp);
  }, py::arg("x"), py::arg("w"), py::arg("stats") = false, py::arg("resident") = true);
  m.def("stem_conv_wgrad", [](at::Tensor dy, at::Tensor xp, int H, int W, int variant, bool unpack) {
    check_cuda(dy, "dy"); check_cuda(xp, "xp");
    TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && xp.scalar_type() == at::kBFloat16, "stem_conv_wgrad: bf16 tensors");
    TORCH_CHECK(dy.dim() == 4 && dy.is_contiguous(at::MemoryFormat::ChannelsLast) && xp.is_contiguous(), "stem_conv_wgrad: dy channels_last, xp packed");
    TORCH_CHECK(variant == 0 || variant == 1, "stem_conv_wgrad: variant 0 (dedicated kernel) or 1 (generic kernel)");
    c10::cuda::CUDAGuard guard(dy.device());
    const int N = (int)dy.size(0), K = (int)dy.size(1);
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g) && dy.size(2) == g.Ho && dy.size(3) == g.Wo && xp.dim() == 4 && xp.size(0) == N && xp.size(1) == g.Hp2 &&
                xp.size(2) == g.Wp && xp.size(3) == 8, "stem_conv_wgrad: geometry mismatch");
    const size_t ws = stem_wgrad_workspace_floats(N, H, W, K, variant);
    TORCH_CHECK(ws > 0, "stem_conv_wgrad: unsupported geometry");
    auto plain = dy.options().memory_format(at::MemoryFormat::Contiguous);
    at::Tensor work = at::empty({(int64_t)ws}, plain.dtype(at::kFloat));
    at::Tensor dw2 = variant == 0 ? at::empty({(int64_t)kStemK, K}, plain) : at::empty({K, (int64_t)kStemK}, plain);
    cudaStream_t st = cur_stream();
    launch_stem_conv_wgrad(dy.data_ptr(), xp.data_ptr(), dw2.data_ptr(), N, H, W, K, variant, work.data_ptr<float>(), st);
    if (!unpack) return dw2;
    at::Tensor dw = at::empty({K, 3, 7, 7}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
    launch_stem_unpack_wgrad(dw2.data_ptr(), dw.data_ptr(), K, variant == 0, st);
    return dw;
  }, py::arg("dy"), py::arg("xp"), py::arg("H"), py::arg("W"), py::arg("variant") = 0, py::arg("unpack") = true);
  m.def("conv_tile_plan", [](int N, int H, int W, int R, int S, int mode) {
    ConvTilePlan pl;
    const bool ok = conv_tile_plan(N, H, W, R, S, mode, &pl);
    return std::make_tuple(ok, pl.mode, pl.BH, pl.BI, pl.num_m_tiles, pl.dense_rows, pl.acc_rows, pl.a_rows);
  });

  // ---- fused BatchNorm ---------------------------------------------------------------------------
  m.def("set_bn_pdl", &set_bn_pdl);
  m.def("set_bn_two_pass", &set_bn_two_pass);
  m.def("bn_resident_error", &bn_resident_error);
  m.def("bn_workspace", [](int R, int C) {
    size_t pf = 0, cn = 0;
    bn_workspace_sizes(R, C, &pf, &cn);
    return std::make_tuple((long long)pf, (long long)cn);
  });
  m.def("bn_forward", [](at::Tensor x, c10::optional<at::Tensor> residual, at::Tensor gamma, at::Tensor beta,
                         c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                         c10::optional<at::Tensor> num_batches, double eps, double momentum, bool relu, at::Tensor partial,
                         at::Tensor counters) {
    check_cuda(x, "x");
    TORCH_CHECK(x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast), "bn_forward: x must be 4-D channels_last");
    TORCH_CHECK(gamma.scalar_type() == at::kFloat && beta.scalar_type() == at::kFloat, "bn_forward: fp32 affine parameters");
    c10::cuda::CUDAGuard guard(x.device());
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    at::Tensor y = at::empty_like(x);
    auto fopt = x.options().dtype(at::kFloat);
    at::Tensor stats = at::empty({4, C}, fopt);   // rows: save_mean, save_rstd, scale, shift
    const void* res = nullptr;
    if (residual.has_value()) {
      TORCH_CHECK(residual->sizes() == x.sizes() && residual->dtype() == x.dtype() && residual->is_contiguous(at::MemoryFormat::ChannelsLast),
                  "bn_forward: residual must match x (shape, dtype, channels_last)");
      res = residual->data_ptr();
    }
    float* st = stats.data_ptr<float>();
    at::Tensor mask = relu ? at::empty({(int64_t)R, (int64_t)(C / 8)}, x.options().dtype(at::kByte)) : at::Tensor();
    launch_bn_forward(x.data_ptr(), res, y.data_ptr(), relu ? mask.data_ptr<uint8_t>() : nullptr, dtype_of(x), R, C, gamma.data_ptr<float>(), beta.data_ptr<float>(),
                      running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
                      running_var.has_value() ? running_var->data_ptr<float>() : nullptr,
                      num_batches.has_value() ? (long long*)num_batches->data_ptr<int64_t>() : nullptr, st, st + C, st + 2 * C, st + 3 * C,
                      partial.data_ptr<float>(), (unsigned int*)counters.data_ptr<int>(), (float)eps, (float)momentum, relu, cur_stream());
    return std::make_tuple(y, stats, mask);
  });
  m.def("bn_forward_partials", [](at::Tensor x, c10::optional<at::Tensor> residual, at::Tensor gamma, at::Tensor beta,
                                  c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                                  c10::optional<at::Tensor> num_batches, double eps, double momentum, bool relu, at::Tensor partial) {
    check_cuda(x, "x"); check_cuda(partial, "partial");
    TORCH_CHECK(x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast), "bn_forward_partials: x must be 4-D channels_last");
    TORCH_CHECK(gamma.scalar_type() == at::kFloat && beta.scalar_type() == at::kFloat, "bn_forward_partials: fp32 affine parameters");
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    TORCH_CHECK(partial.scalar_type() == at::kFloat && partial.dim() == 3 && partial.size(0) == 2 && partial.size(2) == C &&
                partial.is_contiguous(), "bn_forward_partials: partial statistics must be fp32 [2, groups, C]");
    c10::cuda::CUDAGuard guard(x.device());
    at::Tensor y = at::empty_like(x);
    at::Tensor stats = at::empty({4, C}, x.options().dtype(at::kFloat));   // rows: save_mean, save_rstd, scale, shift
    const void* res = nullptr;
    if (residual.has_value()) {
      TORCH_CHECK(residual->sizes() == x.sizes() && residual->dtype() == x.dtype() && residual->is_contiguous(at::MemoryFormat::ChannelsLast),
                  "bn_forward_partials: residual must match x (shape, dtype, channels_last)");
      res = residual->data_ptr();
    }
    float* st = stats.data_ptr<float>();
    at::Tensor mask = relu ? at::empty({(int64_t)R, (int64_t)(C / 8)}, x.options().dtype(at::kByte)) : at::Tensor();
    launch_bn_forward_from_partials(x.data_ptr(), res, y.data_ptr(), relu ? mask.data_ptr<uint8_t>() : nullptr, dtype_of(x), R, C,
                                    gamma.data_ptr<float>(), beta.data_ptr<float>(),
                                    running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
                                    running_var.has_value() ? running_var->data_ptr<float>() : nullptr,
                                    num_batches.has_value() ? (long long*)num_batches->data_ptr<int64_t>() : nullptr, st, st + C, st + 2 * C,
                                    st + 3 * C, partial.data_ptr<float>(), (int)partial.size(1), (float)eps, (float)momentum, relu, cur_stream());
    return std::make_tuple(y, stats, mask);
  });
  m.def("bn_backward_partials", [](at::Tensor dy, at::Tensor x, c10::optional<at::Tensor> y, at::Tensor gamma, at::Tensor stats, bool relu,
                                   bool need_dres, at::Tensor partial) {
    check_cuda(dy, "dy"); check_cuda(partial, "partial");
    c10::cuda::CUDAGuard guard(x.device());
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    TORCH_CHECK(partial.scalar_type() == at::kFloat && partial.dim() == 3 && partial.size(0) == 2 && partial.size(2) == C && partial.is_contiguous(),
                "bn_backward_partials: partial sums must be fp32 [2, groups, C]");
    TORCH_CHECK(dy.is_contiguous(at::MemoryFormat::ChannelsLast) && dy.sizes() == x.sizes() && dy.dtype() == x.dtype(), "bn_backward_partials: dy must match x");
    at::Tensor dx = at::empty_like(x);
    at::Tensor dres = need_dres ? at::empty_like(x) : at::Tensor();
    at::Tensor dparams = at::empty({2, C}, x.options().dtype(at::kFloat));   // rows: dgamma, dbeta
    float* dp = dparams.data_ptr<float>();
    const float* st = stats.data_ptr<float>();
    TORCH_CHECK(!relu || (y.has_value() && y->scalar_type() == at::kByte), "bn_backward_partials: needs the ReLU bitmask written by bn_forward");
    launch_bn_backward_from_partials(dy.data_ptr(), x.data_ptr(), relu ? y->data_ptr() : nullptr, dx.data_ptr(), need_dres ? dres.data_ptr() : nullptr,
                                     dtype_of(x), R, C, gamma.data_ptr<float>(), st, st + C, dp, dp + C, partial.data_ptr<float>(), (int)partial.size(1),
                                     relu, cur_stream());
    return std::make_tuple(dx, dres, dparams);
  });
  m.def("bn_backward", [](at::Tensor dy, at::Tensor x, c10::optional<at::Tensor> y, at::Tensor gamma, at::Tensor stats, bool relu,
                          bool need_dres, at::Tensor partial, at::Tensor counters) {
    check_cuda(dy, "dy");
    c10::cuda::CUDAGuard guard(x.device());
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    at::Tensor dyc = dy.is_contiguous(at::MemoryFormat::ChannelsLast) ? dy : dy.contiguous(at::MemoryFormat::ChannelsLast);
    at::Tensor dx = at::empty_like(x);
    at::Tensor dres = need_dres ? at::empty_like(x) : at::Tensor();
    auto fopt = x.options().dtype(at::kFloat);
    at::Tensor dparams = at::empty({4, C}, fopt);   // rows: dgamma, dbeta, coef1, coef2
    float* dp = dparams.data_ptr<float>();
    const float* st = stats.data_ptr<float>();
    TORCH_CHECK(!relu || (y.has_value() && y->scalar_type() == at::kByte), "bn_backward: needs the ReLU bitmask written by bn_forward");
    launch_bn_backward(dyc.data_ptr(), x.data_ptr(), relu ? y->data_ptr() : nullptr, dx.data_ptr(), need_dres ? dres.data_ptr() : nullptr,
                       dtype_of(x), R, C, gamma.data_ptr<float>(), st, st + C, dp, dp + C, dp + 2 * C, partial.data_ptr<float>(),
                       (unsigned int*)counters.data_ptr<int>(), relu, cur_stream());
    return std::make_tuple(dx, dres, dparams);
  });

  // ---- max pooling ------------------------------------------------------------------------------
  m.def("maxpool3x3s2_fwd", [](at::Tensor x) {
    check_cuda(x, "x");
    TORCH_CHECK(x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast), "maxpool3x3s2_fwd: 4-D channels_last input");
    c10::cuda::CUDAGuard guard(x.device());
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3);
    const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
    at::Tensor y = at::empty({N, C, OH, OW}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    at::Tensor idx = at::empty({N, C, OH, OW}, x.options().dtype(at::kByte).memory_format(at::MemoryFormat::ChannelsLast));
    launch_maxpool3x3s2_fwd(x.data_ptr(), y.data_ptr(), idx.data_ptr<uint8_t>(), dtype_of(x), N, H, W, C, cur_stream());
    return std::make_tuple(y, idx);
  });
  m.def("maxpool3x3s2_bwd", [](at::Tensor dy, at::Tensor idx, int64_t H, int64_t W) {
    check_cuda(dy, "dy");
    c10::cuda::CUDAGuard guard(dy.device());
    at::Tensor dyc = dy.is_contiguous(at::MemoryFormat::ChannelsLast) ? dy : dy.contiguous(at::MemoryFormat::ChannelsLast);
    const int N = (int)dy.size(0), C = (int)dy.size(1);
    at::Tensor dx = at::empty({N, C, H, W}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
    launch_maxpool3x3s2_bwd(dyc.data_ptr(), idx.data_ptr<uint8_t>(), dx.data_ptr(), dtype_of(dy), N, (int)H, (int)W, C, cur_stream());
    return dx;
  });

  // ---- input pipeline ---------------------------------------------------------------------------
  m.def("normalize_to_channels_last", [](at::Tensor src, at::Tensor dst, at::Tensor mean, at::Tensor inv_std, double in_scale) {
    check_cuda(src, "src"); check_cuda(dst, "dst");
    TORCH_CHECK(src.dim() == 4 && src.is_contiguous(), "normalize_to_channels_last: src NCHW contiguous");
    // dst may carry extra (zero-filled) channels: [N, C_out >= C, H, W]
    TORCH_CHECK(dst.dim() == 4 && dst.is_contiguous(at::MemoryFormat::ChannelsLast) && dst.size(0) == src.size(0) &&
                dst.size(1) >= src.size(1) && dst.size(2) == src.size(2) && dst.size(3) == src.size(3),
                "normalize_to_channels_last: dst must be channels_last [N, C_out >= C, H, W]");
    TORCH_CHECK(mean.numel() >= src.size(1) && inv_std.numel() >= src.size(1), "normalize_to_channels_last: mean/inv_std per source channel");
    c10::cuda::CUDAGuard guard(src.device());
    launch_normalize_to_channels_last(src.data_ptr(), dtype_of(src), dst.data_ptr(), dtype_of(dst), (int)src.size(0), (int)src.size(1),
                                      (int)dst.size(1), (int)src.size(2), (int)src.size(3), mean.data_ptr<float>(), inv_std.data_ptr<float>(),
                                      (float)in_scale, cur_stream());
  });
}
