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

// ---- the argument contract: what every binding accepts -------------------------------------------------------------
// A binding first checks each tensor argument's dtype, sizes, layout and alignment (Args::operator()), then that all of
// them are CUDA tensors on one device (Args::device(), which also sets the device guard); only after that does it allocate,
// take pointers or launch.  Errors read "<binding>: <argument> must be <expected>, got <actual>".
constexpr int64_t kAny = -1;   // a size that matches any extent
// kDense: any non-overlapping dense order (the comm bindings); kStrided: any strides, for inputs the binding repairs
enum Layout { kContiguous, kChannelsLast, kDense, kStrided };
using Dtypes = std::initializer_list<at::ScalarType>;   // empty: any dtype
constexpr at::ScalarType kBF16 = at::kBFloat16, kF32 = at::kFloat, kI32 = at::kInt, kI64 = at::kLong, kU8 = at::kByte;

struct Shape {
  enum Kind { kSizes, kNumel, kMinNumel, kLastDim } kind;
  at::IntArrayRef sizes;   // kSizes: a view of the caller's list, used within the call
  int64_t n = 0;
  Shape(std::initializer_list<int64_t> s) : kind(kSizes), sizes(s) {}
  Shape(at::IntArrayRef s) : kind(kSizes), sizes(s) {}
  Shape(Kind k, int64_t v) : kind(k), n(v) {}
};
Shape numel(int64_t n) { return Shape(Shape::kNumel, n); }
Shape min_numel(int64_t n) { return Shape(Shape::kMinNumel, n); }
Shape last_dim(int64_t n) { return Shape(Shape::kLastDim, n); }   // [..., n]; kAny: any tensor of at least one dim

bool misaligned(const at::Tensor& t, int align) { return align > 1 && reinterpret_cast<uintptr_t>(t.data_ptr()) % align != 0; }

// a copy of t when its address is not a multiple of `align` bytes (the kernel's vector width)
at::Tensor aligned(const at::Tensor& t, int align) { return misaligned(t, align) ? t.clone() : t; }

// "[2, *, 4]" (kAny as *)
std::string sizes_str(at::IntArrayRef sizes) {
  std::string s = "[";
  for (size_t i = 0; i < sizes.size(); ++i) s += (i ? ", " : "") + (sizes[i] == kAny ? std::string("*") : std::to_string(sizes[i]));
  return s + "]";
}

std::string describe(const at::Tensor& t, int align = 0) {
  std::string s = std::string(c10::toString(t.scalar_type())) + " " + sizes_str(t.sizes()) +
                  (t.is_contiguous() ? " contiguous" : t.dim() == 4 && t.is_contiguous(at::MemoryFormat::ChannelsLast) ? " channels_last" : " strided");
  if (misaligned(t, align))
    s += " at an address " + std::to_string(reinterpret_cast<uintptr_t>(t.data_ptr()) % align) + " bytes past a multiple of " + std::to_string(align);
  return s;
}

class Args {
 public:
  explicit Args(const char* fn) : fn_(fn) {}
  const char* fn() const { return fn_; }

  // shape check of one tensor argument
  Args& operator()(const char* name, const at::Tensor& t, Dtypes dtypes, const Shape& shape, Layout layout = kContiguous, int align = 0) {
    const bool ok = (dtypes.size() == 0 || std::find(dtypes.begin(), dtypes.end(), t.scalar_type()) != dtypes.end()) && fits(t, shape) &&
                    laid_out(t, layout) && !misaligned(t, align);
    if (!ok) fail(name, expected(dtypes, shape, layout, align), describe(t, align));
    seen_.push_back({name, &t});
    return *this;
  }
  // an optional argument is checked only when present
  Args& operator()(const char* name, const c10::optional<at::Tensor>& t, Dtypes dtypes, const Shape& shape, Layout layout = kContiguous,
                   int align = 0) {
    return t.has_value() ? (*this)(name, *t, dtypes, shape, layout, align) : *this;
  }
  // an optional argument this call needs
  const at::Tensor& required(const char* name, const c10::optional<at::Tensor>& t) const {
    if (!t.has_value()) fail(name, "a tensor", "None");
    return *t;
  }
  // a relation between arguments that their shapes cannot state
  void expect(bool ok, const char* name, const char* what, const at::Tensor& t) const {
    if (!ok) fail(name, what, describe(t));
  }
  // A caller-owned output: when given, it is checked like an argument (contiguous, as many elements as `sizes`, opt's dtype
  // or one of `accept`) and used; otherwise device() allocates it with `sizes` and `opt`.
  void out(at::Tensor& dst, const char* name, const c10::optional<at::Tensor>& given, at::IntArrayRef sizes, const at::TensorOptions& opt,
           int align = 0, Dtypes accept = {}) {
    if (!given.has_value()) {
      pending_.push_back({&dst, c10::SmallVector<int64_t, 4>(sizes.begin(), sizes.end()), opt});
      return;
    }
    const Shape count = numel(c10::multiply_integers(sizes));
    if (accept.size() == 0) (*this)(name, *given, {opt.dtype().toScalarType()}, count, kContiguous, align);
    else (*this)(name, *given, accept, count, kContiguous, align);
    dst = *given;
  }
  // Every tensor argument is a CUDA tensor on one device: set the guard to it, then allocate the outputs not given.
  void device() {
    const at::Tensor& first = *seen_[0].second;
    for (const auto& [name, t] : seen_) {
      if (!t->is_cuda()) fail(name, "a CUDA tensor", t->device().str());
      if (t->device() != first.device()) fail(name, std::string("on ") + seen_[0].first + "'s device " + first.device().str(), t->device().str());
    }
    guard_.set_device(first.device());
    for (auto& p : pending_) *p.dst = at::empty(p.sizes, p.opt);
  }
  [[noreturn]] void fail(const char* name, const std::string& want, const std::string& got) const {
    TORCH_CHECK(false, fn_, ": ", name, " must be ", want, ", got ", got);
  }

 private:
  static bool fits(const at::Tensor& t, const Shape& s) {
    switch (s.kind) {
      case Shape::kNumel: return t.numel() == s.n;
      case Shape::kMinNumel: return t.numel() >= s.n;
      case Shape::kLastDim: return t.dim() >= 1 && (s.n == kAny || t.size(-1) == s.n);
      default:
        if (t.dim() != (int64_t)s.sizes.size()) return false;
        for (size_t i = 0; i < s.sizes.size(); ++i)
          if (s.sizes[i] != kAny && s.sizes[i] != t.size((int64_t)i)) return false;
        return true;
    }
  }
  static bool laid_out(const at::Tensor& t, Layout l) {
    switch (l) {
      case kContiguous: return t.is_contiguous();
      case kChannelsLast: return t.dim() == 4 && t.is_contiguous(at::MemoryFormat::ChannelsLast);
      case kDense: return t.is_contiguous() || t.is_non_overlapping_and_dense();
      default: return true;
    }
  }
  static std::string expected(Dtypes dtypes, const Shape& s, Layout l, int align) {
    std::string o = dtypes.size() == 0 ? "any dtype" : "";
    for (auto it = dtypes.begin(); it != dtypes.end(); ++it) o += (it == dtypes.begin() ? "" : " or ") + std::string(c10::toString(*it));
    switch (s.kind) {
      case Shape::kNumel: o += " of " + std::to_string(s.n) + " elements"; break;
      case Shape::kMinNumel: o += " of at least " + std::to_string(s.n) + " elements"; break;
      case Shape::kLastDim: o += " [..., " + (s.n == kAny ? std::string("*") : std::to_string(s.n)) + "]"; break;
      default: o += " " + sizes_str(s.sizes);
    }
    o += l == kContiguous ? " contiguous" : l == kChannelsLast ? " channels_last" : l == kDense ? " dense" : "";
    return align > 1 ? o + ", " + std::to_string(align) + "-byte aligned" : o;
  }
  struct Pending {
    at::Tensor* dst;
    c10::SmallVector<int64_t, 4> sizes;
    at::TensorOptions opt;
  };
  const char* fn_;
  c10::SmallVector<std::pair<const char*, const at::Tensor*>, 8> seen_;
  c10::SmallVector<Pending, 2> pending_;
  c10::cuda::OptionalCUDAGuard guard_;
};

// the types behind the _C.clip, _C.cross, _C.t5, _C.convnext, _C.swin, _C.swin_v2, _C.mamba, _C.mamba2, _C.whisper and _C.mae
// namespaces of static entry points
struct ClipNamespace {};
struct CrossNamespace {};
struct T5Namespace {};
struct ConvNextNamespace {};
struct SwinNamespace {};
struct SwinV2Namespace {};
struct MambaNamespace {};
struct Mamba2Namespace {};
struct WhisperNamespace {};
struct MaeNamespace {};

// An NHWC activation of the depthwise convolution: bf16 [B, H, W, C] contiguous and 16-byte aligned, B, H, W >= 1,
// 8 <= C <= 1024 with C % 8 == 0 (B is the grid's z extent).  Returns (B, H, W, C).
std::array<int, 4> dwconv_args(Args& args, const char* name, const at::Tensor& x) {
  args(name, x, {kBF16}, {kAny, kAny, kAny, kAny}, kContiguous, 16);
  const int64_t B = x.size(0), H = x.size(1), W = x.size(2), C = x.size(3);
  if (B < 1 || B > 65535 || H < 1 || W < 1 || C < 8 || C > 1024 || C % 8)
    args.fail(name, "bf16 [B, H, W, C] with 1 <= B <= 65535, H, W >= 1, 8 <= C <= 1024 and C % 8 == 0", describe(x));
  return {(int)B, (int)H, (int)W, (int)C};
}

// The window-attention geometry: table fp32 [169, heads] with 1 <= heads <= 65535, batch >= 1, height and width positive
// multiples of 7 and shifts in [0, 7), then qkv bf16 [batch * height * width, 96 heads], contiguous and 16-byte aligned.
// Returns (rows, heads).
std::array<int64_t, 2> swin_args(Args& args, const at::Tensor& qkv, const at::Tensor& table, int64_t batch, int64_t height, int64_t width,
                                 int64_t shift_y, int64_t shift_x) {
  args("table", table, {kF32}, {169, kAny});
  const int64_t heads = table.size(1);
  if (heads < 1 || heads > 65535) args.fail("table", "fp32 [169, heads] with 1 <= heads <= 65535", describe(table));
  const auto geometry = [&] { return std::to_string(batch) + " x " + std::to_string(height) + " x " + std::to_string(width) + ", shift (" +
                                     std::to_string(shift_y) + ", " + std::to_string(shift_x) + ")"; };
  if (batch < 1 || batch > 65535 || height < 7 || width < 7 || height % 7 || width % 7 || height > 65535 || width > 65535 || shift_y < 0 ||
      shift_y >= 7 || shift_x < 0 || shift_x >= 7)
    args.fail("geometry", "batch >= 1, height and width positive multiples of 7 and shifts in [0, 7)", geometry());
  const int64_t rows = batch * height * width;
  if (rows * 96 * heads >= (1ll << 31)) args.fail("geometry", "at most 2^31 qkv elements", geometry());
  args("qkv", qkv, {kBF16}, {rows, 96 * heads}, kContiguous, 16);
  return {rows, heads};
}

// Swin V2's window-attention geometry: table fp32 [225, heads] with 1 <= heads <= 65535, scale fp32 [heads], batch >= 1,
// height and width positive multiples of 8 and shifts in [0, 8), then qkv bf16 [batch * height * width, 96 heads] (head
// dim 32), contiguous and 16-byte aligned.  Returns (rows, heads).
std::array<int64_t, 2> swin_v2_args(Args& args, const at::Tensor& qkv, const at::Tensor& table, const at::Tensor& scale, int64_t batch,
                                    int64_t height, int64_t width, int64_t shift_y, int64_t shift_x) {
  args("table", table, {kF32}, {225, kAny});
  const int64_t heads = table.size(1);
  if (heads < 1 || heads > 65535) args.fail("table", "fp32 [225, heads] with 1 <= heads <= 65535", describe(table));
  args("scale", scale, {kF32}, {heads});
  const auto geometry = [&] { return std::to_string(batch) + " x " + std::to_string(height) + " x " + std::to_string(width) + ", shift (" +
                                     std::to_string(shift_y) + ", " + std::to_string(shift_x) + ")"; };
  if (batch < 1 || batch > 65535 || height < 8 || width < 8 || height % 8 || width % 8 || height > 65535 || width > 65535 || shift_y < 0 ||
      shift_y >= 8 || shift_x < 0 || shift_x >= 8)
    args.fail("geometry", "batch >= 1, height and width positive multiples of 8 and shifts in [0, 8)", geometry());
  const int64_t rows = batch * height * width;
  if (rows * 96 * heads >= (1ll << 31)) args.fail("geometry", "at most 2^31 qkv elements", geometry());
  if (qkv.dim() == 2 && qkv.size(1) != 96 * heads) args.fail("qkv", "bf16 [rows, 96 heads] (head dim 32)", describe(qkv));
  args("qkv", qkv, {kBF16}, {rows, 96 * heads}, kContiguous, 16);
  return {rows, heads};
}

// An image batch of the masked autoencoder: bf16 [B, C, H, W], contiguous or channels_last and 16-byte aligned, with
// 1 <= B <= 65535 and p a multiple of 8 that divides H and W.  Returns (B, C, H, W, N = (H / p)(W / p), channels_last).
struct MaeImages { int64_t B, C, H, W, N; bool cl; };
MaeImages mae_images(Args& args, const at::Tensor& images, int64_t patch) {
  args("images", images, {kBF16}, {kAny, kAny, kAny, kAny}, kStrided, 16);
  const bool cl = !images.is_contiguous();
  args.expect(!cl || images.is_contiguous(at::MemoryFormat::ChannelsLast), "images", "contiguous or channels_last", images);
  const int64_t B = images.size(0), C = images.size(1), H = images.size(2), W = images.size(3);
  if (B < 1 || B > 65535 || C < 1) args.fail("images", "bf16 [B, C, H, W] with 1 <= B <= 65535 and C >= 1", describe(images));
  if (patch < 8 || patch % 8 || H % patch || W % patch)
    args.fail("patch", "a multiple of 8 that divides the image's height and width", std::to_string(patch) + " for " + sizes_str(images.sizes()));
  if (images.numel() >= (1ll << 31)) args.fail("images", "fewer than 2^31 elements", describe(images));
  return {B, C, H, W, (H / patch) * (W / patch), cl};
}

// ids_restore int32 [B, N] (1 <= N <= 1024) and 0 <= keep <= N
void mae_ids(Args& args, const char* name, const at::Tensor& ids, int64_t B, int64_t N, int64_t keep) {
  args(name, ids, {kI32}, {B, N});
  if (N < 1 || N > 1024) args.fail(name, "int32 [B, N] with 1 <= N <= 1024", describe(ids));
  if (keep < 0 || keep > N) args.fail("keep", "in [0, N] = [0, " + std::to_string(N) + "]", std::to_string(keep));
}

// The per-image attention's qkv bf16 [T, 96 heads] (head dim 32), contiguous and 16-byte aligned with 1 <= heads <= 65535 and
// fewer than 2^31 elements, and images of `tokens` rows: batch >= 1, 1 <= tokens <= 256, batch * tokens <= T.  Returns (T, heads).
std::array<int64_t, 2> mae_attention_args(Args& args, const at::Tensor& qkv, int64_t batch, int64_t tokens) {
  args("qkv", qkv, {kBF16}, {kAny, kAny}, kContiguous, 16);
  const int64_t T = qkv.size(0), heads = qkv.size(1) / 96;
  if (qkv.size(1) % 96 || heads < 1 || heads > 65535 || T * qkv.size(1) >= (1ll << 31))
    args.fail("qkv", "bf16 [T, 96 heads] (head dim 32) with 1 <= heads <= 65535 and fewer than 2^31 elements", describe(qkv));
  if (batch < 1 || tokens < 1 || tokens > 256 || batch * tokens > T)
    args.fail("geometry", "batch >= 1, 1 <= tokens <= 256 and batch * tokens <= T = " + std::to_string(T),
              std::to_string(batch) + " x " + std::to_string(tokens));
  return {T, heads};
}

// The reconstruction loss's pred bf16 [Td, C p^2] (C p^2 <= 768, p from its width and the images' C), its images (as
// mae_images), ids_restore int32 [B, N], 0 <= keep < N and Td >= B (N + 1).  Returns the images' geometry and p.
std::pair<MaeImages, int64_t> mae_loss_args(Args& args, const at::Tensor& pred, const at::Tensor& images, const at::Tensor& ids_restore,
                                            int64_t keep) {
  args("pred", pred, {kBF16}, {kAny, kAny}, kContiguous, 16);
  const int64_t C = images.dim() == 4 ? images.size(1) : 1, P = pred.size(1);
  const int64_t patch = C > 0 && P % C == 0 ? (int64_t)std::lround(std::sqrt((double)(P / C))) : 0;
  if (P > 768 || patch * patch * C != P) args.fail("pred", "bf16 [T, C p^2] with C p^2 <= 768", describe(pred));
  const MaeImages im = mae_images(args, images, patch);
  mae_ids(args, "ids_restore", ids_restore, im.B, im.N, keep);
  if (keep >= im.N) args.fail("keep", "below N = " + std::to_string(im.N), std::to_string(keep));
  if (pred.size(0) < im.B * (im.N + 1)) args.fail("pred", "at least B (N + 1) = " + std::to_string(im.B * (im.N + 1)) + " rows", describe(pred));
  return {im, patch};
}

// Mamba's token rows: bounds int32 [B, S, 2] contiguous and 8-byte aligned (the kernels read int2) with 1 <= B <= 65535, then
// xz bf16 [B S, 2E] contiguous and 16-byte aligned with E a positive multiple of 8 and B S 2E < 2^31.  Returns (B, S, E).
std::array<int64_t, 3> mamba_args(Args& args, const at::Tensor& bounds, const at::Tensor& xz) {
  args("bounds", bounds, {kI32}, {kAny, kAny, 2}, kContiguous, 8);
  const int64_t B = bounds.size(0), S = bounds.size(1);
  if (B < 1 || B > 65535 || S < 1) args.fail("bounds", "int32 [B, S, 2] with 1 <= B <= 65535 and S >= 1", describe(bounds));
  args("xz", xz, {kBF16}, {B * S, kAny}, kContiguous, 16);
  const int64_t E = xz.size(1) / 2;
  if (xz.size(1) % 16 || E < 8 || B * S * 2 * E >= (1ll << 31))
    args.fail("xz", "bf16 [B S, 2E] with E a positive multiple of 8 and fewer than 2^31 elements", describe(xz));
  return {B, S, E};
}

// the selective scan's inputs after bounds and xz: u and draw bf16 [T, E], xbc bf16 [T, R + 32] (R >= 0), A_log fp32 [E, 16],
// D and dt_bias fp32 [E], all contiguous.  Returns R.
int64_t mamba_scan_args(Args& args, int64_t T, int64_t E, const at::Tensor& u, const at::Tensor& draw, const at::Tensor& xbc,
                        const at::Tensor& A_log, const at::Tensor& D, const at::Tensor& dt_bias) {
  args("u", u, {kBF16}, {T, E})("draw", draw, {kBF16}, {T, E})("xbc", xbc, {kBF16}, {T, kAny});
  if (xbc.size(1) < 32) args.fail("xbc", "bf16 [T, R + 32] with R >= 0 (dt | B | C)", describe(xbc));
  args("A_log", A_log, {kF32}, {E, 16})("D", D, {kF32}, {E})("dt_bias", dt_bias, {kF32}, {E});
  return xbc.size(1) - 32;
}

// A bf16 row view [rows, cols] read in place through its row pitch (Mamba-2's column windows of in_proj's output): unit
// column stride, a row stride >= cols that is a multiple of 8 elements, 16-byte aligned.  Returns the pitch.
int64_t row_view(Args& args, const char* name, const at::Tensor& t, int64_t rows, int64_t cols) {
  args(name, t, {kBF16}, {rows, cols}, kStrided, 16);
  if (t.stride(1) != 1 || t.stride(0) < cols || t.stride(0) % 8 || t.size(0) * t.stride(0) >= (1ll << 31))
    args.fail(name, "a bf16 [" + std::to_string(rows) + ", " + std::to_string(cols) +
                        "] row view with unit column stride and a row pitch >= the columns, a multiple of 8, under 2^31 elements in all",
              describe(t) + " with strides (" + std::to_string(t.stride(0)) + ", " + std::to_string(t.stride(1)) + ")");
  return t.stride(0);
}

// Mamba-2's bounds int32 [B, S, 2] contiguous and 8-byte aligned with 1 <= B <= 65535, S >= 1.  Returns (B, S).
std::array<int64_t, 2> mamba2_bounds(Args& args, const at::Tensor& bounds) {
  args("bounds", bounds, {kI32}, {kAny, kAny, 2}, kContiguous, 8);
  const int64_t B = bounds.size(0), S = bounds.size(1);
  if (B < 1 || B > 65535 || S < 1) args.fail("bounds", "int32 [B, S, 2] with 1 <= B <= 65535 and S >= 1", describe(bounds));
  return {B, S};
}

// the SSD's inputs: xbc bf16 [B S, 64 H + 256] contiguous, dt a bf16 [B S, H] row view, H a positive multiple of 8 (so E and
// the dt columns stay 16-byte aligned), A_log / D / dt_bias fp32 [H].  Returns (B, S, H, dt pitch).
std::array<int64_t, 4> ssd_args(Args& args, const at::Tensor& xbc, const at::Tensor& dt, const at::Tensor& A_log, const at::Tensor& D,
                                const at::Tensor& dt_bias, const at::Tensor& bounds) {
  const auto [B, S] = mamba2_bounds(args, bounds);
  args("xbc", xbc, {kBF16}, {B * S, kAny}, kContiguous, 16);
  const int64_t H = (xbc.size(1) - 256) / 64;
  if (xbc.size(1) < 256 + 64 * 8 || (xbc.size(1) - 256) % 512 || B * S * xbc.size(1) >= (1ll << 31))
    args.fail("xbc", "bf16 [B S, 64 H + 256] (x | B | C, head dim 64, state 128) with H a positive multiple of 8 and fewer than 2^31 elements",
              describe(xbc));
  const int64_t dtp = row_view(args, "dt", dt, B * S, H);
  args("A_log", A_log, {kF32}, {H})("D", D, {kF32}, {H})("dt_bias", dt_bias, {kF32}, {H});
  return {B, S, H, dtp};
}

// Whisper's stem rows: frames F even and >= 2, rows S >= F / 2, then t bf16 [B * n, cols] contiguous and 16-byte aligned
// with n = F (h1, dh1) or S (P2, dP2), 1 <= B, cols = d or 3 d with d a positive multiple of 8, and fewer than 2^31
// elements on either side.  Returns (B, d).
std::array<int64_t, 2> stem_rows(Args& args, const char* name, const at::Tensor& t, int64_t frames, int64_t rows, bool patches) {
  if (frames < 2 || frames % 2 || rows < frames / 2 || rows > (1ll << 24))
    args.fail("frames", "even and >= 2, with rows >= frames / 2", "frames " + std::to_string(frames) + ", rows " + std::to_string(rows));
  args(name, t, {kBF16}, {kAny, kAny}, kContiguous, 16);
  const int64_t n = patches ? rows : frames, cols = t.size(1), d = patches ? cols / 3 : cols;
  const int64_t B = t.size(0) / n;
  if (t.size(0) < n || t.size(0) % n || d < 8 || d % 8 || (patches && cols % 3) || B * rows * 3 * d >= (1ll << 31) ||
      B * frames * 3 * d >= (1ll << 31))
    args.fail(name, std::string("bf16 [B * ") + (patches ? "rows, 3 d]" : "frames, d]") +
                        " with B >= 1, d a positive multiple of 8 and fewer than 2^31 elements",
              describe(t));
  return {B, d};
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
  Args args("allreduce_tensors");
  args("tensors", tensors[0], {kF32, kBF16}, min_numel(0), kDense);
  for (const at::Tensor& t : tensors) args("tensors", t, {tensors[0].scalar_type()}, min_numel(0), kDense);
  args("sq_partials", sq_partials, {kF32}, min_numel(0));
  args.device();
  const DType in_dt = dtype_of(tensors[0]);
  const DType wire_dt = wire == "fp32" ? DType::F32 : DType::BF16;
  BucketTable tab;
  uint32_t off = 0;
  tab.count = (int)tensors.size();
  for (int k = 0; k < tab.count; ++k) {
    const at::Tensor& t = tensors[k];
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
  if (tensors.empty()) return 0;
  Args args("broadcast_tensors");
  for (const at::Tensor& t : tensors) args("tensors", t, {}, min_numel(0), kDense);
  args.device();
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

// peer_pull / peer_push: `bytes` between the arena and one dense tensor, which must hold them
void peer_copy_args(Args& args, const char* name, const at::Tensor& t, size_t bytes) {
  args(name, t, {}, min_numel(0), kDense);
  if (bytes > (size_t)t.numel() * t.element_size())
    args.fail("bytes", std::string("at most ") + name + "'s " + std::to_string(t.numel() * t.element_size()), std::to_string(bytes));
  args.device();
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

// ---- attention (attention.cu): one body per direction for every mask and head layout ------------------------------
// qkv bf16 [B*S, (heads + 2*kv_heads)*hd], query | key | value column blocks (kv_heads == heads: multi-head), S % 128 == 0;
// the mask is seq_lens int32 [B] (key padding) or bounds int32 [B, S, 2] (documents: packed, causal, grouped-query, head
// dim 128).  The multi-head launchers, which take no kv_heads, are adapted by captureless lambdas at their m.def.
using AttnFwd = void (*)(const void*, const int*, int, int, int, int, void*, float*, cudaStream_t);
using AttnBwd = void (*)(const void*, const void*, const void*, const float*, const int*, int, int, int, int, float*, void*, cudaStream_t);
enum class Mask { kSeqLens, kBounds };

// checks qkv and the mask; returns (B, S)
std::pair<int, int> attn_args(Args& args, const at::Tensor& qkv, const at::Tensor& mask, Mask kind, int heads, int kv_heads, int hd) {
  TORCH_CHECK(heads >= 1 && kv_heads >= 1 && heads % kv_heads == 0, args.fn(), ": kv_heads (", kv_heads, ") must divide heads (", heads, ")");
  const int64_t cols = (int64_t)(heads + 2 * kv_heads) * hd;
  if (kind == Mask::kSeqLens) {
    args("seq_lens", mask, {kI32}, {kAny})("qkv", qkv, {kBF16}, {kAny, cols}, kContiguous, 16);
    const int64_t B = mask.size(0);
    args.expect(B >= 1 && qkv.size(0) % B == 0, "seq_lens", "int32 [B] with B >= 1 dividing qkv's rows", mask);
    return {(int)B, (int)(qkv.size(0) / B)};
  }
  args("bounds", mask, {kI32}, {kAny, kAny, 2}, kContiguous, 8);
  args.expect(mask.numel() >= 2, "bounds", "int32 [B, S, 2] with B, S >= 1", mask);
  args("qkv", qkv, {kBF16}, {mask.size(0) * mask.size(1), cols}, kContiguous, 16);
  return {(int)mask.size(0), (int)mask.size(1)};
}

// (o bf16 [B*S, heads*hd], lse fp32 [B, heads, S]); optional caller-owned outputs
std::tuple<at::Tensor, at::Tensor> attn_fwd(const char* fn, AttnFwd launch, int hd, Mask kind, const at::Tensor& qkv, const at::Tensor& mask,
                                            int heads, int kv_heads, const c10::optional<at::Tensor>& o_out,
                                            const c10::optional<at::Tensor>& lse_out) {
  Args args(fn);
  const auto [B, S] = attn_args(args, qkv, mask, kind, heads, kv_heads, hd);
  at::Tensor o, lse;
  args.out(o, "o", o_out, {qkv.size(0), (int64_t)heads * hd}, qkv.options(), 16);
  args.out(lse, "lse", lse_out, {B, heads, S}, qkv.options().dtype(kF32), 8);
  args.device();
  launch(qkv.data_ptr(), mask.data_ptr<int>(), B, S, heads, kv_heads, o.data_ptr(), lse.data_ptr<float>(), cur_stream());
  return std::make_tuple(o, lse);
}

// dqkv shaped like qkv: the query / key / value column blocks hold dQ / dK / dV
at::Tensor attn_bwd(const char* fn, AttnBwd launch, int hd, Mask kind, const at::Tensor& dout, const at::Tensor& qkv, const at::Tensor& o,
                    const at::Tensor& lse, const at::Tensor& mask, int heads, int kv_heads, const c10::optional<at::Tensor>& dqkv_out) {
  Args args(fn);
  const auto [B, S] = attn_args(args, qkv, mask, kind, heads, kv_heads, hd);
  args("dout", dout, {kBF16}, numel(qkv.size(0) * heads * hd), kContiguous, 16);
  args("o", o, {kBF16}, numel(qkv.size(0) * heads * hd), kContiguous, 16);
  args("lse", lse, {kF32}, numel((int64_t)B * heads * S), kContiguous, 8);
  at::Tensor dqkv;
  args.out(dqkv, "dqkv", dqkv_out, qkv.sizes(), qkv.options(), 4);
  args.device();
  at::Tensor dsum = at::empty({B, heads, S}, qkv.options().dtype(kF32));
  launch(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), mask.data_ptr<int>(), B, S, heads, kv_heads,
         dsum.data_ptr<float>(), dqkv.data_ptr(), cur_stream());
  return dqkv;
}

// checks q, kv and q_bounds of a cross-attention binding (heads * 64 columns per query row); returns (B, Sq, Sk)
std::tuple<int, int, int> cross_args(Args& args, const at::Tensor& q, const at::Tensor& kv, const at::Tensor& q_bounds, int heads) {
  if (heads < 1) args.fail("heads", ">= 1", std::to_string(heads));
  args("q_bounds", q_bounds, {kI32}, {kAny, kAny, 2}, kContiguous, 8);
  args.expect(q_bounds.numel() >= 2, "q_bounds", "int32 [B, Sq, 2] with B, Sq >= 1", q_bounds);
  const int64_t B = q_bounds.size(0), Sq = q_bounds.size(1), hidden = (int64_t)heads * 64;
  args("q", q, {kBF16}, {B * Sq, hidden}, kContiguous, 16)("kv", kv, {kBF16}, {kAny, 2 * hidden}, kContiguous, 16);
  args.expect(kv.size(0) % B == 0 && kv.size(0) >= B, "kv", "bf16 [B*Sk, 2*heads*64] with Sk >= 1", kv);
  return std::make_tuple((int)B, (int)Sq, (int)(kv.size(0) / B));
}

// checks qkv, bounds and table of a relative-bias attention binding (multi-head, head dim 64); returns (B, S)
std::pair<int, int> relative_args(Args& args, const at::Tensor& qkv, const at::Tensor& bounds, const at::Tensor& table, int heads) {
  if (heads < 1) args.fail("heads", ">= 1", std::to_string(heads));
  const auto [B, S] = attn_args(args, qkv, bounds, Mask::kBounds, heads, heads, 64);
  args("table", table, {kF32}, {heads, 257});
  return {B, S};
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
    auto dt = dtype_code == 1 ? kBF16 : dtype_code == 2 ? kU8 : kF32;
    auto opts = at::TensorOptions().dtype(dt).device(at::kCUDA, a.device());
    return at::from_blob(a.local() + offset, {numel}, [](void*) {}, opts);
  });
  m.def("allreduce_symmetric", [](PeerArena& a, size_t buf_off, int64_t numel, int dtype_code, int algo, int blocks, double scale,
                                  int pad_set, double timeout_s) {
    c10::cuda::CUDAGuard guard((c10::DeviceIndex)a.device());
    CommCtx ctx = make_ctx(a, (size_t)pad_set * kPadSetBytes, timeout_s);
    if (algo == kAlgoAuto) algo = a.has_multicast() ? kAlgoNvls : kAlgoTwoShot;
    launch_symmetric_allreduce(ctx, buf_off, (size_t)numel, (DType)dtype_code, algo, blocks, (float)scale, cur_stream());
  });
  m.def("broadcast_tensors", &broadcast_tensors, py::arg("arena"), py::arg("tensors"), py::arg("src") = 0, py::arg("stage_off"),
        py::arg("stage_bytes"), py::arg("use_mc") = false, py::arg("blocks") = 32, py::arg("pad_set") = 1,
        py::arg("timeout_s") = 30.0);
  m.def("peer_pull", [](PeerArena& a, int peer, size_t src_off, at::Tensor dst, size_t bytes, int blocks) {
    Args args("peer_pull");
    peer_copy_args(args, "dst", dst, bytes);
    launch_peer_pull(make_ctx(a, 0, 30.0), peer, src_off, dst.data_ptr(), bytes, blocks, cur_stream());
  });
  m.def("peer_push", [](PeerArena& a, int peer, size_t dst_off, at::Tensor src, size_t bytes, int blocks) {
    Args args("peer_push");
    peer_copy_args(args, "src", src, bytes);
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
    Args args("clip_coef");
    args("partials", partials, {kF32}, min_numel(n))("coef", coef, {kF32}, min_numel(1))("norm", norm, {kF32}, min_numel(1));
    args.device();
    launch_clip_coef(partials.data_ptr<float>(), n, (float)max_norm, (float)grad_scale, coef.data_ptr<float>(),
                     norm.data_ptr<float>(), cur_stream());
  });

  // ---- losses -----------------------------------------------------------------------------------
  m.def("mse_fwd_bwd", [](at::Tensor out, at::Tensor target, double gscale) {
    Args args("mse_fwd_bwd");
    args("out", out, {kF32, kBF16}, min_numel(0))("target", target, {out.scalar_type()}, out.sizes());
    args.device();
    const size_t n = (size_t)out.numel();
    const int blocks = mse_blocks(n);
    at::Tensor loss = at::empty({}, out.options().dtype(kF32));
    at::Tensor dout = at::empty_like(out);
    at::Tensor scratch = at::zeros({blocks + 1}, out.options().dtype(kF32));
    launch_mse_fwd_bwd(out.data_ptr(), target.data_ptr(), dtype_of(out), n, (float)gscale, loss.data_ptr<float>(), dout.data_ptr(),
                       scratch.data_ptr<float>(), blocks, cur_stream());
    return std::make_tuple(loss, dout);
  });
  m.def("xent_fwd_bwd", [](at::Tensor logits, at::Tensor targets, long long ignore_index, double gscale) {
    Args args("xent_fwd_bwd");
    args("logits", logits, {kF32, kBF16}, {kAny, kAny})("targets", targets, {kI64}, numel(logits.size(0)));
    args.device();
    const int rows = (int)logits.size(0), cols = (int)logits.size(1);
    at::Tensor loss = at::empty({}, logits.options().dtype(kF32));
    at::Tensor row_loss = at::empty({rows + 1}, logits.options().dtype(kF32));
    at::Tensor dlogits = at::empty_like(logits);
    launch_xent_fwd_bwd(logits.data_ptr(), (const long long*)targets.data_ptr<int64_t>(), dtype_of(logits), rows, cols, ignore_index,
                        (float)gscale, row_loss.data_ptr<float>(), loss.data_ptr<float>(), dlogits.data_ptr(), cur_stream());
    return std::make_tuple(loss, dlogits);
  });
  // Fused LM-head cross-entropy: mean over non-ignored rows of cross_entropy(hidden [N,H] . weight [V,H]^T + bias [V]) without
  // the [N, V] logits.  Forward -> (loss fp32 [], lse fp32 [N], row_loss fp32 [N+1], row_loss[N] = non-ignored rows).
  // rows (optional): int32 [1] device count of the leading rows that carry labels (compact_rows' count).  Only the 128-row tiles
  // below it are computed; the rows at or past it must be ignored ones, and get lse = row_loss = 0 (dh: zeros).
  auto lm_args = [](Args& args, const at::Tensor& hidden, const at::Tensor& weight, const at::Tensor& targets,
                    const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& rows) {
    args("hidden", hidden, {kBF16}, {kAny, kAny});
    args.expect(hidden.size(0) >= 1 && hidden.size(1) % 8 == 0, "hidden", "[N, H] with N >= 1 and H % 8 == 0 (16-byte rows)", hidden);
    args("weight", weight, {kBF16}, {kAny, hidden.size(1)});
    args.expect(weight.size(0) % 8 == 0, "weight", "[V, H] with V % 8 == 0", weight);
    args("targets", targets, {kI64}, numel(hidden.size(0)))("bias", bias, {kBF16}, numel(weight.size(0)))("rows", rows, {kI32}, numel(1));
  };
  m.def("lm_loss_fwd", [lm_args](at::Tensor hidden, at::Tensor weight, at::Tensor targets, c10::optional<at::Tensor> bias,
                                 long long ignore_index, c10::optional<at::Tensor> lse_out, c10::optional<at::Tensor> row_loss_out,
                                 c10::optional<at::Tensor> rows) {
    Args args("lm_loss_fwd");
    lm_args(args, hidden, weight, targets, bias, rows);
    const int N = (int)hidden.size(0), H = (int)hidden.size(1), V = (int)weight.size(0), tiles = (V + 127) / 128;
    const auto f32 = hidden.options().dtype(kF32);
    at::Tensor lse, row_loss;
    args.out(lse, "lse_out", lse_out, {N}, f32);
    args.out(row_loss, "row_loss_out", row_loss_out, {N + 1}, f32);
    args.device();
    const int* bound = rows.has_value() ? rows->data_ptr<int>() : nullptr;
    at::Tensor loss = at::empty({}, f32);
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
  m.def("lm_loss_bwd", [lm_args](at::Tensor hidden, at::Tensor weight, at::Tensor targets, c10::optional<at::Tensor> bias,
                                 at::Tensor lse, at::Tensor row_loss, at::Tensor gscale, long long ignore_index, int slice,
                                 bool need_dh, bool need_dweight, c10::optional<at::Tensor> dh_out,
                                 c10::optional<at::Tensor> dweight_out, c10::optional<at::Tensor> rows, bool need_dbias) {
    Args args("lm_loss_bwd");
    lm_args(args, hidden, weight, targets, bias, rows);
    if (need_dbias) args.required("bias", bias);
    const int N = (int)hidden.size(0), H = (int)hidden.size(1), V = (int)weight.size(0);
    TORCH_CHECK(slice >= 128 && slice % 128 == 0, "lm_loss_bwd: slice must be a positive multiple of 128, got ", slice);
    args("lse", lse, {kF32}, numel(N))("row_loss", row_loss, {kF32}, numel(N + 1))("gscale", gscale, {kF32}, numel(1));
    const auto bf16 = hidden.options();
    at::Tensor dh, dweight, dbias, dh32, colsum;
    if (need_dh) args.out(dh, "dh_out", dh_out, {N, H}, bf16);
    if (need_dweight) args.out(dweight, "dweight_out", dweight_out, {V, H}, bf16);
    args.device();
    const int* bound = rows.has_value() ? rows->data_ptr<int>() : nullptr;
    // row-bounded: the data-gradient GEMM skips the tiles past the count, whose rows must read as zeros
    if (need_dh) dh32 = bound != nullptr ? at::zeros({N, H}, bf16.dtype(kF32)) : at::empty({N, H}, bf16.dtype(kF32));
    if (need_dbias) dbias = at::empty({V}, bf16);
    if (!need_dh && !need_dweight && !need_dbias) return std::make_tuple(dh, dweight, dbias);
    const int width = slice < V ? slice : V;
    at::Tensor dlogits = at::empty({(int64_t)N * width}, bf16);
    if (need_dbias) colsum = at::empty({(int64_t)column_sum_workspace(N, width)}, bf16.dtype(kF32));
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
    Args args("compact_rows");
    args("targets", targets, {kI64}, {kAny});
    args.expect(targets.numel() >= 1 && targets.numel() < (1LL << 31), "targets", "int64 [T] with 1 <= T < 2^31", targets);
    TORCH_CHECK(vocab >= 1, "compact_rows: vocab must be positive, got ", vocab);
    args.device();
    const int T = (int)targets.numel();
    const auto i32 = targets.options().dtype(kI32);
    at::Tensor index = at::empty({T}, i32), count = at::empty({1}, i32), out = at::empty_like(targets);
    at::Tensor work = at::empty({2 * compact_chunks(T)}, i32);
    launch_compact_rows((const long long*)targets.data_ptr<int64_t>(), T, ignore_index, vocab, work.data_ptr<int>(), index.data_ptr<int>(),
                        count.data_ptr<int>(), (long long*)out.data_ptr<int64_t>(), cur_stream());
    return std::make_tuple(index, count, out);
  }, py::arg("targets"), py::arg("ignore_index"), py::arg("vocab"));
  // x bf16 [T, H] (H % 8 == 0), index int32 [T] and count int32 [1] from compact_rows
  auto rows_args = [](Args& args, const char* name, const at::Tensor& x, const at::Tensor& index, const at::Tensor& count) {
    args(name, x, {kBF16}, {kAny, kAny});
    args.expect(x.size(1) % 8 == 0, name, "bf16 [T, H] with H % 8 == 0", x);
    args("index", index, {kI32}, numel(x.size(0)))("count", count, {kI32}, numel(1));
    args.device();
  };
  // gather_rows(x [T, H], index, count): out[r] = x[index[r]] for r < count, zero rows from count on
  m.def("gather_rows", [rows_args](at::Tensor x, at::Tensor index, at::Tensor count) {
    Args args("gather_rows");
    rows_args(args, "x", x, index, count);
    at::Tensor out = at::empty_like(x);
    launch_gather_rows(x.data_ptr(), index.data_ptr<int>(), count.data_ptr<int>(), (int)x.size(0), (int)x.size(1), out.data_ptr(), cur_stream());
    return out;
  }, py::arg("x"), py::arg("index"), py::arg("count"));
  // scatter_rows(dy [T, H], index, count): dx[index[r]] = dy[r] for r < count, every other row of dx zero
  m.def("scatter_rows", [rows_args](at::Tensor dy, at::Tensor index, at::Tensor count) {
    Args args("scatter_rows");
    rows_args(args, "dy", dy, index, count);
    at::Tensor dx = at::empty_like(dy);
    launch_scatter_rows(dy.data_ptr(), index.data_ptr<int>(), count.data_ptr<int>(), (int)dy.size(0), (int)dy.size(1), dx.data_ptr(),
                        cur_stream());
    return dx;
  }, py::arg("dy"), py::arg("index"), py::arg("count"));

  // tanh = false: the erf form; true: the tanh approximation
  m.def("gelu_fwd", [](at::Tensor pre, bool tanh) {
    Args args("gelu_fwd");
    args("pre", pre, {kF32, kBF16}, min_numel(0));
    args.device();
    at::Tensor out = at::empty_like(pre);
    launch_gelu(pre.data_ptr(), nullptr, out.data_ptr(), dtype_of(pre), (size_t)pre.numel(), false, cur_stream(),
                tanh ? GeluForm::kTanh : GeluForm::kErf);
    return out;
  }, py::arg("pre"), py::arg("tanh") = false);
  m.def("gelu_bwd", [](at::Tensor dy, at::Tensor pre, bool tanh) {
    Args args("gelu_bwd");
    args("pre", pre, {kF32, kBF16}, min_numel(0))("dy", dy, {pre.scalar_type()}, numel(pre.numel()));
    args.device();
    at::Tensor out = at::empty_like(pre);
    launch_gelu(pre.data_ptr(), dy.data_ptr(), out.data_ptr(), dtype_of(pre), (size_t)pre.numel(), true, cur_stream(),
                tanh ? GeluForm::kTanh : GeluForm::kErf);
    return out;
  }, py::arg("dy"), py::arg("pre"), py::arg("tanh") = false);

  // ---- layer norm -------------------------------------------------------------------------------
  m.def("layernorm_fwd", [](at::Tensor x, at::Tensor gamma, at::Tensor beta, double eps) {
    Args args("layernorm_fwd");
    args("x", x, {kF32, kBF16}, last_dim(kAny))("gamma", gamma, {x.scalar_type()}, numel(x.size(-1)));
    args("beta", beta, {x.scalar_type()}, numel(x.size(-1)));
    args.device();
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    at::Tensor y = at::empty_like(x);
    at::Tensor mean = at::empty({rows}, x.options().dtype(kF32));
    at::Tensor rstd = at::empty({rows}, x.options().dtype(kF32));
    launch_layernorm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), dtype_of(x), rows, cols, (float)eps, y.data_ptr(),
                         mean.data_ptr<float>(), rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, mean, rstd);
  });
  m.def("layernorm_bwd", [](at::Tensor dy, at::Tensor x, at::Tensor gamma, at::Tensor mean, at::Tensor rstd) {
    Args args("layernorm_bwd");
    args("x", x, {kF32, kBF16}, last_dim(kAny));
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    args("dy", dy, {x.scalar_type()}, x.sizes())("gamma", gamma, {x.scalar_type()}, numel(cols))("mean", mean, {kF32}, numel(rows));
    args("rstd", rstd, {kF32}, numel(rows));
    args.device();
    const int parts = layernorm_partial_rows(rows);
    at::Tensor dx = at::empty_like(x);
    at::Tensor dgp = at::empty({parts, cols}, x.options().dtype(kF32));
    at::Tensor dbp = at::empty({parts, cols}, x.options().dtype(kF32));
    at::Tensor dgamma = at::empty_like(gamma);
    at::Tensor dbeta = at::empty_like(gamma);
    launch_layernorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(), dtype_of(x),
                         rows, cols, dx.data_ptr(), dgp.data_ptr<float>(), dbp.data_ptr<float>(), parts, dgamma.data_ptr(),
                         dbeta.data_ptr(), cur_stream());
    return std::make_tuple(dx, dgamma, dbeta);
  });

  // ---- linears ----------------------------------------------------------------------------------
  m.def("small_linear_fwd", [](at::Tensor x, at::Tensor w, c10::optional<at::Tensor> b, bool relu) {
    Args args("small_linear_fwd");
    args("x", x, {kF32}, last_dim(kAny))("w", w, {kF32}, {kAny, x.size(-1)})("b", b, {kF32}, numel(w.size(0)));
    args.device();
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
    Args args("small_linear_bwd");
    args("x", x, {kF32}, last_dim(kAny))("w", w, {kF32}, {kAny, x.size(-1)});
    const int K = (int)x.size(-1), N = (int)w.size(0);
    const int M = (int)(x.numel() / K);
    args("y", y, {kF32}, numel((int64_t)M * N))("dy", dy, {kF32}, numel((int64_t)M * N), kStrided);
    args.device();
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
    Args args("gemm_nt");
    args("a", a, {kBF16}, {kAny, kAny})("b", b, {kBF16}, {kAny, a.size(1)});
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    args("bias", bias, {kBF16}, numel(N));
    at::Tensor d;
    args.out(d, "out", out, {M, N}, a.options(), 0, {kBF16, kF32});
    args.device();
    launch_gemm_nt_bf16(a.data_ptr(), b.data_ptr(), d.data_ptr(), bias.has_value() ? bias->data_ptr() : nullptr, M, N, K, epilogue,
                        dtype_of(d), cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("epilogue") = 0, py::arg("out") = py::none());
  // general form: a_mn=false -> a is [M,K]; true -> a is stored [K,M].  b_mn=false -> b is [N,K]; true -> stored [K,N].
  // A given fp32 `out` with out_fp32 is accumulated into.
  m.def("gemm", [](at::Tensor a, at::Tensor b, c10::optional<at::Tensor> bias, bool a_mn, bool b_mn, int epilogue, bool out_fp32,
                   c10::optional<at::Tensor> out) {
    Args args("gemm");
    args("a", a, {kBF16}, {kAny, kAny});
    const int M = (int)(a_mn ? a.size(1) : a.size(0)), K = (int)(a_mn ? a.size(0) : a.size(1));
    if (b_mn) args("b", b, {kBF16}, {K, kAny});
    else args("b", b, {kBF16}, {kAny, K});
    const int N = (int)(b_mn ? b.size(1) : b.size(0));
    args("bias", bias, {kBF16}, numel(N));
    at::Tensor d;
    args.out(d, "out", out, {M, N}, a.options().dtype(out_fp32 ? kF32 : kBF16), 0, {kBF16, kF32});
    args.device();
    const bool accumulate = out.has_value() && out_fp32 && d.scalar_type() == kF32;
    launch_gemm_bf16(a.data_ptr(), b.data_ptr(), d.data_ptr(), bias.has_value() ? bias->data_ptr() : nullptr, M, N, K, a_mn, b_mn, epilogue,
                     dtype_of(d), accumulate, cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("a_mn") = false, py::arg("b_mn") = false,
     py::arg("epilogue") = 0, py::arg("out_fp32") = false, py::arg("out") = py::none());
  // forward GEMM (a [M,K], b [N,K]) that also returns per-32-row partial column statistics of its output: [2][ceil(M/32)][N]
  m.def("gemm_stats", [](at::Tensor a, at::Tensor b) {
    Args args("gemm_stats");
    args("a", a, {kBF16}, {kAny, kAny})("b", b, {kBF16}, {kAny, a.size(1)});
    args.device();
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    at::Tensor d = at::empty({M, N}, a.options());
    at::Tensor stats = at::empty({2, (M + 31) / 32, N}, a.options().dtype(kF32));
    launch_gemm_bf16(a.data_ptr(), b.data_ptr(), d.data_ptr(), nullptr, M, N, K, false, false, 0, DType::BF16, false, cur_stream(),
                     stats.data_ptr<float>());
    return std::make_tuple(d, stats);
  });
  // ---- FP8 (fp8.cu, gemm_wgmma.cu): E4M3 activations / weights, E5M2 gradients, power-of-two per-tensor scales ------------
  m.def("fp8_amax", [](at::Tensor t) {
    Args args("fp8_amax");
    args("t", t, {kBF16}, min_numel(0));
    args.device();
    t = aligned(t, 16);
    at::Tensor amax = at::empty({1}, t.options().dtype(kF32));
    launch_fp8_amax(t.data_ptr(), (size_t)t.numel(), amax.data_ptr<float>(), cur_stream());
    return amax;
  });
  // q (t's shape), q^T [cols, rows] or None, scale_inv [1] (= 1/s), fp32 column sums [cols] or None; s comes from `amax`
  auto fp8_cast = [](const at::Tensor& t, const at::Tensor& amax, bool e5m2, bool want_transpose, bool want_colsum) {
    const int cols = (int)t.size(-1);
    const int rows = (int)(t.numel() / cols);
    at::Tensor q = at::empty(t.sizes(), t.options().dtype(e5m2 ? at::kFloat8_e5m2 : at::kFloat8_e4m3fn));
    at::Tensor qt = want_transpose ? at::empty({cols, rows}, q.options()) : at::Tensor();
    at::Tensor scale_inv = at::empty({1}, t.options().dtype(kF32));
    at::Tensor colsum, partial;
    if (want_colsum) {
      colsum = at::empty({cols}, t.options().dtype(kF32));
      partial = at::empty({fp8_colsum_parts(rows), cols}, t.options().dtype(kF32));
    }
    launch_fp8_cast_transpose(t.data_ptr(), rows, cols, amax.data_ptr<float>(), e5m2, q.data_ptr(),
                              want_transpose ? qt.data_ptr() : nullptr, want_colsum ? partial.data_ptr<float>() : nullptr,
                              want_colsum ? colsum.data_ptr<float>() : nullptr, scale_inv.data_ptr<float>(), cur_stream());
    return py::make_tuple(q, want_transpose ? py::cast(qt) : py::none(), scale_inv, want_colsum ? py::cast(colsum) : py::none());
  };
  m.def("fp8_cast_transpose", [fp8_cast](at::Tensor t, at::Tensor amax, const std::string& fmt, bool want_transpose, bool want_colsum) {
    TORCH_CHECK(fmt == "e4m3" || fmt == "e5m2", "fp8: format must be 'e4m3' or 'e5m2', got '", fmt, "'");
    Args args("fp8_cast_transpose");
    args("t", t, {kBF16}, last_dim(kAny))("amax", amax, {kF32}, numel(1));
    args.device();
    return fp8_cast(aligned(t, 16), amax, fmt == "e5m2", want_transpose, want_colsum);
  }, py::arg("t"), py::arg("amax"), py::arg("fmt"), py::arg("want_transpose") = false, py::arg("want_colsum") = false);
  m.def("fp8_quantize", [fp8_cast](at::Tensor t, const std::string& fmt, bool want_transpose, bool want_colsum) {
    TORCH_CHECK(fmt == "e4m3" || fmt == "e5m2", "fp8: format must be 'e4m3' or 'e5m2', got '", fmt, "'");
    Args args("fp8_quantize");
    args("t", t, {kBF16}, last_dim(kAny));
    args.device();
    t = aligned(t, 16);
    at::Tensor amax = at::empty({1}, t.options().dtype(kF32));
    launch_fp8_amax(t.data_ptr(), (size_t)t.numel(), amax.data_ptr<float>(), cur_stream());
    return fp8_cast(t, amax, fmt == "e5m2", want_transpose, want_colsum);
  }, py::arg("t"), py::arg("fmt"), py::arg("want_transpose") = false, py::arg("want_colsum") = false);
  // D[M,N] bf16 = epi(a_scale_inv * b_scale_inv * A[M,K] @ B[N,K]^T + bias): A e4m3 or e5m2, B e4m3, both K-major
  m.def("gemm_fp8", [](at::Tensor a, at::Tensor b, at::Tensor a_scale_inv, at::Tensor b_scale_inv, c10::optional<at::Tensor> bias,
                       int epilogue) {
    Args args("gemm_fp8");
    args("a", a, {at::kFloat8_e4m3fn, at::kFloat8_e5m2}, {kAny, kAny}, kContiguous, 16);
    args("b", b, {at::kFloat8_e4m3fn}, {kAny, a.size(1)}, kContiguous, 16)("a_scale_inv", a_scale_inv, {kF32}, numel(1));
    args("b_scale_inv", b_scale_inv, {kF32}, numel(1));
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    TORCH_CHECK(K % 16 == 0, "gemm_fp8: K = ", K, " must be a multiple of 16 (row pitch of the 8-bit operands)");
    args("bias", bias, {kBF16}, numel(N));
    args.device();
    at::Tensor d = at::empty({M, N}, a.options().dtype(kBF16));
    launch_gemm_fp8(a.data_ptr(), b.data_ptr(), d.data_ptr(), bias.has_value() ? bias->data_ptr() : nullptr, a_scale_inv.data_ptr<float>(),
                    b_scale_inv.data_ptr<float>(), M, N, K, a.scalar_type() == at::kFloat8_e5m2, epilogue, cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("a_scale_inv"), py::arg("b_scale_inv"), py::arg("bias") = py::none(), py::arg("epilogue") = 0);

  // ---- attention (attention.cu): head dim 64 or 128, S % 128 == 0, masks on the device --------------------------------
  constexpr AttnFwd kPaddedFwd = [](const void* qkv, const int* m, int B, int S, int h, int, void* o, float* l, cudaStream_t s) {
    launch_attention_fwd(qkv, m, B, S, h, o, l, s);
  };
  constexpr AttnFwd kPackedFwd = [](const void* qkv, const int* m, int B, int S, int h, int, void* o, float* l, cudaStream_t s) {
    launch_packed_attention_fwd(qkv, m, B, S, h, o, l, s);
  };
  constexpr AttnFwd kCausalFwd = [](const void* qkv, const int* m, int B, int S, int h, int, void* o, float* l, cudaStream_t s) {
    launch_causal_attention_fwd(qkv, m, B, S, h, o, l, s);
  };
  constexpr AttnBwd kPaddedBwd = [](const void* d, const void* qkv, const void* o, const float* l, const int* m, int B, int S, int h, int,
                                    float* dsum, void* dqkv, cudaStream_t s) { launch_attention_bwd(d, qkv, o, l, m, B, S, h, dsum, dqkv, s); };
  constexpr AttnBwd kPackedBwd = [](const void* d, const void* qkv, const void* o, const float* l, const int* m, int B, int S, int h, int,
                                    float* dsum, void* dqkv, cudaStream_t s) { launch_packed_attention_bwd(d, qkv, o, l, m, B, S, h, dsum, dqkv, s); };
  constexpr AttnBwd kCausalBwd = [](const void* d, const void* qkv, const void* o, const float* l, const int* m, int B, int S, int h, int,
                                    float* dsum, void* dqkv, cudaStream_t s) { launch_causal_attention_bwd(d, qkv, o, l, m, B, S, h, dsum, dqkv, s); };
  // key padding: seq_lens int32 [B]
  m.def("attention_fwd", [](at::Tensor qkv, at::Tensor seq_lens, int heads, c10::optional<at::Tensor> o_out, c10::optional<at::Tensor> lse_out) {
    return attn_fwd("attention_fwd", kPaddedFwd, 64, Mask::kSeqLens, qkv, seq_lens, heads, heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("seq_lens"), py::arg("heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor seq_lens, int heads,
                            c10::optional<at::Tensor> dqkv_out) {
    return attn_bwd("attention_bwd", kPaddedBwd, 64, Mask::kSeqLens, dout, qkv, o, lse, seq_lens, heads, heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("seq_lens"), py::arg("heads"), py::arg("dqkv") = py::none());
  // packed documents: bounds int32 [B, S, 2] (contiguous, so [B*S, 2] rows of (start, end))
  m.def("packed_attention_fwd", [](at::Tensor qkv, at::Tensor bounds, int heads, c10::optional<at::Tensor> o_out,
                                   c10::optional<at::Tensor> lse_out) {
    return attn_fwd("packed_attention_fwd", kPackedFwd, 64, Mask::kBounds, qkv, bounds, heads, heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("packed_attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds, int heads,
                                   c10::optional<at::Tensor> dqkv_out) {
    return attn_bwd("packed_attention_bwd", kPackedBwd, 64, Mask::kBounds, dout, qkv, o, lse, bounds, heads, heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("dqkv") = py::none());
  // causal documents: the same bounds as the packed pair
  m.def("causal_attention_fwd", [](at::Tensor qkv, at::Tensor bounds, int heads, c10::optional<at::Tensor> o_out,
                                   c10::optional<at::Tensor> lse_out) {
    return attn_fwd("causal_attention_fwd", kCausalFwd, 64, Mask::kBounds, qkv, bounds, heads, heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("causal_attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds, int heads,
                                   c10::optional<at::Tensor> dqkv_out) {
    return attn_bwd("causal_attention_bwd", kCausalBwd, 64, Mask::kBounds, dout, qkv, o, lse, bounds, heads, heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("dqkv") = py::none());
  // grouped-query causal documents at head dim 64, and causal documents at head dim 128 (kv_heads == heads included)
  m.def("causal_gqa_attention_fwd", [](at::Tensor qkv, at::Tensor bounds, int heads, int kv_heads, c10::optional<at::Tensor> o_out,
                                       c10::optional<at::Tensor> lse_out) {
    return attn_fwd("causal_gqa_attention_fwd", &launch_causal_gqa_attention_fwd, 64, Mask::kBounds, qkv, bounds, heads, kv_heads, o_out, lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("causal_gqa_attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds, int heads,
                                       int kv_heads, c10::optional<at::Tensor> dqkv_out) {
    return attn_bwd("causal_gqa_attention_bwd", &launch_causal_gqa_attention_bwd, 64, Mask::kBounds, dout, qkv, o, lse, bounds, heads, kv_heads,
                    dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"),
     py::arg("dqkv") = py::none());
  m.def("causal_attention_d128_fwd", [](at::Tensor qkv, at::Tensor bounds, int heads, int kv_heads, c10::optional<at::Tensor> o_out,
                                        c10::optional<at::Tensor> lse_out) {
    return attn_fwd("causal_attention_d128_fwd", &launch_causal_attention_d128_fwd, 128, Mask::kBounds, qkv, bounds, heads, kv_heads, o_out,
                    lse_out);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"), py::arg("o") = py::none(), py::arg("lse") = py::none());
  m.def("causal_attention_d128_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds, int heads,
                                        int kv_heads, c10::optional<at::Tensor> dqkv_out) {
    return attn_bwd("causal_attention_d128_bwd", &launch_causal_attention_d128_bwd, 128, Mask::kBounds, dout, qkv, o, lse, bounds, heads,
                    kv_heads, dqkv_out);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("heads"), py::arg("kv_heads"),
     py::arg("dqkv") = py::none());

  // ---- Llama building blocks: rotary embedding (rotary.cu), RMSNorm (layernorm.cu), SwiGLU (loss.cu) --------------------
  // y = rope(qkv) (backward: the transpose rotation); qkv bf16 [rows, (heads + 2*kv_heads)*d] with d = 64 or 128, positions
  // int32 [rows], table fp32 [max_pos, 2, d/2]
  m.def("rotary", [](at::Tensor x, at::Tensor pos, at::Tensor table, int heads, int kv_heads, bool backward, double q_scale) {
    Args args("rotary");
    TORCH_CHECK(heads >= 1 && kv_heads >= 1, "rotary: heads and kv_heads must be positive, got ", heads, " and ", kv_heads);
    args("cos_sin", table, {kF32}, {kAny, 2, kAny});
    args.expect(table.size(2) == 32 || table.size(2) == 64, "cos_sin", "fp32 [max_position, 2, d/2] with d = 64 or 128", table);
    const int d = (int)table.size(2) * 2;
    args("x", x, {kBF16}, {kAny, (int64_t)(heads + 2 * kv_heads) * d})("position_ids", pos, {kI32}, numel(x.size(0)));
    args.device();
    x = aligned(x, 16);
    at::Tensor y = at::empty_like(x);
    launch_rotary(x.data_ptr(), pos.data_ptr<int>(), table.data_ptr<float>(), (int)table.size(0), (size_t)x.size(0), heads, kv_heads, d,
                  y.data_ptr(), backward, cur_stream(), (float)q_scale);
    return y;
  }, py::arg("x"), py::arg("position_ids"), py::arg("cos_sin"), py::arg("heads"), py::arg("kv_heads"), py::arg("backward") = false,
     py::arg("q_scale") = 1.0);
  // Qwen3's per-head q / k RMSNorm + rotary, d = 128: (y, rstd fp32 [rows, heads + kv_heads]) = fwd(qkv, wq, wk, ...);
  // (dqkv, dwq, dwk) = bwd(dy, qkv, rstd, wq, wk, ...) with qkv the forward's input
  auto qk_norm_args = [](Args& args, const at::Tensor& x, const at::Tensor& wq, const at::Tensor& wk, const at::Tensor& pos,
                         const at::Tensor& table, int heads, int kv_heads) {
    TORCH_CHECK(heads >= 1 && kv_heads >= 1, args.fn(), ": heads and kv_heads must be positive, got ", heads, " and ", kv_heads);
    args("cos_sin", table, {kF32}, {kAny, 2, 64})("x", x, {kBF16}, {kAny, (int64_t)(heads + 2 * kv_heads) * 128});
    args("q_weight", wq, {kBF16}, numel(128))("k_weight", wk, {kBF16}, numel(128))("position_ids", pos, {kI32}, numel(x.size(0)));
  };
  m.def("qk_norm_rotary_fwd", [qk_norm_args](at::Tensor x, at::Tensor wq, at::Tensor wk, at::Tensor pos, at::Tensor table, int heads,
                                             int kv_heads, double eps) {
    Args args("qk_norm_rotary_fwd");
    qk_norm_args(args, x, wq, wk, pos, table, heads, kv_heads);
    args.device();
    at::Tensor y = at::empty_like(x);
    at::Tensor rstd = at::empty({x.size(0), heads + kv_heads}, x.options().dtype(kF32));
    launch_qk_norm_rotary_fwd(x.data_ptr(), wq.data_ptr(), wk.data_ptr(), pos.data_ptr<int>(), table.data_ptr<float>(), (int)table.size(0),
                              (size_t)x.size(0), heads, kv_heads, 128, (float)eps, y.data_ptr(), rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, rstd);
  }, py::arg("x"), py::arg("q_weight"), py::arg("k_weight"), py::arg("position_ids"), py::arg("cos_sin"), py::arg("heads"),
     py::arg("kv_heads"), py::arg("eps"));
  m.def("qk_norm_rotary_bwd", [qk_norm_args](at::Tensor dy, at::Tensor x, at::Tensor rstd, at::Tensor wq, at::Tensor wk, at::Tensor pos,
                                             at::Tensor table, int heads, int kv_heads) {
    Args args("qk_norm_rotary_bwd");
    qk_norm_args(args, x, wq, wk, pos, table, heads, kv_heads);
    args("dy", dy, {kBF16}, x.sizes())("rstd", rstd, {kF32}, numel(x.size(0) * (int64_t)(heads + kv_heads)));
    args.device();
    const int parts = qk_norm_rotary_partials((size_t)x.size(0));
    at::Tensor dx = at::empty_like(x);
    at::Tensor partial = at::empty({2, parts, 128}, x.options().dtype(kF32));
    at::Tensor dwq = at::empty_like(wq), dwk = at::empty_like(wk);
    launch_qk_norm_rotary_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr<float>(), wq.data_ptr(), wk.data_ptr(), pos.data_ptr<int>(),
                              table.data_ptr<float>(), (int)table.size(0), (size_t)x.size(0), heads, kv_heads, 128, dx.data_ptr(),
                              partial.data_ptr<float>(), dwq.data_ptr(), dwk.data_ptr(), cur_stream());
    return std::make_tuple(dx, dwq, dwk);
  }, py::arg("dy"), py::arg("x"), py::arg("rstd"), py::arg("q_weight"), py::arg("k_weight"), py::arg("position_ids"), py::arg("cos_sin"),
     py::arg("heads"), py::arg("kv_heads"));
  m.def("rmsnorm_fwd", [](at::Tensor x, at::Tensor gamma, double eps) {
    Args args("rmsnorm_fwd");
    args("x", x, {kF32, kBF16}, last_dim(kAny))("gamma", gamma, {x.scalar_type()}, numel(x.size(-1)));
    args.device();
    x = aligned(x, 32);
    gamma = aligned(gamma, 32);
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    at::Tensor y = at::empty_like(x);
    at::Tensor rstd = at::empty({rows}, x.options().dtype(kF32));
    launch_rmsnorm_fwd(x.data_ptr(), gamma.data_ptr(), dtype_of(x), rows, cols, (float)eps, y.data_ptr(), rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, rstd);
  });
  m.def("rmsnorm_bwd", [](at::Tensor dy, at::Tensor x, at::Tensor gamma, at::Tensor rstd) {
    Args args("rmsnorm_bwd");
    args("x", x, {kF32, kBF16}, last_dim(kAny));
    const int cols = (int)x.size(-1);
    const int rows = (int)(x.numel() / cols);
    args("dy", dy, {x.scalar_type()}, x.sizes())("gamma", gamma, {x.scalar_type()}, numel(cols), kStrided)("rstd", rstd, {kF32}, numel(rows));
    args.device();
    dy = aligned(dy, 32);
    x = aligned(x, 32);
    gamma = aligned(gamma.contiguous(), 32);
    const int parts = layernorm_partial_rows(rows);
    at::Tensor dx = at::empty_like(x);
    at::Tensor partial = at::empty({2 * parts, cols}, x.options().dtype(kF32));
    at::Tensor counters = at::empty({(cols + 7) / 8}, x.options().dtype(kI32));
    at::Tensor dgamma = at::empty_like(gamma);
    launch_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), rstd.data_ptr<float>(), dtype_of(x), rows, cols, dx.data_ptr(),
                       partial.data_ptr<float>(), reinterpret_cast<unsigned int*>(counters.data_ptr<int>()), parts, dgamma.data_ptr(),
                       cur_stream());
    return std::make_tuple(dx, dgamma);
  });
  // Gated linear units on one projection [M, 2I]: SwiGLU (gate | up, out = silu(gate) * up) and GeGLU (input | gate,
  // out = gelu(input) * gate).  Forward: out [M, I]; backward: the gradient of both column blocks [M, 2I] from dy [M, I].
  using GluLaunch = void (*)(const void*, const void*, void*, size_t, int, bool, cudaStream_t);
  auto glu_fwd = [](const char* fn, const char* name, at::Tensor gate_up, GluLaunch launch) {
    Args args(fn);
    args(name, gate_up, {kBF16}, last_dim(kAny));
    args.expect(gate_up.size(-1) % 16 == 0, name, "bf16 [..., 2I] with I % 8 == 0", gate_up);
    args.device();
    gate_up = aligned(gate_up, 16);
    auto sizes = gate_up.sizes().vec();
    const int inter = (int)(sizes.back() / 2);
    sizes.back() = inter;
    at::Tensor out = at::empty(sizes, gate_up.options());
    launch(gate_up.data_ptr(), nullptr, out.data_ptr(), (size_t)(gate_up.numel() / (2 * inter)), inter, false, cur_stream());
    return out;
  };
  auto glu_bwd = [](const char* fn, const char* name, at::Tensor dy, at::Tensor gate_up, GluLaunch launch) {
    Args args(fn);
    args(name, gate_up, {kBF16}, last_dim(kAny));
    args.expect(gate_up.size(-1) % 16 == 0, name, "bf16 [..., 2I] with I % 8 == 0", gate_up);
    args("dy", dy, {kBF16}, last_dim(gate_up.size(-1) / 2));
    args.expect(dy.numel() * 2 == gate_up.numel(), "dy", "bf16 [..., I] with half the elements of gate_up", dy);
    args.device();
    gate_up = aligned(gate_up, 16);
    dy = aligned(dy, 16);
    const int inter = (int)dy.size(-1);
    at::Tensor out = at::empty_like(gate_up);
    launch(gate_up.data_ptr(), dy.data_ptr(), out.data_ptr(), (size_t)(dy.numel() / inter), inter, true, cur_stream());
    return out;
  };
  m.def("swiglu_fwd", [glu_fwd](at::Tensor gate_up) { return glu_fwd("swiglu_fwd", "gate_up", gate_up, launch_swiglu); });
  m.def("swiglu_bwd", [glu_bwd](at::Tensor dy, at::Tensor gate_up) { return glu_bwd("swiglu_bwd", "gate_up", dy, gate_up, launch_swiglu); });
  m.def("geglu_fwd", [glu_fwd](at::Tensor input_gate) { return glu_fwd("geglu_fwd", "input_gate", input_gate, launch_geglu); });
  m.def("geglu_bwd", [glu_bwd](at::Tensor dy, at::Tensor input_gate) { return glu_bwd("geglu_bwd", "input_gate", dy, input_gate, launch_geglu); });

  // ---- mixture of experts (moe.cu, grouped GEMMs in gemm_wgmma.cu) -------------------------------------------------
  // logits bf16 [T, E] -> (ids int32 [T, k], gates bf16 [T, k], probsum fp32 [E] (aux) or None)
  m.def("moe_route", [](at::Tensor logits, int k, bool aux) {
    Args args("moe_route");
    args("logits", logits, {kBF16}, {kAny, kAny});
    args.device();
    const int T = (int)logits.size(0), E = (int)logits.size(1);
    at::Tensor ids = at::empty({T, k}, logits.options().dtype(kI32));
    at::Tensor gates = at::empty({T, k}, logits.options());
    c10::optional<at::Tensor> probsum;
    at::Tensor partial;
    if (aux) {
      probsum = at::empty({E}, logits.options().dtype(kF32));
      partial = at::empty({(T + 63) / 64, E}, logits.options().dtype(kF32));
    }
    launch_moe_router_fwd(logits.data_ptr(), T, E, k, ids.data_ptr<int>(), gates.data_ptr(), aux ? partial.data_ptr<float>() : nullptr,
                          aux ? probsum->data_ptr<float>() : nullptr, cur_stream());
    return std::make_tuple(ids, gates, probsum);
  });
  // dlogits bf16 [T, E] from d(gates) fp32 [T, k] and d(probsum) fp32 [E] (or None)
  m.def("moe_router_bwd", [](at::Tensor logits, at::Tensor ids, at::Tensor dgates, c10::optional<at::Tensor> dprobsum) {
    Args args("moe_router_bwd");
    args("logits", logits, {kBF16}, {kAny, kAny})("ids", ids, {kI32}, {logits.size(0), kAny});
    const int T = (int)logits.size(0), E = (int)logits.size(1), k = (int)ids.size(1);
    args("dgates", dgates, {kF32}, numel((int64_t)T * k))("dprobsum", dprobsum, {kF32}, numel(E));
    args.device();
    at::Tensor dlogits = at::empty_like(logits);
    launch_moe_router_bwd(logits.data_ptr(), T, E, k, ids.data_ptr<int>(), dgates.data_ptr<float>(),
                          dprobsum.has_value() ? dprobsum->data_ptr<float>() : nullptr, dlogits.data_ptr(), cur_stream());
    return dlogits;
  });
  // ids int32 [T, k] -> (counts [E], offsets [E + 1], fwd_map [capacity], inv_map [T, k], tile_expert [capacity / 128]), int32
  m.def("moe_permute", [](at::Tensor ids, int E) {
    Args args("moe_permute");
    args("ids", ids, {kI32}, {kAny, kAny});
    const int T = (int)ids.size(0), k = (int)ids.size(1);
    TORCH_CHECK(T >= 1 && E >= 1 && E <= kMoeMaxExperts && k >= 1 && k <= kMoeMaxTopK && k <= E,
                "moe_permute: needs T >= 1, 1 <= E <= 64, 1 <= k <= min(E, 8), got T=", T, " E=", E, " k=", k);
    args.device();
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
  m.def("moe_gather", [](at::Tensor x, at::Tensor fwd_map, int k) {
    Args args("moe_gather");
    args("x", x, {kBF16}, {kAny, kAny})("fwd_map", fwd_map, {kI32}, {kAny});
    args.device();
    const int H = (int)x.size(1), cap = (int)fwd_map.numel();
    at::Tensor out = at::empty({cap, H}, x.options());
    launch_moe_gather(x.data_ptr(), fwd_map.data_ptr<int>(), cap, H, k, out.data_ptr(), cur_stream());
    return out;
  });
  // forward: a [capacity, K] . w_e^T with w [E, N, K] -> [capacity, N]; dgrad: a [capacity, K] . w_e with w [E, K, N] -> [capacity, N]
  m.def("moe_gemm", [](at::Tensor a, at::Tensor w, at::Tensor tile_expert, bool dgrad, c10::optional<at::Tensor> out) {
    Args args("moe_gemm");
    args("w", w, {kBF16}, {kAny, kAny, kAny});
    const int E = (int)w.size(0), K = (int)(dgrad ? w.size(1) : w.size(2)), N = (int)(dgrad ? w.size(2) : w.size(1));
    args("a", a, {kBF16}, {kAny, K});
    const int rows = (int)a.size(0);
    args("tile_expert", tile_expert, {kI32}, numel(rows / kMoeAlign));
    at::Tensor d;
    args.out(d, "out", out, {rows, N}, a.options());
    args.device();
    launch_gemm_grouped(a.data_ptr(), w.data_ptr(), d.data_ptr(), rows, N, K, E, dgrad, tile_expert.data_ptr<int>(), cur_stream());
    return d;
  }, py::arg("a"), py::arg("w"), py::arg("tile_expert"), py::arg("dgrad"), py::arg("out") = py::none());
  // weight gradient: dw [E, M, N] (bf16), dw_e = a[s_e]^T . b[s_e] over expert e's segment of a [capacity, M] and b [capacity, N]
  m.def("moe_gemm_wgrad", [](at::Tensor a, at::Tensor b, at::Tensor offsets, c10::optional<at::Tensor> out) {
    Args args("moe_gemm_wgrad");
    args("a", a, {kBF16}, {kAny, kAny})("b", b, {kBF16}, {a.size(0), kAny})("offsets", offsets, {kI32}, {kAny});
    const int rows = (int)a.size(0), M = (int)a.size(1), N = (int)b.size(1), E = (int)offsets.numel() - 1;
    at::Tensor d;
    args.out(d, "out", out, {E, M, N}, a.options());
    args.device();
    launch_gemm_grouped_wgrad(a.data_ptr(), b.data_ptr(), d.data_ptr(), rows, M, N, E, offsets.data_ptr<int>(), cur_stream());
    return d;
  }, py::arg("a"), py::arg("b"), py::arg("offsets"), py::arg("out") = py::none());
  // out [T, H] = sum_j gate[t, j] * y_perm[inv[t, j]] (gates None: weight 1)
  m.def("moe_combine", [](at::Tensor y_perm, at::Tensor inv_map, c10::optional<at::Tensor> gates) {
    Args args("moe_combine");
    args("y_perm", y_perm, {kBF16}, {kAny, kAny})("inv_map", inv_map, {kI32}, {kAny, kAny});
    const int T = (int)inv_map.size(0), k = (int)inv_map.size(1), H = (int)y_perm.size(1);
    args("gates", gates, {kBF16}, numel((int64_t)T * k));
    args.device();
    at::Tensor out = at::empty({T, H}, y_perm.options());
    launch_moe_combine(y_perm.data_ptr(), inv_map.data_ptr<int>(), gates.has_value() ? gates->data_ptr() : nullptr, T, H, k, out.data_ptr(),
                       cur_stream());
    return out;
  });
  // (dy_perm bf16 [capacity, H], dgates fp32 [T, k]) from dout bf16 [T, H]
  m.def("moe_combine_bwd", [](at::Tensor dout, at::Tensor y_perm, at::Tensor fwd_map, at::Tensor gates) {
    Args args("moe_combine_bwd");
    args("dout", dout, {kBF16}, {kAny, kAny})("y_perm", y_perm, {kBF16}, {kAny, dout.size(1)})("gates", gates, {kBF16}, {dout.size(0), kAny});
    const int T = (int)dout.size(0), H = (int)dout.size(1), k = (int)gates.size(1), cap = (int)y_perm.size(0);
    args("fwd_map", fwd_map, {kI32}, numel(cap));
    args.device();
    at::Tensor dy = at::empty_like(y_perm);
    at::Tensor dgates = at::empty({T, k}, dout.options().dtype(kF32));
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
    Args args("conv_fprop");
    args("x", x, {kBF16}, {kAny, kAny, kAny, kAny}, kChannelsLast)("w", w, {kBF16}, {kAny, x.size(1), kAny, kAny}, kChannelsLast);
    args("debug", debug, {kI64}, min_numel(16));
    const int R = (int)w.size(2), S = (int)w.size(3);
    TORCH_CHECK(stride == 1 && R == S && pad == (R - 1) / 2, "conv_fprop: stride 1, 'same' padding");
    args.device();
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), K = (int)w.size(0);
    at::Tensor y = at::empty({N, K, H, W}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    ConvLaunchCfg cfg; cfg.mode = mode; cfg.block_n = block_n; cfg.set_base_offset = base_offset; cfg.kc = kc;
    if (debug.has_value()) cfg.debug_counters = debug->data_ptr();
    at::Tensor st;
    float* stp = nullptr;
    if (stats) {
      const int groups = conv_stat_groups(N, H, W, C, K, R, S, cfg);
      TORCH_CHECK(groups > 0, "conv_fprop: no tile plan");
      st = at::empty({2, groups, K}, x.options().dtype(kF32));
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
    Args args("conv_dgrad");
    args("dy", dy, {kBF16}, {kAny, kAny, kAny, kAny}, kChannelsLast)("w", w, {kBF16}, {dy.size(1), kAny, kAny, kAny}, kChannelsLast);
    const int R = (int)w.size(2), S = (int)w.size(3);
    TORCH_CHECK(stride == 1 && R == S && pad == (R - 1) / 2, "conv_dgrad: stride 1, 'same' padding");
    const int N = (int)dy.size(0), K = (int)dy.size(1), H = (int)dy.size(2), W = (int)dy.size(3), C = (int)w.size(1);
    args("addend", addend, {kBF16}, {N, C, H, W}, kChannelsLast)("bn_x", bn_x, {kBF16}, {N, C, H, W}, kChannelsLast);
    args("bn_mask", bn_mask, {kU8}, numel((int64_t)N * H * W * (C / 8)));
    if (bn_x.has_value()) {
      args("bn_stats", args.required("bn_stats", bn_stats), {kF32}, {kAny, C});
      args.expect(bn_stats->size(0) >= 2, "bn_stats", "fp32 [>= 2, C] (rows: mean, rstd)", *bn_stats);
    }
    args.device();
    at::Tensor dx = at::empty({N, C, H, W}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
    ConvLaunchCfg cfg; cfg.mode = mode; cfg.block_n = block_n; cfg.set_base_offset = base_offset; cfg.kc = kc;
    ConvBwdFusion fuse;
    bool any = false;
    at::Tensor part;
    float* pp = nullptr;
    if (addend.has_value()) { fuse.addend = addend->data_ptr(); any = true; }
    if (bn_x.has_value()) {
      fuse.bn_x = bn_x->data_ptr();
      if (bn_mask.has_value()) fuse.bn_mask = bn_mask->data_ptr();
      fuse.bn_mean = bn_stats->data_ptr<float>();
      fuse.bn_rstd = bn_stats->data_ptr<float>() + C;
      // the statistics workspace of the data gradient has one row per CTA of an n-tile over the Cin columns
      const int groups = conv_stat_groups(N, H, W, K, C, R, S, cfg);
      TORCH_CHECK(groups > 0, "conv_dgrad: no tile plan");
      part = at::empty({2, groups, C}, dy.options().dtype(kF32));
      pp = part.data_ptr<float>();
      any = true;
    }
    launch_conv_tap_gemm(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), N, H, W, C, K, R, S, true, cfg, pp, cur_stream(), any ? &fuse : nullptr);
    return std::make_tuple(dx, part);
  }, py::arg("dy"), py::arg("w"), py::arg("stride") = 1, py::arg("pad") = 0, py::arg("mode") = -1, py::arg("block_n") = 0,
     py::arg("base_offset") = 0, py::arg("kc") = 0, py::arg("addend") = py::none(), py::arg("bn_x") = py::none(),
     py::arg("bn_mask") = py::none(), py::arg("bn_stats") = py::none());
  m.def("conv_wgrad", [](at::Tensor dy, at::Tensor x, int ksize, int stride, int pad, int split, int tile_m, int tile_n) {
    Args args("conv_wgrad");
    args("dy", dy, {kBF16}, {kAny, kAny, kAny, kAny}, kChannelsLast)("x", x, {kBF16}, {dy.size(0), kAny, dy.size(2), dy.size(3)}, kChannelsLast);
    TORCH_CHECK(stride == 1 && pad == (ksize - 1) / 2, "conv_wgrad: stride 1, 'same' padding");
    args.device();
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), K = (int)dy.size(1);
    WgradCfg cfg; cfg.split = split; cfg.tile_m = tile_m; cfg.tile_n = tile_n;
    const size_t ws = conv_wgrad_workspace_floats(N, H, W, C, K, ksize, ksize, cfg);
    TORCH_CHECK(ws > 0, "conv_wgrad: unsupported geometry / tiling");
    at::Tensor work = at::empty({(int64_t)ws}, x.options().dtype(kF32));
    at::Tensor dw = at::empty({K, C, ksize, ksize}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    launch_conv_wgrad(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), N, H, W, C, K, ksize, ksize, cfg, work.data_ptr<float>(), cur_stream());
    return dw;
  }, py::arg("dy"), py::arg("x"), py::arg("ksize"), py::arg("stride") = 1, py::arg("pad") = 0, py::arg("split") = 0,
     py::arg("tile_m") = 0, py::arg("tile_n") = 0);
  // strided 7x7 stem (3 -> 64 channels, stride 2, padding 3) on the wgmma tap-GEMM through an overlapping-window tensor map
  m.def("stem_conv_supported", [](int H, int W) { StemGeom g; return stem_geom(H, W, &g); });
  m.def("stem_pack_input", [](at::Tensor x) {
    Args args("stem_pack_input");
    args("x", x, {kBF16}, {kAny, 3, kAny, kAny}, kChannelsLast);
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g), "stem_pack_input: unsupported image size ", H, "x", W);
    args.device();
    at::Tensor xp = at::empty({N, g.Hp2, g.Wp, 8}, x.options());
    launch_stem_pack_input(x.data_ptr(), xp.data_ptr(), N, H, W, cur_stream());
    return xp;
  });
  m.def("stem_pack_weight", [](at::Tensor w) {
    Args args("stem_pack_weight");
    args("w", w, {kBF16}, {64, 3, 7, 7}, kChannelsLast);
    args.device();
    at::Tensor w2 = at::empty({w.size(0), (int64_t)kStemK}, w.options().memory_format(at::MemoryFormat::Contiguous));
    launch_stem_pack_weight(w.data_ptr(), w2.data_ptr(), (int)w.size(0), cur_stream());
    return w2;
  });
  m.def("stem_conv_fprop_packed", [](at::Tensor xp, at::Tensor w2, int H, int W, bool stats, bool resident, bool debug) {
    Args args("stem_conv_fprop_packed");
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g), "stem_conv_fprop_packed: unsupported image size ", H, "x", W);
    args("xp", xp, {kBF16}, {kAny, g.Hp2, g.Wp, 8})("w2", w2, {kBF16}, {kAny, kStemK});
    args.device();
    const int N = (int)xp.size(0), K = (int)w2.size(0);
    at::Tensor y = at::empty({N, K, g.Ho, g.Wo}, xp.options().memory_format(at::MemoryFormat::ChannelsLast));
    at::Tensor part, dbg;
    float* sp = nullptr;
    if (stats) { part = at::empty({2, stem_stat_groups(N, H, W), K}, xp.options().dtype(kF32)); sp = part.data_ptr<float>(); }
    if (debug) dbg = at::zeros({16}, xp.options().dtype(kI64));
    launch_stem_conv_fprop(xp.data_ptr(), w2.data_ptr(), y.data_ptr(), N, H, W, K, sp, resident, debug ? dbg.data_ptr() : nullptr, cur_stream());
    return std::make_tuple(y, part, dbg);
  }, py::arg("xp"), py::arg("w2"), py::arg("H"), py::arg("W"), py::arg("stats") = false, py::arg("resident") = true, py::arg("debug") = false);
  m.def("stem_conv_fprop", [](at::Tensor x, at::Tensor w, bool stats, bool resident) {
    Args args("stem_conv_fprop");
    args("x", x, {kBF16}, {kAny, 3, kAny, kAny}, kChannelsLast)("w", w, {kBF16}, {64, 3, 7, 7}, kChannelsLast);
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3), K = (int)w.size(0);
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g), "stem_conv_fprop: unsupported image size ", H, "x", W);
    args.device();
    at::Tensor xp = at::empty({N, g.Hp2, g.Wp, 8}, x.options().memory_format(at::MemoryFormat::Contiguous));
    at::Tensor w2 = at::empty({K, (int64_t)kStemK}, x.options().memory_format(at::MemoryFormat::Contiguous));
    at::Tensor y = at::empty({N, K, g.Ho, g.Wo}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    at::Tensor part;
    float* sp = nullptr;
    if (stats) { part = at::empty({2, stem_stat_groups(N, H, W), K}, x.options().dtype(kF32).memory_format(at::MemoryFormat::Contiguous)); sp = part.data_ptr<float>(); }
    cudaStream_t st = cur_stream();
    launch_stem_pack_input(x.data_ptr(), xp.data_ptr(), N, H, W, st);
    launch_stem_pack_weight(w.data_ptr(), w2.data_ptr(), K, st);
    launch_stem_conv_fprop(xp.data_ptr(), w2.data_ptr(), y.data_ptr(), N, H, W, K, sp, resident, nullptr, st);
    return std::make_tuple(y, part, xp);
  }, py::arg("x"), py::arg("w"), py::arg("stats") = false, py::arg("resident") = true);
  m.def("stem_conv_wgrad", [](at::Tensor dy, at::Tensor xp, int H, int W, int variant, bool unpack) {
    Args args("stem_conv_wgrad");
    TORCH_CHECK(variant == 0 || variant == 1, "stem_conv_wgrad: variant 0 (dedicated kernel) or 1 (generic kernel)");
    StemGeom g;
    TORCH_CHECK(stem_geom(H, W, &g), "stem_conv_wgrad: unsupported image size ", H, "x", W);
    args("dy", dy, {kBF16}, {kAny, kAny, g.Ho, g.Wo}, kChannelsLast)("xp", xp, {kBF16}, {dy.size(0), g.Hp2, g.Wp, 8});
    args.device();
    const int N = (int)dy.size(0), K = (int)dy.size(1);
    const size_t ws = stem_wgrad_workspace_floats(N, H, W, K, variant);
    TORCH_CHECK(ws > 0, "stem_conv_wgrad: unsupported geometry");
    auto plain = dy.options().memory_format(at::MemoryFormat::Contiguous);
    at::Tensor work = at::empty({(int64_t)ws}, plain.dtype(kF32));
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

  // ---- fused BatchNorm: x [N, C, H, W] channels_last viewed as [R = N*H*W, C]; gamma, beta and statistics fp32 ----------------
  m.def("set_bn_pdl", &set_bn_pdl);
  m.def("set_bn_two_pass", &set_bn_two_pass);
  m.def("bn_resident_error", &bn_resident_error);
  m.def("bn_workspace", [](int R, int C) {
    size_t pf = 0, cn = 0;
    bn_workspace_sizes(R, C, &pf, &cn);
    return std::make_tuple((long long)pf, (long long)cn);
  });
  // the forward's x, residual and affine / running statistics
  auto bn_fwd_args = [](Args& args, const at::Tensor& x, const c10::optional<at::Tensor>& residual, const at::Tensor& gamma,
                        const at::Tensor& beta, const c10::optional<at::Tensor>& running_mean, const c10::optional<at::Tensor>& running_var,
                        const c10::optional<at::Tensor>& num_batches) {
    args("x", x, {kF32, kBF16}, {kAny, kAny, kAny, kAny}, kChannelsLast);
    const int64_t C = x.size(1);
    args("residual", residual, {x.scalar_type()}, x.sizes(), kChannelsLast)("gamma", gamma, {kF32}, numel(C))("beta", beta, {kF32}, numel(C));
    args("running_mean", running_mean, {kF32}, numel(C))("running_var", running_var, {kF32}, numel(C))("num_batches", num_batches, {kI64}, numel(1));
  };
  // the backward's dy (`dy_layout`: kStrided when the binding makes it channels_last), x, ReLU mask (uint8 [R, C/8], read with
  // relu), gamma and the forward's statistics (save_mean, save_rstd, ...)
  auto bn_bwd_args = [](Args& args, const at::Tensor& dy, Layout dy_layout, const at::Tensor& x, const c10::optional<at::Tensor>& mask, bool relu,
                        const at::Tensor& gamma, const at::Tensor& stats) {
    args("x", x, {kF32, kBF16}, {kAny, kAny, kAny, kAny}, kChannelsLast);
    const int64_t C = x.size(1), R = x.numel() / std::max<int64_t>(C, 1);
    args("dy", dy, {x.scalar_type()}, x.sizes(), dy_layout);
    if (relu) args("y", args.required("y", mask), {kU8}, {R, C / 8});
    args("gamma", gamma, {kF32}, numel(C))("stats", stats, {kF32}, min_numel(2 * C));
  };
  m.def("bn_forward", [bn_fwd_args](at::Tensor x, c10::optional<at::Tensor> residual, at::Tensor gamma, at::Tensor beta,
                                    c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                                    c10::optional<at::Tensor> num_batches, double eps, double momentum, bool relu, at::Tensor partial,
                                    at::Tensor counters) {
    Args args("bn_forward");
    bn_fwd_args(args, x, residual, gamma, beta, running_mean, running_var, num_batches);
    args("partial", partial, {kF32}, min_numel(0))("counters", counters, {kI32}, min_numel(0));
    args.device();
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    size_t pf = 0, cn = 0;
    bn_workspace_sizes(R, C, &pf, &cn);   // reads the device's limits, so after the guard
    args("partial", partial, {kF32}, min_numel((int64_t)pf))("counters", counters, {kI32}, min_numel((int64_t)cn));
    at::Tensor y = at::empty_like(x);
    at::Tensor stats = at::empty({4, C}, x.options().dtype(kF32));   // rows: save_mean, save_rstd, scale, shift
    float* st = stats.data_ptr<float>();
    at::Tensor mask = relu ? at::empty({(int64_t)R, (int64_t)(C / 8)}, x.options().dtype(kU8)) : at::Tensor();
    launch_bn_forward(x.data_ptr(), residual.has_value() ? residual->data_ptr() : nullptr, y.data_ptr(), relu ? mask.data_ptr<uint8_t>() : nullptr,
                      dtype_of(x), R, C, gamma.data_ptr<float>(), beta.data_ptr<float>(),
                      running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
                      running_var.has_value() ? running_var->data_ptr<float>() : nullptr,
                      num_batches.has_value() ? (long long*)num_batches->data_ptr<int64_t>() : nullptr, st, st + C, st + 2 * C, st + 3 * C,
                      partial.data_ptr<float>(), (unsigned int*)counters.data_ptr<int>(), (float)eps, (float)momentum, relu, cur_stream());
    return std::make_tuple(y, stats, mask);
  });
  m.def("bn_forward_partials", [bn_fwd_args](at::Tensor x, c10::optional<at::Tensor> residual, at::Tensor gamma, at::Tensor beta,
                                             c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                                             c10::optional<at::Tensor> num_batches, double eps, double momentum, bool relu, at::Tensor partial) {
    Args args("bn_forward_partials");
    bn_fwd_args(args, x, residual, gamma, beta, running_mean, running_var, num_batches);
    args("partial", partial, {kF32}, {2, kAny, x.size(1)});   // [2, groups, C]
    args.device();
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    at::Tensor y = at::empty_like(x);
    at::Tensor stats = at::empty({4, C}, x.options().dtype(kF32));   // rows: save_mean, save_rstd, scale, shift
    float* st = stats.data_ptr<float>();
    at::Tensor mask = relu ? at::empty({(int64_t)R, (int64_t)(C / 8)}, x.options().dtype(kU8)) : at::Tensor();
    launch_bn_forward_from_partials(x.data_ptr(), residual.has_value() ? residual->data_ptr() : nullptr, y.data_ptr(),
                                    relu ? mask.data_ptr<uint8_t>() : nullptr, dtype_of(x), R, C, gamma.data_ptr<float>(), beta.data_ptr<float>(),
                                    running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
                                    running_var.has_value() ? running_var->data_ptr<float>() : nullptr,
                                    num_batches.has_value() ? (long long*)num_batches->data_ptr<int64_t>() : nullptr, st, st + C, st + 2 * C,
                                    st + 3 * C, partial.data_ptr<float>(), (int)partial.size(1), (float)eps, (float)momentum, relu, cur_stream());
    return std::make_tuple(y, stats, mask);
  });
  m.def("bn_backward_partials", [bn_bwd_args](at::Tensor dy, at::Tensor x, c10::optional<at::Tensor> y, at::Tensor gamma, at::Tensor stats,
                                              bool relu, bool need_dres, at::Tensor partial) {
    Args args("bn_backward_partials");
    bn_bwd_args(args, dy, kChannelsLast, x, y, relu, gamma, stats);
    args("partial", partial, {kF32}, {2, kAny, x.size(1)});   // [2, groups, C]
    args.device();
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    at::Tensor dx = at::empty_like(x);
    at::Tensor dres = need_dres ? at::empty_like(x) : at::Tensor();
    at::Tensor dparams = at::empty({2, C}, x.options().dtype(kF32));   // rows: dgamma, dbeta
    float* dp = dparams.data_ptr<float>();
    const float* st = stats.data_ptr<float>();
    launch_bn_backward_from_partials(dy.data_ptr(), x.data_ptr(), relu ? y->data_ptr() : nullptr, dx.data_ptr(), need_dres ? dres.data_ptr() : nullptr,
                                     dtype_of(x), R, C, gamma.data_ptr<float>(), st, st + C, dp, dp + C, partial.data_ptr<float>(), (int)partial.size(1),
                                     relu, cur_stream());
    return std::make_tuple(dx, dres, dparams);
  });
  m.def("bn_backward", [bn_bwd_args](at::Tensor dy, at::Tensor x, c10::optional<at::Tensor> y, at::Tensor gamma, at::Tensor stats, bool relu,
                                     bool need_dres, at::Tensor partial, at::Tensor counters) {
    Args args("bn_backward");
    bn_bwd_args(args, dy, kStrided, x, y, relu, gamma, stats);
    args("partial", partial, {kF32}, min_numel(0))("counters", counters, {kI32}, min_numel(0));
    args.device();
    const int C = (int)x.size(1);
    const int R = (int)(x.numel() / C);
    size_t pf = 0, cn = 0;
    bn_workspace_sizes(R, C, &pf, &cn);   // reads the device's limits, so after the guard
    args("partial", partial, {kF32}, min_numel((int64_t)pf))("counters", counters, {kI32}, min_numel((int64_t)cn));
    at::Tensor dyc = dy.is_contiguous(at::MemoryFormat::ChannelsLast) ? dy : dy.contiguous(at::MemoryFormat::ChannelsLast);
    at::Tensor dx = at::empty_like(x);
    at::Tensor dres = need_dres ? at::empty_like(x) : at::Tensor();
    at::Tensor dparams = at::empty({4, C}, x.options().dtype(kF32));   // rows: dgamma, dbeta, coef1, coef2
    float* dp = dparams.data_ptr<float>();
    const float* st = stats.data_ptr<float>();
    launch_bn_backward(dyc.data_ptr(), x.data_ptr(), relu ? y->data_ptr() : nullptr, dx.data_ptr(), need_dres ? dres.data_ptr() : nullptr,
                       dtype_of(x), R, C, gamma.data_ptr<float>(), st, st + C, dp, dp + C, dp + 2 * C, partial.data_ptr<float>(),
                       (unsigned int*)counters.data_ptr<int>(), relu, cur_stream());
    return std::make_tuple(dx, dres, dparams);
  });

  // ---- max pooling ------------------------------------------------------------------------------
  m.def("maxpool3x3s2_fwd", [](at::Tensor x) {
    Args args("maxpool3x3s2_fwd");
    args("x", x, {kF32, kBF16}, {kAny, kAny, kAny, kAny}, kChannelsLast);
    args.device();
    const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3);
    const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
    at::Tensor y = at::empty({N, C, OH, OW}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    at::Tensor idx = at::empty({N, C, OH, OW}, x.options().dtype(kU8).memory_format(at::MemoryFormat::ChannelsLast));
    launch_maxpool3x3s2_fwd(x.data_ptr(), y.data_ptr(), idx.data_ptr<uint8_t>(), dtype_of(x), N, H, W, C, cur_stream());
    return std::make_tuple(y, idx);
  });
  m.def("maxpool3x3s2_bwd", [](at::Tensor dy, at::Tensor idx, int64_t H, int64_t W) {
    Args args("maxpool3x3s2_bwd");
    args("dy", dy, {kF32, kBF16}, {kAny, kAny, (H + 1) / 2, (W + 1) / 2}, kStrided)("idx", idx, {kU8}, dy.sizes(), kChannelsLast);
    args.device();
    at::Tensor dyc = dy.is_contiguous(at::MemoryFormat::ChannelsLast) ? dy : dy.contiguous(at::MemoryFormat::ChannelsLast);
    const int N = (int)dy.size(0), C = (int)dy.size(1);
    at::Tensor dx = at::empty({N, C, H, W}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
    launch_maxpool3x3s2_bwd(dyc.data_ptr(), idx.data_ptr<uint8_t>(), dx.data_ptr(), dtype_of(dy), N, (int)H, (int)W, C, cur_stream());
    return dx;
  });

  // ---- input pipeline ---------------------------------------------------------------------------
  m.def("normalize_to_channels_last", [](at::Tensor src, at::Tensor dst, at::Tensor mean, at::Tensor inv_std, double in_scale) {
    Args args("normalize_to_channels_last");
    args("src", src, {kU8, kF32}, {kAny, kAny, kAny, kAny});
    // dst may carry extra (zero-filled) channels: [N, C_out >= C, H, W]
    args("dst", dst, {kBF16, kF32}, {src.size(0), kAny, src.size(2), src.size(3)}, kChannelsLast);
    args.expect(dst.size(1) >= src.size(1), "dst", "channels_last [N, C_out >= C, H, W]", dst);
    args("mean", mean, {kF32}, min_numel(src.size(1)))("inv_std", inv_std, {kF32}, min_numel(src.size(1)));
    args.device();
    launch_normalize_to_channels_last(src.data_ptr(), dtype_of(src), dst.data_ptr(), dtype_of(dst), (int)src.size(0), (int)src.size(1),
                                      (int)dst.size(1), (int)src.size(2), (int)src.size(3), mean.data_ptr<float>(), inv_std.data_ptr<float>(),
                                      (float)in_scale, cur_stream());
  });

  // ---- Vision Transformer patch embedding (vit.cu): images as documents of one token stream ------------------------------
  // The submodule _C.vit holds these entry points; they follow the same argument contract (tests/test_vit_bindings_cpu.py).
  py::module_ vit = m.def_submodule("vit", "Vision Transformer patch embedding (vit.cu)");
  vit.def("patchify", [](at::Tensor images, int64_t patch, int64_t tokens) {
    Args args("patchify");
    args("images", images, {kBF16}, {kAny, kAny, kAny, kAny}, kStrided, 16);
    const bool cl = !images.is_contiguous();
    args.expect(!cl || images.is_contiguous(at::MemoryFormat::ChannelsLast), "images", "contiguous or channels_last", images);
    const int64_t B = images.size(0), C = images.size(1), H = images.size(2), W = images.size(3);
    if (patch < 8 || patch % 8 || H % patch || W % patch)
      args.fail("patch", "a multiple of 8 that divides the image's height and width", std::to_string(patch) + " for " + sizes_str(images.sizes()));
    const int64_t per = (H / patch) * (W / patch) + 1;
    if (tokens < B * per) args.fail("tokens", "at least batch * (patches + 1) = " + std::to_string(B * per), std::to_string(tokens));
    args.device();
    at::Tensor out = at::empty({tokens, C * patch * patch}, images.options().memory_format(at::MemoryFormat::Contiguous));
    launch_patchify(images.data_ptr(), cl, (int)B, (int)C, (int)H, (int)W, (int)patch, (int)tokens, out.data_ptr(), cur_stream());
    return out;
  }, py::arg("images"), py::arg("patch"), py::arg("tokens"));
  vit.def("patch_assemble", [](at::Tensor y, at::Tensor class_token, at::Tensor pos_embedding, int64_t batch) {
    Args args("patch_assemble");
    args("y", y, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t T = y.size(0), D = y.size(1);
    if (D % 8) args.fail("y", "bf16 [T, D] with D % 8 == 0", describe(y));
    args("class_token", class_token, {kBF16}, numel(D), kContiguous, 16)("pos_embedding", pos_embedding, {kBF16}, last_dim(D), kContiguous, 16);
    const int64_t per = pos_embedding.numel() / D;
    if (per < 1 || batch < 0 || batch * per > T)
      args.fail("batch", "at most T / tokens_per_image = " + std::to_string(T / std::max<int64_t>(per, 1)), std::to_string(batch));
    args.device();
    at::Tensor out = at::empty_like(y);
    launch_patch_assemble(y.data_ptr(), class_token.data_ptr(), pos_embedding.data_ptr(), (int)batch, (int)per, (int)D, (int)T, out.data_ptr(),
                          cur_stream());
    return out;
  }, py::arg("y"), py::arg("class_token"), py::arg("pos_embedding"), py::arg("batch"));
  vit.def("patch_embed_bwd", [](at::Tensor dy, int64_t batch, int64_t tokens_per_image) {
    Args args("patch_embed_bwd");
    args("dy", dy, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t T = dy.size(0), D = dy.size(1);
    if (D % 8) args.fail("dy", "bf16 [T, D] with D % 8 == 0", describe(dy));
    if (tokens_per_image < 1 || batch < 0 || batch * tokens_per_image > T)
      args.fail("batch", "batch * tokens_per_image <= T = " + std::to_string(T), std::to_string(batch) + " * " + std::to_string(tokens_per_image));
    args.device();
    at::Tensor dpatch = at::empty_like(dy);
    at::Tensor dpos = at::empty({tokens_per_image, D}, dy.options());
    at::Tensor dcls = at::empty({D}, dy.options());
    launch_patch_embed_bwd(dy.data_ptr(), (int)batch, (int)tokens_per_image, (int)D, (int)T, dpatch.data_ptr(), dpos.data_ptr(), dcls.data_ptr(),
                           cur_stream());
    return std::make_tuple(dpatch, dpos, dcls);
  }, py::arg("dy"), py::arg("batch"), py::arg("tokens_per_image"));

  // ---- CLIP (clip.cu, and QuickGELU in loss.cu): the contrastive loss over the global batch ----------------------------
  // _C.clip is a namespace of static entry points (a class that is never instantiated), not a submodule: the argument-contract
  // tests of the top-level functions and of the vit submodule each list exactly their own bindings, and these have their
  // rows, and their own check that every one has a row, in tests/test_clip_bindings_cpu.py.  Same argument contract.
  py::class_<ClipNamespace> clip(m, "clip", "CLIP contrastive loss and QuickGELU (clip.cu, loss.cu)");
  clip.def_static("quick_gelu_fwd", [](at::Tensor pre) {
    Args args("quick_gelu_fwd");
    args("pre", pre, {kF32, kBF16}, min_numel(0));
    args.device();
    at::Tensor out = at::empty_like(pre);
    launch_gelu(pre.data_ptr(), nullptr, out.data_ptr(), dtype_of(pre), (size_t)pre.numel(), false, cur_stream(), GeluForm::kQuick);
    return out;
  }, py::arg("pre"));
  clip.def_static("quick_gelu_bwd", [](at::Tensor dy, at::Tensor pre) {
    Args args("quick_gelu_bwd");
    args("pre", pre, {kF32, kBF16}, min_numel(0))("dy", dy, {pre.scalar_type()}, numel(pre.numel()));
    args.device();
    at::Tensor out = at::empty_like(pre);
    launch_gelu(pre.data_ptr(), dy.data_ptr(), out.data_ptr(), dtype_of(pre), (size_t)pre.numel(), true, cur_stream(), GeluForm::kQuick);
    return out;
  }, py::arg("dy"), py::arg("pre"));
  clip.def_static("l2norm_fwd", [](at::Tensor x) {
    Args args("l2norm_fwd");
    args("x", x, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t B = x.size(0), D = x.size(1);
    if (B < 1 || D < 8 || D % 8) args.fail("x", "bf16 [B, D] with B >= 1 and D % 8 == 0", describe(x));
    args.device();
    at::Tensor u = at::empty_like(x);
    at::Tensor rnorm = at::empty({B}, x.options().dtype(kF32));
    launch_l2norm_fwd(x.data_ptr(), (int)B, (int)D, u.data_ptr(), rnorm.data_ptr<float>(), cur_stream());
    return std::make_tuple(u, rnorm);
  }, py::arg("x"));
  clip.def_static("l2norm_bwd", [](at::Tensor du, at::Tensor x, at::Tensor rnorm) {
    Args args("l2norm_bwd");
    args("x", x, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t B = x.size(0), D = x.size(1);
    if (B < 1 || D < 8 || D % 8) args.fail("x", "bf16 [B, D] with B >= 1 and D % 8 == 0", describe(x));
    args("du", du, {kBF16}, {B, D}, kContiguous, 16)("rnorm", rnorm, {kF32}, {B});
    args.device();
    at::Tensor dx = at::empty_like(x);
    launch_l2norm_bwd(du.data_ptr(), x.data_ptr(), rnorm.data_ptr<float>(), (int)B, (int)D, dx.data_ptr(), cur_stream());
    return dx;
  }, py::arg("du"), py::arg("x"), py::arg("rnorm"));
  // (loss fp32 [], dscale fp32 [], dz_img bf16 [B, N], dz_txt bf16 [B, N])
  clip.def_static("contrastive_xent", [](at::Tensor z_img, at::Tensor z_txt, at::Tensor logit_scale, int64_t label_offset) {
    Args args("contrastive_xent");
    args("z_img", z_img, {kF32}, {kAny, kAny});
    const int64_t B = z_img.size(0), N = z_img.size(1);
    if (B < 1 || N < B) args.fail("z_img", "fp32 [B, N] with 1 <= B <= N", describe(z_img));
    args("z_txt", z_txt, {kF32}, {B, N})("logit_scale", logit_scale, {kF32}, numel(1));
    if (label_offset < 0 || label_offset + B > N)
      args.fail("label_offset", "in [0, N - B] = [0, " + std::to_string(N - B) + "]", std::to_string(label_offset));
    args.device();
    at::Tensor dz_img = at::empty({B, N}, z_img.options().dtype(kBF16));
    at::Tensor dz_txt = at::empty({B, N}, z_img.options().dtype(kBF16));
    at::Tensor partials = at::empty({4 * B}, z_img.options());
    at::Tensor loss = at::empty({}, z_img.options());
    at::Tensor dscale = at::empty({}, z_img.options());
    launch_contrastive_xent(z_img.data_ptr<float>(), z_txt.data_ptr<float>(), logit_scale.data_ptr<float>(), (int)B, (int)N, (int)label_offset,
                            dz_img.data_ptr(), dz_txt.data_ptr(), partials.data_ptr<float>(), loss.data_ptr<float>(), dscale.data_ptr<float>(),
                            cur_stream());
    return std::make_tuple(loss, dscale, dz_img, dz_txt);
  }, py::arg("z_img"), py::arg("z_txt"), py::arg("logit_scale"), py::arg("label_offset"));

  // ---- cross-attention (cross_attention.cu): decoder queries over another sequence's keys and values, head dim 64 ------
  // _C.cross is a namespace of static entry points like _C.clip; its contract rows are in tests/test_cross_bindings_cpu.py.
  // q bf16 [B*Sq, heads*64], kv bf16 [B*Sk, 2*heads*64] (key | value), q_bounds int32 [B, Sq, 2], kv_bounds int32
  // [B, Sk, 2]; Sq, Sk multiples of 128 (the launcher checks them).
  py::class_<CrossNamespace> cross(m, "cross", "Cross-attention of an encoder-decoder (cross_attention.cu)");
  // (o bf16 [B*Sq, heads*64], lse fp32 [B, heads, Sq])
  cross.def_static("cross_attention_fwd", [](at::Tensor q, at::Tensor kv, at::Tensor q_bounds, int heads) {
    Args args("cross_attention_fwd");
    const auto [B, Sq, Sk] = cross_args(args, q, kv, q_bounds, heads);
    args.device();
    at::Tensor o = at::empty_like(q);
    at::Tensor lse = at::empty({B, heads, Sq}, q.options().dtype(kF32));
    launch_cross_attention_fwd(q.data_ptr(), kv.data_ptr(), q_bounds.data_ptr<int>(), B, Sq, Sk, heads, o.data_ptr(), lse.data_ptr<float>(),
                               cur_stream());
    return std::make_tuple(o, lse);
  }, py::arg("q"), py::arg("kv"), py::arg("q_bounds"), py::arg("heads"));
  // (dq like q, dkv like kv)
  cross.def_static("cross_attention_bwd", [](at::Tensor dout, at::Tensor q, at::Tensor kv, at::Tensor o, at::Tensor lse,
                                                       at::Tensor q_bounds, at::Tensor kv_bounds, int heads) {
    Args args("cross_attention_bwd");
    const auto [B, Sq, Sk] = cross_args(args, q, kv, q_bounds, heads);
    args("kv_bounds", kv_bounds, {kI32}, {B, Sk, 2}, kContiguous, 8);
    args("dout", dout, {kBF16}, numel(q.numel()), kContiguous, 16)("o", o, {kBF16}, numel(q.numel()), kContiguous, 16);
    args("lse", lse, {kF32}, numel((int64_t)B * heads * Sq), kContiguous, 8);
    args.device();
    at::Tensor dq = at::empty_like(q);
    at::Tensor dkv = at::empty_like(kv);
    at::Tensor dsum = at::empty({B, heads, Sq}, q.options().dtype(kF32));
    launch_cross_attention_bwd(dout.data_ptr(), q.data_ptr(), kv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), q_bounds.data_ptr<int>(),
                               kv_bounds.data_ptr<int>(), B, Sq, Sk, heads, dsum.data_ptr<float>(), dq.data_ptr(), dkv.data_ptr(), cur_stream());
    return std::make_tuple(dq, dkv);
  }, py::arg("dout"), py::arg("q"), py::arg("kv"), py::arg("o"), py::arg("lse"), py::arg("q_bounds"), py::arg("kv_bounds"), py::arg("heads"));

  // ---- T5's relative position bias (attention.cu): document attention with a learned bias table, head dim 64 ---------
  // _C.t5 is a namespace of static entry points like _C.cross; its contract rows are in tests/test_t5_bindings_cpu.py.
  // qkv bf16 [B*S, 3*heads*64], bounds int32 [B, S, 2] (segment, or causal inside documents), table fp32 [heads, 257]
  // (launch_relative_attention_fwd); S a multiple of 128 (the launcher checks it).
  py::class_<T5Namespace> t5(m, "t5", "T5's relative position bias inside the attention kernels (attention.cu)");
  // (o bf16 [B*S, heads*64], lse fp32 [B, heads, S])
  t5.def_static("relative_attention_fwd", [](at::Tensor qkv, at::Tensor bounds, at::Tensor table, int heads, bool causal) {
    Args args("relative_attention_fwd");
    const auto [B, S] = relative_args(args, qkv, bounds, table, heads);
    args.device();
    at::Tensor o = at::empty({qkv.size(0), (int64_t)heads * 64}, qkv.options());
    at::Tensor lse = at::empty({B, heads, S}, qkv.options().dtype(kF32));
    launch_relative_attention_fwd(qkv.data_ptr(), bounds.data_ptr<int>(), table.data_ptr<float>(), B, S, heads, causal, o.data_ptr(),
                                  lse.data_ptr<float>(), cur_stream());
    return std::make_tuple(o, lse);
  }, py::arg("qkv"), py::arg("bounds"), py::arg("table"), py::arg("heads"), py::arg("causal"));
  // (dqkv like qkv, dtable fp32 [heads, 257])
  t5.def_static("relative_attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor bounds,
                                             at::Tensor table, int heads, bool causal) {
    Args args("relative_attention_bwd");
    const auto [B, S] = relative_args(args, qkv, bounds, table, heads);
    args("dout", dout, {kBF16}, numel(qkv.size(0) * heads * 64), kContiguous, 16)("o", o, {kBF16}, numel(qkv.size(0) * heads * 64), kContiguous, 16);
    args("lse", lse, {kF32}, numel((int64_t)B * heads * S), kContiguous, 8);
    args.device();
    at::Tensor dqkv = at::empty_like(qkv);
    at::Tensor dtable = at::empty({heads, 257}, qkv.options().dtype(kF32));
    at::Tensor dsum = at::empty({B, heads, S}, qkv.options().dtype(kF32));
    at::Tensor part = at::empty({B, S / 128, heads, 257}, qkv.options().dtype(kF32));
    launch_relative_attention_bwd(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), bounds.data_ptr<int>(),
                                  table.data_ptr<float>(), B, S, heads, causal, dsum.data_ptr<float>(), part.data_ptr<float>(),
                                  dqkv.data_ptr(), dtable.data_ptr<float>(), cur_stream());
    return std::make_tuple(dqkv, dtable);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("bounds"), py::arg("table"), py::arg("heads"), py::arg("causal"));
  // table fp32 [H, 257] = weight[bucket[c], h]: weight fp32 or bf16 [num_buckets, H], bucket int32 [257] in [0, num_buckets)
  t5.def_static("relative_table_fwd", [](at::Tensor weight, at::Tensor bucket) {
    Args args("relative_table_fwd");
    args("weight", weight, {kF32, kBF16}, {kAny, kAny})("bucket", bucket, {kI32}, {257});
    args.expect(weight.size(0) >= 1 && weight.size(1) >= 1, "weight", "[num_buckets, heads] with both >= 1", weight);
    args.device();
    at::Tensor table = at::empty({weight.size(1), 257}, weight.options().dtype(kF32));
    launch_relative_table_fwd(weight.data_ptr(), weight.scalar_type() == kBF16, bucket.data_ptr<int>(), (int)weight.size(1),
                              table.data_ptr<float>(), cur_stream());
    return table;
  }, py::arg("weight"), py::arg("bucket"));
  // d weight like weight: the sum of dtable[h, c] over the c of each bucket, in increasing c
  t5.def_static("relative_table_bwd", [](at::Tensor dtable, at::Tensor bucket, at::Tensor weight) {
    Args args("relative_table_bwd");
    args("weight", weight, {kF32, kBF16}, {kAny, kAny});
    args.expect(weight.size(0) >= 1 && weight.size(1) >= 1, "weight", "[num_buckets, heads] with both >= 1", weight);
    args("dtable", dtable, {kF32}, {weight.size(1), 257})("bucket", bucket, {kI32}, {257});
    args.device();
    at::Tensor dweight = at::empty_like(weight, at::MemoryFormat::Contiguous);
    launch_relative_table_bwd(dtable.data_ptr<float>(), bucket.data_ptr<int>(), (int)weight.size(0), (int)weight.size(1),
                              weight.scalar_type() == kBF16, dweight.data_ptr(), cur_stream());
    return dweight;
  }, py::arg("dtable"), py::arg("bucket"), py::arg("weight"));

  // ---- ConvNeXt's depthwise 7x7 convolution, stride 1, padding 3 (convnext.cu), bf16 NHWC --------------------------------
  // _C.convnext is a namespace of static entry points like _C.t5; its contract rows are in tests/test_convnext_bindings_cpu.py.
  // x, dy [B, H, W, C]; weight bf16 [C, 49] (the memory of a contiguous or channels_last [C, 1, 7, 7]); bias bf16 [C].
  py::class_<ConvNextNamespace> convnext(m, "convnext", "ConvNeXt's depthwise 7x7 convolution on NHWC activations (convnext.cu)");
  convnext.def_static("dwconv_fwd", [](at::Tensor x, at::Tensor weight, at::Tensor bias) {
    Args args("dwconv_fwd");
    const auto [B, H, W, C] = dwconv_args(args, "x", x);
    args("weight", weight, {kBF16}, {C, 49})("bias", bias, {kBF16}, {C});
    args.device();
    at::Tensor y = at::empty_like(x);
    launch_dwconv_fwd(x.data_ptr(), weight.data_ptr(), bias.data_ptr(), B, H, W, C, y.data_ptr(), cur_stream());
    return y;
  }, py::arg("x"), py::arg("weight"), py::arg("bias"));
  convnext.def_static("dwconv_dgrad", [](at::Tensor dy, at::Tensor weight) {
    Args args("dwconv_dgrad");
    const auto [B, H, W, C] = dwconv_args(args, "dy", dy);
    args("weight", weight, {kBF16}, {C, 49});
    args.device();
    at::Tensor dx = at::empty_like(dy);
    launch_dwconv_dgrad(dy.data_ptr(), weight.data_ptr(), B, H, W, C, dx.data_ptr(), cur_stream());
    return dx;
  }, py::arg("dy"), py::arg("weight"));
  // (dweight bf16 [C, 49], dbias bf16 [C])
  convnext.def_static("dwconv_wgrad", [](at::Tensor dy, at::Tensor x) {
    Args args("dwconv_wgrad");
    const auto [B, H, W, C] = dwconv_args(args, "x", x);
    args("dy", dy, {kBF16}, {B, H, W, C}, kContiguous, 16);
    args.device();
    at::Tensor part = at::empty({(int64_t)dwconv_wgrad_slots(B, H, W), 50, C}, x.options().dtype(kF32));
    at::Tensor dweight = at::empty({C, 49}, x.options());
    at::Tensor dbias = at::empty({C}, x.options());
    launch_dwconv_wgrad(dy.data_ptr(), x.data_ptr(), B, H, W, C, part.data_ptr<float>(), dweight.data_ptr(), dbias.data_ptr(), cur_stream());
    return std::make_tuple(dweight, dbias);
  }, py::arg("dy"), py::arg("x"));

  // ---- Swin's shifted-window attention, window 7, head dim 32 (swin.cu), bf16 raster rows ---------------------------------
  // _C.swin is a namespace of static entry points like _C.convnext; its contract rows are in tests/test_swin_bindings_cpu.py.
  // qkv [B H W, 3C] (C = 32 heads), table fp32 [169, heads], o and dout [B H W, C], lse fp32 [B H W, heads].
  py::class_<SwinNamespace> swin(m, "swin", "Swin's shifted-window attention on raster token rows (swin.cu)");
  // (o bf16 [B H W, C], lse fp32 [B H W, heads])
  swin.def_static("attention_fwd", [](at::Tensor qkv, at::Tensor table, int64_t batch, int64_t height, int64_t width, int64_t shift_y,
                                      int64_t shift_x) {
    Args args("attention_fwd");
    const auto [rows, heads] = swin_args(args, qkv, table, batch, height, width, shift_y, shift_x);
    args.device();
    at::Tensor o = at::empty({rows, 32 * heads}, qkv.options());
    at::Tensor lse = at::empty({rows, heads}, qkv.options().dtype(kF32));
    launch_swin_attention_fwd(qkv.data_ptr(), table.data_ptr<float>(), (int)batch, (int)height, (int)width, (int)heads, (int)shift_y,
                              (int)shift_x, o.data_ptr(), lse.data_ptr<float>(), cur_stream());
    return std::make_tuple(o, lse);
  }, py::arg("qkv"), py::arg("table"), py::arg("batch"), py::arg("height"), py::arg("width"), py::arg("shift_y"), py::arg("shift_x"));
  // (dqkv bf16 [B H W, 3C], dtable fp32 [169, heads])
  swin.def_static("attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor table, int64_t batch,
                                      int64_t height, int64_t width, int64_t shift_y, int64_t shift_x) {
    Args args("attention_bwd");
    const auto [rows, heads] = swin_args(args, qkv, table, batch, height, width, shift_y, shift_x);
    args("dout", dout, {kBF16}, {rows, 32 * heads}, kContiguous, 16)("o", o, {kBF16}, {rows, 32 * heads}, kContiguous, 16)
        ("lse", lse, {kF32}, {rows, heads});
    args.device();
    const int windows = swin_windows((int)batch, (int)height, (int)width);
    at::Tensor dqkv = at::empty_like(qkv);
    at::Tensor part = at::empty({heads, (int64_t)windows, 169}, qkv.options().dtype(kF32));
    at::Tensor dtable = at::empty({169, heads}, qkv.options().dtype(kF32));
    launch_swin_attention_bwd(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), table.data_ptr<float>(), (int)batch,
                              (int)height, (int)width, (int)heads, (int)shift_y, (int)shift_x, dqkv.data_ptr(), part.data_ptr<float>(),
                              dtable.data_ptr<float>(), cur_stream());
    return std::make_tuple(dqkv, dtable);
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("table"), py::arg("batch"), py::arg("height"),
     py::arg("width"), py::arg("shift_y"), py::arg("shift_x"));

  // ---- Swin V2's cosine shifted-window attention, window 8, head dim 32 (swin.cu), bf16 raster rows -----------------------
  // _C.swin_v2 is a namespace of static entry points like _C.swin; its contract rows are in tests/test_swin_v2_bindings_cpu.py.
  // qkv [B H W, 3C] (C = 32 heads), table fp32 [225, heads] (16 sigmoid of the cpb MLP), scale fp32 [heads] (exp of the
  // clamped logit_scale), o and dout [B H W, C], lse fp32 [B H W, heads].
  py::class_<SwinV2Namespace> swin_v2(m, "swin_v2", "Swin V2's cosine shifted-window attention on raster token rows (swin.cu)");
  // (o bf16 [B H W, C], lse fp32 [B H W, heads])
  swin_v2.def_static("attention_fwd", [](at::Tensor qkv, at::Tensor table, at::Tensor scale, int64_t batch, int64_t height, int64_t width,
                                         int64_t shift_y, int64_t shift_x) {
    Args args("attention_fwd");
    const auto [rows, heads] = swin_v2_args(args, qkv, table, scale, batch, height, width, shift_y, shift_x);
    args.device();
    at::Tensor o = at::empty({rows, 32 * heads}, qkv.options());
    at::Tensor lse = at::empty({rows, heads}, qkv.options().dtype(kF32));
    launch_swin_v2_attention_fwd(qkv.data_ptr(), table.data_ptr<float>(), scale.data_ptr<float>(), (int)batch, (int)height, (int)width,
                                 (int)heads, (int)shift_y, (int)shift_x, o.data_ptr(), lse.data_ptr<float>(), cur_stream());
    return std::make_tuple(o, lse);
  }, py::arg("qkv"), py::arg("table"), py::arg("scale"), py::arg("batch"), py::arg("height"), py::arg("width"), py::arg("shift_y"),
     py::arg("shift_x"));
  // (dqkv bf16 [B H W, 3C], dtable fp32 [225, heads], dscale fp32 [heads])
  swin_v2.def_static("attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, at::Tensor table, at::Tensor scale,
                                         int64_t batch, int64_t height, int64_t width, int64_t shift_y, int64_t shift_x) {
    Args args("attention_bwd");
    const auto [rows, heads] = swin_v2_args(args, qkv, table, scale, batch, height, width, shift_y, shift_x);
    args("dout", dout, {kBF16}, {rows, 32 * heads}, kContiguous, 16)("o", o, {kBF16}, {rows, 32 * heads}, kContiguous, 16)
        ("lse", lse, {kF32}, {rows, heads});
    args.device();
    const int windows = swin_v2_windows((int)batch, (int)height, (int)width);
    at::Tensor dqkv = at::empty_like(qkv);
    at::Tensor part = at::empty({heads, (int64_t)windows, 226}, qkv.options().dtype(kF32));
    at::Tensor grads = at::empty({226, heads}, qkv.options().dtype(kF32));   // the 225 table rows, then d scale
    launch_swin_v2_attention_bwd(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), table.data_ptr<float>(),
                                 scale.data_ptr<float>(), (int)batch, (int)height, (int)width, (int)heads, (int)shift_y, (int)shift_x,
                                 dqkv.data_ptr(), part.data_ptr<float>(), grads.data_ptr<float>(), cur_stream());
    return std::make_tuple(dqkv, grads.narrow(0, 0, 225), grads.select(0, 225));
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("table"), py::arg("scale"), py::arg("batch"), py::arg("height"),
     py::arg("width"), py::arg("shift_y"), py::arg("shift_x"));

  // ---- Mamba's causal conv1d + SiLU and selective scan (mamba.cu), bf16 token rows ----------------------------------------
  // _C.mamba is a namespace of static entry points like _C.swin; its contract rows are in tests/test_mamba_bindings_cpu.py.
  // bounds int32 [B, S, 2], xz bf16 [B S, 2E] = x | z, conv weight fp32 [E, 4] and bias fp32 [E], u / draw / y bf16 [B S, E],
  // xbc bf16 [B S, R + 32] = dt | B | C, A_log fp32 [E, 16], D / dt_bias fp32 [E].
  py::class_<MambaNamespace> mamba(m, "mamba", "Mamba's causal conv1d and selective scan on token rows (mamba.cu)");
  // u bf16 [B S, E]
  mamba.def_static("conv_fwd", [](at::Tensor xz, at::Tensor weight, at::Tensor bias, at::Tensor bounds) {
    Args args("conv_fwd");
    const auto [B, S, E] = mamba_args(args, bounds, xz);
    args("weight", weight, {kF32}, {E, 4}, kContiguous, 16)("bias", bias, {kF32}, {E});
    args.device();
    at::Tensor u = at::empty({B * S, E}, xz.options());
    launch_mamba_conv_fwd(xz.data_ptr(), weight.data_ptr<float>(), bias.data_ptr<float>(), bounds.data_ptr<int>(), (int)B, (int)S, (int)E,
                          u.data_ptr(), cur_stream());
    return u;
  }, py::arg("xz"), py::arg("weight"), py::arg("bias"), py::arg("bounds"));
  // (dxz bf16 [B S, 2E] with the x half written: dxz_out when given, whose z half is left as it is; dweight fp32 [E, 4];
  // dbias fp32 [E])
  mamba.def_static("conv_bwd", [](at::Tensor du, at::Tensor xz, at::Tensor weight, at::Tensor bias, at::Tensor bounds,
                                  c10::optional<at::Tensor> dxz_out) {
    Args args("conv_bwd");
    const auto [B, S, E] = mamba_args(args, bounds, xz);
    args("du", du, {kBF16}, {B * S, E}, kContiguous, 16)("weight", weight, {kF32}, {E, 4}, kContiguous, 16)("bias", bias, {kF32}, {E});
    at::Tensor dxz;
    args.out(dxz, "dxz_out", dxz_out, {B * S, 2 * E}, xz.options(), 16);
    args.device();
    at::Tensor part = at::empty({(int64_t)mamba_conv_blocks((int)B, (int)S), 5, E}, xz.options().dtype(kF32));
    at::Tensor dweight = at::empty({E, 4}, xz.options().dtype(kF32));
    at::Tensor dbias = at::empty({E}, xz.options().dtype(kF32));
    launch_mamba_conv_bwd(du.data_ptr(), xz.data_ptr(), weight.data_ptr<float>(), bias.data_ptr<float>(), bounds.data_ptr<int>(), (int)B,
                          (int)S, (int)E, dxz.data_ptr(), part.data_ptr<float>(), dweight.data_ptr<float>(), dbias.data_ptr<float>(),
                          cur_stream());
    return std::make_tuple(dxz.view({B * S, 2 * E}), dweight, dbias);
  }, py::arg("du"), py::arg("xz"), py::arg("weight"), py::arg("bias"), py::arg("bounds"), py::arg("dxz_out") = py::none());
  // (y bf16 [B S, E], hstart fp32 [B, chunks, E, 16], sumd fp32 [B, chunks, E]), chunks = ceil(S / 128)
  mamba.def_static("scan_fwd", [](at::Tensor u, at::Tensor draw, at::Tensor xbc, at::Tensor xz, at::Tensor A_log, at::Tensor D,
                                  at::Tensor dt_bias, at::Tensor bounds) {
    Args args("scan_fwd");
    const auto [B, S, E] = mamba_args(args, bounds, xz);
    const int64_t R = mamba_scan_args(args, B * S, E, u, draw, xbc, A_log, D, dt_bias);
    args.device();
    const int64_t nc = mamba_chunks((int)S);
    at::Tensor y = at::empty({B * S, E}, xz.options());
    at::Tensor hst = at::empty({B, nc, E, 16}, xz.options().dtype(kF32));
    at::Tensor sumd = at::empty({B, nc, E}, xz.options().dtype(kF32));
    launch_mamba_scan_fwd(u.data_ptr(), draw.data_ptr(), xbc.data_ptr(), xz.data_ptr(), A_log.data_ptr<float>(), D.data_ptr<float>(),
                          dt_bias.data_ptr<float>(), bounds.data_ptr<int>(), (int)B, (int)S, (int)E, (int)R, y.data_ptr(), hst.data_ptr<float>(),
                          sumd.data_ptr<float>(), cur_stream());
    return std::make_tuple(y, hst, sumd);
  }, py::arg("u"), py::arg("draw"), py::arg("xbc"), py::arg("xz"), py::arg("A_log"), py::arg("D"), py::arg("dt_bias"), py::arg("bounds"));
  // (du bf16 [B S, E], ddraw bf16 [B S, E], dxbc bf16 [B S, R + 32] with zero dt columns, dxz bf16 [B S, 2E] with the z half
  // written and the x half left for conv_bwd, dA_log fp32 [E, 16], dD fp32 [E], ddt_bias fp32 [E])
  mamba.def_static("scan_bwd", [](at::Tensor dy, at::Tensor u, at::Tensor draw, at::Tensor xbc, at::Tensor xz, at::Tensor A_log, at::Tensor D,
                                  at::Tensor dt_bias, at::Tensor bounds, at::Tensor hstart, at::Tensor sumd) {
    Args args("scan_bwd");
    const auto [B, S, E] = mamba_args(args, bounds, xz);
    const int64_t R = mamba_scan_args(args, B * S, E, u, draw, xbc, A_log, D, dt_bias);
    const int64_t nc = mamba_chunks((int)S), groups = mamba_groups((int)E);
    args("dy", dy, {kBF16}, {B * S, E})("hstart", hstart, {kF32}, {B, nc, E, 16})("sumd", sumd, {kF32}, {B, nc, E});
    args.device();
    const auto f32 = xz.options().dtype(kF32);
    at::Tensor dq = at::empty({B, nc, E, 16}, f32), dbc_part = at::empty({B * S, groups, 32}, f32);
    at::Tensor dA_part = at::empty({B * nc, E, 16}, f32), dD_part = at::empty({B * nc, E}, f32), dbias_part = at::empty({B * nc, E}, f32);
    at::Tensor du = at::empty({B * S, E}, xz.options()), ddraw = at::empty({B * S, E}, xz.options());
    at::Tensor dxbc = at::empty({B * S, R + 32}, xz.options()), dxz = at::empty({B * S, 2 * E}, xz.options());
    at::Tensor dA_log = at::empty({E, 16}, f32), dD = at::empty({E}, f32), dbias = at::empty({E}, f32);
    launch_mamba_scan_bwd(dy.data_ptr(), u.data_ptr(), draw.data_ptr(), xbc.data_ptr(), xz.data_ptr(), A_log.data_ptr<float>(),
                          D.data_ptr<float>(), dt_bias.data_ptr<float>(), bounds.data_ptr<int>(), hstart.data_ptr<float>(), sumd.data_ptr<float>(),
                          (int)B, (int)S, (int)E, (int)R, dq.data_ptr<float>(), dbc_part.data_ptr<float>(), dA_part.data_ptr<float>(),
                          dD_part.data_ptr<float>(), dbias_part.data_ptr<float>(), du.data_ptr(), ddraw.data_ptr(), dxbc.data_ptr(), dxz.data_ptr(),
                          dA_log.data_ptr<float>(), dD.data_ptr<float>(), dbias.data_ptr<float>(), cur_stream());
    return std::make_tuple(du, ddraw, dxbc, dxz, dA_log, dD, dbias);
  }, py::arg("dy"), py::arg("u"), py::arg("draw"), py::arg("xbc"), py::arg("xz"), py::arg("A_log"), py::arg("D"), py::arg("dt_bias"),
     py::arg("bounds"), py::arg("hstart"), py::arg("sumd"));

  // ---- Mamba-2's conv, SSD and gated RMSNorm (mamba.cu, mamba2.cu, layernorm.cu), bf16 token rows ----------------------------
  // _C.mamba2 is a namespace of static entry points like _C.mamba; its contract rows are in tests/test_mamba2_bindings_cpu.py.
  // Row views (x, dx_out, dt, ddt_out, z, dz_out) are read and written in place through their row pitch (row_view).
  py::class_<Mamba2Namespace> mamba2(m, "mamba2", "Mamba-2's causal conv1d, chunked SSD scan and gated RMSNorm on token rows");
  // u bf16 [B S, C] = silu(conv(x) + bias) of the row view x [B S, C], C % 8 == 0; weight fp32 [C, 4], bias fp32 [C]
  mamba2.def_static("conv_fwd", [](at::Tensor x, at::Tensor weight, at::Tensor bias, at::Tensor bounds) {
    Args args("conv_fwd");
    const auto [B, S] = mamba2_bounds(args, bounds);
    args("x", x, {kBF16}, {B * S, kAny}, kStrided);
    const int64_t C = x.size(1);
    if (C < 8 || C % 8) args.fail("x", "a bf16 [B S, C] row view with C a positive multiple of 8", describe(x));
    const int64_t xp = row_view(args, "x", x, B * S, C);
    args("weight", weight, {kF32}, {C, 4}, kContiguous, 16)("bias", bias, {kF32}, {C});
    args.device();
    at::Tensor u = at::empty({B * S, C}, x.options().memory_format(at::MemoryFormat::Contiguous));
    launch_mamba2_conv_fwd(x.data_ptr(), xp, weight.data_ptr<float>(), bias.data_ptr<float>(), bounds.data_ptr<int>(), (int)B, (int)S, (int)C,
                           u.data_ptr(), cur_stream());
    return u;
  }, py::arg("x"), py::arg("weight"), py::arg("bias"), py::arg("bounds"));
  // (dx bf16 [B S, C]: dx_out when given (a row view, written in place and returned), else a new contiguous tensor;
  // dweight fp32 [C, 4]; dbias fp32 [C])
  mamba2.def_static("conv_bwd", [](at::Tensor du, at::Tensor x, at::Tensor weight, at::Tensor bias, at::Tensor bounds,
                                   c10::optional<at::Tensor> dx_out) {
    Args args("conv_bwd");
    const auto [B, S] = mamba2_bounds(args, bounds);
    args("x", x, {kBF16}, {B * S, kAny}, kStrided);
    const int64_t C = x.size(1);
    if (C < 8 || C % 8) args.fail("x", "a bf16 [B S, C] row view with C a positive multiple of 8", describe(x));
    const int64_t xp = row_view(args, "x", x, B * S, C);
    args("du", du, {kBF16}, {B * S, C}, kContiguous, 16)("weight", weight, {kF32}, {C, 4}, kContiguous, 16)("bias", bias, {kF32}, {C});
    const int64_t dxp = dx_out.has_value() ? row_view(args, "dx_out", *dx_out, B * S, C) : C;
    args.device();
    at::Tensor dx = dx_out.has_value() ? *dx_out : at::empty({B * S, C}, du.options());
    const auto f32 = du.options().dtype(kF32);
    at::Tensor part = at::empty({(int64_t)mamba_conv_blocks((int)B, (int)S), 5, C}, f32);
    at::Tensor dweight = at::empty({C, 4}, f32), dbias = at::empty({C}, f32);
    launch_mamba2_conv_bwd(du.data_ptr(), x.data_ptr(), xp, weight.data_ptr<float>(), bias.data_ptr<float>(), bounds.data_ptr<int>(), (int)B,
                           (int)S, (int)C, dx.data_ptr(), dxp, part.data_ptr<float>(), dweight.data_ptr<float>(), dbias.data_ptr<float>(),
                           cur_stream());
    return std::make_tuple(dx, dweight, dbias);
  }, py::arg("du"), py::arg("x"), py::arg("weight"), py::arg("bias"), py::arg("bounds"), py::arg("dx_out") = py::none());
  // y bf16 [B S, 64 H]; the chunk states are scratch of this call (the backward recomputes them)
  mamba2.def_static("ssd_fwd", [](at::Tensor xbc, at::Tensor dt, at::Tensor A_log, at::Tensor D, at::Tensor dt_bias, at::Tensor bounds) {
    Args args("ssd_fwd");
    const auto [B, S, H, dtp] = ssd_args(args, xbc, dt, A_log, D, dt_bias, bounds);
    args.device();
    const int64_t nc = ssd_chunks((int)S);
    const auto f32 = xbc.options().dtype(kF32);
    at::Tensor states = at::empty({B, nc, H, 128, 64}, f32), dec = at::empty({B, nc, H}, f32);
    at::Tensor y = at::empty({B * S, 64 * H}, xbc.options());
    launch_ssd_fwd(xbc.data_ptr(), dt.data_ptr(), dtp, A_log.data_ptr<float>(), D.data_ptr<float>(), dt_bias.data_ptr<float>(),
                   bounds.data_ptr<int>(), (int)B, (int)S, (int)H, states.data_ptr<float>(), dec.data_ptr<float>(), y.data_ptr(), cur_stream());
    return y;
  }, py::arg("xbc"), py::arg("dt"), py::arg("A_log"), py::arg("D"), py::arg("dt_bias"), py::arg("bounds"));
  // (dxbc bf16 [B S, 64 H + 256], ddt bf16 [B S, H] (ddt_out when given: a row view, written in place and returned; the
  // gradient of dt through the softplus), dA_log, dD, ddt_bias fp32 [H])
  mamba2.def_static("ssd_bwd", [](at::Tensor dy, at::Tensor xbc, at::Tensor dt, at::Tensor A_log, at::Tensor D, at::Tensor dt_bias,
                                  at::Tensor bounds, c10::optional<at::Tensor> ddt_out) {
    Args args("ssd_bwd");
    const auto [B, S, H, dtp] = ssd_args(args, xbc, dt, A_log, D, dt_bias, bounds);
    args("dy", dy, {kBF16}, {B * S, 64 * H}, kContiguous, 16);
    const int64_t ddtp = ddt_out.has_value() ? row_view(args, "ddt_out", *ddt_out, B * S, H) : H;
    args.device();
    const int64_t nc = ssd_chunks((int)S);
    const auto f32 = xbc.options().dtype(kF32);
    at::Tensor states = at::empty({B, nc, H, 128, 64}, f32), gstates = at::empty({B, nc, H, 128, 64}, f32), dec = at::empty({B, nc, H}, f32);
    at::Tensor dA_part = at::empty({B * nc, H}, f32), dD_part = at::empty({B * nc, H}, f32), dbias_part = at::empty({B * nc, H}, f32);
    at::Tensor dxbc = at::empty_like(xbc), ddt = ddt_out.has_value() ? *ddt_out : at::empty({B * S, H}, xbc.options());
    at::Tensor dA_log = at::empty({H}, f32), dD = at::empty({H}, f32), dbias = at::empty({H}, f32);
    launch_ssd_bwd(dy.data_ptr(), xbc.data_ptr(), dt.data_ptr(), dtp, A_log.data_ptr<float>(), D.data_ptr<float>(), dt_bias.data_ptr<float>(),
                   bounds.data_ptr<int>(), (int)B, (int)S, (int)H, states.data_ptr<float>(), gstates.data_ptr<float>(), dec.data_ptr<float>(),
                   dA_part.data_ptr<float>(), dD_part.data_ptr<float>(), dbias_part.data_ptr<float>(), dxbc.data_ptr(), ddt.data_ptr(), ddtp,
                   dA_log.data_ptr<float>(), dD.data_ptr<float>(), dbias.data_ptr<float>(), cur_stream());
    return std::make_tuple(dxbc, ddt, dA_log, dD, dbias);
  }, py::arg("dy"), py::arg("xbc"), py::arg("dt"), py::arg("A_log"), py::arg("D"), py::arg("dt_bias"), py::arg("bounds"),
     py::arg("ddt_out") = py::none());
  // (out bf16 [rows, E] = weight * rmsnorm(y * silu(z)), rstd fp32 [rows]); y bf16 [rows, E] contiguous, z a row view, weight
  // bf16 [E], 1024 < E <= 4096, E % 8 == 0
  mamba2.def_static("gated_norm_fwd", [](at::Tensor y, at::Tensor z, at::Tensor weight, double eps) {
    Args args("gated_norm_fwd");
    args("y", y, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t rows = y.size(0), E = y.size(1);
    if (rows < 1 || !gated_rmsnorm_supported((int)E) || rows * E >= (1ll << 31))
      args.fail("y", "bf16 [rows, E] with rows >= 1, E % 8 == 0, 1024 < E <= 4096 and fewer than 2^31 elements", describe(y));
    const int64_t zp = row_view(args, "z", z, rows, E);
    args("weight", weight, {kBF16}, {E}, kContiguous, 16);
    args.device();
    at::Tensor out = at::empty_like(y), rstd = at::empty({rows}, y.options().dtype(kF32));
    launch_gated_rmsnorm_fwd(y.data_ptr(), z.data_ptr(), zp, weight.data_ptr(), (int)rows, (int)E, (float)eps, out.data_ptr(),
                             rstd.data_ptr<float>(), cur_stream());
    return std::make_tuple(out, rstd);
  }, py::arg("y"), py::arg("z"), py::arg("weight"), py::arg("eps"));
  // (dy bf16 [rows, E], dz bf16 [rows, E] (dz_out when given: a row view, written in place and returned), dweight bf16 [E])
  mamba2.def_static("gated_norm_bwd", [](at::Tensor dout, at::Tensor y, at::Tensor z, at::Tensor weight, at::Tensor rstd,
                                         c10::optional<at::Tensor> dz_out) {
    Args args("gated_norm_bwd");
    args("y", y, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t rows = y.size(0), E = y.size(1);
    if (rows < 1 || !gated_rmsnorm_supported((int)E) || rows * E >= (1ll << 31))
      args.fail("y", "bf16 [rows, E] with rows >= 1, E % 8 == 0, 1024 < E <= 4096 and fewer than 2^31 elements", describe(y));
    args("dout", dout, {kBF16}, {rows, E}, kContiguous, 16);
    const int64_t zp = row_view(args, "z", z, rows, E);
    args("weight", weight, {kBF16}, {E}, kContiguous, 16)("rstd", rstd, {kF32}, {rows});
    const int64_t dzp = dz_out.has_value() ? row_view(args, "dz_out", *dz_out, rows, E) : E;
    args.device();
    at::Tensor dy = at::empty_like(y), dz = dz_out.has_value() ? *dz_out : at::empty_like(y), dweight = at::empty_like(weight);
    at::Tensor wpart = at::empty({(int64_t)gated_rmsnorm_parts((int)rows), E}, y.options().dtype(kF32));
    launch_gated_rmsnorm_bwd(dout.data_ptr(), y.data_ptr(), z.data_ptr(), zp, weight.data_ptr(), rstd.data_ptr<float>(), (int)rows, (int)E,
                             dy.data_ptr(), dz.data_ptr(), dzp, wpart.data_ptr<float>(), dweight.data_ptr(), cur_stream());
    return std::make_tuple(dy, dz, dweight);
  }, py::arg("dout"), py::arg("y"), py::arg("z"), py::arg("weight"), py::arg("rstd"), py::arg("dz_out") = py::none());

  // ---- Whisper's log-mel front end and stem gathers (whisper.cu) ------------------------------------------------------------
  // _C.whisper is a namespace of static entry points like _C.mamba2; its contract rows are in tests/test_whisper_bindings_cpu.py.
  py::class_<WhisperNamespace> whisper(m, "whisper", "Whisper's log-mel front end and convolution-stem gathers (whisper.cu)");
  // log-mel features [B, 80, 3000] of int16 waveforms [B, 480000] through filters fp32 [201, 80]: bf16 when `bf16`, else fp32;
  // written into `out` when given (contiguous, that dtype, B * 80 * 3000 elements) and returned
  whisper.def_static("log_mel", [](at::Tensor wave, at::Tensor filters, bool bf16, c10::optional<at::Tensor> out) {
    Args args("log_mel");
    args("wave", wave, {at::kShort}, {kAny, 480000});
    const int64_t B = wave.size(0);
    if (B < 1 || B > 65535) args.fail("wave", "int16 [B, 480000] with 1 <= B <= 65535", describe(wave));
    args("filters", filters, {kF32}, {201, 80});
    at::Tensor o;
    args.out(o, "out", out, {B, 80, 3000}, wave.options().dtype(bf16 ? kBF16 : kF32));
    args.device();
    const auto f32 = wave.options().dtype(kF32);
    at::Tensor part = at::empty({B, (int64_t)log_mel_partials()}, f32);
    at::Tensor logmel = bf16 ? at::empty({B, 80, 3000}, f32) : o;
    launch_log_mel(wave.data_ptr(), filters.data_ptr<float>(), (int)B, bf16, logmel.data_ptr<float>(), part.data_ptr<float>(), o.data_ptr(),
                   cur_stream());
    return o.view({B, 80, 3000});
  }, py::arg("wave"), py::arg("filters"), py::arg("bf16"), py::arg("out") = py::none());
  // P1 bf16 [B F, 240] of features bf16 [B, 80, F]
  whisper.def_static("mel_patches", [](at::Tensor features) {
    Args args("mel_patches");
    args("features", features, {kBF16}, {kAny, 80, kAny});
    const int64_t B = features.size(0), F = features.size(2);
    if (B < 1 || F < 1 || B * F * 240 >= (1ll << 31))
      args.fail("features", "bf16 [B, 80, F] with B, F >= 1 and fewer than 2^31 / 3 elements", describe(features));
    args.device();
    at::Tensor p1 = at::empty({B * F, 240}, features.options());
    launch_mel_patches(features.data_ptr(), (int)B, (int)F, p1.data_ptr(), cur_stream());
    return p1;
  }, py::arg("features"));
  // P2 bf16 [B rows, 3 d] of h1 bf16 [B frames, d]
  whisper.def_static("frame_patches", [](at::Tensor h1, int64_t frames, int64_t rows) {
    Args args("frame_patches");
    const auto [B, d] = stem_rows(args, "h1", h1, frames, rows, false);
    args.device();
    at::Tensor p2 = at::empty({B * rows, 3 * d}, h1.options());
    launch_frame_patches(h1.data_ptr(), (int)B, (int)frames, (int)rows, (int)d, p2.data_ptr(), cur_stream());
    return p2;
  }, py::arg("h1"), py::arg("frames"), py::arg("rows"));
  // dh1 bf16 [B frames, d] of dP2 bf16 [B rows, 3 d]
  whisper.def_static("frame_patches_bwd", [](at::Tensor dp2, int64_t frames, int64_t rows) {
    Args args("frame_patches_bwd");
    const auto [B, d] = stem_rows(args, "dp2", dp2, frames, rows, true);
    args.device();
    at::Tensor dh1 = at::empty({B * frames, d}, dp2.options());
    launch_frame_patches_bwd(dp2.data_ptr(), (int)B, (int)frames, (int)rows, (int)d, dh1.data_ptr(), cur_stream());
    return dh1;
  }, py::arg("dp2"), py::arg("frames"), py::arg("rows"));

  // ---- Masked-autoencoder pretraining (mae.cu): shuffle, masked patch embedding, unshuffle, attention, loss ---------------
  // _C.mae is a namespace of static entry points like _C.whisper; its contract rows are in tests/test_vit_mae_bindings_cpu.py.
  py::class_<MaeNamespace> mae(m, "mae", "Masked-autoencoder shuffle, patch embedding, unshuffle, attention and loss (mae.cu)");
  // (ids_keep int32 [B, keep], ids_restore int32 [B, N]) of noise fp32 [B, N]
  mae.def_static("shuffle", [](at::Tensor noise, int64_t keep) {
    Args args("shuffle");
    args("noise", noise, {kF32}, {kAny, kAny});
    const int64_t B = noise.size(0), N = noise.size(1);
    if (B < 1 || N < 1 || N > 1024) args.fail("noise", "fp32 [B, N] with B >= 1 and 1 <= N <= 1024", describe(noise));
    if (keep < 0 || keep > N) args.fail("keep", "in [0, N] = [0, " + std::to_string(N) + "]", std::to_string(keep));
    args.device();
    at::Tensor ids_keep = at::empty({B, keep}, noise.options().dtype(kI32));
    at::Tensor ids_restore = at::empty({B, N}, noise.options().dtype(kI32));
    launch_mae_shuffle(noise.data_ptr<float>(), (int)B, (int)N, (int)keep, ids_keep.data_ptr<int>(), ids_restore.data_ptr<int>(), cur_stream());
    return std::make_tuple(ids_keep, ids_restore);
  }, py::arg("noise"), py::arg("keep"));
  // the kept patches' rows bf16 [tokens, C p p] of images bf16 [B, C, H, W] (NCHW or channels_last); ids_keep int32 [B, keep]
  mae.def_static("patchify", [](at::Tensor images, at::Tensor ids_keep, int64_t patch, int64_t tokens) {
    Args args("patchify");
    const MaeImages im = mae_images(args, images, patch);
    args("ids_keep", ids_keep, {kI32}, {im.B, kAny});
    const int64_t keep = ids_keep.size(1);
    if (keep > im.N) args.fail("ids_keep", "int32 [B, keep] with keep <= patches = " + std::to_string(im.N), describe(ids_keep));
    if (tokens < im.B * (keep + 1) || tokens * im.C * patch * patch >= (1ll << 31))
      args.fail("tokens", "at least batch * (keep + 1) = " + std::to_string(im.B * (keep + 1)) + " and below 2^31 patch elements",
                std::to_string(tokens));
    args.device();
    at::Tensor out = at::empty({tokens, im.C * patch * patch}, images.options().memory_format(at::MemoryFormat::Contiguous));
    launch_mae_patchify(images.data_ptr(), im.cl, ids_keep.data_ptr<int>(), (int)im.B, (int)im.C, (int)im.H, (int)im.W, (int)patch, (int)keep,
                        (int)tokens, out.data_ptr(), cur_stream());
    return out;
  }, py::arg("images"), py::arg("ids_keep"), py::arg("patch"), py::arg("tokens"));
  // encoder tokens bf16 [T, D] of the GEMM output y [T, D], class_token [D], pos_embedding [N + 1, D], ids_keep int32 [B, keep]
  mae.def_static("patch_assemble", [](at::Tensor y, at::Tensor class_token, at::Tensor pos_embedding, at::Tensor ids_keep) {
    Args args("patch_assemble");
    args("y", y, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t T = y.size(0), D = y.size(1);
    if (D % 8 || D < 8) args.fail("y", "bf16 [T, D] with D % 8 == 0", describe(y));
    args("class_token", class_token, {kBF16}, numel(D), kContiguous, 16)("pos_embedding", pos_embedding, {kBF16}, last_dim(D), kContiguous, 16);
    args("ids_keep", ids_keep, {kI32}, {kAny, kAny});
    const int64_t B = ids_keep.size(0), keep = ids_keep.size(1), N = pos_embedding.numel() / D - 1;
    if (B < 1 || keep > N || B * (keep + 1) > T)
      args.fail("ids_keep", "int32 [B, keep] with B >= 1, keep <= patches = " + std::to_string(N) + " and B (keep + 1) <= T = " +
                std::to_string(T), describe(ids_keep));
    args.device();
    at::Tensor out = at::empty_like(y);
    launch_mae_patch_assemble(y.data_ptr(), class_token.data_ptr(), pos_embedding.data_ptr(), ids_keep.data_ptr<int>(), (int)B, (int)keep,
                              (int)D, (int)T, out.data_ptr(), cur_stream());
    return out;
  }, py::arg("y"), py::arg("class_token"), py::arg("pos_embedding"), py::arg("ids_keep"));
  // (dpatch bf16 [T, D], dcls bf16 [D]) of dy bf16 [T, D]
  mae.def_static("patch_embed_bwd", [](at::Tensor dy, int64_t batch, int64_t tokens_per_image) {
    Args args("patch_embed_bwd");
    args("dy", dy, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t T = dy.size(0), D = dy.size(1);
    if (D % 8 || D < 8) args.fail("dy", "bf16 [T, D] with D % 8 == 0", describe(dy));
    if (tokens_per_image < 1 || batch < 1 || batch * tokens_per_image > T)
      args.fail("batch", "batch >= 1 and batch * tokens_per_image <= T = " + std::to_string(T), std::to_string(batch) + " * " +
                std::to_string(tokens_per_image));
    args.device();
    at::Tensor dpatch = at::empty_like(dy);
    at::Tensor dcls = at::empty({D}, dy.options());
    launch_mae_patch_embed_bwd(dy.data_ptr(), (int)batch, (int)tokens_per_image, (int)D, (int)T, dpatch.data_ptr(), dcls.data_ptr(), cur_stream());
    return std::make_tuple(dpatch, dcls);
  }, py::arg("dy"), py::arg("batch"), py::arg("tokens_per_image"));
  // the decoder stream bf16 [rows, E] of y bf16 [Te, E], mask_token [E], pos_embedding [N + 1, E], ids_restore int32 [B, N]
  mae.def_static("unshuffle", [](at::Tensor y, at::Tensor mask_token, at::Tensor pos_embedding, at::Tensor ids_restore, int64_t keep,
                                 int64_t rows) {
    Args args("unshuffle");
    args("y", y, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t Te = y.size(0), E = y.size(1);
    if (E % 8 || E < 8 || E > 2048) args.fail("y", "bf16 [T, E] with E % 8 == 0 and E <= 2048", describe(y));
    args("mask_token", mask_token, {kBF16}, numel(E), kContiguous, 16);
    args("ids_restore", ids_restore, {kI32}, {kAny, kAny});
    const int64_t B = ids_restore.size(0), N = ids_restore.size(1);
    mae_ids(args, "ids_restore", ids_restore, B, N, keep);
    if (B < 1) args.fail("ids_restore", "int32 [B, N] with B >= 1", describe(ids_restore));
    args("pos_embedding", pos_embedding, {kBF16}, numel((N + 1) * E), kContiguous, 16);
    if (B * (keep + 1) > Te) args.fail("y", "at least B (keep + 1) = " + std::to_string(B * (keep + 1)) + " rows", describe(y));
    if (rows < B * (N + 1) || rows * E >= (1ll << 31))
      args.fail("rows", "at least B (N + 1) = " + std::to_string(B * (N + 1)) + " and below 2^31 elements", std::to_string(rows));
    args.device();
    at::Tensor z = at::empty({rows, E}, y.options());
    launch_mae_unshuffle(y.data_ptr(), mask_token.data_ptr(), pos_embedding.data_ptr(), ids_restore.data_ptr<int>(), (int)B, (int)N, (int)keep,
                         (int)E, (int)rows, z.data_ptr(), cur_stream());
    return z;
  }, py::arg("y"), py::arg("mask_token"), py::arg("pos_embedding"), py::arg("ids_restore"), py::arg("keep"), py::arg("rows"));
  // (dy bf16 [rows, E], dmask bf16 [E]) of dz bf16 [Td, E], ids_keep int32 [B, keep], ids_restore int32 [B, N]
  mae.def_static("unshuffle_bwd", [](at::Tensor dz, at::Tensor ids_keep, at::Tensor ids_restore, int64_t rows) {
    Args args("unshuffle_bwd");
    args("dz", dz, {kBF16}, {kAny, kAny}, kContiguous, 16);
    const int64_t Td = dz.size(0), E = dz.size(1);
    if (E % 8 || E < 8 || E > 2048) args.fail("dz", "bf16 [T, E] with E % 8 == 0 and E <= 2048", describe(dz));
    args("ids_keep", ids_keep, {kI32}, {kAny, kAny});
    const int64_t B = ids_keep.size(0), keep = ids_keep.size(1);
    if (B < 1) args.fail("ids_keep", "int32 [B, keep] with B >= 1", describe(ids_keep));
    args("ids_restore", ids_restore, {kI32}, {B, kAny});
    const int64_t N = ids_restore.size(1);
    mae_ids(args, "ids_restore", ids_restore, B, N, keep);
    if (B * (N + 1) > Td) args.fail("dz", "at least B (N + 1) = " + std::to_string(B * (N + 1)) + " rows", describe(dz));
    if (rows < B * (keep + 1) || rows * E >= (1ll << 31))
      args.fail("rows", "at least B (keep + 1) = " + std::to_string(B * (keep + 1)) + " and below 2^31 elements", std::to_string(rows));
    args.device();
    at::Tensor dy = at::empty({rows, E}, dz.options());
    at::Tensor part = at::empty({(int64_t)mae_mask_partials((int)B), E}, dz.options().dtype(kF32));
    at::Tensor dmask = at::empty({E}, dz.options());
    launch_mae_unshuffle_bwd(dz.data_ptr(), ids_keep.data_ptr<int>(), ids_restore.data_ptr<int>(), (int)B, (int)N, (int)keep, (int)E, (int)rows,
                             dy.data_ptr(), part.data_ptr<float>(), dmask.data_ptr(), cur_stream());
    return std::make_tuple(dy, dmask);
  }, py::arg("dz"), py::arg("ids_keep"), py::arg("ids_restore"), py::arg("rows"));
  // (o bf16 [T, C], lse fp32 [T, heads]) of qkv bf16 [T, 3C], C = 32 heads, images of `tokens` rows (1 <= tokens <= 256)
  mae.def_static("attention_fwd", [](at::Tensor qkv, int64_t batch, int64_t tokens) {
    Args args("attention_fwd");
    const auto [T, heads] = mae_attention_args(args, qkv, batch, tokens);
    args.device();
    at::Tensor o = at::empty({T, 32 * heads}, qkv.options());
    at::Tensor lse = at::empty({T, heads}, qkv.options().dtype(kF32));
    launch_image_attention_fwd(qkv.data_ptr(), (int)batch, (int)tokens, (int)heads, (int)T, o.data_ptr(), lse.data_ptr<float>(), cur_stream());
    return std::make_tuple(o, lse);
  }, py::arg("qkv"), py::arg("batch"), py::arg("tokens"));
  // dqkv bf16 [T, 3C]
  mae.def_static("attention_bwd", [](at::Tensor dout, at::Tensor qkv, at::Tensor o, at::Tensor lse, int64_t batch, int64_t tokens) {
    Args args("attention_bwd");
    const auto [T, heads] = mae_attention_args(args, qkv, batch, tokens);
    args("dout", dout, {kBF16}, {T, 32 * heads}, kContiguous, 16)("o", o, {kBF16}, {T, 32 * heads}, kContiguous, 16)("lse", lse, {kF32}, {T, heads});
    args.device();
    at::Tensor dqkv = at::empty_like(qkv);
    launch_image_attention_bwd(dout.data_ptr(), qkv.data_ptr(), o.data_ptr(), lse.data_ptr<float>(), (int)batch, (int)tokens, (int)heads, (int)T,
                               dqkv.data_ptr(), cur_stream());
    return dqkv;
  }, py::arg("dout"), py::arg("qkv"), py::arg("o"), py::arg("lse"), py::arg("batch"), py::arg("tokens"));
  // loss fp32 [] of pred bf16 [Td, C p p] (p from its width), images bf16 [B, C, H, W], ids_restore int32 [B, N], 0 <= keep < N
  mae.def_static("loss", [](at::Tensor pred, at::Tensor images, at::Tensor ids_restore, int64_t keep, bool norm_pix) {
    Args args("loss");
    const auto [im, patch] = mae_loss_args(args, pred, images, ids_restore, keep);
    args.device();
    at::Tensor rowloss = at::empty({im.B * im.N}, pred.options().dtype(kF32));
    at::Tensor loss = at::empty({}, pred.options().dtype(kF32));
    launch_mae_loss_fwd(pred.data_ptr(), images.data_ptr(), im.cl, ids_restore.data_ptr<int>(), (int)im.B, (int)im.C, (int)im.H, (int)im.W,
                        (int)patch, (int)keep, norm_pix, rowloss.data_ptr<float>(), loss.data_ptr<float>(), cur_stream());
    return loss;
  }, py::arg("pred"), py::arg("images"), py::arg("ids_restore"), py::arg("keep"), py::arg("norm_pix"));
  // dpred bf16 [Td, C p p] of dloss fp32 (one element, read on the device)
  mae.def_static("loss_bwd", [](at::Tensor dloss, at::Tensor pred, at::Tensor images, at::Tensor ids_restore, int64_t keep, bool norm_pix) {
    Args args("loss_bwd");
    args("dloss", dloss, {kF32}, numel(1));
    const auto [im, patch] = mae_loss_args(args, pred, images, ids_restore, keep);
    args.device();
    at::Tensor dpred = at::empty_like(pred);
    launch_mae_loss_bwd(dloss.data_ptr<float>(), pred.data_ptr(), images.data_ptr(), im.cl, ids_restore.data_ptr<int>(), (int)im.B, (int)im.C,
                        (int)im.H, (int)im.W, (int)patch, (int)keep, norm_pix, (int)pred.size(0), dpred.data_ptr(), cur_stream());
    return dpred;
  }, py::arg("dloss"), py::arg("pred"), py::arg("images"), py::arg("ids_restore"), py::arg("keep"), py::arg("norm_pix"));
}
