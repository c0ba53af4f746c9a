// Fused loss forward+backward kernels: the stock path runs sub / pow / mean-reduce and a
// separate mse_loss_backward; cross-entropy is log_softmax + nll_loss + their two backwards.
// Each loss here is one launch that emits the scalar loss AND the gradient w.r.t. its input, so the
// autograd Function's backward is just "return the saved tensor (x upstream scale)".
#include "ops.h"

namespace b200 {
namespace {

constexpr int kLossThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kLossThreads) mse_fwd_bwd_kernel(const T* __restrict__ out, const T* __restrict__ tgt, size_t n,
                                                                   float gscale, float* __restrict__ loss, T* __restrict__ dout,
                                                                   float* __restrict__ scratch) {
  __shared__ float red[33];
  __shared__ bool last;
  const float inv_n = 1.f / (float)n;
  const float k = 2.f * inv_n * gscale;
  float acc = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(tgt) | reinterpret_cast<uintptr_t>(dout)) & 31u) == 0;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = n / 8;
    size_t v = tid;
    for (; v + stride < nvec; v += 2 * stride) {            // two independent vector pairs in flight
      float a0[8], b0[8], a1[8], b1[8];
      load8<T>(out + v * 8, a0); load8<T>(tgt + v * 8, b0);
      load8<T>(out + (v + stride) * 8, a1); load8<T>(tgt + (v + stride) * 8, b1);
#pragma unroll
      for (int i = 0; i < 8; ++i) { a0[i] -= b0[i]; acc = fmaf(a0[i], a0[i], acc); a0[i] *= k; a1[i] -= b1[i]; acc = fmaf(a1[i], a1[i], acc); a1[i] *= k; }
      store8<T>(dout + v * 8, a0);
      store8<T>(dout + (v + stride) * 8, a1);
    }
    for (; v < nvec; v += stride) {
      float a0[8], b0[8];
      load8<T>(out + v * 8, a0); load8<T>(tgt + v * 8, b0);
#pragma unroll
      for (int i = 0; i < 8; ++i) { a0[i] -= b0[i]; acc = fmaf(a0[i], a0[i], acc); a0[i] *= k; }
      store8<T>(dout + v * 8, a0);
    }
    done = nvec * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    const float d = to_f32<T>(out[i]) - to_f32<T>(tgt[i]);
    acc += d * d;
    dout[i] = from_f32<T>(k * d);
  }
  const float total = block_sum(acc, red);
  // deterministic two-stage reduction: the last block to arrive sums the partials in index order
  unsigned int* counter = reinterpret_cast<unsigned int*>(scratch + gridDim.x);
  if (threadIdx.x == 0) {
    scratch[blockIdx.x] = total;
    __threadfence();
    const unsigned int ticket = atomicAdd(counter, 1u);
    last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (last) {
    __threadfence();
    float s = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) s += __ldcg(scratch + i);
    s = block_sum(s, red);
    if (threadIdx.x == 0) { *loss = s * inv_n; *counter = 0u; }
  }
}

// One block per row; the row is read once into registers/smem-free streaming form twice (second read
// hits L1/L2: a 30522-wide bf16 row is 61 KB).
template <typename T>
__global__ void __launch_bounds__(kLossThreads) xent_fwd_bwd_kernel(const T* __restrict__ logits, const long long* __restrict__ targets,
                                                                    int rows, int cols, long long ignore_index, float gscale,
                                                                    float* __restrict__ row_loss, T* __restrict__ dlogits) {
  __shared__ float red[33];
  const int row = blockIdx.x;
  const T* x = logits + (size_t)row * cols;
  T* dx = dlogits + (size_t)row * cols;
  const long long t = targets[row];
  const bool ignored = (t == ignore_index) || t < 0 || t >= cols;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) m = fmaxf(m, to_f32<T>(x[i]));
  m = block_max(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) s += __expf(to_f32<T>(x[i]) - m);
  s = block_sum(s, red);
  const float lse = m + __logf(s);
  const float inv_s = 1.f / s;
  if (threadIdx.x == 0) row_loss[row] = ignored ? 0.f : lse - to_f32<T>(x[t]);
  const float valid = row_loss[rows];   // written by count_valid_kernel (mean is over non-ignored rows)
  const float g = (ignored || valid <= 0.f) ? 0.f : gscale / valid;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) {
    float p = __expf(to_f32<T>(x[i]) - m) * inv_s;
    if (i == t) p -= 1.f;
    dx[i] = from_f32<T>(p * g);
  }
}

// Row lives in shared memory: ONE global read of the logits, softmax statistics and the gradient come from smem,
// ONE global write of dlogits; 16-byte accesses with a peeled head/tail (rows of a 30522-wide matrix are only
// 4-byte aligned).  smem index = column + pad so shared and global addresses share their 16-byte phase.
template <typename T>
__global__ void __launch_bounds__(kLossThreads) xent_fwd_bwd_smem_kernel(const T* __restrict__ logits, const long long* __restrict__ targets,
                                                                         int rows, int cols, long long ignore_index, float gscale,
                                                                         float* __restrict__ row_loss, T* __restrict__ dlogits) {
  extern __shared__ __align__(16) unsigned char xsmem[];
  __shared__ float red[33];
  constexpr int EPV = 16 / sizeof(T);                   // elements per 16-byte vector
  const int row = blockIdx.x;
  const T* x = logits + (size_t)row * cols;
  T* dx = dlogits + (size_t)row * cols;
  const int pad = (int)((reinterpret_cast<uintptr_t>(x) & 15u) / sizeof(T));
  T* sx = reinterpret_cast<T*>(xsmem);                   // sx[pad + i] = x[i]
  const int head = min(cols, (EPV - pad) % EPV);         // scalars until the first aligned vector
  const int nvec = (cols - head) / EPV;
  const int tail0 = head + nvec * EPV;
  const long long t = targets[row];
  const bool ignored = (t == ignore_index) || t < 0 || t >= cols;

  float m = -INFINITY;
  for (int i = threadIdx.x; i < head; i += blockDim.x) { const T v = x[i]; sx[pad + i] = v; m = fmaxf(m, to_f32<T>(v)); }
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint4 raw = *reinterpret_cast<const uint4*>(x + head + v * EPV);
    *reinterpret_cast<uint4*>(sx + pad + head + v * EPV) = raw;
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < EPV; ++j) m = fmaxf(m, to_f32<T>(e[j]));
  }
  for (int i = tail0 + threadIdx.x; i < cols; i += blockDim.x) { const T v = x[i]; sx[pad + i] = v; m = fmaxf(m, to_f32<T>(v)); }
  m = block_max(m, red);                                 // (contains the __syncthreads that publishes smem)
  float s = 0.f;
  for (int i = threadIdx.x; i < cols; i += blockDim.x) s += __expf(to_f32<T>(sx[pad + i]) - m);
  s = block_sum(s, red);
  const float lse = m + __logf(s);
  const float valid = row_loss[rows];
  if (threadIdx.x == 0) row_loss[row] = ignored ? 0.f : lse - to_f32<T>(sx[pad + (int)t]);
  const float g = (ignored || valid <= 0.f) ? 0.f : gscale / valid;
  const float coef = g / s;
  const int ti = ignored ? -1 : (int)t;
  for (int i = threadIdx.x; i < head; i += blockDim.x) {
    float p = __expf(to_f32<T>(sx[pad + i]) - m) * coef;
    if (i == ti) p -= g;
    dx[i] = from_f32<T>(p);
  }
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const int base = head + v * EPV;
    const uint4 raw = *reinterpret_cast<const uint4*>(sx + pad + base);
    const T* e = reinterpret_cast<const T*>(&raw);
    uint4 outv;
    T* o = reinterpret_cast<T*>(&outv);
#pragma unroll
    for (int j = 0; j < EPV; ++j) {
      float p = __expf(to_f32<T>(e[j]) - m) * coef;
      if (base + j == ti) p -= g;
      o[j] = from_f32<T>(p);
    }
    *reinterpret_cast<uint4*>(dx + base) = outv;
  }
  for (int i = tail0 + threadIdx.x; i < cols; i += blockDim.x) {
    float p = __expf(to_f32<T>(sx[pad + i]) - m) * coef;
    if (i == ti) p -= g;
    dx[i] = from_f32<T>(p);
  }
}

__global__ void __launch_bounds__(1024) xent_finish_kernel(const float* __restrict__ row_loss, const long long* __restrict__ targets,
                                                           int rows, int cols, long long ignore_index, float* __restrict__ loss) {
  __shared__ float red[33];
  float s = 0.f, cnt = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    const long long t = targets[i];
    if (t != ignore_index && t >= 0 && t < cols) { s += row_loss[i]; cnt += 1.f; }
  }
  s = block_sum(s, red);
  cnt = block_sum(cnt, red);
  if (threadIdx.x == 0) *loss = cnt > 0.f ? s / cnt : 0.f;
}

__global__ void __launch_bounds__(1024) count_valid_kernel(const long long* __restrict__ targets, int rows, int cols,
                                                           long long ignore_index, float* __restrict__ out) {
  __shared__ float red[33];
  float cnt = 0.f;
  for (int i = threadIdx.x; i < rows; i += blockDim.x) {
    const long long t = targets[i];
    if (t != ignore_index && t >= 0 && t < cols) cnt += 1.f;
  }
  cnt = block_sum(cnt, red);
  if (threadIdx.x == 0) *out = cnt;
}

// (max, sum exp(x - max)) pairs; an empty pair (-inf, 0) is the identity
__device__ __forceinline__ float2 lse_merge(float2 a, float2 b) {
  if (b.x == -INFINITY) return a;
  if (a.x == -INFINITY) return b;
  const float m = fmaxf(a.x, b.x);
  return make_float2(m, a.y * __expf(a.x - m) + b.y * __expf(b.x - m));
}

// Block = 32 rows x 8 tile groups: thread (x, y) merges tiles y, y + 8, ... of row x in order (a warp reads 32 consecutive
// rows of one tile: coalesced), then the 8 group results are merged in order.  Deterministic: a fixed order per row.
// BOUNDED: only the rows below the device count *bound have partials (the row-bounded LSE GEMM skipped the other tiles);
// the rest get lse = row_loss = 0 without reading them.
constexpr int kCombineGroups = 8;
template <bool BOUNDED>
__global__ void __launch_bounds__(32 * kCombineGroups) lm_lse_combine_kernel(const float2* __restrict__ partial, const float* __restrict__ target_logit,
                                                                             const long long* __restrict__ targets, int rows, int tiles, int cols,
                                                                             long long ignore_index, float* __restrict__ lse,
                                                                             float* __restrict__ row_loss, const int* __restrict__ bound) {
  __shared__ float2 part[kCombineGroups][32];
  const int row = blockIdx.x * 32 + threadIdx.x;
  const bool live = row < rows && (!BOUNDED || row < __ldg(bound));
  float2 acc = make_float2(-INFINITY, 0.f);
  if (live)
    for (int i = threadIdx.y; i < tiles; i += kCombineGroups) acc = lse_merge(acc, partial[(size_t)i * rows + row]);
  part[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y != 0 || row >= rows) return;
  if (BOUNDED && !live) {
    lse[row] = 0.f;
    row_loss[row] = 0.f;
    return;
  }
#pragma unroll
  for (int g = 1; g < kCombineGroups; ++g) acc = lse_merge(acc, part[g][threadIdx.x]);
  const float l = acc.x + __logf(acc.y);
  lse[row] = l;
  const long long t = targets[row];
  const bool ignored = (t == ignore_index) || t < 0 || t >= cols;
  row_loss[row] = ignored ? 0.f : l - target_logit[row];
}

}  // namespace

int mse_blocks(size_t n) {
  size_t b = (n + kLossThreads * 16 - 1) / (kLossThreads * 16);
  if (b < 1) b = 1;
  if (b > 8 * kNumSMs) b = 8 * kNumSMs;
  return (int)b;
}

void launch_mse_fwd_bwd(const void* out, const void* target, DType dt, size_t n, float gscale, float* loss, void* dout,
                        float* scratch, int blocks, cudaStream_t s) {
  if (dt == DType::BF16)
    mse_fwd_bwd_kernel<__nv_bfloat16><<<blocks, kLossThreads, 0, s>>>((const __nv_bfloat16*)out, (const __nv_bfloat16*)target, n,
                                                                     gscale, loss, (__nv_bfloat16*)dout, scratch);
  else
    mse_fwd_bwd_kernel<float><<<blocks, kLossThreads, 0, s>>>((const float*)out, (const float*)target, n, gscale, loss,
                                                             (float*)dout, scratch);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_xent_fwd_bwd(const void* logits, const long long* targets, DType dt, int rows, int cols, long long ignore_index,
                         float gscale, float* row_loss, float* loss, void* dlogits, cudaStream_t s) {
  // mean over non-ignored rows: count them on device first (row_loss has rows+1 floats; the last
  // one carries the count) so no host round trip is needed.
  const float g = gscale;
  count_valid_kernel<<<1, 1024, 0, s>>>(targets, rows, cols, ignore_index, row_loss + rows);
  const size_t esz = dt == DType::BF16 ? 2 : 4;
  const size_t smem = ((size_t)cols + 16) * esz;
  if (smem <= 200 * 1024 && ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(dlogits)) % esz) == 0 &&
      (reinterpret_cast<uintptr_t>(logits) & 15u) == (reinterpret_cast<uintptr_t>(dlogits) & 15u)) {
    // dlogits rows must share the 16-byte phase of the logits rows (both come from the same allocator: they do)
    static std::atomic<unsigned long long> configured_bf16{0}, configured_f32{0};
    ensure_max_dynamic_smem(xent_fwd_bwd_smem_kernel<__nv_bfloat16>, 200 * 1024, configured_bf16);
    ensure_max_dynamic_smem(xent_fwd_bwd_smem_kernel<float>, 200 * 1024, configured_f32);
    if (dt == DType::BF16)
      xent_fwd_bwd_smem_kernel<__nv_bfloat16><<<rows, kLossThreads, smem, s>>>((const __nv_bfloat16*)logits, targets, rows, cols, ignore_index, g,
                                                                             row_loss, (__nv_bfloat16*)dlogits);
    else
      xent_fwd_bwd_smem_kernel<float><<<rows, kLossThreads, smem, s>>>((const float*)logits, targets, rows, cols, ignore_index, g, row_loss,
                                                                     (float*)dlogits);
  } else if (dt == DType::BF16)
    xent_fwd_bwd_kernel<__nv_bfloat16><<<rows, kLossThreads, 0, s>>>((const __nv_bfloat16*)logits, targets, rows, cols, ignore_index, g,
                                                                   row_loss, (__nv_bfloat16*)dlogits);
  else
    xent_fwd_bwd_kernel<float><<<rows, kLossThreads, 0, s>>>((const float*)logits, targets, rows, cols, ignore_index, g, row_loss,
                                                           (float*)dlogits);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  xent_finish_kernel<<<1, 1024, 0, s>>>(row_loss, targets, rows, cols, ignore_index, loss);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_lm_loss_combine(const float* partial, const float* target_logit, const long long* targets, int rows, int tiles, int cols,
                            long long ignore_index, float* lse, float* row_loss, float* loss, cudaStream_t s, const int* bound) {
  count_valid_kernel<<<1, 1024, 0, s>>>(targets, rows, cols, ignore_index, row_loss + rows);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  const auto* pf2 = reinterpret_cast<const float2*>(partial);
  if (bound != nullptr)
    lm_lse_combine_kernel<true><<<(rows + 31) / 32, dim3(32, kCombineGroups), 0, s>>>(pf2, target_logit, targets, rows, tiles, cols, ignore_index,
                                                                                    lse, row_loss, bound);
  else
    lm_lse_combine_kernel<false><<<(rows + 31) / 32, dim3(32, kCombineGroups), 0, s>>>(pf2, target_logit, targets, rows, tiles, cols, ignore_index,
                                                                                     lse, row_loss, nullptr);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
  xent_finish_kernel<<<1, 1024, 0, s>>>(row_loss, targets, rows, cols, ignore_index, loss);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------------------
// Sparse (masked-row) prediction: the rows that carry a label are compacted to the front on the device, so the LM-head
// loss runs on them alone, and the bias gradient of the fused loss.  Nothing is read back to the host: the number of
// labelled rows is a device scalar that the kernels read, and every buffer is sized for all rows.
//   compact : a stable partition of the rows, labelled first.  Three launches, as the mixture-of-experts sort does it:
//             per-chunk counts, a one-warp scan over the chunks, and a scatter that re-derives each row's rank with
//             warp ballots.  No atomics.
//   gather / scatter : one warp per row, 16-byte copies; rows past the count are written as zeros.
//   column sum : d[rows, cols] bf16 summed over the rows below the count, per 128-row chunk and then over the chunks,
//             both in a fixed order (bitwise repeatable).
namespace b200 {
namespace {

constexpr int kCompactThreads = 256, kCompactWarps = kCompactThreads / 32;
constexpr int kCompactChunk = 4 * kCompactThreads;             // rows per count / scatter block: 4 rounds of 256

__device__ __forceinline__ bool labelled(long long t, long long ignore_index, long long vocab) {
  return t != ignore_index && t >= 0 && t < vocab;
}

__global__ void __launch_bounds__(kCompactThreads) compact_count_kernel(const long long* __restrict__ targets, int n, long long ignore_index,
                                                                        long long vocab, int* __restrict__ chunk_counts) {
  int c = 0;
#pragma unroll
  for (int r = 0; r < kCompactChunk / kCompactThreads; ++r) {
    const int i = blockIdx.x * kCompactChunk + r * kCompactThreads + threadIdx.x;
    c += __syncthreads_count(i < n && labelled(__ldg(targets + i), ignore_index, vocab));
  }
  if (threadIdx.x == 0) chunk_counts[blockIdx.x] = c;
}

// One warp: exclusive prefix sums of the chunk counts in chunk order, and the total.
__global__ void __launch_bounds__(32) compact_scan_kernel(const int* __restrict__ chunk_counts, int chunks, int* __restrict__ chunk_base,
                                                          int* __restrict__ count) {
  const int lane = threadIdx.x;
  int run = 0;
  for (int c0 = 0; c0 < chunks; c0 += 32) {
    const int v = c0 + lane < chunks ? chunk_counts[c0 + lane] : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (c0 + lane < chunks) chunk_base[c0 + lane] = run + inc - v;
    run += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (lane == 0) *count = run;
}

// Labelled row i goes to position (labelled rows before it); unlabelled row i to count + (unlabelled rows before it), with
// its target replaced by ignore_index.  Every position gets exactly one writer.
__global__ void __launch_bounds__(kCompactThreads) compact_scatter_kernel(const long long* __restrict__ targets, int n, long long ignore_index,
                                                                          long long vocab, const int* __restrict__ chunk_base,
                                                                          const int* __restrict__ count, int* __restrict__ index,
                                                                          long long* __restrict__ targets_out) {
  __shared__ int warp_counts[kCompactWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total = __ldg(count);
  int base = __ldg(chunk_base + blockIdx.x);                   // labelled rows before this round
#pragma unroll 1
  for (int r = 0; r < kCompactChunk / kCompactThreads; ++r) {
    const int i = blockIdx.x * kCompactChunk + r * kCompactThreads + threadIdx.x;
    const long long t = i < n ? __ldg(targets + i) : ignore_index;
    const bool lab = i < n && labelled(t, ignore_index, vocab);
    const unsigned ballot = __ballot_sync(0xffffffffu, lab);
    if (lane == 0) warp_counts[warp] = __popc(ballot);
    __syncthreads();
    int before = base + __popc(ballot & ((1u << lane) - 1u)), round = 0;
#pragma unroll
    for (int w = 0; w < kCompactWarps; ++w) {
      before += w < warp ? warp_counts[w] : 0;
      round += warp_counts[w];
    }
    __syncthreads();                                           // warp_counts is rewritten by the next round
    if (i < n) {
      const int pos = lab ? before : total + (i - before);
      index[pos] = i;
      targets_out[pos] = lab ? t : ignore_index;
    }
    base += round;
  }
}

int row_grid(long long rows) {
  const long long b = (rows + kCompactWarps - 1) / kCompactWarps;
  return (int)(b < 1 ? 1 : (b > 16LL * kNumSMs ? 16LL * kNumSMs : b));
}

// out[r] = x[index[r]] for r < *count, zeros after.
__global__ void __launch_bounds__(kCompactThreads) gather_rows_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ index,
                                                                      const int* __restrict__ count, int T, int H,
                                                                      __nv_bfloat16* __restrict__ out) {
  const int lane = threadIdx.x & 31, vecs = H / 8, live = __ldg(count);
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < T; r += (gridDim.x * blockDim.x) >> 5) {
    Bf16x8* o = reinterpret_cast<Bf16x8*>(out + (size_t)r * H);
    if (r < live) {
      const Bf16x8* in = reinterpret_cast<const Bf16x8*>(x + (size_t)__ldg(index + r) * H);
      for (int v = lane; v < vecs; v += 32) o[v] = in[v];
    } else {
      const Bf16x8 z = {};
      for (int v = lane; v < vecs; v += 32) o[v] = z;
    }
  }
}

// dx[index[r]] = dy[r] for r < *count, zeros for the other rows (index is a permutation: one writer per row of dx).
__global__ void __launch_bounds__(kCompactThreads) scatter_rows_kernel(const __nv_bfloat16* __restrict__ dy, const int* __restrict__ index,
                                                                       const int* __restrict__ count, int T, int H,
                                                                       __nv_bfloat16* __restrict__ dx) {
  const int lane = threadIdx.x & 31, vecs = H / 8, live = __ldg(count);
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < T; r += (gridDim.x * blockDim.x) >> 5) {
    Bf16x8* o = reinterpret_cast<Bf16x8*>(dx + (size_t)__ldg(index + r) * H);
    if (r < live) {
      const Bf16x8* in = reinterpret_cast<const Bf16x8*>(dy + (size_t)r * H);
      for (int v = lane; v < vecs; v += 32) o[v] = in[v];
    } else {
      const Bf16x8 z = {};
      for (int v = lane; v < vecs; v += 32) o[v] = z;
    }
  }
}

constexpr int kColSumRows = 128, kColSumThreads = 128;

// partial[chunk][col] = sum of d[row, col] over the chunk's rows below the count, in row order; 8 columns per thread.
__global__ void __launch_bounds__(kColSumThreads) column_sum_kernel(const __nv_bfloat16* __restrict__ d, int rows, int cols,
                                                                    const int* __restrict__ bound, float* __restrict__ partial) {
  const int col = (blockIdx.x * kColSumThreads + threadIdx.x) * 8;
  const int end = bound != nullptr ? min(rows, __ldg(bound)) : rows;
  const int r0 = blockIdx.y * kColSumRows;
  if (col >= cols || r0 >= end) return;
  const int r1 = min(end, r0 + kColSumRows);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
  for (int r = r0; r < r1; ++r) {
    float v[8];
    unpack8(*reinterpret_cast<const Bf16x8*>(d + (size_t)r * cols + col), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += v[i];
  }
  float4* out = reinterpret_cast<float4*>(partial + (size_t)blockIdx.y * cols + col);
  out[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  out[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

__global__ void __launch_bounds__(256) column_sum_finish_kernel(const float* __restrict__ partial, int rows, int cols,
                                                                const int* __restrict__ bound, __nv_bfloat16* __restrict__ out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= cols) return;
  const int end = bound != nullptr ? min(rows, __ldg(bound)) : rows;
  float s = 0.f;
  for (int c = 0; c * kColSumRows < end; ++c) s += partial[(size_t)c * cols + col];
  out[col] = __float2bfloat16_rn(s);
}

void rows_check(const char* name, int T, int H, const void* a, const void* b) {
  if (T < 1 || H < 8 || H % 8 != 0 || ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15u) != 0)
    throw std::runtime_error(std::string(name) + ": needs T >= 1, H a positive multiple of 8 and 16-byte aligned rows, got T=" +
                             std::to_string(T) + " H=" + std::to_string(H));
}

}  // namespace

int compact_chunks(int T) { return ceil_div(T, kCompactChunk); }

void launch_compact_rows(const long long* targets, int T, long long ignore_index, long long vocab, int* workspace, int* index, int* count,
                         long long* targets_out, cudaStream_t s) {
  if (T < 1) throw std::runtime_error("compact_rows: no rows");
  const int chunks = compact_chunks(T);
  int* chunk_counts = workspace;
  int* chunk_base = workspace + chunks;
  compact_count_kernel<<<chunks, kCompactThreads, 0, s>>>(targets, T, ignore_index, vocab, chunk_counts);
  B200_CUDA_CHECK(cudaGetLastError());
  compact_scan_kernel<<<1, 32, 0, s>>>(chunk_counts, chunks, chunk_base, count);
  B200_CUDA_CHECK(cudaGetLastError());
  compact_scatter_kernel<<<chunks, kCompactThreads, 0, s>>>(targets, T, ignore_index, vocab, chunk_base, count, index, targets_out);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(3);
}

void launch_gather_rows(const void* x, const int* index, const int* count, int T, int H, void* out, cudaStream_t s) {
  rows_check("gather_rows", T, H, x, out);
  gather_rows_kernel<<<row_grid(T), kCompactThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), index, count, T, H,
                                                             reinterpret_cast<__nv_bfloat16*>(out));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

void launch_scatter_rows(const void* dy, const int* index, const int* count, int T, int H, void* dx, cudaStream_t s) {
  rows_check("scatter_rows", T, H, dy, dx);
  scatter_rows_kernel<<<row_grid(T), kCompactThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy), index, count, T, H,
                                                              reinterpret_cast<__nv_bfloat16*>(dx));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

size_t column_sum_workspace(int rows, int cols) { return (size_t)ceil_div(rows, kColSumRows) * cols; }

void launch_column_sum(const void* d, int rows, int cols, const int* bound, float* workspace, void* out, cudaStream_t s) {
  rows_check("column_sum", rows, cols, d, workspace);
  const dim3 grid(ceil_div(cols, 8 * kColSumThreads), ceil_div(rows, kColSumRows));
  column_sum_kernel<<<grid, kColSumThreads, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(d), rows, cols, bound, workspace);
  B200_CUDA_CHECK(cudaGetLastError());
  column_sum_finish_kernel<<<ceil_div(cols, 256), 256, 0, s>>>(workspace, rows, cols, bound, reinterpret_cast<__nv_bfloat16*>(out));
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(2);
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------------------
// GELU forward and backward as single vectorised passes, erf form (BERT), tanh approximation (GPT-2) or QuickGELU
// (CLIP).  The stock autograd formula for the backward (cast to fp32, erf, exp, three multiplies, cast back) is ~8 launches
// over a [tokens, 3072] tensor per BERT layer.
namespace b200 {
namespace {

__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad_f(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}
// tanh approximation: gelu(x) = 0.5 x (1 + t), t = tanh(u), u = sqrt(2 / pi) (x + 0.044715 x^3);
// gelu'(x) = 0.5 (1 + t) + 0.5 x (1 - t^2) sqrt(2 / pi) (1 + 3 * 0.044715 x^2)
constexpr float kSqrt2OverPi = 0.7978845608028654f;
constexpr float kGeluTanhC = 0.044715f;
__device__ __forceinline__ float gelu_tanh_f(float x) {
  return 0.5f * x * (1.f + tanhf(kSqrt2OverPi * (x + kGeluTanhC * x * x * x)));
}
__device__ __forceinline__ float gelu_tanh_grad_f(float x) {
  const float t = tanhf(kSqrt2OverPi * (x + kGeluTanhC * x * x * x));
  return 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * kSqrt2OverPi * (1.f + 3.f * kGeluTanhC * x * x);
}
// QuickGELU: x sigmoid(1.702 x); its derivative s + 1.702 x s (1 - s) with s = sigmoid(1.702 x)
constexpr float kQuickGeluC = 1.702f;
__device__ __forceinline__ float quick_gelu_f(float x) { return x / (1.f + __expf(-kQuickGeluC * x)); }
__device__ __forceinline__ float quick_gelu_grad_f(float x) {
  const float s = 1.f / (1.f + __expf(-kQuickGeluC * x));
  return s + kQuickGeluC * x * s * (1.f - s);
}
template <bool BWD, GeluForm FORM>
__device__ __forceinline__ float gelu_op(float x, float g) {
  if constexpr (FORM == GeluForm::kTanh) return BWD ? g * gelu_tanh_grad_f(x) : gelu_tanh_f(x);
  else if constexpr (FORM == GeluForm::kQuick) return BWD ? g * quick_gelu_grad_f(x) : quick_gelu_f(x);
  else return BWD ? g * gelu_grad_f(x) : gelu_f(x);
}

template <typename T, bool BWD, GeluForm FORM>
__global__ void __launch_bounds__(kLossThreads) gelu_kernel(const T* __restrict__ pre, const T* __restrict__ dy, T* __restrict__ out, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(out) | (BWD ? reinterpret_cast<uintptr_t>(dy) : 0)) & 31u) == 0;
  size_t done = 0;
  if (aligned) {
    const size_t nvec = n / 8;
    for (size_t v = tid; v < nvec; v += stride) {
      float a[8], g[8];
      load8<T>(pre + v * 8, a);
      if (BWD) load8<T>(dy + v * 8, g);
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = gelu_op<BWD, FORM>(a[i], g[i]);
      store8<T>(out + v * 8, a);
    }
    done = nvec * 8;
  }
  for (size_t i = done + tid; i < n; i += stride) {
    const float x = to_f32<T>(pre[i]);
    out[i] = from_f32<T>(gelu_op<BWD, FORM>(x, BWD ? to_f32<T>(dy[i]) : 0.f));
  }
}

}  // namespace

template <GeluForm FORM>
void gelu_dispatch(const void* pre, const void* dy, void* out, DType dt, size_t n, bool backward, int blocks, cudaStream_t s) {
  if (dt == DType::BF16) {
    if (backward) gelu_kernel<__nv_bfloat16, true, FORM><<<blocks, kLossThreads, 0, s>>>((const __nv_bfloat16*)pre, (const __nv_bfloat16*)dy, (__nv_bfloat16*)out, n);
    else gelu_kernel<__nv_bfloat16, false, FORM><<<blocks, kLossThreads, 0, s>>>((const __nv_bfloat16*)pre, nullptr, (__nv_bfloat16*)out, n);
  } else {
    if (backward) gelu_kernel<float, true, FORM><<<blocks, kLossThreads, 0, s>>>((const float*)pre, (const float*)dy, (float*)out, n);
    else gelu_kernel<float, false, FORM><<<blocks, kLossThreads, 0, s>>>((const float*)pre, nullptr, (float*)out, n);
  }
}

void launch_gelu(const void* pre, const void* dy, void* out, DType dt, size_t n, bool backward, cudaStream_t s, GeluForm form) {
  size_t b = (n / 8 + kLossThreads - 1) / kLossThreads;
  if (b < 1) b = 1;
  if (b > (size_t)16 * kNumSMs) b = (size_t)16 * kNumSMs;
  const int blocks = (int)b;
  if (form == GeluForm::kTanh) gelu_dispatch<GeluForm::kTanh>(pre, dy, out, dt, n, backward, blocks, s);
  else if (form == GeluForm::kQuick) gelu_dispatch<GeluForm::kQuick>(pre, dy, out, dt, n, backward, blocks, s);
  else gelu_dispatch<GeluForm::kErf>(pre, dy, out, dt, n, backward, blocks, s);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace b200

// ---------------------------------------------------------------------------------------------------------
// SwiGLU (Llama MLP): in = [M, 2I] bf16 with column blocks gate | up, out = silu(gate) * up [M, I].  The backward writes
// d[gate | up] [M, 2I] in one pass: dgate = dy * up * silu'(gate), dup = dy * silu(gate), silu'(g) = s (1 + g (1 - s)),
// s = sigmoid(g).  One thread per 8 consecutive columns (I % 8 == 0), 16-byte loads and stores.
// GeGLU (ModernBERT MLP) is the same kernel with the erf-form GELU on the first block: out = gelu(input) * gate, and
// d[input | gate] = [dy * gate * gelu'(input), dy * gelu(input)].
namespace b200 {
namespace {

enum class GluAct { kSilu, kGelu };

template <bool BWD, GluAct ACT = GluAct::kSilu>
__global__ void __launch_bounds__(kLossThreads) swiglu_kernel(const __nv_bfloat16* __restrict__ in, const __nv_bfloat16* __restrict__ dy,
                                                              __nv_bfloat16* __restrict__ out, size_t rows, int inter) {
  const int vpr = inter / 8;                                    // 8-column vectors per row
  const size_t n = rows * (size_t)vpr;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (size_t)gridDim.x * blockDim.x) {
    const size_t r = v / vpr;
    const int c = (int)(v - r * vpr) * 8;
    const __nv_bfloat16* gp = in + r * 2 * inter + c;
    float g[8], u[8];
    unpack8(*reinterpret_cast<const Bf16x8*>(gp), g);
    unpack8(*reinterpret_cast<const Bf16x8*>(gp + inter), u);
    if constexpr (BWD) {
      float d[8], dg[8], du[8];
      unpack8(*reinterpret_cast<const Bf16x8*>(dy + r * inter + c), d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if constexpr (ACT == GluAct::kGelu) {
          du[i] = d[i] * gelu_f(g[i]);
          dg[i] = d[i] * u[i] * gelu_grad_f(g[i]);
        } else {
          const float sg = 1.f / (1.f + expf(-g[i]));
          du[i] = d[i] * g[i] * sg;
          dg[i] = d[i] * u[i] * sg * (1.f + g[i] * (1.f - sg));
        }
      }
      __nv_bfloat16* op = out + r * 2 * inter + c;
      *reinterpret_cast<Bf16x8*>(op) = pack8(dg);
      *reinterpret_cast<Bf16x8*>(op + inter) = pack8(du);
    } else {
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if constexpr (ACT == GluAct::kGelu) o[i] = gelu_f(g[i]) * u[i];
        else o[i] = g[i] / (1.f + expf(-g[i])) * u[i];
      }
      *reinterpret_cast<Bf16x8*>(out + r * inter + c) = pack8(o);
    }
  }
}

template <GluAct ACT>
void launch_glu(const char* name, const void* in_act, const void* dy, void* out, size_t rows, int inter, bool backward, cudaStream_t s) {
  if (inter % 8 != 0 || ((reinterpret_cast<uintptr_t>(in_act) | reinterpret_cast<uintptr_t>(out) |
                          reinterpret_cast<uintptr_t>(dy)) & 15u) != 0)
    throw std::runtime_error(std::string(name) + ": needs the intermediate size a multiple of 8 and 16-byte aligned tensors (inter=" +
                             std::to_string(inter) + ")");
  size_t b = (rows * (inter / 8) + kLossThreads - 1) / kLossThreads;
  if (b < 1) b = 1;
  if (b > (size_t)16 * kNumSMs) b = (size_t)16 * kNumSMs;
  const auto* in = reinterpret_cast<const __nv_bfloat16*>(in_act);
  if (backward)
    swiglu_kernel<true, ACT><<<(int)b, kLossThreads, 0, s>>>(in, reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<__nv_bfloat16*>(out), rows, inter);
  else
    swiglu_kernel<false, ACT><<<(int)b, kLossThreads, 0, s>>>(in, nullptr, reinterpret_cast<__nv_bfloat16*>(out), rows, inter);
  B200_CUDA_CHECK(cudaGetLastError()); B200_COUNT_LAUNCH(1);
}

}  // namespace

void launch_swiglu(const void* gate_up, const void* dy, void* out, size_t rows, int inter, bool backward, cudaStream_t s) {
  launch_glu<GluAct::kSilu>("swiglu", gate_up, dy, out, rows, inter, backward, s);
}

void launch_geglu(const void* input_gate, const void* dy, void* out, size_t rows, int inter, bool backward, cudaStream_t s) {
  launch_glu<GluAct::kGelu>("geglu", input_gate, dy, out, rows, inter, backward, s);
}

}  // namespace b200
