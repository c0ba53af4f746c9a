// Host-callable entry points of the single-GPU kernels (optimizer, losses, norms, linears).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "common.h"

namespace b200 {

// ---------------- multi-tensor optimizer (optim.cu) ------------------------------------------
constexpr int kMaxOptTensors = 120;
constexpr int kOptChunk = 8192;   // elements per block

struct OptSlot {
  void* p;              // model parameter (fp32 or bf16)
  const void* g;        // gradient (fp32 or bf16), may live anywhere (stolen autograd buffer or bucket view)
  unsigned long long flat_off;  // element offset into the flat fp32 master / momentum buffers
  uint32_t numel;
  uint32_t blk0;        // first block of this tensor inside the launch
};
struct OptTable {
  int count;
  int total_blocks;
  OptSlot t[kMaxOptTensors];
};
struct SgdHyper {
  const float* lr;          // device scalar: never baked into a CUDA graph
  const float* clip_coef;   // device scalar from clip_coef kernel (nullptr = 1)
  float* master;            // flat fp32 master weights (nullptr when params are fp32)
  float* momentum_buf;      // flat fp32 (nullptr when momentum == 0)
  const int* step_count;    // device scalar; 0 on the first step (momentum buffer init)
  float momentum, dampening, weight_decay, grad_scale;
  int nesterov;
  int zero_grad;            // write zeros back into g after use
};
// AdamW (decoupled weight decay).  One launch per (param group, dtype, table): the table fills the kernel-parameter space,
// so per-group hyper-parameters travel here rather than per slot.
struct AdamHyper {
  const float* lr;          // device scalar of this param group
  const float* clip_coef;   // device scalar from clip_coef kernel (nullptr = 1)
  float* master;            // flat fp32 master weights (nullptr when params are fp32)
  float* exp_avg;           // flat fp32 first moment
  float* exp_avg_sq;        // flat fp32 second moment
  const int* step_count;    // device scalar: steps already taken (bias correction uses *step_count + 1)
  float beta1, beta2, eps, weight_decay, grad_scale;
  int zero_grad;            // write zeros back into g after use
};

void launch_multi_sqnorm(const OptTable& tab, DType g_dtype, float* partials /*[total_blocks]*/, cudaStream_t s);
void launch_clip_coef(const float* partials, int n, float max_norm, float grad_scale, float* coef_out,
                      float* norm_out, cudaStream_t s);
void launch_multi_sgd(const OptTable& tab, DType p_dtype, DType g_dtype, const SgdHyper& h, cudaStream_t s);
void launch_multi_adamw(const OptTable& tab, DType p_dtype, DType g_dtype, const AdamHyper& h, cudaStream_t s);
void launch_scale_inplace(float* x, size_t n, const float* scalar, cudaStream_t s);

// ---------------- losses (loss.cu) --------------------------------------------------------------
// MSE: loss = mean((o-t)^2) ; dO = 2 (o-t) / N * gscale      (reference criterion, ddp.py:164)
void launch_mse_fwd_bwd(const void* out, const void* target, DType dt, size_t n, float gscale,
                        float* loss /*1*/, void* dout, float* scratch /*[blocks+1]*/, int blocks, cudaStream_t s);
int mse_blocks(size_t n);
// Softmax cross-entropy over rows: loss = mean_i(lse_i - x[i, t_i]); dX = (softmax - onehot)/rows*gscale
void launch_xent_fwd_bwd(const void* logits, const long long* targets, DType dt, int rows, int cols,
                         long long ignore_index, float gscale, float* row_loss /*[rows+1]*/, float* loss /*1*/,
                         void* dlogits, cudaStream_t s);

// GELU forward: out = gelu(pre); backward: out = dy * gelu'(pre).  One vectorised pass each (loss.cu).  The erf form, or
// with `tanh` the tanh approximation 0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3))) (GPT-2's MLP).
void launch_gelu(const void* pre, const void* dy, void* out, DType dt, size_t n, bool backward, cudaStream_t s, bool tanh = false);

// SwiGLU: forward out[M, I] = silu(gate) * up from gate_up bf16 [M, 2I] (gate | up); backward out[M, 2I] = d[gate | up]
// from dy [M, I].  I % 8 == 0, 16-byte aligned tensors (loss.cu).
void launch_swiglu(const void* gate_up, const void* dy, void* out, size_t rows, int inter, bool backward, cudaStream_t s);

// ---------------- rotary position embedding (rotary.cu) ----------------------------------------------
// qkv bf16 [rows, (heads + 2*kv_heads)*head_dim] -> y (same shape), head_dim 64 or 128: query and key heads rotated by
// position pos[r] (int32, clamped to [0, max_pos)), value heads copied; table fp32 [max_pos, 2, head_dim / 2] (cos | sin).
// backward: the transpose rotation.
void launch_rotary(const void* x, const int* pos, const float* table, int max_pos, size_t rows, int heads, int kv_heads, int head_dim,
                   void* y, bool backward, cudaStream_t s);

// ---------------- layer norm (layernorm.cu) -----------------------------------------------------
void launch_layernorm_fwd(const void* x, const void* gamma, const void* beta, DType dt, int rows, int cols,
                          float eps, void* y, float* mean, float* rstd, cudaStream_t s);
void launch_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                          DType dt, int rows, int cols, void* dx, float* dgamma_partial, float* dbeta_partial,
                          int partial_rows, void* dgamma, void* dbeta, cudaStream_t s);
int layernorm_partial_rows(int rows);
// RMSNorm, y = x * rsqrt(mean(x^2) + eps) * gamma, on the LayerNorm fast path up to 1024 columns and on one CTA per row
// above that: cols % 8 == 0, cols <= 4096, 32-byte aligned tensors.  rstd fp32 [rows]; backward workspace partial fp32
// [2 * partial_rows, cols], counters uint32 [cols / 8].
bool rmsnorm_supported(int cols);
void launch_rmsnorm_fwd(const void* x, const void* gamma, DType dt, int rows, int cols, float eps, void* y, float* rstd, cudaStream_t s);
void launch_rmsnorm_bwd(const void* dy, const void* x, const void* gamma, const float* rstd, DType dt, int rows, int cols, void* dx,
                        float* partial, unsigned int* counters, int partial_rows, void* dgamma, cudaStream_t s);

// ---------------- FP8 quantisation, current per-tensor power-of-two scaling (fp8.cu) ------------------
// amax[0] = max |x| over n bf16 elements (x 16-byte aligned); zeroes amax first, so the two launches are graph-capturable.
void launch_fp8_amax(const void* x, size_t n, float* amax, cudaStream_t s);
// x bf16 [rows, cols] (cols % 16 == 0) -> q [rows, cols] E4M3 (or E5M2), optionally qt = q^T [cols, rows] (rows % 16 == 0)
// and colsum[cols] = fp32 column sums of x (colsum_partial: fp32 [fp8_colsum_parts(rows), cols] workspace).  The scale
// s = 2^e comes from amax in device memory; *scale_inv = 1/s.
void launch_fp8_cast_transpose(const void* x, int rows, int cols, const float* amax, bool e5m2, void* q, void* qt,
                               float* colsum_partial, float* colsum, float* scale_inv, cudaStream_t s);
int fp8_colsum_parts(int rows);

// ---------------- key-padding attention on wgmma, head dim 64 (attention.cu) ------------------------
// qkv bf16 [B*S, 3*heads*64] (16-byte aligned), seq_lens int32 [B] on the device (clamped to [0, S]), S % 128 == 0.
// o bf16 [B*S, heads*64]; lse fp32 [B, heads, S], natural log (-inf where the length is 0).
void launch_attention_fwd(const void* qkv, const int* seq_lens, int B, int S, int heads, void* o, float* lse, cudaStream_t s);
// dout, o bf16 [B*S, heads*64] (16-byte aligned); dsum fp32 [B, heads, S] workspace; dqkv bf16 [B*S, 3*heads*64], every
// element written.  Three launches: rowsum(dO * O), dK / dV, dQ.  Deterministic.
void launch_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* seq_lens, int B, int S,
                          int heads, float* dsum, void* dqkv, cudaStream_t s);
// Packed documents: bounds int32 [B*S, 2] on the device (8-byte aligned), (start, end) per row in its sequence's
// coordinates; query i sees key j of its sequence iff start[i] <= j < end[i] (clamped on the device).  A row with
// start == end gets zero output, lse = -inf and zero gradients.  Same shapes, outputs and workspace as above.
void launch_packed_attention_fwd(const void* qkv, const int* bounds, int B, int S, int heads, void* o, float* lse, cudaStream_t s);
void launch_packed_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                 int S, int heads, float* dsum, void* dqkv, cudaStream_t s);
// Causal documents: the same bounds, and query i also sees no key after itself: key j iff start[i] <= j <= i and
// j < end[i].  Padding rows as above; same shapes, outputs and workspace.
void launch_causal_attention_fwd(const void* qkv, const int* bounds, int B, int S, int heads, void* o, float* lse, cudaStream_t s);
void launch_causal_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                 int S, int heads, float* dsum, void* dqkv, cudaStream_t s);
// Grouped-query causal documents: qkv (and dqkv) bf16 [B*S, (heads + 2*kv_heads)*64], query | key | value column blocks;
// query head h reads K/V head h / (heads / kv_heads).  o, lse, dout and dsum as above (heads query heads).
void launch_causal_gqa_attention_fwd(const void* qkv, const int* bounds, int B, int S, int heads, int kv_heads, void* o, float* lse,
                                     cudaStream_t s);
void launch_causal_gqa_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                     int S, int heads, int kv_heads, float* dsum, void* dqkv, cudaStream_t s);
// The same causal documents at head dim 128: qkv (and dqkv) bf16 [B*S, (heads + 2*kv_heads)*128], o and dout
// [B*S, heads*128]; kv_heads divides heads (kv_heads == heads is multi-head attention).
void launch_causal_attention_d128_fwd(const void* qkv, const int* bounds, int B, int S, int heads, int kv_heads, void* o, float* lse,
                                      cudaStream_t s);
void launch_causal_attention_d128_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds, int B,
                                      int S, int heads, int kv_heads, float* dsum, void* dqkv, cudaStream_t s);

// ---------------- small linears on CUDA cores (linear_small.cu) ------------------------------
// y[M,N] = act(x[M,K] w[N,K]^T + b[N]) ; fp32, dims far below one tensor-core tile (FooModel).
void launch_small_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int N, int K,
                             int relu, cudaStream_t s);
void launch_small_linear_bwd(const float* dy, const float* x, const float* w, const float* y, float* dx,
                             float* dw, float* db, int M, int N, int K, int relu, int accumulate, cudaStream_t s);

// ---------------- fused training BatchNorm (+residual) (+ReLU), channels_last (batchnorm.cu) --------------
// x viewed as row-major [R = N*H*W, C]; C % 8 == 0; gamma/beta/statistics fp32.
void bn_workspace_sizes(int R, int C, size_t* partial_floats, size_t* counters);
// -1 = read B200DDP_PDL (default 0); 1 = statistics -> apply and bwd-reduce -> bwd-apply as programmatic dependent launches
void set_bn_pdl(int on);
// 1 = never select the single-read resident kernels (compare against / benchmark the two-pass kernels); 0 = default
void set_bn_two_pass(int on);
// nonzero once a resident BatchNorm kernel's grid barrier wait has timed out (co-residency failure)
unsigned int bn_resident_error();
void launch_bn_forward(const void* x, const void* residual, void* y, unsigned char* relu_mask /*[R, C/8] or null*/, DType dt, int R, int C, const float* gamma, const float* beta,
                       float* running_mean, float* running_var, long long* num_batches, float* save_mean, float* save_rstd,
                       float* scale, float* shift, float* partial, unsigned int* counters, float eps, float momentum, bool relu,
                       cudaStream_t s);
// Same as launch_bn_forward, but the statistics come from `partial` = [2][groups][C] partial column sums / sums of squares
// (written by the GEMM epilogue that produced x): finish kernel + apply kernel, x is read once instead of twice.
void launch_bn_forward_from_partials(const void* x, const void* residual, void* y, unsigned char* relu_mask, DType dt, int R, int C,
                                     const float* gamma, const float* beta, float* running_mean, float* running_var,
                                     long long* num_batches, float* save_mean, float* save_rstd, float* scale, float* shift,
                                     const float* partial, int groups, float eps, float momentum, bool relu, cudaStream_t s);
// Backward with S1 / S2 partial sums ([2][groups][C]) from the data-gradient epilogue of the consuming convolution: one launch
// (reduce the partials per block, apply), no pass over dy and x for the reduction.
void launch_bn_backward_from_partials(const void* dy, const void* x, const void* relu_mask, void* dx, void* dres, DType dt, int R, int C, const float* gamma,
                                      const float* save_mean, const float* save_rstd, float* dgamma, float* dbeta, const float* partial, int groups,
                                      bool relu, cudaStream_t s);
void launch_bn_backward(const void* dy, const void* x, const void* relu_mask, void* dx, void* dres, DType dt, int R, int C, const float* gamma,
                        const float* save_mean, const float* save_rstd, float* dgamma, float* dbeta, float* coef, float* partial,
                        unsigned int* counters, bool relu, cudaStream_t s);

// ---------------- 3x3/s2/p1 max pooling, channels_last (pool.cu) ------------------------------------------
void launch_maxpool3x3s2_fwd(const void* x, void* y, unsigned char* idx, DType dt, int N, int H, int W, int C, cudaStream_t s);
void launch_maxpool3x3s2_bwd(const void* dy, const unsigned char* idx, void* dx, DType dt, int N, int H, int W, int C, cudaStream_t s);

// ---------------- input pipeline (input.cu) -----------------------------------------------------
// NCHW (u8 or fp32) -> NHWC-in-memory (channels_last) bf16/fp32 with per-channel (x*scale - mean)/std
void launch_normalize_to_channels_last(const void* src, DType src_dt, void* dst, DType dst_dt, int n, int c, int c_out,
                                       int h, int w, const float* mean, const float* inv_std, float in_scale,
                                       cudaStream_t s);

}  // namespace b200
