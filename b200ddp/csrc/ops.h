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
// Fused LM-head cross-entropy, after launch_gemm_lm_lse (gemm.h): lse[row] from the per-tile partials fp32
// [tiles][rows][2] (a fixed-order merge), row_loss [rows+1] (lse - target logit, 0 for ignored rows; row_loss[rows] = the
// number of non-ignored rows) and loss = their mean (0 when every row is ignored).
// bound (optional): int32 device count; rows at or past it get lse = row_loss = 0 and their partials are not read.
void launch_lm_loss_combine(const float* partial, const float* target_logit, const long long* targets, int rows, int tiles, int cols,
                            long long ignore_index, float* lse, float* row_loss, float* loss, cudaStream_t s, const int* bound = nullptr);

// Sparse prediction (loss.cu).  compact_rows: a stable partition of T rows, those whose target is not ignore_index and lies
// in [0, vocab) first.  index int32 [T] (the original row at each position), count int32 [1] (labelled rows), targets_out
// int64 [T] (the labelled targets, then ignore_index); workspace int32 [2 * compact_chunks(T)].
int compact_chunks(int T);
void launch_compact_rows(const long long* targets, int T, long long ignore_index, long long vocab, int* workspace, int* index, int* count,
                         long long* targets_out, cudaStream_t s);
// gather_rows: out[r] = x[index[r]] for r < *count, zero rows after; scatter_rows: dx[index[r]] = dy[r] for r < *count and
// zeros for the other rows of dx (index a permutation of [0, T)).  bf16 [T, H], H % 8 == 0.
void launch_gather_rows(const void* x, const int* index, const int* count, int T, int H, void* out, cudaStream_t s);
void launch_scatter_rows(const void* dy, const int* index, const int* count, int T, int H, void* dx, cudaStream_t s);
// column_sum: out bf16 [cols] = sum over rows r < min(rows, *bound) (all rows when bound is null) of d bf16 [rows, cols],
// in a fixed order; cols % 8 == 0; workspace fp32 [column_sum_workspace(rows, cols)].
size_t column_sum_workspace(int rows, int cols);
void launch_column_sum(const void* d, int rows, int cols, const int* bound, float* workspace, void* out, cudaStream_t s);

// GELU forward: out = gelu(pre); backward: out = dy * gelu'(pre).  One vectorised pass each (loss.cu).  The erf form, the
// tanh approximation 0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3))) (GPT-2's MLP) or QuickGELU x sigmoid(1.702 x) (CLIP's).
enum class GeluForm { kErf, kTanh, kQuick };
void launch_gelu(const void* pre, const void* dy, void* out, DType dt, size_t n, bool backward, cudaStream_t s,
                 GeluForm form = GeluForm::kErf);

// SwiGLU: forward out[M, I] = silu(gate) * up from gate_up bf16 [M, 2I] (gate | up); backward out[M, 2I] = d[gate | up]
// from dy [M, I].  I % 8 == 0, 16-byte aligned tensors (loss.cu).
void launch_swiglu(const void* gate_up, const void* dy, void* out, size_t rows, int inter, bool backward, cudaStream_t s);
// GeGLU: the same with the erf-form GELU, forward out[M, I] = gelu(input) * gate from input_gate bf16 [M, 2I]
// (input | gate); backward out[M, 2I] = d[input | gate] from dy [M, I].  I % 8 == 0, 16-byte aligned tensors (loss.cu).
void launch_geglu(const void* input_gate, const void* dy, void* out, size_t rows, int inter, bool backward, cudaStream_t s);

// ---------------- rotary position embedding (rotary.cu) ----------------------------------------------
// qkv bf16 [rows, (heads + 2*kv_heads)*head_dim] -> y (same shape), head_dim 64 or 128: query and key heads rotated by
// position pos[r] (int32, clamped to [0, max_pos)), value heads copied; table fp32 [max_pos, 2, head_dim / 2] (cos | sin).
// backward: the transpose rotation.  q_scale (a positive power of two) also multiplies the query heads, in both directions
// (Granite's attention multiplier folded into q).
void launch_rotary(const void* x, const int* pos, const float* table, int max_pos, size_t rows, int heads, int kv_heads, int head_dim,
                   void* y, bool backward, cudaStream_t s, float q_scale = 1.f);
// Qwen3's per-head q / k RMSNorm fused with rotary, head_dim 128 only, same layouts, positions and table as launch_rotary.
// Forward: y = rope(x * rstd * w) per query head (w = wq [128]) and key head (w = wk [128]), rstd = rsqrt(mean(x^2) + eps)
// over the head in fp32, one bf16 rounding; value heads copied; rstd fp32 [rows, heads + kv_heads].  Backward from dy and
// the forward's x and rstd: dx (value heads pass through), dwq / dwk bf16 [128] = sum of rope^-1(dy) * x * rstd over rows
// and query / key heads, with no atomics: per-CTA partials in partial fp32 [2, qk_norm_rotary_partials(rows), 128],
// summed in CTA order; the grid depends on rows only, so repeated calls are bitwise identical.
int qk_norm_rotary_partials(size_t rows);
void launch_qk_norm_rotary_fwd(const void* x, const void* wq, const void* wk, const int* pos, const float* table, int max_pos, size_t rows,
                               int heads, int kv_heads, int head_dim, float eps, void* y, float* rstd, cudaStream_t s);
void launch_qk_norm_rotary_bwd(const void* dy, const void* x, const float* rstd, const void* wq, const void* wk, const int* pos,
                               const float* table, int max_pos, size_t rows, int heads, int kv_heads, int head_dim, void* dx,
                               float* partial, void* dwq, void* dwk, cudaStream_t s);

// ---------------- mixture-of-experts routing, permutation and combine (moe.cu) -----------------------------
// T tokens, E <= 64 experts, k <= min(E, 8) experts per token, hidden H % 64 == 0.  Deterministic, no atomics, no host
// synchronisation: every buffer size follows from (T, E, k) alone.
constexpr int kMoeMaxExperts = 64, kMoeMaxTopK = 8, kMoeAlign = 128;
inline int moe_capacity(int T, int E, int k) { return (int)(((long long)T * k + (long long)E * (kMoeAlign - 1) + kMoeAlign - 1) / kMoeAlign * kMoeAlign); }
inline int moe_chunks(int T, int k) { return (int)(((long long)T * k + 1023) / 1024); }
// Router: logits bf16 [T, E] -> ids int32 [T, k] (top-k, ties to the lower expert), gates bf16 [T, k] (softmax of the k
// logits in fp32, rounded once); with probsum != nullptr also probsum fp32 [E] = sum over tokens of softmax(logits)
// (partial: fp32 [ceil(T / 64), E] workspace, reduced in a fixed order).
void launch_moe_router_fwd(const void* logits, int T, int E, int k, int* ids, void* gates, float* partial, float* probsum, cudaStream_t s);
// dlogits bf16 [T, E] = top-k softmax Jacobian . dgates (fp32 [T, k]) + (dprobsum != nullptr) full-softmax Jacobian . dprobsum [E].
void launch_moe_router_bwd(const void* logits, int T, int E, int k, const int* ids, const float* dgates, const float* dprobsum,
                           void* dlogits, cudaStream_t s);
// Stable counting sort of the T*k assignments a = t*k + j by expert: counts int32 [E], offsets int32 [E + 1] (segment
// starts, multiples of 128), fwd_map int32 [capacity] (permuted row -> a, -1 in padding), inv_map int32 [T*k] (a -> row),
// tile_expert int32 [capacity / 128] (-1 for unused tiles).  chunk_counts: int32 [2, moe_chunks(T, k), E] workspace.
void launch_moe_permute(const int* ids, int T, int E, int k, int* chunk_counts, int* counts, int* offsets, int* fwd_map, int* inv_map,
                        int* tile_expert, cudaStream_t s);
// x_perm bf16 [capacity, H]: row r = x[fwd_map[r] / k], zeros where fwd_map[r] < 0.
void launch_moe_gather(const void* x, const int* fwd_map, int capacity, int H, int k, void* x_perm, cudaStream_t s);
// out bf16 [T, H]: out[t] = sum_j gate[t, j] * y_perm[inv_map[t*k + j]] in fp32, slot order (gates == nullptr: weight 1).
void launch_moe_combine(const void* y_perm, const int* inv_map, const void* gates, int T, int H, int k, void* out, cudaStream_t s);
// Combine backward, one writer per row: dy_perm bf16 [capacity, H] = gate * dout[token] (zeros in padding rows) and
// dgates fp32 [T, k] = <dout[token], y_perm[row]>.
void launch_moe_combine_bwd(const void* dout, const void* y_perm, const int* fwd_map, const void* gates, int capacity, int H, int k,
                            void* dy_perm, float* dgates, cudaStream_t s);

// ---------------- layer norm (layernorm.cu) -----------------------------------------------------
void launch_layernorm_fwd(const void* x, const void* gamma, const void* beta, DType dt, int rows, int cols,
                          float eps, void* y, float* mean, float* rstd, cudaStream_t s);
void launch_layernorm_bwd(const void* dy, const void* x, const void* gamma, const float* mean, const float* rstd,
                          DType dt, int rows, int cols, void* dx, float* dgamma_partial, float* dbeta_partial,
                          int partial_rows, void* dgamma, void* dbeta, cudaStream_t s);
int layernorm_partial_rows(int rows);
// out_a / out_b bf16 [cols] = sum over p < parts of partial_a / partial_b fp32 [parts, cols], in part order (the general
// LayerNorm backward's finish kernel)
void launch_column_sum_pair_bf16(const float* partial_a, const float* partial_b, int parts, int cols, void* out_a, void* out_b,
                                 cudaStream_t s);
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

// ---------------- Vision Transformer patch embedding (vit.cu), bf16 --------------------------------
// Token stream of T rows (T >= B (N + 1), N = (H / p) (W / p) patches, per = N + 1): image b owns rows [b per, (b + 1) per),
// its class token first; rows past B per are padding.  p % 8 == 0, H % p == W % p == 0, D % 8 == 0, 16-byte aligned rows.
// out [T, C p p] = the patches in token order, k = (c, ky, kx); zero at class and padding rows
void launch_patchify(const void* img, bool channels_last, int B, int C, int H, int W, int p, int T, void* out, cudaStream_t s);
// out [T, D] = cls + pos[0] at class rows, y + pos[j] at patch rows (fp32 add), 0 at padding rows
void launch_patch_assemble(const void* y, const void* cls, const void* pos, int B, int per, int D, int T, void* out, cudaStream_t s);
// dpatch [T, D] = dy at patch rows, 0 elsewhere; dpos [per, D] = fixed-order fp32 sums over the B images; dcls [D] = dpos[0]
void launch_patch_embed_bwd(const void* dy, int B, int per, int D, int T, void* dpatch, void* dpos, void* dcls, cudaStream_t s);

// ---------------- ConvNeXt depthwise 7x7 convolution, stride 1, padding 3 (convnext.cu), bf16 NHWC ---------------------
// x, y, dy, dx [B, H, W, C] contiguous and 16-byte aligned, 8 <= C <= 1024, C % 8 == 0; w [C, 49] (a contiguous or
// channels_last [C, 1, 7, 7]); bias [C] or null.  fp32 sums in a fixed order, one bf16 rounding, no atomics.
// y = b + sum over the 49 taps of x (zero outside the image) times w
void launch_dwconv_fwd(const void* x, const void* w, const void* bias, int B, int H, int W, int C, void* y, cudaStream_t s);
// dx = the forward of dy with the kernel flipped, no bias
void launch_dwconv_dgrad(const void* dy, const void* w, int B, int H, int W, int C, void* dx, cudaStream_t s);
// dw bf16 [C, 49] and db bf16 [C] through part fp32 [dwconv_wgrad_slots(B, H, W), 50, C]: one slot per (image, spatial
// tile), summed in slot order.  dy is read at real pixels only.
int dwconv_wgrad_slots(int B, int H, int W);
void launch_dwconv_wgrad(const void* dy, const void* x, int B, int H, int W, int C, float* part, void* dw, void* db, cudaStream_t s);

// ---------------- Swin shifted-window attention, window 7, head dim 32 (swin.cu), bf16 raster rows ----------------------
// qkv [B*H*W, 3C] (C = 32 heads, columns q | k | v), 16-byte aligned; table fp32 [169, heads]; H, W multiples of 7,
// 0 <= sy, sx < 7.  o bf16 [B*H*W, C], lse fp32 [B*H*W, heads].  No atomics, no host synchronisation.
int swin_windows(int B, int H, int W);
void launch_swin_attention_fwd(const void* qkv, const float* table, int B, int H, int W, int heads, int sy, int sx, void* o, float* lse,
                               cudaStream_t s);
// dqkv bf16 [B*H*W, 3C]; dtable fp32 [169, heads] through part fp32 [heads, swin_windows(B, H, W), 169]: one partial per
// (head, window), summed in window order
void launch_swin_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const float* table, int B, int H, int W,
                               int heads, int sy, int sx, void* dqkv, float* part, float* dtable, cudaStream_t s);
// Swin V2's cosine attention, window 8: qkv as above; table fp32 [225, heads] (16 sigmoid of the cpb MLP), scale fp32
// [heads] (exp of the clamped logit_scale); H, W multiples of 8, 0 <= sy, sx < 8.  o and lse as above.
int swin_v2_windows(int B, int H, int W);
void launch_swin_v2_attention_fwd(const void* qkv, const float* table, const float* scale, int B, int H, int W, int heads, int sy, int sx,
                                  void* o, float* lse, cudaStream_t s);
// dqkv bf16 [B*H*W, 3C]; dtable fp32 [226, heads], rows 0 .. 224 the table gradient and row 225 d scale, through part fp32
// [heads, swin_v2_windows(B, H, W), 226]: one partial per (head, window), summed in window order
void launch_swin_v2_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const float* table, const float* scale,
                                  int B, int H, int W, int heads, int sy, int sx, void* dqkv, float* part, float* dtable, cudaStream_t s);

// ---------------- Mamba causal conv1d + SiLU and selective scan (mamba.cu), bf16 token rows -------------------------------
// T = B S rows; bounds int32 [B, S, 2] (document (start, end) per position, start == end for padding); E % 8 == 0, N = 16,
// conv width 4.  xz bf16 [T, 2E] = x | z, u / draw / y bf16 [T, E], xbc bf16 [T, R + 32] = dt | B | C; A_log fp32 [E, 16],
// D / dt_bias fp32 [E]; conv weight fp32 [E, 4], bias fp32 [E].  No atomics, no host synchronisation.
int mamba_conv_blocks(int B, int S);
int mamba_chunks(int S);
int mamba_groups(int E);
void launch_mamba_conv_fwd(const void* xz, const float* w, const float* bias, const int* bounds, int B, int S, int E, void* u, cudaStream_t s);
// dx into the x half of dxz [T, 2E]; dw fp32 [E, 4], db fp32 [E] through part fp32 [mamba_conv_blocks(B, S), 5, E]
void launch_mamba_conv_bwd(const void* du, const void* xz, const float* w, const float* bias, const int* bounds, int B, int S, int E, void* dxz,
                           float* part, float* dw, float* db, cudaStream_t s);
// hst fp32 [B, mamba_chunks(S), E, 16] (each chunk's start state, kept for the backward), sumd fp32 [B, chunks, E]
void launch_mamba_scan_fwd(const void* u, const void* draw, const void* xbc, const void* xz, const float* A_log, const float* D,
                           const float* dt_bias, const int* bounds, int B, int S, int E, int R, void* y, float* hst, float* sumd,
                           cudaStream_t s);
// du, ddraw bf16 [T, E]; dz into the z half of dxz [T, 2E]; dxbc bf16 [T, R + 32] (zero dt columns); dA_log fp32 [E, 16],
// dD, dbias fp32 [E].  Scratch: dq fp32 like hst, dbc_part fp32 [T, mamba_groups(E), 32], dA_part fp32 [B chunks, E, 16],
// dD_part and dbias_part fp32 [B chunks, E]
void launch_mamba_scan_bwd(const void* dy, const void* u, const void* draw, const void* xbc, const void* xz, const float* A_log, const float* D,
                           const float* dt_bias, const int* bounds, const float* hst, const float* sumd, int B, int S, int E, int R,
                           float* dq, float* dbc_part, float* dA_part, float* dD_part, float* dbias_part, void* du, void* ddraw, void* dxbc,
                           void* dxz, float* dA_log, float* dD, float* dbias, cudaStream_t s);

// ---------------- Mamba-2 (mamba2.cu, mamba.cu, layernorm.cu), bf16 token rows --------------------------------------------
// T = B S rows, bounds int32 [B, S, 2] as for Mamba-1.  Row views (x, dx, dt, ddt, z, dz) are read and written through their
// row pitch in elements (a multiple of 8), 16-byte aligned.  No atomics, no host synchronisation.
// Conv (width 4) + SiLU over E channels of x [T, *] (pitch x_pitch) -> u bf16 [T, E]; the backward writes dx (pitch
// dx_pitch), dw fp32 [E, 4], db fp32 [E] through part fp32 [mamba_conv_blocks(B, S), 5, E].
void launch_mamba2_conv_fwd(const void* x, long long x_pitch, const float* w, const float* bias, const int* bounds, int B, int S, int E,
                            void* u, cudaStream_t s);
void launch_mamba2_conv_bwd(const void* du, const void* x, long long x_pitch, const float* w, const float* bias, const int* bounds, int B, int S,
                            int E, void* dx, long long dx_pitch, float* part, float* dw, float* db, cudaStream_t s);
// SSD, head dim 64, state 128, one group: xbc bf16 [T, 64 H + 256] = x | B | C, dt bf16 [T, *] (pitch dt_pitch, H columns),
// A_log / D / dt_bias fp32 [H], H % 8 == 0; y bf16 [T, 64 H].  Scratch: states (and gstates) fp32 [B, ssd_chunks(S), H, 128, 64],
// dec fp32 [B, chunks, H], dA_part / dD_part / dbias_part fp32 [B chunks, H].  The backward writes dxbc bf16 [T, 64 H + 256]
// and ddt (pitch ddt_pitch, H columns: the gradient of the dt input), dA_log, dD, dbias fp32 [H].
int ssd_chunks(int S);
void launch_ssd_fwd(const void* xbc, const void* dt, long long dt_pitch, const float* A_log, const float* D, const float* dt_bias,
                    const int* bounds, int B, int S, int H, float* states, float* dec, void* y, cudaStream_t s);
void launch_ssd_bwd(const void* dy, const void* xbc, const void* dt, long long dt_pitch, const float* A_log, const float* D,
                    const float* dt_bias, const int* bounds, int B, int S, int H, float* states, float* gstates, float* dec,
                    float* dA_part, float* dD_part, float* dbias_part, void* dxbc, void* ddt, long long ddt_pitch, float* dA_log,
                    float* dD, float* dbias, cudaStream_t s);
// Gated RMSNorm y = gamma * rmsnorm(x * silu(z)), bf16 x / y [rows, cols], gamma bf16 [cols], rstd fp32 [rows]; the backward
// writes dx [rows, cols], dz (pitch dzp) and dgamma through wpart fp32 [gated_rmsnorm_parts(rows), cols]
bool gated_rmsnorm_supported(int cols);
int gated_rmsnorm_parts(int rows);
void launch_gated_rmsnorm_fwd(const void* x, const void* z, long long zp, const void* gamma, int rows, int cols, float eps, void* y,
                              float* rstd, cudaStream_t s);
void launch_gated_rmsnorm_bwd(const void* dy, const void* x, const void* z, long long zp, const void* gamma, const float* rstd, int rows,
                              int cols, void* dx, void* dz, long long dzp, float* wpart, void* dgamma, cudaStream_t s);

// ---------------- Whisper's log-mel front end and stem gathers (whisper.cu) --------------------------------------------
// Log-mel: wave int16 [B, 480000], filters fp32 [201, 80] -> out [B, 80, 3000] (bf16 when bf16_out, else fp32).  Scratch:
// logmel fp32 [B, 80, 3000] (may be out itself for fp32 output), part_max fp32 [B, log_mel_partials()].
int log_mel_partials();
void launch_log_mel(const void* wave, const float* filters, int B, bool bf16_out, float* logmel, float* part_max, void* out, cudaStream_t s);
// bf16 features [B, 80, F] -> P1 [B F, 240]; h1 [B F, d] -> P2 [B S, 3 d] (F even, S >= F / 2, d % 8 == 0) and its
// backward dP2 [B S, 3 d] -> dh1 [B F, d]
void launch_mel_patches(const void* features, int B, int F, void* p1, cudaStream_t s);
void launch_frame_patches(const void* h1, int B, int F, int S, int d, void* p2, cudaStream_t s);
void launch_frame_patches_bwd(const void* dp2, int B, int F, int S, int d, void* dh1, cudaStream_t s);

// ---------------- Masked-autoencoder pretraining (mae.cu): shuffle, masked patch embedding, unshuffle, loss, attention --
// noise fp32 [B, N] -> ids_keep int32 [B, keep], ids_restore int32 [B, N]: the stable ascending rank of each patch (N <= 1024)
void launch_mae_shuffle(const float* noise, int B, int N, int keep, int* ids_keep, int* ids_restore, cudaStream_t s);
// image bf16 (NCHW or channels_last) -> patch matrix [T, C p p] of the kept patches in (c, ky, kx) order, image b's kept
// patch j at row b (keep + 1) + 1 + j; class and padding rows zero
void launch_mae_patchify(const void* img, bool channels_last, const int* ids_keep, int B, int C, int H, int W, int p, int keep, int T,
                         void* out, cudaStream_t s);
// GEMM output y [T, D] -> tokens: cls + pos[0] at class rows, y + pos[1 + ids_keep] at patch rows, zero padding rows
void launch_mae_patch_assemble(const void* y, const void* cls, const void* pos, const int* ids_keep, int B, int keep, int D, int T, void* out,
                               cudaStream_t s);
// dy [T, D] -> dpatch [T, D] (dy at patch rows, zero elsewhere) and dcls [D] (fixed-order sum over the class rows)
void launch_mae_patch_embed_bwd(const void* dy, int B, int per, int D, int T, void* dpatch, void* dcls, cudaStream_t s);
// y [Te, E] -> z [Td, E]: row b (N + 1) the class row of image b, row b (N + 1) + 1 + i its kept patch ids_restore[b, i] or
// mask_token, plus pos[row in image]; padding rows zero
void launch_mae_unshuffle(const void* y, const void* mask_token, const void* pos, const int* ids_restore, int B, int N, int keep, int E,
                          int Td, void* z, cudaStream_t s);
// dz [Td, E] -> dy [Te, E] (a gather through ids_keep) and dmask [E] through part fp32 [mae_mask_partials(B), E]
int mae_mask_partials(int B);
void launch_mae_unshuffle_bwd(const void* dz, const int* ids_keep, const int* ids_restore, int B, int N, int keep, int E, int Te, void* dy,
                              float* part, void* dmask, cudaStream_t s);
// Per-image attention at head dim 32: qkv bf16 [T, 3C] (C = 32 heads), image b's rows [b tokens, (b + 1) tokens), tokens <= 256,
// rows past B tokens padding (zero o, lse and dqkv).  o bf16 [T, C], lse fp32 [T, heads].
void launch_image_attention_fwd(const void* qkv, int B, int tokens, int heads, int T, void* o, float* lse, cudaStream_t s);
void launch_image_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, int B, int tokens, int heads, int T,
                                void* dqkv, cudaStream_t s);
// Reconstruction loss on the masked patches: pred bf16 [Td, C p p] (rows as the unshuffled stream), the target read from the
// bf16 image in (ky, kx, c) order, optionally per-patch normalised.  rowloss fp32 [B N] is scratch; loss fp32 [1].  The
// backward writes dpred bf16 [Td, C p p] = 2 (pred - target) / (C p p B (N - keep)) * dloss[0] on masked rows, zero elsewhere.
void launch_mae_loss_fwd(const void* pred, const void* img, bool channels_last, const int* ids_restore, int B, int C, int H, int W, int p,
                         int keep, bool norm_pix, float* rowloss, float* loss, cudaStream_t s);
void launch_mae_loss_bwd(const float* dloss, const void* pred, const void* img, bool channels_last, const int* ids_restore, int B, int C,
                         int H, int W, int p, int keep, bool norm_pix, int Td, void* dpred, cudaStream_t s);

// ---------------- CLIP contrastive loss (clip.cu)---------------------------------------------------
// u bf16 [B, D] = x / ||x|| per row (fp32, one rounding), rnorm fp32 [B] = 1 / ||x||; D % 8 == 0, 16-byte aligned rows
void launch_l2norm_fwd(const void* x, int B, int D, void* u, float* rnorm, cudaStream_t s);
// dx bf16 [B, D] = rnorm (du - u <u, du>) with u = x rnorm in fp32
void launch_l2norm_bwd(const void* du, const void* x, const float* rnorm, int B, int D, void* dx, cudaStream_t s);
// z_img, z_txt fp32 [B, N] (unscaled similarities), logit_scale fp32 [1], labels offset + r (0 <= offset, offset + B <= N):
// dz_* bf16 [B, N] = s (softmax(s z) - onehot) / (2B), loss fp32 [1] = mean of the 2B cross-entropies, dscale fp32 [1] =
// d loss / d logit_scale; row_partials fp32 [4B] is scratch.  Two launches, fixed-order sums.
void launch_contrastive_xent(const float* z_img, const float* z_txt, const float* logit_scale, int B, int N, int offset, void* dz_img,
                             void* dz_txt, float* row_partials, float* loss, float* dscale, cudaStream_t s);

// ---------------- T5 relative position bias (attention.cu) ------------------------
// The segment (causal = false) or causal attention of launch_packed_attention_* / launch_causal_attention_*, multi-head
// at head dim 64, with table fp32 [heads, 257] added to the unscaled scores: score(i, j) = q_i . k_j + table[h, clamp(j - i,
// -128, 128) + 128].  lse is that of the biased scores.  The backward also writes dtable fp32 [heads, 257], the sum of dS
// over the pairs at each clamped distance, through dtable_part fp32 [B, S / 128, heads, 257]; no atomics.
void launch_relative_attention_fwd(const void* qkv, const int* bounds, const float* table, int B, int S, int heads, bool causal,
                                   void* o, float* lse, cudaStream_t s);
void launch_relative_attention_bwd(const void* dout, const void* qkv, const void* o, const float* lse, const int* bounds,
                                   const float* table, int B, int S, int heads, bool causal, float* dsum, float* dtable_part,
                                   void* dqkv, float* dtable, cudaStream_t s);
// table fp32 [heads, 257] = weight[bucket[c], h] (weight [num_buckets, heads], fp32 or bf16; bucket int32 [257]), and its
// backward: dweight[k, h] = the sum of dtable[h, c] over the c with bucket[c] == k, in increasing c
void launch_relative_table_fwd(const void* weight, bool bf16, const int* bucket, int heads, float* table, cudaStream_t s);
void launch_relative_table_bwd(const float* dtable, const int* bucket, int num_buckets, int heads, bool bf16, void* dweight,
                               cudaStream_t s);

// ---------------- cross-attention on wgmma, head dim 64 (cross_attention.cu) ------------------------
// q bf16 [B*Sq, heads*64], kv bf16 [B*Sk, 2*heads*64] (key block | value block), o bf16 [B*Sq, heads*64], lse fp32
// [B, heads, Sq]; q_bounds int32 [B*Sq, 2] (the keys each query sees), kv_bounds int32 [B*Sk, 2] (the queries that see
// each key, the same mask); Sq, Sk multiples of 128.  Backward: dsum fp32 [B, heads, Sq] scratch, dq like q, dkv like kv.
void launch_cross_attention_fwd(const void* q, const void* kv, const int* q_bounds, int B, int Sq, int Sk, int heads, void* o, float* lse,
                                cudaStream_t s);
void launch_cross_attention_bwd(const void* dout, const void* q, const void* kv, const void* o, const float* lse, const int* q_bounds,
                                const int* kv_bounds, int B, int Sq, int Sk, int heads, float* dsum, void* dq, void* dkv, cudaStream_t s);

}  // namespace b200
