// wgmma / TMA bf16 GEMM entry points (gemm_wgmma.cu).
#pragma once
#include <cuda_runtime.h>
#include "common.h"

#ifdef __CUDACC__
#define B200_HD __host__ __device__
#else
#define B200_HD
#endif

namespace b200 {

// D[M,N] = epi( sum_k A(m,k) * B(n,k) ).  a_mn=false: A stored [M,K]; a_mn=true: A stored [K,M].
// b_mn=false: B stored [N,K]; b_mn=true: B stored [K,N].  All operands bf16 row-major, D bf16 or fp32.
// epilogue: 0 none, 1 +bias[N], 2 +bias then ReLU, 3 +bias then GELU(erf).
// col_stats (optional): fp32 workspace [2][ceil(M/32)][N]; the epilogue writes, per group of 32 output rows, the column sums
// and sums of squares of the output as stored - BatchNorm statistics of a 1x1 convolution without re-reading its output.
void launch_gemm_bf16(const void* a, const void* b, void* d, const void* bias, int M, int N, int K, bool a_mn, bool b_mn,
                      int epilogue, DType out_dtype, bool accumulate, cudaStream_t stream, float* col_stats = nullptr);
void launch_gemm_nt_bf16(const void* a, const void* b, void* d, const void* bias, int M, int N, int K, int epilogue,
                         DType out_dtype, cudaStream_t stream);
bool gemm_shape_supported(int M, int N, int K, bool a_mn, bool b_mn);
// FP8: D[M,N] (bf16) = epi( a_scale_inv * b_scale_inv * sum_k A[m,k] * B[n,k] ), A stored [M,K] (e4m3, or e5m2 with
// a_e5m2), B stored [N,K] e4m3 - both K-major, the only layout FP8 wgmma takes.  The scale factors are fp32 device scalars
// (no host round trip).  K % 16 == 0 (16-byte row pitch).  Same epilogue codes as launch_gemm_bf16.
void launch_gemm_fp8(const void* a, const void* b, void* d, const void* bias, const float* a_scale_inv, const float* b_scale_inv,
                     int M, int N, int K, bool a_e5m2, int epilogue, cudaStream_t stream);

// Fused LM-head cross-entropy GEMMs: logits x = bf16(hidden[M,K] . weight[V,K]^T + bias) on 128 x 128 tiles, never stored.
// LSE: partial fp32 [ceil(V/128)][M][2] gets each row's (max, sum exp(x - max)) per 128-column tile; target_logit [M] gets
// x[row, targets[row]] for targets in [0, V) (other rows are not written).  K % 8 == 0.
// rows (optional): int32 device count; only the 128-row tiles below it are computed, and the other rows of partial and
// target_logit are not written.
void launch_gemm_lm_lse(const void* hidden, const void* weight, const void* bias, int M, int V, int K, const long long* targets,
                        float* partial, float* target_logit, cudaStream_t stream, const int* rows = nullptr);
// Logit gradient of vocabulary columns [col_offset, col_offset + N): weight and bias point at that slice's first row.
// dlogits bf16 [M, N] = (exp(x - lse[row]) - [col == target]) * gscale / valid, zero for rows whose target is ignore_index
// or outside [0, vocab); gscale and valid are fp32 device scalars (valid <= 0 gives zeros).  rows (optional): as for the LSE
// GEMM; the dlogits rows of skipped tiles are not written.
void launch_gemm_lm_dlogits(const void* hidden, const void* weight, const void* bias, int M, int N, int K, int col_offset, int vocab,
                            const long long* targets, long long ignore_index, const float* lse, const float* gscale,
                            const float* valid, void* dlogits, cudaStream_t stream, const int* rows = nullptr);
// The two backward GEMMs of the row-bounded LM loss, bf16 operands, B MN-major, 128 x 128 tiles; rows: int32 device count.
// a_mn=false (data gradient): A [M, K] K-major, only the 128-row tiles below *rows are computed, D's other rows are not
// written.  a_mn=true (weight gradient): A stored [K, M], B stored [K, N], the k-loop runs over the first *rows rows rounded
// up to 64 (those rows must be finite; zero-padded beyond *rows), and zero rows store zeros.
void launch_gemm_bf16_rows(const void* a, const void* b, void* d, int M, int N, int K, bool a_mn, DType out_dtype, bool accumulate,
                           const int* rows, cudaStream_t stream);

// Grouped (mixture-of-experts) GEMMs on 128 x 128 tiles, bf16 in and out.  A's rows are sorted by expert into segments that
// start at multiples of 128, so each 128-row tile belongs to one expert; rows % 128 == 0, N and K multiples of 64.
// launch_gemm_grouped: D [rows, N] = A [rows, K] . B_e^T per tile, B_e the tile's expert's [N, K] block of B stored
// [E * N, K] (b_mn=false, forward), or D = A . B_e with B_e the [K, N] block of B stored [E * K, N] (b_mn=true, data
// gradient).  tile_expert int32 [rows / 128] on the device: the tile's expert, -1 for unused tiles, whose D rows are not
// written.
void launch_gemm_grouped(const void* a, const void* b, void* d, int rows, int N, int K, int experts, bool b_mn, const int* tile_expert,
                         cudaStream_t stream);
// Weight gradient: D [E, M, N] with D_e = A[s_e]^T . B[s_e] over expert e's rows s_e = [offsets[e], offsets[e+1]) of
// A [rows, M] and B [rows, N]; offsets int32 [E + 1] on the device, multiples of 64.  An expert without rows gets zeros.
void launch_gemm_grouped_wgrad(const void* a, const void* b, void* d, int rows, int M, int N, int experts, const int* offsets,
                               cudaStream_t stream);

// Persistent-tile rasterisation shared by the producer, issuer and epilogue roles (and mirrored on the host for
// tests).  group_m <= 0: m-fastest over the whole problem (default).  group_m > 0: bands of `group_m` m-tiles
// are swept n-major, so the ~132 tiles in flight form a near-square patch and both operands are reused out of L2.
B200_HD inline void gemm_tile_coords(int tile, int num_m, int num_n, int group_m, int* m_blk, int* n_blk) {
  if (group_m <= 0) { *m_blk = tile % num_m; *n_blk = tile / num_m; return; }
  const int per_group = group_m * num_n;
  const int g = tile / per_group;
  const int first_m = g * group_m;
  const int rows = (num_m - first_m) < group_m ? (num_m - first_m) : group_m;   // last band may be short
  const int r = tile - g * per_group;
  *m_blk = first_m + r % rows;
  *n_blk = r / rows;
}
// 0 = auto, 1 = always single-CTA tiles, 2 = always cluster pairs (two CTAs share the B tile through TMA multicast)
void set_gemm_cta_mode(int mode);
// -1 = read B200DDP_GEMM_GROUP_M (default 0 = m-fastest)
void set_gemm_group_m(int group_m);
// -1 = read B200DDP_GEMM_TMA_STORE (default 0); 1 = bf16 outputs leave through shared memory + TMA stores
void set_gemm_tma_store(int on);

}  // namespace b200
