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
