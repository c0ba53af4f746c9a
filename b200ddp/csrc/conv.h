// wgmma convolution entry points (conv_wgmma.cu, conv_wgrad_wgmma.cu) for channels_last bf16 activations.
// They replace the cuDNN calls behind the model's forward / backward (reference hot path: the reference ddp.py:221,231).
#pragma once
#include <cuda_runtime.h>
#include "common.h"

namespace b200 {

// How an output tile of <= 128 accumulator rows is cut out of the N x H x W output grid.
//   mode 0 "flat" : 1x1 convolutions - the NHWC tensor is the row-major [N*H*W, C] matrix, a tile is 128 consecutive pixels.
//   mode 1 "patch": filter taps re-fetch their (shifted) input patch: tile = BI images x BH rows x W columns, dense.
//   mode 2 "halo" : the (BH+2) x (W+2) input halo is fetched ONCE per 64-channel block and the nine taps are nine
//                   shared-memory descriptors into it (row offsets of the K-major, 128B-swizzled tile); accumulator rows
//                   enumerate BH x (W+2) positions, the two extra columns per row are discarded by the epilogue.
struct ConvTilePlan {
  int mode = 0;
  int BH = 0, BI = 0, tiles_h = 0;
  int Wp = 0;            // halo row pitch (W + 2)
  int num_m_tiles = 0;
  int dense_rows = 0;    // output rows stored per tile
  int acc_rows = 0;      // accumulator rows in use (<= 128)
  int a_rows = 0;        // shared-memory rows one A load delivers
};
// want_mode: -1 auto, else force (returns false if the geometry does not fit the mode)
bool conv_tile_plan(int N, int H, int W, int R, int S, int want_mode, ConvTilePlan* plan);

struct ConvLaunchCfg {
  int mode = -1;             // -1 auto
  int block_n = 0;           // 0 auto; 64 / 128; 256 runs as two 128-wide n-tiles (a wider accumulator does not fit in registers)
  int kc = 0;                // 0 auto; 64-deep k chunks per pipeline stage (flat / patch tilings)
  void* debug_counters = nullptr;   // device int64[16]: cycle breakdown of CTA 0's producer / issuer / epilogue (diagnostics)
  int set_base_offset = 0;   // halo mode experiment knob: 1 = fill the A descriptors' base-offset field with the 128-byte row phase of
                             // their start address (default 0: the swizzle phase is taken from the absolute address)
};

// Forward (dgrad = false):  y[N,H,W,Cout] = conv(x[N,H,W,Cin], w[Cout,R,S,Cin]),  stride 1, padding (R-1)/2.
// Data gradient (dgrad = true): dx[N,H,W,Cin] = conv^T(dy[N,H,W,Cout], w[Cout,R,S,Cin]) - same kernel, mirrored taps, filter read MN-major.
// `a` is x (or dy), `d` the output; R = S in {1, 3}.  col_stats (forward only, optional): [2][conv_stat_groups(...)][Cout] fp32 partial
// column sums / sums of squares of the stored output (BatchNorm statistics from the epilogue).
// Data-gradient epilogue fusion (optional): `addend` [N,H,W,Cin] is added to dx (the shortcut gradient of a residual block - no
// separate add kernel); and if `bn_x` is given, dx is the output gradient of the BatchNorm(+ReLU) whose input was bn_x: the
// epilogue then also writes per-CTA partial sums S1 = sum dx*m, S2 = sum dx*m*xhat into col_stats ([2][conv_stat_groups][Cin]),
// which replaces that BatchNorm's backward reduction pass over dx and bn_x.
struct ConvBwdFusion {
  const void* addend = nullptr;
  const void* bn_x = nullptr;
  const void* bn_mask = nullptr;     // [N*H*W, Cin / 8] bit mask (ReLU) or nullptr
  const float* bn_mean = nullptr;
  const float* bn_rstd = nullptr;
};
void launch_conv_tap_gemm(const void* a, const void* w, void* d, int N, int H, int W, int Cin, int Cout, int R, int S, bool dgrad,
                          const ConvLaunchCfg& cfg, float* col_stats, cudaStream_t stream, const ConvBwdFusion* fuse = nullptr);


// rows G of the column-statistics workspace [2][G][Cout] the forward launch with this configuration will write
int conv_stat_groups(int N, int H, int W, int Cin, int Cout, int R, int S, const ConvLaunchCfg& cfg);

// Weight gradient: dw[Cout,R,S,Cin] = sum over pixels of dy[n,h,w,co] * x[n,h+r-pad,w+s-pad,ci]  (stride 1).
// Split over the pixel dimension across all SMs; fp32 partials in `workspace`, reduced by a second (fully parallel,
// fixed-order -> deterministic) kernel that writes bf16.  workspace_floats(...) sizes the scratch.
struct WgradCfg {
  int split = 0;             // 0 auto
  int tile_m = 0, tile_n = 0;   // 0 auto: output tile (Cout x Cin-per-tap) handled by one CTA
};
size_t conv_wgrad_workspace_floats(int N, int H, int W, int Cin, int Cout, int R, int S, const WgradCfg& cfg);
void launch_conv_wgrad(const void* dy, const void* x, void* dw, int N, int H, int W, int Cin, int Cout, int R, int S,
                       const WgradCfg& cfg, float* workspace, cudaStream_t stream);


// ---- the strided 7x7 stem (3 input channels, stride 2, padding 3) as a 4-tap implicit GEMM -------------------------------
// The [N,H,W,3] input is repacked once per step into a zero-bordered image of ROW PAIRS, xp[N, H/2+3, W+8, 8]: "pixel"
// (i, wp) holds padded rows 2i and 2i+1 (4 channels each, the 4th zero) of padded column wp; image pixel (h,w) sits at padded
// (h+3, w+4).  A 16-byte pixel makes the 8-pixel window that starts at padded column 2*ow a 128-byte row whose start advances
// by 32 bytes per output column - a legal TMA stride - so "im2col" is a tensor map with OVERLAPPING rows
// {64 elements, Wo windows (stride 32 B), H/2+3 pair rows, N} and never exists in memory.  Output row oh reads pair rows
// oh .. oh+3: four taps of 64 reduction elements each (K = 256 for 147 real filter taps; the rest meets zero weights).
struct StemGeom { int Ho, Wo, Hp2, Wp; };
inline bool stem_geom(int H, int W, StemGeom* g) {
  if (H < 8 || W < 32 || H % 2 != 0 || W % 2 != 0) return false;
  g->Ho = H / 2; g->Wo = W / 2; g->Hp2 = H / 2 + 3; g->Wp = W + 8;
  return g->Wo <= 128 && g->Wo % 16 == 0;
}
constexpr int kStemTaps = 4;
constexpr int kStemK = kStemTaps * 64;      // packed filter row: 4 pair rows x 8 window pixels x (2 rows x 4 channels)
void launch_stem_pack_input(const void* x_nhwc3, void* xp, int N, int H, int W, cudaStream_t stream);
void launch_stem_pack_weight(const void* w_krsc3, void* w2, int Cout, cudaStream_t stream);            // [Cout,7,7,3] -> [Cout,4,8,8]
// packed weight gradient -> [Cout,7,7,3]; transposed: dw2 is [kStemK, Cout] (the dedicated kernel) instead of [Cout, kStemK]
void launch_stem_unpack_wgrad(const void* dw2, void* dw_krsc3, int Cout, bool transposed, cudaStream_t stream);
// y[N,Ho,Wo,Cout] = conv7x7s2(x) from the packed operands; col_stats optional [2][stem_stat_groups][Cout] (BatchNorm statistics).
// resident_filter: the 32 KB packed filter is loaded into shared memory once per CTA instead of once per tile.
int stem_stat_groups(int N, int H, int W);
void launch_stem_conv_fprop(const void* xp, const void* w2, void* y, int N, int H, int W, int Cout, float* col_stats, bool resident_filter,
                            void* debug_counters, cudaStream_t stream);
// Weight gradient over the same windows.  variant 0: the dedicated kernel (window elements on the accumulator rows, two taps per
// MMA, dw2 comes out transposed [kStemK, Cout]); variant 1: the generic split-pixel kernel with four taps (dw2 [Cout, kStemK]).
size_t stem_wgrad_workspace_floats(int N, int H, int W, int Cout, int variant);
void launch_stem_conv_wgrad(const void* dy, const void* xp, void* dw2, int N, int H, int W, int Cout, int variant, float* workspace,
                            cudaStream_t stream);

}  // namespace b200
