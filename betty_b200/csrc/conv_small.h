// Argument block of the small-channel direct convolution kernels (conv_small.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct SmallConvArgs {
  const void* in[2];  // input feature maps [N, CI, H, W] per operand pair
  int dt_in[2];
  const void* w[2];   // weights in their ORIGINAL [O][C][KH][KW] layout (corr kernel)
  int dt_w[2];
  const void* g[2];   // output-side maps [N, CO, HO, WO] (wgrad kernel)
  int dt_g[2];
  int npairs;
  int mode;           // corr: 0 forward indexing, 1 data-gradient indexing (transposed + flipped)
  float* out;
  float* part;        // wgrad: per-block partials [gridDim.x][CO][CI][KH][KW] (the launcher adds them onto out in order)
  const float* bias;
  int beta;
  int N, CI, H, W, CO, KH, KW, HO, WO, ph, pw;
  int C_orig;         // C of the original weight tensor (row pitch for both modes)
};

bool bb_conv_small_corr_ok(int CI, int CO, int KH, int KW, int npairs);
int bb_conv_small_corr(const SmallConvArgs& A, cudaStream_t s);
bool bb_conv_small_wgrad_ok(int O, int C, int H, int W, int HO, int WO, int KH, int KW);
int bb_conv_small_wgrad(const SmallConvArgs& A, cudaStream_t s);

// second generation (conv_small2.cu): shared-memory staged, warp-per-output-row correlation and channel-blocked weight
// gradient; BB_DECLINED when the geometry does not fit (the callers then use the kernels above)
int bb_conv_small_corr2(const SmallConvArgs& A, cudaStream_t s);
int bb_conv_small_wgrad2(const SmallConvArgs& A, cudaStream_t s);

// The planning of the launchers above without a launch (bb_conv_small_geometry): false when the kernel declines.
// corr2: geo = {grid, units, PX, IMGS, RY, bands, CIC, nstages, VW, groups}
bool bb_conv_small_corr2_geometry(const SmallConvArgs& A, int64_t* geo);
// wgrad2: geo = {grid, OB, tasks, ns, partial floats per block};  first generation: grid and partial floats per block
bool bb_conv_small_wgrad2_geometry(const SmallConvArgs& A, int64_t* geo);
void bb_conv_small_wgrad_geometry(const SmallConvArgs& A, int64_t* geo);
