// TMA-fed tensor-core path of the Conv2d second-order rules (conv_tma.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "plan.h"

// node shape / pass this path handles (stride 1, <= 9 taps, 32..64 channels each way, bf16-autocast graph, scratch set)
bool bb_conv_tma_ok(const bb_node& nd, int pass);
// base-backward pass hook: packs the node's K-loop constants into the plan's persistent arena (no-op otherwise)
int bb_conv_tma_prepare(const bb_node& nd, cudaStream_t s);
// scratch bytes the node's packs need (plan.py mirrors this bound)
size_t bb_conv_tma_scratch(const bb_node& nd);
// TF: writes t_y.  TB: writes at_x and at_W (the bias adjoint stays with the caller).  BB_DECLINED: nothing usable was
// produced, caller takes its other path.
int bb_conv_tma_run(const bb_node& nd, int pass, cudaStream_t s);

// ---- building blocks for fused blocks (convblock2.cu) that bring their own bf16 NHWC operands (64-channel padded) ----
struct BbConvGeo {
  int N, C, H, W, O, KH, KW, HO, WO, ph, pw;
};
// forward-form product on a GH x GW pixel grid: out[img][n][pixel] (fp32 NCHW planes, beta: accumulate) =
//   sum_pairs sum_(tap, ch) src[pair][pixel + disp(tap)][ch] * wmat[pair][n][tap][ch]   (+ bias[n]);
// src: bf16 NHWC [N][SH][SW][64]; wmat: bf16 [ncols][taps][64] (bb_pack_convw); flip = 1: input-gradient form
int bb_conv_tma_corr(const BbConvGeo& g, int npairs, const void* const* src_nhwc, int SH, int SW, const void* const* wmat,
                     int ncols, int GH, int GW, int flip, float* out, int beta, const float* bias, cudaStream_t s,
                     bool padded = false);   // padded: the operands are [N][SH+2][SW+2][64] with a zero border
// weight gradient: out[o][c][tap] += sum_pairs sum_pixels gy[pair][pixel][o] * x[pair][pixel + disp(tap)][c]
// x: bf16 NHWC [N][H][W][64], gy: bf16 NHWC [N][HO][WO][64]; out accumulates (per-CTA partials added in CTA order)
int bb_conv_tma_wgrad(const BbConvGeo& g, int npairs, const void* const* x_nhwc, const void* const* gy_nhwc, float* out,
                      cudaStream_t s, bool padded = false);
