// Halo-resident implicit-GEMM 3x3 convolution (conv_halo.cu): 64 -> 64 channels, stride 1, padding 1, activations in the
// PADDED NHWC layout [N][H+2][W+2][64] (bf16, zero border).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// shape this kernel takes (a band of 128 + 2(W+2) + 2 pixel rows must fit one 256-row TMA box)
bool bb_conv_halo_ok(int C, int O, int H, int W);
// out[img][n][y][x] (fp32 NCHW planes; beta: accumulate) = sum_pairs sum_(tap,ch) act[pair][img][y+dy][x+dx][ch] *
// wmat[pair][n][tap][ch] (+ bias[n]);  wmat: bf16 [64][9][64] (bb_pack_convw);  flip = 1: input-gradient form
int bb_conv_halo_run(int N, int H, int W, int npairs, const void* const* act_padded, const void* const* wmat, int flip,
                     float* out, int beta, const float* bias, cudaStream_t s, void* out_bf16_padded = nullptr);
// out_bf16_padded != nullptr: the result is written as bf16 in the padded NHWC layout instead (one contiguous 16 KB
// block per 128-pixel tile, border rows zero) -- directly the next kernel's TMA operand; `out` / `beta` unused
// weight gradient over padded operands: out[o][c][tap] += sum_pairs sum_pixels gy[pair][pixel][o] * x[pair][pixel + d(tap)][c]
// (out: fp32 [O][C][9], accumulated: per-CTA partials added in CTA order)
int bb_wgrad_halo_run(int N, int H, int W, int C, int O, int npairs, const void* const* x_padded, const void* const* gy_padded,
                      float* out, cudaStream_t s);
