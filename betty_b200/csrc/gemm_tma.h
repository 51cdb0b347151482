// TMA-fed wgmma dual-product GEMM / 3x3-style convolution (gemm_tma.cu, conv_tma.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define BB_DECLINED 1   // launcher did not take the job (nothing was launched): caller uses its other path

// An operand as a strided matrix view: element (row, k) = p[row*rs + k*cs]; rows index m (A) or n (B).
struct TmaView {
  const void* p;
  int dt;
  int64_t rs, cs;
  int64_t bs = 0;   // batch stride (elements); ignored when batch == 1
};

// D[m][n] (beta)= sum_p sum_k A_p[m][k] * B_p[n][k]  (+ bias[n]),  out[m*ors + n*ocs].
// Operands that are not already TMA-addressable bf16 are packed into bb_scratch first.
// batch > 1: `batch` independent products (operand / output batch strides TmaView::bs / obs), one grid.z slice each.
// plane_ohw > 0: the rows are pixels (img, q) of planes with plane_ohw pixels and the output is NCHW,
// out[(img*N + n)*plane_ohw + q] (ors / ocs unused).  min_n: smallest N accepted (64 for Linear layers).
int bb_gemm_tma_run(int64_t M, int64_t N, int64_t K, int npairs, const TmaView* A, const TmaView* B, float* out,
                    int64_t ors, int64_t ocs, int beta, const float* bias, int64_t bias_stride, bool out_dense,
                    cudaStream_t s, int plane_ohw = 0, int min_n = 64, int64_t batch = 1, int64_t obs = 0);

// Pack, in as few launches as possible (four operands per launch), every listed view that is not TMA-addressable as
// it stands; the bb_gemm_tma_run calls of the same node then find the packs in the per-node cache.  rows / k as in
// bb_gemm_tma_run (A: rows = M, B: rows = N).
struct TmaPackReq {
  TmaView v;
  int64_t rows, k;
};
int bb_gemm_tma_prepack(const TmaPackReq* reqs, int n, int64_t batch, cudaStream_t s);

enum { TMA_KMAJ = 0, TMA_MNMAJ = 1, TMA_CONV = 2 };

struct alignas(64) TmaGemmArgs {
  CUtensorMap a[2], b[2];
  int a_kind[2], b_kind[2];
  int64_t M, N, K;
  int npairs, ksplit;
  int stages;                  // ring depth (2..8): deep when the grid leaves SMs idle, 3-4 with two CTAs per SM otherwise
  uint32_t a_bytes, b_bytes;   // bytes one stage receives per operand (mbarrier expect_tx)
  // TMA_CONV: the M tile is a (Wb x Hb) box of pixels of one image, the k-blocks walk (tap, 64-channel block)
  int Wb, Hb, tiles_per_img, KW, ph, pw, flip, cblocks;
  float* out;
  int omode;                   // 0: out[m*ors + n*ocs]; 1 (plane, TMA_CONV tiles): out[(img*OCH + n)*OHW + pixel];
                               // 2 (plane, flat rows): m = img*OHW + q
  int64_t ors, ocs, obs;
  int OCH, OHW;
  int beta;
  const float* bias;
  int64_t bias_stride;
};

int bb_gemm_tma_launch(TmaGemmArgs& G, int bn, int64_t mtiles, cudaStream_t s, int batch = 1);

// ---- packs (gemm_tma.cu) ----
// dst[o][i] = bf16(src[o*os + i*is]), o < outer, i < inner; dst pitch dp (>= inner, multiple of 8), tail zero-filled
int bb_pack2d(const void* src, int dt, int64_t os, int64_t is, int64_t outer, int64_t inner, void* dst, int64_t dp,
              cudaStream_t s);
// NCHW (contiguous, dt) -> NHWC bf16 with Cp = roundup(C, 64) channels (zero padded)
int bb_pack_nhwc(const void* src, int dt, int N, int C, int HW, void* dst, int Cp, cudaStream_t s);
// conv weights W[o][c][i][j] (dt) -> dst[r][tap][q] bf16, q padded to Qp:
//   transpose = 0: r = o, q = c (forward operand);  transpose = 1: r = c, q = o (input-gradient operand)
int bb_pack_convw(const void* src, int dt, int O, int C, int taps, int transpose, void* dst, int Qp, cudaStream_t s);
// im2col of an NCHW tensor: dst[pixel (img,y,x) of the HO x WO grid][k = (c,i,j)] bf16, pitch kp (>= C*KH*KW, mult of 8)
struct Im2colGeom {
  int N, C, H, W, KH, KW, HO, WO, sh, sw, ph, pw, dh, dw;
};
int bb_pack_im2col(const void* src, int dt, const Im2colGeom& g, void* dst, int kp, cudaStream_t s);
