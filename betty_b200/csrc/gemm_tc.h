// Argument block of the wgmma dual-product GEMM / implicit-GEMM convolution kernel (gemm_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// How element (row, k) of an operand tile is found in global memory.
enum { TC_STRIDED = 0, TC_PIXROW = 1, TC_PIXK = 2, TC_WDGRAD = 3 };

struct TcSrc {
  const void* p;
  int dt;            // BB_F32 / BB_BF16 (converted to bf16 while staging)
  int mode;
  int64_t rs, cs;    // TC_STRIDED: elem = p[row*rs + k*cs]
  // convolution gathers over a source tensor [NIMG, CH, H, W] and a KH x KW window:
  //   TC_PIXROW  row = pixel (img,y,x) of a GH x GW grid, k = (ch,i,j)
  //   TC_PIXK    row = (ch,i,j),                          k = pixel (img,y,x)
  //     value = src[img, ch, flip ? y+py-i : y-py+i, flip ? x+px-j : x-px+j]  (0 outside the source)
  //   TC_WDGRAD  row = c (< C2), k = (o,i,j): value = p[((o*C2 + c)*KH + i)*KW + j]
  int CH, H, W, KH, KW, GH, GW, py, px, flip, C2;
  int mn_major;      // set by bb_gemm_tc_run: stage this (row-contiguous) operand in the MN-major smem layout
};

struct TcGemmArgs {
  int64_t M, N, K;
  int npairs, ksplit;
  TcSrc a[2];        // A_p: rows = m
  TcSrc b[2];        // B_p: rows = n   (D[m][n] += sum_k A[m][k] * B[n][k])
  float* out;
  int omode;         // 0: out[m*ors + n*ocs]; 1 (plane): m = pixel (img,q), n = channel: out[(img*OCH + n)*OHW + q]
  int64_t ors, ocs;
  int OCH, OHW;
  int beta;
  const float* bias; // indexed by n
  int64_t bias_stride;
  int allow_split, out_dense;
  int lut_k;         // set by bb_gemm_tc_run: entries of the k -> gather-offset tables (0 if unused)
};

inline TcSrc tc_strided(const void* p, int dt, int64_t rs, int64_t cs) {
  TcSrc s{};
  s.p = p; s.dt = dt; s.mode = TC_STRIDED; s.rs = rs; s.cs = cs;
  return s;
}

bool bb_gemm_tc_eligible(int64_t M, int64_t N, int64_t K, int64_t batch);
int bb_gemm_tc_run(const TcGemmArgs& G, cudaStream_t s);
