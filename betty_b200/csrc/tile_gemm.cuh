// Tiled fp32-accumulate SIMT GEMM skeleton shared by the Linear (K5) and Conv2d implicit-GEMM (K6)
// second-order kernels.  C[b][m][n] (+)= sum over up to two operand pairs of A_p[b][m][k] * B_p[b][k][n]:
// the "dual" form is what every second-order product needs (e.g. t_y = t_x W^T + x t_W^T), so the
// output tile is produced once instead of round-tripping through HBM between the two products.
//
// Operand access goes through loader functors so the same kernel serves strided matrices (Linear,
// bmm, transposed views of parameter/arena slices) and the three im2col gathers of a convolution.
// This is the exact-fp32 path (fp32 configs must hold rtol 1e-4, BASELINE.json); the bf16 tensor-core
// path lives in gemm_tc.cu.
#pragma once
#include "bb_common.cuh"
#include "plan.h"

namespace bb {

template <int BM, int BN, int BK, int TM, int TN, class LA, class LB, class SC>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
tile_gemm_kernel(const __grid_constant__ LA la, const __grid_constant__ LB lb, const __grid_constant__ SC sc,
                 int64_t M, int64_t N, int64_t K, int npairs, int ksplit,
                 float* __restrict__ part = nullptr) {
  constexpr int THREADS = (BM / TM) * (BN / TN);
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN;
  const int64_t bz = blockIdx.z / ksplit;
  const int split = blockIdx.z % ksplit;
  const int64_t kchunk = ((K + ksplit - 1) / ksplit + BK - 1) / BK * BK;
  const int64_t kbeg = (int64_t)split * kchunk;
  const int64_t kend = (kbeg + kchunk < K) ? kbeg + kchunk : K;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int pair = 0; pair < npairs; ++pair) {
    for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
      // stage A tile (BM x BK) and B tile (BK x BN); thread->element order follows the fast axis in memory
#pragma unroll
      for (int e = tid; e < BM * BK; e += THREADS) {
        int m, k;
        if (la.k_fast) { k = e % BK; m = e / BK; } else { m = e % BM; k = e / BM; }
        const int64_t gm = m0 + m, gk = k0 + k;
        As[k][m] = (gm < M && gk < kend) ? la.load(pair, bz, gm, gk) : 0.f;
      }
#pragma unroll
      for (int e = tid; e < BK * BN; e += THREADS) {
        int k, n;
        if (lb.k_fast) { k = e % BK; n = e / BK; } else { n = e % BN; k = e / BN; }
        const int64_t gk = k0 + k, gn = n0 + n;
        Bs[k][n] = (gk < kend && gn < N) ? lb.load(pair, bz, gk, gn) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[TM], b[TN];
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t gm = m0 + ty * TM + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int64_t gn = n0 + tx * TN + j;
      if (gn >= N) continue;
      if (part != nullptr) part[(((int64_t)split * (gridDim.z / ksplit) + bz) * M + gm) * N + gn] = acc[i][j];
      else sc.store(bz, gm, gn, acc[i][j], split == 0, ksplit > 1);
    }
  }
}

// ---- fast path: fp32 operands with a unit-stride dimension, 128-bit global loads ----------------------
// A_p[m][k] = a[p][m*ars + k*acs] with (AK ? acs == 1 : ars == 1); B_p[k][n] = b[p][k*brs + n*bcs] with
// (BK_ ? brs == 1 : bcs == 1).  The caller guarantees 16-byte alignment of every row start and that the
// unit-stride extent (K for k-fast, M/N otherwise) is a multiple of 4.  Same dual-product semantics and the same
// store functor as tile_gemm_kernel.
struct VecOperands {
  const float* a[2];
  const float* b[2];
  int64_t ars, acs, brs, bcs;   // shared by both pairs
};

template <int BM, int BN, int TM, int TN, bool AK, bool BKF, class SC>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
tile_gemm_vec_kernel(const __grid_constant__ VecOperands op, const __grid_constant__ SC sc, int64_t M, int64_t N,
                     int64_t K, int npairs, int ksplit,
                     float* __restrict__ part = nullptr) {
  constexpr int BK = 16;
  constexpr int THREADS = (BM / TM) * (BN / TN);
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN;
  const int split = blockIdx.z % ksplit;
  const int64_t kchunk = ((K + ksplit - 1) / ksplit + BK - 1) / BK * BK;
  const int64_t kbeg = (int64_t)split * kchunk;
  const int64_t kend = (kbeg + kchunk < K) ? kbeg + kchunk : K;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int pair = 0; pair < npairs; ++pair) {
    const float* __restrict__ A = op.a[pair];
    const float* __restrict__ B = op.b[pair];
    for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
      // ---- A tile: BM x 16 ----
      for (int f = tid; f < BM * BK / 4; f += THREADS) {
        if (AK) {   // 4 consecutive k of one row
          const int m = f / (BK / 4), k4 = (f % (BK / 4)) * 4;
          const int64_t gm = m0 + m, gk = k0 + k4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (gm < M && gk < kend) v = *reinterpret_cast<const float4*>(A + gm * op.ars + gk);
          As[k4 + 0][m] = v.x; As[k4 + 1][m] = v.y; As[k4 + 2][m] = v.z; As[k4 + 3][m] = v.w;
        } else {    // 4 consecutive m of one k
          const int k = f / (BM / 4), m4 = (f % (BM / 4)) * 4;
          const int64_t gm = m0 + m4, gk = k0 + k;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (gm < M && gk < kend) v = *reinterpret_cast<const float4*>(A + gk * op.acs + gm);
          *reinterpret_cast<float4*>(&As[k][m4]) = v;
        }
      }
      // ---- B tile: 16 x BN ----
      for (int f = tid; f < BN * BK / 4; f += THREADS) {
        if (BKF) {  // 4 consecutive k of one column n
          const int n = f / (BK / 4), k4 = (f % (BK / 4)) * 4;
          const int64_t gn = n0 + n, gk = k0 + k4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (gn < N && gk < kend) v = *reinterpret_cast<const float4*>(B + gn * op.bcs + gk);
          Bs[k4 + 0][n] = v.x; Bs[k4 + 1][n] = v.y; Bs[k4 + 2][n] = v.z; Bs[k4 + 3][n] = v.w;
        } else {    // 4 consecutive n of one k
          const int k = f / (BN / 4), n4 = (f % (BN / 4)) * 4;
          const int64_t gn = n0 + n4, gk = k0 + k;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (gn < N && gk < kend) v = *reinterpret_cast<const float4*>(B + gk * op.brs + gn);
          *reinterpret_cast<float4*>(&Bs[k][n4]) = v;
        }
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[TM], b[TN];
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t gm = m0 + ty * TM + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int64_t gn = n0 + tx * TN + j;
      if (gn >= N) continue;
      if (part != nullptr) part[((int64_t)split * M + gm) * N + gn] = acc[i][j];
      else sc.store(0, gm, gn, acc[i][j], split == 0, ksplit > 1);
    }
  }
}

// ---- strided operands --------------------------------------------------------------------------
struct StridedLoad {
  const void* p[2];
  int dt[2];
  int64_t rs[2], cs[2], bs[2];  // row / col / batch strides (elements)
  int k_fast;                   // 1 if consecutive k are adjacent in memory for this operand
  __device__ __forceinline__ float load(int pair, int64_t b, int64_t r, int64_t c) const {
    return ldf(p[pair], b * bs[pair] + r * rs[pair] + c * cs[pair], dt[pair]);
  }
};

// Split-K partials part[split][b][m][n] (written by the kernels above when `part` is set) summed in split order, then
// stored through the caller's store once (bias, beta): the result does not depend on the order the CTAs ran in.
template <class SC>
__global__ void __launch_bounds__(256) splitk_reduce_kernel(SC sc, const float* __restrict__ part, int64_t M, int64_t N,
                                                            int64_t batch, int ksplit) {
  const int64_t mn = M * N, total = mn * batch;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int sp = 0; sp < ksplit; ++sp) v += part[sp * total + t];
    const int64_t b = t / mn, r = t - b * mn, m = r / N;
    sc.store(b, m, r - m * N, v, true, false);
  }
}

template <class SC>
inline int splitk_reduce(const SC& sc, const float* part, int64_t M, int64_t N, int64_t batch, int ksplit, cudaStream_t s) {
  if (part == nullptr || ksplit <= 1) return 0;
  int64_t blocks = (M * N * batch + 255) / 256;
  if (blocks > 4096) blocks = 4096;
  splitk_reduce_kernel<SC><<<(unsigned)blocks, 256, 0, s>>>(sc, part, M, N, batch, ksplit);
  bb_launch_tally += 1;
  const cudaError_t e = cudaPeekAtLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

struct StridedStore {
  float* p;
  int64_t rs, cs, bs;
  int beta;            // 1: accumulate into existing contents
  const float* bias;   // optional, indexed by column
  int64_t bias_stride;
  __device__ __forceinline__ void store(int64_t b, int64_t m, int64_t n, float v, bool first_split, bool atomic) const {
    float* q = p + b * bs + m * rs + n * cs;
    if (bias != nullptr && first_split) v += bias[n * bias_stride];
    if (atomic) atomicAdd(q, v);
    else *q = beta ? *q + v : v;
  }
};

}  // namespace bb
