// K7 / K8: second-order rules of BatchNorm2d with batch statistics (NCHW) and LayerNorm (last dim).
//   y = gamma * xhat + beta,  xhat = (x - mu) * rstd
//   TF   tc = t_x - mean(t_x); sdot = mean(xhat*tc); dxhat = (tc - xhat*sdot)*rstd
//        t_y = gamma*dxhat + t_gamma*xhat + t_beta
//   BB   gh = a_y*gamma; a_x = rstd*(gh - mean(gh) - xhat*mean(gh*xhat))
//   TB   ght = at_y*gamma + a_y*t_gamma; u = gh - m1 - xhat*m2
//        ut = ght - mean(ght) - dxhat*m2 - xhat*mean(ght*xhat + gh*dxhat)
//        at_x = -rstd^2*sdot*u + rstd*ut ; at_gamma = sum(at_y*xhat + a_y*dxhat) ; at_beta = sum(at_y)
// (SURVEY.md Appendix B; verified against jvp-of-vjp in float64 through oracle/plan_interp.py
// _tf_norm/_bb_norm/_tb_norm.)  BatchNorm statistics couple every pixel of a channel, so each pass is
// a per-channel reduction kernel followed by an apply kernel; LayerNorm rows fit in one warp.
#include <stdlib.h>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "plan.h"
#include "tma.h"

namespace {

// ---------------------------------------------------------------------------------------------------
// BatchNorm.  scratch: double[16][C]; slots 0,1 stats | 2,3 BB | 4,5 TF | 6..9 TB
// ---------------------------------------------------------------------------------------------------
struct BnArgs {
  const void* x;
  int dtx;
  const float* gamma;   // may be null (affine=False) -> 1
  const float* tx;
  const float* tgamma;  // may be null
  const float* tbeta;   // may be null
  const float* g;       // a_y
  const float* gt;      // at_y
  float* ty;
  float* dst;           // a_x or at_x
  float* at_gamma;
  float* at_beta;
  double* S;
  int N, C, HW;
  float eps;
  int beta;
};

enum { BN_STATS = 0, BN_BB = 1, BN_TF = 2, BN_TB = 3 };

struct ChanConst {
  float mean, rstd, m1, m2, mean_t, sdot, gamma, tgamma, tbeta;
};

__device__ __forceinline__ ChanConst chan_const(const BnArgs& A, int c) {
  ChanConst k;
  const double cnt = (double)A.N * A.HW;
  const double mean = A.S[0 * A.C + c] / cnt;
  const double var = A.S[1 * A.C + c] / cnt - mean * mean;
  k.mean = (float)mean;
  k.rstd = (float)rsqrt((var > 0 ? var : 0) + (double)A.eps);
  k.m1 = (float)(A.S[2 * A.C + c] / cnt);
  k.m2 = (float)(A.S[3 * A.C + c] / cnt);
  k.mean_t = (float)(A.S[4 * A.C + c] / cnt);
  k.sdot = (float)(A.S[5 * A.C + c] / cnt);
  k.gamma = A.gamma ? A.gamma[c] : 1.f;
  k.tgamma = A.tgamma ? A.tgamma[c] : 0.f;
  k.tbeta = A.tbeta ? A.tbeta[c] : 0.f;
  return k;
}

// 4 consecutive elements of a base tensor (fp32 / bf16 / fp16) as floats; i must be a multiple of 4, p 16-byte
// (fp32) or 8-byte (16-bit types) aligned
__device__ __forceinline__ void ld_base4(const void* p, int64_t i, int dt, float* o) {
  if (dt == BB_F32) {
    const float4 q = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + i);
    o[0] = q.x; o[1] = q.y; o[2] = q.z; o[3] = q.w;
    return;
  }
  const uint2 r = *reinterpret_cast<const uint2*>(reinterpret_cast<const unsigned short*>(p) + i);
  if (dt == BB_BF16) {
    o[0] = __uint_as_float(r.x << 16); o[1] = __uint_as_float(r.x & 0xffff0000u);
    o[2] = __uint_as_float(r.y << 16); o[3] = __uint_as_float(r.y & 0xffff0000u);
  } else {
    const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
    const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
    o[0] = f0.x; o[1] = f0.y; o[2] = f1.x; o[3] = f1.y;
  }
}
__device__ __forceinline__ void ld_f4(const float* p, int64_t i, float* o) {
  const float4 q = *reinterpret_cast<const float4*>(p + i);
  o[0] = q.x; o[1] = q.y; o[2] = q.z; o[3] = q.w;
}

// per-element bodies shared by the scalar and the 128-bit variants
template <int MODE>
__device__ __forceinline__ void bn_reduce_elem(const ChanConst& k, float x, float tx, float g, float gt, float& s0, float& s1,
                                               float& s2, float& s3) {
  if (MODE == BN_STATS) {
    s0 += x;
    s1 += x * x;
    return;
  }
  const float xh = (x - k.mean) * k.rstd;
  if (MODE == BN_BB) {
    const float gh = g * k.gamma;
    s0 += gh;
    s1 += gh * xh;
  } else if (MODE == BN_TF) {
    s0 += tx;
    s1 += xh * tx;
  } else {
    const float dxh = (tx - k.mean_t - xh * k.sdot) * k.rstd;
    const float gh = g * k.gamma, ght = gt * k.gamma + g * k.tgamma;
    s0 += ght;
    s1 += ght * xh + gh * dxh;
    s2 += gt * xh + g * dxh;
    s3 += gt;
  }
}

template <int MODE>
__device__ __forceinline__ float bn_apply_elem(const ChanConst& k, float mt1, float mt2, float x, float tx, float g, float gt) {
  const float xh = (x - k.mean) * k.rstd;
  if (MODE == BN_TF) {
    const float dxh = (tx - k.mean_t - xh * k.sdot) * k.rstd;
    return k.gamma * dxh + k.tgamma * xh + k.tbeta;
  }
  if (MODE == BN_BB) {
    const float gh = g * k.gamma;
    return k.rstd * (gh - k.m1 - xh * k.m2);
  }
  const float dxh = (tx - k.mean_t - xh * k.sdot) * k.rstd;
  const float gh = g * k.gamma, ght = gt * k.gamma + g * k.tgamma;
  const float u = gh - k.m1 - xh * k.m2;
  const float ut = ght - mt1 - dxh * k.m2 - xh * mt2;
  return -k.rstd * k.rstd * k.sdot * u + k.rstd * ut;
}

// VEC = 4: planes of HW % 4 == 0 elements with 16-byte aligned operands are streamed with 128-bit loads (the scalar
// version kept ~2 MB in flight chip-wide and ran at a third of the HBM rate)
template <int MODE, int VEC>
__global__ void __launch_bounds__(256) bn_reduce_kernel(const __grid_constant__ BnArgs A) {
  __shared__ double red[32];
  const int c = blockIdx.x;
  ChanConst k{};
  if (MODE != BN_STATS) k = chan_const(A, c);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  for (int n = blockIdx.y; n < A.N; n += gridDim.y) {
    const int64_t off = ((int64_t)n * A.C + c) * A.HW;
    if (VEC == 4) {
      for (int q = threadIdx.x * 4; q < A.HW; q += blockDim.x * 4) {
        float x[4], tx[4] = {0.f, 0.f, 0.f, 0.f}, g[4] = {0.f, 0.f, 0.f, 0.f}, gt[4] = {0.f, 0.f, 0.f, 0.f};
        ld_base4(A.x, off + q, A.dtx, x);
        if (MODE == BN_TF || MODE == BN_TB) ld_f4(A.tx, off + q, tx);
        if (MODE == BN_BB || MODE == BN_TB) ld_f4(A.g, off + q, g);
        if (MODE == BN_TB) ld_f4(A.gt, off + q, gt);
#pragma unroll
        for (int e = 0; e < 4; ++e) bn_reduce_elem<MODE>(k, x[e], tx[e], g[e], gt[e], s0, s1, s2, s3);
      }
    } else {
      for (int q = threadIdx.x; q < A.HW; q += blockDim.x) {
        const float x = bb::ldf(A.x, off + q, A.dtx);
        const float tx = (MODE == BN_TF || MODE == BN_TB) ? A.tx[off + q] : 0.f;
        const float g = (MODE == BN_BB || MODE == BN_TB) ? A.g[off + q] : 0.f;
        const float gt = MODE == BN_TB ? A.gt[off + q] : 0.f;
        bn_reduce_elem<MODE>(k, x, tx, g, gt, s0, s1, s2, s3);
      }
    }
  }
  constexpr int slot = MODE == BN_STATS ? 0 : MODE == BN_BB ? 2 : MODE == BN_TF ? 4 : 6;
  double b0 = bb::block_sum<double>((double)s0, red);
  double b1 = bb::block_sum<double>((double)s1, red);
  if (threadIdx.x == 0) {
    atomicAdd(&A.S[(slot + 0) * A.C + c], b0);
    atomicAdd(&A.S[(slot + 1) * A.C + c], b1);
  }
  if (MODE == BN_TB) {
    double b2 = bb::block_sum<double>((double)s2, red);
    double b3 = bb::block_sum<double>((double)s3, red);
    if (threadIdx.x == 0) {
      atomicAdd(&A.S[8 * A.C + c], b2);
      atomicAdd(&A.S[9 * A.C + c], b3);
    }
  }
}

template <int MODE, int VEC>
__global__ void __launch_bounds__(256) bn_apply_kernel(const __grid_constant__ BnArgs A) {
  const int c = blockIdx.x;
  const ChanConst k = chan_const(A, c);
  const double cnt = (double)A.N * A.HW;
  float mt1 = 0.f, mt2 = 0.f;
  if (MODE == BN_TB) {
    mt1 = (float)(A.S[6 * A.C + c] / cnt);
    mt2 = (float)(A.S[7 * A.C + c] / cnt);
    if (blockIdx.y == 0 && threadIdx.x == 0) {
      if (A.at_gamma) A.at_gamma[c] += (float)A.S[8 * A.C + c];  // parameter slices always accumulate
      if (A.at_beta) A.at_beta[c] += (float)A.S[9 * A.C + c];
    }
  }
  float* const out = MODE == BN_TF ? A.ty : A.dst;
  const bool acc = MODE != BN_TF && A.beta;
  for (int n = blockIdx.y; n < A.N; n += gridDim.y) {
    const int64_t off = ((int64_t)n * A.C + c) * A.HW;
    if (VEC == 4) {
      for (int q = threadIdx.x * 4; q < A.HW; q += blockDim.x * 4) {
        float x[4], tx[4] = {0.f, 0.f, 0.f, 0.f}, g[4] = {0.f, 0.f, 0.f, 0.f}, gt[4] = {0.f, 0.f, 0.f, 0.f}, o[4];
        ld_base4(A.x, off + q, A.dtx, x);
        if (MODE == BN_TF || MODE == BN_TB) ld_f4(A.tx, off + q, tx);
        if (MODE == BN_BB || MODE == BN_TB) ld_f4(A.g, off + q, g);
        if (MODE == BN_TB) ld_f4(A.gt, off + q, gt);
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = bn_apply_elem<MODE>(k, mt1, mt2, x[e], tx[e], g[e], gt[e]);
        float4* dst = reinterpret_cast<float4*>(out + off + q);
        float4 w = make_float4(o[0], o[1], o[2], o[3]);
        if (acc) {
          const float4 old = *dst;
          w.x += old.x; w.y += old.y; w.z += old.z; w.w += old.w;
        }
        *dst = w;
      }
    } else {
      for (int q = threadIdx.x; q < A.HW; q += blockDim.x) {
        const float x = bb::ldf(A.x, off + q, A.dtx);
        const float tx = (MODE == BN_TF || MODE == BN_TB) ? A.tx[off + q] : 0.f;
        const float g = (MODE == BN_BB || MODE == BN_TB) ? A.g[off + q] : 0.f;
        const float gt = MODE == BN_TB ? A.gt[off + q] : 0.f;
        const float v = bn_apply_elem<MODE>(k, mt1, mt2, x, tx, g, gt);
        out[off + q] = acc ? out[off + q] + v : v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, statistics recomputed per pass.  Parameter adjoints: each block writes its per-column
// sums to part[block][D] (gamma) and part[gridDim.x + block][D] (beta), and ln_params_finish_kernel adds them in a
// fixed order, so the result does not depend on the order the blocks ran in.
// ---------------------------------------------------------------------------------------------------
struct LnArgs {
  const void* x;
  int dtx;
  const float* gamma;
  const float* tx;
  const float* tgamma;
  const float* tbeta;
  const float* g;
  const float* gt;
  float* ty;
  float* dst;
  float* at_gamma;
  float* at_beta;
  float* part;   // BN_TB: [2][gridDim.x][D] per-block partials of at_gamma, at_beta
  int64_t rows;
  int D;
  float eps;
  int beta;
};

// one row per warp and small blocks: the rows are short (hidden size), so parallelism across rows -- not work per
// warp -- is what keeps the SMs busy (profile: 25 blocks of 8 warps x 4 rows took 0.18 ms per LayerNorm)
constexpr int kLnWarps = 4;
constexpr int kLnRowsPerWarp = 1;

template <int MODE>  // BN_BB / BN_TF / BN_TB reuse the enum
__global__ void __launch_bounds__(kLnWarps * 32) ln_kernel(const __grid_constant__ LnArgs A) {
  extern __shared__ float colsm[];  // [kLnWarps][2][D] for MODE == TB: one slot per warp, added in warp order
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int D = A.D;
  float* colacc = colsm + (int64_t)warp * 2 * D;
  if (MODE == BN_TB) {
    for (int c = lane; c < 2 * D; c += 32) colacc[c] = 0.f;
    __syncwarp();
  }
  const float invD = 1.f / (float)D;
  for (int rr = 0; rr < kLnRowsPerWarp; ++rr) {
    const int64_t row = ((int64_t)blockIdx.x * kLnWarps + warp) * kLnRowsPerWarp + rr;
    if (row >= A.rows) break;
    const int64_t off = row * D;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s += bb::ldf(A.x, off + c, A.dtx);
    const float mean = bb::warp_sum(s) * invD;
    float v = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float d = bb::ldf(A.x, off + c, A.dtx) - mean;
      v += d * d;
    }
    const float rstd = rsqrtf(bb::warp_sum(v) * invD + A.eps);
    auto XH = [&](int c) { return (bb::ldf(A.x, off + c, A.dtx) - mean) * rstd; };
    auto GAM = [&](int c) { return A.gamma ? A.gamma[c] : 1.f; };
    float mean_t = 0.f, sdot = 0.f;
    if (MODE != BN_BB) {
      float a = 0.f;
      for (int c = lane; c < D; c += 32) a += A.tx[off + c];
      mean_t = bb::warp_sum(a) * invD;
      float b = 0.f;
      for (int c = lane; c < D; c += 32) b += XH(c) * (A.tx[off + c] - mean_t);
      sdot = bb::warp_sum(b) * invD;
    }
    if (MODE == BN_TF) {
      for (int c = lane; c < D; c += 32) {
        const float xh = XH(c);
        const float dxh = (A.tx[off + c] - mean_t - xh * sdot) * rstd;
        A.ty[off + c] = GAM(c) * dxh + (A.tgamma ? A.tgamma[c] * xh : 0.f) + (A.tbeta ? A.tbeta[c] : 0.f);
      }
      continue;
    }
    float a1 = 0.f, a2 = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float gh = A.g[off + c] * GAM(c);
      a1 += gh;
      a2 += gh * XH(c);
    }
    const float m1 = bb::warp_sum(a1) * invD, m2 = bb::warp_sum(a2) * invD;
    if (MODE == BN_BB) {
      for (int c = lane; c < D; c += 32) {
        const float xh = XH(c);
        const float val = rstd * (A.g[off + c] * GAM(c) - m1 - xh * m2);
        A.dst[off + c] = A.beta ? A.dst[off + c] + val : val;
      }
      continue;
    }
    float b1 = 0.f, b2 = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float xh = XH(c);
      const float dxh = (A.tx[off + c] - mean_t - xh * sdot) * rstd;
      const float g = A.g[off + c], gt = A.gt[off + c];
      const float gh = g * GAM(c), ght = gt * GAM(c) + (A.tgamma ? g * A.tgamma[c] : 0.f);
      b1 += ght;
      b2 += ght * xh + gh * dxh;
      colacc[c] += gt * xh + g * dxh;
      colacc[D + c] += gt;
    }
    const float mt1 = bb::warp_sum(b1) * invD, mt2 = bb::warp_sum(b2) * invD;
    for (int c = lane; c < D; c += 32) {
      const float xh = XH(c);
      const float dxh = (A.tx[off + c] - mean_t - xh * sdot) * rstd;
      const float g = A.g[off + c], gt = A.gt[off + c];
      const float gh = g * GAM(c), ght = gt * GAM(c) + (A.tgamma ? g * A.tgamma[c] : 0.f);
      const float u = gh - m1 - xh * m2;
      const float ut = ght - mt1 - dxh * m2 - xh * mt2;
      const float val = -rstd * rstd * sdot * u + rstd * ut;
      A.dst[off + c] = A.beta ? A.dst[off + c] + val : val;
    }
  }
  if (MODE == BN_TB) {
    __syncthreads();
    for (int c = threadIdx.x; c < 2 * D; c += blockDim.x) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kLnWarps; ++w) v += colsm[w * 2 * D + c];
      const int half = c >= D;
      A.part[((int64_t)half * gridDim.x + blockIdx.x) * D + (c - half * D)] = v;
    }
  }
}

// ---- wide rows (D % 4 == 0, 256 <= D <= 1024): one 256-thread block walks a few rows; every thread owns four
// consecutive columns, keeps x / t_x / a_y / at_y of the row in registers (each operand is read once, 128-bit), and
// the statistics need three block reductions instead of the warp kernel's eight dependent passes over L1:
//   P1 {sum x, sum t_x}   P2 {sum dx^2, sum dx*dt}   P3 {sum gh, sum gh*xh, sum ght, sum ght*xh + gh*dxh}
// The per-column parameter adjoints accumulate in registers over the block's rows -> one partial per column per block.
__device__ __forceinline__ void block_sum4(float& a, float& b, float& c, float& d, float (*red)[8]) {
  a = bb::warp_sum(a); b = bb::warp_sum(b); c = bb::warp_sum(c); d = bb::warp_sum(d);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();   // previous use of red is over
  if (lane == 0) { red[0][w] = a; red[1][w] = b; red[2][w] = c; red[3][w] = d; }
  __syncthreads();
  a = b = c = d = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { a += red[0][i]; b += red[1][i]; c += red[2][i]; d += red[3][i]; }
}

__device__ __forceinline__ float4 ld_x4(const void* p, int64_t i, int dt) {
  if (dt == BB_F32) return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + i);
  const uint2 r = *reinterpret_cast<const uint2*>(reinterpret_cast<const unsigned short*>(p) + i);
  float4 o;
  if (dt == BB_BF16) {
    o.x = __uint_as_float(r.x << 16); o.y = __uint_as_float(r.x & 0xffff0000u);
    o.z = __uint_as_float(r.y << 16); o.w = __uint_as_float(r.y & 0xffff0000u);
  } else {
    const __half2 h0 = *reinterpret_cast<const __half2*>(&r.x), h1 = *reinterpret_cast<const __half2*>(&r.y);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    o.x = f0.x; o.y = f0.y; o.z = f1.x; o.w = f1.y;
  }
  return o;
}

template <int MODE>
__global__ void __launch_bounds__(256) ln_row_kernel(const __grid_constant__ LnArgs A, int rows_per_block) {
  __shared__ float red[4][8];
  const int D = A.D, c0 = threadIdx.x * 4;
  const bool on = c0 < D;
  const float invD = 1.f / (float)D;
  float gam[4] = {1.f, 1.f, 1.f, 1.f}, tgam[4] = {0.f, 0.f, 0.f, 0.f}, tbet[4] = {0.f, 0.f, 0.f, 0.f};
  if (on) {
    if (A.gamma) { const float4 q = *reinterpret_cast<const float4*>(A.gamma + c0); gam[0] = q.x; gam[1] = q.y; gam[2] = q.z; gam[3] = q.w; }
    if (MODE != BN_BB && A.tgamma) { const float4 q = *reinterpret_cast<const float4*>(A.tgamma + c0); tgam[0] = q.x; tgam[1] = q.y; tgam[2] = q.z; tgam[3] = q.w; }
    if (MODE == BN_TF && A.tbeta) { const float4 q = *reinterpret_cast<const float4*>(A.tbeta + c0); tbet[0] = q.x; tbet[1] = q.y; tbet[2] = q.z; tbet[3] = q.w; }
  }
  float cg[4] = {0.f, 0.f, 0.f, 0.f}, cb[4] = {0.f, 0.f, 0.f, 0.f};   // at_gamma / at_beta partial sums
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  for (int rr = 0; rr < rows_per_block; ++rr) {
    const int64_t row = r0 + rr;
    if (row >= A.rows) break;   // uniform across the block
    const int64_t off = row * D + c0;
    float x[4] = {0.f, 0.f, 0.f, 0.f}, t[4] = {0.f, 0.f, 0.f, 0.f}, g[4] = {0.f, 0.f, 0.f, 0.f}, gt[4] = {0.f, 0.f, 0.f, 0.f};
    if (on) {
      const float4 q = ld_x4(A.x, off, A.dtx);
      x[0] = q.x; x[1] = q.y; x[2] = q.z; x[3] = q.w;
      if (MODE != BN_BB) { const float4 u = *reinterpret_cast<const float4*>(A.tx + off); t[0] = u.x; t[1] = u.y; t[2] = u.z; t[3] = u.w; }
      if (MODE != BN_TF) { const float4 u = *reinterpret_cast<const float4*>(A.g + off); g[0] = u.x; g[1] = u.y; g[2] = u.z; g[3] = u.w; }
      if (MODE == BN_TB) { const float4 u = *reinterpret_cast<const float4*>(A.gt + off); gt[0] = u.x; gt[1] = u.y; gt[2] = u.z; gt[3] = u.w; }
    }
    float s0 = x[0] + x[1] + x[2] + x[3], s1 = t[0] + t[1] + t[2] + t[3], s2 = 0.f, s3 = 0.f;
    block_sum4(s0, s1, s2, s3, red);
    const float mean = s0 * invD, mean_t = s1 * invD;
    float v0 = 0.f, v1 = 0.f;
    if (on) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float d = x[e] - mean;
        v0 += d * d;
        v1 += d * (t[e] - mean_t);
      }
    }
    s2 = s3 = 0.f;
    block_sum4(v0, v1, s2, s3, red);
    const float rstd = rsqrtf(v0 * invD + A.eps);
    const float sdot = rstd * v1 * invD;
    float xh[4], dxh[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      xh[e] = (x[e] - mean) * rstd;
      dxh[e] = (t[e] - mean_t - xh[e] * sdot) * rstd;
    }
    if (MODE == BN_TF) {
      if (on) {
        float4 o;
        o.x = gam[0] * dxh[0] + tgam[0] * xh[0] + tbet[0]; o.y = gam[1] * dxh[1] + tgam[1] * xh[1] + tbet[1];
        o.z = gam[2] * dxh[2] + tgam[2] * xh[2] + tbet[2]; o.w = gam[3] * dxh[3] + tgam[3] * xh[3] + tbet[3];
        *reinterpret_cast<float4*>(A.ty + off) = o;
      }
      continue;
    }
    float gh[4], ght[4], a1 = 0.f, a2 = 0.f, b1 = 0.f, b2 = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      gh[e] = g[e] * gam[e];
      ght[e] = gt[e] * gam[e] + g[e] * tgam[e];
      if (on) {
        a1 += gh[e];
        a2 += gh[e] * xh[e];
        b1 += ght[e];
        b2 += ght[e] * xh[e] + gh[e] * dxh[e];
        cg[e] += gt[e] * xh[e] + g[e] * dxh[e];
        cb[e] += gt[e];
      }
    }
    block_sum4(a1, a2, b1, b2, red);
    const float m1 = a1 * invD, m2 = a2 * invD, mt1 = b1 * invD, mt2 = b2 * invD;
    if (on) {
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float u = gh[e] - m1 - xh[e] * m2;
        if (MODE == BN_BB) {
          o[e] = rstd * u;
        } else {
          const float ut = ght[e] - mt1 - dxh[e] * m2 - xh[e] * mt2;
          o[e] = -rstd * rstd * sdot * u + rstd * ut;
        }
      }
      float4* dst = reinterpret_cast<float4*>(A.dst + off);
      float4 w = make_float4(o[0], o[1], o[2], o[3]);
      if (A.beta) {
        const float4 old = *dst;
        w.x += old.x; w.y += old.y; w.z += old.z; w.w += old.w;
      }
      *dst = w;
    }
  }
  if (MODE == BN_TB && on) {
    *reinterpret_cast<float4*>(A.part + (int64_t)blockIdx.x * D + c0) = make_float4(cg[0], cg[1], cg[2], cg[3]);
    *reinterpret_cast<float4*>(A.part + ((int64_t)gridDim.x + blockIdx.x) * D + c0) = make_float4(cb[0], cb[1], cb[2], cb[3]);
  }
}

// at_gamma[c] += sum_b part[b][c], at_beta[c] += sum_b part[parts + b][c].  Block = 8 lanes x 32 columns: lane l adds
// the partials b = l, l + 8, ... in order, then the lanes are added in lane order.  (One thread per column walking
// all the partials would wait on a memory round trip per partial.)
__global__ void __launch_bounds__(256) ln_params_finish_kernel(const float* __restrict__ part, int parts, int D,
                                                               float* at_gamma, float* at_beta) {
  __shared__ float red[8][32];
  const int cl = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;   // 0 .. 2D-1: gamma columns, then beta columns
  const int half = c >= D ? 1 : 0;
  float v = 0.f;
  if (c < 2 * D) {
    const float* p = part + (int64_t)half * parts * D + (c - half * D);
    for (int b = pl; b < parts; b += 8) v += p[(int64_t)b * D];
  }
  red[pl][cl] = v;
  __syncthreads();
  if (pl == 0 && c < 2 * D) {
    float sum = red[0][cl];
#pragma unroll
    for (int i = 1; i < 8; ++i) sum += red[i][cl];
    float* out = half ? at_beta : at_gamma;
    if (out) out[c - half * D] += sum;
  }
}

}  // namespace

int bb_launch_batchnorm(const bb_node& nd, int pass, cudaStream_t s) {
  BnArgs A{};
  A.x = nd.base[0]; A.dtx = nd.dt[0];
  A.gamma = reinterpret_cast<const float*>(nd.base[1]);
  A.tx = reinterpret_cast<const float*>(nd.t[0]);
  A.tgamma = (nd.active & 2) ? reinterpret_cast<const float*>(nd.t[1]) : nullptr;
  A.tbeta = (nd.active & 4) ? reinterpret_cast<const float*>(nd.t[2]) : nullptr;
  A.g = reinterpret_cast<const float*>(nd.a[3]);
  A.gt = reinterpret_cast<const float*>(nd.at[3]);
  A.ty = reinterpret_cast<float*>(nd.t[3]);
  A.at_gamma = (nd.active & 2) ? reinterpret_cast<float*>(nd.at[1]) : nullptr;
  A.at_beta = (nd.active & 4) ? reinterpret_cast<float*>(nd.at[2]) : nullptr;
  A.S = reinterpret_cast<double*>(nd.aux[0]);
  A.N = (int)nd.dims[0]; A.C = (int)nd.dims[1]; A.HW = (int)nd.dims[2];
  A.eps = (float)nd.f[0];
  A.beta = nd.beta[0];
  int split = (4 * BB_SM_COUNT + A.C - 1) / A.C;
  if (split > A.N) split = A.N;
  if (split < 1) split = 1;
  const dim3 grid(A.C, split);
  const size_t cbytes = sizeof(double) * A.C;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (pass == BB_PASS_BASE_BWD) A.dst = reinterpret_cast<float*>(nd.a[0]);
  if (pass == BB_PASS_TAN_BWD) A.dst = reinterpret_cast<float*>(nd.at[0]);
  const bool vec = A.HW % 4 == 0 && al16(A.tx) && al16(A.g) && al16(A.gt) && al16(A.ty) && al16(A.dst) &&
                   (A.dtx == BB_F32 ? al16(A.x) : (reinterpret_cast<uintptr_t>(A.x) & 7) == 0) && !getenv("BB200_BN_SCALAR");
#define BB_BN_LAUNCH(KERNEL, MODE)                          \
  do {                                                      \
    if (vec) KERNEL<MODE, 4><<<grid, 256, 0, s>>>(A);       \
    else KERNEL<MODE, 1><<<grid, 256, 0, s>>>(A);           \
  } while (0)
  if (pass == BB_PASS_BASE_BWD) {
    BB_CUDA_TRY(cudaMemsetAsync(A.S, 0, 4 * cbytes, s));
    BB_BN_LAUNCH(bn_reduce_kernel, BN_STATS);
    BB_BN_LAUNCH(bn_reduce_kernel, BN_BB);
    BB_BN_LAUNCH(bn_apply_kernel, BN_BB);
    bb_launch_tally += 4;
  } else if (pass == BB_PASS_TAN_FWD) {
    BB_CUDA_TRY(cudaMemsetAsync(A.S + 4 * A.C, 0, 2 * cbytes, s));
    BB_BN_LAUNCH(bn_reduce_kernel, BN_TF);
    BB_BN_LAUNCH(bn_apply_kernel, BN_TF);
    bb_launch_tally += 3;
  } else {
    BB_CUDA_TRY(cudaMemsetAsync(A.S + 6 * A.C, 0, 4 * cbytes, s));
    BB_BN_LAUNCH(bn_reduce_kernel, BN_TB);
    BB_BN_LAUNCH(bn_apply_kernel, BN_TB);
    bb_launch_tally += 3;
  }
#undef BB_BN_LAUNCH
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_launch_layernorm(const bb_node& nd, int pass, cudaStream_t s) {
  LnArgs A{};
  A.x = nd.base[0]; A.dtx = nd.dt[0];
  A.gamma = reinterpret_cast<const float*>(nd.base[1]);
  A.tx = reinterpret_cast<const float*>(nd.t[0]);
  A.tgamma = (nd.active & 2) ? reinterpret_cast<const float*>(nd.t[1]) : nullptr;
  A.tbeta = (nd.active & 4) ? reinterpret_cast<const float*>(nd.t[2]) : nullptr;
  A.g = reinterpret_cast<const float*>(nd.a[3]);
  A.gt = reinterpret_cast<const float*>(nd.at[3]);
  A.ty = reinterpret_cast<float*>(nd.t[3]);
  A.at_gamma = (nd.active & 2) ? reinterpret_cast<float*>(nd.at[1]) : nullptr;
  A.at_beta = (nd.active & 4) ? reinterpret_cast<float*>(nd.at[2]) : nullptr;
  A.rows = nd.dims[0]; A.D = (int)nd.dims[1];
  A.eps = (float)nd.f[0];
  A.beta = nd.beta[0];
  if (A.rows <= 0) return BB_OK;
  // BN_TB: per-block partials of the parameter adjoints, added in a fixed order into at_gamma / at_beta
  auto finish_params = [&](unsigned grid) -> int {
    if (!A.at_gamma && !A.at_beta) return BB_OK;
    ln_params_finish_kernel<<<(unsigned)((2 * A.D + 31) / 32), 256, 0, s>>>(A.part, (int)grid, A.D, A.at_gamma, A.at_beta);
    bb_launch_tally += 1;
    return (int)cudaPeekAtLastError();
  };
  bool owned = false;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool wide = A.D % 4 == 0 && A.D >= 256 && A.D <= 1024 && al16(A.tx) && al16(A.g) && al16(A.gt) && al16(A.ty) &&
                    al16(A.gamma) && al16(A.tgamma) && al16(A.tbeta) && (reinterpret_cast<uintptr_t>(A.x) & 7) == 0 &&
                    al16(pass == BB_PASS_BASE_BWD ? nd.a[0] : nd.at[0]) && (A.dtx != BB_F32 || al16(A.x)) &&
                    !getenv("BB200_LN_WARP");
  if (wide) {
    int rpb = (int)(A.rows / BB_SM_COUNT);
    if (rpb < 1) rpb = 1;
    if (rpb > 8) rpb = 8;
    const unsigned grid = (unsigned)((A.rows + rpb - 1) / rpb);
    if (pass == BB_PASS_BASE_BWD) {
      A.dst = reinterpret_cast<float*>(nd.a[0]);
      ln_row_kernel<BN_BB><<<grid, 256, 0, s>>>(A, rpb);
    } else if (pass == BB_PASS_TAN_FWD) {
      ln_row_kernel<BN_TF><<<grid, 256, 0, s>>>(A, rpb);
    } else {
      A.dst = reinterpret_cast<float*>(nd.at[0]);
      if ((A.part = bb_partials_acquire(sizeof(float) * 2 * grid * A.D, s, &owned)) == nullptr)
        return (int)cudaErrorMemoryAllocation;
      ln_row_kernel<BN_TB><<<grid, 256, 0, s>>>(A, rpb);
    }
    bb_launch_tally += 1;
    int rc = (int)cudaPeekAtLastError();
    if (rc == BB_OK && A.part) rc = finish_params(grid);
    bb_partials_release(A.part, owned, s);
    return rc;
  }
  const int rows_per_block = kLnWarps * kLnRowsPerWarp;
  const unsigned grid = (unsigned)((A.rows + rows_per_block - 1) / rows_per_block);
  if (pass == BB_PASS_BASE_BWD) {
    A.dst = reinterpret_cast<float*>(nd.a[0]);
    ln_kernel<BN_BB><<<grid, kLnWarps * 32, 0, s>>>(A);
  } else if (pass == BB_PASS_TAN_FWD) {
    ln_kernel<BN_TF><<<grid, kLnWarps * 32, 0, s>>>(A);
  } else {
    A.dst = reinterpret_cast<float*>(nd.at[0]);
    const size_t smem = sizeof(float) * kLnWarps * 2 * A.D;
    if (smem > 200 * 1024) return BB_ERR_UNSUPPORTED;
    static BbOncePerDevice configured;
    if (configured.need())
      BB_CUDA_TRY(cudaFuncSetAttribute(ln_kernel<BN_TB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    if ((A.part = bb_partials_acquire(sizeof(float) * 2 * grid * A.D, s, &owned)) == nullptr)
      return (int)cudaErrorMemoryAllocation;
    ln_kernel<BN_TB><<<grid, kLnWarps * 32, smem, s>>>(A);
  }
  bb_launch_tally += 1;
  int rc = (int)cudaPeekAtLastError();
  if (rc == BB_OK && A.part) rc = finish_params(grid);
  bb_partials_release(A.part, owned, s);
  return rc;
}
