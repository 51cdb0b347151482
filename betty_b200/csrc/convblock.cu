// Fused second-order rules of a DATA-INPUT convolution block
//
//     x (data) --conv3x3(W,b)--> y --BatchNorm2d(batch stats; gamma,beta)--> z --[ReLU]--> MaxPool2d(2)--> q
//
// (reference examples/implicit_maml/models.py:9-24; the first block of the 4-conv backbone is 2/3 of the K-loop's
// algorithmic bytes, SURVEY.md 8d).  Because x is data, the tangent t_y = X t_W + t_b (X = im2col(x), P x CKK) is
// LINEAR in the direction, so every full-resolution reduction of the BatchNorm rules collapses to a product with a
// per-call constant:
//
//     s[k]    = sum_p X[p,k]                 sx[o]   = sum_p xhat[p,o]
//     G[o,k]  = sum_p xhat[p,o] X[p,k]       S2[k,l] = sum_p X[p,k] X[p,l]
//
//   TF   mean_t = (t_W.s)/P + t_b            sdot = (t_W.G + t_b sx - mean_t sx)/P
//        t_q[w,o] = mask * (gamma*rstd*(t_y[p*] + ... ) ...)   only at the arg-max pixel p*(w,o) of each window
//   TB   at_y = sparse + d0 + xhat d1 + t_y d2   (norm.cu's rule expanded; sparse lives on the arg-max pixels)
//        at_W = sum_p at_y X = rstd gamma GW + (rstd t_gamma - rstd^2 sdot gamma) Gd + d0 s + d1 G + d2 (t_W S2 + t_b s)
//        with GW[o,k] = sum_w mask at_q[w,o] X[p*(w,o),k]  -- the only per-iteration pass, at POOLED resolution.
//
// So neither y-sized tangents nor y-sized adjoints exist: per iteration the block reads x and streams pooled-size
// arrays (a quarter of y).  All arithmetic fp32 (x / y / q are read in the dtype the forward recorded).
// Verified against the composition of the three member rules (oracle/plan_interp.py) and autograd's double backward.
#include <algorithm>
#include <cuda_bf16.h>
#include <stdlib.h>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "plan.h"

namespace {

constexpr int KP = 28;          // padded CKK (<= 27 used)
constexpr int NT = 256;         // threads per CTA
constexpr int MAXO = 64;
constexpr int NSUM = 4;         // per-channel scalar sums carried next to GW

// pooled arrays (xhat*, dxhat*, mask a_q) are fp32 for fp32 graphs and bf16 for reduced-precision graphs (they are
// streamed once per iteration: 13 -> 7 bytes per pooled element)
template <typename PT> __device__ __forceinline__ float ldp(const PT* p, int64_t i);
template <> __device__ __forceinline__ float ldp<float>(const float* p, int64_t i) { return p[i]; }
template <> __device__ __forceinline__ float ldp<__nv_bfloat16>(const __nv_bfloat16* p, int64_t i) { return __bfloat162float(p[i]); }
template <typename PT> __device__ __forceinline__ void stp(PT* p, int64_t i, float v);
template <> __device__ __forceinline__ void stp<float>(float* p, int64_t i, float v) { p[i] = v; }
template <> __device__ __forceinline__ void stp<__nv_bfloat16>(__nv_bfloat16* p, int64_t i, float v) { p[i] = __float2bfloat16(v); }

struct CbGeom {
  int N, C, H, W, O, HO, WO, ph, pw, HP, WP, relu;
  int ps;         // bytes per pooled-array element (4 or 2)
  int R;          // window rows per tile
  int tiles_per_img, ntiles;
  int xrows, xpitch;   // input tile rows / pitch in shared memory
  int wpitch;          // pooled tile pitch in shared memory
};

// workspace layout (floats unless noted); offsets in bytes, filled by cb_layout()
struct CbWs {
  double* dsum;     // [2*O] sum y, sum y^2  + [KP + O + O*KP + KP*KP] double accumulators of the Gram pass
  float* mean;      // [O]
  float* rstd;      // [O]
  float* s;         // [KP]
  float* sx;        // [O]
  float* G;         // [O*KP]
  float* S2;        // [KP*KP]
  float* Gd;        // [O*KP]   gather-wgrad of the masked base adjoint
  float* Sa;        // [O]      sum mask a_q
  float* Saxh;      // [O]      sum mask a_q xhat_sel
  float* mean_t;    // [O]      written by the tangent-forward pass
  float* sdot;      // [O]
  float* part;      // [grid][O][KP + NSUM] per-CTA partial sums of the reduce kernels
  unsigned char* sel;   // [N*HP*WP*O] NHWC: code (dy*2+dx) | mask << 2
  void* xh;         // [N*HP*WP*O] NHWC xhat at the arg-max pixel          (fp32 or bf16, CbGeom::ps)
  void* dxh;        // [N*HP*WP*O] NHWC dxhat at the arg-max pixel (per iteration)
  void* aqm;        // [N*HP*WP*O] NHWC mask * a_q
  void* pfrag;      // [ceil(N*HP*WP/16)][8][32] uint4: patch fragments of the tensor-core path (O == 64 only)
  void* pfragT;     // same size: the transposed fragments (reduce kernel)
  size_t bytes;
};

constexpr int GRID_MAX = 4 * BB_SM_COUNT;

__host__ __device__ inline size_t up(size_t x) { return (x + 255) & ~(size_t)255; }

CbWs cb_layout(void* base, const CbGeom& g) {
  CbWs w{};
  size_t at = 0;
  uint8_t* b = reinterpret_cast<uint8_t*>(base);
  auto take = [&](size_t bytes) { size_t o = at; at = up(at + bytes); return b ? b + o : nullptr; };
  const size_t O = g.O, pooled = (size_t)g.N * g.HP * g.WP * g.O;
  w.dsum = reinterpret_cast<double*>(take(sizeof(double) * (2 * O + KP + O + O * KP + KP * KP)));
  w.mean = reinterpret_cast<float*>(take(4 * O));
  w.rstd = reinterpret_cast<float*>(take(4 * O));
  w.s = reinterpret_cast<float*>(take(4 * KP));
  w.sx = reinterpret_cast<float*>(take(4 * O));
  w.G = reinterpret_cast<float*>(take(4 * O * KP));
  w.S2 = reinterpret_cast<float*>(take(4 * KP * KP));
  w.Gd = reinterpret_cast<float*>(take(4 * O * KP));
  w.Sa = reinterpret_cast<float*>(take(4 * O));
  w.Saxh = reinterpret_cast<float*>(take(4 * O));
  w.mean_t = reinterpret_cast<float*>(take(4 * O));
  w.sdot = reinterpret_cast<float*>(take(4 * O));
  w.part = reinterpret_cast<float*>(take(4 * (size_t)GRID_MAX * O * (KP + NSUM)));
  w.sel = reinterpret_cast<unsigned char*>(take(pooled));
  const size_t ps = g.ps == 2 ? 2 : 4;
  w.xh = take(ps * pooled);
  w.dxh = take(ps * pooled);
  w.aqm = take(ps * pooled);
  if (g.O == 64) {
    const size_t nmt = ((size_t)g.N * g.HP * g.WP + 15) / 16;
    w.pfrag = take(nmt * 8 * 32 * 16);
    w.pfragT = take(nmt * 8 * 32 * 16);
  }
  w.bytes = at;
  return w;
}

struct CbArgs {
  CbGeom g;
  CbWs w;
  const void* x; int dtx;
  const void* y; int dty;
  const void* q; int dtq;
  const int64_t* idx;
  const float* gamma;
  float eps;
  // parameter tangents (direction arena slices) and adjoint-tangent slices (H.d arena); null when absent
  const float *t_W, *t_b, *t_gamma, *t_beta;
  float *at_W, *at_b, *at_gamma, *at_beta;
  // pooled output buffers of the plan (fp32, NCHW)
  float* t_q;
  __nv_bfloat16* tq_nhwc;     // when the consumer is a fused block: t_q as bf16 NHWC (its TMA operand), t_q unused
  const float* a_q;
  const float* at_q;
  // when the consumer is a fused inner block it hands a_q / at_q over as bf16 padded NHWC [N][HP+2][WP+2][64]
  const __nv_bfloat16* aq_nhwc;
  const __nv_bfloat16* atq_nhwc;
  int nparts;     // CTAs that wrote partials
};

CbGeom make_geom(const bb_node& nd) {
  CbGeom g{};
  g.N = (int)nd.dims[0]; g.C = (int)nd.dims[1]; g.H = (int)nd.dims[2]; g.W = (int)nd.dims[3]; g.O = (int)nd.dims[4];
  g.HO = (int)nd.dims[7]; g.WO = (int)nd.dims[8]; g.ph = (int)nd.dims[11]; g.pw = (int)nd.dims[12];
  g.HP = (int)nd.dims[13]; g.WP = (int)nd.dims[14]; g.relu = (int)nd.dims[15];
  g.ps = (nd.kind & 1) ? 2 : 4;
  int R = 96 / (g.WP > 0 ? g.WP : 1);     // ~96 windows x O channels per tile (two pooled rows of the 84x84 layer)
  if (R < 1) R = 1;
  if (R > g.HP) R = g.HP;
  g.R = R;
  g.tiles_per_img = (g.HP + R - 1) / R;
  g.ntiles = g.N * g.tiles_per_img;
  g.xrows = 2 * R + 2;
  g.xpitch = (g.WO + 2) | 1;              // odd pitch: the four candidate pixels of a window fall into distinct banks
  g.wpitch = (R * g.WP) | 1;
  return g;
}

// ---------------------------------------------------------------------------------------------------------------
// base statistics of y (once per call)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cb_stats_kernel(const CbArgs A) {
  // grid (O, chunks): each block sums a slice of the channel's N*HO*WO values
  __shared__ double red[32];
  const int o = blockIdx.x, HW = A.g.HO * A.g.WO;
  const int64_t per = (int64_t)A.g.N * HW;
  double s0 = 0, s1 = 0;
  for (int64_t i = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.y * blockDim.x) {
    const int64_t n = i / HW, r = i - n * HW;
    const float v = bb::ldf(A.y, (n * A.g.O + o) * HW + r, A.dty);
    s0 += v;
    s1 += (double)v * v;
  }
  s0 = bb::block_sum<double>(s0, red);
  s1 = bb::block_sum<double>(s1, red);
  if (threadIdx.x == 0) {
    atomicAdd(&A.w.dsum[o], s0);
    atomicAdd(&A.w.dsum[A.g.O + o], s1);
  }
}

// bf16 y with HO*WO % 8 == 0: a warp per (image, channel) plane, 16-byte loads (the generic kernel above pays a 64-bit
// division per element: 1.08 ms for 722 MB; this one streams)
__global__ void __launch_bounds__(256) cb_stats_bf16_kernel(const CbArgs A) {
  const int HW = A.g.HO * A.g.WO, lane = threadIdx.x & 31;
  const int64_t planes = (int64_t)A.g.N * A.g.O;
  const int64_t warp0 = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  const __nv_bfloat16* y = reinterpret_cast<const __nv_bfloat16*>(A.y);
  for (int64_t pl = warp0; pl < planes; pl += nwarps) {
    const uint4* src = reinterpret_cast<const uint4*>(y + pl * HW);
    float s0 = 0.f, s1 = 0.f;
    for (int i = lane; i < HW / 8; i += 32) {
      const uint4 r = src[i];
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float a = __uint_as_float(w[e] << 16), b = __uint_as_float(w[e] & 0xffff0000u);
        s0 += a + b;
        s1 = fmaf(a, a, fmaf(b, b, s1));
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, off);
      s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    }
    if (lane == 0) {
      const int o = (int)(pl % A.g.O);
      atomicAdd(&A.w.dsum[o], (double)s0);
      atomicAdd(&A.w.dsum[A.g.O + o], (double)s1);
    }
  }
}

__global__ void cb_stats_finish_kernel(const CbArgs A) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= A.g.O) return;
  const double cnt = (double)A.g.N * A.g.HO * A.g.WO;
  const double mean = A.w.dsum[o] / cnt;
  const double var = A.w.dsum[A.g.O + o] / cnt - mean * mean;
  A.w.mean[o] = (float)mean;
  A.w.rstd[o] = (float)rsqrt((var > 0 ? var : 0) + (double)A.eps);
}

// ---------------------------------------------------------------------------------------------------------------
// shared tile helpers
// ---------------------------------------------------------------------------------------------------------------
// input rows needed by window rows [hp0, hp0+R): conv-output rows 2*hp0 .. 2*(hp0+R)-1, taps -ph .. 2-ph
template <int C>
__device__ __forceinline__ void load_x_tile(const CbArgs& A, int n, int hp0, float* xs) {
  const CbGeom& g = A.g;
  const int rows = g.xrows, pitch = g.xpitch, cols = g.WO + 2;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // warp per (channel, row), lanes along the row: no divisions, coalesced reads
  for (int cr = wid; cr < C * rows; cr += NT / 32) {
    const int c = cr / rows, r = cr - c * rows;
    const int iy = 2 * hp0 - g.ph + r;
    float* d = xs + cr * pitch;
    if (iy < 0 || iy >= g.H) {
      for (int col = lane; col < cols; col += 32) d[col] = 0.f;
      continue;
    }
    const int64_t rowbase = (((int64_t)n * C + c) * g.H + iy) * g.W - g.pw;
    for (int col = lane; col < cols; col += 32) {
      const int ix = col - g.pw;
      d[col] = (ix >= 0 && ix < g.W) ? bb::ldf(A.x, rowbase + col, A.dtx) : 0.f;
    }
  }
}

// Bulk copy of a contiguous global range into shared memory with cp.async (no register staging: every thread has
// several independent 16-byte requests in flight, so the pooled arrays of a whole tile stream in at DRAM latency
// once instead of once per window -- the first version of these kernels ran at 10 % of DRAM throughput on exactly
// that dependency).  Falls back to plain loads for unaligned ranges.
__device__ __forceinline__ void tile_copy_async(void* dst_smem, const void* src, int nbytes) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  const uintptr_t a = reinterpret_cast<uintptr_t>(src);
  if (((a | d | (uintptr_t)nbytes) & 15) == 0) {
    for (int i = threadIdx.x * 16; i < nbytes; i += NT * 16)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + i), "l"(a + i) : "memory");
  } else if (((a | d | (uintptr_t)nbytes) & 3) == 0) {
    for (int i = threadIdx.x * 4; i < nbytes; i += NT * 4)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d + i), "l"(a + i) : "memory");
  } else {
    const unsigned char* sp = reinterpret_cast<const unsigned char*>(src);
    unsigned char* dp = reinterpret_cast<unsigned char*>(dst_smem);
    for (int i = threadIdx.x; i < nbytes; i += NT) dp[i] = sp[i];
  }
}
__device__ __forceinline__ void tile_copy_wait() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// dot of the 3x3xC patch whose top-left tap sits at xs[base] with per-lane weights tw[C*9]
template <int C>
__device__ __forceinline__ float patch_dot(const float* xs, int base, int plane, int pitch, const float* tw) {
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c)
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) acc = fmaf(xs[base + c * plane + i * pitch + j], tw[(c * 3 + i) * 3 + j], acc);
  return acc;
}

// ---------------------------------------------------------------------------------------------------------------
// base-backward preparation: arg-max codes, ReLU mask, xhat at the arg-max pixel, masked base adjoint (NHWC)
// ---------------------------------------------------------------------------------------------------------------
// One block per (image, pooled row): phase 1 walks the NCHW pooled tensors (idx / q / a_q: runs of WP contiguous
// elements per channel) and fills a [WP][O] shared tile, phase 2 writes the channels-last rows in full 128-byte lines
// (the element-per-thread version scattered three 1-2 byte stores per element: 2.45 ms at N=800).
template <typename PT>
__global__ void __launch_bounds__(256) cb_prep_kernel(const CbArgs A) {
  extern __shared__ float prep_sm[];
  const CbGeom& g = A.g;
  const int n = blockIdx.x / g.HP, hp = blockIdx.x - n * g.HP;
  const int cnt = g.WP * g.O;
  float* xh_t = prep_sm;                       // [WP][O]
  float* aq_t = prep_sm + cnt;                 // [WP][O]   (NCHW a_q only)
  unsigned char* sel_t = reinterpret_cast<unsigned char*>(prep_sm + 2 * cnt);
  for (int e = threadIdx.x; e < cnt; e += blockDim.x) {
    const int o = e / g.WP, wp = e - o * g.WP;
    const int64_t i = (((int64_t)n * g.O + o) * g.HP + hp) * g.WP + wp;
    const int64_t id = A.idx[i];
    const int iy = (int)(id / g.WO), ix = (int)(id - (int64_t)iy * g.WO);
    const int dy = iy - 2 * hp, dx = ix - 2 * wp;
    const bool m = g.relu ? (bb::ldf(A.q, i, A.dtq) > 0.f) : true;
    const float yv = bb::ldf(A.y, ((int64_t)n * g.O + o) * g.HO * g.WO + id, A.dty);
    const int t = wp * g.O + o;
    sel_t[t] = (unsigned char)((dy & 1) * 2 + (dx & 1) + (m ? 4 : 0));
    xh_t[t] = (yv - A.w.mean[o]) * A.w.rstd[o];
    if (!A.aq_nhwc) aq_t[t] = A.a_q[i];
  }
  __syncthreads();
  const int64_t p0 = ((int64_t)n * g.HP + hp) * g.WP * g.O;
  for (int t = threadIdx.x; t < cnt; t += blockDim.x) {
    const unsigned char code = sel_t[t];
    float aq;
    if (A.aq_nhwc) {
      const int wp = t / g.O, o = t - wp * g.O;
      aq = __bfloat162float(A.aq_nhwc[((((int64_t)n * (g.HP + 2) + hp + 1) * (g.WP + 2)) + wp + 1) * 64 + o]);
    } else {
      aq = aq_t[t];
    }
    A.w.sel[p0 + t] = code;
    stp<PT>(reinterpret_cast<PT*>(A.w.xh), p0 + t, xh_t[t]);
    stp<PT>(reinterpret_cast<PT*>(A.w.aqm), p0 + t, (code & 4) ? aq : 0.f);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Gram pass (once per call): s, sx, G, S2 over every pixel of y
// ---------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(NT) cb_gram_kernel(const CbArgs A) {
  // tile = (image n, band of 2R conv-output rows) -- the same input tile as the K-loop kernels.
  //   warps 0 .. NW-3: lane <-> channel o, warp <-> (channel group, pixel group); per-lane G[o,:] / sx[o] accumulators,
  //                    the pixel's patch is a shared-memory broadcast
  //   warps NW-2, NW-1: lane k < CKK owns row k of S2 and s[k] (even / odd pixels)
  extern __shared__ float sm[];
  const CbGeom& g = A.g;
  constexpr int CKK = C * 9;
  constexpr int NW = NT / 32;
  const int band = 2 * g.R;
  const int bands = (g.HO + band - 1) / band;
  float* xs = sm;
  const int plane = g.xrows * g.xpitch;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int cgs = (g.O + 31) / 32, pgs = (NW - 2) / cgs;     // channel groups x pixel groups among the G warps
  const bool s2warp = wid >= NW - 2;
  const int cg = wid % cgs, pg = wid / cgs;
  const int o = cg * 32 + lane;
  const bool gwarp = !s2warp && pg < pgs;
  const bool och = gwarp && o < g.O;
  float acc[CKK];
#pragma unroll
  for (int k = 0; k < CKK; ++k) acc[k] = 0.f;
  float a1 = 0.f;
  const float mean = och ? A.w.mean[o] : 0.f, rstd = och ? A.w.rstd[o] : 0.f;
  const int HW = g.HO * g.WO;
  for (int tile = blockIdx.x; tile < g.N * bands; tile += gridDim.x) {
    const int n = tile / bands, b = tile - n * bands;
    __syncthreads();
    load_x_tile<C>(A, n, b * g.R, xs);
    __syncthreads();
    const int row0 = b * band;
    const int npix = min(band, g.HO - row0) * g.WO;
    if (s2warp) {
      if (lane < CKK) {
        for (int p = wid - (NW - 2); p < npix; p += 2) {
          const int oy = p / g.WO, ox = p - oy * g.WO;
          const int base = oy * g.xpitch + ox;
          const int c0 = lane / 9, r0 = lane - c0 * 9, i0 = r0 / 3, j0 = r0 - i0 * 3;
          const float mine = xs[base + c0 * plane + i0 * g.xpitch + j0];
          a1 += mine;
#pragma unroll
          for (int c = 0; c < C; ++c)
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
              for (int j = 0; j < 3; ++j)
                acc[(c * 3 + i) * 3 + j] = fmaf(mine, xs[base + c * plane + i * g.xpitch + j], acc[(c * 3 + i) * 3 + j]);
        }
      }
    } else if (och) {
      const int64_t ybase = ((int64_t)n * g.O + o) * HW + (int64_t)row0 * g.WO;
      for (int p = pg; p < npix; p += pgs) {
        const int oy = p / g.WO, ox = p - oy * g.WO;
        const int base = oy * g.xpitch + ox;
        const float xh = (bb::ldf(A.y, ybase + p, A.dty) - mean) * rstd;
        a1 += xh;
#pragma unroll
        for (int c = 0; c < C; ++c)
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j)
              acc[(c * 3 + i) * 3 + j] = fmaf(xh, xs[base + c * plane + i * g.xpitch + j], acc[(c * 3 + i) * 3 + j]);
      }
    }
  }
  // one double atomic per accumulator and thread (once per call)
  double* D = A.w.dsum + 2 * g.O;                         // [KP] s | [O] sx | [O*KP] G | [KP*KP] S2
  if (s2warp) {
    if (lane < CKK) {
      atomicAdd(&D[lane], (double)a1);
#pragma unroll
      for (int k = 0; k < CKK; ++k) atomicAdd(&D[KP + g.O + g.O * KP + lane * KP + k], (double)acc[k]);
    }
  } else if (och) {
    atomicAdd(&D[KP + o], (double)a1);
#pragma unroll
    for (int k = 0; k < CKK; ++k) atomicAdd(&D[KP + g.O + o * KP + k], (double)acc[k]);
  }
}

__global__ void cb_gram_finish_kernel(const CbArgs A) {
  const CbGeom& g = A.g;
  const double* D = A.w.dsum + 2 * g.O;
  const int n = KP + g.O + g.O * KP + KP * KP;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = (float)D[i];
    if (i < KP) A.w.s[i] = v;
    else if (i < KP + g.O) A.w.sx[i - KP] = v;
    else if (i < KP + g.O + g.O * KP) A.w.G[i - KP - g.O] = v;
    else A.w.S2[i - KP - g.O - g.O * KP] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// tangent forward: t_q and dxhat at the arg-max pixels
//   lane <-> channel (its 27 direction weights live in registers), warp <-> (channel group, window group); the four
//   candidate pixels of a window are four distinct shared-memory words -> conflict-free broadcast reads.  Window
//   indices advance without divisions; the pooled NHWC arrays (code, xhat) of the next window are fetched while the
//   current one is being computed.
// ---------------------------------------------------------------------------------------------------------------
template <int C, typename PT>
__global__ void __launch_bounds__(NT, 4) cb_tf_kernel(const CbArgs A) {
  extern __shared__ float sm[];
  const CbGeom g = A.g;
  constexpr int CKK = C * 9;
  const int plane = g.xrows * g.xpitch;
  float* xs = sm;
  float* outs = sm + C * plane;                    // [O][wpitch] pooled tile, transposed for the NCHW store
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int cgs = (g.O + 31) / 32, wgs = (NT / 32) / cgs;   // channel groups x window groups
  const int cg = wid % cgs, wg = wid / cgs;
  const int o = cg * 32 + lane;
  const bool och = o < g.O && wg < wgs;
  const double invP = 1.0 / ((double)g.N * g.HO * g.WO);
  const unsigned char* __restrict__ sel = A.w.sel;
  const PT* __restrict__ xhp = reinterpret_cast<const PT*>(A.w.xh);
  PT* __restrict__ dxhp = reinterpret_cast<PT*>(A.w.dxh);
  // per-lane channel constants
  float tw[CKK];
  float mean_t = 0.f, sdot = 0.f, rstd = 0.f, gam = 1.f, tgam = 0.f, tbeta = 0.f, tb = 0.f;
  if (och) {
    double d0 = 0, d1 = 0;
#pragma unroll
    for (int k = 0; k < CKK; ++k) {
      tw[k] = A.t_W[o * CKK + k];
      d0 += (double)tw[k] * A.w.s[k];
      d1 += (double)tw[k] * A.w.G[o * KP + k];
    }
    tb = A.t_b ? A.t_b[o] : 0.f;
    const double mt = d0 * invP + tb;
    const double sx = A.w.sx[o];
    mean_t = (float)mt;
    sdot = (float)((d1 + tb * sx - mt * sx) * invP);
    rstd = A.w.rstd[o];
    gam = A.gamma ? A.gamma[o] : 1.f;
    tgam = A.t_gamma ? A.t_gamma[o] : 0.f;
    tbeta = A.t_beta ? A.t_beta[o] : 0.f;
    if (blockIdx.x == 0 && wg == 0) {
      A.w.mean_t[o] = mean_t;
      A.w.sdot[o] = sdot;
    }
  } else {
#pragma unroll
    for (int k = 0; k < CKK; ++k) tw[k] = 0.f;
  }
  // t_q = mask * (c_y * t_y + c_x * xhat + c_0)
  const float c_y = gam * rstd, c_x = tgam - gam * rstd * sdot, c_0 = tbeta + gam * rstd * (tb - mean_t);
  const float e_0 = (tb - mean_t) * rstd, e_x = -sdot * rstd;          // dxhat = rstd*t_y + e_x*xhat + e_0
  const int pitch = g.xpitch, WPc = g.WP, Oc = g.O;
  int roff[C * 3];                                                      // (channel, tap row) offsets inside the x tile
#pragma unroll
  for (int r = 0; r < C * 3; ++r) roff[r] = (r / 3) * plane + (r % 3) * pitch;
  const int tcap = g.R * g.WP * g.O;                 // pooled elements of a full tile
  PT* xh_s = reinterpret_cast<PT*>(outs + (A.tq_nhwc ? 0 : g.O * g.wpitch));   // [nw][O] xhat* of the tile (no NCHW
                                                                                // staging tile in NHWC mode)
  unsigned char* sel_s = reinterpret_cast<unsigned char*>(xh_s + tcap);
  for (int tile = blockIdx.x; tile < g.ntiles; tile += gridDim.x) {
    const int n = tile / g.tiles_per_img, tr = tile - n * g.tiles_per_img;
    const int hp0 = tr * g.R, rows = min(g.R, g.HP - hp0), nw = rows * g.WP;
    const int64_t t0 = ((int64_t)n * g.HP + hp0) * g.WP * g.O;             // NHWC index of (window 0, channel 0)
    __syncthreads();
    tile_copy_async(xh_s, xhp + t0, nw * g.O * (int)sizeof(PT));
    tile_copy_async(sel_s, sel + t0, nw * g.O);
    load_x_tile<C>(A, n, hp0, xs);
    tile_copy_wait();
    __syncthreads();
    if (och) {
      // strength-reduced indices: everything below advances by additions (the first version spent ~50 integer
      // multiply-adds per window on address arithmetic)
      int wr = 0, wc = wg;
      while (wc >= WPc) { wc -= WPc; ++wr; }
      int rowbase = 2 * wr * pitch + 2 * wc;                    // xs offset of the window's top-left candidate pixel
      int sidx = wg * Oc + o;                                   // index into the staged pooled arrays
      PT* dxo = dxhp + t0 + sidx;                               // global dxhat* slot
      __nv_bfloat16* tqo = A.tq_nhwc
          ? A.tq_nhwc + ((((int64_t)n * (g.HP + 2) + hp0 + wr + 1) * (WPc + 2)) + wc + 1) * 64 + o : nullptr;
      for (int wl = wg; wl < nw; wl += wgs) {
        const unsigned code_c = sel_s[sidx];
        const float xh_c = ldp<PT>(xh_s, sidx);
        const float* px = xs + rowbase + ((code_c & 2) ? pitch : 0) + (code_c & 1);
        float ty = 0.f;
#pragma unroll
        for (int r = 0; r < C * 3; ++r) {
          const float* q = px + roff[r];
          ty = fmaf(q[0], tw[3 * r], ty);
          ty = fmaf(q[1], tw[3 * r + 1], ty);
          ty = fmaf(q[2], tw[3 * r + 2], ty);
        }
        stp<PT>(dxo, 0, fmaf(rstd, ty, fmaf(e_x, xh_c, e_0)));
        const float tq = (code_c & 4) ? fmaf(c_y, ty, fmaf(c_x, xh_c, c_0)) : 0.f;
        if (tqo)
          *tqo = __float2bfloat16(tq);
        else
          outs[o * g.wpitch + wl] = tq;
        sidx += wgs * Oc;
        dxo += wgs * Oc;
        wc += wgs;
        rowbase += 2 * wgs;
        if (tqo) tqo += wgs * 64;
        while (wc >= WPc) {
          wc -= WPc; ++wr;
          rowbase += 2 * pitch - 2 * WPc;
          if (tqo) tqo += 2 * 64;                                // skip the right border of this row and the left of the next
        }
      }
    }
    if (!A.tq_nhwc) {
      __syncthreads();
      // NCHW store: for each channel the tile's windows are `nw` consecutive floats; warp per channel, lanes along them
      float* dst = A.t_q + (((int64_t)n * g.O) * g.HP + hp0) * g.WP;
      for (int oo = wid; oo < g.O; oo += NT / 32) {
        float* d = dst + (int64_t)oo * g.HP * g.WP;
        const float* sp = outs + oo * g.wpitch;
        for (int wl = lane; wl < nw; wl += 32) d[wl] = sp[wl];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// pooled-resolution reduction (tangent backward; BASE = the same sums for the base adjoint, once per call)
//   part[cta][o][k < KP]  = sum_w v(w,o) X[p*(w,o), k]         v = mask*at_q   (BASE: mask*a_q)
//   part[cta][o][KP + 0]  = sum_w v
//   part[cta][o][KP + 1]  = sum_w v * xhat_sel
//   part[cta][o][KP + 2]  = sum_w mask*a_q * dxhat_sel         (TB only)
// ---------------------------------------------------------------------------------------------------------------
template <int C, bool BASE, typename PT>
__global__ void __launch_bounds__(NT) cb_reduce_kernel(const CbArgs A) {
  extern __shared__ float sm[];
  const CbGeom g = A.g;
  constexpr int CKK = C * 9;
  const int plane = g.xrows * g.xpitch;
  float* xs = sm;
  float* ins = sm + C * plane;                     // [O][wpitch] at_q tile (NCHW load, transposed reads)
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int cgs = (g.O + 31) / 32, wgs = (NT / 32) / cgs;
  const int cg = wid % cgs, wg = wid / cgs;
  const int o = cg * 32 + lane;
  const bool och = o < g.O && wg < wgs;
  const unsigned char* __restrict__ sel = A.w.sel;
  const PT* __restrict__ xhp = reinterpret_cast<const PT*>(A.w.xh);
  const PT* __restrict__ dxhp = reinterpret_cast<const PT*>(A.w.dxh);
  const PT* __restrict__ aqm = reinterpret_cast<const PT*>(A.w.aqm);
  float gw[CKK];
#pragma unroll
  for (int k = 0; k < CKK; ++k) gw[k] = 0.f;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  const int pitch = g.xpitch, WPc = g.WP, Oc = g.O;
  int roff[C * 3];
#pragma unroll
  for (int r = 0; r < C * 3; ++r) roff[r] = (r / 3) * plane + (r % 3) * pitch;
  const int tcap = g.R * g.WP * g.O;
  // pooled arrays of the tile; in NHWC mode the transposed NCHW staging tile `ins` is not needed and its place is taken
  // by the adjoint-tangent rows themselves ([rows][WP][64] bf16, copied row by row out of the padded array)
  const bool nhwc_mode = A.atq_nhwc != nullptr || A.tq_nhwc != nullptr;     // (the launcher sizes shared memory by this)
  const bool nhwc_in = !BASE && A.atq_nhwc != nullptr;
  PT* xh_s = reinterpret_cast<PT*>(ins + (nhwc_mode ? 0 : g.O * g.wpitch));
  PT* aq_s = xh_s + tcap;
  PT* dx_s = aq_s + tcap;
  unsigned char* sel_s = reinterpret_cast<unsigned char*>(dx_s + tcap);
  __nv_bfloat16* at_s = reinterpret_cast<__nv_bfloat16*>(sel_s + ((tcap + 15) & ~15));
  for (int tile = blockIdx.x; tile < g.ntiles; tile += gridDim.x) {
    const int n = tile / g.tiles_per_img, tr = tile - n * g.tiles_per_img;
    const int hp0 = tr * g.R, rows = min(g.R, g.HP - hp0), nw = rows * g.WP;
    const int64_t t0 = ((int64_t)n * g.HP + hp0) * g.WP * g.O;
    __syncthreads();
    tile_copy_async(xh_s, xhp + t0, nw * g.O * (int)sizeof(PT));
    tile_copy_async(aq_s, aqm + t0, nw * g.O * (int)sizeof(PT));
    if (!BASE) tile_copy_async(dx_s, dxhp + t0, nw * g.O * (int)sizeof(PT));
    tile_copy_async(sel_s, sel + t0, nw * g.O);
    if (nhwc_in)
      for (int rr = 0; rr < rows; ++rr)
        tile_copy_async(at_s + rr * WPc * 64, A.atq_nhwc + ((((int64_t)n * (g.HP + 2) + hp0 + rr + 1) * (WPc + 2)) + 1) * 64,
                        WPc * 64 * 2);
    load_x_tile<C>(A, n, hp0, xs);
    if (!BASE && !A.atq_nhwc) {
      const float* src = A.at_q + (((int64_t)n * g.O) * g.HP + hp0) * g.WP;
      for (int oo = wid; oo < g.O; oo += NT / 32) {
        const float* sp = src + (int64_t)oo * g.HP * g.WP;
        float* d = ins + oo * g.wpitch;
        for (int wl = lane; wl < nw; wl += 32) d[wl] = sp[wl];
      }
    }
    tile_copy_wait();
    __syncthreads();
    if (och) {
      int wr = 0, wc = wg;
      while (wc >= WPc) { wc -= WPc; ++wr; }
      int rowbase = 2 * wr * pitch + 2 * wc;
      int si = wg * Oc + o;
      for (int wl = wg; wl < nw; wl += wgs) {
        const unsigned code_c = sel_s[si];
        const float xh_c = ldp<PT>(xh_s, si), aq_c = ldp<PT>(aq_s, si);
        float v;
        if (BASE) {
          v = aq_c;
        } else {
          const float a = nhwc_in ? __bfloat162float(at_s[wl * 64 + o]) : ins[o * g.wpitch + wl];
          v = (code_c & 4) ? a : 0.f;
          s2 = fmaf(aq_c, ldp<PT>(dx_s, si), s2);
        }
        s0 += v;
        s1 = fmaf(v, xh_c, s1);
        const float* px = xs + rowbase + ((code_c & 2) ? pitch : 0) + (code_c & 1);
#pragma unroll
        for (int r = 0; r < C * 3; ++r) {
          const float* q = px + roff[r];
          gw[3 * r] = fmaf(v, q[0], gw[3 * r]);
          gw[3 * r + 1] = fmaf(v, q[1], gw[3 * r + 1]);
          gw[3 * r + 2] = fmaf(v, q[2], gw[3 * r + 2]);
        }
        si += wgs * Oc;
        wc += wgs;
        rowbase += 2 * wgs;
        while (wc >= WPc) {
          wc -= WPc; ++wr;
          rowbase += 2 * pitch - 2 * WPc;
        }
      }
    }
  }
  // cross-window-group reduction through shared memory, then one partial row per (cta, channel)
  __syncthreads();
  float* red = sm;      // [wgs][O][KP + NSUM] -- reuses the tile memory
  const int stride = KP + NSUM;
  if (och) {
    float* r = red + ((size_t)wg * g.O + o) * stride;
#pragma unroll
    for (int k = 0; k < CKK; ++k) r[k] = gw[k];
    for (int k = CKK; k < KP; ++k) r[k] = 0.f;
    r[KP + 0] = s0; r[KP + 1] = s1; r[KP + 2] = s2; r[KP + 3] = 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < g.O * stride; i += NT) {
    float acc = 0.f;
    for (int w = 0; w < wgs; ++w) acc += red[(size_t)w * g.O * stride + i];
    A.w.part[(size_t)blockIdx.x * g.O * stride + i] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// finish: combine the per-CTA partials (fixed order: deterministic) and write the parameter slices of H.d
// ---------------------------------------------------------------------------------------------------------------
template <bool BASE>
__global__ void __launch_bounds__(64) cb_finish_kernel(const CbArgs A, int CKK) {
  // one block per channel; thread k < KP + NSUM owns one column of the partial rows
  const CbGeom& g = A.g;
  const int o = blockIdx.x, k = threadIdx.x;
  const int stride = KP + NSUM;
  __shared__ float col[KP + NSUM];
  __shared__ float tyx[KP];
  if (k < stride) {
    double acc = 0.0;
    for (int c = 0; c < A.nparts; ++c) acc += A.w.part[((size_t)c * g.O + o) * stride + k];
    col[k] = (float)acc;
  }
  __syncthreads();
  if (BASE) {
    if (k < KP) A.w.Gd[o * KP + k] = col[k];
    if (k == 0) { A.w.Sa[o] = col[KP + 0]; A.w.Saxh[o] = col[KP + 1]; }
    return;
  }
  const double P = (double)g.N * g.HO * g.WO;
  const float rstd = A.w.rstd[o], sdot = A.w.sdot[o], mean_t = A.w.mean_t[o];
  const float gam = A.gamma ? A.gamma[o] : 1.f, tgam = A.t_gamma ? A.t_gamma[o] : 0.f;
  const float tb = A.t_b ? A.t_b[o] : 0.f;
  const float Sa = A.w.Sa[o], Saxh = A.w.Saxh[o];
  const float S_at = col[KP + 0], S_atxh = col[KP + 1], S_adxh = col[KP + 2];
  const float m1 = (float)(gam * Sa / P), m2 = (float)(gam * Saxh / P);
  const float mt1 = (float)((gam * S_at + tgam * Sa) / P);
  const float mt2 = (float)(((double)gam * S_atxh + (double)tgam * Saxh + (double)gam * S_adxh) / P);
  const float d2 = -rstd * rstd * m2;
  const float d1 = -rstd * mt2 + 2.f * rstd * rstd * sdot * m2;
  const float d0 = -rstd * mt1 + rstd * rstd * sdot * m1 + rstd * rstd * m2 * mean_t;
  const float cw = rstd * gam, cd = rstd * tgam - rstd * rstd * sdot * gam;
  if (k < CKK) {
    // (t_W S2)[o,k] + t_b s[k]
    double acc = 0.0;
    for (int l = 0; l < CKK; ++l) acc += (double)A.t_W[o * CKK + l] * A.w.S2[l * KP + k];
    tyx[k] = (float)(acc + (double)tb * A.w.s[k]);
    const float v = cw * col[k] + cd * A.w.Gd[o * KP + k] + d0 * A.w.s[k] + d1 * A.w.G[o * KP + k] + d2 * tyx[k];
    A.at_W[o * CKK + k] += v;
  }
  if (k == 0) {
    if (A.at_gamma) A.at_gamma[o] += S_atxh + S_adxh;
    if (A.at_beta) A.at_beta[o] += S_at;
    if (A.at_b) A.at_b[o] += (float)((double)cw * S_at + (double)cd * Sa + (double)d0 * P + (double)d1 * A.w.sx[o] +
                                     (double)d2 * P * mean_t);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Tensor-core path of the K-loop kernels (O == 64, bf16 pooled arrays, NHWC neighbours on both sides).
//
// x is data, so the 3x3xC patch of each of the four candidate pixels of a window never changes during a call: the base
// pass writes them once as bf16 mma.sync fragments (`pfrag`: rows = 16 consecutive windows, columns = the C*9 taps
// padded to 32; `pfragT`: the transpose).  The tangent-forward kernel is then, per 16 windows, 64 m16n8k16 products
// [windows x taps] x [taps x channels] for the four candidates plus a register select by the arg-max code; the
// reduce kernel is 64 products [taps x windows] x [windows x channels] of the code-masked adjoint tangent.  The SIMT
// kernels above spent ~105 instructions per (window, channel) on 27 multiply-adds; column C*9 of the patch matrix
// holds 1, so the plain channel sum of the masked adjoint falls out of the same product.
// ---------------------------------------------------------------------------------------------------------------
constexpr int MT = 16;            // windows per m-tile
constexpr int STG_V = 144;        // bytes per staged row of 64 bf16 (128 + 16: conflict-free for ldmatrix and pair reads)
constexpr int STG_C = 80;         // bytes per staged row of 64 code bytes

__device__ __forceinline__ void mma16816(float (&c)[4], const uint4& a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&p);
}
__device__ __forceinline__ uint4 ldg_nc16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// patch matrix: window w (flat over N*HP*WP), candidate d = dy*2+dx, column k = (c*3+i)*3+j; column C*9 holds 1
struct WinPos {
  int64_t base;     // index of x[n][0][2hp + dy - ph][2wp + dx - pw]
  int iy0, ix0;
  bool live;
};
__device__ __forceinline__ WinPos win_pos(const CbGeom& g, int C, int64_t w, int64_t total, int d) {
  WinPos p;
  p.live = w < total;
  const int64_t ww = p.live ? w : 0;
  const int wp = (int)(ww % g.WP);
  const int64_t r = ww / g.WP;
  const int hp = (int)(r % g.HP), n = (int)(r / g.HP);
  p.iy0 = 2 * hp + (d >> 1) - g.ph;
  p.ix0 = 2 * wp + (d & 1) - g.pw;
  p.base = (((int64_t)n * C) * g.H + p.iy0) * g.W + p.ix0;
  return p;
}
template <int C>
__device__ __forceinline__ float patch_value(const CbArgs& A, const WinPos& p, int k) {
  if (!p.live || k > C * 9) return 0.f;
  if (k == C * 9) return 1.f;
  const int c = k / 9, i = (k % 9) / 3, j = k % 3;
  const int iy = p.iy0 + i, ix = p.ix0 + j;
  if (iy < 0 || iy >= A.g.H || ix < 0 || ix >= A.g.W) return 0.f;
  return bb::ldf(A.x, p.base + ((int64_t)c * A.g.H + i) * A.g.W + j, A.dtx);
}

// one thread per (m-tile, candidate d, lane): the four fragments pfrag[d*2+ks] (rows = windows, columns = taps) and
// pfragT[d*2+mk] (rows = taps, columns = windows) of its candidate
template <int C>
__global__ void __launch_bounds__(256) cb_patch_frag_kernel(const CbArgs A, int64_t nmt) {
  const int64_t total = (int64_t)A.g.N * A.g.HP * A.g.WP;
  const int64_t nthreads = nmt * 4 * 32;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nthreads; i += (int64_t)gridDim.x * blockDim.x) {
    const int lane = (int)(i & 31), d = (int)((i >> 5) & 3);
    const int64_t mt = i >> 7;
    const int gq = lane >> 2, t = lane & 3;
    const int64_t w0 = mt * MT;
    uint4* pf = reinterpret_cast<uint4*>(A.w.pfrag) + (mt * 8 + d * 2) * 32 + lane;
    uint4* pt = reinterpret_cast<uint4*>(A.w.pfragT) + (mt * 8 + d * 2) * 32 + lane;
    {
      const WinPos r0 = win_pos(A.g, C, w0 + gq, total, d), r1 = win_pos(A.g, C, w0 + gq + 8, total, d);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = patch_value<C>(A, ((e >> 1) & 1) ? r1 : r0, ks * 16 + 2 * t + (e & 1) + (e >> 2) * 8);
        pf[ks * 32] = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
      }
    }
    {
      const WinPos c0 = win_pos(A.g, C, w0 + 2 * t, total, d), c1 = win_pos(A.g, C, w0 + 2 * t + 1, total, d);
      const WinPos c2 = win_pos(A.g, C, w0 + 2 * t + 8, total, d), c3 = win_pos(A.g, C, w0 + 2 * t + 9, total, d);
#pragma unroll
      for (int mk = 0; mk < 2; ++mk) {
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int k = mk * 16 + gq + ((e >> 1) & 1) * 8;
          v[e] = patch_value<C>(A, (e >> 2) ? ((e & 1) ? c3 : c2) : ((e & 1) ? c1 : c0), k);
        }
        pt[mk * 32] = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
      }
    }
  }
}

// padded-NHWC pixel index of window w (the fused neighbour's [N][HP+2][WP+2][64] layout)
__device__ __forceinline__ int64_t padded_pixel(const CbGeom& g, int64_t w) {
  const int wp = (int)(w % g.WP);
  const int64_t r = w / g.WP;
  const int hp = (int)(r % g.HP);
  const int64_t n = r / g.HP;
  return ((n * (g.HP + 2) + hp + 1) * (g.WP + 2)) + wp + 1;
}

template <int C>
__global__ void __launch_bounds__(256) cb_tf_mma_kernel(const CbArgs A, int64_t nmt) {
  constexpr int CKK = C * 9;
  __shared__ uint2 bfrag[8 * 2 * 32];
  __shared__ __align__(16) float cst[6][64];                 // rstd, e_x, e_0, c_y, c_x, c_0
  extern __shared__ __align__(16) uint8_t stage_raw[];         // [8 warps][MT * (STG_C + 2 * STG_V)]
  const CbGeom& g = A.g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gq = lane >> 2, t = lane & 3;
  const int64_t total = (int64_t)g.N * g.HP * g.WP;
  if (tid < 64) {
    const int o = tid;
    const double invP = 1.0 / ((double)g.N * g.HO * g.WO);
    double d0 = 0, d1 = 0;
    for (int k = 0; k < CKK; ++k) {
      const double tw = A.t_W[o * CKK + k];
      d0 += tw * A.w.s[k];
      d1 += tw * A.w.G[o * KP + k];
    }
    const float tb = A.t_b ? A.t_b[o] : 0.f;
    const double mt = d0 * invP + tb;
    const double sx = A.w.sx[o];
    const float mean_t = (float)mt;
    const float sdot = (float)((d1 + tb * sx - mt * sx) * invP);
    const float rstd = A.w.rstd[o];
    const float gam = A.gamma ? A.gamma[o] : 1.f, tgam = A.t_gamma ? A.t_gamma[o] : 0.f;
    const float tbeta = A.t_beta ? A.t_beta[o] : 0.f;
    if (blockIdx.x == 0) {
      A.w.mean_t[o] = mean_t;
      A.w.sdot[o] = sdot;
    }
    cst[0][o] = rstd;
    cst[1][o] = -sdot * rstd;
    cst[2][o] = (tb - mean_t) * rstd;
    cst[3][o] = gam * rstd;
    cst[4][o] = tgam - gam * rstd * sdot;
    cst[5][o] = tbeta + gam * rstd * (tb - mean_t);
  }
  for (int i = tid; i < 8 * 2 * 32; i += 256) {
    const int ln = i & 31, ks = (i >> 5) & 1, j = i >> 6;
    const int o = j * 8 + (ln >> 2), k0 = ks * 16 + 2 * (ln & 3);
    auto tw = [&](int k) { return k < CKK ? A.t_W[o * CKK + k] : 0.f; };
    bfrag[i] = make_uint2(pack_bf16(tw(k0), tw(k0 + 1)), pack_bf16(tw(k0 + 8), tw(k0 + 9)));
  }
  __syncthreads();
  uint8_t* codes_s = stage_raw + warp * (MT * (STG_C + 2 * STG_V));
  uint8_t* xh_s = codes_s + MT * STG_C;
  uint8_t* tq_s = xh_s + MT * STG_V;
  const uint4* pf = reinterpret_cast<const uint4*>(A.w.pfrag);
  const uint8_t* xhg = reinterpret_cast<const uint8_t*>(A.w.xh);
  uint8_t* dxg = reinterpret_cast<uint8_t*>(A.w.dxh);
  const int srow = lane >> 1, shalf = lane & 1;               // staging role: (window row, 32-channel half)
  for (int64_t mt = (int64_t)blockIdx.x * 8 + warp; mt < nmt; mt += (int64_t)gridDim.x * 8) {
    const int64_t w0 = mt * MT;
    uint4 af[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) af[q] = ldg_nc16(pf + (mt * 8 + q) * 32 + lane);
    const int64_t ws = w0 + srow;
    const bool live = ws < total;
    {
      uint4 c0 = make_uint4(0, 0, 0, 0), c1 = c0, x0 = c0, x1 = c0, x2 = c0, x3 = c0;
      if (live) {
        const uint8_t* cs = A.w.sel + ws * 64 + shalf * 32;
        c0 = ldg_nc16(cs); c1 = ldg_nc16(cs + 16);
        const uint8_t* xs = xhg + (ws * 64 + shalf * 32) * 2;
        x0 = ldg_nc16(xs); x1 = ldg_nc16(xs + 16); x2 = ldg_nc16(xs + 32); x3 = ldg_nc16(xs + 48);
      }
      uint4* cd = reinterpret_cast<uint4*>(codes_s + srow * STG_C + shalf * 32);
      cd[0] = c0; cd[1] = c1;
      uint4* xd = reinterpret_cast<uint4*>(xh_s + srow * STG_V + shalf * 64);
      xd[0] = x0; xd[1] = x1; xd[2] = x2; xd[3] = x3;
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float acc[4][4][4];
#pragma unroll
      for (int d = 0; d < 4; ++d)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int r = 0; r < 4; ++r) acc[d][j][r] = 0.f;
      // ks outermost: 16 independent products between two that touch the same accumulator
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint2 b = bfrag[((h * 4 + j) * 2 + ks) * 32 + lane];
#pragma unroll
          for (int d = 0; d < 4; ++d) mma16816(acc[d][j], af[d * 2 + ks], b.x, b.y);
        }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = (h * 4 + j) * 8 + 2 * t;
        const float2 k_r = *reinterpret_cast<const float2*>(&cst[0][col]), k_ex = *reinterpret_cast<const float2*>(&cst[1][col]);
        const float2 k_e0 = *reinterpret_cast<const float2*>(&cst[2][col]), k_cy = *reinterpret_cast<const float2*>(&cst[3][col]);
        const float2 k_cx = *reinterpret_cast<const float2*>(&cst[4][col]), k_c0 = *reinterpret_cast<const float2*>(&cst[5][col]);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int row = gq + 8 * rr;
          const unsigned cp = *reinterpret_cast<const unsigned short*>(codes_s + row * STG_C + col);
          uint32_t* xp = reinterpret_cast<uint32_t*>(xh_s + row * STG_V + col * 2);
          const uint32_t xr = *xp;
          const float xa = __uint_as_float(xr << 16), xb = __uint_as_float(xr & 0xffff0000u);
          const unsigned ca = cp & 0xffu, cb = cp >> 8;
          const unsigned sa = ca & 3u, sb = cb & 3u;
          const float ta = sa == 0 ? acc[0][j][2 * rr] : sa == 1 ? acc[1][j][2 * rr] : sa == 2 ? acc[2][j][2 * rr] : acc[3][j][2 * rr];
          const float tb2 = sb == 0 ? acc[0][j][2 * rr + 1] : sb == 1 ? acc[1][j][2 * rr + 1] : sb == 2 ? acc[2][j][2 * rr + 1]
                                                                                                    : acc[3][j][2 * rr + 1];
          const float da = fmaf(k_r.x, ta, fmaf(k_ex.x, xa, k_e0.x)), db = fmaf(k_r.y, tb2, fmaf(k_ex.y, xb, k_e0.y));
          const float qa = (ca & 4u) ? fmaf(k_cy.x, ta, fmaf(k_cx.x, xa, k_c0.x)) : 0.f;
          const float qb = (cb & 4u) ? fmaf(k_cy.y, tb2, fmaf(k_cx.y, xb, k_c0.y)) : 0.f;
          *xp = pack_bf16(da, db);                                            // dxhat* over xhat* (same owner thread)
          *reinterpret_cast<uint32_t*>(tq_s + row * STG_V + col * 2) = pack_bf16(qa, qb);
        }
      }
    }
    __syncwarp();
    if (live) {
      const uint4* xd = reinterpret_cast<const uint4*>(xh_s + srow * STG_V + shalf * 64);
      uint4* dd = reinterpret_cast<uint4*>(dxg + (ws * 64 + shalf * 32) * 2);
      dd[0] = xd[0]; dd[1] = xd[1]; dd[2] = xd[2]; dd[3] = xd[3];
      const uint4* td = reinterpret_cast<const uint4*>(tq_s + srow * STG_V + shalf * 64);
      uint4* qd = reinterpret_cast<uint4*>(A.tq_nhwc + padded_pixel(g, ws) * 64 + shalf * 32);
      qd[0] = td[0]; qd[1] = td[1]; qd[2] = td[2]; qd[3] = td[3];
    }
    __syncwarp();
  }
}

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem_row);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

// GW[o][k] = sum_w v[w][o] patch_{code(w,o)}[w][k]  (+ the channel sums s0 = sum v, s1 = sum v xhat*, s2 = sum a_q dxhat*)
// v = mask a_q (BASE) or the masked adjoint tangent at_q.  Per 16 windows: the [w][o] tile of v and of the codes (as
// 16-bit) are staged in shared memory, ldmatrix.trans turns them into B fragments (pairs along w), the per-candidate
// mask is two SIMD-in-word compares per register.
template <int C, bool BASE>
__global__ void __launch_bounds__(256, 2) cb_reduce_mma_kernel(const CbArgs A, int64_t nmt) {
  constexpr int CKK = C * 9;
  __shared__ __align__(16) uint8_t stage[8][2 * MT * STG_V];
  __shared__ float red[64][KP + NSUM];
  const CbGeom& g = A.g;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gq = lane >> 2, t = lane & 3;
  const int64_t total = (int64_t)g.N * g.HP * g.WP;
  for (int i = tid; i < 64 * (KP + NSUM); i += 256) (&red[0][0])[i] = 0.f;
  __syncthreads();
  uint8_t* v_s = stage[warp];
  uint8_t* c_s = v_s + MT * STG_V;
  const uint4* pf = reinterpret_cast<const uint4*>(A.w.pfragT);
  const uint8_t* xhg = reinterpret_cast<const uint8_t*>(A.w.xh);
  const uint8_t* dxg = reinterpret_cast<const uint8_t*>(A.w.dxh);
  const uint8_t* aqg = reinterpret_cast<const uint8_t*>(A.w.aqm);
  const int srow = lane >> 1, shalf = lane & 1;
  float gw[2][8][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) gw[m][j][r] = 0.f;
  float s1a = 0.f, s1b = 0.f, s2a = 0.f, s2b = 0.f;     // channels 2*lane, 2*lane+1
  // ldmatrix row address of this lane: matrix mi = lane>>3 -> (window block mi&1, channel block + (mi>>1))
  const int lm_row = ((lane >> 3) & 1) * 8 + (lane & 7), lm_jo = lane >> 4;
  for (int64_t mt = (int64_t)blockIdx.x * 8 + warp; mt < nmt; mt += (int64_t)gridDim.x * 8) {
    const int64_t w0 = mt * MT;
    uint4 af[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) af[q] = ldg_nc16(pf + (mt * 8 + q) * 32 + lane);
    const int64_t ws = w0 + srow;
    const bool live = ws < total;
    {
      uint4 c0 = make_uint4(0, 0, 0, 0), c1 = c0;
      uint32_t v[16];
#pragma unroll
      for (int e = 0; e < 16; ++e) v[e] = 0u;
      if (live) {
        const uint8_t* cs = A.w.sel + ws * 64 + shalf * 32;
        c0 = ldg_nc16(cs); c1 = ldg_nc16(cs + 16);
        const uint8_t* vs = BASE ? aqg + (ws * 64 + shalf * 32) * 2
                                 : reinterpret_cast<const uint8_t*>(A.atq_nhwc) + (padded_pixel(g, ws) * 64 + shalf * 32) * 2;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const uint4 r = BASE ? ldg_nc16(vs + 16 * e) : *reinterpret_cast<const uint4*>(vs + 16 * e);
          v[4 * e] = r.x; v[4 * e + 1] = r.y; v[4 * e + 2] = r.z; v[4 * e + 3] = r.w;
        }
      }
      const uint32_t cw[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      uint32_t c16[16];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        c16[2 * e] = __byte_perm(cw[e], 0u, 0x4140);          // codes 0,1 of the word as two 16-bit lanes
        c16[2 * e + 1] = __byte_perm(cw[e], 0u, 0x4342);      // codes 2,3
      }
      if (!BASE) {
#pragma unroll
        for (int e = 0; e < 16; ++e) v[e] &= __vcmpne2(c16[e] & 0x00040004u, 0u);      // relu mask (a_q m is pre-masked)
      }
      uint4* vd = reinterpret_cast<uint4*>(v_s + srow * STG_V + shalf * 64);
      uint4* cd = reinterpret_cast<uint4*>(c_s + srow * STG_V + shalf * 64);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        vd[e] = make_uint4(v[4 * e], v[4 * e + 1], v[4 * e + 2], v[4 * e + 3]);
        cd[e] = make_uint4(c16[4 * e], c16[4 * e + 1], c16[4 * e + 2], c16[4 * e + 3]);
      }
    }
    __syncwarp();
    // channel sums: lane <-> channels 2*lane, 2*lane+1, loop over the tile's windows
    {
      const int nlive = (int)((total - w0) < MT ? (total - w0) : MT);
#pragma unroll 4
      for (int r = 0; r < MT; ++r) {
        if (r >= nlive) break;
        const int64_t gi = ((w0 + r) * 64 + 2 * lane) * 2;
        const uint32_t vv = *reinterpret_cast<const uint32_t*>(v_s + r * STG_V + lane * 4);
        const uint32_t xx = *reinterpret_cast<const uint32_t*>(xhg + gi);
        const float va = __uint_as_float(vv << 16), vb = __uint_as_float(vv & 0xffff0000u);
        s1a = fmaf(va, __uint_as_float(xx << 16), s1a);
        s1b = fmaf(vb, __uint_as_float(xx & 0xffff0000u), s1b);
        if (!BASE) {
          const uint32_t aa = *reinterpret_cast<const uint32_t*>(aqg + gi), dd = *reinterpret_cast<const uint32_t*>(dxg + gi);
          s2a = fmaf(__uint_as_float(aa << 16), __uint_as_float(dd << 16), s2a);
          s2b = fmaf(__uint_as_float(aa & 0xffff0000u), __uint_as_float(dd & 0xffff0000u), s2b);
        }
      }
    }
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      uint32_t bv[4], bc[4];
      ldmatrix_x4_trans(bv, v_s + lm_row * STG_V + (2 * jp + lm_jo) * 16);
      ldmatrix_x4_trans(bc, c_s + lm_row * STG_V + (2 * jp + lm_jo) * 16);
#pragma unroll
      for (int e = 0; e < 4; ++e) bc[e] &= 0x00030003u;
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        const uint32_t want = (uint32_t)d * 0x00010001u;
        uint32_t m[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) m[e] = bv[e] & __vcmpeq2(bc[e], want);
#pragma unroll
        for (int mk = 0; mk < 2; ++mk) {
          mma16816(gw[mk][2 * jp], af[d * 2 + mk], m[0], m[1]);
          mma16816(gw[mk][2 * jp + 1], af[d * 2 + mk], m[2], m[3]);
        }
      }
    }
    __syncwarp();
  }
  // per-CTA partial row: taps k < CKK -> GW columns, k == CKK -> s0.  The lanes of a warp own distinct entries, so the
  // warps add in turn (warp order, not arrival order: the partial is the same every run)
  for (int w = 0; w < 8; ++w) {
    if (warp == w) {
#pragma unroll
      for (int mk = 0; mk < 2; ++mk)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int k = mk * 16 + gq + (r >> 1) * 8, o = j * 8 + 2 * t + (r & 1);
            if (k < CKK)
              red[o][k] += gw[mk][j][r];
            else if (k == CKK)
              red[o][KP + 0] += gw[mk][j][r];
          }
      red[2 * lane][KP + 1] += s1a;
      red[2 * lane + 1][KP + 1] += s1b;
      if (!BASE) {
        red[2 * lane][KP + 2] += s2a;
        red[2 * lane + 1][KP + 2] += s2b;
      }
    }
    __syncthreads();
  }
  for (int i = tid; i < 64 * (KP + NSUM); i += 256) A.w.part[(size_t)blockIdx.x * 64 * (KP + NSUM) + i] = (&red[0][0])[i];
}

template <int C, typename PT>
int run(const CbArgs& A0, int pass, cudaStream_t s) {
  CbArgs A = A0;
  const CbGeom& g = A.g;
  // x tile + transposed pooled tile (+ staged pooled arrays of one tile: xhat*, mask a_q, dxhat* 4 B each, codes 1 B)
  const size_t tcap = (size_t)g.R * g.WP * g.O;
  const size_t tile = 4 * ((size_t)C * g.xrows * g.xpitch + (size_t)g.O * g.wpitch);
  const int wgs = (NT / 32) / ((g.O + 31) / 32);
  const size_t smem_part = 4 * (size_t)wgs * g.O * (KP + NSUM);
  // NHWC mode (fused neighbour): no transposed NCHW staging tile; the reduce kernel stages the bf16 adjoint-tangent rows
  const bool nhwc = A.tq_nhwc != nullptr || A.atq_nhwc != nullptr;
  const size_t xt = 4 * (size_t)C * g.xrows * g.xpitch, nchw_tile = nhwc ? 0 : 4 * (size_t)g.O * g.wpitch;
  const size_t smem_tf = xt + nchw_tile + (sizeof(PT) + 1) * tcap + 64;
  size_t smem_red = xt + nchw_tile + (3 * sizeof(PT) + 1) * tcap + (nhwc ? 2 * (size_t)g.R * g.WP * 64 : 0) + 128;
  if (smem_red < smem_part) smem_red = smem_part;
  static BbOncePerDevice once;
  if (once.need()) {
    BB_CUDA_TRY(cudaFuncSetAttribute(cb_tf_kernel<C, PT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    BB_CUDA_TRY(cudaFuncSetAttribute(cb_reduce_kernel<C, false, PT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    BB_CUDA_TRY(cudaFuncSetAttribute(cb_reduce_kernel<C, true, PT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    BB_CUDA_TRY(cudaFuncSetAttribute(cb_gram_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    BB_CUDA_TRY(cudaFuncSetAttribute(cb_prep_kernel<PT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  if (smem_red > 200 * 1024 || (size_t)g.WP * g.O * 9 > 200 * 1024) return BB_ERR_UNSUPPORTED;
  // tensor-core path of the K-loop kernels: bf16 pooled arrays, 64 channels, NHWC neighbour on the pooled side.
  // BB200_NO_CBMMA is read at each launch, so a process can run both routes; a plan must keep one route for all passes
  // (the base pass builds the state its tangent passes read).
  const bool no_mma = getenv("BB200_NO_CBMMA") != nullptr;
  const bool mma = !no_mma && g.O == 64 && sizeof(PT) == 2 && A.tq_nhwc && A.atq_nhwc && A.w.pfrag;
  const int64_t nmt = ((int64_t)g.N * g.HP * g.WP + MT - 1) / MT;
  auto mma_blocks = [&](const void* fn, size_t smem) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    return (int)std::min<int64_t>((nmt + 7) / 8, (int64_t)std::min(per_sm * BB_SM_COUNT, GRID_MAX));
  };
  const size_t smem_tf_mma = 8 * MT * (STG_C + 2 * STG_V);
  static BbOncePerDevice once_mma;
  if (mma && once_mma.need())
    BB_CUDA_TRY(cudaFuncSetAttribute(cb_tf_mma_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tf_mma));
  // persistent grids: exactly the CTAs that are resident at once (a partial second wave would run at a fraction of
  // the occupancy for as long as a full one)
  auto resident = [&](const void* fn, size_t smem) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, NT, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    int gmax = per_sm * BB_SM_COUNT;
    if (gmax > GRID_MAX) gmax = GRID_MAX;
    return g.ntiles < gmax ? (g.ntiles < 1 ? 1 : g.ntiles) : gmax;
  };
  if (pass == BB_PASS_BASE_BWD) {
    const size_t nd = sizeof(double) * (2 * g.O + KP + g.O + g.O * KP + KP * KP);
    BB_CUDA_TRY(cudaMemsetAsync(A.w.dsum, 0, nd, s));
    const int64_t per = (int64_t)g.N * g.HO * g.WO;
    int chunks = (int)((per + 256 * 64 - 1) / (256 * 64));
    if (chunks > 64) chunks = 64;
    if (chunks < 1) chunks = 1;
    if (A.dty == BB_BF16 && (g.HO * g.WO) % 8 == 0)
      cb_stats_bf16_kernel<<<8 * BB_SM_COUNT, 256, 0, s>>>(A);
    else
      cb_stats_kernel<<<dim3(g.O, chunks), 256, 0, s>>>(A);
    cb_stats_finish_kernel<<<1, 64, 0, s>>>(A);
    cb_prep_kernel<PT><<<g.N * g.HP, 256, (size_t)g.WP * g.O * 9, s>>>(A);
    const int bands = (g.HO + 2 * g.R - 1) / (2 * g.R);
    int ggrid = g.N * bands < GRID_MAX ? g.N * bands : GRID_MAX;
    cb_gram_kernel<C><<<ggrid, NT, tile, s>>>(A);
    cb_gram_finish_kernel<<<8, 256, 0, s>>>(A);
    if (mma) {
      cb_patch_frag_kernel<C><<<8 * BB_SM_COUNT, 256, 0, s>>>(A, nmt);
      const int mma_grid = mma_blocks((const void*)cb_reduce_mma_kernel<C, true>, 0);
      A.nparts = mma_grid;
      cb_reduce_mma_kernel<C, true><<<mma_grid, 256, 0, s>>>(A, nmt);
      bb_launch_tally += 1;
    } else {
      const int grid = resident((const void*)cb_reduce_kernel<C, true, PT>, smem_red);
      A.nparts = grid;
      cb_reduce_kernel<C, true, PT><<<grid, NT, smem_red, s>>>(A);
    }
    cb_finish_kernel<true><<<g.O, 64, 0, s>>>(A, C * 9);
    bb_launch_tally += 9;
    BB_LAUNCH_CHECK();
    return BB_OK;
  }
  if (pass == BB_PASS_TAN_FWD) {
    if (mma) {
      cb_tf_mma_kernel<C><<<mma_blocks((const void*)cb_tf_mma_kernel<C>, smem_tf_mma), 256, smem_tf_mma, s>>>(A, nmt);
      bb_launch_tally += 1;
      BB_LAUNCH_CHECK();
      return BB_OK;
    }
    const int grid = resident((const void*)cb_tf_kernel<C, PT>, smem_tf);
    cb_tf_kernel<C, PT><<<grid, NT, smem_tf, s>>>(A);
    bb_launch_tally += 1;
    BB_LAUNCH_CHECK();
    return BB_OK;
  }
  if (mma) {
    const int mma_grid = mma_blocks((const void*)cb_reduce_mma_kernel<C, false>, 0);
    A.nparts = mma_grid;
    cb_reduce_mma_kernel<C, false><<<mma_grid, 256, 0, s>>>(A, nmt);
  } else {
    const int grid = resident((const void*)cb_reduce_kernel<C, false, PT>, smem_red);
    A.nparts = grid;
    cb_reduce_kernel<C, false, PT><<<grid, NT, smem_red, s>>>(A);
  }
  cb_finish_kernel<false><<<g.O, 64, 0, s>>>(A, C * 9);
  bb_launch_tally += 2;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace

// node layout (plan.py _n_convblock):
//   dims = N,C,H,W,O,KH,KW,HO,WO,sh,sw,ph,pw,HP,WP,relu      f[0] = eps
//   slot 0 = W (t, at), slot 1 = conv bias (t, at; may be 0), slot 2 = gamma (base = fp32 values; t, at; may be 0)
//   slot 3 = pooled output q (base, t, a, at)
//   base[0] = x (dt[0]), base[1] = y = conv output (dt[1])
//   aux[0] = workspace (bb_convblock_ws_bytes), aux[1] = t_beta, aux[2] = at_beta, aux[3] = int64 arg-max indices
int bb_launch_convblock(const bb_node& nd, int pass, cudaStream_t s) {
  CbArgs A{};
  A.g = make_geom(nd);
  if (nd.dims[5] != 3 || nd.dims[6] != 3 || A.g.O > MAXO || (A.g.C != 1 && A.g.C != 3)) return BB_ERR_UNSUPPORTED;
  A.w = cb_layout(nd.aux[0], A.g);
  A.x = nd.base[0]; A.dtx = nd.dt[0];
  A.y = nd.base[1]; A.dty = nd.dt[1];
  A.q = nd.base[3]; A.dtq = nd.dt[3];
  A.idx = reinterpret_cast<const int64_t*>(nd.aux[3]);
  A.gamma = reinterpret_cast<const float*>(nd.base[2]);
  A.eps = (float)nd.f[0];
  A.t_W = reinterpret_cast<const float*>(nd.t[0]); A.at_W = reinterpret_cast<float*>(nd.at[0]);
  A.t_b = reinterpret_cast<const float*>(nd.t[1]); A.at_b = reinterpret_cast<float*>(nd.at[1]);
  A.t_gamma = reinterpret_cast<const float*>(nd.t[2]); A.at_gamma = reinterpret_cast<float*>(nd.at[2]);
  A.t_beta = reinterpret_cast<const float*>(nd.aux[1]); A.at_beta = reinterpret_cast<float*>(nd.aux[2]);
  // kind bit 2: the pooled tangent is the next fused block's bf16 padded-NHWC operand ([N][HP+2][WP+2][64], O == 64)
  const bool tq_nhwc = (nd.kind & 4) && A.g.O == 64;
  A.t_q = tq_nhwc ? nullptr : reinterpret_cast<float*>(nd.t[3]);
  A.tq_nhwc = tq_nhwc ? reinterpret_cast<__nv_bfloat16*>(nd.t[3]) : nullptr;
  // kind bit 3: a_q / at_q arrive as bf16 padded NHWC too (written by the next fused block's input-gradient epilogue)
  const bool adj_nhwc = (nd.kind & 8) && A.g.O == 64;
  A.a_q = adj_nhwc ? nullptr : reinterpret_cast<const float*>(nd.a[3]);
  A.at_q = adj_nhwc ? nullptr : reinterpret_cast<const float*>(nd.at[3]);
  A.aq_nhwc = adj_nhwc ? reinterpret_cast<const __nv_bfloat16*>(nd.a[3]) : nullptr;
  A.atq_nhwc = adj_nhwc ? reinterpret_cast<const __nv_bfloat16*>(nd.at[3]) : nullptr;
  if (A.g.ps == 2) return A.g.C == 1 ? run<1, __nv_bfloat16>(A, pass, s) : run<3, __nv_bfloat16>(A, pass, s);
  return A.g.C == 1 ? run<1, float>(A, pass, s) : run<3, float>(A, pass, s);
}

extern "C" int64_t bb_convblock_ws_bytes(int N, int C, int H, int W, int O, int HO, int WO, int HP, int WP) {
  CbGeom g{};
  g.ps = 4;    // upper bound (fp32 pooled arrays)
  g.N = N; g.C = C; g.H = H; g.W = W; g.O = O; g.HO = HO; g.WO = WO; g.HP = HP; g.WP = WP;
  return (int64_t)cb_layout(nullptr, g).bytes;
}
