// K6, small-channel convolutions (LeNet-class), second generation of conv_small.cu (which stays as the fallback for
// geometries these kernels decline).  Exact fp32 on the FMA pipe: the 1e-4 parity bar rules out single-pass TF32 and
// these layers (<= 16 channels) are FMA-bound, not HBM-bound -- LeNet B=4096 needs 10.3 G multiply-adds per K-loop
// iteration against 0.72 GB of HBM traffic (SURVEY 8d bytes).  The first-generation kernels issue a shared-memory or
// global load for every 2.5 ... 5 FMAs and do 2x zero-padding work in the data-gradient form.
//
//   conv_small_corr2_kernel   out[n,co,y,x] = sum_p sum_{ci,i,j} in_p[n,ci,y-ph+i,x-pw+j] * w_p(co,ci,i,j)  (+bias)
//       (forward and data-gradient indexing as in conv_small.cu).  A warp owns ONE output row y of IMGS images: lane =
//       (image, x-group of PX pixels); the input rows of the block's images are staged in shared memory with zero
//       column padding, so the inner loop has no predicates, no 64-bit address arithmetic and no global loads, and the
//       rows a data-gradient output does not touch (y-ph+i outside the image) are skipped warp-uniformly.  Per (ci, i):
//       PX+KW-1 input words + KW * CO/4 weight vectors (broadcast) feed PX*KW*CO FMAs (10 ... 14 FMAs per load).
//   conv_small_wgrad2_kernel  dW[o,c,i,j] += sum_p sum_{n,y,x} g_p[n,o,y,x] * in_p[n,c,y-ph+i,x-pw+j]
//       A thread owns (block of OB output channels, c, i) x KW taps = OB*KW accumulators; g is staged channels-last so
//       the OB values of a pixel are one vector load, the input row slides through a register window: 2 loads per
//       OB*KW FMAs (10:1; first generation 2.5:1).  Each block writes its sum over its images as one partial; the
//       partials are added onto dW in block order, so the result does not depend on which block finishes first.
#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "conv_small.h"
#include "gemm_tma.h"   // BB_DECLINED
#include "plan.h"
#include "tma.h"
#include <stdlib.h>

namespace {

// ---- asynchronous staging (cp.async, 4-byte granules; src_size 0 = zero fill) -------------------------------------
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct Corr2Geom {
  int XG, IMGS, RY, RS, CIC, pitch, S, nbuf, VW, bands, groups;
  // x-groups per row, images per unit, output rows per unit, staged rows (max over the bands), channel chunk, staged row
  // pitch, image stride (floats), staging buffers, staging vector width (floats), row bands, image groups
};

template <int VW>
__device__ __forceinline__ void cp_async_vec(float* smem_dst, const float* gsrc, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 4 * VW : 0;
  if (VW == 4) asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
  else if (VW == 2) asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
  else asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}

// accumulator-heavy instantiations (16 channels x 5 pixels) run with at most 12 warps so that ptxas may use 170 registers
template <int CO_T, int PX>
constexpr int corr2_max_threads() { return CO_T * PX > 64 ? 384 : 512; }

// Persistent: a block walks work units u = blockIdx.x, +gridDim.x, ...; unit = (image group, row band).  The stages of
// all its units -- (unit, operand pair, channel chunk) -- form one sequence that is double buffered: while stage k is
// being computed the cp.asyncs of stage k+1 (possibly the next unit's images) are in flight.  The weights are staged once.
template <int OP, int KW, int CO_T, int PX>
__global__ void __launch_bounds__(corr2_max_threads<CO_T, PX>()) conv_small_corr2_kernel(const __grid_constant__ SmallConvArgs A,
                                                                const __grid_constant__ Corr2Geom G) {
  extern __shared__ float sm2[];
  const int K = A.CI * A.KH * KW;
  float* wsm = sm2;                                  // [npairs][K][OP]
  float* xs = sm2 + ((A.npairs * K * OP + 3) & ~3);  // nbuf x [IMGS][CIC][RS][pitch] (image stride S)
  for (int e = threadIdx.x; e < A.npairs * K * OP; e += blockDim.x) {
    const int co = e % OP, k = (e / OP) % K, p = e / (OP * K);
    float v = 0.f;
    if (co < A.CO) {
      const int ci = k / (A.KH * KW), r = k - ci * (A.KH * KW), i = r / KW, j = r - i * KW;
      int64_t idx;
      if (A.mode == 0) idx = (((int64_t)co * A.C_orig + ci) * A.KH + i) * KW + j;
      else idx = (((int64_t)ci * A.C_orig + co) * A.KH + (A.KH - 1 - i)) * KW + (KW - 1 - j);
      v = bb::ldf(A.w[p], idx, A.dt_w[p]);
    }
    wsm[e] = v;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int img_l = lane / G.XG, xg = lane - img_l * G.XG;
  const int x0 = xg * PX;
  constexpr int NV = PX + KW - 1;
  const int nchunks = (A.CI + G.CIC - 1) / G.CIC;
  const int nstages = A.npairs * nchunks;            // stages per unit
  const int bufsz = G.IMGS * G.S;
  const int units = G.groups * G.bands;
  const int my_units = units > (int)blockIdx.x ? (units - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  const int total = my_units * nstages;
  const int vpl = G.pitch / G.VW;                    // vectors per staged row

  // geometry of unit k of this block
  auto unit_geom = [&](int k, int& grp, int& y0, int& r0, int& rs) {
    const int u = (int)blockIdx.x + k * (int)gridDim.x;
    grp = u / G.bands;
    y0 = (u - grp * G.bands) * G.RY;
    r0 = max(y0 - A.ph, 0);     // input rows the band touches: [r0, r0 + rs), clipped to the image
    rs = min(y0 + G.RY - 1 - A.ph + A.KH - 1, A.H - 1) - r0 + 1;
  };

  // issue the copies of global stage gst into buffer b; nothing waits here
  auto stage = [&](int gst, int b) {
    const int k = gst / nstages, st = gst - k * nstages;
    int grp, y0, r0, rs;
    unit_geom(k, grp, y0, r0, rs);
    const int p = st / nchunks, c0 = (st - p * nchunks) * G.CIC;
    const int cic = min(G.CIC, A.CI - c0);
    const int imgs_here = (int)min((int64_t)G.IMGS, A.N - (int64_t)grp * G.IMGS);
    float* buf = xs + b * bufsz;
    const float* src0 = reinterpret_cast<const float*>(A.in[p]);
    const bool f32 = A.dt_in[p] == BB_F32;
    const int nvec = imgs_here * cic * rs * vpl;
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
      const int ln = v / vpl, pc = (v - ln * vpl) * G.VW;
      const int r = ln % rs, t = ln / rs, cl = t % cic, im = t / cic;
      const int64_t base = ((((int64_t)grp * G.IMGS + im) * A.CI + c0 + cl) * A.H + (r0 + r)) * A.W;
      float* dst = buf + im * G.S + (cl * G.RS + r) * G.pitch + pc;
      const int col = pc - A.pw;
      const bool ok = col >= 0 && col < A.W;          // a vector is entirely inside or outside (VW divides pw and W)
      if (f32) {
        const float* src = ok ? src0 + base + col : src0;
        if (G.VW == 4) cp_async_vec<4>(dst, src, ok);
        else if (G.VW == 2) cp_async_vec<2>(dst, src, ok);
        else cp_async_vec<1>(dst, src, ok);
      } else {
        for (int q = 0; q < G.VW; ++q) dst[q] = ok ? bb::ldf(A.in[p], base + col + q, A.dt_in[p]) : 0.f;
      }
    }
    cp_async_commit();
  };

  float acc[CO_T][PX];
  if (total > 0) stage(0, 0);
  for (int gst = 0; gst < total; ++gst) {
    const int b = G.nbuf == 2 ? (gst & 1) : 0;
    if (G.nbuf == 2 && gst + 1 < total) {
      stage(gst + 1, b ^ 1);         // prefetch the next stage while this one is computed
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int k = gst / nstages, st = gst - k * nstages;
    int grp, y0, r0, rs;
    unit_geom(k, grp, y0, r0, rs);
    const int y = y0 + warp;
    const int64_t n = (int64_t)grp * G.IMGS + img_l;
    const bool active = img_l < G.IMGS && n < A.N && warp < G.RY && y < A.HO;
    if (st == 0) {
#pragma unroll
      for (int o = 0; o < CO_T; ++o)
#pragma unroll
        for (int q = 0; q < PX; ++q) acc[o][q] = 0.f;
    }
    if (active) {
      const int p = st / nchunks, c0 = (st - p * nchunks) * G.CIC;
      const int cic = min(G.CIC, A.CI - c0);
      const float* wp = wsm + (int64_t)p * K * OP;
      const float* img = xs + b * bufsz + img_l * G.S + x0;
      for (int cl = 0; cl < cic; ++cl) {
        for (int i = 0; i < A.KH; ++i) {
          const int hy = y - A.ph + i;
          if (hy < 0 || hy >= A.H) continue;                  // warp-uniform: all lanes share y
          const float* src = img + (cl * G.RS + (hy - r0)) * G.pitch;
          float v[NV];
#pragma unroll
          for (int q = 0; q < NV; ++q) v[q] = src[q];
          const float* wr = wp + (((c0 + cl) * A.KH + i) * KW) * OP;
#pragma unroll
          for (int j = 0; j < KW; ++j) {
#pragma unroll
            for (int o = 0; o < OP; o += 4) {
              if (o >= CO_T) break;
              float w4[4];
              if (o + 4 <= CO_T) {
                const float4 t4 = *reinterpret_cast<const float4*>(wr + j * OP + o);
                w4[0] = t4.x; w4[1] = t4.y; w4[2] = t4.z; w4[3] = t4.w;
              } else {
                const float2 t2 = *reinterpret_cast<const float2*>(wr + j * OP + o);
                w4[0] = t2.x; w4[1] = t2.y; w4[2] = 0.f; w4[3] = 0.f;
                if (o + 2 < CO_T) w4[2] = wr[j * OP + o + 2];
              }
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                if (o + u < CO_T) {
#pragma unroll
                  for (int q = 0; q < PX; ++q) acc[o + u][q] = fmaf(v[q + j], w4[u], acc[o + u][q]);
                }
              }
            }
          }
        }
      }
      if (st == nstages - 1) {
#pragma unroll
        for (int o = 0; o < CO_T; ++o) {
          if (o >= A.CO) break;
          const float bv = A.bias ? A.bias[o] : 0.f;
          float* dst = A.out + ((n * A.CO + o) * A.HO + y) * A.WO + x0;
#pragma unroll
          for (int q = 0; q < PX; ++q) {
            if (x0 + q < A.WO) dst[q] = A.beta ? dst[q] + acc[o][q] + bv : acc[o][q] + bv;
          }
        }
      }
    }
    if (G.nbuf == 1 && gst + 1 < total) {
      __syncthreads();
      stage(gst + 1, 0);
    } else if (gst + 2 < total) {
      __syncthreads();               // buffer b is overwritten by the prefetch issued in the next iteration
    }
  }
}

struct Wgrad2Geom {
  int OPs, gp, ip, iplane, OG, tasks, ns;   // padded channel count of the staged g, its row pitch, input row pitch / plane,
                                            // channel groups, tasks = OG*C*KH, row slices per task
};

template <int KW, int OB>
__global__ void __launch_bounds__(256) conv_small_wgrad2_kernel(const __grid_constant__ SmallConvArgs A,
                                                                 const __grid_constant__ Wgrad2Geom G) {
  extern __shared__ float sm3[];
  const int O = A.CO, C = A.CI;
  const int bufsz = (A.HO * G.gp + C * G.iplane + 3) & ~3;   // one staged (image, pair): gs [HO][gp] pixel-major, channels
                                                             // last | is [C][iplane], rows of pitch ip
  const int t = threadIdx.x;
  const int task = t % G.tasks, slice = t / G.tasks;
  const bool live = slice < G.ns;
  const int og = task / (C * A.KH), tc = (task / A.KH) % C, ti = task % A.KH;
  float acc[OB][KW];
#pragma unroll
  for (int o = 0; o < OB; ++o)
#pragma unroll
    for (int j = 0; j < KW; ++j) acc[o][j] = 0.f;
  const int HWo = A.HO * A.WO, gsz = O * HWo, HWi = A.H * A.W, isz = C * HWi;
  // the padding channels (o >= O) of both buffers are never staged: zero them once
  for (int e = t; e < 2 * bufsz; e += blockDim.x) sm3[e] = 0.f;
  __syncthreads();

  // stage image n, pair p into buffer b.  g[n][o][y][x] -> gs[y][x][o]: the threads run along the pixels of one channel
  // plane (coalesced global reads), every element is one 4-byte cp.async; indices advance without divisions.
  auto stage = [&](int64_t n, int p, int b) {
    float* gs = sm3 + b * bufsz;
    float* is = gs + A.HO * G.gp;
    const bool gf32 = A.dt_g[p] == BB_F32, if32 = A.dt_in[p] == BB_F32;
    const float* gsrc = reinterpret_cast<const float*>(A.g[p]) + n * gsz;
    const float* isrc = reinterpret_cast<const float*>(A.in[p]) + n * isz;
    {
      int yy = t / A.WO, xx = t - yy * A.WO;
      const int dy = (int)blockDim.x / A.WO, dx = (int)blockDim.x - dy * A.WO;
      for (int px = t; px < HWo; px += blockDim.x) {
        float* dst = gs + yy * G.gp + xx * G.OPs;
        for (int o = 0; o < O; ++o) {
          if (gf32) cp_async4(dst + o, gsrc + (int64_t)o * HWo + px, true);
          else dst[o] = bb::ldf(A.g[p], n * gsz + (int64_t)o * HWo + px, A.dt_g[p]);
        }
        xx += dx; yy += dy;
        if (xx >= A.WO) { xx -= A.WO; ++yy; }
      }
    }
    {
      int yy = t / A.W, xx = t - yy * A.W;
      const int dy = (int)blockDim.x / A.W, dx = (int)blockDim.x - dy * A.W;
      for (int px = t; px < HWi; px += blockDim.x) {
        float* dst = is + yy * G.ip + xx;
        for (int c = 0; c < C; ++c) {
          if (if32) cp_async4(dst + c * G.iplane, isrc + (int64_t)c * HWi + px, true);
          else dst[c * G.iplane] = bb::ldf(A.in[p], n * isz + (int64_t)c * HWi + px, A.dt_in[p]);
        }
        xx += dx; yy += dy;
        if (xx >= A.W) { xx -= A.W; ++yy; }
      }
    }
    cp_async_commit();
  };

  // work items of this block: (image, pair) pairs, double buffered
  const int64_t nimg = A.N > blockIdx.x ? (A.N - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const int64_t items = nimg * A.npairs;
  if (items > 0) stage(blockIdx.x, 0, 0);
  for (int64_t it = 0; it < items; ++it) {
    const int b = (int)(it & 1);
    if (it + 1 < items) {
      const int64_t nx = (it + 1) / A.npairs;
      stage(blockIdx.x + nx * gridDim.x, (int)(it + 1 - nx * A.npairs), b ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* gs = sm3 + b * bufsz;
    const float* is = gs + A.HO * G.gp;
    if (live) {
      for (int y = slice; y < A.HO; y += G.ns) {
        const int hy = y - A.ph + ti;
        if (hy < 0 || hy >= A.H) continue;
        const float* grow = gs + y * G.gp + og * OB;
        const float* irow = is + tc * G.iplane + hy * G.ip;
        float win[KW + 3];
#pragma unroll
        for (int j = 0; j < KW - 1; ++j) {
          const int xx = j - A.pw;
          win[j] = (xx >= 0 && xx < A.W) ? irow[xx] : 0.f;
        }
        int x = 0;
        for (; x + 4 <= A.WO; x += 4) {
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int xx = x + u + KW - 1 - A.pw;
            win[KW - 1 + u] = (xx >= 0 && xx < A.W) ? irow[xx] : 0.f;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            float gv[OB];
            const float* gpx = grow + (x + u) * G.OPs;
            if (OB % 4 == 0) {
#pragma unroll
              for (int o = 0; o < OB; o += 4) {
                const float4 t4 = *reinterpret_cast<const float4*>(gpx + o);
                gv[o] = t4.x; gv[o + 1] = t4.y; gv[o + 2] = t4.z; gv[o + 3] = t4.w;
              }
            } else {
#pragma unroll
              for (int o = 0; o < OB; o += 2) {
                const float2 t2 = *reinterpret_cast<const float2*>(gpx + o);
                gv[o] = t2.x; gv[o + 1] = t2.y;
              }
            }
#pragma unroll
            for (int o = 0; o < OB; ++o)
#pragma unroll
              for (int j = 0; j < KW; ++j) acc[o][j] = fmaf(gv[o], win[u + j], acc[o][j]);
          }
#pragma unroll
          for (int j = 0; j < KW - 1; ++j) win[j] = win[j + 4];
        }
        for (; x < A.WO; ++x) {   // tail
          const int xx = x + KW - 1 - A.pw;
          win[KW - 1] = (xx >= 0 && xx < A.W) ? irow[xx] : 0.f;
          const float* gpx = grow + x * G.OPs;
#pragma unroll
          for (int o = 0; o < OB; ++o) {
            const float gvo = gpx[o];
#pragma unroll
            for (int j = 0; j < KW; ++j) acc[o][j] = fmaf(gvo, win[j], acc[o][j]);
          }
#pragma unroll
          for (int j = 0; j < KW - 1; ++j) win[j] = win[j + 1];
        }
      }
    }
    if (it + 2 < items) __syncthreads();   // buffer b is refilled by the prefetch of the next iteration
  }
  // fixed-order finish: the ns row slices of each task are added in slice order through the staging memory, which is
  // idle now, and the block writes its partial dW[O][C][KH][KW] to A.part[blockIdx.x]
  float* red = sm3;   // [ns][tasks][OB][KW]
  __syncthreads();
  if (live) {
#pragma unroll
    for (int o = 0; o < OB; ++o)
#pragma unroll
      for (int j = 0; j < KW; ++j) red[((slice * G.tasks + task) * OB + o) * KW + j] = acc[o][j];
  }
  __syncthreads();
  float* dst = A.part + (int64_t)blockIdx.x * O * C * A.KH * KW;
  const int per_slice = G.tasks * OB * KW;
  for (int e = t; e < per_slice; e += blockDim.x) {
    const int tk = e / (OB * KW), r = e - tk * (OB * KW), o = r / KW, j = r - o * KW;
    const int oo = (tk / (C * A.KH)) * OB + o;
    if (oo >= O) continue;
    float v = red[e];
    for (int sl = 1; sl < G.ns; ++sl) v += red[sl * per_slice + e];
    dst[(((int64_t)oo * C + (tk / A.KH) % C) * A.KH + tk % A.KH) * KW + j] = v;
  }
}

// ---- host side --------------------------------------------------------------------------------------------------
constexpr int kCorr2SmemCap = 216 * 1024;   // one block per SM, double-buffered staging

bool corr2_plan(const SmallConvArgs& A, int OP, int& PX, Corr2Geom& G, size_t& smem) {
  if (A.HO < 1 || A.WO < 1) return false;
  const int cands[3] = {7, 5, 4};
  int best = 0;
  double best_cost = 1e30;
  const char* force = getenv("BB200_CORR2_PX");       // tuning: force the pixels-per-lane choice
  for (int c = 0; c < 3; ++c) {
    const int px = cands[c];
    if (force && atoi(force) != px) continue;
    if (OP * px > 80 && !(OP == 8 && px == 7)) continue;   // accumulator registers: CO_T * PX <= 80 (6 x 7, 8 x 7 allowed)
    const int xg = (A.WO + px - 1) / px;
    if (xg > 32) continue;
    const int imgs = 32 / xg;
    const double cost = (double)xg * px / A.WO * 32.0 / (imgs * xg);   // padded columns x idle lanes
    if (cost < best_cost - 1e-9) { best_cost = cost; best = px; }
  }
  if (!best) return false;
  PX = best;
  G.XG = (A.WO + PX - 1) / PX;
  G.IMGS = 32 / G.XG;
  if ((int64_t)G.IMGS > A.N) G.IMGS = (int)A.N;
  const int maxw = (OP * PX > 64 ? 384 : 512) / 32;    // == corr2_max_threads / 32 (CO_T * PX > 64 only for OP = 16)
  const int nb = (A.HO + maxw - 1) / maxw;
  G.RY = (A.HO + nb - 1) / nb;                         // equal bands of <= maxw rows
  G.RS = G.RY + A.KH - 1 < A.H ? G.RY + A.KH - 1 : A.H;   // a band never needs more rows than the image has
  G.pitch = G.XG * PX + A.KW - 1;
  // staging vector width: columns [-pw, 0) and [W, ...) are zero fill, so a vector must not straddle those borders
  G.VW = 1;
  if (A.W % 2 == 0 && A.pw % 2 == 0) G.VW = 2;
  if (A.W % 4 == 0 && A.pw % 4 == 0) G.VW = 4;
  for (int p = 0; p < A.npairs; ++p)
    if (reinterpret_cast<uintptr_t>(A.in[p]) % 16) G.VW = 1;
  if (getenv("BB200_CORR2_VW1")) G.VW = 1;
  G.pitch = (G.pitch + G.VW - 1) / G.VW * G.VW;
  G.bands = (A.HO + G.RY - 1) / G.RY;
  G.groups = (int)((A.N + G.IMGS - 1) / G.IMGS);
  const size_t wbytes = sizeof(float) * (((size_t)A.npairs * A.CI * A.KH * A.KW * OP + 3) & ~(size_t)3);
  for (int cic = A.CI; cic >= 1; --cic) {
    int S = cic * G.RS * G.pitch;
    // image stride residue mod 32 that spreads (image, x-group) lanes over the banks
    int best_s = 0, best_conf = 1 << 30;
    for (int s = 0; s < 32; ++s) {
      int cnt[32] = {0}, conf = 0;
      for (int l = 0; l < G.IMGS * G.XG; ++l) conf += cnt[((l / G.XG) * s + (l % G.XG) * PX) & 31]++;
      if (conf < best_conf) { best_conf = conf; best_s = s; }
    }
    // image stride: multiple of the staging vector width, residue (mod 32) as close to the conflict-free one as that allows
    S += ((best_s - S) % 32 + 32) % 32;
    S = (S + G.VW - 1) / G.VW * G.VW;
    const int nbuf = 2;
    const size_t bytes = wbytes + sizeof(float) * (size_t)nbuf * G.IMGS * S;
    if (bytes <= (size_t)kCorr2SmemCap) {
      G.CIC = cic;
      G.S = S;
      G.nbuf = nbuf;
      smem = bytes;
      return true;
    }
  }
  return false;
}

int corr2_grid(const Corr2Geom& G) {
  const int units = G.groups * G.bands;
  return units < BB_SM_COUNT ? units : BB_SM_COUNT;     // one persistent block per SM
}

template <int OP, int KW, int CO_T, int PX>
int launch_corr2(const SmallConvArgs& A, const Corr2Geom& G, size_t smem, cudaStream_t s) {
  static BbOncePerDevice configured;
  if (configured.need())
    BB_CUDA_TRY(cudaFuncSetAttribute(conv_small_corr2_kernel<OP, KW, CO_T, PX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     kCorr2SmemCap));
  const int grid = corr2_grid(G);
  conv_small_corr2_kernel<OP, KW, CO_T, PX><<<grid, G.RY * 32, smem, s>>>(A, G);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

template <int OP, int KW, int CO_T>
int dispatch_px(const SmallConvArgs& A, int PX, const Corr2Geom& G, size_t smem, cudaStream_t s) {
  if (PX == 4) return launch_corr2<OP, KW, CO_T, 4>(A, G, smem, s);
  if (PX == 5) return launch_corr2<OP, KW, CO_T, 5>(A, G, smem, s);
  if constexpr (OP == 8) {
    if (PX == 7) return launch_corr2<OP, KW, CO_T, 7>(A, G, smem, s);
  }
  return BB_DECLINED;
}

constexpr int kWgrad2SmemCap = 100 * 1024;

bool wgrad2_plan(const SmallConvArgs& A, int OB, Wgrad2Geom& G, size_t& smem) {
  const int O = A.CO, C = A.CI;
  G.OG = (O + OB - 1) / OB;
  G.OPs = (G.OG * OB + 3) & ~3;
  G.tasks = G.OG * C * A.KH;
  if (G.tasks > 256 || G.tasks < 1) return false;
  // with few tasks per image (LeNet conv1: 15) a block needs ~17 row slices and its per-image barriers dominate -- the
  // first-generation kernel is faster there
  if (G.tasks < 64 && !getenv("BB200_WGRAD2_ALWAYS")) return false;
  G.ns = 256 / G.tasks;
  if (G.ns > A.HO) G.ns = A.HO;
  {   // fewest slices with the same maximum of rows per slice: every slice gets (nearly) the same work between barriers
    const int rows = (A.HO + G.ns - 1) / G.ns;
    G.ns = (A.HO + rows - 1) / rows;
  }
  const int row = A.WO * G.OPs;
  G.gp = row + (((G.OPs - row) % 32) + 32) % 32;      // gp mod 32 == OPs mod 32: the row slices of a warp hit distinct banks
  G.ip = A.W | 1;
  G.iplane = (A.H * G.ip) | 1;
  smem = sizeof(float) * 2 * (((size_t)A.HO * G.gp + (size_t)C * G.iplane + 3) & ~(size_t)3);   // double buffered
  const size_t red = sizeof(float) * (size_t)G.ns * G.tasks * OB * A.KW;   // slice sums of the finish
  if (smem < red) smem = red;
  return smem <= (size_t)kWgrad2SmemCap;
}

int wgrad2_grid(const SmallConvArgs& A, size_t smem) {
  int per_sm = (int)((200 * 1024) / (smem + 1024));
  if (per_sm > 6) per_sm = 6;
  if (per_sm < 1) per_sm = 1;
  int grid = BB_SM_COUNT * per_sm;
  if (grid > A.N) grid = A.N;
  const size_t n = (size_t)A.CO * A.CI * A.KH * A.KW;
  if (bb_reduce_ws.base != nullptr) grid = bb_reduce_ws_splits(grid, sizeof(float) * n);   // a plan never allocates
  return grid;
}

template <int KW, int OB>
int launch_wgrad2(const SmallConvArgs& A, const Wgrad2Geom& G, size_t smem, cudaStream_t s) {
  static BbOncePerDevice configured;
  if (configured.need())
    BB_CUDA_TRY(cudaFuncSetAttribute(conv_small_wgrad2_kernel<KW, OB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     kWgrad2SmemCap));
  const int grid = wgrad2_grid(A, smem);
  const int64_t n = (int64_t)A.CO * A.CI * A.KH * A.KW;
  bool owned = false;
  SmallConvArgs B = A;
  if ((B.part = bb_partials_acquire(sizeof(float) * grid * n, s, &owned)) == nullptr) return cudaErrorMemoryAllocation;
  conv_small_wgrad2_kernel<KW, OB><<<grid, 256, smem, s>>>(B, G);
  bb_launch_tally += 1;
  int rc = (int)cudaPeekAtLastError();
  if (rc == BB_OK) rc = bb_partials_reduce_lanes(B.part, grid, n, A.out, s);
  bb_partials_release(B.part, owned, s);
  return rc;
}

int pick_ob(int O) { return O % 4 == 0 || O > 6 ? 4 : (O <= 2 ? 2 : 6); }

bool corr2_setup(const SmallConvArgs& A, int& OP, int& PX, Corr2Geom& G, size_t& smem) {
  if (A.CO > 16 || (A.KW != 3 && A.KW != 5) || A.HO > 512) return false;
  OP = A.CO <= 8 ? 8 : 16;
  return corr2_plan(A, OP, PX, G, smem);
}

}  // namespace

bool bb_conv_small_corr2_geometry(const SmallConvArgs& A, int64_t* geo) {
  int OP = 0, PX = 0;
  Corr2Geom G{};
  size_t smem = 0;
  if (!corr2_setup(A, OP, PX, G, smem)) return false;
  const int64_t v[10] = {corr2_grid(G), (int64_t)G.groups * G.bands, PX, G.IMGS, G.RY, G.bands, G.CIC,
                         (int64_t)A.npairs * ((A.CI + G.CIC - 1) / G.CIC), G.VW, G.groups};
  for (int i = 0; i < 10; ++i) geo[i] = v[i];
  return true;
}

bool bb_conv_small_wgrad2_geometry(const SmallConvArgs& A, int64_t* geo) {
  if (A.KW != 3 && A.KW != 5) return false;
  const int OB = pick_ob(A.CO);
  Wgrad2Geom G{};
  size_t smem = 0;
  if (!wgrad2_plan(A, OB, G, smem)) return false;
  const int64_t v[5] = {wgrad2_grid(A, smem), OB, G.tasks, G.ns, (int64_t)A.CO * A.CI * A.KH * A.KW};
  for (int i = 0; i < 5; ++i) geo[i] = v[i];
  return true;
}

int bb_conv_small_corr2(const SmallConvArgs& A, cudaStream_t s) {
  int OP = 0, PX = 0;
  Corr2Geom G{};
  size_t smem = 0;
  if (!corr2_setup(A, OP, PX, G, smem)) return BB_DECLINED;
  if (A.KW == 3) {
    if (A.CO == 6) return dispatch_px<8, 3, 6>(A, PX, G, smem, s);
    if (A.CO <= 8) return dispatch_px<8, 3, 8>(A, PX, G, smem, s);
    return dispatch_px<16, 3, 16>(A, PX, G, smem, s);
  }
  if (A.CO == 6) return dispatch_px<8, 5, 6>(A, PX, G, smem, s);
  if (A.CO <= 8) return dispatch_px<8, 5, 8>(A, PX, G, smem, s);
  return dispatch_px<16, 5, 16>(A, PX, G, smem, s);
}

int bb_conv_small_wgrad2(const SmallConvArgs& A, cudaStream_t s) {
  if (A.KW != 3 && A.KW != 5) return BB_DECLINED;
  const int OB = pick_ob(A.CO);
  Wgrad2Geom G{};
  size_t smem = 0;
  if (!wgrad2_plan(A, OB, G, smem)) return BB_DECLINED;
  if (A.KW == 3) {
    if (OB == 2) return launch_wgrad2<3, 2>(A, G, smem, s);
    if (OB == 4) return launch_wgrad2<3, 4>(A, G, smem, s);
    return launch_wgrad2<3, 6>(A, G, smem, s);
  }
  if (OB == 2) return launch_wgrad2<5, 2>(A, G, smem, s);
  if (OB == 4) return launch_wgrad2<5, 4>(A, G, smem, s);
  return launch_wgrad2<5, 6>(A, G, smem, s);
}
