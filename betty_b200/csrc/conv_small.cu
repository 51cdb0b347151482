// K6 fast path for small-channel convolutions (LeNet-class: <=16 output channels, stride 1, no dilation):
// direct kernels with the (dual) weights staged in shared memory and register tiling, instead of the
// generic implicit-GEMM tile kernel whose 64-wide tiles are mostly padding at 6/16 channels.
//
//   conv_small_corr_kernel   out[n,co,y,x] = sum_p sum_{ci,i,j} in_p[n,ci,y-ph+i,x-pw+j] * w_p(co,ci,i,j) (+bias)
//        mode FWD  : w(co,ci,i,j) = W[co][ci][i][j]                 -> tangent forward (dual: t_x*W + x*t_W)
//        mode DGRAD: w(co,ci,i,j) = W[ci][co][KH-1-i][KW-1-j], padding K-1-p
//                                                               -> a_x / at_x (dual: at_y*W + a_y*t_W)
//   conv_small_wgrad_kernel  dW[o,c,i,j] += sum_p sum_{n,y,x} g_p[n,o,y,x] * in_p[n,c,y-ph+i,x-pw+j]
//                                                               -> at_W (dual: at_y*x + a_y*t_x)
//        each block writes its sum over its images as one partial; the partials are added onto dW in block order
// Same maths as conv.cu (spec: oracle/plan_interp.py tf_conv2d/bb_conv2d/tb_conv2d).
#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "conv_small.h"
#include "plan.h"
#include "tma.h"

namespace {

constexpr int PX = 4;  // output pixels per thread along x

// OP = padded channel count of the shared-memory weight rows (8 / 16), CO_T = channels actually accumulated
// (compile time, so a 6-channel layer issues 6/8 of the FMAs), F32IN = every input map is fp32.
template <int OP, int KW, int CO_T, bool F32IN>
__global__ void __launch_bounds__(256, 2) conv_small_corr_kernel(const __grid_constant__ SmallConvArgs A) {
  extern __shared__ float wsm[];  // [npairs][K][OP], K = CI*KH*KW
  const int K = A.CI * A.KH * KW;
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
  __syncthreads();
  const int G = (A.WO + PX - 1) / PX;
  const int64_t total = (int64_t)A.N * A.HO * G;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int xg = (int)(gid % G);
  const int y = (int)((gid / G) % A.HO);
  const int n = (int)(gid / ((int64_t)G * A.HO));
  const int x0 = xg * PX;

  // column validity of the PX+KW-1 inputs this thread reads in every row: hoisted out of the channel / row loops
  // (a 0/1 multiplier and a clamped column instead of per-load predicates)
  constexpr int NV = PX + KW - 1;
  float fm[NV];
  int col[NV];
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    const int xx = x0 - A.pw + q;
    const bool ok = xx >= 0 && xx < A.W;
    fm[q] = ok ? 1.f : 0.f;
    col[q] = ok ? xx : 0;
  }

  float acc[OP][PX];
#pragma unroll
  for (int o = 0; o < OP; ++o)
#pragma unroll
    for (int q = 0; q < PX; ++q) acc[o][q] = 0.f;

  for (int p = 0; p < A.npairs; ++p) {
    const float* wp = wsm + (int64_t)p * K * OP;
    const float* inf = reinterpret_cast<const float*>(A.in[p]);
    for (int ci = 0; ci < A.CI; ++ci) {
      const int64_t plane = ((int64_t)n * A.CI + ci) * A.H;
      for (int i = 0; i < A.KH; ++i) {
        const int hy = y - A.ph + i;
        if (hy < 0 || hy >= A.H) continue;
        const int64_t rowb = (plane + hy) * A.W;
        float v[NV];
#pragma unroll
        for (int q = 0; q < NV; ++q) {
          if (F32IN) v[q] = inf[rowb + col[q]] * fm[q];
          else v[q] = bb::ldf(A.in[p], rowb + col[q], A.dt_in[p]) * fm[q];
        }
        const float* wr = wp + (int64_t)((ci * A.KH + i) * KW) * OP;
#pragma unroll
        for (int j = 0; j < KW; ++j) {
#pragma unroll
          for (int o = 0; o < OP; o += 4) {
            if (o >= CO_T) break;
            const float4 w4 = *reinterpret_cast<const float4*>(wr + j * OP + o);
#pragma unroll
            for (int q = 0; q < PX; ++q) {
              acc[o + 0][q] = fmaf(v[q + j], w4.x, acc[o + 0][q]);
              if (o + 1 < CO_T) acc[o + 1][q] = fmaf(v[q + j], w4.y, acc[o + 1][q]);
              if (o + 2 < CO_T) acc[o + 2][q] = fmaf(v[q + j], w4.z, acc[o + 2][q]);
              if (o + 3 < CO_T) acc[o + 3][q] = fmaf(v[q + j], w4.w, acc[o + 3][q]);
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int o = 0; o < OP; ++o) {
    if (o >= A.CO || o >= CO_T) break;
    const float b = A.bias ? A.bias[o] : 0.f;
    float* dst = A.out + (((int64_t)n * A.CO + o) * A.HO + y) * A.WO + x0;
#pragma unroll
    for (int q = 0; q < PX; ++q) {
      if (x0 + q < A.WO) dst[q] = A.beta ? dst[q] + acc[o][q] + b : acc[o][q] + b;
    }
  }
}

// One block walks images n = blockIdx.x, +gridDim.x, ...; per image and pair it stages g[n] (O x HO x WO)
// and in[n] (C x H x W) in shared memory.  A thread owns task (o, c, i) [+ a row slice] and keeps the KW
// partial sums of dW[o,c,i,:] in registers, sliding a KW-wide window along each input row.
template <int KW, int TPT>  // TPT = tasks per thread (1 or 2)
__global__ void __launch_bounds__(256) conv_small_wgrad_kernel(const __grid_constant__ SmallConvArgs A) {
  extern __shared__ float sm[];
  const int O = A.CO, C = A.CI;  // here CO = O (rows of dW), CI = C
  // odd row pitches: tasks of a warp read the same column of different rows/planes -- with W = 32 every
  // row would otherwise start in the same shared-memory bank
  const int gp = A.WO | 1, ip = A.W | 1;
  const int gplane = (A.HO * gp) | 1, iplane = (A.H * ip) | 1;
  const int gsz = O * A.HO * A.WO, isz = C * A.H * A.W;
  float* gs = sm;
  float* is = sm + O * gplane;
  const int tasks = O * C * A.KH;
  int ns = 1;
  if (TPT == 1) {
    ns = blockDim.x / tasks;
    if (ns < 1) ns = 1;
  }
  float acc[TPT][KW];
  int tk[TPT], to[TPT], tc[TPT], ti[TPT], slice[TPT];
  bool live[TPT];
#pragma unroll
  for (int u = 0; u < TPT; ++u) {
    const int t = threadIdx.x + u * blockDim.x;
    const int task = (TPT == 1) ? t % tasks : t;
    tk[u] = task;
    slice[u] = (TPT == 1) ? t / tasks : 0;
    live[u] = (TPT == 1) ? (slice[u] < ns) : (task < tasks);
    const int tt = live[u] ? task : 0;
    to[u] = tt / (C * A.KH);
    tc[u] = (tt / A.KH) % C;
    ti[u] = tt % A.KH;
#pragma unroll
    for (int j = 0; j < KW; ++j) acc[u][j] = 0.f;
  }
  for (int n = blockIdx.x; n < A.N; n += gridDim.x) {
    for (int p = 0; p < A.npairs; ++p) {
      __syncthreads();
      for (int e = threadIdx.x; e < gsz; e += blockDim.x) {
        const int pl = e / (A.HO * A.WO), r = e - pl * (A.HO * A.WO), yy = r / A.WO, xx = r - yy * A.WO;
        gs[pl * gplane + yy * gp + xx] = bb::ldf(A.g[p], (int64_t)n * gsz + e, A.dt_g[p]);
      }
      for (int e = threadIdx.x; e < isz; e += blockDim.x) {
        const int pl = e / (A.H * A.W), r = e - pl * (A.H * A.W), yy = r / A.W, xx = r - yy * A.W;
        is[pl * iplane + yy * ip + xx] = bb::ldf(A.in[p], (int64_t)n * isz + e, A.dt_in[p]);
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < TPT; ++u) {
        if (!live[u]) continue;
        for (int y = slice[u]; y < A.HO; y += ns) {
          const int hy = y - A.ph + ti[u];
          if (hy < 0 || hy >= A.H) continue;
          const float* grow = gs + to[u] * gplane + y * gp;
          const float* irow = is + tc[u] * iplane + hy * ip;
          // sliding window over the input row, 4 output pixels per step: win[u + j] = in[x + u + j - pw]
          float win[KW + 3];
#pragma unroll
          for (int j = 0; j < KW - 1; ++j) {
            const int xx = j - A.pw;
            win[j] = (xx >= 0 && xx < A.W) ? irow[xx] : 0.f;
          }
          int x = 0;
          for (; x + 4 <= A.WO; x += 4) {
            float gv[4];
#pragma unroll
            for (int u4 = 0; u4 < 4; ++u4) {
              const int xx = x + u4 + KW - 1 - A.pw;
              win[KW - 1 + u4] = (xx >= 0 && xx < A.W) ? irow[xx] : 0.f;
              gv[u4] = grow[x + u4];
            }
#pragma unroll
            for (int u4 = 0; u4 < 4; ++u4)
#pragma unroll
              for (int j = 0; j < KW; ++j) acc[u][j] = fmaf(gv[u4], win[u4 + j], acc[u][j]);
#pragma unroll
            for (int j = 0; j < KW - 1; ++j) win[j] = win[j + 4];
          }
          for (; x < A.WO; ++x) {   // tail
            const int xx = x + KW - 1 - A.pw;
            win[KW - 1] = (xx >= 0 && xx < A.W) ? irow[xx] : 0.f;
            const float gv = grow[x];
#pragma unroll
            for (int j = 0; j < KW; ++j) acc[u][j] = fmaf(gv, win[j], acc[u][j]);
#pragma unroll
            for (int j = 0; j < KW - 1; ++j) win[j] = win[j + 1];
          }
        }
      }
    }
  }
  // fixed-order finish: the row slices of each task are added in slice order through the staging memory, which is idle
  // now, and the block writes its partial dW (task (o, c, i) x KW taps is dW's own layout) to A.part[blockIdx.x]
  float* red = sm;   // [ns][tasks][KW]
  __syncthreads();
#pragma unroll
  for (int u = 0; u < TPT; ++u) {
    if (!live[u]) continue;
#pragma unroll
    for (int j = 0; j < KW; ++j) red[(slice[u] * tasks + tk[u]) * KW + j] = acc[u][j];
  }
  __syncthreads();
  float* dst = A.part + (int64_t)blockIdx.x * tasks * KW;
  for (int e = threadIdx.x; e < tasks * KW; e += blockDim.x) {
    float v = red[e];
    for (int sl = 1; sl < ns; ++sl) v += red[sl * tasks * KW + e];
    dst[e] = v;
  }
}

template <int OP, int KW, int CO_T>
int launch_corr(const SmallConvArgs& A, cudaStream_t s) {
  const int K = A.CI * A.KH * KW;
  const size_t smem = sizeof(float) * (size_t)A.npairs * K * OP;
  const int G = (A.WO + PX - 1) / PX;
  const int64_t total = (int64_t)A.N * A.HO * G;
  bool f32 = true;
  for (int p = 0; p < A.npairs; ++p) f32 = f32 && A.dt_in[p] == BB_F32;
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (f32) conv_small_corr_kernel<OP, KW, CO_T, true><<<grid, 256, smem, s>>>(A);
  else conv_small_corr_kernel<OP, KW, CO_T, false><<<grid, 256, smem, s>>>(A);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace

bool bb_conv_small_corr_ok(int CI, int CO, int KH, int KW, int npairs) {
  if (CO > 16 || (KW != 3 && KW != 5)) return false;
  const int OP = CO <= 8 ? 8 : 16;
  return sizeof(float) * (size_t)npairs * CI * KH * KW * OP <= 48 * 1024;
}

int bb_conv_small_corr(const SmallConvArgs& A, cudaStream_t s) {
  if (A.CO == 6) return A.KW == 3 ? launch_corr<8, 3, 6>(A, s) : launch_corr<8, 5, 6>(A, s);   // LeNet: 6 maps
  if (A.CO <= 8) return A.KW == 3 ? launch_corr<8, 3, 8>(A, s) : launch_corr<8, 5, 8>(A, s);
  return A.KW == 3 ? launch_corr<16, 3, 16>(A, s) : launch_corr<16, 5, 16>(A, s);
}

// staging of one image (g and input planes), and at least the [ns][tasks][KW] slice sums of the finish (<= 512 x 5)
static size_t wgrad_smem_bytes(int O, int C, int H, int W, int HO, int WO) {
  const size_t gplane = (size_t)(HO * (WO | 1)) | 1, iplane = (size_t)(H * (W | 1)) | 1;
  const size_t stage = sizeof(float) * (O * gplane + C * iplane), red = sizeof(float) * 512 * 5;
  return stage > red ? stage : red;
}

bool bb_conv_small_wgrad_ok(int O, int C, int H, int W, int HO, int WO, int KH, int KW) {
  if (KW != 3 && KW != 5) return false;
  if (O * C * KH > 512) return false;
  return wgrad_smem_bytes(O, C, H, W, HO, WO) <= 48 * 1024;
}

void bb_conv_small_wgrad_geometry(const SmallConvArgs& A, int64_t* geo) {
  const int64_t n = (int64_t)A.CO * A.CI * A.KH * A.KW;
  int grid = BB_SM_COUNT * 4;
  if (grid > A.N) grid = A.N;
  if (bb_reduce_ws.base != nullptr) grid = bb_reduce_ws_splits(grid, sizeof(float) * n);   // a plan never allocates
  geo[0] = grid;
  geo[1] = n;
}

int bb_conv_small_wgrad(const SmallConvArgs& A, cudaStream_t s) {
  const int tasks = A.CO * A.CI * A.KH;
  const size_t smem = wgrad_smem_bytes(A.CO, A.CI, A.H, A.W, A.HO, A.WO);
  int64_t geo[2];
  bb_conv_small_wgrad_geometry(A, geo);
  const int grid = (int)geo[0];
  bool owned = false;
  SmallConvArgs B = A;
  if ((B.part = bb_partials_acquire(sizeof(float) * grid * geo[1], s, &owned)) == nullptr) return cudaErrorMemoryAllocation;
  if (tasks <= 256) {
    if (A.KW == 3) conv_small_wgrad_kernel<3, 1><<<grid, 256, smem, s>>>(B);
    else conv_small_wgrad_kernel<5, 1><<<grid, 256, smem, s>>>(B);
  } else {
    if (A.KW == 3) conv_small_wgrad_kernel<3, 2><<<grid, 256, smem, s>>>(B);
    else conv_small_wgrad_kernel<5, 2><<<grid, 256, smem, s>>>(B);
  }
  bb_launch_tally += 1;
  int rc = (int)cudaPeekAtLastError();
  if (rc == BB_OK) rc = bb_partials_reduce_lanes(B.part, grid, geo[1], A.out, s);
  bb_partials_release(B.part, owned, s);
  return rc;
}
