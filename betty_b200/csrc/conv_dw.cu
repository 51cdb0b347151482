// Second-order rules of a depthwise Conv2d (groups == C_in == C_out, channel multiplier 1), NCHW fp32, any kernel size,
// stride, padding and dilation.  Conv2d's rules of SURVEY.md Appendix B, applied per channel:
//
//   TF  t_y  = dw(t_x, W) + dw(x, t_W) (+ t_b)
//   BB  a_x  = dwT(a_y, W)                       g_W  = sum_{n,yo,xo} a_y (x) x
//   TB  at_x = dwT(at_y, W) + dwT(a_y, t_W)       at_W = sum_{n,yo,xo} at_y (x) x + a_y (x) t_x
//
// (the bias terms are conv.cu's channel sums).  Spec: oracle/plan_interp.py tf_conv2d/bb_conv2d/tb_conv2d with groups.
//
// At the shapes depthwise convolutions run at (DARTS cells: 16..64 channels of 8x8..32x32 planes, 9 or 25 taps) every
// product is memory-bound.  A block owns one channel of a group of images and walks them one (image, channel) plane at a
// time: it stages the plane of each operand in shared memory -- inputs with their zero halo, so the tap loop has no
// bounds checks -- and computes every product of the pass from the staged planes, so each operand is read from global
// memory once per pass.  The data adjoint is a gather over the output windows covering each input pixel (no atomics).
// The weight gradient keeps per-thread tap sums across the block's images, closes them with a fixed-shape block
// reduction into one partial per (image group, channel) and adds the partials in image-group order with
// bb_partials_reduce: the result does not depend on scheduling.
#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "plan.h"
#include "tma.h"

namespace {

constexpr int kThreads = 128;
constexpr int kMaxTaps = 49;                 // KH*KW of the register tap sums of the weight gradient
constexpr size_t kMaxSmem = 160 * 1024;      // staged planes of one block

struct DwGeom {
  int N, C, H, W, KH, KW, HO, WO, sh, sw, ph, pw, dh, dw;
  int ipb;                                   // images per block
  __host__ __device__ int Hp() const { return H + 2 * ph; }
  __host__ __device__ int Wp() const { return W + 2 * pw; }
};

// Operands of one launch.  Forward: out = sum_p dw(in[p], w[p]) (+ bias).  Backward: dx (beta)= sum_p dwT(g[p], w[p]);
// weight-gradient partials of sum_p g[p] (x) xin[p].  A null pointer drops its term.
struct DwArgs {
  const float* in[2];
  const float* w[2];
  const float* bias;
  float* out;
  const float* g[2];
  const float* xin[2];
  float* dx;
  int beta_dx;
  float* part;                               // [image groups][C][KH*KW]
};

__device__ __forceinline__ void stage_padded(float* dst, const float* src, const DwGeom& g) {
  const int Wp = g.Wp(), n = g.Hp() * Wp;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int r = i / Wp - g.ph, c = i % Wp - g.pw;
    dst[i] = (r >= 0 && r < g.H && c >= 0 && c < g.W) ? src[r * g.W + c] : 0.f;
  }
}

__device__ __forceinline__ void stage_plain(float* dst, const float* src, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// grid (image groups, C)
__global__ void __launch_bounds__(kThreads) dw_fwd_kernel(DwArgs A, DwGeom g) {
  extern __shared__ float sm[];
  const int c = blockIdx.y, KK = g.KH * g.KW, Wp = g.Wp(), plane = g.Hp() * Wp;
  float* inS[2] = {sm, sm + plane};
  float* wS[2] = {sm + 2 * plane, sm + 2 * plane + KK};
  int* offS = reinterpret_cast<int*>(sm + 2 * plane + 2 * KK);
  for (int t = threadIdx.x; t < KK; t += blockDim.x) {
    offS[t] = (t / g.KW) * g.dh * Wp + (t % g.KW) * g.dw;
    for (int p = 0; p < 2; ++p)
      if (A.in[p]) wS[p][t] = A.w[p][(int64_t)c * KK + t];
  }
  const float b = A.bias ? A.bias[c] : 0.f;
  const int n0 = blockIdx.x * g.ipb, n1 = min(g.N, n0 + g.ipb), nout = g.HO * g.WO;
  for (int n = n0; n < n1; ++n) {
    const int64_t pl = (int64_t)n * g.C + c;
    __syncthreads();
    for (int p = 0; p < 2; ++p)
      if (A.in[p]) stage_padded(inS[p], A.in[p] + pl * g.H * g.W, g);
    __syncthreads();
    for (int o = threadIdx.x; o < nout; o += blockDim.x) {
      const int yo = o / g.WO, xo = o % g.WO;
      const int at = yo * g.sh * Wp + xo * g.sw;
      float acc = b;
      for (int p = 0; p < 2; ++p) {
        if (!A.in[p]) continue;
        const float* s = inS[p] + at;
        for (int t = 0; t < KK; ++t) acc += s[offS[t]] * wS[p][t];
      }
      A.out[pl * nout + o] = acc;
    }
  }
}

// grid (image groups, C).  KT >= KH*KW: register tap sums of the weight gradient.
template <int KT>
__global__ void __launch_bounds__(kThreads) dw_bwd_kernel(DwArgs A, DwGeom g) {
  extern __shared__ float sm[];
  const int c = blockIdx.y, KK = g.KH * g.KW, Wp = g.Wp(), plane = g.Hp() * Wp, nout = g.HO * g.WO;
  const bool wgrad = A.part != nullptr;
  float* gS[2] = {sm, sm + nout};
  float* xS[2] = {sm + 2 * nout, sm + 2 * nout + plane};
  float* wS[2] = {sm + 2 * nout + 2 * plane, sm + 2 * nout + 2 * plane + KK};
  int* offS = reinterpret_cast<int*>(sm + 2 * nout + 2 * plane + 2 * KK);
  __shared__ float red[kThreads / 32][KT];
  for (int t = threadIdx.x; t < KK; t += blockDim.x) {
    offS[t] = (t / g.KW) * g.dh * Wp + (t % g.KW) * g.dw;
    for (int p = 0; p < 2; ++p)
      if (A.dx && A.w[p]) wS[p][t] = A.w[p][(int64_t)c * KK + t];
  }
  bool useg[2];
  for (int p = 0; p < 2; ++p) useg[p] = A.g[p] && ((A.dx && A.w[p]) || (wgrad && A.xin[p]));
  float acc[KT];
#pragma unroll
  for (int t = 0; t < KT; ++t) acc[t] = 0.f;
  const int n0 = blockIdx.x * g.ipb, n1 = min(g.N, n0 + g.ipb);
  for (int n = n0; n < n1; ++n) {
    const int64_t pl = (int64_t)n * g.C + c;
    __syncthreads();
    for (int p = 0; p < 2; ++p) {
      if (useg[p]) stage_plain(gS[p], A.g[p] + pl * nout, nout);
      if (wgrad && A.xin[p]) stage_padded(xS[p], A.xin[p] + pl * g.H * g.W, g);
    }
    __syncthreads();
    if (A.dx) {
      float* dst = A.dx + pl * g.H * g.W;
      for (int i = threadIdx.x; i < g.H * g.W; i += blockDim.x) {
        const int h = i / g.W, w = i % g.W;
        float v = 0.f;
        for (int a = 0; a < g.KH; ++a) {
          const int hh = h + g.ph - a * g.dh;
          if (hh < 0 || hh % g.sh) continue;
          const int yo = hh / g.sh;
          if (yo >= g.HO) continue;
          for (int b = 0; b < g.KW; ++b) {
            const int ww = w + g.pw - b * g.dw;
            if (ww < 0 || ww % g.sw) continue;
            const int xo = ww / g.sw;
            if (xo >= g.WO) continue;
            const int o = yo * g.WO + xo, t = a * g.KW + b;
            for (int p = 0; p < 2; ++p)
              if (A.w[p] && A.g[p]) v += gS[p][o] * wS[p][t];
          }
        }
        dst[i] = A.beta_dx ? dst[i] + v : v;
      }
    }
    if (wgrad) {
      for (int o = threadIdx.x; o < nout; o += blockDim.x) {
        const int yo = o / g.WO, xo = o % g.WO;
        const int at = yo * g.sh * Wp + xo * g.sw;
        for (int p = 0; p < 2; ++p) {
          if (!A.xin[p]) continue;
          const float gv = gS[p][o];
          const float* s = xS[p] + at;
#pragma unroll
          for (int t = 0; t < KT; ++t)
            if (t < KK) acc[t] += gv * s[offS[t]];
        }
      }
    }
  }
  if (!wgrad) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int t = 0; t < KT; ++t) {
    const float v = bb::warp_sum(acc[t]);
    if (lane == 0) red[wid][t] = v;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < KK; t += blockDim.x) {
    float s = red[0][t];
    for (int k = 1; k < kThreads / 32; ++k) s += red[k][t];
    A.part[((int64_t)blockIdx.x * g.C + c) * KK + t] = s;
  }
}

DwGeom geom(const bb_node& nd) {
  DwGeom g;
  g.N = (int)nd.dims[0]; g.C = (int)nd.dims[1]; g.H = (int)nd.dims[2]; g.W = (int)nd.dims[3];
  g.KH = (int)nd.dims[5]; g.KW = (int)nd.dims[6]; g.HO = (int)nd.dims[7]; g.WO = (int)nd.dims[8];
  g.sh = (int)nd.dims[9]; g.sw = (int)nd.dims[10]; g.ph = (int)nd.dims[11]; g.pw = (int)nd.dims[12];
  g.dh = (int)nd.dims[13]; g.dw = (int)nd.dims[14];
  // a few hundred outputs per image group, as long as the grid still covers every SM twice
  int ipb = 1;
  while (2 * ipb <= g.N && (int64_t)ipb * g.HO * g.WO < 512 &&
         (int64_t)((g.N + 2 * ipb - 1) / (2 * ipb)) * g.C >= 2 * BB_SM_COUNT)
    ipb *= 2;
  g.ipb = ipb;
  return g;
}

size_t bwd_smem(const DwGeom& g) {
  const int KK = g.KH * g.KW;
  return sizeof(float) * (2 * (size_t)g.HO * g.WO + 2 * (size_t)g.Hp() * g.Wp() + 2 * KK) + sizeof(int) * KK;
}

template <int KT>
int launch_bwd(const DwArgs& A, const DwGeom& g, dim3 grid, size_t smem, cudaStream_t s) {
  static BbOncePerDevice once;
  if (once.need())
    BB_CUDA_TRY(cudaFuncSetAttribute(dw_bwd_kernel<KT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
  dw_bwd_kernel<KT><<<grid, kThreads, smem, s>>>(A, g);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace

// Shapes the staged kernels take: C_out == C_in == groups, at most kMaxTaps taps, fp32 operands, planes that fit the
// shared-memory budget.  plan.py refuses every other grouped convolution before a descriptor is built.
extern "C" int bb_conv_dw_ok(int C, int O, int groups, int H, int W, int KH, int KW, int HO, int WO, int ph, int pw) {
  if (groups != C || O != C || KH * KW > kMaxTaps || HO < 1 || WO < 1) return 0;
  DwGeom g{};
  g.H = H; g.W = W; g.KH = KH; g.KW = KW; g.HO = HO; g.WO = WO; g.ph = ph; g.pw = pw;
  return bwd_smem(g) <= kMaxSmem ? 1 : 0;
}

// Depthwise products of the input and weight operands of a conv2d node (dims[15] = groups > 1); the bias terms are
// left to bb_launch_conv2d.
int bb_conv_dw_run(const bb_node& nd, int pass, cudaStream_t s) {
  const DwGeom g = geom(nd);
  const int KK = g.KH * g.KW;
  if (!bb_conv_dw_ok(g.C, (int)nd.dims[4], (int)nd.dims[15], g.H, g.W, g.KH, g.KW, g.HO, g.WO, g.ph, g.pw) ||
      nd.dt[0] != BB_F32 || nd.dt[1] != BB_F32)
    return BB_ERR_UNSUPPORTED;
  const bool actX = nd.active & 1, actW = nd.active & 2, actB = nd.active & 4;
  const dim3 grid((unsigned)((g.N + g.ipb - 1) / g.ipb), (unsigned)g.C);
  if (pass == BB_PASS_TAN_FWD) {
    DwArgs A{};
    if (actX) { A.in[0] = reinterpret_cast<const float*>(nd.t[0]); A.w[0] = reinterpret_cast<const float*>(nd.base[1]); }
    if (actW) { A.in[1] = reinterpret_cast<const float*>(nd.base[0]); A.w[1] = reinterpret_cast<const float*>(nd.t[1]); }
    A.bias = actB ? reinterpret_cast<const float*>(nd.t[2]) : nullptr;
    A.out = reinterpret_cast<float*>(nd.t[3]);
    const size_t smem = sizeof(float) * (2 * (size_t)g.Hp() * g.Wp() + 2 * KK) + sizeof(int) * KK;
    static BbOncePerDevice once;
    if (once.need())
      BB_CUDA_TRY(cudaFuncSetAttribute(dw_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    dw_fwd_kernel<<<grid, kThreads, smem, s>>>(A, g);
    bb_launch_tally += 1;
    BB_LAUNCH_CHECK();
    return BB_OK;
  }
  const bool base = pass == BB_PASS_BASE_BWD;
  const int need = base ? nd.pad0 : nd.active;
  if (!(need & 3)) return BB_OK;
  DwArgs A{};
  A.g[0] = reinterpret_cast<const float*>(base ? nd.a[3] : nd.at[3]);
  if (!base) A.g[1] = reinterpret_cast<const float*>(nd.a[3]);
  if (need & 1) {
    A.dx = reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]);
    A.beta_dx = nd.beta[0];
    A.w[0] = reinterpret_cast<const float*>(nd.base[1]);
    if (!base && actW) A.w[1] = reinterpret_cast<const float*>(nd.t[1]);
  }
  float* wout = reinterpret_cast<float*>(base ? nd.a[1] : nd.at[1]);
  const int64_t nw = (int64_t)g.C * KK;
  bool owned = false;
  if (need & 2) {
    A.xin[0] = reinterpret_cast<const float*>(nd.base[0]);
    if (!base && actX) A.xin[1] = reinterpret_cast<const float*>(nd.t[0]);
    A.part = bb_partials_acquire(sizeof(float) * grid.x * nw, s, &owned);
    if (A.part == nullptr) return cudaErrorMemoryAllocation;
    if (!nd.beta[1]) {
      BB_CUDA_TRY(cudaMemsetAsync(wout, 0, sizeof(float) * nw, s));
      bb_launch_tally += 1;
    }
  }
  const size_t smem = bwd_smem(g);
  int rc = KK <= 9 ? launch_bwd<9>(A, g, grid, smem, s)
         : KK <= 25 ? launch_bwd<25>(A, g, grid, smem, s)
                    : launch_bwd<kMaxTaps>(A, g, grid, smem, s);
  if (rc == BB_OK && A.part != nullptr) rc = bb_partials_reduce(A.part, (int)grid.x, nw, wout, s);
  if (A.part != nullptr) bb_partials_release(A.part, owned, s);
  return rc;
}
