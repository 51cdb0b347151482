// K6: second-order rules of Conv2d (NCHW, groups=1, any stride/padding/dilation) as implicit GEMMs on
// the shared SIMT tile kernel -- the three im2col gathers are loader functors, nothing is materialised.
//
//   TF  t_y  = conv(t_x, W) + conv(x, t_W) (+ t_b)                         C[o][p]     K = C*KH*KW
//   BB  a_x  = dgrad(a_y, W)                                              C[c][p_in]  K = O*KH*KW
//   TB  at_x = dgrad(at_y, W) + dgrad(a_y, t_W)
//       at_W = wgrad(at_y, x) + wgrad(a_y, t_x)   (split-K, fixed order)  C[o][cij]   K = N*HO*WO
//       at_b = sum_{n,y,x} at_y
// (SURVEY.md Appendix B "Conv2d".)  Spec: oracle/plan_interp.py tf_conv2d/bb_conv2d/tb_conv2d.
#include <stdlib.h>

#include "../../include/betty_b200.h"
#include "conv_small.h"
#include "conv_tma.h"
#include "gemm_tma.h"
#include "tma.h"
#include "gemm_tc.h"
#include "plan.h"
#include "tile_gemm.cuh"

namespace {

struct Geom {
  int N, C, H, W, O, KH, KW, HO, WO, sh, sw, ph, pw, dh, dw;
};

// B operand of the forward product: In[(c,i,j)][p], p = (img, y, x)
struct ImLoad {
  const void* p[2];
  int dt[2];
  Geom g;
  int k_fast;
  __device__ __forceinline__ float load(int pair, int64_t, int64_t k, int64_t pix) const {
    const int kk = g.KH * g.KW;
    const int c = (int)(k / kk), r = (int)(k - (int64_t)c * kk), i = r / g.KW, j = r - i * g.KW;
    const int hw = g.HO * g.WO;
    const int img = (int)(pix / hw), q = (int)(pix - (int64_t)img * hw), y = q / g.WO, x = q - y * g.WO;
    const int h = y * g.sh - g.ph + i * g.dh, w = x * g.sw - g.pw + j * g.dw;
    if (h < 0 || h >= g.H || w < 0 || w >= g.W) return 0.f;
    return bb::ldf(p[pair], (((int64_t)img * g.C + c) * g.H + h) * g.W + w, dt[pair]);
  }
};

// same gather, transposed roles: In[p][(c,i,j)]  (B operand of the weight-gradient product)
struct ImLoadT {
  ImLoad im;
  int k_fast;
  __device__ __forceinline__ float load(int pair, int64_t b, int64_t pix, int64_t k) const {
    return im.load(pair, b, k, pix);
  }
};

// A operand of the forward product: W[o][(c,i,j)] (row-major as stored)
struct WLoad {
  const void* p[2];
  int dt[2];
  int64_t ckk;
  int k_fast;
  __device__ __forceinline__ float load(int pair, int64_t, int64_t o, int64_t k) const {
    return bb::ldf(p[pair], o * ckk + k, dt[pair]);
  }
};

// A operand of the data-gradient product: Wd[c][(o,i,j)] = W[o][c][i][j]
struct WLoadD {
  const void* p[2];
  int dt[2];
  Geom g;
  int k_fast;
  __device__ __forceinline__ float load(int pair, int64_t, int64_t c, int64_t k) const {
    const int kk = g.KH * g.KW;
    const int o = (int)(k / kk), r = (int)(k - (int64_t)o * kk);
    return bb::ldf(p[pair], ((int64_t)o * g.C + c) * kk + r, dt[pair]);
  }
};

// B operand of the data-gradient product: G[(o,i,j)][p_in], p_in = (img, h, w)
struct GLoadD {
  const void* p[2];
  int dt[2];
  Geom g;
  int k_fast;
  __device__ __forceinline__ float load(int pair, int64_t, int64_t k, int64_t pix) const {
    const int kk = g.KH * g.KW;
    const int o = (int)(k / kk), r = (int)(k - (int64_t)o * kk), i = r / g.KW, j = r - i * g.KW;
    const int hw = g.H * g.W;
    const int img = (int)(pix / hw), q = (int)(pix - (int64_t)img * hw), h = q / g.W, w = q - h * g.W;
    const int yy = h + g.ph - i * g.dh, xx = w + g.pw - j * g.dw;
    if (yy < 0 || xx < 0 || yy % g.sh || xx % g.sw) return 0.f;
    const int y = yy / g.sh, x = xx / g.sw;
    if (y >= g.HO || x >= g.WO) return 0.f;
    return bb::ldf(p[pair], (((int64_t)img * g.O + o) * g.HO + y) * g.WO + x, dt[pair]);
  }
};

// A operand of the weight-gradient product: G[o][p], p = (img, y, x)
struct GLoadW {
  const void* p[2];
  int dt[2];
  Geom g;
  int k_fast;
  __device__ __forceinline__ float load(int pair, int64_t, int64_t o, int64_t pix) const {
    const int hw = g.HO * g.WO;
    const int img = (int)(pix / hw), q = (int)(pix - (int64_t)img * hw);
    return bb::ldf(p[pair], ((int64_t)img * g.O + o) * hw + q, dt[pair]);
  }
};

// C[ch][pix] -> NCHW tensor with `CH` channels and `HW` pixels per plane
struct PlaneStore {
  float* p;
  int CH, HW;
  int beta;
  const float* bias;
  __device__ __forceinline__ void store(int64_t, int64_t ch, int64_t pix, float v, bool first, bool atomic) const {
    const int img = (int)(pix / HW), q = (int)(pix - (int64_t)img * HW);
    float* dst = p + ((int64_t)img * CH + ch) * HW + q;
    if (bias != nullptr && first) v += bias[ch];
    if (atomic) atomicAdd(dst, v);
    else *dst = beta ? *dst + v : v;
  }
};

template <class LA, class LB, class SC>
int launch(const LA& la, const LB& lb, const SC& sc, int64_t M, int64_t N, int64_t K, int npairs, int ksplit,
           cudaStream_t s) {
  // ksplit > 1: partials in the plan's reduction workspace, summed in split order (tile_gemm.cuh splitk_reduce)
  ksplit = bb_reduce_ws_splits(ksplit, sizeof(float) * M * N);
  float* part = ksplit > 1 ? bb_reduce_ws.base : nullptr;
  if (M <= 16) {
    dim3 grid((unsigned)((N + 63) / 64), (unsigned)((M + 15) / 16), (unsigned)ksplit);
    bb::tile_gemm_kernel<16, 64, 16, 1, 4, LA, LB, SC><<<grid, 256, 0, s>>>(la, lb, sc, M, N, K, npairs, ksplit, part);
  } else {
    dim3 grid((unsigned)((N + 63) / 64), (unsigned)((M + 63) / 64), (unsigned)ksplit);
    bb::tile_gemm_kernel<64, 64, 16, 4, 4, LA, LB, SC><<<grid, 256, 0, s>>>(la, lb, sc, M, N, K, npairs, ksplit, part);
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return bb::splitk_reduce(sc, part, M, N, 1, ksplit, s);
}

__device__ __forceinline__ void chansum_store(float* out, float* part, int ch, int CH, float acc) {
  if (part != nullptr) part[(int64_t)blockIdx.y * CH + ch] = acc;
  else out[ch] += acc;
}

// out[ch] += sum_{img, q} g[(img*CH + ch)*HW + q].  With part != nullptr, block (ch, y) writes its sum to part[y*CH + ch]
// and bb_partials_reduce adds the gridDim.y partials in order; without, gridDim.y is 1 and the block adds to out itself.
__global__ void __launch_bounds__(256) chansum_kernel(const float* __restrict__ g, float* out, int NIMG, int CH, int HW,
                                                      int small_max, float* __restrict__ part) {
  __shared__ float red[32];
  const int ch = blockIdx.x;
  float acc = 0.f;
  const bool vec = (HW & 3) == 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  if (HW <= small_max) {
    // small planes (LeNet conv2: 100 elements): a block per plane would keep 25 of 256 threads busy.  A warp per
    // plane instead, four planes in flight per warp.
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int wstride = gridDim.y * nw;
    for (int img0 = blockIdx.y * nw + warp; img0 < NIMG; img0 += 4 * wstride) {
      float part[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int img = img0 + u * wstride;
        if (img < NIMG) {
          const float* src = g + ((int64_t)img * CH + ch) * HW;
          if (vec) {
            for (int q = lane * 4; q < HW; q += 128) {
              const float4 v = bb::ld4_stream(src + q);
              part[u] += (v.x + v.y) + (v.z + v.w);
            }
          } else {
            for (int q = lane; q < HW; q += 32) part[u] += src[q];
          }
        }
      }
      acc += (part[0] + part[1]) + (part[2] + part[3]);
    }
    acc = bb::block_sum<float>(acc, red);
    if (threadIdx.x == 0) chansum_store(out, part, ch, CH, acc);
    return;
  }
  for (int img = blockIdx.y; img < NIMG; img += gridDim.y) {
    const float* src = g + ((int64_t)img * CH + ch) * HW;
    if (vec) {
      for (int q = threadIdx.x * 4; q < HW; q += blockDim.x * 4) {
        const float4 v = bb::ld4_stream(src + q);
        acc += (v.x + v.y) + (v.z + v.w);
      }
    } else {
      for (int q = threadIdx.x; q < HW; q += blockDim.x) acc += src[q];
    }
  }
  acc = bb::block_sum<float>(acc, red);
  if (threadIdx.x == 0) chansum_store(out, part, ch, CH, acc);
}

// ---- tensor-core (wgmma) implicit-GEMM operands, bf16-autocast graphs with >= 32 channels ----------
TcSrc pixrow(const void* p, int dt, int CH, int H, int W, const Geom& g, int GH, int GW, int flip) {
  TcSrc s{};
  s.p = p; s.dt = dt; s.mode = TC_PIXROW;
  s.CH = CH; s.H = H; s.W = W; s.KH = g.KH; s.KW = g.KW; s.GH = GH; s.GW = GW; s.py = g.ph; s.px = g.pw; s.flip = flip;
  return s;
}
TcSrc pixk(const void* p, int dt, int CH, int H, int W, int KH, int KW, int GH, int GW, int py, int px) {
  TcSrc s{};
  s.p = p; s.dt = dt; s.mode = TC_PIXK;
  s.CH = CH; s.H = H; s.W = W; s.KH = KH; s.KW = KW; s.GH = GH; s.GW = GW; s.py = py; s.px = px; s.flip = 0;
  return s;
}
TcSrc wdgrad(const void* p, int dt, const Geom& g) {
  TcSrc s{};
  s.p = p; s.dt = dt; s.mode = TC_WDGRAD; s.KH = g.KH; s.KW = g.KW; s.C2 = g.C;
  return s;
}

// the small-channel kernels' view of a stride-1 node: its own geometry (tangent forward and weight gradient), and the
// data gradient as a correlation with the transposed, flipped weights over the output-side maps; launchers add pointers
SmallConvArgs small_fwd_args(const Geom& g) {
  SmallConvArgs A{};
  A.mode = 0;
  A.N = g.N; A.CI = g.C; A.H = g.H; A.W = g.W; A.CO = g.O; A.KH = g.KH; A.KW = g.KW; A.HO = g.HO; A.WO = g.WO;
  A.ph = g.ph; A.pw = g.pw; A.C_orig = g.C;
  return A;
}
SmallConvArgs small_dgrad_args(const Geom& g) {
  SmallConvArgs A{};
  A.mode = 1;
  A.N = g.N; A.CI = g.O; A.H = g.HO; A.W = g.WO; A.CO = g.C; A.KH = g.KH; A.KW = g.KW; A.HO = g.H; A.WO = g.W;
  A.ph = g.KH - 1 - g.ph; A.pw = g.KW - 1 - g.pw; A.C_orig = g.C;
  return A;
}

// second-generation small-channel kernels first (conv_small2.cu), the first generation when they decline
int small_corr(const SmallConvArgs& A, cudaStream_t s) {
  if (!getenv("BB200_CONV_SMALL_V1")) {
    const int rc = bb_conv_small_corr2(A, s);
    if (rc != BB_DECLINED) return rc;
  }
  return bb_conv_small_corr(A, s);
}
int small_wgrad(const SmallConvArgs& A, cudaStream_t s) {
  if (!getenv("BB200_CONV_SMALL_V1")) {
    const int rc = bb_conv_small_wgrad2(A, s);
    if (rc != BB_DECLINED) return rc;
  }
  return bb_conv_small_wgrad(A, s);
}

// a_b / at_b = per-channel sum of a_y / at_y
int bias_grad(const bb_node& nd, const Geom& g, bool base, cudaStream_t s) {
  const void* gy = base ? nd.a[3] : nd.at[3];
  float* out = reinterpret_cast<float*>(base ? nd.a[2] : nd.at[2]);
  if (!nd.beta[2]) {
    BB_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * g.O, s));
    bb_launch_tally += 1;
  }
  int gy_blocks = g.N < 64 ? g.N : 64;
  gy_blocks = bb_reduce_ws_splits(gy_blocks, sizeof(float) * g.O);     // 1 outside a plan: no partials
  float* part = gy_blocks > 1 ? bb_reduce_ws.base : nullptr;
  static const int small_max = getenv("BB200_CHANSUM_V1") ? 0 : 512;
  chansum_kernel<<<dim3(g.O, gy_blocks), 256, 0, s>>>(reinterpret_cast<const float*>(gy), out, g.N, g.O, g.HO * g.WO,
                                                      small_max, part);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  if (part != nullptr) return bb_partials_reduce(part, gy_blocks, g.O, out, s);
  return BB_OK;
}

}  // namespace

int bb_launch_conv2d(const bb_node& nd, int pass, cudaStream_t s) {
  Geom g;
  g.N = (int)nd.dims[0]; g.C = (int)nd.dims[1]; g.H = (int)nd.dims[2]; g.W = (int)nd.dims[3]; g.O = (int)nd.dims[4];
  g.KH = (int)nd.dims[5]; g.KW = (int)nd.dims[6]; g.HO = (int)nd.dims[7]; g.WO = (int)nd.dims[8];
  g.sh = (int)nd.dims[9]; g.sw = (int)nd.dims[10]; g.ph = (int)nd.dims[11]; g.pw = (int)nd.dims[12];
  g.dh = (int)nd.dims[13]; g.dw = (int)nd.dims[14];
  const bool actX = nd.active & 1, actW = nd.active & 2, actB = nd.active & 4;
  int rc;
  if (nd.dims[15] > 1) {
    // depthwise (groups = C = O): staged per-plane kernels for x and W, the channel sums here for the bias
    if ((rc = bb_conv_dw_run(nd, pass, s))) return rc;
    const bool base = pass == BB_PASS_BASE_BWD;
    if (pass == BB_PASS_TAN_FWD || !((base ? nd.pad0 : nd.active) & 4)) return BB_OK;
    return bias_grad(nd, g, base, s);
  }
  const int64_t CKK = (int64_t)g.C * g.KH * g.KW, OKK = (int64_t)g.O * g.KH * g.KW;
  const int64_t P = (int64_t)g.N * g.HO * g.WO, PIN = (int64_t)g.N * g.H * g.W;
  const bool unit = g.sh == 1 && g.sw == 1 && g.dh == 1 && g.dw == 1 && !getenv("BB200_CONV_IGEMM");
  const bool tc = (nd.kind & 1) && unit && !getenv("BB200_NO_TC") && g.O >= 32 && CKK <= 2048 && OKK <= 2048;
  // preferred tensor-core route: NHWC bf16 packs + TMA box loads (conv_tma.cu)
  bool tma_done = false;
  if (pass == BB_PASS_BASE_BWD && (rc = bb_conv_tma_prepare(nd, s))) return rc;
  if (bb_conv_tma_ok(nd, pass)) {
    rc = bb_conv_tma_run(nd, pass, s);
    if (rc == BB_OK) {
      if (pass == BB_PASS_TAN_FWD) return BB_OK;
      tma_done = true;
    } else if (rc != BB_DECLINED) {
      return rc;
    }
  }
  if (pass == BB_PASS_TAN_FWD && tc) {
    // D[pixel][o] = sum_(c,i,j) im2col(t_x)[pixel][cij] * W[o][cij] + im2col(x)[pixel][cij] * t_W[o][cij]
    TcGemmArgs G{};
    G.M = P; G.N = g.O; G.K = CKK;
    int np = 0;
    if (actX) { G.a[np] = pixrow(nd.t[0], BB_F32, g.C, g.H, g.W, g, g.HO, g.WO, 0); G.b[np] = tc_strided(nd.base[1], nd.dt[1], CKK, 1); ++np; }
    if (actW) { G.a[np] = pixrow(nd.base[0], nd.dt[0], g.C, g.H, g.W, g, g.HO, g.WO, 0); G.b[np] = tc_strided(nd.t[1], BB_F32, CKK, 1); ++np; }
    G.npairs = np;
    G.out = reinterpret_cast<float*>(nd.t[3]); G.omode = 1; G.OCH = g.O; G.OHW = g.HO * g.WO; G.beta = 0;
    G.bias = actB ? reinterpret_cast<const float*>(nd.t[2]) : nullptr; G.bias_stride = 1;
    G.allow_split = 0;
    return bb_gemm_tc_run(G, s);
  }
  if (pass == BB_PASS_TAN_FWD && unit && bb_conv_small_corr_ok(g.C, g.O, g.KH, g.KW, (actX ? 1 : 0) + (actW ? 1 : 0))) {
    SmallConvArgs A = small_fwd_args(g);
    int np = 0;
    if (actX) { A.in[np] = nd.t[0]; A.dt_in[np] = BB_F32; A.w[np] = nd.base[1]; A.dt_w[np] = nd.dt[1]; ++np; }
    if (actW) { A.in[np] = nd.base[0]; A.dt_in[np] = nd.dt[0]; A.w[np] = nd.t[1]; A.dt_w[np] = BB_F32; ++np; }
    A.npairs = np;
    A.out = reinterpret_cast<float*>(nd.t[3]);
    A.bias = actB ? reinterpret_cast<const float*>(nd.t[2]) : nullptr;
    A.beta = 0;
    return small_corr(A, s);
  }
  if (pass == BB_PASS_TAN_FWD) {
    WLoad la{};
    ImLoad lb{};
    la.ckk = CKK; la.k_fast = 1;
    lb.g = g; lb.k_fast = 0;
    int np = 0;
    if (actX) { la.p[np] = nd.base[1]; la.dt[np] = nd.dt[1]; lb.p[np] = nd.t[0]; lb.dt[np] = BB_F32; ++np; }
    if (actW) { la.p[np] = nd.t[1]; la.dt[np] = BB_F32; lb.p[np] = nd.base[0]; lb.dt[np] = nd.dt[0]; ++np; }
    PlaneStore sc{reinterpret_cast<float*>(nd.t[3]), g.O, g.HO * g.WO, 0,
                  actB ? reinterpret_cast<const float*>(nd.t[2]) : nullptr};
    return launch(la, lb, sc, g.O, P, CKK, np, 1, s);
  }
  const bool base = pass == BB_PASS_BASE_BWD;
  const void* gy = base ? nd.a[3] : nd.at[3];
  const int need = (base ? nd.pad0 : nd.active) & (tma_done ? ~3 : ~0);
  if ((need & 1) && tc && g.C >= 32) {
    // D[in-pixel][c] = sum_(o,i,j) g[img,o,y+ph-i,x+pw-j] * W[o][c][i][j]  (+ a_y with t_W)
    TcGemmArgs G{};
    G.M = PIN; G.N = g.C; G.K = OKK;
    int np = 0;
    G.a[np] = pixrow(gy, BB_F32, g.O, g.HO, g.WO, g, g.H, g.W, 1); G.b[np] = wdgrad(nd.base[1], nd.dt[1], g); ++np;
    if (!base && actW) { G.a[np] = pixrow(nd.a[3], BB_F32, g.O, g.HO, g.WO, g, g.H, g.W, 1); G.b[np] = wdgrad(nd.t[1], BB_F32, g); ++np; }
    G.npairs = np;
    G.out = reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]); G.omode = 1; G.OCH = g.C; G.OHW = g.H * g.W;
    G.beta = nd.beta[0]; G.bias = nullptr; G.allow_split = 0;
    rc = bb_gemm_tc_run(G, s);
    if (rc) return rc;
  } else if ((need & 1) && unit && bb_conv_small_corr_ok(g.O, g.C, g.KH, g.KW, (!base && actW) ? 2 : 1)) {
    SmallConvArgs A = small_dgrad_args(g);
    int np = 0;
    A.in[np] = gy; A.dt_in[np] = BB_F32; A.w[np] = nd.base[1]; A.dt_w[np] = nd.dt[1]; ++np;
    if (!base && actW) { A.in[np] = nd.a[3]; A.dt_in[np] = BB_F32; A.w[np] = nd.t[1]; A.dt_w[np] = BB_F32; ++np; }
    A.npairs = np;
    A.out = reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]);
    A.bias = nullptr;
    A.beta = nd.beta[0];
    rc = small_corr(A, s);
    if (rc) return rc;
  } else if (need & 1) {
    WLoadD la{};
    GLoadD lb{};
    la.g = g; la.k_fast = 1;
    lb.g = g; lb.k_fast = 0;
    int np = 0;
    la.p[np] = nd.base[1]; la.dt[np] = nd.dt[1]; lb.p[np] = gy; lb.dt[np] = BB_F32; ++np;
    if (!base && actW) { la.p[np] = nd.t[1]; la.dt[np] = BB_F32; lb.p[np] = nd.a[3]; lb.dt[np] = BB_F32; ++np; }
    PlaneStore sc{reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]), g.C, g.H * g.W, nd.beta[0], nullptr};
    rc = launch(la, lb, sc, g.C, PIN, OKK, np, 1, s);
    if (rc) return rc;
  }
  if ((need & 2) && tc && nd.beta[1]) {
    // D[(c,i,j)][o] = sum_pixels im2col(x)[cij][pixel] * at_y[o][pixel]  (+ t_x with a_y); split-K, fixed-order reduce
    TcGemmArgs G{};
    G.M = CKK; G.N = g.O; G.K = P;
    int np = 0;
    G.a[np] = pixk(nd.base[0], nd.dt[0], g.C, g.H, g.W, g.KH, g.KW, g.HO, g.WO, g.ph, g.pw);
    G.b[np] = pixk(gy, BB_F32, g.O, g.HO, g.WO, 1, 1, g.HO, g.WO, 0, 0); ++np;
    if (!base && actX) {
      G.a[np] = pixk(nd.t[0], BB_F32, g.C, g.H, g.W, g.KH, g.KW, g.HO, g.WO, g.ph, g.pw);
      G.b[np] = pixk(nd.a[3], BB_F32, g.O, g.HO, g.WO, 1, 1, g.HO, g.WO, 0, 0); ++np;
    }
    G.npairs = np;
    G.out = reinterpret_cast<float*>(base ? nd.a[1] : nd.at[1]); G.omode = 0; G.ors = 1; G.ocs = CKK;
    G.beta = 1; G.bias = nullptr; G.allow_split = 1;
    rc = bb_gemm_tc_run(G, s);
    if (rc) return rc;
  } else if ((need & 2) && unit && bb_conv_small_wgrad_ok(g.O, g.C, g.H, g.W, g.HO, g.WO, g.KH, g.KW)) {
    SmallConvArgs A = small_fwd_args(g);
    int np = 0;
    A.g[np] = gy; A.dt_g[np] = BB_F32; A.in[np] = nd.base[0]; A.dt_in[np] = nd.dt[0]; ++np;
    if (!base && actX) { A.g[np] = nd.a[3]; A.dt_g[np] = BB_F32; A.in[np] = nd.t[0]; A.dt_in[np] = BB_F32; ++np; }
    A.npairs = np;
    float* out = reinterpret_cast<float*>(base ? nd.a[1] : nd.at[1]);
    if (!nd.beta[1]) {
      BB_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * g.O * CKK, s));
      bb_launch_tally += 1;
    }
    A.out = out;
    rc = small_wgrad(A, s);
    if (rc) return rc;
  } else if (need & 2) {
    GLoadW la{};
    ImLoadT lb{};
    la.g = g; la.k_fast = 1;
    lb.im.g = g; lb.k_fast = 1;
    int np = 0;
    la.p[np] = gy; la.dt[np] = BB_F32; lb.im.p[np] = nd.base[0]; lb.im.dt[np] = nd.dt[0]; ++np;
    if (!base && actX) { la.p[np] = nd.a[3]; la.dt[np] = BB_F32; lb.im.p[np] = nd.t[0]; lb.im.dt[np] = BB_F32; ++np; }
    float* out = reinterpret_cast<float*>(base ? nd.a[1] : nd.at[1]);
    const int64_t tiles = ((g.O + (g.O <= 16 ? 15 : 63)) / (g.O <= 16 ? 16 : 64)) * ((CKK + 63) / 64);
    int64_t want = (4 * BB_SM_COUNT + tiles - 1) / tiles, maxs = (P + 511) / 512;
    int ksplit = (int)(want < maxs ? want : maxs);
    if (ksplit < 1) ksplit = 1;
    if (ksplit > 1024) ksplit = 1024;
    bb::StridedStore sc{out, CKK, 1, 0, nd.beta[1], nullptr, 0};
    rc = launch(la, lb, sc, g.O, CKK, P, np, ksplit, s);
    if (rc) return rc;
  }
  if (need & 4) return bias_grad(nd, g, base, s);
  return BB_OK;
}

// The route and geometry the small-channel launchers would choose for a stride-1 fp32 node (N, C, H, W) -> O, KHxKW,
// padding (ph, pw), without launching anything (tests).  which: 0 tangent forward, 1 data gradient, 2 weight gradient.
// out[15]: route (0 generic implicit GEMM, 1 corr2, 2 first-generation correlation, 3 wgrad2, 4 first-generation
// weight gradient), grid, work units (correlation) or images per block (weight gradient), then for corr2 PX, IMGS, RY,
// bands, CIC, nstages, VW, image groups, for wgrad2 OB, tasks, row slices, and for both weight gradients the floats of
// one block's partial; -1 where a field does not apply.  The environment switches the launchers read are honoured.
extern "C" int bb_conv_small_geometry(int which, int N, int CI, int H, int W, int CO, int KH, int KW, int ph, int pw,
                                      int npairs, int64_t* out, int cap) {
  if (cap < 15 || which < 0 || which > 2 || npairs < 1 || npairs > 2 || N < 1) return BB_ERR_ARG;
  for (int i = 0; i < 15; ++i) out[i] = -1;
  Geom g{};
  g.N = N; g.C = CI; g.H = H; g.W = W; g.O = CO; g.KH = KH; g.KW = KW; g.ph = ph; g.pw = pw;
  g.HO = H + 2 * ph - KH + 1; g.WO = W + 2 * pw - KW + 1;
  g.sh = g.sw = g.dh = g.dw = 1;
  if (g.HO < 1 || g.WO < 1) return BB_ERR_ARG;
  const bool v1 = getenv("BB200_CONV_SMALL_V1") != nullptr;
  out[0] = 0;
  if (which < 2) {
    SmallConvArgs A = which == 0 ? small_fwd_args(g) : small_dgrad_args(g);
    A.npairs = npairs;
    if (getenv("BB200_CONV_IGEMM") || !bb_conv_small_corr_ok(A.CI, A.CO, A.KH, A.KW, npairs)) return BB_OK;
    int64_t geo[10];
    if (!v1 && bb_conv_small_corr2_geometry(A, geo)) {
      out[0] = 1;
      out[1] = geo[0];
      for (int i = 1; i < 10; ++i) out[1 + i] = geo[i];
    } else {
      const int64_t total = (int64_t)A.N * A.HO * ((A.WO + 3) / 4);   // conv_small.cu: PX = 4, 256 threads per block
      out[0] = 2; out[1] = (total + 255) / 256; out[2] = total; out[3] = 4;
    }
    return BB_OK;
  }
  SmallConvArgs A = small_fwd_args(g);
  A.npairs = npairs;
  if (getenv("BB200_CONV_IGEMM") || !bb_conv_small_wgrad_ok(g.O, g.C, g.H, g.W, g.HO, g.WO, g.KH, g.KW)) return BB_OK;
  int64_t geo[5];
  if (!v1 && bb_conv_small_wgrad2_geometry(A, geo)) {
    out[0] = 3; out[1] = geo[0];
    out[11] = geo[1]; out[12] = geo[2]; out[13] = geo[3]; out[14] = geo[4];
  } else {
    bb_conv_small_wgrad_geometry(A, geo);
    out[0] = 4; out[1] = geo[0]; out[14] = geo[1];
  }
  out[2] = (N + out[1] - 1) / out[1];
  return BB_OK;
}
