// K6 tensor-core path, TMA-fed: second-order rules of a stride-1 Conv2d on bf16-autocast graphs.
//
//   TF  t_y  = conv(t_x, W) + conv(x, t_W) (+ t_b)            gemm_tma_kernel, A = shifted NHWC boxes (TMA_CONV)
//   TB  at_x = dgrad(at_y, W) + dgrad(a_y, t_W)               same kernel, flipped displacements, transposed weights
//       at_W = wgrad(at_y, x) + wgrad(a_y, t_x)               wgrad_tma_kernel below
//
// Activations / adjoints (NCHW, fp32 or bf16) are first repacked to NHWC bf16 with the channel count padded to 64
// (one streaming transpose per operand, written to the plan scratch): a (tap, 64-channel block) operand tile is then a
// single 4-D TMA box whose out-of-bounds rows/columns are the zero padding, and the weight operand is a plain K-major
// matrix [rows][tap][channel].
//
// wgrad: D_tap[c][o] = sum_pixels X[pixel + tap][c] * G[pixel][o] has its reduction over pixels, so both operands are
// MN-major tiles (rows = pixels = k) -- exactly what the NHWC boxes are.  One CTA walks a strided set of pixel tiles;
// per tile the TMA brings one G box and one shifted X box per tap; three consumer warpgroups split the taps (warpgroup
// g owns taps g, g+3, g+6) and issue one wgmma m64n64 per tap and 16-pixel step into register accumulators that live
// over all tiles of the CTA; the epilogue writes the CTA's partial sums to its own slice of `part`, and
// bb_partials_reduce adds the slices into the fp32 weight adjoint in CTA order.
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "conv_tma.h"
#include "gemm_tma.h"
#include "plan.h"
#include "tc_ptx.cuh"
#include "tma.h"

namespace {

using namespace bbtc;

constexpr int WG_CONSUMERS = 3;                      // warpgroups; up to 3 taps each
constexpr int WG_THREADS = WG_CONSUMERS * 128 + 32;    // + the TMA producer warp
constexpr int WG_MAX_TAPS = 9;

struct alignas(64) WgradArgs {
  CUtensorMap x[2], g[2];   // NHWC bf16: X over (64, W, H, N), G over (64, WO, HO, N); box (64, WO, Hb, 1)
  int npairs;
  int taps, KW, ph, pw;
  int Hb, rows, RK;         // box height, valid rows per tile (WO*Hb), rows rounded up to 16
  int tiles_per_img, ntiles;
  int stages;
  int C, O;                 // real channel counts (<= 64)
  float* part;              // [gridDim.x][O][C][taps] fp32 per-CTA partial sums
};

__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_tma_kernel(const __grid_constant__ WgradArgs G) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tile_bytes = G.RK * 128;
  const int stage_bytes = (G.taps + 1) * tile_bytes;   // X tile per tap + G tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + G.stages * stage_bytes);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + 4);
  const int tid = threadIdx.x, warp = tid >> 5;

  // zero the stage buffers once: rows the TMA never writes (tile tail) must read as 0
  {
    uint4* z = reinterpret_cast<uint4*>(smem);
    const int n16 = G.stages * stage_bytes / 16;
    for (int i = tid; i < n16; i += WG_THREADS) z[i] = make_uint4(0, 0, 0, 0);
  }
  fence_proxy_async();
  if (tid == 0) {
    for (int s = 0; s < G.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, WG_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int my_tiles = ((int)blockIdx.x < G.ntiles) ? (G.ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int total = my_tiles * G.npairs;

  if (warp == WG_CONSUMERS * 4) {
    if (elect_one()) {
      for (int p = 0; p < G.npairs; ++p) {
        tma_prefetch_desc(&G.x[p]);
        tma_prefetch_desc(&G.g[p]);
      }
      const uint32_t bytes = (uint32_t)(G.taps + 1) * (uint32_t)G.rows * 128u;
      for (int it = 0; it < total; ++it) {
        const int s = it % G.stages;
        if (it >= G.stages) mbar_wait(empty0 + 8 * s, ((it / G.stages) - 1) & 1);
        const int pair = it % G.npairs;
        const int tile = (int)blockIdx.x + (it / G.npairs) * (int)gridDim.x;
        const int img = tile / G.tiles_per_img, h0 = (tile - img * G.tiles_per_img) * G.Hb;
        const uint32_t bar = full0 + 8 * s;
        const uint32_t base = smem_u32(smem + s * stage_bytes);
        mbar_expect_tx(bar, bytes);
        tma_load_4d(base + G.taps * tile_bytes, &G.g[pair], bar, 0, 0, h0, img);
        for (int t = 0; t < G.taps; ++t) {
          const int i = t / G.KW, j = t - i * G.KW;
          tma_load_4d(base + t * tile_bytes, &G.x[pair], bar, 0, j - G.pw, h0 + i - G.ph, img);
        }
      }
    }
  } else {
    const int wg = tid >> 7, t = tid & 127;
    float acc[3][32];
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
    const int ksteps = G.RK / 16;
    for (int it = 0; it < total; ++it) {
      const int s = it % G.stages;
      mbar_wait(full0 + 8 * s, (it / G.stages) & 1);
      const uint32_t base = smem_u32(smem + s * stage_bytes);
      const uint32_t g_addr = base + G.taps * tile_bytes;
#pragma unroll
      for (int q = 0; q < 3; ++q) fence_acc(acc[q]);
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int tap = wg + WG_CONSUMERS * q;
        if (tap < G.taps) {
          const uint32_t x_addr = base + tap * tile_bytes;
          for (int ks = 0; ks < ksteps; ++ks)
            wgmma_n64<1, 1>(acc[q], desc_mn(x_addr + ks * 2048, 8192), desc_mn(g_addr + ks * 2048, 8192),
                            (it > 0 || ks > 0) ? 1u : 0u);
        }
      }
      wgmma_commit();
#pragma unroll
      for (int q = 0; q < 3; ++q) fence_acc(acc[q]);
      wgmma_wait<1>();
      if (it > 0 && t == 0) mbar_arrive(empty0 + 8 * ((it - 1) % G.stages));
    }
    wgmma_wait<0>();
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      fence_acc(acc[q]);
      const int tap = wg + WG_CONSUMERS * q;
      if (tap >= G.taps) continue;
      // d[4j + 2h + e]: row c = frag_row + 8h, column o = 8j + frag_col + e
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = frag_row(t) + 8 * h;
        if (c >= G.C) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int o = 8 * j + frag_col(t) + e;
            if (o < G.O)
              G.part[((int64_t)blockIdx.x * G.O * G.C + (int64_t)o * G.C + c) * G.taps + tap] = acc[q][4 * j + 2 * h + e];
          }
      }
    }
  }
}

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct Geo {
  int N, C, H, W, O, KH, KW, HO, WO, ph, pw;
};

// forward-form launch: D[pixel of a GH x GW grid][n] = sum_(tap, ch) SRC[pixel + disp(tap)][ch] * WM[n][tap][ch]
int launch_corr(const Geo& g, int npairs, const void* const* src_nhwc, int SH, int SW, int SCp, const void* const* wmat,
                int ncols, int GH, int GW, int flip, float* out, int beta, const float* bias, cudaStream_t s,
                bool padded = false) {
  alignas(64) TmaGemmArgs G;
  memset(&G, 0, sizeof(G));
  const int taps = g.KH * g.KW;
  const int Hb = GH < 128 / GW ? GH : 128 / GW;
  const int bn = ncols <= 64 ? 64 : 128;
  const int64_t Kdim = (int64_t)taps * SCp;
  for (int p = 0; p < npairs; ++p) {
    int rc = padded ? bb_tma_map_nhwc_padded(&G.a[p], src_nhwc[p], g.N, SH, SW, GW, Hb)
                    : bb_tma_map_nhwc(&G.a[p], src_nhwc[p], g.N, SH, SW, SCp, GW, Hb);
    if (rc) return rc;
    rc = bb_tma_map_2d(&G.b[p], wmat[p], ncols, Kdim, Kdim, bn);
    if (rc) return rc;
    G.a_kind[p] = TMA_CONV;
    G.b_kind[p] = TMA_KMAJ;
  }
  G.M = (int64_t)g.N * GH * GW; G.N = ncols; G.K = Kdim; G.npairs = npairs; G.ksplit = 1;
  G.a_bytes = (uint32_t)GW * Hb * 128u; G.b_bytes = (uint32_t)bn * 128u;
  G.Wb = GW; G.Hb = Hb; G.tiles_per_img = (GH + Hb - 1) / Hb; G.KW = g.KW; G.ph = g.ph; G.pw = g.pw; G.flip = flip;
  G.cblocks = SCp / 64;
  G.out = out; G.omode = 1; G.OCH = ncols; G.OHW = GH * GW; G.beta = beta; G.bias = bias; G.bias_stride = 1;
  return bb_gemm_tma_launch(G, bn, (int64_t)g.N * G.tiles_per_img, s);
}

// weight-gradient launch over caller-provided bf16 NHWC operands (accumulates into `out`)
int launch_wgrad(const Geo& g, int npairs, const void* const* xs, const void* const* gs, float* out, cudaStream_t s,
                 bool padded = false) {
  alignas(64) WgradArgs A;
  memset(&A, 0, sizeof(A));
  const int taps = g.KH * g.KW;
  const int Hb = g.HO < 64 / g.WO ? g.HO : 64 / g.WO;
  int rc;
  for (int p = 0; p < npairs; ++p) {
    if (padded) {
      if ((rc = bb_tma_map_nhwc_padded(&A.x[p], xs[p], g.N, g.H, g.W, g.WO, Hb))) return rc;
      if ((rc = bb_tma_map_nhwc_padded(&A.g[p], gs[p], g.N, g.HO, g.WO, g.WO, Hb))) return rc;
    } else {
      if ((rc = bb_tma_map_nhwc(&A.x[p], xs[p], g.N, g.H, g.W, 64, g.WO, Hb))) return rc;
      if ((rc = bb_tma_map_nhwc(&A.g[p], gs[p], g.N, g.HO, g.WO, 64, g.WO, Hb))) return rc;
    }
  }
  A.npairs = npairs; A.taps = taps; A.KW = g.KW; A.ph = g.ph; A.pw = g.pw;
  A.Hb = Hb; A.rows = g.WO * Hb; A.RK = round_up(A.rows, 16);
  A.tiles_per_img = (g.HO + Hb - 1) / Hb; A.ntiles = g.N * A.tiles_per_img;
  A.C = g.C; A.O = g.O;
  const size_t stage = (size_t)(taps + 1) * A.RK * 128;
  int stages = (int)((220 * 1024 - 2048) / stage);
  if (stages > 4) stages = 4;
  if (stages < 2) return BB_DECLINED;
  A.stages = stages;
  const size_t smem = stages * stage + 1024 + 256;
  static BbOncePerDevice configured;
  if (configured.need()) {
    BB_CUDA_TRY(cudaFuncSetAttribute(wgrad_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024));
  }
  const int grid = A.ntiles < BB_SM_COUNT ? A.ntiles : BB_SM_COUNT;
  const int64_t n = (int64_t)g.O * g.C * taps;
  bool owned = false;
  A.part = bb_partials_acquire(sizeof(float) * grid * n, s, &owned);
  if (A.part == nullptr) return cudaErrorMemoryAllocation;
  wgrad_tma_kernel<<<grid, WG_THREADS, smem, s>>>(A);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  rc = bb_partials_reduce(A.part, grid, n, out, s);
  bb_partials_release(A.part, owned, s);
  return rc;
}

// ---- first-layer convolutions (few input channels, input is data: no tangent, no input gradient) -------------------
// With C*KH*KW <= 64 the reduction fits one k-block, so the im2col matrix is materialised once per pass as bf16
// [pixels][k] (TMA-addressable, any stride / dilation) and both products are plain GEMMs on gemm_tma_kernel:
//   TF  t_y[pixel][o]  = Xcol[pixel][k] . t_W[o][k]        (NCHW plane output)
//   TB  at_W[o][k]     = sum_pixels at_y[pixel][o] * Xcol[pixel][k]      (both operands MN-major, split-K)
bool small_c_ok(const bb_node& nd) {
  const int64_t C = nd.dims[1], O = nd.dims[4], KH = nd.dims[5], KW = nd.dims[6];
  if (nd.active & 1) return false;                    // t_x / at_x exist: not a data-input layer
  if (!(nd.active & 2)) return false;
  return C * KH * KW <= 64 && C * KH * KW >= 8 && O >= 32 && O <= 128 && nd.dims[0] * nd.dims[7] * nd.dims[8] >= 128;
}

size_t small_c_scratch(const bb_node& nd) {
  const int64_t P = nd.dims[0] * nd.dims[7] * nd.dims[8], O = nd.dims[4];
  const int64_t kp = (nd.dims[1] * nd.dims[5] * nd.dims[6] + 7) / 8 * 8, op = (O + 63) / 64 * 64;
  return (size_t)(2 * P * kp + 2 * P * op + 2 * (O + 8) * (kp + 8) + 16384);
}

int run_small_c(const bb_node& nd, int pass, cudaStream_t s) {
  Im2colGeom ig;
  ig.N = (int)nd.dims[0]; ig.C = (int)nd.dims[1]; ig.H = (int)nd.dims[2]; ig.W = (int)nd.dims[3];
  ig.KH = (int)nd.dims[5]; ig.KW = (int)nd.dims[6]; ig.HO = (int)nd.dims[7]; ig.WO = (int)nd.dims[8];
  ig.sh = (int)nd.dims[9]; ig.sw = (int)nd.dims[10]; ig.ph = (int)nd.dims[11]; ig.pw = (int)nd.dims[12];
  ig.dh = (int)nd.dims[13]; ig.dw = (int)nd.dims[14];
  const int O = (int)nd.dims[4];
  const int64_t CKK = (int64_t)ig.C * ig.KH * ig.KW, P = (int64_t)ig.N * ig.HO * ig.WO;
  const int kp = (int)((CKK + 7) / 8 * 8), op = (O + 63) / 64 * 64;
  if (small_c_scratch(nd) > bb_scratch.bytes) return BB_DECLINED;
  bb_scratch_reset();
  // the input is data: its im2col matrix is a K-loop constant -> plan-lifetime buffer when one is configured
  bool fresh = false;
  void* xcol = bb_persist_get((size_t)P * kp * 2, &fresh);
  if (!xcol) {
    xcol = bb_scratch_alloc((size_t)P * kp * 2);
    fresh = true;
  }
  if (!xcol) return BB_DECLINED;
  int rc = BB_OK;
  if (fresh && (rc = bb_pack_im2col(nd.base[0], nd.dt[0], ig, xcol, kp, s))) return rc;
  if (pass == BB_PASS_BASE_BWD) return BB_OK;   // bb_conv_tma_prepare: only the constant pack
  if (pass == BB_PASS_TAN_FWD) {
    const TmaView a{xcol, BB_BF16, kp, 1};                 // rows = pixels
    const TmaView b{nd.t[1], BB_F32, CKK, 1};              // rows = o
    return bb_gemm_tma_run(P, O, CKK, 1, &a, &b, reinterpret_cast<float*>(nd.t[3]), 0, 0, 0,
                           (nd.active & 4) ? reinterpret_cast<const float*>(nd.t[2]) : nullptr, 1, false, s,
                           ig.HO * ig.WO, 32);
  }
  void* gy = bb_scratch_alloc((size_t)P * op * 2);
  if (!gy) return BB_DECLINED;
  if ((rc = bb_pack_nhwc(nd.at[3], BB_F32, ig.N, O, ig.HO * ig.WO, gy, op, s))) return rc;
  const TmaView a{gy, BB_BF16, 1, op};                     // rows = o, k = pixel
  const TmaView b{xcol, BB_BF16, 1, kp};                   // rows = k of the window, k = pixel
  return bb_gemm_tma_run(O, CKK, P, 1, &a, &b, reinterpret_cast<float*>(nd.at[1]), CKK, 1, nd.beta[1], nullptr, 0, true, s,
                         0, 8);
}

}  // namespace

bool bb_conv_tma_ok(const bb_node& nd, int pass) {
  static const bool off = getenv("BB200_NO_TMA") != nullptr || getenv("BB200_NO_TC") != nullptr;
  if (off || !(nd.kind & 1) || bb_scratch.base == nullptr || pass == BB_PASS_BASE_BWD) return false;
  if (small_c_ok(nd)) return true;
  const int C = (int)nd.dims[1], H = (int)nd.dims[2], W = (int)nd.dims[3], O = (int)nd.dims[4];
  const int KH = (int)nd.dims[5], KW = (int)nd.dims[6], HO = (int)nd.dims[7], WO = (int)nd.dims[8];
  if (nd.dims[9] != 1 || nd.dims[10] != 1 || nd.dims[13] != 1 || nd.dims[14] != 1) return false;
  if (KH * KW > WG_MAX_TAPS || KH * KW < 1) return false;
  if (C < 32 || O < 32 || C > 64 || O > 64) return false;        // one 64-channel block each way (for now)
  if (WO > 64 || W > 128 || WO < 4 || HO < 1) return false;
  (void)H;
  return true;
}

// NHWC bf16 pack of a K-loop constant (slot 0: the layer input x, slot 1: the base output adjoint a_y) in the plan's
// persistent arena; nullptr if there is none.  Packed on first use, which bb_conv_tma_prepare makes the eager
// base-backward pass.
void* const_nhwc(const void* src, int dt, int N, int C, int HW, int slot, cudaStream_t s, int* rc) {
  bool fresh = false;
  void* p = bb_persist_get((size_t)N * HW * 64 * 2, &fresh, slot);
  *rc = BB_OK;
  if (p && fresh) *rc = bb_pack_nhwc(src, dt, N, C, HW, p, 64, s);
  return p;
}

int bb_conv_tma_prepare(const bb_node& nd, cudaStream_t s) {
  static const bool off = getenv("BB200_NO_TMA") != nullptr || getenv("BB200_NO_TC") != nullptr;
  if (off || !(nd.kind & 1) || bb_scratch.base == nullptr) return BB_OK;
  if (small_c_ok(nd)) {
    const int rc = run_small_c(nd, BB_PASS_BASE_BWD, s);
    return rc == BB_DECLINED ? BB_OK : rc;
  }
  if (!bb_conv_tma_ok(nd, BB_PASS_TAN_BWD)) return BB_OK;
  // called at the node's base-backward visit: x is a base value, a_y (nd.a[3]) is final by now
  int rc = BB_OK;
  if (nd.active & 2) const_nhwc(nd.base[0], nd.dt[0], (int)nd.dims[0], (int)nd.dims[1], (int)(nd.dims[2] * nd.dims[3]), 0, s, &rc);
  if (rc) return rc;
  const_nhwc(nd.a[3], BB_F32, (int)nd.dims[0], (int)nd.dims[4], (int)(nd.dims[7] * nd.dims[8]), 1, s, &rc);
  return rc;
}

size_t bb_conv_tma_scratch(const bb_node& nd) {
  if (small_c_ok(nd)) return small_c_scratch(nd);
  const int64_t N = nd.dims[0], H = nd.dims[2], W = nd.dims[3], KH = nd.dims[5], KW = nd.dims[6], HO = nd.dims[7],
                WO = nd.dims[8];
  return (size_t)(2 * (2 * N * H * W * 64 + 2 * N * HO * WO * 64) + 2 * 4 * 64 * KH * KW * 64 + 16384);
}

int bb_conv_tma_run(const bb_node& nd, int pass, cudaStream_t s) {
  if (small_c_ok(nd)) return run_small_c(nd, pass, s);
  Geo g;
  g.N = (int)nd.dims[0]; g.C = (int)nd.dims[1]; g.H = (int)nd.dims[2]; g.W = (int)nd.dims[3]; g.O = (int)nd.dims[4];
  g.KH = (int)nd.dims[5]; g.KW = (int)nd.dims[6]; g.HO = (int)nd.dims[7]; g.WO = (int)nd.dims[8];
  g.ph = (int)nd.dims[11]; g.pw = (int)nd.dims[12];
  const int taps = g.KH * g.KW;
  const bool actX = nd.active & 1, actW = nd.active & 2, actB = nd.active & 4;
  if (bb_conv_tma_scratch(nd) > bb_scratch.bytes) return BB_DECLINED;
  bb_scratch_reset();
  const size_t in_bytes = (size_t)g.N * g.H * g.W * 64 * 2, out_bytes = (size_t)g.N * g.HO * g.WO * 64 * 2;
  const size_t w_bytes = (size_t)64 * taps * 64 * 2;
  int rc;
  if (pass == BB_PASS_TAN_FWD) {
    const void* src[2];
    const void* wm[2];
    int np = 0;
    if (actX) {
      void* a = bb_scratch_alloc(in_bytes);
      void* w = bb_scratch_alloc(w_bytes);
      if (!a || !w) return BB_DECLINED;
      if ((rc = bb_pack_nhwc(nd.t[0], BB_F32, g.N, g.C, g.H * g.W, a, 64, s))) return rc;
      if ((rc = bb_pack_convw(nd.base[1], nd.dt[1], g.O, g.C, taps, 0, w, 64, s))) return rc;
      src[np] = a; wm[np] = w; ++np;
    }
    if (actW) {
      void* a = const_nhwc(nd.base[0], nd.dt[0], g.N, g.C, g.H * g.W, 0, s, &rc);
      if (rc) return rc;
      void* w = bb_scratch_alloc(w_bytes);
      if (!a) {
        a = bb_scratch_alloc(in_bytes);
        if (a && (rc = bb_pack_nhwc(nd.base[0], nd.dt[0], g.N, g.C, g.H * g.W, a, 64, s))) return rc;
      }
      if (!a || !w) return BB_DECLINED;
      if ((rc = bb_pack_convw(nd.t[1], BB_F32, g.O, g.C, taps, 0, w, 64, s))) return rc;
      src[np] = a; wm[np] = w; ++np;
    }
    if (np == 0) return BB_DECLINED;
    return launch_corr(g, np, src, g.H, g.W, 64, wm, g.O, g.HO, g.WO, 0, reinterpret_cast<float*>(nd.t[3]), 0,
                       actB ? reinterpret_cast<const float*>(nd.t[2]) : nullptr, s);
  }
  // ---- tangent backward ----
  const int need = nd.active;
  void* gy = bb_scratch_alloc(out_bytes);     // at_y
  if (!gy) return BB_DECLINED;
  if ((rc = bb_pack_nhwc(nd.at[3], BB_F32, g.N, g.O, g.HO * g.WO, gy, 64, s))) return rc;
  const bool need_ay = ((need & 1) && actW) || ((need & 2) && actX);
  void* ay = nullptr;                         // a_y: a K-loop constant
  if (need_ay) {
    ay = const_nhwc(nd.a[3], BB_F32, g.N, g.O, g.HO * g.WO, 1, s, &rc);
    if (rc) return rc;
    if (!ay) {
      ay = bb_scratch_alloc(out_bytes);
      if (!ay) return BB_DECLINED;
      if ((rc = bb_pack_nhwc(nd.a[3], BB_F32, g.N, g.O, g.HO * g.WO, ay, 64, s))) return rc;
    }
  }
  if (need & 1) {
    const void* src[2];
    const void* wm[2];
    int np = 0;
    void* w0 = bb_scratch_alloc(w_bytes);
    if (!w0) return BB_DECLINED;
    if ((rc = bb_pack_convw(nd.base[1], nd.dt[1], g.O, g.C, taps, 1, w0, 64, s))) return rc;
    src[np] = gy; wm[np] = w0; ++np;
    if (actW) {
      void* w1 = bb_scratch_alloc(w_bytes);
      if (!w1) return BB_DECLINED;
      if ((rc = bb_pack_convw(nd.t[1], BB_F32, g.O, g.C, taps, 1, w1, 64, s))) return rc;
      src[np] = ay; wm[np] = w1; ++np;
    }
    rc = launch_corr(g, np, src, g.HO, g.WO, 64, wm, g.C, g.H, g.W, 1, reinterpret_cast<float*>(nd.at[0]), nd.beta[0],
                     nullptr, s);
    if (rc) return rc;
  }
  if (need & 2) {
    void* xs = const_nhwc(nd.base[0], nd.dt[0], g.N, g.C, g.H * g.W, 0, s, &rc);
    if (rc) return rc;
    if (!xs) {
      xs = bb_scratch_alloc(in_bytes);
      if (!xs) return BB_DECLINED;
      if ((rc = bb_pack_nhwc(nd.base[0], nd.dt[0], g.N, g.C, g.H * g.W, xs, 64, s))) return rc;
    }
    const void* xs_[2] = {xs, nullptr};
    const void* gs_[2] = {gy, nullptr};
    int np = 1;
    if (actX) {
      void* txs = bb_scratch_alloc(in_bytes);
      if (!txs) return BB_DECLINED;
      if ((rc = bb_pack_nhwc(nd.t[0], BB_F32, g.N, g.C, g.H * g.W, txs, 64, s))) return rc;
      xs_[1] = txs; gs_[1] = ay;
      np = 2;
    }
    float* out = reinterpret_cast<float*>(nd.at[1]);
    if (!nd.beta[1]) {
      BB_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * g.O * g.C * taps, s));
      bb_launch_tally += 1;
    }
    if ((rc = launch_wgrad(g, np, xs_, gs_, out, s))) return rc;
  }
  return BB_OK;
}

int bb_conv_tma_corr(const BbConvGeo& c, int npairs, const void* const* src_nhwc, int SH, int SW, const void* const* wmat,
                     int ncols, int GH, int GW, int flip, float* out, int beta, const float* bias, cudaStream_t s,
                     bool padded) {
  Geo g{c.N, c.C, c.H, c.W, c.O, c.KH, c.KW, c.HO, c.WO, c.ph, c.pw};
  return launch_corr(g, npairs, src_nhwc, SH, SW, 64, wmat, ncols, GH, GW, flip, out, beta, bias, s, padded);
}

int bb_conv_tma_wgrad(const BbConvGeo& c, int npairs, const void* const* x_nhwc, const void* const* gy_nhwc, float* out,
                      cudaStream_t s, bool padded) {
  Geo g{c.N, c.C, c.H, c.W, c.O, c.KH, c.KW, c.HO, c.WO, c.ph, c.pw};
  const int rc = launch_wgrad(g, npairs, x_nhwc, gy_nhwc, out, s, padded);
  return rc == BB_DECLINED ? BB_ERR_UNSUPPORTED : rc;
}
