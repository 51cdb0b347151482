// K8/K9 (row-structured part): softmax / log-softmax over the last dim (attention probabilities, CE
// head), NLL pick, BCE-with-logits, embedding gather / scatter-add, max-pool gather / scatter.
// Spec: oracle/plan_interp.py (tf_/bb_/tb_ softmax, logsoftmax, nll, bce_logits, embedding, maxpool2d);
// formulas: SURVEY.md Appendix B.
#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "plan.h"

namespace {

constexpr int kWarpsPerBlock = 8;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per row.  mode: 0 softmax, 1 log-softmax.
//   TF:  softmax  t_y = p*(t_z - <p,t_z>)                 logsm  t_y = t_z - <p,t_z>
//   BB:  softmax  a_z = p*(g - <p,g>)                     logsm  a_z = g - p*sum(g)
//   TB:  softmax  at_z = pt*(g - <p,g>) + p*(gt - <pt,g> - <p,gt>)
//        logsm    at_z = gt - p*sum(gt) - pt*sum(g),      pt = p*(t_z - <p,t_z>)
__global__ void __launch_bounds__(kWarpsPerBlock * 32) softmax_rule_kernel(
    const void* __restrict__ z, int dtz, const float* __restrict__ tz, float* ty, const float* __restrict__ g,
    const float* __restrict__ gt, float* gz, int64_t rows, int D, int mode, int pass, int beta) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int64_t off = row * D;
  float mx = -INFINITY;
  for (int c = lane; c < D; c += 32) mx = fmaxf(mx, bb::ldf(z, off + c, dtz));
  mx = warp_max(mx);
  float se = 0.f;
  for (int c = lane; c < D; c += 32) se += __expf(bb::ldf(z, off + c, dtz) - mx);
  se = bb::warp_sum(se);
  const float inv = 1.f / se;
  auto P = [&](int c) { return __expf(bb::ldf(z, off + c, dtz) - mx) * inv; };
  if (pass == BB_PASS_TAN_FWD) {
    float d = 0.f;
    for (int c = lane; c < D; c += 32) d += P(c) * tz[off + c];
    d = bb::warp_sum(d);
    for (int c = lane; c < D; c += 32) {
      const float v = tz[off + c] - d;
      ty[off + c] = mode == 0 ? P(c) * v : v;
    }
  } else if (pass == BB_PASS_BASE_BWD) {
    float d = 0.f;
    for (int c = lane; c < D; c += 32) d += (mode == 0 ? P(c) : 1.f) * g[off + c];
    d = bb::warp_sum(d);
    for (int c = lane; c < D; c += 32) {
      const float p = P(c);
      const float v = mode == 0 ? p * (g[off + c] - d) : g[off + c] - p * d;
      gz[off + c] = beta ? gz[off + c] + v : v;
    }
  } else {
    float ptz = 0.f;
    for (int c = lane; c < D; c += 32) ptz += P(c) * tz[off + c];
    ptz = bb::warp_sum(ptz);
    float s1 = 0.f, s2 = 0.f, s3 = 0.f;  // softmax: <p,g>, <pt,g>, <p,gt> ; logsm: sum g, sum gt
    for (int c = lane; c < D; c += 32) {
      const float p = P(c), pt = p * (tz[off + c] - ptz);
      if (mode == 0) {
        s1 += p * g[off + c];
        s2 += pt * g[off + c];
        s3 += p * gt[off + c];
      } else {
        s1 += g[off + c];
        s2 += gt[off + c];
      }
    }
    s1 = bb::warp_sum(s1);
    s2 = bb::warp_sum(s2);
    s3 = bb::warp_sum(s3);
    for (int c = lane; c < D; c += 32) {
      const float p = P(c), pt = p * (tz[off + c] - ptz);
      float v;
      if (mode == 0) v = pt * (g[off + c] - s1) + p * (gt[off + c] - s2 - s3);
      else v = gt[off + c] - p * s2 - pt * s1;
      gz[off + c] = beta ? gz[off + c] + v : v;
    }
  }
}

// ---- NLL: y_i = -z[i, t_i] (none) or scale * sum_i (mean / sum); linear in z ------------------------
__global__ void nll_fwd_kernel(const float* __restrict__ tz, const int64_t* __restrict__ target, float* ty, int B, int C,
                               int reduction, float scale) {
  if (reduction == 0) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) ty[i] = -tz[(int64_t)i * C + target[i]];
  } else {  // single block
    __shared__ float red[32];
    float acc = 0.f;
    for (int i = threadIdx.x; i < B; i += blockDim.x) acc -= tz[(int64_t)i * C + target[i]];
    acc = bb::block_sum<float>(acc, red);
    if (threadIdx.x == 0) ty[0] = scale * acc;
  }
}

__global__ void nll_bwd_kernel(float* gz, const float* __restrict__ gy, const int64_t* __restrict__ target, int B, int C,
                               int reduction, float scale, int beta) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * C) return;
  const int r = (int)(i / C), c = (int)(i - (int64_t)r * C);
  const float g = reduction == 0 ? gy[r] : scale * gy[0];
  const float v = (c == (int)target[r]) ? -g : 0.f;
  gz[i] = beta ? gz[i] + v : v;
}

// ---- BCE with logits, mean reduction -----------------------------------------------------------------
__global__ void __launch_bounds__(512) bce_fwd_kernel(const void* __restrict__ z, int dtz, const float* __restrict__ y,
                                                      const float* __restrict__ tz, float* ty, int64_t n) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float s = 1.f / (1.f + __expf(-bb::ldf(z, i, dtz)));
    acc += (s - y[i]) * tz[i];
  }
  acc = bb::block_sum<float>(acc, red);
  if (threadIdx.x == 0) ty[0] = acc / (float)n;
}

__global__ void bce_bwd_kernel(const void* __restrict__ z, int dtz, const float* __restrict__ y,
                               const float* __restrict__ tz, const float* __restrict__ g, const float* __restrict__ gt,
                               float* gz, int64_t n, int pass, int beta) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = 1.f / (1.f + __expf(-bb::ldf(z, i, dtz)));
  float v;
  if (pass == BB_PASS_BASE_BWD) v = g[0] * (s - y[i]) / (float)n;
  else v = (gt[0] * (s - y[i]) + g[0] * s * (1.f - s) * tz[i]) / (float)n;
  gz[i] = beta ? gz[i] + v : v;
}

// ---- embedding ---------------------------------------------------------------------------------------
__global__ void emb_fwd_kernel(const float* __restrict__ tw, const int64_t* __restrict__ idx, float* ty, int64_t nidx,
                               int D) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nidx * D) return;
  const int64_t r = i / D;
  ty[i] = tw[idx[r] * D + (i - r * D)];
}

// gw[row] += sum of gy over the tokens that gathered row, in a fixed order.  seg[0..nidx) = the token positions stably
// sorted by table row, seg[nidx + j] = end of the row's run in that order if j starts one, else 0 (built with the plan).
// Block = 16 token lanes x 32 columns, walking the runs that start at j = blockIdx.y, +gridDim.y, ...: lane l adds the
// run's tokens l, l + 16, ... in order, then the lanes are added in lane order (a row every token shares, such as the
// token-type row, is one run of all nidx tokens).
constexpr int kEmbLanes = 16;
__global__ void __launch_bounds__(kEmbLanes * 32) emb_bwd_kernel(float* gw, const int64_t* __restrict__ idx,
                                                                 const int64_t* __restrict__ seg,
                                                                 const float* __restrict__ gy, int64_t nidx, int D,
                                                                 int64_t padding_idx) {
  __shared__ float red[kEmbLanes][32];
  const int cl = threadIdx.x & 31, tl = threadIdx.x >> 5;
  const int64_t col = (int64_t)blockIdx.x * 32 + cl;
  for (int64_t j = blockIdx.y; j < nidx; j += gridDim.y) {
    const int64_t end = seg[nidx + j];
    if (end == 0) continue;   // uniform over the block
    const int64_t row = idx[seg[j]];
    if (row == padding_idx) continue;
    float v = 0.f;
    if (col < D) {
#pragma unroll 4
      for (int64_t k = j + tl; k < end; k += kEmbLanes) v += gy[seg[k] * D + col];
    }
    red[tl][cl] = v;
    __syncthreads();
    if (tl == 0 && col < D) {
      float sum = red[0][cl];
#pragma unroll
      for (int i = 1; i < kEmbLanes; ++i) sum += red[i][cl];
      gw[row * D + col] += sum;
    }
    __syncthreads();
  }
}

// ---- max-pool: gather / scatter with the base argmax ---------------------------------------------------
// relu != 0: a ReLU in front of the pool was folded into the node (ir._fuse_relu_maxpool): its derivative at the
// arg-max position is [pooled base output y > 0]
__global__ void pool_fwd_kernel(const float* __restrict__ tx, const int64_t* __restrict__ idx, float* ty, int64_t nout,
                                int hw_in, int hw_out, const void* __restrict__ y, int dty, int relu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nout) return;
  const int64_t plane = i / hw_out;
  float v = tx[plane * hw_in + idx[i]];
  if (relu && !(bb::ldf(y, i, dty) > 0.f)) v = 0.f;
  ty[i] = v;
}
__global__ void pool_bwd_kernel(float* gx, const int64_t* __restrict__ idx, const float* __restrict__ gy, int64_t nout,
                                int hw_in, int hw_out, const void* __restrict__ y, int dty, int relu) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nout) return;
  if (relu && !(bb::ldf(y, i, dty) > 0.f)) return;
  const int64_t plane = i / hw_out;
  atomicAdd(gx + plane * hw_in + idx[i], gy[i]);  // gx is zeroed at the start of the pass
}
// Disjoint windows (kernel == stride, no padding): every input position belongs to at most one window, so the
// adjoint needs no zero-fill of the buffer and no atomics.  One thread per WINDOW writes its kh x kw input positions
// (the arg-max gets the adjoint, the others 0; 64-bit stores for 2-wide windows); the threads of the last window
// column / row also clear the positions no window covers (odd H or W in floor mode).
template <int KW>
__global__ void __launch_bounds__(256) pool_bwd_window_kernel(float* gx, const int64_t* __restrict__ idx,
                                                              const float* __restrict__ gy, int64_t nout, int H, int W, int HO,
                                                              int WO, int kh, int kw_rt, const void* __restrict__ y, int dty,
                                                              int relu, int beta) {
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= nout) return;
  const int kw = KW > 0 ? KW : kw_rt;
  const int hwo = HO * WO;
  const int64_t plane = o / hwo;
  const int r = (int)(o - plane * hwo), ho = r / WO, wo = r - ho * WO;
  const int am = (int)idx[o];                       // arg-max position inside the plane
  float g = gy[o];
  if (relu && !(bb::ldf(y, o, dty) > 0.f)) g = 0.f;
  float* base = gx + plane * ((int64_t)H * W);
  const int h0 = ho * kh, w0 = wo * kw;
  const int wend = (wo == WO - 1) ? W : w0 + kw;    // last window column also covers the uncovered tail columns
  const int hend = (ho == HO - 1) ? H : h0 + kh;
  for (int h = h0; h < hend; ++h) {
    float* row = base + (int64_t)h * W;
    if (KW == 2 && wend == w0 + 2 && (W & 1) == 0) {
      const int p = h * W + w0;
      float2 v = make_float2(p == am ? g : 0.f, p + 1 == am ? g : 0.f);
      float2* q = reinterpret_cast<float2*>(row + w0);
      if (beta) {
        const float2 old = *q;
        v.x += old.x; v.y += old.y;
      }
      *q = v;
    } else {
      for (int w = w0; w < wend; ++w) {
        const float v = (h * W + w == am) ? g : 0.f;
        row[w] = beta ? row[w] + v : v;
      }
    }
  }
}

// ---- average pooling (linear, floor mode) -------------------------------------------------------------------------
// exclude = 0: every window is divided by the constant divisor (inv = 1/divisor; count_include_pad or an override).
// exclude = 1: count_include_pad=False -- each window is divided by the number of its taps inside the image.
struct AvgGeom {
  int H, W, HO, WO, kh, kw, sh, sw, ph, pw;
  float inv;
  int exclude;
};

// taps of output window (yo, xo) that lie inside the image
__device__ __forceinline__ float avg_count(const AvgGeom& g, int yo, int xo) {
  const int h0 = yo * g.sh - g.ph, w0 = xo * g.sw - g.pw;
  const int rows = min(h0 + g.kh, g.H) - max(h0, 0), cols = min(w0 + g.kw, g.W) - max(w0, 0);
  return (float)(rows * cols);
}

__global__ void avgpool_fwd_kernel(const float* __restrict__ tx, float* ty, int64_t nout, AvgGeom g) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nout) return;
  const int xo = (int)(i % g.WO), yo = (int)((i / g.WO) % g.HO);
  const int64_t plane = i / ((int64_t)g.WO * g.HO);
  const float* src = tx + plane * g.H * g.W;
  float acc = 0.f;
  for (int a = 0; a < g.kh; ++a) {
    const int h = yo * g.sh - g.ph + a;
    if (h < 0 || h >= g.H) continue;
    for (int b = 0; b < g.kw; ++b) {
      const int w = xo * g.sw - g.pw + b;
      if (w >= 0 && w < g.W) acc += src[h * g.W + w];
    }
  }
  ty[i] = g.exclude ? acc / avg_count(g, yo, xo) : acc * g.inv;
}

// gather form of the adjoint: every input pixel sums the windows that cover it (no atomics)
__global__ void avgpool_bwd_kernel(float* gx, const float* __restrict__ gy, int64_t nin, AvgGeom g, int beta) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nin) return;
  const int w = (int)(i % g.W), h = (int)((i / g.W) % g.H);
  const int64_t plane = i / ((int64_t)g.W * g.H);
  const float* src = gy + plane * g.HO * g.WO;
  float acc = 0.f;
  for (int a = 0; a < g.kh; ++a) {
    const int hh = h + g.ph - a;
    if (hh < 0 || hh % g.sh) continue;
    const int yo = hh / g.sh;
    if (yo >= g.HO) continue;
    for (int b = 0; b < g.kw; ++b) {
      const int ww = w + g.pw - b;
      if (ww < 0 || ww % g.sw) continue;
      const int xo = ww / g.sw;
      if (xo < g.WO) acc += g.exclude ? src[yo * g.WO + xo] / avg_count(g, yo, xo) : src[yo * g.WO + xo];
    }
  }
  const float v = g.exclude ? acc : acc * g.inv;
  gx[i] = beta ? gx[i] + v : v;
}

inline unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

int bb_launch_softmax(const bb_node& nd, int pass, cudaStream_t s) {
  if (pass == BB_PASS_BASE_BWD && !(nd.pad0 & 1)) return BB_OK;
  const int64_t rows = nd.dims[0];
  const int D = (int)nd.dims[1];
  const int mode = nd.op == BB_OP_SOFTMAX ? 0 : 1;
  if (rows <= 0) return BB_OK;
  const bool base = pass == BB_PASS_BASE_BWD;
  softmax_rule_kernel<<<blocks(rows, kWarpsPerBlock), kWarpsPerBlock * 32, 0, s>>>(
      nd.base[0], nd.dt[0], reinterpret_cast<const float*>(nd.t[0]), reinterpret_cast<float*>(nd.t[3]),
      reinterpret_cast<const float*>(nd.a[3]), reinterpret_cast<const float*>(nd.at[3]),
      reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]), rows, D, mode, pass, nd.beta[0]);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_launch_nll(const bb_node& nd, int pass, cudaStream_t s) {
  if (pass == BB_PASS_BASE_BWD && !(nd.pad0 & 1)) return BB_OK;
  const int B = (int)nd.dims[0], C = (int)nd.dims[1];
  const int64_t* target = reinterpret_cast<const int64_t*>(nd.aux[0]);
  const float scale = (float)nd.f[0];
  if (pass == BB_PASS_TAN_FWD) {
    if (nd.kind == 0)
      nll_fwd_kernel<<<blocks(B, 256), 256, 0, s>>>(reinterpret_cast<const float*>(nd.t[0]), target,
                                                    reinterpret_cast<float*>(nd.t[3]), B, C, 0, scale);
    else
      nll_fwd_kernel<<<1, 512, 0, s>>>(reinterpret_cast<const float*>(nd.t[0]), target,
                                        reinterpret_cast<float*>(nd.t[3]), B, C, nd.kind, scale);
  } else {
    const bool base = pass == BB_PASS_BASE_BWD;
    nll_bwd_kernel<<<blocks((int64_t)B * C, 256), 256, 0, s>>>(
        reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]), reinterpret_cast<const float*>(base ? nd.a[3] : nd.at[3]),
        target, B, C, nd.kind, scale, nd.beta[0]);
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_launch_bce(const bb_node& nd, int pass, cudaStream_t s) {
  if (pass == BB_PASS_BASE_BWD && !(nd.pad0 & 1)) return BB_OK;
  const int64_t n = nd.n;
  const float* y = reinterpret_cast<const float*>(nd.aux[0]);
  if (pass == BB_PASS_TAN_FWD) {
    bce_fwd_kernel<<<1, 512, 0, s>>>(nd.base[0], nd.dt[0], y, reinterpret_cast<const float*>(nd.t[0]),
                                      reinterpret_cast<float*>(nd.t[3]), n);
  } else {
    const bool base = pass == BB_PASS_BASE_BWD;
    bce_bwd_kernel<<<blocks(n, 256), 256, 0, s>>>(nd.base[0], nd.dt[0], y, reinterpret_cast<const float*>(nd.t[0]),
                                                  reinterpret_cast<const float*>(nd.a[3]),
                                                  reinterpret_cast<const float*>(nd.at[3]),
                                                  reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]), n, pass, nd.beta[0]);
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_launch_embedding(const bb_node& nd, int pass, cudaStream_t s) {
  const int64_t nidx = nd.dims[0];
  const int D = (int)nd.dims[1];
  const int64_t* idx = reinterpret_cast<const int64_t*>(nd.aux[0]);
  if (nidx <= 0) return BB_OK;
  if (pass == BB_PASS_TAN_FWD) {
    emb_fwd_kernel<<<blocks(nidx * D, 256), 256, 0, s>>>(reinterpret_cast<const float*>(nd.t[0]), idx,
                                                         reinterpret_cast<float*>(nd.t[3]), nidx, D);
  } else if (pass == BB_PASS_TAN_BWD) {
    const int64_t* seg = reinterpret_cast<const int64_t*>(nd.aux[1]);
    if (seg == nullptr) return BB_ERR_ARG;
    const dim3 grid((unsigned)((D + 31) / 32), (unsigned)(nidx < 128 ? nidx : 128));
    emb_bwd_kernel<<<grid, kEmbLanes * 32, 0, s>>>(reinterpret_cast<float*>(nd.at[0]), idx, seg,
                                                   reinterpret_cast<const float*>(nd.at[3]), nidx, D, nd.dims[3]);
  } else {
    return BB_OK;  // base adjoint of a parameter table is never needed
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_launch_maxpool2d(const bb_node& nd, int pass, cudaStream_t s) {
  if (pass == BB_PASS_BASE_BWD && !(nd.pad0 & 1)) return BB_OK;
  const int64_t planes = nd.dims[0];
  const int hw_in = (int)nd.dims[1], hw_out = (int)nd.dims[2];
  const int64_t nout = planes * hw_out;
  const int64_t* idx = reinterpret_cast<const int64_t*>(nd.aux[0]);
  if (nout <= 0) return BB_OK;
  const int relu = nd.kind & 1, disjoint = (nd.kind >> 1) & 1;
  if (pass == BB_PASS_TAN_FWD) {
    pool_fwd_kernel<<<blocks(nout, 256), 256, 0, s>>>(reinterpret_cast<const float*>(nd.t[0]), idx,
                                                      reinterpret_cast<float*>(nd.t[3]), nout, hw_in, hw_out, nd.base[3],
                                                      nd.dt[3], relu);
  } else {
    const bool base = pass == BB_PASS_BASE_BWD;
    float* gx = reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]);
    const float* gy = reinterpret_cast<const float*>(base ? nd.a[3] : nd.at[3]);
    if (disjoint) {
      const int H = (int)nd.dims[3], W = (int)nd.dims[4], HO = (int)nd.dims[5], WO = (int)nd.dims[6];
      const int kh = (int)nd.dims[7], kw = (int)nd.dims[8];
      if (kw == 2)
        pool_bwd_window_kernel<2><<<blocks(nout, 256), 256, 0, s>>>(gx, idx, gy, nout, H, W, HO, WO, kh, kw, nd.base[3],
                                                                    nd.dt[3], relu, nd.beta[0]);
      else
        pool_bwd_window_kernel<0><<<blocks(nout, 256), 256, 0, s>>>(gx, idx, gy, nout, H, W, HO, WO, kh, kw, nd.base[3],
                                                                    nd.dt[3], relu, nd.beta[0]);
    } else {
      pool_bwd_kernel<<<blocks(nout, 256), 256, 0, s>>>(gx, idx, gy, nout, hw_in, hw_out, nd.base[3], nd.dt[3], relu);
    }
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_launch_avgpool2d(const bb_node& nd, int pass, cudaStream_t s) {
  if (pass == BB_PASS_BASE_BWD && !(nd.pad0 & 1)) return BB_OK;
  AvgGeom g;
  const int64_t planes = nd.dims[0];
  g.H = (int)nd.dims[1]; g.W = (int)nd.dims[2]; g.HO = (int)nd.dims[3]; g.WO = (int)nd.dims[4];
  g.kh = (int)nd.dims[5]; g.kw = (int)nd.dims[6]; g.sh = (int)nd.dims[7]; g.sw = (int)nd.dims[8];
  g.ph = (int)nd.dims[9]; g.pw = (int)nd.dims[10];
  g.inv = (float)nd.f[0];
  g.exclude = nd.kind & 1;
  if (pass == BB_PASS_TAN_FWD) {
    const int64_t nout = planes * g.HO * g.WO;
    if (nout <= 0) return BB_OK;
    avgpool_fwd_kernel<<<blocks(nout, 256), 256, 0, s>>>(reinterpret_cast<const float*>(nd.t[0]),
                                                         reinterpret_cast<float*>(nd.t[3]), nout, g);
  } else {
    const bool base = pass == BB_PASS_BASE_BWD;
    const int64_t nin = planes * g.H * g.W;
    if (nin <= 0) return BB_OK;
    avgpool_bwd_kernel<<<blocks(nin, 256), 256, 0, s>>>(reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]),
                                                        reinterpret_cast<const float*>(base ? nd.a[3] : nd.at[3]), nin, g,
                                                        nd.beta[0]);
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}
