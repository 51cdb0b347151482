// K1-K4: flat-arena kernels of the Neumann / CG / finite-difference K-loops (SURVEY.md §8a).
//
// All vectors (v, p, x, r, hv) are fp32 arenas with the lower problem's parameters laid out back to
// back, every tensor's offset rounded up to 4 floats, padding zero -- so each kernel is a pure
// 128-bit streaming pass and the dot products need no masking.  CG's alpha/beta and the finite
// difference eps never leave the device (the reference does a host sync per call, darts.py:35).
//
//   K1  bb_neumann_update   v <- v - alpha*hv ; p <- p + v              (reference neumann.py:63-64)
//   K2  bb_cg_dots          rr = r.r (first iter), php=(cg_alpha*hp).p ; alpha = rr/php   (cg.py:42-47)
//   K3  bb_cg_update_xr     x += alpha p ; r -= alpha hp ; rr' = r.r ; beta = rr'/rr      (cg.py:49-52)
//       bb_cg_update_p      p <- r + beta p                                                (cg.py:53)
//   K4  bb_mt_sumsq / bb_fd_eps / bb_mt_axpby / bb_mt_fd_combine                            (darts.py:30-67)
#include "bb_common.cuh"
#include "../../include/betty_b200.h"

namespace {

constexpr int kThreads = 512;
constexpr int kBlocksPerSM = 4;
constexpr int kMaxGrid = BB_SM_COUNT * kBlocksPerSM;  // 528 persistent-ish blocks, grid-stride

inline int grid_for(int64_t n4) {
  int64_t want = (n4 + kThreads - 1) / kThreads;
  if (want < 1) want = 1;
  if (want > kMaxGrid) want = kMaxGrid;
  return (int)want;
}

// ---- K1 -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) neumann_update_kernel(float* __restrict__ v, float* __restrict__ p,
                                                                  const float* __restrict__ hv, float alpha,
                                                                  float shift, int64_t n4) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 a = bb::ld4(v + 4 * i);
    const float4 h = bb::ld4_stream(hv + 4 * i);
    float4 q = bb::ld4(p + 4 * i);
    // v - alpha*(hv + shift*v): `shift` folds a declared c*I curvature term into the update
    if (shift != 0.f) {
      a.x = a.x - alpha * fmaf(shift, a.x, h.x); a.y = a.y - alpha * fmaf(shift, a.y, h.y);
      a.z = a.z - alpha * fmaf(shift, a.z, h.z); a.w = a.w - alpha * fmaf(shift, a.w, h.w);
    } else {
      a.x = a.x - alpha * h.x; a.y = a.y - alpha * h.y; a.z = a.z - alpha * h.z; a.w = a.w - alpha * h.w;
    }
    q.x += a.x; q.y += a.y; q.z += a.z; q.w += a.w;
    bb::st4(v + 4 * i, a);
    bb::st4(p + 4 * i, q);
  }
}

__global__ void __launch_bounds__(kThreads) scale_kernel(float* __restrict__ out, const float* __restrict__ in,
                                                         float c, int64_t n4) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 a = bb::ld4(in + 4 * i);
    a.x *= c; a.y *= c; a.z *= c; a.w *= c;
    bb::st4(out + 4 * i, a);
  }
}

// ---- K2 -------------------------------------------------------------------------------------
struct Ws {
  bb_kloop_scalars* s;
  unsigned int* ticket;
  double* partials;  // 2 * kMaxGrid (overwritten by every reduction)
  double* slots;     // kMaxGrid accumulation slots, kept zero between launches
};

__device__ __forceinline__ Ws ws_view(void* ws) {
  Ws w;
  char* b = reinterpret_cast<char*>(ws);
  w.s = reinterpret_cast<bb_kloop_scalars*>(b);
  w.ticket = reinterpret_cast<unsigned int*>(b + 256);
  w.partials = reinterpret_cast<double*>(b + 512);
  w.slots = w.partials + 2 * kMaxGrid;
  return w;
}

__global__ void __launch_bounds__(kThreads) cg_dots_kernel(const float* __restrict__ r, const float* __restrict__ hp,
                                                           const float* __restrict__ p, float cg_alpha,
                                                           float shift, int first, int64_t n4, void* wsraw) {
  __shared__ double red[32];
  Ws w = ws_view(wsraw);
  float acc_php = 0.f, acc_rr = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 h = bb::ld4(hp + 4 * i);
    const float4 q = bb::ld4(p + 4 * i);
    if (shift != 0.f) {   // H p = hp + shift p: a declared c*I curvature term folded into the vector pass
      h.x = fmaf(shift, q.x, h.x); h.y = fmaf(shift, q.y, h.y); h.z = fmaf(shift, q.z, h.z); h.w = fmaf(shift, q.w, h.w);
    }
    acc_php += (cg_alpha * h.x) * q.x + (cg_alpha * h.y) * q.y + (cg_alpha * h.z) * q.z + (cg_alpha * h.w) * q.w;
    if (first) {
      const float4 a = bb::ld4(r + 4 * i);
      acc_rr += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
    }
  }
  double b_php = bb::block_sum<double>((double)acc_php, red);
  double b_rr = first ? bb::block_sum<double>((double)acc_rr, red) : 0.0;
  // two partial arrays; one ticket covers both
  if (threadIdx.x == 0 && first) w.partials[kMaxGrid + blockIdx.x] = b_rr;
  double php;
  if (bb::grid_sum_finish(b_php, w.partials, w.ticket, &php, red)) {
    if (first) {
      double rr = 0.0;
      for (unsigned int i = 0; i < gridDim.x; ++i) rr += w.partials[kMaxGrid + i];
      w.s->rr = rr;
    }
    w.s->php = php;
    w.s->alpha = w.s->rr / php;
  }
}

// rr = r.r before the first iteration (so that the captured iteration body is identical for all k)
__global__ void __launch_bounds__(kThreads) cg_init_kernel(const float* __restrict__ r, int64_t n4, void* wsraw) {
  __shared__ double red[32];
  Ws w = ws_view(wsraw);
  float acc = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 a = bb::ld4(r + 4 * i);
    acc += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
  }
  double b = bb::block_sum<double>((double)acc, red);
  double rr;
  if (bb::grid_sum_finish(b, w.partials, w.ticket, &rr, red)) w.s->rr = rr;
}

// ---- K3 -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) cg_update_xr_kernel(float* __restrict__ x, float* __restrict__ r,
                                                                const float* __restrict__ p,
                                                                const float* __restrict__ hp, float shift,
                                                                int64_t n4, void* wsraw) {
  __shared__ double red[32];
  Ws w = ws_view(wsraw);
  const float alpha = (float)w.s->alpha;
  float acc = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 xx = bb::ld4(x + 4 * i);
    float4 rr = bb::ld4(r + 4 * i);
    const float4 q = bb::ld4(p + 4 * i);
    float4 h = bb::ld4_stream(hp + 4 * i);
    if (shift != 0.f) {
      h.x = fmaf(shift, q.x, h.x); h.y = fmaf(shift, q.y, h.y); h.z = fmaf(shift, q.z, h.z); h.w = fmaf(shift, q.w, h.w);
    }
    xx.x += alpha * q.x; xx.y += alpha * q.y; xx.z += alpha * q.z; xx.w += alpha * q.w;
    rr.x -= alpha * h.x; rr.y -= alpha * h.y; rr.z -= alpha * h.z; rr.w -= alpha * h.w;
    acc += rr.x * rr.x + rr.y * rr.y + rr.z * rr.z + rr.w * rr.w;
    bb::st4(x + 4 * i, xx);
    bb::st4(r + 4 * i, rr);
  }
  double b = bb::block_sum<double>((double)acc, red);
  double rr_new;
  if (bb::grid_sum_finish(b, w.partials, w.ticket, &rr_new, red)) {
    w.s->rr_new = rr_new;
    w.s->beta = rr_new / w.s->rr;
    w.s->rr = rr_new;
  }
}

__global__ void __launch_bounds__(kThreads) cg_update_p_kernel(float* __restrict__ p, const float* __restrict__ r,
                                                               int64_t n4, const void* wsraw) {
  const float beta = (float)reinterpret_cast<const bb_kloop_scalars*>(wsraw)->beta;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 rr = bb::ld4(r + 4 * i);
    float4 q = bb::ld4(p + 4 * i);
    q.x = rr.x + beta * q.x; q.y = rr.y + beta * q.y; q.z = rr.z + beta * q.z; q.w = rr.w + beta * q.w;
    bb::st4(p + 4 * i, q);
  }
}

// ---- K4 + arena packing: multi-tensor kernels driven by a chunk table -----------------------
// table[c] = {a, b, n}: chunk c covers n (<= BB_MT_CHUNK) floats at a / b.
constexpr int kMtThreads = 256;

__global__ void __launch_bounds__(kMtThreads) mt_copy_kernel(const bb_mt_chunk* __restrict__ tab, int dir) {
  const bb_mt_chunk c = tab[blockIdx.x];
  const float* src = reinterpret_cast<const float*>(dir == 0 ? c.a : c.b);
  float* dst = reinterpret_cast<float*>(dir == 0 ? c.b : c.a);
  const bool vec = (((uintptr_t)src | (uintptr_t)dst) & 15) == 0;
  const int n4 = vec ? c.n >> 2 : 0;
  for (int i = threadIdx.x; i < n4; i += kMtThreads) bb::st4(dst + 4 * i, bb::ld4(src + 4 * i));
  for (int i = 4 * n4 + threadIdx.x; i < c.n; i += kMtThreads) dst[i] = src[i];
}

// b <- coef_a * scale_dev * a + coef_b * b   (scale_dev may be null => 1; a may alias b)
__global__ void __launch_bounds__(kMtThreads) mt_axpby_kernel(const bb_mt_chunk* __restrict__ tab, float coef_a,
                                                              const double* __restrict__ scale_dev, float coef_b) {
  const bb_mt_chunk c = tab[blockIdx.x];
  const float s = coef_a * (scale_dev ? (float)(*scale_dev) : 1.f);
  const float* a = reinterpret_cast<const float*>(c.a);
  float* b = reinterpret_cast<float*>(c.b);
  // 128-bit body when both chunk pointers are 16-byte aligned (chunks start at tensor base + k*BB_MT_CHUNK floats,
  // so this is the case for every chunk of an allocator-aligned tensor), scalar tail / fallback otherwise
  const bool vec = (((uintptr_t)a | (uintptr_t)b) & 15) == 0;
  const int n4 = vec ? c.n >> 2 : 0;
  for (int i = threadIdx.x; i < n4; i += kMtThreads) {
    const float4 va = bb::ld4(a + 4 * i);
    float4 vb;
    if (coef_b == 0.f) {
      vb = make_float4(s * va.x, s * va.y, s * va.z, s * va.w);
    } else {
      vb = bb::ld4(b + 4 * i);
      vb.x = s * va.x + coef_b * vb.x; vb.y = s * va.y + coef_b * vb.y;
      vb.z = s * va.z + coef_b * vb.z; vb.w = s * va.w + coef_b * vb.w;
    }
    bb::st4(b + 4 * i, vb);
  }
  if (coef_b == 0.f) {
    for (int i = 4 * n4 + threadIdx.x; i < c.n; i += kMtThreads) b[i] = s * a[i];
  } else {
    for (int i = 4 * n4 + threadIdx.x; i < c.n; i += kMtThreads) b[i] = s * a[i] + coef_b * b[i];
  }
}

__global__ void __launch_bounds__(kMtThreads) mt_sumsq_kernel(const bb_mt_chunk* __restrict__ tab, void* wsraw) {
  __shared__ double red[32];
  Ws w = ws_view(wsraw);
  const bb_mt_chunk c = tab[blockIdx.x];
  const float* a = reinterpret_cast<const float*>(c.a);
  float acc = 0.f;
  const int n4 = (((uintptr_t)a) & 15) == 0 ? c.n >> 2 : 0;
  for (int i = threadIdx.x; i < n4; i += kMtThreads) {
    const float4 v = bb::ld4(a + 4 * i);
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (int i = 4 * n4 + threadIdx.x; i < c.n; i += kMtThreads) acc += a[i] * a[i];
  double b = bb::block_sum<double>((double)acc, red);
  // chunk count can exceed kMaxGrid: accumulate with a fixed-order scheme per slot
  if (threadIdx.x == 0) atomicAdd(&w.slots[blockIdx.x % kMaxGrid], b);
  __shared__ bool last;
  if (threadIdx.x == 0) {
    __threadfence();
    last = (atomicAdd(w.ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double s = 0.0;
    for (int i = 0; i < kMaxGrid; ++i) {
      s += w.slots[i];
      w.slots[i] = 0.0;
    }
    w.s->sumsq = s;
    *w.ticket = 0u;
  }
}

__global__ void fd_eps_kernel(void* wsraw, double darts_alpha) {
  bb_kloop_scalars* s = reinterpret_cast<bb_kloop_scalars*>(wsraw);
  // reference darts.py:30-35: eps = R / (||v|| + 1e-15); fp32 norm in the reference
  const float nrm = sqrtf((float)s->sumsq);
  s->eps = darts_alpha / ((double)nrm + 1e-15);
  s->inv_2eps = 1.0 / (2.0 * s->eps);
}

// out(a) = (a - b) * inv_2eps   (a = g_minus, b = g_plus, in place on a)
__global__ void __launch_bounds__(kMtThreads) mt_fd_combine_kernel(const bb_mt_chunk* __restrict__ tab,
                                                                   const void* wsraw) {
  const float s = (float)reinterpret_cast<const bb_kloop_scalars*>(wsraw)->inv_2eps;
  const bb_mt_chunk c = tab[blockIdx.x];
  float* a = reinterpret_cast<float*>(c.a);
  const float* b = reinterpret_cast<const float*>(c.b);
  const bool vec = (((uintptr_t)a | (uintptr_t)b) & 15) == 0;
  const int n4 = vec ? c.n >> 2 : 0;
  for (int i = threadIdx.x; i < n4; i += kMtThreads) {
    float4 va = bb::ld4(a + 4 * i);
    const float4 vb = bb::ld4(b + 4 * i);
    va.x = (va.x - vb.x) * s; va.y = (va.y - vb.y) * s; va.z = (va.z - vb.z) * s; va.w = (va.w - vb.w) * s;
    bb::st4(a + 4 * i, va);
  }
  for (int i = 4 * n4 + threadIdx.x; i < c.n; i += kMtThreads) a[i] = (a[i] - b[i]) * s;
}

// SAMA's Adam preconditioner (reference hypergradient/utils.py:37-63), one chunk row per <= BB_MT_CHUNK floats:
//   m_old = (m - (1-b1) g)/b1 (0 if b1 == 0);  s_old = (s - (1-b2) g^2)/b2
//   out = v * lr * ((1-b1) b2 s_old - b1 (1-b2) g m_old) / (sqrt(s) + eps)^3        missing state tensors read as 0
__global__ void __launch_bounds__(kMtThreads) mt_adam_precondition_kernel(const bb_mt_adam_chunk* __restrict__ tab) {
  const bb_mt_adam_chunk c = tab[blockIdx.x];
  const float* v = reinterpret_cast<const float*>(c.v);
  const float* g = reinterpret_cast<const float*>(c.g);
  const float* m = reinterpret_cast<const float*>(c.m);
  const float* q = reinterpret_cast<const float*>(c.s);
  float* out = reinterpret_cast<float*>(c.out);
  const float b1 = c.beta1, b2 = c.beta2;
  for (int i = threadIdx.x; i < c.n; i += kMtThreads) {
    const float gi = g ? g[i] : 0.f, mi = m ? m[i] : 0.f, si = q ? q[i] : 0.f;
    const float m_old = b1 != 0.f ? (mi - (1.f - b1) * gi) / b1 : 0.f;
    const float s_old = (si - (1.f - b2) * gi * gi) / b2;
    float scale = (1.f - b1) * b2 * s_old - b1 * (1.f - b2) * gi * m_old;
    const float d = sqrtf(si) + c.eps;
    scale /= d * d * d;
    out[i] = v[i] * scale * c.lr;
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
extern "C" {

int bb_mt_adam_precondition(const bb_mt_adam_chunk* table_dev, int nchunks, void* stream) {
  if (nchunks <= 0) return BB_OK;
  mt_adam_precondition_kernel<<<nchunks, kMtThreads, 0, (cudaStream_t)stream>>>(table_dev);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_kloop_ws_bytes(void) { return 512 + 3 * kMaxGrid * (int)sizeof(double); }

int bb_neumann_update(float* v, float* p, const float* hv, float alpha, float shift, int64_t n, void* stream) {
  if ((n & 3) != 0) return BB_ERR_ARG;
  if (n == 0) return BB_OK;
  const int64_t n4 = n >> 2;
  neumann_update_kernel<<<grid_for(n4), kThreads, 0, (cudaStream_t)stream>>>(v, p, hv, alpha, shift, n4);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_scale(float* out, const float* in, float c, int64_t n, void* stream) {
  if ((n & 3) != 0) return BB_ERR_ARG;
  if (n == 0) return BB_OK;
  const int64_t n4 = n >> 2;
  scale_kernel<<<grid_for(n4), kThreads, 0, (cudaStream_t)stream>>>(out, in, c, n4);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_cg_dots(const float* r, const float* hp, const float* p, float cg_alpha, float shift, int first, int64_t n,
               void* ws, void* stream) {
  if ((n & 3) != 0) return BB_ERR_ARG;
  const int64_t n4 = n >> 2;
  cg_dots_kernel<<<grid_for(n4), kThreads, 0, (cudaStream_t)stream>>>(r, hp, p, cg_alpha, shift, first, n4, ws);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_cg_init(const float* r, int64_t n, void* ws, void* stream) {
  if ((n & 3) != 0) return BB_ERR_ARG;
  const int64_t n4 = n >> 2;
  cg_init_kernel<<<grid_for(n4), kThreads, 0, (cudaStream_t)stream>>>(r, n4, ws);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_cg_update_xr(float* x, float* r, const float* p, const float* hp, float shift, int64_t n, void* ws,
                    void* stream) {
  if ((n & 3) != 0) return BB_ERR_ARG;
  const int64_t n4 = n >> 2;
  cg_update_xr_kernel<<<grid_for(n4), kThreads, 0, (cudaStream_t)stream>>>(x, r, p, hp, shift, n4, ws);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_cg_update_p(float* p, const float* r, int64_t n, const void* ws, void* stream) {
  if ((n & 3) != 0) return BB_ERR_ARG;
  const int64_t n4 = n >> 2;
  cg_update_p_kernel<<<grid_for(n4), kThreads, 0, (cudaStream_t)stream>>>(p, r, n4, ws);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_mt_copy(const bb_mt_chunk* table_dev, int nchunks, int dir, void* stream) {
  if (nchunks <= 0) return BB_OK;
  mt_copy_kernel<<<nchunks, kMtThreads, 0, (cudaStream_t)stream>>>(table_dev, dir);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_mt_axpby(const bb_mt_chunk* table_dev, int nchunks, float coef_a, const double* scale_dev, float coef_b,
                void* stream) {
  if (nchunks <= 0) return BB_OK;
  mt_axpby_kernel<<<nchunks, kMtThreads, 0, (cudaStream_t)stream>>>(table_dev, coef_a, scale_dev, coef_b);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_mt_sumsq(const bb_mt_chunk* table_dev, int nchunks, void* ws, void* stream) {
  if (nchunks <= 0) return BB_ERR_ARG;
  mt_sumsq_kernel<<<nchunks, kMtThreads, 0, (cudaStream_t)stream>>>(table_dev, ws);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_fd_eps(void* ws, double darts_alpha, void* stream) {
  fd_eps_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(ws, darts_alpha);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_mt_fd_combine(const bb_mt_chunk* table_dev, int nchunks, const void* ws, void* stream) {
  if (nchunks <= 0) return BB_OK;
  mt_fd_combine_kernel<<<nchunks, kMtThreads, 0, (cudaStream_t)stream>>>(table_dev, ws);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // extern "C"
