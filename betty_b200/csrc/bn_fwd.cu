// Prologue (SURVEY.md 8 f2): training-mode BatchNorm FORWARD of the lower problem's own forward pass.
//
// The prologue of every plugin call runs the user's lower forward once (reference neumann.py:31, cg.py:27).  On a
// channels-first activation of 64 channels PyTorch's `batch_norm_collect_statistics_kernel` launches one block per
// channel (64 blocks for the whole GPU, strided bf16 reads).  When asked to (BB200_PROLOGUE_BN_MIN, opt-in: see
// betty_b200/trace.py for why bit-identical base activations matter for the bf16 parity bar) the dispatch-mode recorder (betty_b200/trace.py) executes aten.native_batch_norm(training=True) on
// large CUDA inputs with these three kernels instead -- same outputs (out, save_mean, save_invstd), same formula
//     out = gamma * (x - mean) * invstd + beta,   invstd = rsqrt(biased_var + eps)
// with the statistics reduced in fp64 in a fixed order (bit-reproducible run to run):
//
//   bn_fwd_stats_kernel    grid (S, C): block (s, c) sums x and x^2 of channel c over the planes n = s, s+S, ...
//                          with 16-byte loads; one fp64 (sum, sumsq) partial per block
//   bn_fwd_finalize_kernel one thread per channel adds the S partials in order -> mean, invstd, unbiased variance
//   bn_fwd_apply_kernel    one pass: 16-byte loads / stores over the N*C planes
//
// HBM bound: x read twice, out written once (the second read partly hits L2 when the tensor is not much larger).
#include "../../include/betty_b200.h"
#include "bb_common.cuh"

namespace {

template <typename T>
struct Vec16;   // 16-byte vector of T and its conversion to floats
template <>
struct Vec16<float> {
  static constexpr int N = 4;
  __device__ static void load(const float* p, float* v) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  }
  __device__ static void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <>
struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static void load(const __nv_bfloat16* p, float* v) {
    const uint4 q = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[2 * i] = __uint_as_float(w[i] << 16);
      v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static void store(__nv_bfloat16* p, const float* v) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  }
};

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ void from_f(float* p, float v) { *p = v; }
__device__ __forceinline__ void from_f(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// VEC: every plane (HW elements) starts 16-byte aligned and HW is a multiple of the vector length
template <typename T, bool VEC>
__global__ void __launch_bounds__(256) bn_fwd_stats_kernel(const T* __restrict__ x, double* __restrict__ partials,
                                                           int64_t N, int C, int64_t HW) {
  constexpr int V = Vec16<T>::N;
  const int c = blockIdx.y, S = gridDim.x;
  double sum = 0.0, sq = 0.0;
  for (int64_t n = blockIdx.x; n < N; n += S) {
    const T* plane = x + (n * C + c) * HW;
    // fp32 accumulation inside one plane slice per thread (<= HW / 256 + 1 terms), fp64 across planes
    float s = 0.f, q = 0.f;
    if (VEC) {
      const int64_t nv = HW / V;
      for (int64_t i = threadIdx.x; i < nv; i += blockDim.x) {
        float v[V];
        Vec16<T>::load(plane + i * V, v);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          s += v[k];
          q = fmaf(v[k], v[k], q);
        }
      }
    } else {
      for (int64_t i = threadIdx.x; i < HW; i += blockDim.x) {
        const float v = to_f(plane[i]);
        s += v;
        q = fmaf(v, v, q);
      }
    }
    sum += (double)s;
    sq += (double)q;
  }
  __shared__ double red[32];
  sum = bb::block_sum<double>(sum, red);
  sq = bb::block_sum<double>(sq, red);
  if (threadIdx.x == 0) {
    partials[((int64_t)c * S + blockIdx.x) * 2] = sum;
    partials[((int64_t)c * S + blockIdx.x) * 2 + 1] = sq;
  }
}

__global__ void bn_fwd_finalize_kernel(const double* __restrict__ partials, int S, int C, double count, double eps,
                                       float* __restrict__ mean, float* __restrict__ invstd,
                                       float* __restrict__ var_unbiased) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double sum = 0.0, sq = 0.0;
  for (int s = 0; s < S; ++s) {
    sum += partials[((int64_t)c * S + s) * 2];
    sq += partials[((int64_t)c * S + s) * 2 + 1];
  }
  const double m = sum / count;
  double var = sq / count - m * m;
  if (var < 0.0) var = 0.0;
  mean[c] = (float)m;
  invstd[c] = (float)(1.0 / sqrt(var + eps));
  if (var_unbiased) var_unbiased[c] = (float)(count > 1.0 ? var * count / (count - 1.0) : var);
}

template <typename T, bool VEC>
__global__ void __launch_bounds__(256) bn_fwd_apply_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                           const float* __restrict__ mean,
                                                           const float* __restrict__ invstd,
                                                           const float* __restrict__ weight,
                                                           const float* __restrict__ bias, int64_t planes, int C,
                                                           int64_t HW) {
  constexpr int V = Vec16<T>::N;
  for (int64_t pl = blockIdx.x; pl < planes; pl += gridDim.x) {
    const int c = (int)(pl % C);
    const float m = mean[c], is = invstd[c];
    const float g = weight ? weight[c] : 1.f, b = bias ? bias[c] : 0.f;
    const T* src = x + pl * HW;
    T* dst = y + pl * HW;
    if (VEC) {
      const int64_t nv = HW / V;
      for (int64_t i = threadIdx.x; i < nv; i += blockDim.x) {
        float v[V];
        Vec16<T>::load(src + i * V, v);
#pragma unroll
        for (int k = 0; k < V; ++k) v[k] = g * (v[k] - m) * is + b;
        Vec16<T>::store(dst + i * V, v);
      }
    } else {
      for (int64_t i = threadIdx.x; i < HW; i += blockDim.x) from_f(dst + i, g * (to_f(src[i]) - m) * is + b);
    }
  }
}

template <typename T>
int run(const T* x, const float* w, const float* b, double eps, T* y, float* mean, float* invstd, float* var_unb,
        double* ws, int S, int64_t N, int C, int64_t HW, cudaStream_t s) {
  constexpr int V = Vec16<T>::N;
  const bool vec = (HW % V == 0) && (reinterpret_cast<uintptr_t>(x) % 16 == 0) && (reinterpret_cast<uintptr_t>(y) % 16 == 0);
  if (vec) bn_fwd_stats_kernel<T, true><<<dim3(S, C), 256, 0, s>>>(x, ws, N, C, HW);
  else bn_fwd_stats_kernel<T, false><<<dim3(S, C), 256, 0, s>>>(x, ws, N, C, HW);
  BB_LAUNCH_CHECK();
  bn_fwd_finalize_kernel<<<(C + 127) / 128, 128, 0, s>>>(ws, S, C, (double)N * (double)HW, eps, mean, invstd, var_unb);
  BB_LAUNCH_CHECK();
  const int64_t planes = N * C;
  const int64_t cap = (int64_t)BB_SM_COUNT * 8;
  const unsigned grid = (unsigned)(planes < cap ? planes : cap);
  if (vec) bn_fwd_apply_kernel<T, true><<<grid, 256, 0, s>>>(x, y, mean, invstd, w, b, planes, C, HW);
  else bn_fwd_apply_kernel<T, false><<<grid, 256, 0, s>>>(x, y, mean, invstd, w, b, planes, C, HW);
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace

extern "C" int bb_bn_forward_splits(int64_t N, int C) {
  // enough blocks for ~8 per SM, never more than one plane stride per image
  int64_t S = ((int64_t)BB_SM_COUNT * 8 + C - 1) / C;
  if (S > N) S = N;
  if (S < 1) S = 1;
  if (S > 4096) S = 4096;
  return (int)S;
}

extern "C" int bb_bn_forward(const void* x, int dtype, const float* weight, const float* bias, double eps, void* y,
                             float* mean, float* invstd, float* var_unbiased, double* ws, int64_t N, int C, int64_t HW,
                             void* stream) {
  if (!x || !y || !mean || !invstd || !ws || N < 1 || C < 1 || HW < 1 || C > 65535) return BB_ERR_ARG;
  const int S = bb_bn_forward_splits(N, C);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == BB_F32)
    return run<float>(reinterpret_cast<const float*>(x), weight, bias, eps, reinterpret_cast<float*>(y), mean, invstd,
                      var_unbiased, ws, S, N, C, HW, s);
  if (dtype == BB_BF16)
    return run<__nv_bfloat16>(reinterpret_cast<const __nv_bfloat16*>(x), weight, bias, eps,
                              reinterpret_cast<__nv_bfloat16*>(y), mean, invstd, var_unbiased, ws, S, N, C, HW, s);
  return BB_ERR_UNSUPPORTED;
}
