// Shared device helpers for the betty_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define BB_OK 0
#define BB_ERR_ARG (-1)
#define BB_ERR_UNSUPPORTED (-2)

#define BB_SM_COUNT 132  // H100 SXM; grids are sized in multiples of this

#define BB_CUDA_TRY(expr)                 \
  do {                                    \
    cudaError_t _e = (expr);              \
    if (_e != cudaSuccess) return (int)_e; \
  } while (0)

#define BB_LAUNCH_CHECK()                    \
  do {                                       \
    cudaError_t _e = cudaPeekAtLastError();  \
    if (_e != cudaSuccess) return (int)_e;   \
  } while (0)

// dtype tags for *base* tensors recorded from the forward pass (tangents/adjoints are always fp32)
#define BB_F32 0
#define BB_BF16 1
#define BB_F16 2

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device setting: a launcher remembers it per device,
// so a process driving several GPUs opts in on each of them.
struct BbOncePerDevice {
  unsigned long long done = 0;
  bool need() {
    int d = 0;
    cudaGetDevice(&d);
    const unsigned long long bit = 1ull << (d & 63);
    if (done & bit) return false;
    done |= bit;
    return true;
  }
};

namespace bb {

__device__ __forceinline__ float ldf(const void* p, int64_t i, int dt) {
  if (dt == BB_F32) return reinterpret_cast<const float*>(p)[i];
  if (dt == BB_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  return __half2float(reinterpret_cast<const __half*>(p)[i]);   // fp16 autocast (reference precision="fp16")
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// streaming (read-once) 128-bit load that does not allocate in L1
__device__ __forceinline__ float4 ld4_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum (all threads get nothing; thread 0 gets the result). `red` needs 32 slots.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (threadIdx.x < nw) ? red[threadIdx.x] : T(0);
  if (wid == 0) r = warp_sum(r);
  __syncthreads();
  return r;
}

// Deterministic two-stage grid reduction: every block stores its partial, the last block to arrive
// (ticket) adds the partials in block order in fp64.  Returns true in thread 0 of the last block,
// with *out set.  `ticket` must be zero on entry and is reset for the next launch.
__device__ __forceinline__ bool grid_sum_finish(double partial, double* partials, unsigned int* ticket,
                                                double* out, double* red /*32*/) {
  __shared__ bool is_last;
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = partial;
    __threadfence();
    unsigned int t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  double acc = 0.0;
  for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) acc += partials[i];
  // fixed-shape tree => deterministic for a fixed grid
  acc = block_sum<double>(acc, red);
  if (threadIdx.x == 0) {
    *out = acc;
    *ticket = 0u;
    return true;
  }
  return false;
}

}  // namespace bb
