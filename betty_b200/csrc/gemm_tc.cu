// K5 tensor-core path: dual-product GEMM on the Hopper tensor cores (wgmma.mma_async with bf16 operands from
// shared memory, fp32 accumulation in registers) for the bf16-autocast configurations.
//
//   D[m][n] (beta/atomic)= sum over up to two operand pairs p of  sum_k A_p[m][k] * B_p[k][n]   (+ bias[n])
//
// Operand staging is done by the threads themselves rather than by TMA because the second-order operands are
// heterogeneous: base activations / weights are bf16 (autocast), tangents and adjoints are fp32 slices of arenas,
// and half of them are consumed through transposed views.  The threads read global memory with whatever strides
// the operand has, convert to bf16 and write the canonical K-major SWIZZLE_128B layout the wgmma shared-memory
// descriptors expect (row pitch 128 B, 16-byte chunk index XOR (row % 8), 8-row groups 1024 B apart), then publish
// the stage with a generic->async proxy fence and a CTA barrier.  Each of the two warpgroups then issues
// 4 x wgmma m64nBNk16 per 64-wide k-block for its 64 rows of the 128-row tile; the MMAs of k-block i run while
// k-block i+1 is staged (3-stage ring, wait_group 1).  The epilogue stores the register accumulators with beta /
// atomic split-K / bias handling.
//
// 256 threads = 2 warpgroups, 24-32 KB per stage.
#include <cuda_bf16.h>
#include <stdlib.h>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "gemm_tc.h"
#include "plan.h"
#include "tc_ptx.cuh"

namespace {

constexpr int BM = 128, BK = 64, STAGES = 3;   // BN = 64 or 128 (template)
constexpr int NPROD = 256;                   // staging threads (2 warpgroups)
constexpr int NTHREADS = NPROD;
constexpr int TILE_BYTES = BM * BK * 2;      // 16 KB per operand per stage

using namespace bbtc;

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ------------------------------------------------------------------------------------------------
// Operand staging.  One tile = ROWS rows x 64 k of bf16 in the K-major SWIZZLE_128B layout:
// byte offset(row, k) = row*128 + (((k>>3) ^ (row&7)) << 4) + (k&7)*2.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_chunk(uint8_t* tile, int row, int chunk, const float* v) {
  uint4 q;
  q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]); q.z = pack_bf16(v[4], v[5]); q.w = pack_bf16(v[6], v[7]);
  *reinterpret_cast<uint4*>(tile + row * 128 + ((chunk ^ (row & 7)) << 4)) = q;
}

// The staging code is written so that the compiler emits straight-line batches of independent loads
// (addresses first, then all loads, then convert/pack/store): a per-element "load -> use" chain is
// latency-serialised and was 10-20x slower.  Mode and dtype are template parameters (one warp-uniform
// switch per tile), out-of-range elements load from offset 0 and are masked afterwards.
template <int DT>
struct Raw;
template <>
struct Raw<BB_F32> {
  using T = float;
  static __device__ __forceinline__ float cvt(float v) { return v; }
};
template <>
struct Raw<BB_BF16> {
  using T = unsigned short;
  static __device__ __forceinline__ float cvt(unsigned short v) { return __uint_as_float(((uint32_t)v) << 16); }
};
template <>
struct Raw<BB_F16> {
  using T = unsigned short;
  static __device__ __forceinline__ float cvt(unsigned short v) { return __half2float(__ushort_as_half(v)); }
};

// --- SEG threads per row, each a contiguous run of BK/SEG k's: STRIDED (row-contiguous), PIXROW, WDGRAD.
//     All index arithmetic is 32-bit and incremental (one division per thread per tile); loads go out in
//     batches of 16. ---
template <int MODE, int DT, int ROWS>
__device__ __forceinline__ void stage_by_row_t(uint8_t* tile, const TcSrc& S, int64_t row0, int64_t nrows, int64_t k0,
                                               int64_t kend, int tid, const int2* lut) {
  using R = Raw<DT>;
  constexpr int SEG = NPROD / ROWS;   // 2 (128 rows) or 4 (64 rows)
  constexpr int EPS = BK / SEG;       // elements per thread: 32 or 16
  const int row = tid % ROWS, seg = tid / ROWS;
  const int64_t gr = row0 + row;
  const bool row_ok = gr < nrows;
  const typename R::T* p = reinterpret_cast<const typename R::T*>(S.p);
  const int kb = (int)k0 + seg * EPS;
  int nvalid = (int)(kend - kb);
  nvalid = !row_ok ? 0 : (nvalid > EPS ? EPS : (nvalid < 0 ? 0 : nvalid));
  int y = 0, x = 0, pixoff = 0, cs32 = 0;
  if (MODE == TC_STRIDED) {
    p += (row_ok ? gr : 0) * S.rs + (int64_t)kb * S.cs;
    cs32 = (int)S.cs;
  } else if (MODE == TC_PIXROW) {
    const int64_t g = row_ok ? gr : 0;
    const int hw = S.GH * S.GW;
    const int img = (int)(g / hw), q = (int)(g - (int64_t)img * hw);
    y = q / S.GW;
    x = q - y * S.GW;
    p += (int64_t)img * S.CH * S.H * S.W;
    pixoff = y * S.W + x;
  } else {  // TC_WDGRAD: offset(k) from the table, relative to p + c*KH*KW
    p += (row_ok ? gr : 0) * (S.KH * S.KW);
  }
#pragma unroll
  for (int b = 0; b < EPS / 16; ++b) {
    int off[16];
    uint32_t mask = 0;
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      bool ok = (b * 16 + e) < nvalid;
      int o;
      if (MODE == TC_STRIDED) {
        o = (b * 16 + e) * cs32;
      } else {
        // table entry (same for every thread of the warp: a broadcast shared-memory read)
        const int2 t = lut[ok ? kb + b * 16 + e : 0];
        if (MODE == TC_PIXROW) {
          const int sy = y + (t.y >> 16), sx = x + (int)(short)(t.y & 0xffff);
          ok = ok && (unsigned)sy < (unsigned)S.H && (unsigned)sx < (unsigned)S.W;
          o = pixoff + t.x;
        } else {
          o = t.x;
        }
      }
      off[e] = ok ? o : 0;
      mask |= (ok ? 1u : 0u) << e;
    }
    typename R::T raw[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) raw[e] = p[off[e]];
    float v[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] = ((mask >> e) & 1u) ? R::cvt(raw[e]) : 0.f;
    const int chunk0 = (seg * EPS + b * 16) >> 3;
    store_chunk(tile, row, chunk0, v);
    store_chunk(tile, row, chunk0 + 1, v + 8);
  }
}

// k -> gather-offset table of a PIXROW / WDGRAD operand, built once per CTA.
//   PIXROW: .x = ch*H*W + dy*W + dx, .y = (dy << 16) | (dx & 0xffff)   (dy, dx = window displacement)
//   WDGRAD: .x = ch*C2*KH*KW + i*KW + j
__device__ __forceinline__ void build_lut(int2* lut, const TcSrc& S, int K, int tid) {
  const int KK = S.KH * S.KW;
  for (int k = tid; k < K; k += NTHREADS) {
    const int ch = k / KK, r = k - ch * KK, i = r / S.KW, j = r - i * S.KW;
    int2 t;
    if (S.mode == TC_PIXROW) {
      const int dy = S.flip ? S.py - i : i - S.py, dx = S.flip ? S.px - j : j - S.px;
      t.x = ch * S.H * S.W + dy * S.W + dx;
      t.y = (dy << 16) | (dx & 0xffff);
    } else {
      t.x = ch * S.C2 * KK + r;
      t.y = 0;
    }
    lut[k] = t;
  }
}

// --- 8 threads per row, one 8-element chunk each: STRIDED (k-contiguous) and PIXK; up to 4 rows per batch ---
template <int MODE, int DT, int ROWS>
__device__ __forceinline__ void stage_by_chunk_t(uint8_t* tile, const TcSrc& S, int64_t row0, int64_t nrows, int64_t k0,
                                                 int64_t kend, int tid) {
  using R = Raw<DT>;
  const typename R::T* p = reinterpret_cast<const typename R::T*>(S.p);
  const int chunk = tid & 7;
  const int64_t gk = k0 + chunk * 8;
  constexpr int RPP = NPROD / 8;      // rows per pass (32)
  constexpr int PASSES = ROWS / RPP;  // 4 or 2
  constexpr int BATCH = PASSES < 4 ? PASSES : 4;
  if (MODE == TC_STRIDED) {
    const bool full_k = gk + 8 <= kend;
    const bool vec_ok = full_k && ((S.rs * (int64_t)sizeof(typename R::T)) % 16 == 0) &&
                        ((reinterpret_cast<uintptr_t>(p + gk) & 15) == 0);
#pragma unroll 1
    for (int b0 = 0; b0 < PASSES; b0 += BATCH) {
      if (vec_ok) {
        uint4 raw[BATCH][DT == BB_F32 ? 2 : 1];
        bool okr[BATCH];
#pragma unroll
        for (int b = 0; b < BATCH; ++b) {
          const int row = (tid >> 3) + (b0 + b) * RPP;
          const int64_t gr = row0 + row;
          okr[b] = gr < nrows;
          const uint4* q = reinterpret_cast<const uint4*>(p + (okr[b] ? gr : 0) * S.rs + gk);
          raw[b][0] = q[0];
          if (DT == BB_F32) raw[b][DT == BB_F32 ? 1 : 0] = q[1];
        }
#pragma unroll
        for (int b = 0; b < BATCH; ++b) {
          const int row = (tid >> 3) + (b0 + b) * RPP;
          uint4 out;
          if (DT == BB_F32) {
            const float* f0 = reinterpret_cast<const float*>(&raw[b][0]);
            const float* f1 = reinterpret_cast<const float*>(&raw[b][DT == BB_F32 ? 1 : 0]);
            out.x = pack_bf16(f0[0], f0[1]); out.y = pack_bf16(f0[2], f0[3]);
            out.z = pack_bf16(f1[0], f1[1]); out.w = pack_bf16(f1[2], f1[3]);
          } else if (DT == BB_BF16) {
            out = raw[b][0];   // already bf16: pass the 16-byte chunk through
          } else {
            const unsigned short* h = reinterpret_cast<const unsigned short*>(&raw[b][0]);
            out.x = pack_bf16(R::cvt(h[0]), R::cvt(h[1])); out.y = pack_bf16(R::cvt(h[2]), R::cvt(h[3]));
            out.z = pack_bf16(R::cvt(h[4]), R::cvt(h[5])); out.w = pack_bf16(R::cvt(h[6]), R::cvt(h[7]));
          }
          if (!okr[b]) out = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(tile + row * 128 + ((chunk ^ (row & 7)) << 4)) = out;
        }
      } else {
        typename R::T raw[BATCH][8];
        uint32_t mask = 0;
#pragma unroll
        for (int b = 0; b < BATCH; ++b) {
          const int row = (tid >> 3) + (b0 + b) * RPP;
          const int64_t gr = row0 + row;
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const bool ok = gr < nrows && gk + e < kend;
            mask |= (ok ? 1u : 0u) << (b * 8 + e);
            raw[b][e] = p[ok ? gr * S.rs + gk + e : 0];
          }
        }
#pragma unroll
        for (int b = 0; b < BATCH; ++b) {
          const int row = (tid >> 3) + (b0 + b) * RPP;
          float v[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = ((mask >> (b * 8 + e)) & 1u) ? R::cvt(raw[b][e]) : 0.f;
          store_chunk(tile, row, chunk, v);
        }
      }
    }
  } else {  // TC_PIXK: row = (ch,i,j), k = pixel.  offset = pixbase[e] + rowconst, both 32-bit
    const int KK = S.KH * S.KW;
    const int hw = S.GH * S.GW;
    int pixbase[8], cy[8], cx[8];
    {
      const int64_t g = gk < kend ? gk : 0;
      int ci = (int)(g / hw);
      const int q0 = (int)(g - (int64_t)ci * hw);
      int y = q0 / S.GW, x = q0 - y * S.GW;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const bool kok = gk + e < kend;
        cy[e] = kok ? y : -0x40000000;     // pushes sy out of range -> element masked
        cx[e] = x;
        pixbase[e] = (ci * S.CH * S.H + y) * S.W + x;
        if (++x == S.GW) {
          x = 0;
          if (++y == S.GH) { y = 0; ++ci; }
        }
      }
    }
#pragma unroll 1
    for (int b0 = 0; b0 < PASSES; b0 += BATCH) {
      typename R::T raw[BATCH][8];
      uint32_t mask = 0;
#pragma unroll
      for (int b = 0; b < BATCH; ++b) {
        const int row = (tid >> 3) + (b0 + b) * RPP;
        const int64_t gr = row0 + row;
        const bool rok = gr < nrows;
        const int rr = (int)(rok ? gr : 0);
        const int ch = rr / KK, r = rr - ch * KK, i = r / S.KW, j = r - i * S.KW;
        const int dy = i - S.py, dx = j - S.px;
        const int rowconst = (ch * S.H + dy) * S.W + dx;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const bool ok = rok && (unsigned)(cy[e] + dy) < (unsigned)S.H && (unsigned)(cx[e] + dx) < (unsigned)S.W;
          mask |= (ok ? 1u : 0u) << (b * 8 + e);
          raw[b][e] = p[ok ? pixbase[e] + rowconst : 0];
        }
      }
#pragma unroll
      for (int b = 0; b < BATCH; ++b) {
        const int row = (tid >> 3) + (b0 + b) * RPP;
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = ((mask >> (b * 8 + e)) & 1u) ? R::cvt(raw[b][e]) : 0.f;
        store_chunk(tile, row, chunk, v);
      }
    }
  }
}

// --- MN-major tile from a source whose ROWS are adjacent in memory (rs == 1): element(row,k) = p[row + k*cs].
//     One 8-row chunk (16 B of bf16) per (k, chunk): the global read is contiguous, no transposition is needed,
//     the tensor core reads the tile through an MN-major descriptor.  byte(row,k) = ((row/64)*8 + k/8)*1024 +
//     (k%8)*128 + ((((row%64)/8) ^ (k%8)) << 4) + (row%8)*2
template <int DT, int ROWS>
__device__ __forceinline__ void stage_mn_t(uint8_t* tile, const TcSrc& S, int64_t row0, int64_t nrows, int64_t k0,
                                           int64_t kend, int tid) {
  using R = Raw<DT>;
  const typename R::T* p = reinterpret_cast<const typename R::T*>(S.p);
  constexpr int CPR = ROWS / 8;                 // 8-row chunks per k
  constexpr int TOTAL = CPR * BK;               // chunks per tile
  constexpr int PER = TOTAL / NPROD;            // 4 (128 rows) or 2 (64 rows)
  constexpr int VEC = DT == BB_F32 ? 2 : 1;     // 16-byte loads per chunk
  const bool vec_ok = ((S.cs * (int64_t)sizeof(typename R::T)) % 16 == 0) &&
                      ((reinterpret_cast<uintptr_t>(p + row0) & 15) == 0) && (row0 + ROWS <= nrows);
  auto dst_of = [&](int c, int k) {
    const int blk = c >> 3, cc = c & 7, kb = k >> 3, r = k & 7;
    return reinterpret_cast<uint4*>(tile + (blk * (BK / 8) + kb) * 1024 + r * 128 + ((cc ^ r) << 4));
  };
  if (vec_ok) {
    uint4 raw[PER][VEC];
#pragma unroll
    for (int it = 0; it < PER; ++it) {
      const int q = tid + it * NPROD;
      const int c = q % CPR, k = q / CPR;
      const int64_t gk = (k0 + k < kend) ? k0 + k : k0;
      const uint4* src = reinterpret_cast<const uint4*>(p + row0 + c * 8 + gk * S.cs);
      raw[it][0] = src[0];
      if (VEC == 2) raw[it][VEC - 1] = src[1];
    }
#pragma unroll
    for (int it = 0; it < PER; ++it) {
      const int q = tid + it * NPROD;
      const int c = q % CPR, k = q / CPR;
      uint4 out;
      if (DT == BB_F32) {
        const float* f0 = reinterpret_cast<const float*>(&raw[it][0]);
        const float* f1 = reinterpret_cast<const float*>(&raw[it][VEC - 1]);
        out.x = pack_bf16(f0[0], f0[1]); out.y = pack_bf16(f0[2], f0[3]);
        out.z = pack_bf16(f1[0], f1[1]); out.w = pack_bf16(f1[2], f1[3]);
      } else if (DT == BB_BF16) {
        out = raw[it][0];
      } else {
        const unsigned short* h = reinterpret_cast<const unsigned short*>(&raw[it][0]);
        out.x = pack_bf16(R::cvt(h[0]), R::cvt(h[1])); out.y = pack_bf16(R::cvt(h[2]), R::cvt(h[3]));
        out.z = pack_bf16(R::cvt(h[4]), R::cvt(h[5])); out.w = pack_bf16(R::cvt(h[6]), R::cvt(h[7]));
      }
      if (k0 + k >= kend) out = make_uint4(0, 0, 0, 0);
      *dst_of(c, k) = out;
    }
  } else {
#pragma unroll 1
    for (int it = 0; it < PER; ++it) {
      const int q = tid + it * NPROD;
      const int c = q % CPR, k = q / CPR;
      const int64_t gk = k0 + k, gr = row0 + c * 8;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = (gk < kend && gr + e < nrows) ? R::cvt(p[gr + e + gk * S.cs]) : 0.f;
      uint4 out;
      out.x = pack_bf16(v[0], v[1]); out.y = pack_bf16(v[2], v[3]); out.z = pack_bf16(v[4], v[5]); out.w = pack_bf16(v[6], v[7]);
      *dst_of(c, k) = out;
    }
  }
}

template <int DT, int ROWS>
__device__ __forceinline__ void stage_tile_dt(uint8_t* tile, const TcSrc& S, int64_t row0, int64_t nrows, int64_t k0,
                                              int64_t kend, int tid, const int2* lut) {
  switch (S.mode) {
    case TC_STRIDED:
      if (S.cs == 1) stage_by_chunk_t<TC_STRIDED, DT, ROWS>(tile, S, row0, nrows, k0, kend, tid);
      else if (S.mn_major) stage_mn_t<DT, ROWS>(tile, S, row0, nrows, k0, kend, tid);
      else stage_by_row_t<TC_STRIDED, DT, ROWS>(tile, S, row0, nrows, k0, kend, tid, lut);
      break;
    case TC_PIXROW:
      stage_by_row_t<TC_PIXROW, DT, ROWS>(tile, S, row0, nrows, k0, kend, tid, lut);
      break;
    case TC_PIXK:
      stage_by_chunk_t<TC_PIXK, DT, ROWS>(tile, S, row0, nrows, k0, kend, tid);
      break;
    default:
      stage_by_row_t<TC_WDGRAD, DT, ROWS>(tile, S, row0, nrows, k0, kend, tid, lut);
  }
}

template <int ROWS>
__device__ __forceinline__ void stage_tile(uint8_t* tile, const TcSrc& S, int64_t row0, int64_t nrows, int64_t k0,
                                           int64_t kend, int tid, const int2* lut) {
  if (S.dt == BB_F32) stage_tile_dt<BB_F32, ROWS>(tile, S, row0, nrows, k0, kend, tid, lut);
  else if (S.dt == BB_BF16) stage_tile_dt<BB_BF16, ROWS>(tile, S, row0, nrows, k0, kend, tid, lut);
  else stage_tile_dt<BB_F16, ROWS>(tile, S, row0, nrows, k0, kend, tid, lut);
}

constexpr int kMaxLutK = 2048;   // 2 tables x 8 B x 2048 = 32 KB

template <int BN_>
struct Cfg {
  static constexpr int kBTile = BN_ * BK * 2;
  static constexpr int kStage = TILE_BYTES + kBTile;
  static constexpr size_t kSmem = (size_t)STAGES * kStage + 1024;
};

template <int BN_, int MINB>
__global__ void __launch_bounds__(NTHREADS, MINB) gemm_tc_kernel(const __grid_constant__ TcGemmArgs G) {
  using C = Cfg<BN_>;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B atoms must start on a 1024-byte boundary of the *shared* address space
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  int2* lut_a = reinterpret_cast<int2*>(smem + STAGES * C::kStage);
  int2* lut_b = lut_a + G.lut_k;

  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;
  const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN_;
  const int split = blockIdx.z;
  // k range of this split, in whole k-blocks
  const int64_t kblocks_total = (G.K + BK - 1) / BK;
  const int64_t kb_per = (kblocks_total + G.ksplit - 1) / G.ksplit;
  const int64_t kb_beg = (int64_t)split * kb_per;
  int64_t kb_end = kb_beg + kb_per;
  if (kb_end > kblocks_total) kb_end = kblocks_total;
  const int nkb = (int)(kb_end > kb_beg ? kb_end - kb_beg : 0);
  const int total_kb = nkb * G.npairs;

  if (G.a[0].mode == TC_PIXROW || G.a[0].mode == TC_WDGRAD) build_lut(lut_a, G.a[0], G.lut_k, threadIdx.x);
  if (G.b[0].mode == TC_PIXROW || G.b[0].mode == TC_WDGRAD) build_lut(lut_b, G.b[0], G.lut_k, threadIdx.x);
  __syncthreads();

  float acc[BN_ / 2];
#pragma unroll
  for (int i = 0; i < BN_ / 2; ++i) acc[i] = 0.f;
  // Stage s is rewritten at iteration it + 3.  Every warpgroup passed the barrier of iteration it + 2 only after its
  // wait_group<1> of iteration it + 1, which retires the MMAs of iteration it: the ring needs no other barrier.
  for (int it = 0; it < total_kb; ++it) {
    const int s = it % STAGES;
    const int pair = it / nkb;
    const int64_t k0 = (kb_beg + (it % nkb)) * BK;
    const int64_t kend = (kb_end * BK < G.K) ? kb_end * BK : G.K;
    uint8_t* st = smem + s * C::kStage;
    stage_tile<BM>(st, G.a[pair], m0, G.M, k0, kend, tid, lut_a);
    stage_tile<BN_>(st + TILE_BYTES, G.b[pair], n0, G.N, k0, kend, tid, lut_b);
    fence_proxy_async();
    __syncthreads();
    const bool a_mn = G.a[pair].mn_major != 0, b_mn = G.b[pair].mn_major != 0;
    // this warpgroup's 64 rows: +8 KB in both layouts (64 K-major rows, or the second 64-wide MN block)
    const uint32_t a_addr = smem_u32(st) + (uint32_t)wg * 8192u, b_addr = smem_u32(st) + TILE_BYTES;
    fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      // K-major tiles advance 32 B per 16-wide k-step inside the 128-byte rows; MN-major tiles advance two
      // 1024-byte k-atoms
      const uint64_t da = a_mn ? desc_mn(a_addr + k * 2048, (BK / 8) * 1024) : desc_k(a_addr + k * 32);
      const uint64_t db = b_mn ? desc_mn(b_addr + k * 2048, (BK / 8) * 1024) : desc_k(b_addr + k * 32);
      wgmma_bf16<BN_>(acc, da, db, (it > 0 || k > 0) ? 1u : 0u, a_mn, b_mn);
    }
    wgmma_commit();
    fence_acc(acc);
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  fence_acc(acc);

  // ---------------- epilogue: d[4j + 2h + e] = (row frag_row + 8h, column 8j + frag_col + e) ----------------
  const int64_t col_stride = G.omode == 1 ? (int64_t)G.OHW : G.ocs;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t row = m0 + wg * 64 + frag_row(t) + 8 * h;
    if (row >= G.M) continue;
    int64_t row_base;
    if (G.omode == 1) {
      const int64_t img = row / G.OHW, q = row - img * G.OHW;
      row_base = img * G.OCH * G.OHW + q;
    } else {
      row_base = row * G.ors;
    }
#pragma unroll
    for (int j = 0; j < BN_ / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t col = n0 + 8 * j + frag_col(t) + e;
        if (col < G.N) {
          float v = acc[4 * j + 2 * h + e];
          if (G.bias != nullptr && split == 0) v += G.bias[col * G.bias_stride];
          float* dst = G.out + row_base + col * col_stride;
          if (G.ksplit > 1) atomicAdd(dst, v);
          else *dst = G.beta ? *dst + v : v;
        }
      }
    }
  }
}

template <int BN_, int MINB>
int launch_tc(const TcGemmArgs& G, int ksplit, cudaStream_t s) {
  static BbOncePerDevice configured;
  if (configured.need()) {
    BB_CUDA_TRY(cudaFuncSetAttribute(gemm_tc_kernel<BN_, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(Cfg<BN_>::kSmem + 2 * sizeof(int2) * kMaxLutK)));
  }
  dim3 grid((unsigned)((G.N + BN_ - 1) / BN_), (unsigned)((G.M + BM - 1) / BM), (unsigned)ksplit);
  gemm_tc_kernel<BN_, MINB><<<grid, NTHREADS, Cfg<BN_>::kSmem + 2 * sizeof(int2) * G.lut_k, s>>>(G);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

}  // namespace

bool bb_gemm_tc_eligible(int64_t M, int64_t N, int64_t K, int64_t batch) {
  return batch == 1 && M >= 64 && N >= 64 && K >= 64;
}

int bb_gemm_tc_run(const TcGemmArgs& G0, cudaStream_t s) {
  TcGemmArgs G = G0;
  const int bn = G.N <= 64 ? 64 : 128;
  const int64_t tiles = ((G.M + BM - 1) / BM) * ((G.N + bn - 1) / bn);
  const int64_t kblocks = (G.K + BK - 1) / BK;
  int ksplit = 1;
  if (G.allow_split && tiles < BB_SM_COUNT && kblocks >= 8) {
    int64_t want = (2 * BB_SM_COUNT + tiles - 1) / tiles, maxs = kblocks / 4;
    ksplit = (int)(want < maxs ? want : maxs);
    if (ksplit > 64) ksplit = 64;
    if (ksplit < 1) ksplit = 1;
  }
  if (ksplit > 1 && !G.beta) {
    if (!G.out_dense) {
      ksplit = 1;
    } else {
      BB_CUDA_TRY(cudaMemsetAsync(G.out, 0, sizeof(float) * G.M * G.N, s));
      bb_launch_tally += 1;
    }
  }
  G.ksplit = ksplit;
  // row-contiguous strided operands (transposed views) are staged MN-major: contiguous 16-byte reads, no transpose
  static const bool no_mn = getenv("BB200_TC_NO_MN") != nullptr;
  for (int p = 0; p < G.npairs; ++p) {
    G.a[p].mn_major = (!no_mn && G.a[p].mode == TC_STRIDED && G.a[p].rs == 1 && G.a[p].cs != 1) ? 1 : 0;
    G.b[p].mn_major = (!no_mn && G.b[p].mode == TC_STRIDED && G.b[p].rs == 1 && G.b[p].cs != 1) ? 1 : 0;
  }
  const bool need_lut = G.a[0].mode == TC_PIXROW || G.a[0].mode == TC_WDGRAD || G.b[0].mode == TC_PIXROW ||
                        G.b[0].mode == TC_WDGRAD;
  G.lut_k = need_lut ? (int)G.K : 0;
  if (G.lut_k > kMaxLutK) return BB_ERR_UNSUPPORTED;
  // Two register budgets are compiled: 1 CTA/SM and, for 64-wide tiles, 2 CTAs/SM (capped at 128 registers).  The convolution gathers
  // are issue-latency bound and gain from a second resident CTA; plain strided GEMMs keep the larger budget.
  static const int forced = getenv("BB200_TC_OCC") ? atoi(getenv("BB200_TC_OCC")) : 0;
  const int occ = forced ? forced : (need_lut || G.a[0].mode == TC_PIXK ? 2 : 1);
  // (128 accumulator registers of a 128-wide tile do not fit the 2-CTA budget: those tiles always run one per SM)
  if (occ >= 2 && bn == 64) return launch_tc<64, 2>(G, ksplit, s);
  return bn == 64 ? launch_tc<64, 1>(G, ksplit, s) : launch_tc<128, 1>(G, ksplit, s);
}

extern "C" int bb_gemm_bf16_tc(int64_t M, int64_t N, int64_t K, const void* A, int dtA, int64_t ars, int64_t acs,
                               const void* B, int dtB, int64_t brs, int64_t bcs, float* C, int64_t crs, int64_t ccs,
                               int beta, void* stream) {
  TcGemmArgs G{};
  G.M = M; G.N = N; G.K = K; G.npairs = 1;
  G.a[0] = tc_strided(A, dtA, ars, acs);
  G.b[0] = tc_strided(B, dtB, bcs, brs);   // B tile rows = n: elem(n,k) = B[k*brs + n*bcs]
  G.out = C; G.omode = 0; G.ors = crs; G.ocs = ccs; G.beta = beta; G.bias = nullptr; G.bias_stride = 0;
  G.allow_split = 1;
  G.out_dense = (ccs == 1 && crs == N) || (crs == 1 && ccs == M);
  return bb_gemm_tc_run(G, (cudaStream_t)stream);
}
