// K5/K6 tensor-core path, TMA-fed: dual-product GEMM and stride-1 convolution (forward / input-gradient form) on
// wgmma.mma_async with operands brought into shared memory by the TMA unit.
//
//   D[m][n] (beta/atomic)= sum over up to two operand pairs p of  sum_k A_p[m][k] * B_p[n][k]   (+ bias[n])
//
// The software-staged kernel in gemm_tc.cu spends most of its time staging operands (address arithmetic, 4-byte
// gathers, bf16 conversion, swizzled stores).  Here every operand is first made TMA-addressable -- bf16, unit stride
// along one matrix dimension, 16-byte aligned rows; base activations and autocast weight copies already are,
// tangents / adjoints (fp32 arena slices) go through a streaming pack kernel -- and one elected thread issues
// cp.async.bulk.tensor loads that land in the SWIZZLE_128B layout the wgmma descriptors read:
//   K-major operand  (k contiguous in memory): one box of 64 k x ROWS rows      -> rows of 128 B
//   MN-major operand (m/n contiguous):         ROWS/64 boxes of 64 mn x 64 k    -> 8x64 atoms, SBO 1024 B, LBO 8 KB
//   convolution A    (NHWC bf16 activations):  one 4-D box 64 ch x Wb x Hb x 1 per (tap, channel block); the
//                    window displacement is a coordinate offset, zero padding is TMA out-of-bounds fill
// so transposed views cost nothing and an implicit-GEMM convolution is nine shifted box loads per 64 channels.
//
// Roles (288 threads): warps 0-7 = two consumer warpgroups (warpgroup g issues wgmma m64nBNk16 for rows 64g..64g+63
// of the 128-row tile and stores them from its registers), warp 8 = TMA producer (one lane).  3-8 stage mbarrier
// ring; two CTAs per SM on full grids so one CTA's epilogue overlaps the other's main loop.
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <string>
#include <unordered_map>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "gemm_tma.h"
#include "plan.h"
#include "tc_ptx.cuh"
#include "tma.h"

thread_local BbScratch bb_scratch = {nullptr, 0, 0};
thread_local uint64_t bb_scratch_gen = 0;
thread_local BbReduceWs bb_reduce_ws = {nullptr, 0};

namespace {

using namespace bbtc;

constexpr int BM = 128, BK = 64;
constexpr int NTHREADS = 288;
constexpr int PRODUCER_WARP = 8;
constexpr int A_TILE = BM * BK * 2;   // 16 KB

constexpr int MAX_STAGES = 8;

template <int BN_>
struct Cfg {
  static constexpr int kStagesShared = BN_ == 64 ? 4 : 3;   // two CTAs per SM
  static constexpr int kStagesDeep = BN_ == 64 ? 8 : 6;     // one CTA per SM, ~190 KB in flight
  static constexpr int kBTile = BN_ * BK * 2;
  static constexpr int kStage = A_TILE + kBTile;
  static constexpr size_t smem(int stages) { return (size_t)stages * kStage + 1024 + 256; }
};

// Where the rows of an output tile go: row r (0..127) of the tile -> base offset, column stride, validity.
struct OutRows {
  int omode, img, h0;
  int64_t m0, bz;
  __device__ __forceinline__ bool map(const TmaGemmArgs& G, int r, int64_t* base, int64_t* col_stride) const {
    if (omode == 1) {
      const int64_t q = (int64_t)h0 * G.Wb + r;   // Wb == output width
      *base = (int64_t)img * G.OCH * G.OHW + q;
      *col_stride = G.OHW;
      return r < G.Wb * G.Hb && q < G.OHW;
    }
    const int64_t row = m0 + r;
    if (omode == 2) {
      const int64_t im = row / G.OHW;
      *base = im * G.OCH * G.OHW + (row - im * G.OHW);
      *col_stride = G.OHW;
    } else {
      *base = bz * G.obs + row * G.ors;
      *col_stride = G.ocs;
    }
    return row < G.M;
  }
};

// Epilogue of one warpgroup's 64 x BN accumulator fragment (d[4j + 2h + e] = row frag_row + 8h, column
// 8j + frag_col + e).  Mode decisions are made once per row; row-major fp32 outputs are written as float2.
template <int BN_>
__device__ __forceinline__ void epi_store(const TmaGemmArgs& G, const float (&acc)[BN_ / 2], const OutRows& R, int wg, int t,
                                          int n0, bool add_bias) {
  const bool vec = G.omode == 0 && G.ocs == 1 && (G.ors & 1) == 0 && (G.obs & 1) == 0 &&
                   ((reinterpret_cast<uintptr_t>(G.out) & 7) == 0) && G.ksplit == 1;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int64_t base, cs;
    if (!R.map(G, wg * 64 + frag_row(t) + 8 * h, &base, &cs)) continue;
#pragma unroll
    for (int j = 0; j < BN_ / 8; ++j) {
      const int col = n0 + 8 * j + frag_col(t);
      if (col >= G.N) continue;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      const bool two = col + 1 < G.N;
      if (add_bias) {
        v0 += G.bias[(int64_t)col * G.bias_stride];
        if (two) v1 += G.bias[(int64_t)(col + 1) * G.bias_stride];
      }
      float* q = G.out + base + (int64_t)col * cs;
      if (vec && two) {
        float2* q2 = reinterpret_cast<float2*>(q);
        float2 o = make_float2(v0, v1);
        if (G.beta) {
          const float2 old = *q2;
          o.x += old.x; o.y += old.y;
        }
        *q2 = o;
      } else if (G.ksplit > 1) {
        atomicAdd(q, v0);
        if (two) atomicAdd(q + cs, v1);
      } else if (G.beta) {
        *q += v0;
        if (two) q[cs] += v1;
      } else {
        *q = v0;
        if (two) q[cs] = v1;
      }
    }
  }
}

// TMA loads of k-block `it` of a tile into stage buffer sa / sb (one elected producer thread)
template <int BN_>
__device__ __forceinline__ void produce(const TmaGemmArgs& G, int pair, int kb, uint32_t sa, uint32_t sb, uint32_t bar,
                                        int m0, int n0, int img, int h0, int bz) {
  const int k0 = kb * BK;
  mbar_expect_tx(bar, G.a_bytes + G.b_bytes);
  const int ak = G.a_kind[pair];
  if (ak == TMA_KMAJ) {
    tma_load_3d(sa, &G.a[pair], bar, k0, m0, bz);
  } else if (ak == TMA_MNMAJ) {
    tma_load_3d(sa, &G.a[pair], bar, m0, k0, bz);
    tma_load_3d(sa + 8192, &G.a[pair], bar, m0 + 64, k0, bz);
  } else {
    const int tap = kb / G.cblocks, cb = kb - tap * G.cblocks;
    const int i = tap / G.KW, j = tap - i * G.KW;
    const int dy = G.flip ? G.ph - i : i - G.ph, dx = G.flip ? G.pw - j : j - G.pw;
    tma_load_4d(sa, &G.a[pair], bar, cb * 64, dx, h0 + dy, img);
  }
  const int bzb = ak == TMA_CONV ? 0 : bz;
  if (G.b_kind[pair] == TMA_KMAJ) {
    tma_load_3d(sb, &G.b[pair], bar, k0, n0, bzb);
  } else {
#pragma unroll
    for (int q = 0; q < BN_ / 64; ++q) tma_load_3d(sb + q * 8192, &G.b[pair], bar, n0 + q * 64, k0, bzb);
  }
}

// The MMAs of one k-block for this warpgroup's 64 rows; the previous k-block's stage is handed back once its MMAs
// have retired (wait_group 1), so one stage per warpgroup stays in flight.
template <int BN_>
__device__ __forceinline__ void consume(const TmaGemmArgs& G, float (&acc)[BN_ / 2], int pair, uint32_t a_addr, uint32_t b_addr,
                                        bool first) {
  const bool a_mn = G.a_kind[pair] == TMA_MNMAJ, b_mn = G.b_kind[pair] == TMA_MNMAJ;
  fence_acc(acc);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint64_t da = a_mn ? desc_mn(a_addr + k * 2048, 8192) : desc_k(a_addr + k * 32);
    const uint64_t db = b_mn ? desc_mn(b_addr + k * 2048, 8192) : desc_k(b_addr + k * 32);
    wgmma_bf16<BN_>(acc, da, db, (!first || k > 0) ? 1u : 0u, a_mn, b_mn);
  }
  wgmma_commit();
  fence_acc(acc);
  wgmma_wait<1>();
}

template <int BN_>
__global__ void __launch_bounds__(NTHREADS, 2) gemm_tma_kernel(const __grid_constant__ TmaGemmArgs G) {
  using C = Cfg<BN_>;
  const int STAGES = G.stages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * C::kStage);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + MAX_STAGES);

  const int tid = threadIdx.x, warp = tid >> 5;
  const int n0 = blockIdx.x * BN_;
  const int bz = blockIdx.z / G.ksplit;            // batch index (ksplit == 1 when batched)
  const int split = blockIdx.z - bz * G.ksplit;
  const int64_t kblocks_total = (G.K + BK - 1) / BK;
  const int64_t kb_per = (kblocks_total + G.ksplit - 1) / G.ksplit;
  const int64_t kb_beg = (int64_t)split * kb_per;
  int64_t kb_end = kb_beg + kb_per;
  if (kb_end > kblocks_total) kb_end = kblocks_total;
  const int nkb = (int)(kb_end > kb_beg ? kb_end - kb_beg : 0);
  const int total_kb = nkb * G.npairs;

  const bool conv = G.a_kind[0] == TMA_CONV;
  int m0 = 0, img = 0, h0 = 0;
  if (conv) {
    img = blockIdx.y / G.tiles_per_img;
    h0 = (blockIdx.y - img * G.tiles_per_img) * G.Hb;
  } else {
    m0 = blockIdx.y * BM;
  }

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ---------------- TMA producer ----------------
    if (elect_one()) {
      for (int p = 0; p < G.npairs; ++p) {
        tma_prefetch_desc(&G.a[p]);
        tma_prefetch_desc(&G.b[p]);
      }
      for (int it = 0; it < total_kb; ++it) {
        const int s = it % STAGES;
        if (it >= STAGES) mbar_wait(empty0 + 8 * s, ((it / STAGES) - 1) & 1);
        const int pair = it / nkb;
        const uint32_t sa = smem_u32(smem + s * C::kStage);
        produce<BN_>(G, pair, (int)kb_beg + (it - pair * nkb), sa, sa + A_TILE, full0 + 8 * s, m0, n0, img, h0, bz);
      }
    }
  } else {
    // ---------------- consumers (warpgroups 0, 1) ----------------
    const int wg = tid >> 7, t = tid & 127;
    float acc[BN_ / 2];
#pragma unroll
    for (int i = 0; i < BN_ / 2; ++i) acc[i] = 0.f;
    for (int it = 0; it < total_kb; ++it) {
      const int s = it % STAGES;
      mbar_wait(full0 + 8 * s, (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + s * C::kStage);
      consume<BN_>(G, acc, it / nkb, a_addr + (uint32_t)wg * 8192u, a_addr + A_TILE, it == 0);
      if (it > 0 && t == 0) mbar_arrive(empty0 + 8 * ((it - 1) % STAGES));
    }
    wgmma_wait<0>();
    fence_acc(acc);
    const OutRows R{G.omode, img, h0, (int64_t)m0, (int64_t)bz};
    epi_store<BN_>(G, acc, R, wg, t, n0, G.bias != nullptr && split == 0);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Persistent variant for launches with many more tiles than SMs (convolutions: one tile per 128 pixels).  A CTA
// walks tiles blockIdx.x, +gridDim.x, ...; the TMA producer runs ahead across tile boundaries on the same stage ring,
// so the loads of tile i+1 overlap the epilogue of tile i (register accumulators: the consumers store a tile, then
// start the next).  The one-tile-per-CTA kernel above pays barrier init and a cold TMA round trip per tile.
// No split-K, no batch (conv and plane-output GEMMs only).
template <int BN_>
__global__ void __launch_bounds__(NTHREADS, 2) gemm_tma_persist_kernel(const __grid_constant__ TmaGemmArgs G, int ntiles_n,
                                                                       int total_tiles) {
  using C = Cfg<BN_>;
  const int STAGES = G.stages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * C::kStage);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + MAX_STAGES);

  const int tid = threadIdx.x, warp = tid >> 5;
  const int nkb = (int)((G.K + BK - 1) / BK);
  const int per_tile = nkb * G.npairs;
  const bool conv = G.a_kind[0] == TMA_CONV;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // ---------------- TMA producer ----------------
    if (elect_one()) {
      for (int p = 0; p < G.npairs; ++p) {
        tma_prefetch_desc(&G.a[p]);
        tma_prefetch_desc(&G.b[p]);
      }
      int git = 0;   // stage-ring position, continues across tiles
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int mt = tile / ntiles_n, n0 = (tile - mt * ntiles_n) * BN_;
        int m0 = 0, img = 0, h0 = 0;
        if (conv) {
          img = mt / G.tiles_per_img;
          h0 = (mt - img * G.tiles_per_img) * G.Hb;
        } else {
          m0 = mt * BM;
        }
        for (int it = 0; it < per_tile; ++it, ++git) {
          const int s = git % STAGES;
          if (git >= STAGES) mbar_wait(empty0 + 8 * s, ((git / STAGES) - 1) & 1);
          const int pair = it / nkb;
          const uint32_t sa = smem_u32(smem + s * C::kStage);
          produce<BN_>(G, pair, it - pair * nkb, sa, sa + A_TILE, full0 + 8 * s, m0, n0, img, h0, 0);
        }
      }
    }
  } else {
    // ---------------- consumers ----------------
    const int wg = tid >> 7, t = tid & 127;
    float acc[BN_ / 2];
    int git = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int mt = tile / ntiles_n, n0 = (tile - mt * ntiles_n) * BN_;
      for (int it = 0; it < per_tile; ++it, ++git) {
        const int s = git % STAGES;
        mbar_wait(full0 + 8 * s, (git / STAGES) & 1);
        const uint32_t a_addr = smem_u32(smem + s * C::kStage);
        consume<BN_>(G, acc, it / nkb, a_addr + (uint32_t)wg * 8192u, a_addr + A_TILE, it == 0);
        if (it > 0 && t == 0) mbar_arrive(empty0 + 8 * ((git - 1) % STAGES));
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (t == 0) mbar_arrive(empty0 + 8 * ((git - 1) % STAGES));
      OutRows R{G.omode, 0, 0, (int64_t)mt * BM, 0};
      if (conv) {
        R.img = mt / G.tiles_per_img;
        R.h0 = (mt - R.img * G.tiles_per_img) * G.Hb;
      }
      epi_store<BN_>(G, acc, R, wg, t, n0, G.bias != nullptr);
    }
  }
}

template <int BN_>
int launch_tma(TmaGemmArgs& G, int64_t mtiles, cudaStream_t s, int batch) {
  using C = Cfg<BN_>;
  static BbOncePerDevice configured;
  if (configured.need()) {
    BB_CUDA_TRY(cudaFuncSetAttribute(gemm_tma_kernel<BN_>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)C::smem(C::kStagesDeep)));
  }
  dim3 grid((unsigned)((G.N + BN_ - 1) / BN_), (unsigned)mtiles, (unsigned)(G.ksplit * batch));
  // A grid that does not fill the machine is latency-bound on its k-loop (each TMA round trip is ~1.5 us): give the
  // lone CTA of each SM the whole shared memory as prefetch depth.  Full grids keep two CTAs per SM instead, so one
  // CTA's epilogue overlaps the other's main loop.
  static const int forced = getenv("BB200_TMA_STAGES") ? atoi(getenv("BB200_TMA_STAGES")) : 0;
  const int64_t ctas = (int64_t)grid.x * grid.y * grid.z;
  G.stages = ctas <= BB_SM_COUNT ? C::kStagesDeep : C::kStagesShared;
  if (forced >= 2 && forced <= C::kStagesDeep) G.stages = forced;
  static const bool no_persist = getenv("BB200_TMA_NO_PERSIST") != nullptr;
  if (!no_persist && G.ksplit == 1 && batch == 1 && ctas > 4 * BB_SM_COUNT) {
    static BbOncePerDevice configured_p;
    if (configured_p.need()) {
      BB_CUDA_TRY(cudaFuncSetAttribute(gemm_tma_persist_kernel<BN_>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)C::smem(C::kStagesDeep)));
    }
    G.stages = C::kStagesShared;
    gemm_tma_persist_kernel<BN_><<<2 * BB_SM_COUNT, NTHREADS, C::smem(G.stages), s>>>(G, (int)grid.x, (int)(grid.x * grid.y));
    bb_launch_tally += 1;
    BB_LAUNCH_CHECK();
    return BB_OK;
  }
  gemm_tma_kernel<BN_><<<grid, NTHREADS, C::smem(G.stages), s>>>(G);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// ------------------------------------------------------------------------------------------------
// tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess) return nullptr;
    if (q != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<EncodeTiledFn>(f);
  }();
  return fn;
}

std::mutex g_map_mu;
std::unordered_map<std::string, CUtensorMap> g_maps;

int encode_cached(CUtensorMap* out, int rank, const void* p, const cuuint64_t* dims, const cuuint64_t* strides,
                  const cuuint32_t* box) {
  std::string key(reinterpret_cast<const char*>(&p), sizeof(p));
  key.append(reinterpret_cast<const char*>(dims), sizeof(cuuint64_t) * rank);
  key.append(reinterpret_cast<const char*>(strides), sizeof(cuuint64_t) * (rank - 1));
  key.append(reinterpret_cast<const char*>(box), sizeof(cuuint32_t) * rank);
  std::lock_guard<std::mutex> lock(g_map_mu);
  auto it = g_maps.find(key);
  if (it != g_maps.end()) {
    *out = it->second;
    return BB_OK;
  }
  EncodeTiledFn fn = encode_fn();
  if (fn == nullptr) return BB_ERR_UNSUPPORTED;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  alignas(64) CUtensorMap m;
  const CUresult rc = fn(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(p), dims, strides, box,
                         estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) return BB_ERR_ARG;
  if (g_maps.size() > 65536) g_maps.clear();
  g_maps.emplace(std::move(key), m);
  *out = m;
  return BB_OK;
}

// ------------------------------------------------------------------------------------------------
// packs
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// dst[o][i] = bf16(src[o*os + i*is]); one thread = 8 consecutive destination elements (16 bytes).  Up to four
// operands per launch (blockIdx.y = job): a dual product needs at most four packs, and launches -- not bytes -- are
// what a 1 us pack costs.
struct PackJob {
  const void* src;
  uint4* dst;
  int64_t os, is, outer, inner, dp8;
  int64_t batch, sbs;   // batches (>= 1) and source batch stride; destination batches are dense (outer*dp8 chunks)
  int dt, vec;          // vec: fp32, is == 1, rows 16-byte aligned, inner % 8 == 0, dp == inner
};
struct PackJobs {
  PackJob j[4];
  int n;
};

__global__ void __launch_bounds__(256) pack2d_kernel(const __grid_constant__ PackJobs J) {
  const PackJob& q = J.j[blockIdx.y];
  const int64_t per = q.outer * q.dp8, total = per * q.batch;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = t / per, tb = t - b * per;
    const int64_t o = tb / q.dp8, i0 = (tb - o * q.dp8) * 8;
    const int64_t sb = b * q.sbs;
    float v[8];
    if (q.vec) {
      const float* f = reinterpret_cast<const float*>(q.src) + sb + o * q.os + i0;
      const float4 a = bb::ld4_stream(f), b = bb::ld4_stream(f + 4);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = (i0 + e < q.inner) ? bb::ldf(q.src, sb + o * q.os + (i0 + e) * q.is, q.dt) : 0.f;
    }
    uint4 out;
    out.x = pack_bf16(v[0], v[1]); out.y = pack_bf16(v[2], v[3]); out.z = pack_bf16(v[4], v[5]); out.w = pack_bf16(v[6], v[7]);
    q.dst[t] = out;
  }
}

// NCHW -> NHWC bf16: block = 64 channels x 64 pixels of one image through shared memory
__global__ void __launch_bounds__(256) pack_nhwc_kernel(const void* __restrict__ src, int dt, int C, int HW,
                                                        __nv_bfloat16* __restrict__ dst, int Cp) {
  __shared__ float tile[64][65];
  const int img = blockIdx.z, c0 = blockIdx.y * 64, p0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;   // 64 x 4
  const int64_t sbase = (int64_t)img * C * HW;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = c0 + ty + k * 4, p = p0 + tx;
    tile[ty + k * 4][tx] = (c < C && p < HW) ? bb::ldf(src, sbase + (int64_t)c * HW + p, dt) : 0.f;
  }
  __syncthreads();
  // write: 32 threads cover 64 channels (2 each) of one pixel; 8 pixels per pass
  const int cx = (threadIdx.x & 31) * 2, py = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int pl = py + k * 8, p = p0 + pl;
    if (p < HW) {
      const uint32_t w = pack_bf16(tile[cx][pl], tile[cx + 1][pl]);
      *reinterpret_cast<uint32_t*>(dst + ((int64_t)img * HW + p) * Cp + c0 + cx) = w;
    }
  }
}

__global__ void __launch_bounds__(256) pack_convw_kernel(const void* __restrict__ src, int dt, int O, int C, int taps,
                                                         int transpose, __nv_bfloat16* __restrict__ dst, int Qp) {
  const int R = transpose ? C : O, Q = transpose ? O : C;
  const int64_t total = (int64_t)R * taps * Qp;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int q = (int)(t % Qp);
    const int64_t rt = t / Qp;
    const int tap = (int)(rt % taps), r = (int)(rt / taps);
    float v = 0.f;
    if (q < Q) {
      const int o = transpose ? q : r, c = transpose ? r : q;
      v = bb::ldf(src, ((int64_t)o * C + c) * taps + tap, dt);
    }
    dst[t] = __float2bfloat16(v);
  }
}

// im2col: one thread = one pixel x 8 consecutive k
__global__ void __launch_bounds__(256) pack_im2col_kernel(const void* __restrict__ src, int dt, const Im2colGeom g,
                                                          uint4* __restrict__ dst, int kp8) {
  const int64_t P = (int64_t)g.N * g.HO * g.WO, total = P * kp8;
  const int KK = g.KH * g.KW, CKK = g.C * KK;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = t / kp8;
    const int k0 = (int)(t - pix * kp8) * 8;
    const int hw = g.HO * g.WO;
    const int img = (int)(pix / hw), q = (int)(pix - (int64_t)img * hw), y = q / g.WO, x = q - y * g.WO;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = k0 + e;
      float val = 0.f;
      if (k < CKK) {
        const int c = k / KK, r = k - c * KK, i = r / g.KW, j = r - i * g.KW;
        const int h = y * g.sh - g.ph + i * g.dh, w = x * g.sw - g.pw + j * g.dw;
        if ((unsigned)h < (unsigned)g.H && (unsigned)w < (unsigned)g.W)
          val = bb::ldf(src, (((int64_t)img * g.C + c) * g.H + h) * g.W + w, dt);
      }
      v[e] = val;
    }
    uint4 out;
    out.x = pack_bf16(v[0], v[1]); out.y = pack_bf16(v[2], v[3]); out.z = pack_bf16(v[4], v[5]); out.w = pack_bf16(v[6], v[7]);
    dst[t] = out;
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline int64_t round8(int64_t x) { return (x + 7) / 8 * 8; }

// Packs already written to the scratch since the last bb_scratch_reset() (= by earlier launches of the same node):
// the output adjoints of a Linear feed both its input-gradient and its weight-gradient products, and a K-major view
// and its transposed MN-major view are the same bytes.
struct PackKey {
  const void* src;
  int64_t os, is, outer, inner, batch, sbs;
  int dt;
  void* dst;
};
thread_local PackKey t_cache[16];
thread_local int t_ncache = 0;
thread_local uint64_t t_cache_gen = 0;   // bb_scratch_gen the entries belong to

void* cached_pack(const PackKey& want) {
  if (t_cache_gen != bb_scratch_gen) {   // scratch was reset since
    t_ncache = 0;
    t_cache_gen = bb_scratch_gen;
  }
  for (int i = 0; i < t_ncache; ++i) {
    const PackKey& k = t_cache[i];
    if (k.src == want.src && k.dt == want.dt && k.os == want.os && k.is == want.is && k.outer == want.outer &&
        k.inner == want.inner && k.batch == want.batch && k.sbs == want.sbs)
      return k.dst;
  }
  return nullptr;
}

int queue_pack(PackJobs& J, const void* src, int dt, int64_t os, int64_t is, int64_t outer, int64_t inner, int64_t batch,
               int64_t sbs, void** dst, int64_t* dp) {
  *dp = round8(inner);
  PackKey key{src, os, is, outer, inner, batch, batch > 1 ? sbs : 0, dt, nullptr};
  if (void* hit = cached_pack(key)) {
    *dst = hit;
    return BB_OK;
  }
  void* d = bb_scratch_alloc((size_t)batch * outer * *dp * 2);
  if (!d || J.n >= 4) return BB_DECLINED;
  PackJob& q = J.j[J.n++];
  q.src = src; q.dst = reinterpret_cast<uint4*>(d); q.os = os; q.is = is; q.outer = outer; q.inner = inner;
  q.dp8 = *dp / 8; q.dt = dt; q.batch = batch; q.sbs = key.sbs;
  q.vec = (dt == BB_F32 && is == 1 && inner % 8 == 0 && os % 4 == 0 && key.sbs % 4 == 0 && aligned16(src)) ? 1 : 0;
  key.dst = d;
  if (t_ncache < 16) t_cache[t_ncache++] = key;
  *dst = d;
  return BB_OK;
}

int flush_packs(const PackJobs& J, cudaStream_t s) {
  if (J.n == 0) return BB_OK;
  int64_t most = 0;
  for (int i = 0; i < J.n; ++i) {
    const int64_t t = J.j[i].batch * J.j[i].outer * J.j[i].dp8;
    if (t > most) most = t;
  }
  int64_t blocks = (most + 255) / 256;
  if (blocks > 8 * BB_SM_COUNT) blocks = 8 * BB_SM_COUNT;
  if (blocks < 1) blocks = 1;
  pack2d_kernel<<<dim3((unsigned)blocks, (unsigned)J.n), 256, 0, s>>>(J);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// An operand after preparation: a bf16 matrix (per batch) whose rows are the view's rows (TMA_KMAJ, pitch >= K) or the
// view's k (TMA_MNMAJ, pitch >= R), `bstride` elements between batches.
struct Prepared {
  const void* mat;
  int64_t pitch, bstride;
  int kind;
};

inline bool batch_ok(const TmaView& v, int64_t batch) { return batch == 1 || (v.bs % 8 == 0 && v.bs > 0); }
inline bool direct_k(const TmaView& v, int64_t K, int64_t batch) {
  return v.cs == 1 && v.dt == BB_BF16 && v.rs % 8 == 0 && v.rs >= K && aligned16(v.p) && batch_ok(v, batch);
}
inline bool direct_mn(const TmaView& v, int64_t R, int64_t batch) {
  return v.rs == 1 && v.cs != 1 && v.dt == BB_BF16 && v.cs % 8 == 0 && v.cs >= R && aligned16(v.p) && batch_ok(v, batch);
}
size_t pack_bytes(const TmaView& v, int64_t R, int64_t K, int64_t batch) {
  if (v.cs == 1 || v.rs != 1) return direct_k(v, K, batch) ? 0 : (size_t)batch * R * round8(K) * 2;
  return direct_mn(v, R, batch) ? 0 : (size_t)batch * K * round8(R) * 2;
}

// Make one operand view TMA-addressable; packs are queued in J.
int prepare_operand(PackJobs& J, const TmaView& v, int64_t R, int64_t K, int64_t batch, Prepared* out) {
  void* d = nullptr;
  if (v.cs == 1 || v.rs != 1) {
    // K-major (or neither stride unit: gathered into K-major)
    out->kind = TMA_KMAJ;
    if (direct_k(v, K, batch)) {
      out->mat = v.p; out->pitch = v.rs; out->bstride = batch > 1 ? v.bs : R * v.rs;
      return BB_OK;
    }
    const int rc = queue_pack(J, v.p, v.dt, v.rs, v.cs, R, K, batch, v.bs, &d, &out->pitch);
    out->mat = d; out->bstride = R * out->pitch;
    return rc;
  }
  out->kind = TMA_MNMAJ;
  if (direct_mn(v, R, batch)) {
    out->mat = v.p; out->pitch = v.cs; out->bstride = batch > 1 ? v.bs : K * v.cs;
    return BB_OK;
  }
  const int rc = queue_pack(J, v.p, v.dt, v.cs, 1, K, R, batch, v.bs, &d, &out->pitch);
  out->mat = d; out->bstride = K * out->pitch;
  return rc;
}

}  // namespace

int bb_tma_map_3d(CUtensorMap* out, const void* p, int64_t batch, int64_t rows, int64_t cols, int64_t pitch,
                  int64_t bstride, int box_rows) {
  const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
  const cuuint64_t strides[2] = {(cuuint64_t)pitch * 2, (cuuint64_t)bstride * 2};
  const cuuint32_t box[3] = {64u, (cuuint32_t)box_rows, 1u};
  return encode_cached(out, 3, p, dims, strides, box);
}

int bb_tma_map_2d(CUtensorMap* out, const void* p, int64_t rows, int64_t cols, int64_t pitch, int box_rows) {
  return bb_tma_map_3d(out, p, 1, rows, cols, pitch, rows * pitch, box_rows);
}

int bb_tma_map_nhwc(CUtensorMap* out, const void* p, int N, int H, int W, int Cp, int bw, int bh) {
  const cuuint64_t dims[4] = {(cuuint64_t)Cp, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)Cp * 2, (cuuint64_t)W * Cp * 2, (cuuint64_t)H * W * Cp * 2};
  const cuuint32_t box[4] = {64u, (cuuint32_t)bw, (cuuint32_t)bh, 1u};
  return encode_cached(out, 4, p, dims, strides, box);
}

int bb_tma_map_nhwc_padded(CUtensorMap* out, const void* p, int N, int H, int W, int bw, int bh) {
  const cuuint64_t Wp = (cuuint64_t)W + 2, Hp = (cuuint64_t)H + 2;
  const cuuint64_t dims[4] = {64u, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {64u * 2, Wp * 64 * 2, Hp * Wp * 64 * 2};
  const cuuint32_t box[4] = {64u, (cuuint32_t)bw, (cuuint32_t)bh, 1u};
  const char* interior = reinterpret_cast<const char*>(p) + (Wp + 1) * 64 * 2;
  return encode_cached(out, 4, interior, dims, strides, box);
}

int bb_pack2d(const void* src, int dt, int64_t os, int64_t is, int64_t outer, int64_t inner, void* dst, int64_t dp,
              cudaStream_t s) {
  if (outer <= 0 || inner <= 0) return BB_OK;
  PackJobs J{};
  PackJob& q = J.j[0];
  J.n = 1;
  q.src = src; q.dst = reinterpret_cast<uint4*>(dst); q.os = os; q.is = is; q.outer = outer; q.inner = inner;
  q.dp8 = dp / 8; q.dt = dt; q.batch = 1; q.sbs = 0;
  q.vec = (dt == BB_F32 && is == 1 && inner % 8 == 0 && dp == inner && os % 4 == 0 && aligned16(src)) ? 1 : 0;
  return flush_packs(J, s);
}

int bb_pack_nhwc(const void* src, int dt, int N, int C, int HW, void* dst, int Cp, cudaStream_t s) {
  dim3 grid((unsigned)((HW + 63) / 64), (unsigned)(Cp / 64), (unsigned)N);
  pack_nhwc_kernel<<<grid, 256, 0, s>>>(src, dt, C, HW, reinterpret_cast<__nv_bfloat16*>(dst), Cp);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_pack_convw(const void* src, int dt, int O, int C, int taps, int transpose, void* dst, int Qp, cudaStream_t s) {
  const int64_t total = (int64_t)(transpose ? C : O) * taps * Qp;
  int64_t blocks = (total + 255) / 256;
  if (blocks > 4 * BB_SM_COUNT) blocks = 4 * BB_SM_COUNT;
  pack_convw_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dt, O, C, taps, transpose, reinterpret_cast<__nv_bfloat16*>(dst), Qp);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_pack_im2col(const void* src, int dt, const Im2colGeom& g, void* dst, int kp, cudaStream_t s) {
  const int64_t total = (int64_t)g.N * g.HO * g.WO * (kp / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 16 * BB_SM_COUNT) blocks = 16 * BB_SM_COUNT;
  if (blocks < 1) blocks = 1;
  pack_im2col_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dt, g, reinterpret_cast<uint4*>(dst), kp / 8);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_gemm_tma_launch(TmaGemmArgs& G, int bn, int64_t mtiles, cudaStream_t s, int batch) {
  return bn == 64 ? launch_tma<64>(G, mtiles, s, batch) : launch_tma<128>(G, mtiles, s, batch);
}

int bb_gemm_tma_prepack(const TmaPackReq* reqs, int n, int64_t batch, cudaStream_t s) {
  if (encode_fn() == nullptr || bb_scratch.base == nullptr) return BB_OK;
  PackJobs J{};
  for (int i = 0; i < n; ++i) {
    const size_t need = pack_bytes(reqs[i].v, reqs[i].rows, reqs[i].k, batch);
    if (need == 0) continue;
    if (bb_scratch.used + need + 512 > bb_scratch.bytes) break;   // the products will decline or pack on their own
    Prepared pr;
    if (prepare_operand(J, reqs[i].v, reqs[i].rows, reqs[i].k, batch, &pr) != BB_OK) break;
    if (J.n == 4) {
      const int rc = flush_packs(J, s);
      if (rc) return rc;
      J.n = 0;
    }
  }
  return flush_packs(J, s);
}

int bb_gemm_tma_run(int64_t M, int64_t N, int64_t K, int npairs, const TmaView* A, const TmaView* B, float* out,
                    int64_t ors, int64_t ocs, int beta, const float* bias, int64_t bias_stride, bool out_dense,
                    cudaStream_t s, int plane_ohw, int min_n, int64_t batch, int64_t obs) {
  if (npairs < 1 || npairs > 2 || batch < 1) return BB_DECLINED;
  if (batch == 1) {
    if (M < 64 || N < min_n || K < 8) return BB_DECLINED;
    if (K < 64 && min_n >= 64) return BB_DECLINED;
  } else {
    // batched (attention score / context products): the tiles are mostly padding, but a 128 x 64 wgmma tile costs
    // less than the SIMT kernel's inner loop as soon as the products are not tiny
    if (M < 32 || N < 32 || K < 32 || batch > 65535 || plane_ohw > 0 || bias != nullptr) return BB_DECLINED;
  }
  if (M > INT32_MAX / 2 || N > INT32_MAX / 2 || K > INT32_MAX / 2) return BB_DECLINED;
  if (encode_fn() == nullptr || bb_scratch.base == nullptr) return BB_DECLINED;
  // scratch admission: bytes of the operands that need a pack (plan.py sizes the scratch with an upper bound of this)
  {
    size_t need = 1024;
    for (int p = 0; p < npairs; ++p) need += pack_bytes(A[p], M, K, batch) + pack_bytes(B[p], N, K, batch) + 512;
    if (bb_scratch.used + need > bb_scratch.bytes) return BB_DECLINED;
  }
  alignas(64) TmaGemmArgs G;
  memset(&G, 0, sizeof(G));
  // Tile width and split-K by a cost model.  The kernel is bound by what one SM can pull through the TMA unit (a
  // 128 x bn x 64 k-block costs 16 + bn/8 KB), so the time of a configuration is (waves of CTAs) x (k-blocks per CTA)
  // x (bytes per k-block) / per-SM rate; split-K adds a memset launch and the reduction traffic of its partial tiles.
  const int64_t mtiles = (M + BM - 1) / BM;
  const int64_t kblocks = (K + BK - 1) / BK;
  const bool can_split = batch == 1 && plane_ohw == 0 && (beta || out_dense) && kblocks >= 8;
  int bn = 64, ksplit = 1;
  {
    double best = 1e30;
    const int bn_opts[2] = {128, 64};
    for (int bi = 0; bi < 2; ++bi) {
      const int cand = bn_opts[bi];
      if (cand == 128 && N <= 64) continue;
      const int64_t tiles = mtiles * ((N + cand - 1) / cand) * batch;
      for (int sp = 1; sp <= 256; sp = sp < 4 ? sp + 1 : sp * 2) {
        if (sp > 1 && (!can_split || kblocks / sp < 4)) break;
        const int64_t ctas = tiles * sp;
        const int64_t waves = (ctas + BB_SM_COUNT - 1) / BB_SM_COUNT;
        const int64_t iters = (kblocks + sp - 1) / sp * npairs;
        double us = (double)waves * (double)iters * (16.0 + cand / 8.0) * 1024.0 / 84e3 + 2.0;   // 84 GB/s per SM
        if (sp > 1) us += (beta ? 0.0 : 2.5) + (double)M * (double)N * 4.0 * sp / 2.0e6;          // ~2 TB/s of reductions
        if (us < best) {
          best = us;
          bn = cand;
          ksplit = sp;
        }
      }
    }
  }
  PackJobs J{};
  Prepared pa[2], pb[2];
  for (int p = 0; p < npairs; ++p) {
    int rc = prepare_operand(J, A[p], M, K, batch, &pa[p]);
    if (rc) return rc;
    rc = prepare_operand(J, B[p], N, K, batch, &pb[p]);
    if (rc) return rc;
  }
  {
    const int rc = flush_packs(J, s);
    if (rc) return rc;
  }
  for (int p = 0; p < npairs; ++p) {
    G.a_kind[p] = pa[p].kind;
    G.b_kind[p] = pb[p].kind;
    int rc = pa[p].kind == TMA_KMAJ ? bb_tma_map_3d(&G.a[p], pa[p].mat, batch, M, K, pa[p].pitch, pa[p].bstride, BM)
                                    : bb_tma_map_3d(&G.a[p], pa[p].mat, batch, K, M, pa[p].pitch, pa[p].bstride, 64);
    if (rc) return rc;
    rc = pb[p].kind == TMA_KMAJ ? bb_tma_map_3d(&G.b[p], pb[p].mat, batch, N, K, pb[p].pitch, pb[p].bstride, bn)
                                : bb_tma_map_3d(&G.b[p], pb[p].mat, batch, K, N, pb[p].pitch, pb[p].bstride, 64);
    if (rc) return rc;
  }
  G.M = M; G.N = N; G.K = K; G.npairs = npairs;
  G.a_bytes = A_TILE; G.b_bytes = (uint32_t)bn * BK * 2;
  G.out = out; G.omode = 0; G.ors = ors; G.ocs = ocs; G.obs = obs; G.beta = beta; G.bias = bias; G.bias_stride = bias_stride;
  if (plane_ohw > 0) {
    G.omode = 2; G.OCH = (int)N; G.OHW = plane_ohw;
  }
  if (ksplit > 1 && !beta) {
    BB_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * M * N, s));
    bb_launch_tally += 1;
  }
  G.ksplit = ksplit;
  return bb_gemm_tma_launch(G, bn, mtiles, s, (int)batch);
}

extern "C" int bb_gemm_bf16_tma(int64_t M, int64_t N, int64_t K, const void* A, int dtA, int64_t ars, int64_t acs,
                                const void* B, int dtB, int64_t brs, int64_t bcs, float* C, int64_t crs, int64_t ccs,
                                int beta, void* scratch, int64_t scratch_bytes, void* stream) {
  const BbScratch saved = bb_scratch;
  bb_scratch = BbScratch{reinterpret_cast<uint8_t*>(scratch), (size_t)scratch_bytes, 0};
  bb_scratch_reset();
  const TmaView a{A, dtA, ars, acs}, b{B, dtB, bcs, brs};   // rows of the B view = n
  const bool dense = (ccs == 1 && crs == N) || (crs == 1 && ccs == M);
  const int rc = bb_gemm_tma_run(M, N, K, 1, &a, &b, C, crs, ccs, beta, nullptr, 0, dense, (cudaStream_t)stream);
  bb_scratch = saved;
  bb_scratch_reset();
  return rc;
}
