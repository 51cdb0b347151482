// Halo-resident implicit-GEMM 3x3 convolution on wgmma (64 -> 64 channels, stride 1, padding 1), forward and
// input-gradient form, up to two operand pairs accumulated into one register tile:
//
//     out[img][n][y][x] (beta)= sum_pairs sum_(tap, ch) A_p[img][y + dy(tap)][x + dx(tap)][ch] * B_p[n][tap][ch]  (+ bias[n])
//
// gemm_tma_kernel's TMA_CONV mode brings one 128-pixel x 64-channel box per TAP into shared memory: nine shifted
// copies of (almost) the same pixels per tile, 24 KB of shared-memory fill per 2.1 MFLOP, which bounds that kernel
// by the fill rate rather than by the tensor cores.  Here the activation lives in a PADDED NHWC layout
// [N][H+2][W+2][64] (zero border), i.e. one long matrix of 128-byte pixel rows in which a tap displacement (dy, dx)
// is the constant row offset dy*(W+2) + dx.  A tile is 128 consecutive pixel rows; ONE TMA box of 128 + 2(W+2) + 2
// rows is loaded per (tile, pair) and the nine taps are nine wgmma descriptors pointing at different 128-byte row
// offsets inside that band (SWIZZLE_128B is a function of the shared-memory address bits alone, so a descriptor may
// start on any 128-byte row of a 1024-byte-aligned band with base offset 0).  The 2 x 9 weight tiles (144 KB) are
// loaded once per CTA and stay resident.  Shared-memory fill per tile: 2 x 28 KB instead of 2 x 9 x 24 KB.  Rows that
// fall on the zero border compute garbage-free zeros' neighbours and are simply not stored.
//
// Roles (288 threads, one CTA per SM, persistent over tiles): warps 0-7 = two consumer warpgroups (register
// accumulators, epilogue -> bf16 padded NHWC or fp32 NCHW planes), warp 8 = TMA producer.  With bf16 output the
// warpgroups take the CTA's tiles in turn, all 128 rows each, so that one issues a tile's wgmma while the other drains
// its tile and runs the epilogue; with fp32 output both work on every tile, 64 rows each.  Up to four band buffers are
// in flight.
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "conv_halo.h"
#include "gemm_tma.h"
#include "plan.h"
#include "tc_ptx.cuh"
#include "tma.h"

namespace {

using namespace bbtc;

constexpr int BM = 128, BN = 64;
constexpr int NTHREADS = 288;                 // 2 consumer warpgroups + the TMA producer warp
constexpr int PRODUCER_WARP = 8;
constexpr int BAND_ROWS = 256;                 // TMA box limit; a band needs 128 + 2*(W+2) + 2 rows
constexpr int BAND_BYTES = BAND_ROWS * 128;    // 32 KB
constexpr int W_TILE = 64 * 128;               // one tap's weights: 64 rows (n) x 64 ch
constexpr int MAXBAND = 4;                     // activation bands in flight: 4 with one operand pair, 2 with two
constexpr uint32_t HALF16 = 64 * 128 / 16;     // rows 64-127 of a tile: 64 band rows further, in 16-byte units
constexpr int STG_BYTES = 64 * 128;            // 64 output rows in bf16: one warpgroup's staging, used per tile half
constexpr int STG_BAR = 1, TURN_BAR = 3;       // named barriers: 1, 2 = staging of warpgroup 0, 1; 3, 4 = issue turn of
                                               // warpgroup 0, 1; 5 = end of the phase-timing run

struct alignas(64) HaloArgs {
  CUtensorMap a[2];          // padded activation as a matrix [rows][64] (rank-3 map, batch 1), box (64, band_rows)
  CUtensorMap b[2];          // weights [64][9*64], box (64, 64)
  int npairs;
  int Wp, HpWp;              // W+2, (H+2)*(W+2)
  int H, W, N;
  int band_rows;
  int band_alloc;            // bytes reserved per band buffer (band_rows * 128 rounded up to 1 KB)
  int nband;                 // band buffers (2 ... MAXBAND)
  int flip;
  int64_t total_rows;        // N * (H+2) * (W+2)
  int ntiles;
  float* out;
  __nv_bfloat16* out_bf16;   // when set: the result goes out as bf16 in the SAME padded NHWC layout (row r of a tile is
                             // row tile*128 + r of the output matrix: one contiguous 16 KB block per tile), border rows 0
  int beta;
  const float* bias;
  unsigned long long* phases;   // PHASES variant only: see bb_conv_halo_phases
  int phase_slots;              // tile slots per CTA in `phases` (tiles per CTA + 1)
};

// Phase timing (conv_halo_kernel<..., PHASES = true>, reached only through bb_conv_halo_phases): thread 0 of the
// consumer warpgroup that owns a tile writes clock64() at the points named by PHASE_NAMES, in program order, into
//   phases[4 * grid + ((cta * phase_slots + slot) * 2 + wg) * NSTAMP + k]
// and thread 0 of the CTA writes {globaltimer, clock64} at the start and the end of its tile loop into phases[4 * cta ...]
// (so the SM clock can be recovered).  Slot = the CTA's local tile index; wg = slot & 1, the other entry stays 0.
constexpr int NSTAMP = 8;
constexpr const char* PHASE_NAMES = "top,turn,p0_band,last_band,issued,drained,epilogue";

__device__ __forceinline__ uint64_t globaltimer() {
  uint64_t v;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(v));
  return v;
}


// Shared memory: [npairs x 9 x 8 KB] weights (resident for the whole kernel) | [NB x band_alloc] activation bands |
// [2 x 8 KB] bf16 output staging, one 64-row block per consumer warpgroup, filled and copied out once per tile half
// (BF16OUT only) | barriers.  The MMA issue loop stays free of waits: both pairs' weights are resident rather than streamed through a
// ring with a wait per tap, and two bands are in flight.
template <int NB, bool BF16OUT, bool PHASES>
__global__ void __launch_bounds__(NTHREADS, 1) conv_halo_kernel(const __grid_constant__ HaloArgs G) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* wsm = smem;                                    // [npairs][9][W_TILE]
  uint8_t* bands = smem + (size_t)G.npairs * 9 * W_TILE;  // [NB][band_alloc]
  uint8_t* stg = bands + (size_t)NB * G.band_alloc;      // [2][64 rows x 128 B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg + (BF16OUT ? 2 * STG_BYTES : 0));
  const uint32_t wfull = smem_u32(bars);
  const uint32_t bfull0 = smem_u32(bars + 1), bempty0 = smem_u32(bars + 1 + MAXBAND);

  const int tid = threadIdx.x, warp = tid >> 5;
  if (tid == 0) {
    mbar_init(wfull, 1);
    for (int b = 0; b < MAXBAND; ++b) {
      mbar_init(bfull0 + 8 * b, 1);
      mbar_init(bempty0 + 8 * b, BF16OUT ? 1 : 2);   // consumer warpgroups that read each band
    }
    fence_barrier_init();
  }
  __syncthreads();
  const uint32_t band_bytes = (uint32_t)G.band_rows * 128u;

  if (warp == PRODUCER_WARP) {
    // ---------------- TMA producer: activation bands (+ the resident weights once) ----------------
    if (elect_one()) {
      for (int p = 0; p < G.npairs; ++p) {
        tma_prefetch_desc(&G.a[p]);
        tma_prefetch_desc(&G.b[p]);
      }
      mbar_expect_tx(wfull, (uint32_t)(G.npairs * 9 * W_TILE));
      for (int p = 0; p < G.npairs; ++p)
        for (int t = 0; t < 9; ++t) tma_load_3d(smem_u32(wsm + (p * 9 + t) * W_TILE), &G.b[p], wfull, t * 64, 0, 0);
      int git = 0;
      for (int tile = blockIdx.x; tile < G.ntiles; tile += gridDim.x) {
        const int row0 = tile * BM - G.Wp - 1;             // first band row (may be negative: zero fill)
        for (int p = 0; p < G.npairs; ++p, ++git) {
          const int b = git % NB;
          if (git >= NB) mbar_wait(bempty0 + 8 * b, ((git / NB) - 1) & 1);
          mbar_expect_tx(bfull0 + 8 * b, band_bytes);
          tma_load_3d(smem_u32(bands + (size_t)b * G.band_alloc), &G.a[p], bfull0 + 8 * b, 0, row0, 0);
        }
      }
    }
    return;
  }
  // ---------------- consumers (warpgroups 0, 1) ----------------
  // Everything the 36 wgmma of a (tile, pair) need is a 32-bit add away: the descriptors' constant upper half, the nine
  // tap offsets (in 16-byte units) and the weight tiles' addresses are set up once.
  const int wg = tid >> 7, t = tid & 127;
  const uint64_t dhi = ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | kDescSw128;
  uint32_t tap16[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) {
    const int i = q / 3, j = q - 3 * i;
    const int dy = G.flip ? 1 - i : i - 1, dx = G.flip ? 1 - j : j - 1;
    tap16[q] = (uint32_t)((G.Wp + 1 + dy * G.Wp + dx) * 8);
  }
  const uint32_t w16 = (smem_u32(wsm) & 0x3FFFF) >> 4, band16_0 = (smem_u32(bands) & 0x3FFFF) >> 4;
  const uint32_t band16_step = (uint32_t)G.band_alloc >> 4;
  const int64_t HW = (int64_t)G.H * G.W;
  // Epilogue without divisions: each thread's output rows are a fixed offset rb into the tile half plus steps of ST rows
  // (bf16 copy-out: rows t/8 + 16 it; fp32 NCHW: rows frag_row + 8 h).  The first row's (image, y, x) is found once
  // per half and the next ones by adding the step's precomputed (dy, dx) with a carry.
  constexpr int ST = BF16OUT ? 16 : 8;
  const int rb = BF16OUT ? (t >> 3) : frag_row(t);
  const int Hp = G.HpWp / G.Wp, sy = ST / G.Wp, sx = ST - sy * G.Wp;
  // this thread's 16 output channels' bias, read once
  const bool has_bias = G.bias != nullptr;
  // (bf16 output, transposed product: channels frag_row and frag_row + 8; fp32 output: channels 8 j + frag_col + e)
  float bz[BN / 4];
  if constexpr (BF16OUT) {
    bz[0] = has_bias ? G.bias[frag_row(t)] : 0.f;
    bz[1] = has_bias ? G.bias[frag_row(t) + 8] : 0.f;
  } else {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) bz[2 * j + e] = has_bias ? G.bias[8 * j + frag_col(t) + e] : 0.f;
  }
  mbar_wait(wfull, 0);
  unsigned long long* ph = nullptr;
  if constexpr (PHASES) {
    ph = G.phases + 4 * gridDim.x + ((size_t)blockIdx.x * G.phase_slots * 2 + wg) * NSTAMP;
    if (tid == 0) { G.phases[4 * blockIdx.x] = globaltimer(); G.phases[4 * blockIdx.x + 1] = clock64(); }
  }
  auto stamp = [&](int slot, int k) {
    if constexpr (PHASES) { if (t == 0) ph[(size_t)slot * 2 * NSTAMP + k] = clock64(); }
  };

  // ---------------- epilogue: d[4j + 2h + e] = (row frag_row + 8h, channel 8j + frag_col + e) ----------------
  auto epilogue = [&](auto& a, int tile, int half) {
    int row = tile * BM + half * 64 + rb;   // padded-linear pixel index of this thread's first row
    int img = (int)((unsigned)row / (unsigned)G.HpWp);
    int yy = row - img * G.HpWp;
    int xx = yy;
    yy = (int)((unsigned)yy / (unsigned)G.Wp);
    xx -= yy * G.Wp;
    auto next_row = [&]() {
      row += ST; xx += sx; yy += sy;
      if (xx >= G.Wp) { xx -= G.Wp; ++yy; }
      if (yy >= Hp) { yy -= Hp; ++img; }
    };
    if constexpr (BF16OUT) {
      // bf16 padded-NHWC output: the half's 64 rows are one contiguous 8 KB block of the output.  The accumulator is
      // the transposed tile (row = channel, column = pixel); stmatrix.trans writes its 8x8 blocks back as pixel rows
      // into shared memory (16-byte chunk c of row r at r*128 + 16 (c ^ (r & 7)), free of bank conflicts), and the
      // block goes out as whole 16-byte chunks, border rows as zeros.
      uint8_t* st = stg + wg * STG_BYTES;
      named_barrier_sync(STG_BAR + wg, 128);    // the previous half's copy-out has read the staging block
      {
        // block q of the x4 = (pixels 8 (j + q/2) .. + 7 of the half, channels 16 warp + 8 (q & 1) .. + 7); lane L
        // addresses the pixel row L % 8 of block L / 8
        const int lane = t & 31, blk = lane >> 3, chunk = 2 * (t >> 5) + (blk & 1);
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          uint32_t v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int jj = 8 * half + j + (q >> 1), h = q & 1;
            float f0 = a[4 * jj + 2 * h], f1 = a[4 * jj + 2 * h + 1];
            if (has_bias) { f0 += bz[h]; f1 += bz[h]; }
            const __nv_bfloat162 b2 = __floats2bfloat162_rn(f0, f1);
            v[q] = *reinterpret_cast<const uint32_t*>(&b2);
          }
          const int r = 8 * (j + (blk >> 1)) + (lane & 7);
          stmatrix_x4_trans(smem_u32(st) + (uint32_t)(r * 128 + 16 * (chunk ^ (r & 7))), v[0], v[1], v[2], v[3]);
        }
      }
      named_barrier_sync(STG_BAR + wg, 128);
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int r = (t >> 3) + 16 * it, c = t & 7;
        if (row >= G.total_rows) break;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if ((unsigned)(yy - 1) < (unsigned)G.H && (unsigned)(xx - 1) < (unsigned)G.W)
          v = *reinterpret_cast<const uint4*>(st + r * 128 + 16 * (c ^ (r & 7)));
        *reinterpret_cast<uint4*>(G.out_bf16 + (int64_t)row * 64 + 8 * c) = v;
        next_row();
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (row < G.total_rows && (unsigned)(yy - 1) < (unsigned)G.H && (unsigned)(xx - 1) < (unsigned)G.W) {
          float* q = G.out + (int64_t)img * BN * HW + (int64_t)(yy - 1) * G.W + (xx - 1);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int n = 8 * j + frag_col(t) + e;
              float v = a[4 * j + 2 * h + e];
              if (has_bias) v += bz[2 * j + e];
              float* d = q + (int64_t)n * HW;
              *d = G.beta ? *d + v : v;
            }
          }
        }
        next_row();
      }
    }
  };

  // bf16 output -- ping-pong over whole tiles: local tile lt of this CTA belongs to warpgroup lt & 1, which accumulates
  // all 128 rows.  Issue is ordered: a warpgroup starts tile lt once the other
  // one has committed the last wgmma of tile lt - 1, so the tensor pipe has one warpgroup's work queued while the other
  // drains and runs its epilogue.  A warpgroup arrives on the other's turn barrier only when a next tile exists, so every
  // arrival meets exactly one wait (0 or 1 tiles: no barrier at all; odd or even counts: each tile lt >= 1 waits once,
  // on the arrival its predecessor made).
  // fp32 NCHW output -- both warpgroups take every tile, rows 64 wg .. 64 wg + 63: that epilogue is a strided
  // read-modify-write bound by memory, which gains more from both warpgroups writing at once than from overlapping it
  // with the MMA (tools/halo_bench.py, DESIGN section 7).
  // The ping-pong warpgroup computes the tile transposed, out^T[channel][pixel] = W . band^T, as one wgmma m64n128k16
  // per k-step with the weights as A and the 128 band rows as B: 6 KB of shared-memory operands per step where two
  // m64n64k16 over the two 64-row halves read 8 KB.  Per element the sum runs over the same products in the same order.
  constexpr bool PP = BF16OUT;
  const uint32_t row16 = PP ? 0u : (uint32_t)wg * HALF16;
  const int my_tiles = (int)blockIdx.x < G.ntiles ? (G.ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  float acc[PP ? BN : BN / 2];
  auto fence_all = [&]() { fence_acc(acc); };
  for (int lt = PP ? wg : 0; lt < my_tiles; lt += PP ? 2 : 1) {
    const int tile = (int)blockIdx.x + lt * (int)gridDim.x;
    stamp(lt, 0);
    if (PP && lt > 0) named_barrier_sync(TURN_BAR + wg, 256);
    stamp(lt, 1);
    int git = lt * G.npairs;
    for (int p = 0; p < G.npairs; ++p, ++git) {
      const int b = git % NB;
      mbar_wait(bfull0 + 8 * b, (git / NB) & 1);
      if (p == 0) stamp(lt, 2);
      if (p == G.npairs - 1) stamp(lt, 3);
      const uint32_t band16 = band16_0 + (uint32_t)b * band16_step + row16;
      const uint32_t wp16 = w16 + (uint32_t)p * (9 * W_TILE >> 4);
      fence_all();
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < 9; ++q) {
        const uint32_t alo = band16 + tap16[q], blo = wp16 + (uint32_t)q * (W_TILE >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t sc = (p > 0 || q > 0 || k > 0) ? 1u : 0u;
          if constexpr (PP)
            wgmma_n128<0, 0>(acc, dhi | (uint64_t)(blo + 2 * k), dhi | (uint64_t)(alo + 2 * k), sc);
          else
            wgmma_n64<0, 0>(acc, dhi | (uint64_t)(alo + 2 * k), dhi | (uint64_t)(blo + 2 * k), sc);
        }
        if (q == 0) {
          // tap 0 is a group of its own: once the group before it (the previous pair) completes, that pair's band is
          // released and the producer reloads it while this pair's remaining eight taps are issued
          wgmma_commit();
          fence_all();
          wgmma_wait<1>();
          if (p > 0 && t == 0) mbar_arrive(bempty0 + 8 * ((git - 1) % NB));
        }
      }
      wgmma_commit();
    }
    stamp(lt, 4);
    if (PP && lt + 1 < my_tiles) named_barrier_arrive(TURN_BAR + (wg ^ 1), 256);
    fence_all();
    wgmma_wait<0>();
    fence_all();
    stamp(lt, 5);
    if (t == 0) mbar_arrive(bempty0 + 8 * ((git - 1) % NB));
    if constexpr (PP) {
      epilogue(acc, tile, 0);
      epilogue(acc, tile, 1);
    } else {
      epilogue(acc, tile, wg);
    }
    stamp(lt, 6);
  }
  if constexpr (PHASES) {
    named_barrier_sync(TURN_BAR + 2, 256);
    if (tid == 0) { G.phases[4 * blockIdx.x + 2] = globaltimer(); G.phases[4 * blockIdx.x + 3] = clock64(); }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Weight gradient with the same halo trick:  D[tap][c][o] += sum_pixels X[pixel + d(tap)][c] * G[pixel][o]
// Both operands are MN-major (rows = pixels = the reduction dimension), X and G in the padded NHWC layout.  Per tile of
// 128 padded-linear pixels: ONE TMA box of G (128 rows) and ONE band of X (128 + 2(W+2) + 2 rows); the nine taps are
// nine row offsets into the X band.  Three consumer warpgroups split the taps (warpgroup g owns taps g, g+3, g+6, one
// wgmma m64n64 per tap and 16-pixel step); wgrad_tma_kernel (conv_tma.cu) loads one X box per tap and tile of <= 64
// pixels.  Accumulators stay in registers over all tiles of the CTA; each CTA writes them to its own slice of `part` and
// bb_partials_reduce adds the slices in CTA order (the result does not depend on which CTA finished first).
// ---------------------------------------------------------------------------------------------------------------
struct alignas(64) WHaloArgs {
  CUtensorMap x[2], g[2];
  int npairs;
  int Wp;
  int band_rows;
  int64_t total_rows;
  int ntiles;
  int stages;
  float* part;                // [gridDim.x][O][C][9] fp32 per-CTA partial sums
  int C, O;
};

constexpr int WH_G_BYTES = 128 * 128;     // 16 KB
constexpr int WH_STAGE = BAND_BYTES + WH_G_BYTES;
constexpr int WH_CONSUMERS = 3;
constexpr int WH_THREADS = WH_CONSUMERS * 128 + 32;
static_assert(64 * 64 * 9 * 4 <= 4 * WH_STAGE, "the weight-gradient partial is staged in the four stage buffers");

__global__ void __launch_bounds__(WH_THREADS, 1) wgrad_halo_kernel(const __grid_constant__ WHaloArgs G) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + G.stages * WH_STAGE);
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + 4);
  const int tid = threadIdx.x, warp = tid >> 5;
  if (tid == 0) {
    for (int s = 0; s < G.stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, WH_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int my_tiles = ((int)blockIdx.x < G.ntiles) ? (G.ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  const int total = my_tiles * G.npairs;
  const uint32_t bytes = (uint32_t)G.band_rows * 128u + (uint32_t)WH_G_BYTES;

  if (warp == WH_CONSUMERS * 4) {
    if (elect_one()) {
      for (int p = 0; p < G.npairs; ++p) {
        tma_prefetch_desc(&G.x[p]);
        tma_prefetch_desc(&G.g[p]);
      }
      for (int it = 0; it < total; ++it) {
        const int s = it % G.stages;
        if (it >= G.stages) mbar_wait(empty0 + 8 * s, ((it / G.stages) - 1) & 1);
        const int pair = it % G.npairs;
        const int tile = (int)blockIdx.x + (it / G.npairs) * (int)gridDim.x;
        const int m0 = tile * BM;
        const uint32_t bar = full0 + 8 * s;
        const uint32_t base = smem_u32(smem + s * WH_STAGE);
        mbar_expect_tx(bar, bytes);
        tma_load_3d(base, &G.x[pair], bar, 0, m0 - G.Wp - 1, 0);
        tma_load_3d(base + BAND_BYTES, &G.g[pair], bar, 0, m0, 0);
      }
    }
    return;
  }
  const int wg = tid >> 7, t = tid & 127;
  // descriptor halves set up once (see conv_halo_kernel): per instruction only the 32-bit start addresses change; one
  // 64-wide MN block per operand, so the leading byte offset is never used
  const uint64_t dhi = ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | kDescSw128;
  uint32_t x16[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int tap = wg + WH_CONSUMERS * q;
    x16[q] = (uint32_t)((G.Wp + 1 + (tap / 3 - 1) * G.Wp + (tap % 3 - 1)) * 8);
  }
  float acc[3][32];
#pragma unroll
  for (int q = 0; q < 3; ++q)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
  for (int it = 0; it < total; ++it) {
    const int s = it % G.stages;
    mbar_wait(full0 + 8 * s, (it / G.stages) & 1);
    const uint32_t band16 = (smem_u32(smem + s * WH_STAGE) & 0x3FFFF) >> 4, g16 = band16 + (BAND_BYTES >> 4);
#pragma unroll
    for (int q = 0; q < 3; ++q) fence_acc(acc[q]);
    wgmma_fence();
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const uint32_t xa = band16 + x16[q];
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
        wgmma_n64<1, 1>(acc[q], dhi | (uint64_t)(xa + ks * 128), dhi | (uint64_t)(g16 + ks * 128), (it > 0 || ks > 0) ? 1u : 0u);
    }
    wgmma_commit();
#pragma unroll
    for (int q = 0; q < 3; ++q) fence_acc(acc[q]);
    wgmma_wait<1>();
    if (it > 0 && t == 0) mbar_arrive(empty0 + 8 * ((it - 1) % G.stages));
  }
  wgmma_wait<0>();
  // The CTA's partial [O][C][9] goes out through shared memory: written straight from the fragments, every 4-byte
  // store would land in its own 32-byte sector (consecutive taps of one (o, c) sit in different warpgroups).  The
  // stage buffers are idle once every consumer has drained its last wgmma.
  named_barrier_sync(1, WH_CONSUMERS * 128);
  float* stage = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    fence_acc(acc[q]);
    const int tap = wg + WH_CONSUMERS * q;
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
          if (o < G.O) stage[(o * G.C + c) * 9 + tap] = acc[q][4 * j + 2 * h + e];
        }
    }
  }
  named_barrier_sync(1, WH_CONSUMERS * 128);
  const int n = G.O * G.C * 9;
  float* dst = G.part + (int64_t)blockIdx.x * n;
  for (int i = tid; i < n; i += WH_CONSUMERS * 128) dst[i] = stage[i];
}

__global__ void __launch_bounds__(256) partials_reduce_kernel(const float* __restrict__ part, int parts, int64_t n,
                                                              float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int b = 0; b < parts; ++b) v += part[(int64_t)b * n + i];
    out[i] += v;
  }
}

// Same sum for hundreds of partials of a few thousand elements.  Block = 32 elements x 32 lanes: lane l adds the
// partials b = l, l + 32, ... in order (four loads in flight), then the lanes are added in lane order.  (One thread per
// element walking all the partials would wait on a memory round trip per partial.)
__global__ void __launch_bounds__(1024) partials_reduce_lanes_kernel(const float* __restrict__ part, int parts, int64_t n,
                                                                     float* __restrict__ out) {
  __shared__ float red[32][33];
  const int c = threadIdx.x & 31, l = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * 32 + c;
  float v = 0.f;
  if (i < n) {
    const float* p = part + i;
    int b = l;
    for (; b + 96 < parts; b += 128) {
      const float v0 = p[(int64_t)b * n], v1 = p[(int64_t)(b + 32) * n], v2 = p[(int64_t)(b + 64) * n],
                  v3 = p[(int64_t)(b + 96) * n];
      v += v0;
      v += v1;
      v += v2;
      v += v3;
    }
    for (; b < parts; b += 32) v += p[(int64_t)b * n];
  }
  red[l][c] = v;
  __syncthreads();
  if (l == 0 && i < n) {
    float sum = red[0][c];
#pragma unroll
    for (int k = 1; k < 32; ++k) sum += red[k][c];
    out[i] += sum;
  }
}

}  // namespace

int bb_partials_reduce(const float* part, int parts, int64_t n, float* out, cudaStream_t s) {
  int64_t blocks = (n + 255) / 256;
  if (blocks > 4 * BB_SM_COUNT) blocks = 4 * BB_SM_COUNT;
  partials_reduce_kernel<<<(unsigned)blocks, 256, 0, s>>>(part, parts, n, out);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

int bb_partials_reduce_lanes(const float* part, int parts, int64_t n, float* out, cudaStream_t s) {
  partials_reduce_lanes_kernel<<<(unsigned)((n + 31) / 32), 1024, 0, s>>>(part, parts, n, out);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

float* bb_partials_acquire(size_t bytes, cudaStream_t s, bool* owned) {
  *owned = false;
  if (float* p = bb_reduce_ws_get(bytes)) return p;
  void* p = nullptr;
  if (cudaMallocAsync(&p, bytes, s) != cudaSuccess) return nullptr;
  *owned = true;
  return reinterpret_cast<float*>(p);
}

void bb_partials_release(float* p, bool owned, cudaStream_t s) {
  if (owned) cudaFreeAsync(p, s);
}

bool bb_conv_halo_ok(int C, int O, int H, int W) {
  static const bool off = getenv("BB200_NO_HALO") != nullptr;
  return !off && C == 64 && O == 64 && W >= 4 && 128 + 2 * (W + 2) + 2 <= BAND_ROWS && H >= 1;
}

namespace {
// Launches conv_halo_kernel; with `phases` set, the phase-timing variant (bf16 output only) writes its stamps there.
// layout (optional) receives {grid, tile slots per CTA, NSTAMP}.
int conv_halo_launch(int N, int H, int W, int npairs, const void* const* act_padded, const void* const* wmat, int flip,
                     float* out, int beta, const float* bias, cudaStream_t s, void* out_bf16_padded,
                     unsigned long long* phases, int* layout) {
  if (npairs < 1 || npairs > 2 || !bb_conv_halo_ok(64, 64, H, W)) return BB_ERR_UNSUPPORTED;
  alignas(64) HaloArgs G;
  memset(&G, 0, sizeof(G));
  G.npairs = npairs;
  G.Wp = W + 2; G.HpWp = (H + 2) * (W + 2);
  G.H = H; G.W = W; G.N = N;
  G.band_rows = BM + 2 * G.Wp + 2;
  G.flip = flip;
  G.total_rows = (int64_t)N * G.HpWp;
  G.ntiles = (int)((G.total_rows + BM - 1) / BM);
  G.out = out; G.beta = beta; G.bias = bias;
  G.out_bf16 = reinterpret_cast<__nv_bfloat16*>(out_bf16_padded);
  if (G.out_bf16 ? beta != 0 : out == nullptr) return BB_ERR_ARG;
  G.band_rows = (G.band_rows + 7) & ~7;
  int rc;
  for (int p = 0; p < npairs; ++p) {
    if ((rc = bb_tma_map_2d(&G.a[p], act_padded[p], G.total_rows, 64, 64, G.band_rows))) return rc;
    if ((rc = bb_tma_map_2d(&G.b[p], wmat[p], 64, 9 * 64, 9 * 64, 64))) return rc;
  }
  G.band_alloc = (G.band_rows * 128 + 1023) & ~1023;
  const bool bf = G.out_bf16 != nullptr;
  const size_t fixed = (size_t)npairs * 9 * W_TILE + (bf ? 2 * STG_BYTES : 0) + 512 + 1024;
  const int fit = (int)((227 * 1024 - fixed) / (size_t)G.band_alloc);
  if (fit < 2) return BB_ERR_UNSUPPORTED;
  const int nb = fit >= 4 ? 4 : 2;
  G.nband = nb;
  const size_t smem = fixed + (size_t)nb * G.band_alloc;
  const int grid = G.ntiles < BB_SM_COUNT ? G.ntiles : BB_SM_COUNT;
  G.phase_slots = (G.ntiles + grid - 1) / grid + 1;
  if (layout) { layout[0] = grid; layout[1] = G.phase_slots; layout[2] = NSTAMP; }
  if (layout && !phases) return BB_OK;
  G.phases = phases;
  if (phases && !bf) return BB_ERR_ARG;
  static BbOncePerDevice configured[6];
  auto launch = [&](auto kern, int slot) -> int {
    if (configured[slot].need())
      BB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    kern<<<grid, NTHREADS, smem, s>>>(G);
    return BB_OK;
  };
  if (phases)
    rc = nb == 4 ? launch(conv_halo_kernel<4, true, true>, 4) : launch(conv_halo_kernel<2, true, true>, 5);
  else if (nb == 4)
    rc = bf ? launch(conv_halo_kernel<4, true, false>, 0) : launch(conv_halo_kernel<4, false, false>, 1);
  else
    rc = bf ? launch(conv_halo_kernel<2, true, false>, 2) : launch(conv_halo_kernel<2, false, false>, 3);
  if (rc) return rc;
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}
}  // namespace

int bb_conv_halo_run(int N, int H, int W, int npairs, const void* const* act_padded, const void* const* wmat, int flip,
                     float* out, int beta, const float* bias, cudaStream_t s, void* out_bf16_padded) {
  return conv_halo_launch(N, H, W, npairs, act_padded, wmat, flip, out, beta, bias, s, out_bf16_padded, nullptr, nullptr);
}

// C-ABI hook for the unit test (tests/test_conv_halo_gpu.py)
extern "C" int bb_conv_halo_bf16(int N, int H, int W, int npairs, const void* act0, const void* act1, const void* w0,
                                 const void* w1, int flip, float* out, int beta, const float* bias, void* stream) {
  const void* acts[2] = {act0, act1};
  const void* ws[2] = {w0, w1};
  return bb_conv_halo_run(N, H, W, npairs, acts, ws, flip, out, beta, bias, (cudaStream_t)stream, nullptr);
}

// same product written as bf16 in the padded NHWC layout (out_padded: [N][H+2][W+2][64], border rows written as zeros)
extern "C" int bb_conv_halo_bf16_nhwc(int N, int H, int W, int npairs, const void* act0, const void* act1, const void* w0,
                                      const void* w1, int flip, void* out_padded, const float* bias, void* stream) {
  const void* acts[2] = {act0, act1};
  const void* ws[2] = {w0, w1};
  return bb_conv_halo_run(N, H, W, npairs, acts, ws, flip, nullptr, 0, bias, (cudaStream_t)stream, out_padded);
}

// Phase timing of the bf16 padded-NHWC product (tools/halo_phases.py).  With stamps == NULL only layout is filled:
// {grid, tile slots per CTA, stamps per slot}; stamps then needs 4 * grid + grid * slots * 2 * NSTAMP entries, zeroed.
extern "C" int bb_conv_halo_phases(int N, int H, int W, int npairs, const void* act0, const void* act1, const void* w0,
                                   const void* w1, int flip, void* out_padded, const float* bias,
                                   unsigned long long* stamps, int* layout, void* stream) {
  if (layout == nullptr) return BB_ERR_ARG;
  const void* acts[2] = {act0, act1};
  const void* ws[2] = {w0, w1};
  return conv_halo_launch(N, H, W, npairs, acts, ws, flip, nullptr, 0, bias, (cudaStream_t)stream, out_padded, stamps,
                          layout);
}

// names of the stamp points of bb_conv_halo_phases, comma-separated, in the order of k
extern "C" int bb_conv_halo_phase_names(char* buf, int cap) {
  const int n = (int)strlen(PHASE_NAMES);
  if (buf == nullptr || cap <= n) return BB_ERR_ARG;
  memcpy(buf, PHASE_NAMES, n + 1);
  return BB_OK;
}

int bb_wgrad_halo_run(int N, int H, int W, int C, int O, int npairs, const void* const* x_padded, const void* const* gy_padded,
                      float* out, cudaStream_t s) {
  if (npairs < 1 || npairs > 2 || C > 64 || O > 64 || !bb_conv_halo_ok(64, 64, H, W)) return BB_ERR_UNSUPPORTED;
  alignas(64) WHaloArgs G;
  memset(&G, 0, sizeof(G));
  G.npairs = npairs;
  G.Wp = W + 2;
  G.band_rows = BM + 2 * G.Wp + 2;
  G.total_rows = (int64_t)N * (H + 2) * (W + 2);
  G.ntiles = (int)((G.total_rows + BM - 1) / BM);
  G.stages = 4;
  G.C = C; G.O = O;
  int rc;
  for (int p = 0; p < npairs; ++p) {
    if ((rc = bb_tma_map_2d(&G.x[p], x_padded[p], G.total_rows, 64, 64, G.band_rows))) return rc;
    if ((rc = bb_tma_map_2d(&G.g[p], gy_padded[p], G.total_rows, 64, 64, BM))) return rc;
  }
  const size_t smem = (size_t)G.stages * WH_STAGE + 256 + 1024;
  static BbOncePerDevice configured;
  if (configured.need())
    BB_CUDA_TRY(cudaFuncSetAttribute(wgrad_halo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = G.ntiles < BB_SM_COUNT ? G.ntiles : BB_SM_COUNT;
  const int64_t n = (int64_t)O * C * 9;
  bool owned = false;
  G.part = bb_partials_acquire(sizeof(float) * grid * n, s, &owned);
  if (G.part == nullptr) return cudaErrorMemoryAllocation;
  wgrad_halo_kernel<<<grid, WH_THREADS, smem, s>>>(G);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  rc = bb_partials_reduce(G.part, grid, n, out, s);
  bb_partials_release(G.part, owned, s);
  return rc;
}

extern "C" int bb_wgrad_halo_bf16(int N, int H, int W, int npairs, const void* x0, const void* x1, const void* g0, const void* g1,
                                  float* out, void* stream) {
  const void* xs[2] = {x0, x1};
  const void* gs[2] = {g0, g1};
  const BbReduceWs saved = bb_reduce_ws;   // not a plan pass: no plan workspace (its stream may be elsewhere)
  bb_reduce_ws = BbReduceWs{nullptr, 0};
  const int rc = bb_wgrad_halo_run(N, H, W, 64, 64, npairs, xs, gs, out, (cudaStream_t)stream);
  bb_reduce_ws = saved;
  return rc;
}
