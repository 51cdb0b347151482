// Host-side helpers of the TMA-fed tensor-core path (gemm_tma.cu, conv_tma.cu): tensor-map encoding through the
// driver entry point (no link-time dependency on libcuda), a cache of encoded maps, and the per-plan scratch the
// bf16 operand packs are written to.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

// Scratch for packed (bf16, TMA-addressable) copies of operands.  Owned by the caller of the plan (Python allocates
// it once per plan, bb_plan_set_scratch); the executor publishes it here for the node launchers.  Every launcher
// bump-allocates from offset 0: launches on one stream are ordered, so the previous node's packs are dead.
struct BbScratch {
  uint8_t* base;
  size_t bytes;
  size_t used;
};
extern thread_local BbScratch bb_scratch;
extern thread_local uint64_t bb_scratch_gen;   // bumped by every reset: invalidates the launcher's pack cache

inline void bb_scratch_reset() {
  bb_scratch.used = 0;
  ++bb_scratch_gen;
}
inline void* bb_scratch_alloc(size_t bytes) {
  const size_t at = (bb_scratch.used + 255) & ~(size_t)255;
  if (bb_scratch.base == nullptr || at + bytes > bb_scratch.bytes) return nullptr;
  bb_scratch.used = at + bytes;
  return bb_scratch.base + at;
}

// Workspace of the fixed-order reductions (split-K partial products, per-CTA weight-gradient partials): the launcher
// writes partial sums here and a second kernel adds them in a fixed order, so results do not depend on which CTA
// finishes first (fp32 atomics would).  Owned by the plan (plan.cu) and published for the duration of its passes; empty
// outside a plan, where launchers fall back to unsplit reductions.
struct BbReduceWs {
  float* base;
  size_t bytes;
};
extern thread_local BbReduceWs bb_reduce_ws;
inline float* bb_reduce_ws_get(size_t bytes) { return bytes <= bb_reduce_ws.bytes ? bb_reduce_ws.base : nullptr; }
// Largest split count <= want whose partials (`per_split` bytes each) fit the workspace (1: no split).
inline int bb_reduce_ws_splits(int want, size_t per_split) {
  const size_t fit = per_split ? bb_reduce_ws.bytes / per_split : 0;
  return want <= 1 || fit < 2 ? 1 : (int)(fit < (size_t)want ? fit : (size_t)want);
}

// out[i] += sum_{b < parts} part[b*n + i], b in order (the second half of a fixed-order reduction; conv_halo.cu)
int bb_partials_reduce(const float* part, int parts, int64_t n, float* out, cudaStream_t s);
// the same sum with each element's partials split over 32 lanes that are then added in lane order: for hundreds of
// partials of few elements (the small-channel weight gradients, conv_small*.cu)
int bb_partials_reduce_lanes(const float* part, int parts, int64_t n, float* out, cudaStream_t s);
// A partial buffer of `bytes` for launcher-side reductions: the plan's workspace when it is large enough, otherwise a
// stream-ordered allocation released by bb_partials_release (launches outside a plan, e.g. the C-ABI unit hooks).
float* bb_partials_acquire(size_t bytes, cudaStream_t s, bool* owned);
void bb_partials_release(float* p, bool owned, cudaStream_t s);
// Second half of a split-K product (gemm_tma.cu, gemm_tc.cu): out[m*ors + n*ocs] (beta)= bias[n*bias_stride] + the
// ksplit partials part[sp][m][n] (col_major: part[sp][n][m]) added in split order.
int bb_splitk_finish(const float* part, int ksplit, int64_t M, int64_t N, bool col_major, float* out, int64_t ors,
                     int64_t ocs, int beta, const float* bias, int64_t bias_stride, cudaStream_t s);

// Per-node buffer that lives as long as the plan, for packs of operands that are constant across the K-loop (the
// im2col matrix of a data-input convolution).  Returns nullptr when the plan has no persistent arena (or it is full);
// *fresh = true means the caller has to fill it.  Filled eagerly in the base-backward pass (plan creation), so the
// captured K-loop iterations only read it.
void* bb_persist_get(size_t bytes, bool* fresh, int slot = 0);   // slot: 0..BB_PERSIST_SLOTS-1 per node
#define BB_PERSIST_SLOTS 4

// bf16 row-major matrix [rows][cols], `pitch` elements between rows (multiple of 8, base 16-byte aligned):
// box = (64 columns, box_rows rows), SWIZZLE_128B.  Returns 0 or an error code.
int bb_tma_map_2d(CUtensorMap* out, const void* p, int64_t rows, int64_t cols, int64_t pitch, int box_rows);
// batched form: `batch` such matrices `bstride` elements apart (multiple of 8); box = (64, box_rows, 1).  The kernels
// always address matrices through this rank-3 form (bb_tma_map_2d is batch = 1).
int bb_tma_map_3d(CUtensorMap* out, const void* p, int64_t batch, int64_t rows, int64_t cols, int64_t pitch,
                  int64_t bstride, int box_rows);
// bf16 NHWC tensor [N][H][W][Cp] (Cp multiple of 64): box = (64 channels, bw, bh, 1), SWIZZLE_128B.
int bb_tma_map_nhwc(CUtensorMap* out, const void* p, int N, int H, int W, int Cp, int bw, int bh);
// the same view of a PADDED array [N][H+2][W+2][64] (zero border): `p` = the padded base; coordinates address the
// interior, out-of-range taps are zero-filled by TMA as before
int bb_tma_map_nhwc_padded(CUtensorMap* out, const void* p, int N, int H, int W, int bw, int bh);
