// K5: second-order rules of C = A.B (+ bias) -- Linear layers (addmm with a transposed-view weight),
// attention score/context products (bmm), and any mm/mv in user loss code.  Exact-fp32 SIMT path.
//
//   TF  t_C  = t_A.B + A.t_B (+ t_bias)                       one dual-product launch
//   BB  a_A  = a_C.B^T            a_B  = A^T.a_C
//   TB  at_A = at_C.B^T + a_C.t_B^T      at_B = A^T.at_C + t_A^T.a_C      at_bias = colsum(at_C)
//
// (SURVEY.md Appendix B "Linear": 6 GEMMs per iteration; here 3 dual launches.)  Spec:
// oracle/plan_interp.py tf_gemm/bb_gemm/tb_gemm.
#include <stdlib.h>

#include "../../include/betty_b200.h"
#include "gemm_tc.h"
#include "gemm_tma.h"
#include "tma.h"
#include "plan.h"
#include "tile_gemm.cuh"

namespace {

using bb::StridedLoad;
using bb::StridedStore;

struct Mat {  // a (possibly transposed) strided matrix view
  const void* p;
  int dt;
  int64_t rs, cs, bs;
};

inline Mat T(const Mat& m) { return Mat{m.p, m.dt, m.cs, m.rs, m.bs}; }

// does {m*rs + n*cs (+ b*bs)} cover exactly [0, M*N*batch)?  (needed before the memset + atomic split-K of the tensor-core kernels)
inline bool dense_block(int64_t M, int64_t N, int64_t batch, int64_t rs, int64_t cs, int64_t bs) {
  bool ok;
  if (M == 1) ok = (cs == 1 || N == 1);
  else if (N == 1) ok = (rs == 1);
  else ok = (cs == 1 && rs == N) || (rs == 1 && cs == M);
  return ok && (batch == 1 || bs == M * N);
}

// ---- vectorised fp32 fast path ----------------------------------------------------------------------------
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// 0: not eligible; otherwise bit0 = A k-fast, bit1 = B k-fast, bit2 = eligible
int vec_mode(int64_t M, int64_t N, int64_t K, int64_t batch, int npairs, const Mat* L, const Mat* R) {
  if (batch != 1 || npairs < 1) return 0;
  for (int p = 0; p < npairs; ++p) {
    if (L[p].dt != BB_F32 || R[p].dt != BB_F32 || !aligned16(L[p].p) || !aligned16(R[p].p)) return 0;
    if (L[p].rs != L[0].rs || L[p].cs != L[0].cs || R[p].rs != R[0].rs || R[p].cs != R[0].cs) return 0;
  }
  int mode = 4;
  if (L[0].cs == 1 && K % 4 == 0 && L[0].rs % 4 == 0) mode |= 1;             // A[m][k], k contiguous
  else if (!(L[0].rs == 1 && M % 4 == 0 && L[0].cs % 4 == 0)) return 0;       // A[m][k], m contiguous
  if (R[0].rs == 1 && K % 4 == 0 && R[0].cs % 4 == 0) mode |= 2;             // B[k][n], k contiguous
  else if (!(R[0].cs == 1 && N % 4 == 0 && R[0].rs % 4 == 0)) return 0;       // B[k][n], n contiguous
  return mode;
}

template <int BM, int BN, int TM, int TN>
int launch_vec(int mode, const bb::VecOperands& op, const StridedStore& sc, int64_t M, int64_t N, int64_t K, int npairs,
               int ksplit, dim3 grid, float* part, cudaStream_t s) {
  constexpr int T = (BM / TM) * (BN / TN);
  switch (mode & 3) {
    case 0: bb::tile_gemm_vec_kernel<BM, BN, TM, TN, false, false, StridedStore><<<grid, T, 0, s>>>(op, sc, M, N, K, npairs, ksplit, part); break;
    case 1: bb::tile_gemm_vec_kernel<BM, BN, TM, TN, true, false, StridedStore><<<grid, T, 0, s>>>(op, sc, M, N, K, npairs, ksplit, part); break;
    case 2: bb::tile_gemm_vec_kernel<BM, BN, TM, TN, false, true, StridedStore><<<grid, T, 0, s>>>(op, sc, M, N, K, npairs, ksplit, part); break;
    default: bb::tile_gemm_vec_kernel<BM, BN, TM, TN, true, true, StridedStore><<<grid, T, 0, s>>>(op, sc, M, N, K, npairs, ksplit, part);
  }
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return BB_OK;
}

// out (M x N) (beta)= sum_p L_p (M x K) . R_p (K x N)  [+ bias]
int run_gemm(int64_t M, int64_t N, int64_t K, int64_t batch, int npairs, const Mat* L, const Mat* R, float* out,
             int64_t ors, int64_t ocs, int64_t obs, int beta, const float* bias, int64_t bias_stride,
             cudaStream_t s, bool tensor_cores = false) {
  if (M <= 0 || N <= 0 || batch <= 0) return BB_OK;
  static const bool no_tma = getenv("BB200_NO_TMA") != nullptr;
  if (tensor_cores && npairs > 0 && batch > 1 && !no_tma) {
    // batched products (attention): TMA-fed wgmma kernel, one grid.z slice per batch
    TmaView a[2], b[2];
    for (int p = 0; p < npairs; ++p) {
      a[p] = TmaView{L[p].p, L[p].dt, L[p].rs, L[p].cs, L[p].bs};
      b[p] = TmaView{R[p].p, R[p].dt, R[p].cs, R[p].rs, R[p].bs};
    }
    const int rc = bb_gemm_tma_run(M, N, K, npairs, a, b, out, ors, ocs, beta, bias, bias_stride, false, s, 0, 64, batch, obs);
    if (rc != BB_DECLINED) return rc;
  }
  if (tensor_cores && npairs > 0 && bb_gemm_tc_eligible(M, N, K, batch)) {
    // bf16-autocast configuration: wgmma path (operands rounded to bf16, fp32 accumulation in registers).
    // Preferred: operands packed to TMA-addressable bf16 and fed by the TMA unit (gemm_tma.cu); the software-staged
    // kernel takes what that launcher declines (no scratch, odd shapes).
    if (!no_tma) {
      TmaView a[2], b[2];
      for (int p = 0; p < npairs; ++p) {
        a[p] = TmaView{L[p].p, L[p].dt, L[p].rs, L[p].cs};
        b[p] = TmaView{R[p].p, R[p].dt, R[p].cs, R[p].rs};   // rows of the B view = n
      }
      const int rc = bb_gemm_tma_run(M, N, K, npairs, a, b, out, ors, ocs, beta, bias, bias_stride,
                                     dense_block(M, N, 1, ors, ocs, 0), s);
      if (rc != BB_DECLINED) return rc;
    }
    TcGemmArgs G{};
    G.M = M; G.N = N; G.K = K; G.npairs = npairs;
    for (int p = 0; p < npairs; ++p) {
      G.a[p] = tc_strided(L[p].p, L[p].dt, L[p].rs, L[p].cs);
      G.b[p] = tc_strided(R[p].p, R[p].dt, R[p].cs, R[p].rs);   // rows of the B tile = n
    }
    G.out = out; G.omode = 0; G.ors = ors; G.ocs = ocs; G.beta = beta; G.bias = bias; G.bias_stride = bias_stride;
    G.allow_split = 1;
    return bb_gemm_tc_run(G, s);
  }
  StridedLoad la{}, lb{};
  for (int p = 0; p < npairs; ++p) {
    la.p[p] = L[p].p; la.dt[p] = L[p].dt; la.rs[p] = L[p].rs; la.cs[p] = L[p].cs; la.bs[p] = L[p].bs;
    lb.p[p] = R[p].p; lb.dt[p] = R[p].dt; lb.rs[p] = R[p].rs; lb.cs[p] = R[p].cs; lb.bs[p] = R[p].bs;
  }
  la.k_fast = (npairs > 0 && L[0].cs == 1) ? 1 : 0;
  lb.k_fast = (npairs > 0 && R[0].rs == 1) ? 1 : 0;
  StridedStore sc{out, ors, ocs, obs, beta, bias, bias_stride};

  const bool small_m = M <= 16, small_n = N <= 16 && !small_m;
  // 64x64 tiles unless that leaves most SMs idle: then 32x32 tiles (4x the CTAs)
  const int64_t tiles64 = ((M + 63) / 64) * ((N + 63) / 64) * batch;
  // 64x64 tiles (4x4 per thread) do four times the FMAs per shared-memory load of 32x32 tiles (2x2 per thread) -- only
  // below ~64 big tiles do the small ones pay
  static const int mid_below = getenv("BB200_GEMM_MID") ? atoi(getenv("BB200_GEMM_MID")) : 64;
  const bool mid = !small_m && !small_n && tiles64 < mid_below;
  const int BM = small_m ? 16 : (mid ? 32 : 64), BN = small_n ? 16 : (mid ? 32 : 64);
  const int64_t tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN) * batch;
  int ksplit = 1;
  if (npairs > 0 && tiles < BB_SM_COUNT && K >= 256 && dense_block(M, N, batch, ors, ocs, obs)) {
    int64_t want = (2 * BB_SM_COUNT + tiles - 1) / tiles;
    int64_t maxs = K / 64;
    ksplit = (int)(want < maxs ? want : maxs);
    if (ksplit > 64) ksplit = 64;
    if (ksplit < 1) ksplit = 1;
  }
  // split-K partials go to the plan's reduction workspace and are summed in split order (splitk_reduce_kernel)
  ksplit = bb_reduce_ws_splits(ksplit, sizeof(float) * M * N * batch);
  float* part = ksplit > 1 ? bb_reduce_ws.base : nullptr;
  dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM), (unsigned)(batch * ksplit));
  const int vmode = (small_m || small_n || getenv("BB200_NO_VEC_GEMM")) ? 0 : vec_mode(M, N, K, batch, npairs, L, R);
  if (vmode) {
    bb::VecOperands op{};
    for (int p = 0; p < npairs; ++p) {
      op.a[p] = reinterpret_cast<const float*>(L[p].p);
      op.b[p] = reinterpret_cast<const float*>(R[p].p);
    }
    op.ars = L[0].rs; op.acs = L[0].cs; op.brs = R[0].rs; op.bcs = R[0].cs;
    const int rc = mid ? launch_vec<32, 32, 2, 2>(vmode, op, sc, M, N, K, npairs, ksplit, grid, part, s)
                       : launch_vec<64, 64, 4, 4>(vmode, op, sc, M, N, K, npairs, ksplit, grid, part, s);
    return rc ? rc : bb::splitk_reduce(sc, part, M, N, batch, ksplit, s);
  }
  if (small_m)
    bb::tile_gemm_kernel<16, 64, 16, 1, 4, StridedLoad, StridedLoad, StridedStore><<<grid, 256, 0, s>>>(la, lb, sc, M, N, K, npairs, ksplit, part);
  else if (small_n)
    bb::tile_gemm_kernel<64, 16, 16, 4, 1, StridedLoad, StridedLoad, StridedStore><<<grid, 256, 0, s>>>(la, lb, sc, M, N, K, npairs, ksplit, part);
  else if (mid)
    bb::tile_gemm_kernel<32, 32, 16, 2, 2, StridedLoad, StridedLoad, StridedStore><<<grid, 256, 0, s>>>(la, lb, sc, M, N, K, npairs, ksplit, part);
  else
    bb::tile_gemm_kernel<64, 64, 16, 4, 4, StridedLoad, StridedLoad, StridedStore><<<grid, 256, 0, s>>>(la, lb, sc, M, N, K, npairs, ksplit, part);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  return bb::splitk_reduce(sc, part, M, N, batch, ksplit, s);
}

// out[n] += sum_{b,m} g[b*bs + m*rs + n*cs]   (out must hold the value to accumulate onto).  With more than one block
// row (gridDim.y > 1) every block writes its partial to part[blockIdx.y][n] and colsum_finish_kernel adds them in order.
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ g, float* out, int64_t rows_per_b,
                                                     int64_t batch, int64_t N, int64_t rs, int64_t cs, int64_t bs,
                                                     int64_t out_stride, float* __restrict__ part) {
  __shared__ float sm[8][33];
  const int64_t n = (int64_t)blockIdx.x * 32 + threadIdx.x;
  const int64_t total = rows_per_b * batch;
  float acc = 0.f;
  if (n < N) {
    for (int64_t r = (int64_t)blockIdx.y * 8 + threadIdx.y; r < total; r += (int64_t)gridDim.y * 8) {
      const int64_t b = r / rows_per_b, m = r - b * rows_per_b;
      acc += g[b * bs + m * rs + n * cs];
    }
  }
  sm[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
    if (part != nullptr) part[(int64_t)blockIdx.y * N + n] = t;
    else out[n * out_stride] += t;
  }
}

__global__ void __launch_bounds__(256) colsum_finish_kernel(const float* __restrict__ part, int parts, float* out, int64_t N,
                                                            int64_t out_stride) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float t = 0.f;
  for (int i = 0; i < parts; ++i) t += part[(int64_t)i * N + n];
  out[n * out_stride] += t;
}

int run_colsum(const float* g, float* out, int64_t M, int64_t batch, int64_t N, int64_t rs, int64_t cs, int64_t bs,
               int64_t out_stride, int beta, cudaStream_t s) {
  if (!beta) {
    if (out_stride != 1) return BB_ERR_UNSUPPORTED;
    BB_CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * N, s));
    bb_launch_tally += 1;
  }
  const int64_t rows = M * batch;
  int gy = (int)((rows + 63) / 64);
  if (gy < 1) gy = 1;
  if (gy > 64) gy = 64;
  gy = bb_reduce_ws_splits(gy, sizeof(float) * N);
  float* part = gy > 1 ? bb_reduce_ws.base : nullptr;
  dim3 grid((unsigned)((N + 31) / 32), (unsigned)gy);
  colsum_kernel<<<grid, dim3(32, 8), 0, s>>>(g, out, M, batch, N, rs, cs, bs, out_stride, part);
  bb_launch_tally += 1;
  BB_LAUNCH_CHECK();
  if (part != nullptr) {
    colsum_finish_kernel<<<(unsigned)((N + 255) / 256), 256, 0, s>>>(part, gy, out, N, out_stride);
    bb_launch_tally += 1;
    BB_LAUNCH_CHECK();
  }
  return BB_OK;
}

}  // namespace

int bb_launch_gemm(const bb_node& nd, int pass, cudaStream_t s) {
  const int64_t M = nd.dims[0], N = nd.dims[1], K = nd.dims[2], batch = nd.dims[3];
  const bool actA = nd.active & 1, actB = nd.active & 2, actBias = nd.active & 4;
  const int64_t* sa = nd.stride[0];  // A: m, k, b
  const int64_t* sb = nd.stride[1];  // B: k, n, b
  const int64_t* sc = nd.stride[3];  // C: m, n, b
  const Mat A{nd.base[0], nd.dt[0], sa[0], sa[1], sa[2]};
  const Mat B{nd.base[1], nd.dt[1], sb[0], sb[1], sb[2]};
  const Mat tA{nd.t[0], BB_F32, sa[0], sa[1], sa[2]};
  const Mat tB{nd.t[1], BB_F32, sb[0], sb[1], sb[2]};
  int rc;
  const bool tc = (nd.kind & 1) && !getenv("BB200_NO_TC");   // set by plan.py for bf16-autocast graphs
  bb_scratch_reset();   // operand packs of the TMA-fed path live for one node
  if (pass == BB_PASS_TAN_FWD) {
    Mat L[2], R[2];
    int np = 0;
    if (actA) { L[np] = tA; R[np] = B; ++np; }
    if (actB) { L[np] = A; R[np] = tB; ++np; }
    return run_gemm(M, N, K, batch, np, L, R, reinterpret_cast<float*>(nd.t[3]), sc[0], sc[1], sc[2], 0,
                    actBias ? reinterpret_cast<const float*>(nd.t[2]) : nullptr, nd.stride[2][0], s, tc);
  }
  const bool base = pass == BB_PASS_BASE_BWD;
  const Mat gC{base ? nd.a[3] : nd.at[3], BB_F32, sc[0], sc[1], sc[2]};   // adjoint being propagated
  const Mat aC{nd.a[3], BB_F32, sc[0], sc[1], sc[2]};                      // base adjoint (curvature terms)
  const int need = base ? nd.pad0 : nd.active;                              // pad0 = need_a mask
  Mat Ld[2] = {gC, aC}, Rd[2] = {T(B), T(tB)};        // (M x K) = gC (M x N) . B^T (N x K)  [+ aC . tB^T]
  Mat Lw[2] = {T(A), T(tA)}, Rw[2] = {gC, aC};        // (K x N) = A^T (K x M) . gC (M x N)  [+ tA^T . aC]
  const int npd = (!base && actB) ? 2 : 1, npw = (!base && actA) ? 2 : 1;
  if (tc && !base && batch == 1 && M >= 64 && N >= 64 && K >= 64 && (need & 3) == 3 && !getenv("BB200_NO_TMA")) {
    // tensor-core route: pack the operands of BOTH products in one launch (the adjoints are shared between them)
    TmaPackReq rq[8];
    int nr = 0;
    for (int p = 0; p < npd; ++p) {
      rq[nr++] = TmaPackReq{TmaView{Ld[p].p, Ld[p].dt, Ld[p].rs, Ld[p].cs}, M, N};
      rq[nr++] = TmaPackReq{TmaView{Rd[p].p, Rd[p].dt, Rd[p].cs, Rd[p].rs}, K, N};
    }
    for (int p = 0; p < npw; ++p) {
      rq[nr++] = TmaPackReq{TmaView{Lw[p].p, Lw[p].dt, Lw[p].rs, Lw[p].cs}, K, M};
      rq[nr++] = TmaPackReq{TmaView{Rw[p].p, Rw[p].dt, Rw[p].cs, Rw[p].rs}, N, M};
    }
    rc = bb_gemm_tma_prepack(rq, nr, 1, s);
    if (rc) return rc;
  }
  if (need & 1) {
    rc = run_gemm(M, K, N, batch, npd, Ld, Rd, reinterpret_cast<float*>(base ? nd.a[0] : nd.at[0]), sa[0], sa[1], sa[2],
                  nd.beta[0], nullptr, 0, s, tc);
    if (rc) return rc;
  }
  if (need & 2) {
    rc = run_gemm(K, N, M, batch, npw, Lw, Rw, reinterpret_cast<float*>(base ? nd.a[1] : nd.at[1]), sb[0], sb[1], sb[2],
                  nd.beta[1], nullptr, 0, s, tc);
    if (rc) return rc;
  }
  if (need & 4) {
    rc = run_colsum(reinterpret_cast<const float*>(gC.p), reinterpret_cast<float*>(base ? nd.a[2] : nd.at[2]), M, batch,
                    N, sc[0], sc[1], sc[2], nd.stride[2][0], nd.beta[2], s);
    if (rc) return rc;
  }
  return BB_OK;
}
