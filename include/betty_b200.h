/* betty_b200 -- C ABI of the H100-native hypergradient engine.
 *
 * The reference (leopard-ai/betty) has NO native layer and no FFI: its extension point for this path
 * is the Python plugin table `jvp_fn_mapping[Config.type](vector, curr, prev, sync)`
 * (reference betty/hypergradient/__init__.py:13-19,33-37).  This header is therefore the engine's own
 * boundary: plain pointers, sizes and a `cudaStream_t` passed as `void*`; no torch types.  The Python
 * plugins in betty_b200/hypergradient bind it through ctypes (see INTEGRATION.md for the stub a
 * reference maintainer would add).  Every entry point returns 0 on success, a negative BB_ERR_* code
 * for argument errors, or a positive cudaError_t.  Nothing here allocates inside the K-loop.
 *
 * Each group cites the reference computation it replaces.
 */
#ifndef BETTY_B200_H
#define BETTY_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- workspace shared by the K-loop kernels (device memory, zero-initialised by the caller) ---- */
typedef struct {
  double rr;       /* r.r                        reference cg.py:45   */
  double php;      /* (cg_alpha*Hp).p            reference cg.py:46   */
  double rr_new;   /* r'.r'                      reference cg.py:52   */
  double alpha;    /* rr / php                   reference cg.py:47   */
  double beta;     /* rr_new / rr                reference cg.py:52   */
  double sumsq;    /* ||v||^2                    reference darts.py:30 */
  double eps;      /* darts_alpha/(||v||+1e-15)  reference darts.py:35 */
  double inv_2eps; /* 1/(2 eps)                  reference darts.py:45,53,67 */
} bb_kloop_scalars;

int bb_kloop_ws_bytes(void); /* scalars at offset 0, tickets at 256, reduction slots from 512 */

/* ---- K1: Neumann accumulate.  Replaces reference neumann.py:63-64 (two list comprehensions, three
 *      elementwise launches + two allocations per parameter tensor).  n % 4 == 0.
 *      v <- v - alpha*(hv + shift*v);  p <- p + v                                              */
int bb_neumann_update(float* v, float* p, const float* hv, float alpha, float shift, int64_t n, void* stream);
/* out <- c * in   (final alpha*p, reference neumann.py:66; cg_alpha*x, reference cg.py:56) */
int bb_scale(float* out, const float* in, float c, int64_t n, void* stream);

/* ---- K2/K3: conjugate-gradient inner products and updates.  Replaces reference cg.py:42-53
 *      (three to_vec concatenations, three dots, three list-comprehension AXPYs per iteration).
 *      alpha and beta stay in `ws`; `first` != 0 also computes rr = r.r.                        */
/* `shift`: H p = hp + shift * p -- a declared c*I curvature term (folded L2 / proximal regulariser) applied inside
 * the vector passes instead of a separate sweep over the arenas (same argument as bb_neumann_update's) */
int bb_cg_dots(const float* r, const float* hp, const float* p, float cg_alpha, float shift, int first, int64_t n,
               void* ws, void* stream);
int bb_cg_init(const float* r, int64_t n, void* ws, void* stream); /* ws.rr = r.r */
int bb_cg_update_xr(float* x, float* r, const float* p, const float* hp, float shift, int64_t n, void* ws,
                    void* stream);
int bb_cg_update_p(float* p, const float* r, int64_t n, const void* ws, void* stream);

/* ---- K4 + packing: multi-tensor kernels over a chunk table.  Replaces reference darts.py:30-38,
 *      49-50,61-67 (per-tensor add_/sub_ loops, to_vec().norm().item(), (x-y).div_(2 eps)).      */
#define BB_MT_CHUNK 16384
typedef struct {
  void* a;
  void* b;
  int32_t n; /* <= BB_MT_CHUNK floats */
  int32_t pad;
} bb_mt_chunk;
int bb_mt_copy(const bb_mt_chunk* table_dev, int nchunks, int dir /*0: a->b, 1: b->a*/, void* stream);
/* b <- coef_a * (*scale_dev) * a + coef_b * b   (scale_dev may be NULL => 1) */
int bb_mt_axpby(const bb_mt_chunk* table_dev, int nchunks, float coef_a, const double* scale_dev, float coef_b,
                void* stream);
int bb_mt_sumsq(const bb_mt_chunk* table_dev, int nchunks, void* ws, void* stream); /* -> ws.sumsq */
int bb_fd_eps(void* ws, double darts_alpha, void* stream);                          /* -> ws.eps, inv_2eps */
/* a <- (a - b) * ws.inv_2eps */
int bb_mt_fd_combine(const bb_mt_chunk* table_dev, int nchunks, const void* ws, void* stream);
/* K4 epilogue for `sama` (reference betty/hypergradient/sama.py:24, utils.py:37-63): the Adam preconditioner of the
 * direction, out = v * lr * ((1-b1) b2 s_old - b1 (1-b2) g m_old) / (sqrt(s) + eps)^3 per element, multi-tensor */
typedef struct bb_mt_adam_chunk {
  const void* v;   /* direction                       */
  const void* g;   /* optimizer state "last_grad"  (0 => zeros) */
  const void* m;   /* optimizer state "exp_avg"    (0 => zeros) */
  const void* s;   /* optimizer state "exp_avg_sq" (0 => zeros) */
  void* out;
  int32_t n;
  float beta1, beta2, eps, lr;
  int32_t pad;
} bb_mt_adam_chunk;
int bb_mt_adam_precondition(const bb_mt_adam_chunk* table_dev, int nchunks, void* stream);

/* ---- prologue (SURVEY.md 8 f2): training-mode BatchNorm forward of the lower problem's own forward pass.
 *      Replaces the aten.native_batch_norm(training=True) call PyTorch makes inside curr.training_step_exec
 *      (reference neumann.py:31 / cg.py:27 run that forward once per call) for large channels-first CUDA
 *      activations -- opt-in, BB200_PROLOGUE_BN_MIN (betty_b200/trace.py): x, y [N][C][HW] (dtype BB_F32 | BB_BF16), weight / bias fp32 [C] or NULL,
 *      mean / invstd / var_unbiased fp32 [C] (var_unbiased may be NULL), ws >= 2 * C * bb_bn_forward_splits(N, C)
 *      doubles.  out = weight * (x - mean) * invstd + bias, invstd = rsqrt(biased variance + eps); the statistics
 *      are reduced in fp64 in a fixed order.  csrc/bn_fwd.cu                                                  */
int bb_bn_forward_splits(int64_t N, int C);
int bb_bn_forward(const void* x, int dtype, const float* weight, const float* bias, double eps, void* y, float* mean,
                  float* invstd, float* var_unbiased, double* ws, int64_t N, int C, int64_t HW, void* stream);

/* ---- K5-K9: second-order tape ("HVP plan").  Replaces reference neumann.py:62 / cg.py:39-41
 *      (torch.autograd.grad(in_grad, params, grad_outputs=v, retain_graph=True): reverse-over-reverse
 *      through the retained autograd graph) with forward-over-reverse over a recorded op list.
 *      See betty_b200/csrc/plan.h for the node descriptor.                                        */
struct bb_node;
typedef struct bb_plan bb_plan;
#define BB_PASS_BASE_BWD 0 /* delta from the loss seed, once per call                */
#define BB_PASS_TAN_FWD 1  /* tangents along the direction arena                     */
#define BB_PASS_TAN_BWD 2  /* adjoint-tangents -> Hv slices of the hv arena          */
int bb_node_bytes(void);
int bb_plan_create(const struct bb_node* nodes, int n_nodes, bb_plan** out);
int bb_plan_destroy(bb_plan* plan);
int bb_plan_set_zero_regions(bb_plan* plan, int pass, void* const* ptrs, const int64_t* bytes, int n);
/* device scratch for the bf16 operand packs of the TMA-fed tensor-core kernels (caller-owned, >= the largest
 * node's need; without it those nodes use the software-staged kernel) */
int bb_plan_set_scratch(bb_plan* plan, void* ptr, int64_t bytes);
/* device buffer that lives as long as the plan, for packs of K-loop constants (im2col matrix of a data-input
 * convolution): filled once during BB_PASS_BASE_BWD, read by every iteration; optional */
int bb_plan_set_persistent(bb_plan* plan, void* ptr, int64_t bytes);
int bb_plan_run(bb_plan* plan, int pass, void* stream);
int bb_plan_launch_count(const bb_plan* plan, int pass);
/* eager run of one pass with a CUDA event pair around every node: ms_per_node[n_nodes] */
int bb_plan_profile(bb_plan* plan, int pass, float* ms_per_node, void* stream);
/* one H.d product: zero regions, tangent forward, tangent backward */
int bb_plan_hvp(bb_plan* plan, void* stream);
/* node `node` is a BB_OP_DIAGSHIFT that adds coef * d to EVERY parameter slice of H.d: the K-loops skip it and hand
 * `coef` to K1 / K2 / K3 as their `shift` (one pass over the arenas less per iteration); bb_plan_hvp still runs it */
int bb_plan_set_uniform_shift(bb_plan* plan, int node, double coef);
/* the same product as ONE graph launch (captured at the first call, kept for the plan's lifetime) */
int bb_plan_hvp_replay(bb_plan* plan, void* stream);
/* a cached plan is about to serve new base values written in place behind the same pointers: rebuild the packs of
 * K-loop constants at the next BB_PASS_BASE_BWD (captured graphs stay valid, addresses do not change) */
int bb_plan_invalidate_constants(bb_plan* plan);
int bb_plan_graph_captures(const bb_plan* plan); /* how many times a K-loop iteration was captured (tests) */
int bb_plan_node_route(bb_plan* plan, int node, int pass); /* tests: 2 = TMA tensor-core convolution path */
/* bytes of the per-node workspace of a fused data-input convolution block (BB_OP_CONVBLOCK, csrc/convblock.cu) */
/* ---- K6 building block exposed for unit tests: halo-resident 3x3 convolution (csrc/conv_halo.cu), 64 -> 64 channels,
 *      activations bf16 in the padded NHWC layout [N][H+2][W+2][64] (zero border), weights bf16 [64][9][64] (n, tap, ch);
 *      out fp32 NCHW; flip = 1: tap (i, j) reads the pixel at (+1-i, +1-j) (input-gradient form) */
int bb_conv_halo_bf16(int N, int H, int W, int npairs, const void* act0, const void* act1, const void* w0, const void* w1,
                      int flip, float* out, int beta, const float* bias, void* stream);
int bb_conv_halo_bf16_nhwc(int N, int H, int W, int npairs, const void* act0, const void* act1, const void* w0,
                           const void* w1, int flip, void* out_padded /* bf16 [N][H+2][W+2][64] */, const float* bias,
                           void* stream);
/* phase timing of the bf16 padded-NHWC product (tools/halo_phases.py): a separate instantiation writes clock64 stamps
 * at the points bb_conv_halo_phase_names lists; with stamps == NULL only layout = {grid, tile slots per CTA, stamps per
 * slot} is filled, and stamps then needs 4*grid + grid*slots*2*stamps_per_slot zeroed entries */
int bb_conv_halo_phases(int N, int H, int W, int npairs, const void* act0, const void* act1, const void* w0, const void* w1,
                        int flip, void* out_padded, const float* bias, unsigned long long* stamps, int* layout, void* stream);
int bb_conv_halo_phase_names(char* buf, int cap);
/* weight-gradient companion (wgrad_halo_kernel): out[o][c][tap] (fp32 [64][64][9], accumulated) +=
 * sum_pixels gy[pixel][o] * x[pixel + d(tap)][c], x / gy bf16 padded NHWC */
int bb_wgrad_halo_bf16(int N, int H, int W, int npairs, const void* x0, const void* x1, const void* g0, const void* g1,
                       float* out, void* stream);
int64_t bb_convblock_ws_bytes(int N, int C, int H, int W, int O, int HO, int WO, int HP, int WP);
/* same for a fused inner block of a bf16 graph (BB_OP_CONVBLOCK2, csrc/convblock2.cu) */
int64_t bb_convblock2_ws_bytes(int N, int C, int H, int W, int O, int HO, int WO, int HP, int WP);
/* whole K-loops: one iteration is captured into a CUDA graph at the first call and relaunched by every later
 * call with the same arenas / alpha (direction arena `d`, result `hv`) */
int bb_plan_neumann_loop(bb_plan* plan, int iterations, float alpha, float* v /*direction*/, float* p,
                         const float* hv, int64_t n, int use_graph, void* stream);
int bb_plan_cg_loop(bb_plan* plan, int iterations, float cg_alpha, float* x, float* r, float* p /*direction*/,
                    const float* hp, int64_t n, void* ws, int use_graph, void* stream);

/* ---- K5 tensor-core building block, exposed for unit tests: C (beta)= A.B with operands rounded to bf16,
 *      fp32 accumulation in registers (wgmma.mma_async).  A[m][k] = A[m*ars+k*acs], B[k][n] = B[k*brs+n*bcs]; dt: 0 f32, 1 bf16 */
int bb_gemm_bf16_tc(int64_t M, int64_t N, int64_t K, const void* A, int dtA, int64_t ars, int64_t acs, const void* B,
                    int dtB, int64_t brs, int64_t bcs, float* C, int64_t crs, int64_t ccs, int beta, void* stream);

/* same contract, operands made TMA-addressable (bf16 packs written to `scratch`) and loaded by the TMA unit;
 * returns 1 if the shape is declined (M, N or K < 64, scratch too small) */
int bb_gemm_bf16_tma(int64_t M, int64_t N, int64_t K, const void* A, int dtA, int64_t ars, int64_t acs, const void* B,
                     int dtB, int64_t brs, int64_t bcs, float* C, int64_t crs, int64_t ccs, int beta, void* scratch,
                     int64_t scratch_bytes, void* stream);

/* every option of the TMA-fed product, for unit tests: npairs (1-2) operand pairs summed into one output,
 *   C[b][m][n] (beta)= sum_p sum_k A_p[b][m][k] B_p[b][k][n] (+ bias[n*bias_stride]),
 * A_p[b][m][k] = A[p][b*a_desc[4p+3] + m*a_desc[4p+1] + k*a_desc[4p+2]] with dtype a_desc[4p] (B likewise:
 * b_desc[4p..4p+3] = dt, brs, bcs, bbs), C[b][m][n] = C[b*cbs + m*crs + n*ccs], or the NCHW plane layout
 * C[(img*N + n)*plane_ohw + q] for m = img*plane_ohw + q when plane_ohw > 0.  flags force the tile width (1: 64,
 * 2: 128), turn the persistent kernel off (4) or force a split-K count (n << 8).  route (7 ints) receives the
 * configuration launched: bn, ksplit, persistent, then the operand layouts of A_0, B_0, A_1, B_1 (0 k-major,
 * 1 m/n-major, -1 absent).  Returns 1 if the launcher declines the job. */
int bb_gemm_bf16_tma_ex(int64_t M, int64_t N, int64_t K, int npairs, int64_t batch, const void* const* A,
                        const int64_t* a_desc, const void* const* B, const int64_t* b_desc, float* C, int64_t crs,
                        int64_t ccs, int64_t cbs, int beta, const float* bias, int64_t bias_stride, int plane_ohw,
                        int min_n, int flags, void* scratch, int64_t scratch_bytes, int* route, void* stream);

const char* bb_version(void);

#ifdef __cplusplus
}
#endif
#endif
