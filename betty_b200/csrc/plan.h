// Node descriptor of the second-order tape ("HVP plan").  Filled by betty_b200/plan.py through a numpy
// structured dtype with the same layout (checked against bb_node_bytes()).  Semantics of the three
// passes are specified in betty_b200/ir.py and restated executable in oracle/plan_interp.py.
#pragma once
#include <stdint.h>

#define BB_MAX_DIMS 6

enum bb_op {
  BB_OP_UNARY = 1,    // y = f(x)                       kind = bb_unary_kind, f[0] = scalar
  BB_OP_COPY = 2,     // y = x (strided gather)
  BB_OP_ADD2 = 3,     // y = f[1]*a + f[2]*b
  BB_OP_MULC = 4,     // y = c * x, c constant tensor (aux[0], fp32, strides in stride[2])
  BB_OP_MUL2 = 5,     // y = a * b
  BB_OP_SUMALL = 6,   // y = f[0] * sum(x)
  BB_OP_GEMM = 7,     // C = A.B (+ bias)               dims = M,N,K,batch
  BB_OP_CONV2D = 8,   // NCHW direct/implicit-GEMM conv dims = N,C,H,W,O,KH,KW,HO,WO,sh,sw,ph,pw,dh,dw,groups
  BB_OP_MAXPOOL2D = 9,  // gather/scatter with the base argmax (aux[0] = int64 indices) dims = NC, HW, HOWO
  BB_OP_BATCHNORM = 10, // batch statistics, NCHW       dims = N,C,HW   f[0]=eps  aux[0]=double scratch[C*16]
  BB_OP_LAYERNORM = 11, // last-dim statistics          dims = rows,D   f[0]=eps  aux[0]=float stats[rows*4]
  BB_OP_SOFTMAX = 12,   // last dim                     dims = rows,D
  BB_OP_LOGSOFTMAX = 13,
  BB_OP_NLL = 14,       // dims = B,C  aux[0]=int64 target  kind=reduction(0 none,1 mean,2 sum) f[0]=scale
  BB_OP_BCE_LOGITS = 15,// mean reduction               n  aux[0] = fp32 targets
  BB_OP_EMBEDDING = 16, // dims = nidx,D,V,padding_idx  aux[0] = int64 indices, aux[1] = sorted token positions + run ends (plan.py _n_embedding)
  BB_OP_AVGPOOL2D = 18, // linear: dims = NC,H,W,HO,WO,kh,kw,sh,sw,ph,pw  f[0] = 1/divisor
                        // kind bit 0: count_include_pad=False, each window divided by its in-image taps (f[0] unused)
  BB_OP_CONVBLOCK = 19, // fused data-input conv3x3 -> BatchNorm -> [ReLU] -> MaxPool2d(2) (convblock.cu)
  BB_OP_CONVBLOCK2 = 20, // fused inner conv3x3 -> BatchNorm -> [ReLU] -> MaxPool2d(2) of a bf16 graph (convblock2.cu)
  BB_OP_DIAGSHIFT = 17, // folded c*sum((w-const)^2): at_w += f[0]*t_w over aux[0] = bb_mt_chunk[dims[0]] {a=t_w, b=at_w}
};

enum bb_unary_kind { BB_U_RELU = 1, BB_U_GELU = 2, BB_U_TANH = 3, BB_U_SIGMOID = 4, BB_U_POW = 5, BB_U_SCALE = 6 };

// operand slots: 0,1,2 = inputs, 3 = output
struct bb_node {
  int32_t op;
  int32_t kind;
  int32_t active;   // bit i: input i is parameter-dependent (has t / a / at buffers)
  int32_t linear;   // elementwise ops: every operand is dense with identical strides -> index memory linearly
  int32_t beta[4];  // adjoint write mode per input: 0 overwrite, 1 accumulate
  int32_t dt[4];    // dtype of base[s]: BB_F32 / BB_BF16
  int32_t ndim;
  int32_t pad0;
  int64_t n;        // elements of the output (elementwise) / of the input (sumall)
  int64_t dims[16];
  double f[4];
  void* base[4];
  void* t[4];
  void* a[4];
  void* at[4];
  void* aux[4];
  int64_t sizes[BB_MAX_DIMS];
  int64_t stride[4][BB_MAX_DIMS];
};

#ifdef __cplusplus
#include <cuda_runtime.h>
// per-op launchers (each returns 0 or an error code); `pass` is BB_PASS_*
int bb_launch_ew(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_sumall(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_gemm(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_conv2d(const bb_node& nd, int pass, cudaStream_t s);
// depthwise conv2d (dims[15] = groups = C = O): input and weight terms of every pass (conv_dw.cu)
int bb_conv_dw_run(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_maxpool2d(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_batchnorm(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_layernorm(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_softmax(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_nll(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_bce(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_embedding(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_avgpool2d(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_convblock(const bb_node& nd, int pass, cudaStream_t s);
int bb_launch_convblock2(const bb_node& nd, int pass, cudaStream_t s);
// number of kernel launches (incl. memsets) the call above makes, for bench.py's gpu_launches
extern thread_local int bb_launch_tally;
#endif
