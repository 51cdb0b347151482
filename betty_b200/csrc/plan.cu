// Executor of the second-order tape: walks the node list (forward for tangents, reverse for adjoints),
// and drives whole Neumann / CG K-loops natively so Python is out of the loop: one iteration
// (tangent forward, tangent backward, vector update kernels) is captured into a CUDA graph and replayed.
// Replaces reference neumann.py:61-64 and cg.py:38-55 (Python loops around autograd.grad).
#include <vector>

#include "../../include/betty_b200.h"
#include "bb_common.cuh"
#include "plan.h"
#include "tma.h"
#include "conv_tma.h"

struct bb_plan {
  std::vector<bb_node> nodes;
  std::vector<void*> zero_ptr[3];
  std::vector<int64_t> zero_bytes[3];
  int launches[3] = {0, 0, 0};
  void* scratch = nullptr;      // bf16 operand packs of the TMA-fed tensor-core path (tma.h)
  int64_t scratch_bytes = 0;
  float* reduce_ws = nullptr;   // fixed-order reductions of the node launchers (tma.h BbReduceWs), allocated on first run
  uint8_t* persist = nullptr;   // plan-lifetime packs of K-loop constants, bump-allocated per node
  int64_t persist_bytes = 0, persist_used = 0;
  std::vector<void*> node_persist;
  // One captured iteration per loop kind (0 Neumann, 1 CG, 2 bare H.d), kept for the plan's lifetime and relaunched
  // by every later K-loop on the same arenas: capture + instantiate (0.5 ms ... 15 ms for ~1000 nodes) is paid
  // once per plan, not once per solve.  The key holds everything the captured kernels have baked in.
  struct LoopKey {
    const void* ptr[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    int64_t n = 0;
    float alpha = 0.f;
    bool operator==(const LoopKey& o) const {
      for (int i = 0; i < 5; ++i)
        if (ptr[i] != o.ptr[i]) return false;
      return n == o.n && alpha == o.alpha;
    }
  };
  int shift_node = -1;          // BB_OP_DIAGSHIFT covering every parameter: applied by K1-K3 inside the K-loops
  float shift = 0.f;
  cudaGraphExec_t exec[3] = {nullptr, nullptr, nullptr};
  LoopKey key[3];
  int graph_captures = 0;
  void drop_graphs() {
    for (auto& e : exec) {
      if (e) cudaGraphExecDestroy(e);
      e = nullptr;
    }
  }
  ~bb_plan() { drop_graphs(); }
};

namespace {
thread_local bb_plan* t_plan = nullptr;
thread_local int t_node = -1;
}  // namespace

void* bb_persist_get(size_t bytes, bool* fresh, int slot_id) {
  *fresh = false;
  bb_plan* p = t_plan;
  if (!p || !p->persist || t_node < 0 || slot_id < 0 || slot_id >= BB_PERSIST_SLOTS) return nullptr;
  const size_t at_slot = (size_t)t_node * BB_PERSIST_SLOTS + slot_id;
  if (at_slot >= p->node_persist.size()) return nullptr;
  void*& slot = p->node_persist[at_slot];
  if (slot) return slot;
  const int64_t at = (p->persist_used + 255) & ~(int64_t)255;
  if (at + (int64_t)bytes > p->persist_bytes) return nullptr;
  slot = p->persist + at;
  p->persist_used = at + (int64_t)bytes;
  *fresh = true;
  return slot;
}

namespace {

int dispatch(const bb_node& nd, int pass, cudaStream_t s) {
  switch (nd.op) {
    case BB_OP_UNARY:
    case BB_OP_COPY:
    case BB_OP_ADD2:
    case BB_OP_MULC:
    case BB_OP_MUL2:
      return bb_launch_ew(nd, pass, s);
    case BB_OP_SUMALL:
      return bb_launch_sumall(nd, pass, s);
    case BB_OP_GEMM:
      return bb_launch_gemm(nd, pass, s);
    case BB_OP_CONV2D:
      return bb_launch_conv2d(nd, pass, s);
    case BB_OP_MAXPOOL2D:
      return bb_launch_maxpool2d(nd, pass, s);
    case BB_OP_BATCHNORM:
      return bb_launch_batchnorm(nd, pass, s);
    case BB_OP_LAYERNORM:
      return bb_launch_layernorm(nd, pass, s);
    case BB_OP_SOFTMAX:
    case BB_OP_LOGSOFTMAX:
      return bb_launch_softmax(nd, pass, s);
    case BB_OP_NLL:
      return bb_launch_nll(nd, pass, s);
    case BB_OP_BCE_LOGITS:
      return bb_launch_bce(nd, pass, s);
    case BB_OP_EMBEDDING:
      return bb_launch_embedding(nd, pass, s);
    case BB_OP_AVGPOOL2D:
      return bb_launch_avgpool2d(nd, pass, s);
    case BB_OP_CONVBLOCK:
      return bb_launch_convblock(nd, pass, s);
    case BB_OP_CONVBLOCK2:
      return bb_launch_convblock2(nd, pass, s);
    case BB_OP_DIAGSHIFT: {
      if (pass != BB_PASS_TAN_BWD) return BB_OK;
      bb_launch_tally += 1;
      return bb_mt_axpby(reinterpret_cast<const bb_mt_chunk*>(nd.aux[0]), (int)nd.dims[0], (float)nd.f[0], nullptr, 1.0f,
                         (void*)s);
    }
    default:
      return BB_ERR_UNSUPPORTED;
  }
}

// 24 MB holds the per-CTA weight-gradient partials of a 64 -> 64 channel 3x3 convolution on every SM (132 x 144 KB) and
// the split-K partials of the SIMT products; launchers split less when a reduction would not fit.
constexpr size_t kReduceWsBytes = 24u << 20;

// Allocated by the first pass, which runs eagerly before any K-loop capture.
cudaError_t publish_reduce_ws(bb_plan* p) {
  if (p->reduce_ws == nullptr) {
    const cudaError_t e = cudaMalloc(&p->reduce_ws, kReduceWsBytes);
    if (e != cudaSuccess) {
      p->reduce_ws = nullptr;
      return e;
    }
  }
  bb_reduce_ws = BbReduceWs{p->reduce_ws, kReduceWsBytes};
  return cudaSuccess;
}

int run_pass(bb_plan* p, int pass, cudaStream_t s, bool in_loop = false) {
  if (pass < 0 || pass > 2) return BB_ERR_ARG;
  const int skip = in_loop ? p->shift_node : -1;
  BB_CUDA_TRY(publish_reduce_ws(p));
  bb_scratch = BbScratch{reinterpret_cast<uint8_t*>(p->scratch), (size_t)p->scratch_bytes, 0};
  bb_scratch_reset();
  const int tally0 = bb_launch_tally;
  for (size_t i = 0; i < p->zero_ptr[pass].size(); ++i) {
    BB_CUDA_TRY(cudaMemsetAsync(p->zero_ptr[pass][i], 0, (size_t)p->zero_bytes[pass][i], s));
    bb_launch_tally += 1;
  }
  const int n = (int)p->nodes.size();
  t_plan = p;
  if (pass == BB_PASS_TAN_FWD) {
    for (int i = 0; i < n; ++i) {
      t_node = i;
      const int rc = dispatch(p->nodes[i], pass, s);
      if (rc) return rc;
    }
  } else {
    for (int i = n - 1; i >= 0; --i) {
      if (i == skip) continue;
      t_node = i;
      const int rc = dispatch(p->nodes[i], pass, s);
      if (rc) return rc;
    }
  }
  t_node = -1;
  if (!in_loop) p->launches[pass] = bb_launch_tally - tally0;
  return BB_OK;
}

template <class Body>
int loop_with_graph(bb_plan* plan, int kind, const bb_plan::LoopKey& key, int iterations, int use_graph, cudaStream_t s,
                    Body body) {
  if (iterations <= 0) return BB_OK;
  if (!use_graph) {
    for (int k = 0; k < iterations; ++k) {
      const int rc = body();
      if (rc) return rc;
    }
    return BB_OK;
  }
  if (plan->exec[kind] && !(plan->key[kind] == key)) {
    cudaGraphExecDestroy(plan->exec[kind]);
    plan->exec[kind] = nullptr;
  }
  if (!plan->exec[kind]) {
    cudaGraph_t graph = nullptr;
    BB_CUDA_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
    const int rc = body();
    cudaError_t e = cudaStreamEndCapture(s, &graph);
    if (rc) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (e != cudaSuccess) return (int)e;
    e = cudaGraphInstantiate(&plan->exec[kind], graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
      plan->exec[kind] = nullptr;
      return (int)e;
    }
    plan->key[kind] = key;
    plan->graph_captures += 1;
  }
  for (int k = 0; k < iterations; ++k) BB_CUDA_TRY(cudaGraphLaunch(plan->exec[kind], s));
  return BB_OK;
}

}  // namespace

extern "C" {

int bb_node_bytes(void) { return (int)sizeof(bb_node); }

int bb_plan_create(const struct bb_node* nodes, int n_nodes, bb_plan** out) {
  if (!out || n_nodes < 0 || (n_nodes > 0 && !nodes)) return BB_ERR_ARG;
  bb_plan* p = new bb_plan();
  p->nodes.assign(nodes, nodes + n_nodes);
  p->node_persist.assign((size_t)n_nodes * BB_PERSIST_SLOTS, nullptr);
  *out = p;
  return BB_OK;
}

int bb_plan_destroy(bb_plan* plan) {
  if (plan && plan->reduce_ws) {
    if (bb_reduce_ws.base == plan->reduce_ws) bb_reduce_ws = BbReduceWs{nullptr, 0};
    cudaFree(plan->reduce_ws);
  }
  delete plan;
  return BB_OK;
}

int bb_plan_set_zero_regions(bb_plan* plan, int pass, void* const* ptrs, const int64_t* bytes, int n) {
  if (!plan || pass < 0 || pass > 2) return BB_ERR_ARG;
  plan->zero_ptr[pass].assign(ptrs, ptrs + n);
  plan->zero_bytes[pass].assign(bytes, bytes + n);
  return BB_OK;
}

int bb_plan_set_scratch(bb_plan* plan, void* ptr, int64_t bytes) {
  if (!plan || bytes < 0) return BB_ERR_ARG;
  plan->scratch = ptr;
  plan->scratch_bytes = bytes;
  return BB_OK;
}

int bb_plan_set_persistent(bb_plan* plan, void* ptr, int64_t bytes) {
  if (!plan || bytes < 0) return BB_ERR_ARG;
  plan->persist = reinterpret_cast<uint8_t*>(ptr);
  plan->persist_bytes = bytes;
  plan->persist_used = 0;
  plan->node_persist.assign(plan->nodes.size() * BB_PERSIST_SLOTS, nullptr);
  plan->drop_graphs();
  return BB_OK;
}

int bb_plan_invalidate_constants(bb_plan* plan) {
  // the base values behind the plan's pointers were refreshed in place (a cached plan serving a new batch): packs of
  // K-loop constants must be rebuilt by the next base-backward pass.  Addresses are unchanged, so captured graphs stay.
  if (!plan) return BB_ERR_ARG;
  plan->persist_used = 0;
  plan->node_persist.assign(plan->nodes.size() * BB_PERSIST_SLOTS, nullptr);
  return BB_OK;
}

int bb_plan_graph_captures(const bb_plan* plan) { return plan ? plan->graph_captures : BB_ERR_ARG; }

int bb_plan_node_route(bb_plan* plan, int node, int pass) {
  // introspection for the unit tests: 2 = TMA-fed tensor-core convolution path takes (node, pass), 0 = another path
  if (!plan || node < 0 || node >= (int)plan->nodes.size()) return BB_ERR_ARG;
  BB_CUDA_TRY(publish_reduce_ws(plan));
  bb_scratch = BbScratch{reinterpret_cast<uint8_t*>(plan->scratch), (size_t)plan->scratch_bytes, 0};
  const bb_node& nd = plan->nodes[node];
  if (nd.op == BB_OP_CONV2D && bb_conv_tma_ok(nd, pass)) return 2;
  return 0;
}

int bb_plan_run(bb_plan* plan, int pass, void* stream) {
  if (!plan) return BB_ERR_ARG;
  return run_pass(plan, pass, (cudaStream_t)stream);
}

int bb_plan_launch_count(const bb_plan* plan, int pass) {
  if (!plan || pass < 0 || pass > 2) return BB_ERR_ARG;
  return plan->launches[pass];
}

int bb_plan_hvp(bb_plan* plan, void* stream) {
  if (!plan) return BB_ERR_ARG;
  int rc = run_pass(plan, BB_PASS_TAN_FWD, (cudaStream_t)stream);
  if (rc) return rc;
  return run_pass(plan, BB_PASS_TAN_BWD, (cudaStream_t)stream);
}

// H.d without the uniform c*I term (the K-loop kernels apply it as their `shift`)
static int hvp_in_loop(bb_plan* plan, cudaStream_t s) {
  int rc = run_pass(plan, BB_PASS_TAN_FWD, s, true);
  if (rc) return rc;
  return run_pass(plan, BB_PASS_TAN_BWD, s, true);
}

int bb_plan_set_uniform_shift(bb_plan* plan, int node, double coef) {
  if (!plan || node >= (int)plan->nodes.size()) return BB_ERR_ARG;
  if (node >= 0 && plan->nodes[node].op != BB_OP_DIAGSHIFT) return BB_ERR_ARG;
  plan->shift_node = node;
  plan->shift = node >= 0 ? (float)coef : 0.f;
  plan->drop_graphs();
  return BB_OK;
}

int bb_plan_hvp_replay(bb_plan* plan, void* stream) {
  // H.d as one graph launch (epilogue pass along x, benchmarks of the bare product)
  if (!plan) return BB_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  bb_plan::LoopKey key;
  return loop_with_graph(plan, 2, key, 1, 1, s, [&]() -> int { return bb_plan_hvp(plan, s); });
}

int bb_plan_profile(bb_plan* plan, int pass, float* ms_per_node, void* stream) {
  if (!plan || pass < 0 || pass > 2 || !ms_per_node) return BB_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  BB_CUDA_TRY(publish_reduce_ws(plan));
  bb_scratch = BbScratch{reinterpret_cast<uint8_t*>(plan->scratch), (size_t)plan->scratch_bytes, 0};
  bb_scratch_reset();
  const int n = (int)plan->nodes.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) BB_CUDA_TRY(cudaEventCreate(&e));
  for (size_t i = 0; i < plan->zero_ptr[pass].size(); ++i)
    BB_CUDA_TRY(cudaMemsetAsync(plan->zero_ptr[pass][i], 0, (size_t)plan->zero_bytes[pass][i], s));
  int rc = BB_OK;
  for (int j = 0; j < n && !rc; ++j) {
    const int i = (pass == BB_PASS_TAN_FWD) ? j : n - 1 - j;
    cudaEventRecord(ev[j], s);
    t_plan = plan;
    t_node = i;
    rc = dispatch(plan->nodes[i], pass, s);
    ms_per_node[i] = 0.f;
  }
  cudaEventRecord(ev[n], s);
  cudaStreamSynchronize(s);
  if (!rc) {
    for (int j = 0; j < n; ++j) {
      const int i = (pass == BB_PASS_TAN_FWD) ? j : n - 1 - j;
      cudaEventElapsedTime(&ms_per_node[i], ev[j], ev[j + 1]);
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

int bb_plan_neumann_loop(bb_plan* plan, int iterations, float alpha, float* v, float* p, const float* hv, int64_t n,
                         int use_graph, void* stream) {
  if (!plan) return BB_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  bb_plan::LoopKey key;
  key.ptr[0] = v; key.ptr[1] = p; key.ptr[2] = hv; key.n = n; key.alpha = alpha;
  return loop_with_graph(plan, 0, key, iterations, use_graph, s, [&]() -> int {
    int rc = hvp_in_loop(plan, s);                                    // hv <- H v        (neumann.py:62)
    if (rc) return rc;
    return bb_neumann_update(v, p, hv, alpha, plan->shift, n, s);     // v, p updates     (neumann.py:63-64)
  });
}

int bb_plan_cg_loop(bb_plan* plan, int iterations, float cg_alpha, float* x, float* r, float* p, const float* hp,
                    int64_t n, void* ws, int use_graph, void* stream) {
  if (!plan) return BB_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  int rc = bb_cg_init(r, n, ws, s);                           // rr = r.r         (cg.py:45, first iteration)
  if (rc) return rc;
  bb_plan::LoopKey key;
  key.ptr[0] = x; key.ptr[1] = r; key.ptr[2] = p; key.ptr[3] = hp; key.ptr[4] = ws; key.n = n; key.alpha = cg_alpha;
  return loop_with_graph(plan, 1, key, iterations, use_graph, s, [&]() -> int {
    int rc2 = hvp_in_loop(plan, s);                                   // hp <- H p        (cg.py:39-41)
    if (rc2) return rc2;
    rc2 = bb_cg_dots(r, hp, p, cg_alpha, plan->shift, 0, n, ws, s);   // alpha            (cg.py:42-47)
    if (rc2) return rc2;
    rc2 = bb_cg_update_xr(x, r, p, hp, plan->shift, n, ws, s);        // x, r, beta       (cg.py:49-52)
    if (rc2) return rc2;
    return bb_cg_update_p(p, r, n, ws, s);                    // p                (cg.py:53)
  });
}

const char* bb_version(void) { return "betty_b200 0.1.0 (sm_90a)"; }

}  // extern "C"
