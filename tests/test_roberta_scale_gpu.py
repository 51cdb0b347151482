"""The transformer kernels at the scale of the benchmark's bert_data_reweighting line: RoBERTa-base, B=16 x L=50 = 800
tokens, hidden 768, 12 heads, FFN 3072, vocabulary 50 265.

At this size the code takes branches that the small RoBERTa cases of tests/test_plan_gpu.py never reach:
ln_row_kernel (norm.cu) handles rows / 132 = 6 rows per block and carries its parameter-adjoint sums across them,
D = 768 leaves two of its eight warps idle, the GEMM cost model (gemm_tma.cu) picks split-K at 800 x 768 x 3072 and
at the K = 800 weight gradients, and the attention products run batched over 192 (sequence, head) slices.

Checks:
  * every tangent and adjoint tangent against the float64 interpreter of the same IR (oracle/plan_interp.py), one
    sequence at a time (a lost 128-row tile spans 2.5 sequences and moves them by far more than a global norm shows),
    each failure named by its producer op; each H.v tensor by parameter name (the word-embedding, position-embedding
    and LayerNorm gamma / beta adjoints each on their own).  fp32 at 2 layers (the float64 interpreter of the full
    depth is large; the peak is printed), bf16 at the benchmark's full depth;
  * LayerNorm's two routes (ln_row_kernel, and ln_kernel under BB200_LN_WARP) against each other and against fp64;
  * run-to-run and plan-to-plan bit identity of H.v and of a K=3 CG loop;
  * the benchmark's own configuration against autograd's bf16 double backward.
Each case prints its worst errors and its peak device memory; DESIGN.md section 4 records them."""
import gc

import pytest
import torch

from betty_b200 import workloads as W
from betty_b200.arena import ArenaLayout, pack
from betty_b200.engine import Workspace
from betty_b200.ir import lower_tape
from betty_b200.plan import HvpPlan
from betty_b200.trace import record_tape
from oracle.plan_interp import Interp
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu

SM = 132
BATCH, SEQ, HEADS = 16, 50, 12
PEAK_MAX = 40 * 2 ** 30           # the GPUs are shared: every case stays well under this

# name: (factory kwargs, per-sequence bars of the tangents and of the adjoint tangents, per-tensor H.v bar, whole H.v
# bar).  fp32: the plan tests' 1e-4 scale; measured worst 4.8e-6 / 3.0e-6 / 1.8e-6 / 1.3e-6.  bf16: about 3.5 x the
# measured worst 4.5e-3 / 5.9e-3 / 3.7e-3 / 2.5e-3 (H100 SXM 80 GB, 700 W; DESIGN.md section 4).
CASES = {
    "fp32_l2": (dict(layers=2), 1e-4, 1e-4, 1e-4, 1e-4),
    "bf16": (dict(precision="bf16"), 1.5e-2, 2e-2, 1.5e-2, 1e-2),
}


def _fresh():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def _peak(what):
    peak = torch.cuda.max_memory_allocated()
    print(f"[roberta scale] {what}: peak device memory {peak / 2 ** 30:.2f} GiB")
    assert peak < PEAK_MAX, f"{what}: {peak / 2 ** 30:.2f} GiB"


def _workload(case):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    kw = dict(method="cg", batch=BATCH, seq=SEQ, K=10, **CASES[case][0])
    wl = W.FACTORIES["bert_data_reweighting"](device="cuda", **kw)
    names = [nm for nm, _ in wl.lower.module.named_parameters()]
    params = wl.lower.trainable_parameters()
    assert len(names) == len(params)
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    return wl, names, params, loss, tape


def _plan(tape, params):
    lay = ArenaLayout.like(params)
    d, hv = lay.new(params[0].device), lay.new(params[0].device)
    return lay, d, hv, HvpPlan(tape, params, lay, d, hv, cuda_graph=False)


def _hvp(plan, lay, d, hv, vec):
    pack(lay, vec, d)
    plan()
    torch.cuda.synchronize()
    return hv.clone()


def _where(plan, vn):
    prod = [n for n in plan.g.nodes if n.out is vn]
    cons = [n.op for n in plan.g.nodes if any(x is not None and x.root is vn for x in n.ins)]
    return f"producer={prod[0].op if prod else None} consumers={cons}"


def _per_sequence(a, b):
    """Relative L2 per sequence of a token-major value ([16][...], [800][...] or [192 = 16 x 12][...]); None when the
    value is not laid out by sequence."""
    if a.dim() == 0 or a.shape[0] not in (BATCH, BATCH * SEQ, BATCH * HEADS):
        return None
    a, b = a.double().reshape(BATCH, -1), b.double().reshape(BATCH, -1)
    bn, dn = b.norm(dim=1), (a - b).norm(dim=1)
    return torch.where(bn > 0, dn / bn.clamp_min(1e-300), dn)


def _compare_per_sequence(plan, interp, kind, tol, what):
    """Every value: per sequence where it is laid out by sequence, else one relative L2.  Returns the worst."""
    bad, worst = [], (0.0, "")
    for vn, vi in zip(plan.g.values, interp.g.values):
        if vn.parent is not None or not vn.needed or vn.param_index is not None:
            continue
        a, b = getattr(vn, kind), getattr(vi, kind)
        per = _per_sequence(a, b)
        if per is None:
            e, s = (float((a.double() - b).norm() / b.norm()) if float(b.norm()) > 0 else float(a.double().norm())), -1
        else:
            e, s = (float(x) for x in per.max(0))
        desc = f"{what}: value #{vn.vid} {tuple(vn.base.shape)} kind={kind} worst sequence {int(s)} rel={e:.3e} {_where(plan, vn)}"
        if e > worst[0]:
            worst = (e, desc)
        if not (e <= tol):
            bad.append(desc)
    assert not bad, "\n".join(bad[:12])
    return worst


def _check_params(names, got, want, tol, what):
    """Per-parameter relative L2 of H.v, named.  Returns {name: error}."""
    errs, bad = {}, []
    for nm, g_, w_ in zip(names, got, want):
        if float(w_.norm()) > 0:
            errs[nm] = rel_l2([g_], [w_])
            if not (errs[nm] < tol):
                bad.append(f"{what}: H.v {nm} {tuple(g_.shape)}: rel={errs[nm]:.3e}")
    assert not bad, "\n".join(bad)
    return errs


def _embedding_and_ln(errs):
    keys = [k for k in errs if "embeddings." in k]
    return ", ".join(f"{k.replace('roberta.embeddings.', '')} {errs[k]:.2e}" for k in keys)


# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(CASES))
def test_roberta_matches_interpreter_per_sequence(case):
    _fresh()
    _, tol_t, tol_at, tol_param, tol_hv = CASES[case]
    wl, names, params, loss, tape = _workload(case)
    lay, d, hv, plan = _plan(tape, params)
    ln = [n for n in plan.g.nodes if n.op == "layernorm"]
    assert ln and all(tuple(n.out.base.shape[-1:]) == (768,) for n in ln)
    assert any(n.out.base.numel() // 768 // SM == 6 for n in ln), "no LayerNorm with 6 rows per ln_row_kernel block"
    vec = list(wl.vector)
    got = [g_.clone() for g_ in lay.views(_hvp(plan, lay, d, hv, vec))]
    interp = Interp(lower_tape(tape), torch.float64)
    interp.base_backward()
    want = interp.hvp(vec)
    wt = _compare_per_sequence(plan, interp, "t", tol_t, f"{case} tangent-forward")
    wat = _compare_per_sequence(plan, interp, "at", tol_at, f"{case} tangent-backward")
    print(f"[roberta scale] {case}: worst per-sequence t {wt[0]:.3e} ({wt[1]})")
    print(f"[roberta scale] {case}: worst per-sequence at {wat[0]:.3e} ({wat[1]})")
    errs = _check_params(names, got, want, tol_param, f"{case} vs fp64 interpreter")
    for must in ("roberta.embeddings.word_embeddings.weight", "roberta.embeddings.position_embeddings.weight",
                 "roberta.embeddings.LayerNorm.weight", "roberta.embeddings.LayerNorm.bias"):
        assert must in errs, f"{case}: H.v of {must} is zero or missing"
    worst = max(errs, key=errs.get)
    e = rel_l2(got, want)
    print(f"[roberta scale] {case}: H.v vs fp64 interpreter {e:.3e}; worst tensor {worst} {errs[worst]:.3e}; "
          f"{_embedding_and_ln(errs)}")
    assert e < tol_hv, f"{case}: H.v vs fp64 interpreter {e:.3e}"
    _peak(f"{case} with the float64 interpreter")


def test_layernorm_routes_agree(monkeypatch):
    """ln_row_kernel (6 rows per block at 800 rows) against ln_kernel (BB200_LN_WARP, read at each launch), fp32:
    every LayerNorm's tangent, adjoint tangent and gamma / beta adjoints; both against float64."""
    _fresh()
    case = "fp32_l2"
    wl, names, params, loss, tape = _workload(case)
    vec = list(wl.vector)
    res = {}
    for route in ("row", "warp"):
        if route == "warp":
            monkeypatch.setenv("BB200_LN_WARP", "1")
        lay, d, hv, plan = _plan(tape, params)
        got = [g_.clone() for g_ in lay.views(_hvp(plan, lay, d, hv, vec))]
        ln = [n for n in plan.g.nodes if n.op == "layernorm"]
        vids = [plan.g.values.index(n.out) for n in ln]
        res[route] = (got, [(n.out.t.clone(), n.ins[0].root.at.clone()) for n in ln])
        del plan, d, hv
    monkeypatch.delenv("BB200_LN_WARP")
    interp = Interp(lower_tape(tape), torch.float64)
    interp.base_backward()
    want = interp.hvp(vec)
    ln_i = [next(n for n in interp.g.nodes if n.out is interp.g.values[v]) for v in vids]
    lnp = [i for i, nm in enumerate(names) if "LayerNorm" in nm]
    assert len(lnp) == 2 * len(ln_i)
    differ = False
    for k, ((t_r, at_r), (t_w, at_w)) in enumerate(zip(res["row"][1], res["warp"][1])):
        differ |= not (torch.equal(t_r, t_w) and torch.equal(at_r, at_w))
        for nm, a, b in (("t_y", t_r, t_w), ("at_x", at_r, at_w)):
            e = rel_l2([a], [b])
            assert e < 1e-5, f"LayerNorm {k} {nm}: ln_row_kernel vs ln_kernel {e:.3e}"
        for route, t_, at_ in (("row", t_r, at_r), ("warp", t_w, at_w)):
            for nm, a, b in (("t_y", t_, ln_i[k].out.t), ("at_x", at_, ln_i[k].ins[0].root.at)):
                e = float(_per_sequence(a, b).max())
                assert e < 1e-4, f"LayerNorm {k} {nm} ({route} route) vs fp64: worst sequence {e:.3e}"
    assert differ, "BB200_LN_WARP did not switch the LayerNorm route (both routes returned the same bits)"
    worst = 0.0
    for i in lnp:
        e_rw = rel_l2([res["row"][0][i]], [res["warp"][0][i]])
        for route in ("row", "warp"):
            e = rel_l2([res[route][0][i]], [want[i]])
            worst = max(worst, e)
            assert e < 3e-4, f"H.v {names[i]} ({route} route) vs fp64 {e:.3e}"
        assert e_rw < 1e-4, f"H.v {names[i]}: routes differ by {e_rw:.3e}"
    print(f"[roberta scale] LayerNorm routes: gamma/beta H.v worst vs fp64 {worst:.3e}")
    _peak("LayerNorm routes")


def test_run_to_run_bit_identity():
    """The benchmark's configuration: the same plan twice, two plans of one tape, and a K=3 CG loop twice return the
    same bits."""
    _fresh()
    wl, names, params, loss, tape = _workload("bf16")
    vec = list(wl.vector)
    lay, d, hv, plan = _plan(tape, params)
    a = _hvp(plan, lay, d, hv, vec)
    b = _hvp(plan, lay, d, hv, vec)

    def first_diff(x, y):
        views_x, views_y = lay.views(x), lay.views(y)
        return next((nm for nm, u, v in zip(names, views_x, views_y) if not torch.equal(u, v)), None)

    assert torch.equal(a, b), f"two runs of one plan differ (first: {first_diff(a, b)})"
    lay2, d2, hv2, plan2 = _plan(tape, params)
    c = _hvp(plan2, lay2, d2, hv2, vec)
    assert torch.equal(a, c), f"two plans of one tape differ (first: {first_diff(a, c)})"
    del plan2, d2, hv2
    loops = []
    for _ in range(2):
        pack(lay, vec, d)
        r, acc, ws = d.clone(), torch.zeros_like(d), Workspace(d.device)
        plan.cg_loop(3, 1.0, acc, r, d, hv, ws)
        torch.cuda.synchronize()
        loops.append((acc.clone(), r.clone()))
    assert torch.equal(loops[0][0], loops[1][0]) and torch.equal(loops[0][1], loops[1][1]), "CG K=3 differs"
    print("[roberta scale] bf16: H.v and CG K=3 bit-identical across runs and plans")
    _peak("bf16 identity")


def test_benchmark_configuration_matches_autograd():
    """bench.py's bert_data_reweighting workload exactly: one H.v against autograd's bf16 double backward."""
    from bench import WORKLOADS

    _fresh()
    fac, kw, _ = WORKLOADS["bert_data_reweighting"]
    assert fac == "bert_data_reweighting" and (kw["batch"], kw["seq"], kw["precision"]) == (BATCH, SEQ, "bf16")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    wl = W.FACTORIES[fac](device="cuda", **kw)
    names = [nm for nm, _ in wl.lower.module.named_parameters()]
    params = wl.lower.trainable_parameters()
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    lay, d, hv, plan = _plan(tape, params)
    vec = list(wl.vector)
    got = [g_.clone() for g_ in lay.views(_hvp(plan, lay, d, hv, vec))]
    del plan, d, hv
    gc.collect()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    want = torch.autograd.grad(in_grad, params, grad_outputs=vec)
    e = rel_l2(got, want)
    errs = _check_params(names, got, want, 1.5e-1, "bench RoBERTa vs autograd")
    worst = max(errs, key=errs.get)
    print(f"[roberta scale] bench bert_data_reweighting: H.v vs autograd bf16 double backward {e:.3e}, "
          f"worst tensor {worst} {errs[worst]:.3e}; {_embedding_and_ln(errs)}")
    assert e < 2e-2, f"H.v vs autograd double backward {e:.3e}"
    _peak("bench bert_data_reweighting")
