"""Neumann and CG hypergradients through the DARTS search networks on the GPU: the native plan against the float64
interpreter of the same IR per value, CUDA-graph replay against the eager loop, and ``betty_b200.install()`` against
the real reference on the same GPU -- including a second call with a new batch and new architecture weights, which
must not serve stale softmax-weight constants.  The second call is asserted to be a plan-cache hit, so it runs through
HvpPlan.rebind: the new forward's values behind the cached pointers, the mixed-op weights rebuilt by their recipes, the
cat slices refreshed through their tape tensors and the contiguous copies of strided conv inputs recomputed.

Mutants these tests catch: cat writing an input at the wrong channel offset (the per-value plan-vs-interpreter compare;
on CPU the interpreter-vs-autograd test of tests/test_darts_implicit_cpu.py), the excluded-padding divisor counting
padded taps (per-value compare of the pooled tangent), a rebind that leaves a contiguous copy or a softmax-weight
constant stale (the second reference call)."""
import pytest
import torch
import torch.nn.functional as F

from betty_b200 import engine as E
from betty_b200 import workloads as W
from betty_b200.arena import ArenaLayout, pack
from betty_b200.ir import lower_tape
from betty_b200.plan import HvpPlan
from betty_b200.trace import record_tape
from oracle import reference as R
from tests.helpers import assert_close, rel_l2
from tests.interp_ext import Interp

pytestmark = pytest.mark.gpu

NETS = {
    "lite": ("neural_architecture_search", dict(batch=4, c=8, cells=2)),
    "full": ("neural_architecture_search_full", dict(batch=4, c=8, layers=3)),
}


def _fp32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _compare(plan, interp, kind, tol, what):
    bad = []
    for vn, vi in zip(plan.g.values, interp.g.values):
        if vn.parent is not None or not vn.needed or vn.param_index is not None:
            continue
        a, b = getattr(vn, kind), getattr(vi, kind)
        err = float((a.double() - b).norm() / (b.norm() + 1e-30)) if float(b.norm()) > 0 else float(a.double().norm())
        if not err <= tol:
            prod = [n.op for n in plan.g.nodes if n.out is vn]
            bad.append(f"{what}: value #{vn.vid} {tuple(vn.base.shape)} {kind} rel={err:.3e} producer={prod}")
    assert not bad, "\n".join(bad[:12])


@pytest.mark.parametrize("net", sorted(NETS))
def test_darts_plan_matches_interpreter(net):
    _fp32()
    fac, kw = NETS[net]
    wl = W.FACTORIES[fac](device="cuda", method="neumann", l2=0.01, **kw)
    params = wl.lower.trainable_parameters()
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    lay = ArenaLayout.like(params)
    d, hv = lay.new(params[0].device), lay.new(params[0].device)
    plan = HvpPlan(tape, params, lay, d, hv, cuda_graph=False)
    assert any(n.op == "conv2d" and n.attrs["groups"] > 1 for n in plan.g.nodes)
    interp = Interp(lower_tape(tape), torch.float64)
    interp.base_backward()
    _compare(plan, interp, "a", 2e-5, "base-backward")
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    for trial in range(2):
        vec = [torch.randn_like(p) for p in params] if trial else list(wl.vector)
        pack(lay, vec, d)
        plan()
        want_i = interp.hvp(vec)
        _compare(plan, interp, "t", 5e-5, "tangent-forward")
        _compare(plan, interp, "at", 2e-4, "tangent-backward")
        got = lay.views(hv)
        assert rel_l2(got, want_i) < 1e-4
        want_a = torch.autograd.grad(in_grad, params, grad_outputs=vec, retain_graph=True)
        assert rel_l2(got, want_a) < 1e-4
        for g_, i_ in zip(got, want_i):
            if float(i_.norm()) > 0:
                assert rel_l2([g_], [i_]) < 1e-3, f"{net}: tensor {tuple(g_.shape)}"


@pytest.mark.parametrize("method", ("neumann", "cg"))
def test_darts_graph_replay_equals_eager_loop(method):
    _fp32()
    outs = []
    try:
        for graph in (False, True):
            E.settings.cuda_graph = graph
            wl = W.darts_search_full(device="cuda", batch=4, c=8, layers=3, method=method, K=6, l2=0.01)
            call = E.HypergradientCall(wl.lower, method)
            outs.append([t.clone() for t in call.solve(wl.vector)])
            outs.append([t.clone() for t in call.solve(wl.vector)])
    finally:
        E.settings.cuda_graph = True
    for o in outs[1:]:
        assert rel_l2(o, outs[0]) < 1e-5


def _upper_step(p, batch):
    x, y = batch
    return F.cross_entropy(p.peers["lower"].module(x, p.module()), y)


REF_CASES = {f"{net}_{m}": (net, m) for net in NETS for m in ("neumann", "cg")}


@pytest.fixture
def reference_table():
    R.load()
    import betty.hypergradient as RH

    keep = dict(RH.jvp_fn_mapping)
    yield RH
    RH.jvp_fn_mapping.clear()
    RH.jvp_fn_mapping.update(keep)


def _tolerance(upper, lower, want):
    again = R.hypergradient_through_reference(upper, lower)
    self_dist = rel_l2(again, want)
    return self_dist, (1e-4 if self_dist <= 2e-5 else 1e-4 + self_dist)


@pytest.mark.skipif(not R.available(), reason="oracle/_ref not fetched (bash oracle/fetch_ref.sh)")
@pytest.mark.parametrize("case", sorted(REF_CASES))
def test_install_matches_reference_on_darts(case, reference_table):
    import betty_b200

    _fp32()
    net, method = REF_CASES[case]
    fac, kw = NETS[net]
    wl = W.FACTORIES[fac](device="cpu", method=method, K=5, alpha=0.01, l2=0.01, **kw)
    engine, upper, lower = R.real_problems(wl, _upper_step, strategy="gpu")
    want = R.hypergradient_through_reference(upper, lower)
    self_dist, tol = _tolerance(upper, lower, want)
    keep = dict(reference_table.jvp_fn_mapping)
    betty_b200.install()
    got = R.hypergradient_through_reference(upper, lower)
    e = assert_close(got, want, tol, case)
    print(f"[darts reference parity] {case}: rel-L2 {e:.3e}, reference-vs-reference {self_dist:.3e}, tol {tol:.2e}")

    # second call: new batch and new architecture weights (new softmax-weight constants in the lower forward)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for a in upper.module.parameters():
            a.add_(0.5 * torch.randn(a.shape, generator=g).to(a.device))
    x, y = lower.cur_batch
    lower.cur_batch = (torch.randn(x.shape, generator=g).to(x.device), y.flip(0))
    hits = E.plan_cache.hits
    got2 = R.hypergradient_through_reference(upper, lower)
    assert E.plan_cache.hits == hits + 1, "the second call did not reuse the cached plan"
    reference_table.jvp_fn_mapping.update(keep)
    want2 = R.hypergradient_through_reference(upper, lower)
    self2, tol2 = _tolerance(upper, lower, want2)
    assert rel_l2(want2, want) > 1e-3, "the second call did not change the problem"
    e2 = assert_close(got2, want2, tol2, case + " second call")
    print(f"[darts reference parity] {case} second call: rel-L2 {e2:.3e}, reference self {self2:.3e}")

