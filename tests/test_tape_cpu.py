"""CPU tests of the tape tracer + IR lowering (betty_b200/trace.py, ir.py): the torch interpreter of the
IR (oracle/plan_interp.py) must reproduce autograd's double-backward HVP -- the quantity the reference
evaluates at neumann.py:62 / cg.py:39-41 -- on every workload family, in float64."""
import pytest
import torch

from betty_b200 import workloads as W
from betty_b200.ir import UnsupportedGraph, lower_tape
from betty_b200.trace import record_tape
from oracle.plan_interp import Interp
from tests.helpers import rel_l2, to_double

CASES = {
    "logistic": ("logistic_regression_hpo", dict()),
    "mlp": ("mlp_reweight", dict(batch=16)),
    "lenet": ("learning_to_reweight", dict(batch=4)),
    "fourconv": ("implicit_maml", dict(n=6, hidden=8)),
    "fourconv_mini": ("implicit_maml", dict(n=2, hidden=4, image="miniimagenet")),
    "roberta": ("bert_data_reweighting", dict(batch=3, seq=7, tiny=True)),
    "resnet": ("learning_to_reweight_resnet", dict(batch=4, n=1, width=4)),
}


def trace(wl):
    params = wl.lower.trainable_parameters()
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    assert any(o.out is loss or (isinstance(o.out, (tuple, list)) and any(x is loss for x in o.out)) for o in tape.ops)
    return loss, tape, params


@pytest.mark.parametrize("case", sorted(CASES))
def test_interp_hvp_matches_autograd_double_backward(case):
    fac, kw = CASES[case]
    wl = to_double(W.FACTORIES[fac](device="cpu", **kw))
    loss, tape, params = trace(wl)
    g = lower_tape(tape)
    it = Interp(g, torch.float64)
    it.base_backward()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    # base backward reproduces the plain gradient
    assert rel_l2([p.a for p in g.params], in_grad) < 1e-10
    want = torch.autograd.grad(in_grad, params, grad_outputs=wl.vector, retain_graph=True)
    got = it.hvp(list(wl.vector))
    assert rel_l2(got, want) < 1e-9, case
    # a second direction through the same plan (buffers are reused across K-loop iterations)
    v2 = [torch.randn_like(v) for v in wl.vector]
    want2 = torch.autograd.grad(in_grad, params, grad_outputs=v2, retain_graph=True)
    assert rel_l2(it.hvp(v2), want2) < 1e-9, case


def test_unsupported_graph_raises_instead_of_falling_back():
    wl = W.mlp_reweight(device="cpu", batch=4)

    def step(p, batch):
        x, y = batch
        return torch.cumsum(p.module(x), 1).mean()

    wl.lower._training_step = step
    _, tape, _ = trace(wl)
    with pytest.raises(UnsupportedGraph):
        lower_tape(tape)


def test_dead_branches_and_unused_parameters():
    wl = to_double(W.mlp_reweight(device="cpu", batch=4, l2=0.0))
    extra = torch.nn.Parameter(torch.randn(3, dtype=torch.float64))
    wl.lower.module.register_parameter("unused", extra)
    loss, tape, params = trace(wl)
    vec = [torch.randn_like(p) for p in params]
    k = [i for i, p in enumerate(params) if p is extra][0]
    g = lower_tape(tape)
    it = Interp(g)
    it.base_backward()
    got = it.hvp(vec)
    assert float(got[k].abs().sum()) == 0.0
    in_grad = torch.autograd.grad(loss, params, create_graph=True, allow_unused=True)
    keep = [i for i in range(len(params)) if i != k]
    want = torch.autograd.grad([in_grad[i] for i in keep], [params[i] for i in keep],
                               grad_outputs=[vec[i] for i in keep])
    assert rel_l2([got[i] for i in keep], want) < 1e-9


@pytest.mark.parametrize("case", sorted(CASES))
def test_native_descriptors_build_on_cpu(case):
    """Dry run of betty_b200/plan.py: buffer arenas + bb_node descriptors for every workload family (no launch)."""
    import numpy as np

    from betty_b200.arena import ArenaLayout
    from betty_b200.plan import NODE_DTYPE, OPS, HvpPlan

    fac, kw = CASES[case]
    wl = W.FACTORIES[fac](device="cpu", **kw)
    loss, tape, params = trace(wl)
    lay = ArenaLayout.like(params)
    d, hv = lay.new("cpu"), lay.new("cpu")
    plan = HvpPlan(tape, params, lay, d, hv, dry_run=True)
    assert len(plan.recs) == len(plan.g.nodes) > 0
    assert plan.recs.dtype.itemsize == NODE_DTYPE.itemsize
    assert set(int(o) for o in plan.recs["op"]) <= set(OPS.values())
    # every active input of every node has tangent and adjoint-tangent pointers; outputs too
    for r, n in zip(plan.recs, plan.g.nodes):
        for k, v in enumerate(n.ins[:3] if n.op != "diagshift" else []):
            if v is not None:
                assert r["t"][k] != 0 and r["at"][k] != 0, (n, k)
        if n.op != "diagshift":
            assert r["t"][3] != 0 and r["at"][3] != 0 and r["a"][3] != 0
    # parameter tangents alias the direction arena, adjoint tangents the H.d arena
    lo, hi = d.data_ptr(), d.data_ptr() + 4 * d.numel()
    for p in plan.g.params:
        assert lo <= p.t.data_ptr() < hi and p.at.data_ptr() - hv.data_ptr() == p.t.data_ptr() - lo


@pytest.mark.parametrize("case", sorted(CASES))
def test_native_epilogue_seeds_reproduce_the_mixed_product(case):
    """-(d^2 L/d lambda d w)^T x from the boundary adjoint-tangents of one extra pass + a first-order backward
    through the upper graph == the reference's double backward (neumann.py:50-54), in float64."""
    from betty_b200.engine import chain_boundary_seeds

    fac, kw = CASES[case]
    wl = to_double(W.FACTORIES[fac](device="cpu", **kw))
    loss, tape, params = trace(wl)
    g = lower_tape(tape)
    assert g.native_epilogue_ok and len(g.boundaries) >= 1, case
    it = Interp(g, torch.float64)
    it.base_backward()
    x = [torch.randn_like(p) for p in params]
    lam = wl.upper.trainable_parameters()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    want = torch.autograd.grad(in_grad, lam, grad_outputs=x, allow_unused=True, retain_graph=True)
    want = [torch.zeros_like(p) if t is None else -t for t, p in zip(want, lam)]
    got = chain_boundary_seeds(it.mixed_seeds(x), wl.upper, False)
    assert rel_l2(got, want) < 1e-9, case


def test_uncaptured_upper_dependence_disables_the_native_epilogue():
    wl = W.mlp_reweight(device="cpu", batch=4)
    scale = torch.nn.Parameter(torch.tensor(2.0))
    wl.upper.module.register_parameter("gain", scale)

    def step(p, batch):
        x, y = batch
        out = p.module(x)
        lv = torch.nn.functional.cross_entropy(out, y, reduction="none")
        return (lv * scale).mean()      # broadcast of a 0-dim upper parameter: not captured as a boundary

    wl.lower._training_step = step
    _, tape, _ = trace(wl)
    assert lower_tape(tape).native_epilogue_ok is False


class _PoolNet(torch.nn.Module):
    """conv -> relu -> max-pool variants for the ReLU->pool fold: `share` feeds the ReLU output to a second consumer
    (the fold must not fire), `kernel`/`stride` choose disjoint (2,2), overlapping (3,2) or odd-size windows."""

    def __init__(self, kernel, stride, share, size):
        super().__init__()
        self.conv = torch.nn.Conv2d(2, 3, 3, padding=1)
        self.kernel, self.stride, self.share = kernel, stride, share
        ho = (size - kernel) // stride + 1
        self.fc = torch.nn.Linear(3 * ho * ho, 4)
        self.fc2 = torch.nn.Linear(3, 4)
        self.size = size

    def forward(self, x):
        h = torch.relu(self.conv(x))
        p = torch.nn.functional.max_pool2d(h, self.kernel, self.stride)
        out = self.fc(p.flatten(1))
        if self.share:   # second consumer of the ReLU output
            out = out + self.fc2(torch.nn.functional.avg_pool2d(h, self.size).flatten(1))
        return out


@pytest.mark.parametrize("kernel,stride,share,size,fused", [(2, 2, False, 8, True), (2, 2, False, 7, True),
                                                            (3, 2, False, 9, True), (2, 2, True, 8, False),
                                                            (3, 3, False, 10, True)])
def test_relu_maxpool_fold(kernel, stride, share, size, fused):
    """ir._fuse_relu_maxpool: same H.v as autograd (fp64) whether or not the fold fires; disjoint windows get the
    overwrite (beta = 0) window-form adjoint, overlapping ones keep the accumulate/scatter form."""
    torch.manual_seed(0)
    wl = to_double(W.mlp_reweight(device="cpu", batch=5))
    net = _PoolNet(kernel, stride, share, size).double()
    wl.lower.module = net
    x = torch.randn(5, 2, size, size, dtype=torch.float64)
    y = torch.randint(0, 4, (5,))
    wl.lower.cur_batch = (x, y)
    wl.lower._training_step = lambda p, batch: torch.nn.functional.cross_entropy(p.module(batch[0]), batch[1])
    params = [p for p in net.parameters() if share or p is not net.fc2.weight and p is not net.fc2.bias]
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    g = lower_tape(tape)
    pools = [n for n in g.nodes if n.op == "maxpool2d"]
    assert len(pools) == 1
    assert bool(pools[0].attrs.get("relu")) == fused
    assert bool(pools[0].attrs.get("disjoint")) == (kernel == stride)
    if fused:
        assert not any(n.op == "unary" and n.attrs.get("kind") == "relu" for n in g.nodes)
        assert pools[0].beta[0] == (0 if kernel == stride else 1)
    it = Interp(g, torch.float64)
    it.base_backward()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    assert rel_l2([p.a for p in g.params], in_grad) < 1e-10
    vec = [torch.randn_like(p) for p in params]
    want = torch.autograd.grad(in_grad, params, grad_outputs=vec, retain_graph=True)
    assert rel_l2(it.hvp(vec), want) < 1e-9


def _golden_records():
    import glob
    import os

    from tests.helpers import GOLDEN

    recs = {}
    for d in (GOLDEN, os.path.join(os.path.dirname(GOLDEN), "golden_cpu")):
        for p in sorted(glob.glob(os.path.join(d, "*.pt"))):
            recs[os.path.basename(p)[:-3]] = p
    return recs


@pytest.mark.parametrize("case", sorted(c for c in _golden_records() if "darts" not in c and "sama" not in c))
def test_interpreted_engine_matches_the_real_reference(case):
    """Whole algorithm, no CUDA: tape -> IR (folds included) -> second-order rules (fp64 interpreter) -> the
    reference's Neumann / CG recurrence -> native epilogue seeds, against the hypergradient the REAL
    betty.hypergradient function returned for the same seeded inputs (oracle/make_golden.py).  The golden vectors
    are fp32, so the bar is the reference's own rounding: 1e-4 for the Neumann series, 2e-3 for CG (its fp32
    recurrence amplifies rounding on the small un-shifted problems, cf. tools/parity_margin.py)."""
    from betty_b200.engine import chain_boundary_seeds
    from oracle import ref_port

    rec = torch.load(_golden_records()[case], weights_only=False)
    wl = to_double(W.FACTORIES[rec["factory"]](device="cpu", **rec["kwargs"]))
    loss, tape, params = trace(wl)
    g = lower_tape(tape)
    it = Interp(g, torch.float64)
    it.base_backward()
    cfg = wl.lower.config
    vec = [v.double() for v in wl.vector]
    if rec["method"] == "neumann":
        x = ref_port.neumann_series(vec, it.hvp, cfg.neumann_iterations, cfg.neumann_alpha)
    else:
        x = ref_port.cg_solve(vec, it.hvp, cfg.cg_iterations, cfg.cg_alpha)
    if "ihvp" in rec:
        assert rel_l2(x, rec["ihvp"]) < 1e-4, case
    assert g.native_epilogue_ok
    got = chain_boundary_seeds(it.mixed_seeds(x), wl.upper, False)
    tol = 2e-3 if rec["method"] == "cg" else 1e-4
    assert rel_l2(got, rec["hypergrad"]) < tol, (case, rel_l2(got, rec["hypergrad"]))


def _hvp_against_autograd(wl, step):
    wl.lower._training_step = step
    loss, tape, params = trace(wl)
    g = lower_tape(tape)
    it = Interp(g, torch.float64)
    it.base_backward()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    assert rel_l2([p.a for p in g.params], in_grad) < 1e-10
    vec = [torch.randn_like(p) for p in params]
    want = torch.autograd.grad(in_grad, params, grad_outputs=vec, retain_graph=True)
    assert rel_l2(it.hvp(vec), want) < 1e-9
    return g


def test_no_grad_results_are_constants():
    """Values computed under torch.no_grad() are constants for autograd (hence for the reference); the lowering must
    not differentiate through them (only aten.detach used to be recognised)."""
    wl = to_double(W.mlp_reweight(device="cpu", batch=8, l2=0.0))

    def step(p, batch):
        x, y = batch
        out = p.module(x)
        with torch.no_grad():
            w = torch.sigmoid(out)
        return (w * torch.tanh(out)).mean()

    _hvp_against_autograd(wl, step)


def test_loss_that_is_one_element_of_a_larger_tensor():
    """``per_sample[0]``: only that element is seeded, not the whole root buffer."""
    wl = to_double(W.mlp_reweight(device="cpu", batch=8, l2=0.0))

    def step(p, batch):
        x, y = batch
        per_sample = torch.tanh(p.module(x)) ** 2
        return per_sample.view(-1)[3]

    _hvp_against_autograd(wl, step)


def test_side_computations_without_a_rule_do_not_abort():
    """loss.item(), an accuracy metric, an op without a rule on a dead branch: all fine in the reference, so fine
    here; the same unknown op raises once it feeds the loss."""
    wl = to_double(W.mlp_reweight(device="cpu", batch=8, l2=0.0))
    seen = {}

    def step(p, batch):
        x, y = batch
        out = p.module(x)
        loss = torch.nn.functional.cross_entropy(out, y)
        seen["loss"] = loss.item()                                   # aten._local_scalar_dense
        with torch.no_grad():
            seen["acc"] = (out.argmax(1) == y).float().mean()        # argmax / eq / mean under no_grad
        seen["dead"] = torch.cumsum(out, 1).sum()                    # no rule, requires grad, never reaches the loss
        return loss

    g = _hvp_against_autograd(wl, step)
    assert all(n.op != "poison" for n in g.nodes)


def test_native_prologue_batchnorm_is_opt_in_and_never_touches_cpu_tensors(monkeypatch):
    """The recorder substitutes aten.native_batch_norm only when asked to (BB200_PROLOGUE_BN_MIN) and only for CUDA
    inputs (betty_b200/trace.py): by default the lower forward is PyTorch's, bit for bit."""
    import torch

    from betty_b200 import trace as T

    assert T.native_bn_min_numel <= 0 or "BB200_PROLOGUE_BN_MIN" in __import__("os").environ
    net = torch.nn.Sequential(torch.nn.Conv2d(2, 4, 3, padding=1), torch.nn.BatchNorm2d(4))
    x = torch.randn(3, 2, 6, 6)
    want = net(x).sum()
    for thr in (0, 1):
        monkeypatch.setattr(T, "native_bn_min_numel", thr)
        before = T.native_bn_calls
        loss, tape = T.record_tape(lambda: net(x).sum(), list(net.parameters()))
        assert T.native_bn_calls == before                       # CPU input: left to PyTorch even when switched on
        assert any(op.name in T._BN_FWD_OPS or "batch_norm" in op.name for op in tape.ops)
        assert torch.equal(loss.detach(), want.detach())
