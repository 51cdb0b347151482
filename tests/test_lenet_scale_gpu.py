"""The LeNet line of the benchmark (learning_to_reweight: LeNet-5, B=4096, CG K=20, fp32) at its own size.

Its hot path is the small-channel convolutions (conv_small2.cu, conv_small.cu) and the SIMT GEMM (gemm.cu).  At
B=4096 the correlation kernel runs 256...1 024 units over 132 blocks, the weight gradients walk 6...8 images per block
and the Linear layers take the 64x64 tile kernel with ragged N (120, 84); at the B=300 of tests/test_plan_gpu.py none
of that runs.  Checks:
  * every tangent, adjoint and adjoint tangent against the float64 interpreter of the same IR, per sample (leading
    dimension N: conv / pool maps and Linear activations), with the global number next to it;
  * H.v per named parameter against the interpreter and against autograd's fp32 double backward;
  * H.v bit-identical from run to run and across plans;
  * the benchmark's own call (HypergradientCall(...).solve, CUDA graph on, what bench.py --dump-outputs writes):
    bit-identical over two calls and two plans, and within 1e-4 of a float64 CG of the same system.
Each check prints its measured values and the peak device memory."""
import gc

import pytest
import torch

from betty_b200 import engine as E
from betty_b200 import workloads as W
from betty_b200.ir import lower_tape
from oracle import ref_port
from oracle.plan_interp import Interp
from tests.helpers import rel_l2, to_double
from tests.test_conv_small_scale_gpu import CORR2, WGRAD2, WGRAD_V1, geometry
from tests.test_fused_scale_gpu import _dense, _hvp, _plan, _record, _where

pytestmark = pytest.mark.gpu

BATCH, K = 4096, 20                # bench.py WORKLOADS["learning_to_reweight"]
PEAK_MAX = 20 * 2 ** 30            # the GPUs are shared: stay well under this
FP32_BAR = 1e-4                    # the project's fp32 protocol for H.v and hypergradients
# per-sample bars, from the worst measured on an H100 SXM 80 GB (700 W): a 3.1e-7, t 1.3e-6, at 1.3e-6
PER_SAMPLE_BAR = {"a": 2e-6, "t": 1e-5, "at": 1e-5}


def _flat(xs):
    return torch.cat([x.reshape(-1) for x in xs])


def _fresh():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def _peak(what):
    peak = torch.cuda.max_memory_allocated()
    print(f"[lenet scale] {what}: peak device memory {peak / 2 ** 30:.2f} GiB")
    assert peak < PEAK_MAX, f"{what}: {peak / 2 ** 30:.2f} GiB"


def _workload():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return W.lenet_reweight(device="cuda", batch=BATCH, method="cg", K=K)


def _names(wl):
    return [nm for nm, _ in wl.lower.module.named_parameters()]


def _check_conv_routes(plan):
    """Both convolutions run on the small-channel kernels at this size (the launchers' own planning code)."""
    convs = [nd for nd in plan.g.nodes if nd.op == "conv2d"]
    assert len(convs) == 2, [nd.op for nd in plan.g.nodes]
    seen = []
    for i, nd in enumerate(convs):
        n, c, h, w = nd.attrs["X"].shape
        o, _, kh, kw = nd.attrs["W"].shape
        (ph, pw) = nd.attrs["padding"]
        act_x = i > 0                  # conv1 reads the data batch: only its weight tangent is active
        np_ = 2 if act_x else 1
        tf = geometry(0, n, c, h, w, o, kh, kw, ph, pw, np_)
        wg = geometry(2, n, c, h, w, o, kh, kw, ph, pw, np_)
        assert tf["route"] == CORR2 and tf["units"] > tf["grid"], f"conv{i + 1} tangent forward: {tf}"
        assert wg["route"] == (WGRAD2 if act_x else WGRAD_V1) and wg["units"] > 1, f"conv{i + 1} weight gradient: {wg}"
        assert wg["grid"] * wg["part_floats"] * 4 <= 24 << 20, f"conv{i + 1}: partials exceed the plan workspace {wg}"
        desc = f"conv{i + 1}: tf {tf['units']} units / {tf['grid']} blocks, wgrad route {wg['route']} {wg['grid']} blocks"
        if act_x:
            dg = geometry(1, n, c, h, w, o, kh, kw, ph, pw, 2)
            assert dg["route"] == CORR2 and dg["CIC"] < o, f"conv{i + 1} data gradient: {dg}"
            desc += f", dgrad {dg['units']} units (CIC {dg['CIC']} of {o})"
        seen.append(desc)
    print("[lenet scale] " + "; ".join(seen))


def _per_sample(a, b, n):
    """Error norm of each sample (leading dim) over the larger of its reference norm and the RMS of all samples'
    reference norms.  A value with one element per sample (the weighted per-sample losses) can cancel to far below
    its typical size, where its own relative error says nothing; a dropped or stale sample still counts ~1."""
    a, b = a.double().reshape(n, -1), b.double().reshape(n, -1)
    bn, dn = b.norm(dim=1), (a - b).norm(dim=1)
    return dn / torch.maximum(bn, bn.pow(2).mean().sqrt()).clamp_min(1e-300)


def _compare_per_sample(plan, interp, kind, tol, what, n):
    """Per-sample error (_per_sample) of every value with leading dimension N (4-D maps and 2-D Linear activations),
    and the global relative L2 of each.  Returns the worst per-sample and worst global values."""
    bad, worst, worst_g = [], (0.0, ""), 0.0
    for vn, vi in zip(plan.g.values, interp.g.values):
        if vn.parent is not None or not vn.needed or vn.param_index is not None:
            continue
        if vn.base.dim() not in (2, 4) or vn.base.shape[0] != n:
            continue
        a, b = _dense(vn, kind), getattr(vi, kind)
        if float(b.norm()) == 0 and float(a.norm()) == 0:
            continue
        err = _per_sample(a, b, n)
        e, i = (float(x) for x in err.max(0))
        g = float((a.double() - b).norm() / b.norm().clamp_min(1e-300))
        worst_g = max(worst_g, g)
        desc = (f"{what}: value #{vn.vid} {tuple(vn.base.shape)} kind={kind} worst sample {int(i)} rel={e:.3e} "
                f"(global {g:.3e}) {_where(plan, vn)}")
        if e > worst[0]:
            worst = (e, desc)
        if not (e <= tol):
            bad.append(desc)
    assert not bad, "\n".join(bad[:12])
    return worst, worst_g


def _check_named(names, got, want, tol, what):
    bad, worst = [], (0.0, "")
    for nm, g_, w_ in zip(names, got, want):
        e = rel_l2([g_], [w_])
        if e > worst[0]:
            worst = (e, nm)
        if not (e <= tol):
            bad.append(f"{what}: H.v {nm} {tuple(g_.shape)} rel={e:.3e}")
    assert not bad, "\n".join(bad)
    return worst


def test_lenet_b4096_against_fp64_interpreter_and_autograd():
    _fresh()
    wl = _workload()
    names = _names(wl)
    vec = list(wl.vector)
    params, loss, tape = _record(wl)
    lay, d, hv, plan = _plan(tape, params)
    _check_conv_routes(plan)
    interp = Interp(lower_tape(tape), torch.float64)
    interp.base_backward()
    worst = {}
    worst["a"] = _compare_per_sample(plan, interp, "a", PER_SAMPLE_BAR["a"], "base-backward", BATCH)
    got = lay.views(_hvp(plan, lay, d, hv, vec))
    want = interp.hvp(vec)
    worst["t"] = _compare_per_sample(plan, interp, "t", PER_SAMPLE_BAR["t"], "tangent-forward", BATCH)
    worst["at"] = _compare_per_sample(plan, interp, "at", PER_SAMPLE_BAR["at"], "tangent-backward", BATCH)
    for k, ((e, desc), g) in worst.items():
        print(f"[lenet scale] per-sample {k}: worst {e:.3e}, worst global {g:.3e} ({desc})")
    got = [g_.clone() for g_ in got]
    t_int = _check_named(names, got, want, FP32_BAR, "vs fp64 interpreter")
    e_int = rel_l2(got, want)
    del interp, want
    gc.collect()
    # bit identity: one plan twice, and a second plan of the same tape
    first = _flat(got)
    again = _flat(lay.views(_hvp(plan, lay, d, hv, vec)))
    assert torch.equal(again, first), f"two runs of one plan differ (max {float((again - first).abs().max()):.3e})"
    lay2, d2, hv2, plan2 = _plan(tape, params)
    other = _flat(lay2.views(_hvp(plan2, lay2, d2, hv2, vec)))
    assert torch.equal(other, first), f"two plans of one tape differ (max {float((other - first).abs().max()):.3e})"
    del plan, plan2, d, d2, hv, hv2
    gc.collect()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    ag = torch.autograd.grad(in_grad, params, grad_outputs=vec)
    t_ag = _check_named(names, got, ag, FP32_BAR, "vs autograd fp32 double backward")
    e_ag = rel_l2(got, ag)
    print(f"[lenet scale] H.v vs fp64 interpreter {e_int:.3e} (worst tensor {t_int[1]} {t_int[0]:.3e}); "
          f"vs autograd fp32 {e_ag:.3e} (worst tensor {t_ag[1]} {t_ag[0]:.3e}); bit-identical across runs and plans")
    assert e_int <= FP32_BAR and e_ag <= FP32_BAR
    _peak("H.v per sample")


def _solve_bench_call(wl):
    call = E.HypergradientCall(wl.lower, "cg")
    try:
        return [x.clone() for x in call.solve(wl.vector)]
    finally:
        call.release()


def test_benchmark_cg_call_reproducible_and_against_fp64_cg():
    """The benchmark's K-loop call exactly as bench.py times it (plan cache and CUDA graph as configured by default)."""
    _fresh()
    wl = _workload()
    a = _solve_bench_call(wl)
    b = _solve_bench_call(wl)            # second call: the cached plan, its captured graph replayed
    E.plan_cache.clear()
    c = _solve_bench_call(wl)            # a new plan
    fa, fb, fc = _flat(a), _flat(b), _flat(c)
    assert torch.equal(fa, fb), f"two calls differ (max {float((fa - fb).abs().max()):.3e})"
    assert torch.equal(fa, fc), f"two plans differ (max {float((fa - fc).abs().max()):.3e})"
    names = _names(wl)
    _peak("bench call")
    del wl
    E.plan_cache.clear()
    _fresh()
    w64 = to_double(_workload())
    in_grad = ref_port.lower_gradient(w64.lower)
    x64 = ref_port.cg_solve(list(w64.vector), ref_port.make_hvp(in_grad, w64.lower.parameters()), K,
                            float(w64.lower.config.cg_alpha))
    e = rel_l2(a, x64)
    worst = max((rel_l2([g_], [w_]), nm) for nm, g_, w_ in zip(names, a, x64))
    print(f"[lenet scale] bench CG K={K} B={BATCH}: bit-identical over two calls and two plans; vs fp64 CG {e:.3e} "
          f"(worst tensor {worst[1]} {worst[0]:.3e})")
    assert e <= FP32_BAR, f"CG K={K} hypergradient vs fp64 CG {e:.3e}"
    _peak("fp64 CG")
