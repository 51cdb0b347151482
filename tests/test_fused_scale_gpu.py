"""The fused 4-conv kernels at the scale of the benchmark's headline line (mini-ImageNet N=800, 64 channels, bf16).

convblock.cu (data-input block), convblock2.cu (inner blocks) and conv_halo.cu run persistent or grid-stride grids,
and the partial sums they leave for the fixed-order reductions have one slot per CTA.  At the sizes of
tests/test_plan_gpu.py every warp handles one m-tile and every grid-stride loop runs a single round, so loop-carried
state, a ragged last m-tile landing in a later round and partial arrays with hundreds of slots are never exercised
there.  The cases below are sized from the grid caps in the code (not from occupancy), so that they reach a second
round whatever occupancy the driver reports:

    convblock.cu   tensor-core grids <= GRID_MAX = 4 x 132 CTAs x 8 warps, 16 windows per m-tile
                   SIMT grids        <= GRID_MAX CTAs, one tile of R pooled rows per CTA and round
    convblock2.cu  stream_grid       <= 8 x 132 blocks x 32 windows per round

Checks, per case:
  * every activation-sized value against the float64 interpreter of the same IR with a per-image relative L2 (a lost
    16-window tile moves its image by ~10 %; a global norm over the batch only sees ~1 %), next to the global one;
  * block 1 on its tensor-core route against its SIMT route (BB200_NO_CBMMA): with bf16 input images and a
    bf16-representable direction the two differ only in fp32 summation order, so the bar is tight;
  * the inner blocks fused (convblock2 + halo kernels) against unfused (conv_tma, norm.cu, pooling);
  * run-to-run bit identity of H.v and of the Neumann loop;
  * the benchmark's own N=800 configuration against autograd's bf16 double backward.
Each case prints its worst errors and its peak device memory."""
import gc

import pytest
import torch

from betty_b200 import _native as N
from betty_b200 import workloads as W
from betty_b200.arena import ArenaLayout, pack
from betty_b200.ir import lower_tape
from betty_b200.plan import PASS_BB, HvpPlan
from betty_b200.trace import record_tape
from oracle.plan_interp import Interp
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu

SM = 132
GRID_MAX = 4 * SM                 # convblock.cu: CTAs of the block-1 grids (both routes)
CB_WARPS, CB_MT = 8, 16           # convblock.cu: warps per CTA, windows per m-tile of the tensor-core kernels
STREAM_ROUND = 8 * SM * 32        # convblock2.cu stream_grid: windows per round
PEAK_MAX = 20 * 2 ** 30           # the GPUs are shared: every case stays well under this

# name: (factory kwargs, tolerance, fused inner blocks expected)
CASES = {
    # 97 x 42 x 42 = 171 108 windows -> 10 695 m-tiles (last one holds 4 windows); block 2: 42 777 windows
    "mini_bf16_n97": (dict(n=97, hidden=64, image="miniimagenet", precision="bf16"), 5e-2, 3),
    # the C = 1 instantiation: 347 x 14 x 14 = 68 012 windows -> 4 251 m-tiles > 4 224 (last one holds 12 windows)
    "omniglot_bf16_n347": (dict(n=347, hidden=64, precision="bf16"), 5e-2, 2),
    # block 1 with fp32 pooled arrays (SIMT cb_tf_kernel / cb_reduce_kernel, 2 037 tiles); inner blocks unfused
    "mini_fp32_n97": (dict(n=97, hidden=64, image="miniimagenet"), 5e-5, 0),
}
BF16_CASES = ("mini_bf16_n97", "omniglot_bf16_n347")


def _fresh():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def _peak(what):
    peak = torch.cuda.max_memory_allocated()
    print(f"[fused scale] {what}: peak device memory {peak / 2 ** 30:.2f} GiB")
    assert peak < PEAK_MAX, f"{what}: {peak / 2 ** 30:.2f} GiB"


def _workload(case, bf16_inputs=False):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    wl = W.FACTORIES["implicit_maml"](device="cuda", **CASES[case][0])
    vec = list(wl.vector)
    if bf16_inputs:
        # bf16 images and direction: the tensor-core route's bf16 patch / weight-tangent fragments are then exact
        x = wl.lower.cur_batch[0]
        x.copy_(x.bfloat16().float())
        vec = [v.bfloat16().float() for v in vec]
    return wl, vec


def _record(wl):
    params = wl.lower.trainable_parameters()
    loss, tape = record_tape(lambda: wl.lower.training_step_exec(wl.lower.cur_batch), params)
    return params, loss, tape


def _plan(tape, params):
    lay = ArenaLayout.like(params)
    d, hv = lay.new(params[0].device), lay.new(params[0].device)
    return lay, d, hv, HvpPlan(tape, params, lay, d, hv, cuda_graph=False)


def _hvp(plan, lay, d, hv, vec):
    pack(lay, vec, d)
    plan()
    torch.cuda.synchronize()
    return hv.clone()


def _check_nodes(plan, case):
    ops = [n.op for n in plan.g.nodes]
    n_inner = CASES[case][2]
    assert ops.count("convblock") == 1, f"{case}: data-input block not fused: {ops}"
    assert ops.count("convblock2") == n_inner, f"{case}: expected {n_inner} fused inner blocks: {ops}"
    if n_inner == 0:
        assert ops.count("conv2d") == 3 and ops.count("batchnorm") == 3, f"{case}: {ops}"


def _check_rounds(plan, case):
    """The sizes reach the loops' second round: computed from the plan's own shapes and the grid caps."""
    cb = next(n for n in plan.g.nodes if n.op == "convblock")
    n, _, hp, wp = cb.out.base.shape
    nwin = n * hp * wp
    if CASES[case][0].get("precision") == "bf16":
        nmt = -(-nwin // CB_MT)
        assert nmt > CB_WARPS * GRID_MAX and nwin % CB_MT, (case, nwin, nmt)
    else:
        r = min(max(96 // wp, 1), hp)
        assert n * -(-hp // r) > GRID_MAX, (case, n, hp, wp)
    cb2 = [nd for nd in plan.g.nodes if nd.op == "convblock2"]
    if cb2 and CASES[case][0].get("image") == "miniimagenet":     # omniglot's block 2 (17 003 windows) fits one round
        n2, _, hp2, wp2 = cb2[0].out.base.shape
        assert n2 * hp2 * wp2 > STREAM_ROUND, (case, n2, hp2, wp2)


def _dense(vn, kind):
    a = getattr(vn, kind)
    if getattr(vn, "tfmt", None) == "nhwc_bf16":
        a = a[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2).float()     # bf16 padded-NHWC TMA operand of the next fused block
    return a


def _where(plan, vn):
    prod = [n for n in plan.g.nodes if n.out is vn]
    cons = [n.op for n in plan.g.nodes if any(x is not None and x.root is vn for x in n.ins)]
    return f"producer={prod[0].op if prod else None} consumers={cons}"


def _compare(plan, interp, kinds, tol, what):
    bad = []
    for vn, vi in zip(plan.g.values, interp.g.values):
        if vn.parent is not None or not vn.needed or vn.param_index is not None:
            continue
        for k in kinds:
            a, b = _dense(vn, k), getattr(vi, k)
            err = float((a.double() - b).norm() / (b.norm() + 1e-30)) if float(b.norm()) > 0 else float(a.double().norm())
            if not (err <= tol):
                bad.append(f"{what}: value #{vn.vid} {tuple(vn.base.shape)} kind={k} rel={err:.3e} {_where(plan, vn)}")
    assert not bad, "\n".join(bad[:12])


def _per_image(a, b, n):
    """Relative L2 of each image (leading dim); an image whose reference is 0 counts its absolute norm."""
    a, b = a.double().reshape(n, -1), b.double().reshape(n, -1)
    bn, dn = b.norm(dim=1), (a - b).norm(dim=1)
    return torch.where(bn > 0, dn / bn.clamp_min(1e-300), dn)


def _compare_per_image(plan, interp, kinds, tol, what, n):
    """Per-image relative L2 of every feature-map value (N, C, H, W).  Returns the worst (error, description)."""
    bad, worst = [], (0.0, "")
    for vn, vi in zip(plan.g.values, interp.g.values):
        if vn.parent is not None or not vn.needed or vn.param_index is not None:
            continue
        if vn.base.dim() != 4 or vn.base.shape[0] != n:
            continue
        for k in kinds:
            err = _per_image(_dense(vn, k), getattr(vi, k), n)
            e, i = (float(x) for x in err.max(0))
            desc = f"{what}: value #{vn.vid} {tuple(vn.base.shape)} kind={k} worst image {int(i)} rel={e:.3e} {_where(plan, vn)}"
            if e > worst[0]:
                worst = (e, desc)
            if not (e <= tol):
                bad.append(desc)
    assert not bad, "\n".join(bad[:12])
    return worst


def _param_index(v):
    while v is not None and v.parent is not None and v.ident:
        v = v.parent
    return None if v is None else v.param_index


def _owner(plan, i):
    """The node that reads parameter i (the fused block it belongs to), for failure messages."""
    for k, nd in enumerate(plan.g.nodes):
        if nd.op != "diagshift" and any(_param_index(v) == i for v in nd.ins if v is not None):
            return f"{nd.op} (node {k})"
    return "no node"


def _check_params(plan, got, want, tol, what):
    """Per-tensor relative L2 of H.v, each parameter named by its block (``plan``: a plan, or the list of names).
    Returns the worst one."""
    owners = plan if isinstance(plan, list) else [_owner(plan, i) for i in range(len(got))]
    bad, worst = [], 0.0
    for i, (g_, w_) in enumerate(zip(got, want)):
        if float(w_.norm()) > 0:
            e = rel_l2([g_], [w_])
            worst = max(worst, e)
            if not (e < tol):
                bad.append(f"{what}: H.v parameter {i} {tuple(g_.shape)} of {owners[i]}: rel={e:.3e}")
    e = rel_l2(got, want)
    assert not bad, "\n".join(bad + [f"{what}: whole H.v rel={e:.3e}"])
    return worst


# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(CASES))
def test_fused_blocks_match_interpreter_per_image(case):
    _fresh()
    tol = CASES[case][1]
    reduced = tol >= 1e-2
    wl, vec = _workload(case)
    params, loss, tape = _record(wl)
    lay, d, hv, plan = _plan(tape, params)
    _check_nodes(plan, case)
    _check_rounds(plan, case)
    n = CASES[case][0]["n"]
    interp = Interp(lower_tape(tape), torch.float64)
    interp.base_backward()
    _compare(plan, interp, ["a"], tol, "base-backward")
    got = lay.views(_hvp(plan, lay, d, hv, vec))
    want = interp.hvp(vec)
    _compare(plan, interp, ["t"], tol, "tangent-forward")
    _compare(plan, interp, ["at"], tol * 5, "tangent-backward")
    wt = _compare_per_image(plan, interp, ["t"], tol, "tangent-forward", n)
    wat = _compare_per_image(plan, interp, ["at"], tol * 5, "tangent-backward", n)
    print(f"[fused scale] {case}: worst per-image t {wt[0]:.3e} ({wt[1]})")
    print(f"[fused scale] {case}: worst per-image at {wat[0]:.3e} ({wat[1]})")
    per_tensor = _check_params(plan, got, want, 1.5e-1 if reduced else max(3e-4, tol * 20), f"{case} vs fp64 interpreter")
    e = rel_l2(got, want)
    print(f"[fused scale] {case}: H.v vs fp64 interpreter {e:.3e}, worst tensor {per_tensor:.3e}")
    assert e < tol * 5, f"{case}: H.v vs fp64 interpreter {e:.3e}"
    _peak(case)


def _block1(plan):
    return next(n for n in plan.g.nodes if n.op == "convblock")


def _block1_slices(plan, lay, hv):
    views = lay.views(hv)
    ins = zip(("W", "b", "gamma", "beta"), _block1(plan).ins)
    return {f"at_{nm}": views[_param_index(v)].clone() for nm, v in ins if _param_index(v) is not None}


def _bf16_ulps(a, b):
    """Distance of two bf16 tensors in units in the last place, elementwise (ordered bit patterns; -0 == +0)."""
    def ordered(x):
        u = x.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
        return torch.where(u < 0x8000, u, 0x8000 - u)
    return (ordered(a) - ordered(b)).abs()


@pytest.mark.parametrize("case", BF16_CASES)
def test_block1_tensor_core_route_matches_simt_route(case, monkeypatch):
    """Block 1 on mma.sync (cb_tf_mma_kernel / cb_reduce_mma_kernel) against cb_tf_kernel / cb_reduce_kernel.  Both
    keep bf16 pooled arrays and write the same bf16 NHWC tangent; with bf16 images and direction they differ only in
    fp32 summation order.

    * tangent forward: the pooled tangent of block 1 from identical inputs, element by element.
    * tangent backward: with the direction zero on block 1's parameters its pooled tangent is exactly 0 on both
      routes, so blocks 2-4 hand both routes the same bits of at_q, and at_W / at_b / at_gamma / at_beta isolate the
      reduce kernels.  (With a nonzero block-1 direction the last-bit differences of t_q flip bf16 roundings in
      blocks 2-4 and the comparison measures those, not block 1.)"""
    _fresh()
    wl, vec = _workload(case, bf16_inputs=True)
    params, loss, tape = _record(wl)
    out = {}
    for route in ("mma", "simt"):
        if route == "simt":
            monkeypatch.setenv("BB200_NO_CBMMA", "1")
        lay, d, hv, plan = _plan(tape, params)
        _check_nodes(plan, case)
        _hvp(plan, lay, d, hv, vec)
        tq = _block1(plan).out.t.clone()
        own = {_param_index(v) for v in _block1(plan).ins if _param_index(v) is not None}
        vec0 = [torch.zeros_like(v) if i in own else v for i, v in enumerate(vec)]
        _hvp(plan, lay, d, hv, vec0)
        assert not _block1(plan).out.t.any()
        out[route] = (tq, _block1_slices(plan, lay, hv), N.lib().bb_plan_launch_count(plan.handle, PASS_BB))
        del plan, d, hv
    monkeypatch.delenv("BB200_NO_CBMMA")
    (tq_m, at_m, nb_m), (tq_s, at_s, nb_s) = out["mma"], out["simt"]
    # the tensor-core base pass adds one launch (patch fragments + the mma reduce, against the SIMT reduce)
    assert nb_m == nb_s + 1, f"{case}: BB200_NO_CBMMA did not switch the block-1 route ({nb_m} vs {nb_s} launches)"
    n = CASES[case][0]["n"]
    ulps = _bf16_ulps(tq_m, tq_s)
    # where |t_q| is far below its RMS the value is a cancellation of fp32 terms: there, count ulps of the RMS instead
    ref = tq_s.float()
    big = ref.abs() >= ref.pow(2).mean().sqrt() / 16
    ulp_big = int(ulps[big].max())
    img = float(_per_image(tq_m[:, 1:-1, 1:-1, :].float(), ref[:, 1:-1, 1:-1, :], n).max())
    frac = float((ulps > 0).double().mean())
    errs = {k: rel_l2([at_m[k]], [at_s[k]]) for k in at_m}
    # at_b is 0 in exact arithmetic (the batch norm removes the conv bias), so both routes return rounding residue:
    # reported, not compared
    at_b = errs.pop("at_b", None)
    print(f"[fused scale] {case}: block 1 tensor-core vs SIMT: t_q max {ulp_big} bf16 ulp where |t_q| >= rms/16 "
          f"(max {int(ulps.max())} anywhere, {frac:.2e} of elements differ), worst image {img:.3e}; "
          + ", ".join(f"{k} {v:.3e}" for k, v in errs.items()) + f" (at_b residue {at_b:.1e})")
    assert ulp_big <= 1, f"{case}: block 1 (convblock) pooled tangent differs by {ulp_big} bf16 ulp between routes"
    assert img <= 2 ** -8, f"{case}: block 1 (convblock) pooled tangent: worst image {img:.3e} between routes"
    for k, v in errs.items():
        assert v <= 1e-4, f"{case}: block 1 (convblock) {k} differs by {v:.3e} between the tensor-core and SIMT routes"
    _peak(f"{case} routes")


def test_inner_blocks_fused_match_unfused(monkeypatch):
    """convblock2 + halo kernels against the unfused chain (conv_tma, norm.cu, pooling) of the same tape.  The chains
    round to bf16 at different points, so the bar is the bf16 one."""
    _fresh()
    case = "mini_bf16_n97"
    tol = CASES[case][1]
    n = CASES[case][0]["n"]
    wl, vec = _workload(case)
    params, loss, tape = _record(wl)
    res = {}
    for fused in (True, False):
        if not fused:
            monkeypatch.setenv("BB200_NO_CONVBLOCK2", "1")
        lay, d, hv, plan = _plan(tape, params)
        ops = [nd.op for nd in plan.g.nodes]
        assert ops.count("convblock2") == (3 if fused else 0), ops
        got = lay.views(_hvp(plan, lay, d, hv, vec))
        pooled = {nd.out.base.data_ptr(): _dense(nd.out, "t").float().clone()
                  for nd in plan.g.nodes if nd.op in ("convblock2", "maxpool2d")}
        res[fused] = ([g_.clone() for g_ in got], pooled)
        if fused:
            res["plan"] = plan          # names the fused block of a failing parameter
        del plan, d, hv
    monkeypatch.delenv("BB200_NO_CONVBLOCK2")
    (hv_f, tq_f), (hv_u, tq_u) = res[True], res[False]
    assert len(tq_f) == 3 and set(tq_f) == set(tq_u), (len(tq_f), len(tq_u))
    worst = 0.0
    for i, key in enumerate(sorted(tq_f)):
        e = float(_per_image(tq_f[key], tq_u[key], n).max())
        worst = max(worst, e)
        assert e <= tol, f"inner block pooled tangent {tuple(tq_f[key].shape)}: worst image {e:.3e} fused vs unfused"
    per_tensor = _check_params(res["plan"], hv_f, hv_u, 1.5e-1, "fused vs unfused inner blocks")
    e = rel_l2(hv_f, hv_u)
    print(f"[fused scale] inner blocks fused vs unfused: pooled tangents worst image {worst:.3e}; "
          f"H.v {e:.3e}, worst tensor {per_tensor:.3e}")
    assert e < 2e-2, f"H.v fused vs unfused inner blocks {e:.3e}"
    _peak("fused vs unfused")


@pytest.mark.parametrize("case", ("mini_bf16_n97", "mini_fp32_n97"))
def test_run_to_run_bit_identity(case):
    """Fixed-order reductions: the same plan twice, two plans of one tape, and the Neumann loop return the same bits."""
    _fresh()
    wl, vec = _workload(case)
    params, loss, tape = _record(wl)
    lay, d, hv, plan = _plan(tape, params)
    a = _hvp(plan, lay, d, hv, vec)
    b = _hvp(plan, lay, d, hv, vec)
    assert torch.equal(a, b), f"{case}: two runs of one plan differ (max {float((a - b).abs().max()):.3e})"
    lay2, d2, hv2, plan2 = _plan(tape, params)
    c = _hvp(plan2, lay2, d2, hv2, vec)
    assert torch.equal(a, c), f"{case}: two plans of one tape differ (max {float((a - c).abs().max()):.3e})"
    del plan2, d2, hv2
    loops = []
    for _ in range(2):
        pack(lay, vec, d)
        acc = d.clone()
        plan.neumann_loop(5, 0.01, d, acc, hv)
        torch.cuda.synchronize()
        loops.append((acc.clone(), d.clone()))
    assert torch.equal(loops[0][0], loops[1][0]) and torch.equal(loops[0][1], loops[1][1]), f"{case}: Neumann K=5 differs"
    print(f"[fused scale] {case}: H.v and Neumann K=5 bit-identical across runs and plans")
    _peak(f"{case} identity")


def test_benchmark_configuration_matches_autograd():
    """bench.py's headline workload exactly (mini-ImageNet N=800, bf16): one H.v against autograd's bf16 double
    backward.  (No float64 interpreter here: its activations alone would not fit the memory budget.)"""
    from bench import WORKLOADS

    _fresh()
    fac, kw, _ = WORKLOADS["implicit_maml"]
    assert fac == "implicit_maml" and kw["n"] == 800
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    wl = W.FACTORIES[fac](device="cuda", **kw)
    params, loss, tape = _record(wl)
    lay, d, hv, plan = _plan(tape, params)
    ops = [nd.op for nd in plan.g.nodes]
    assert ops.count("convblock") == 1 and ops.count("convblock2") == 3, ops
    vec = list(wl.vector)
    got = lay.views(_hvp(plan, lay, d, hv, vec))
    owners = [_owner(plan, i) for i in range(len(params))]
    del plan, d, hv                  # the plan's buffers are not needed by autograd's double backward: lower the peak
    gc.collect()
    in_grad = torch.autograd.grad(loss, params, create_graph=True)
    want = torch.autograd.grad(in_grad, params, grad_outputs=vec)
    e = rel_l2(got, want)
    per_tensor = _check_params(owners, got, want, 1.5e-1, "N=800 vs autograd")
    print(f"[fused scale] bench implicit_maml N=800: H.v vs autograd bf16 double backward {e:.3e}, "
          f"worst tensor {per_tensor:.3e}")
    assert e < 2e-2, f"N=800: H.v vs autograd double backward {e:.3e}"
    _peak("bench implicit_maml N=800")
