"""The small-channel convolution kernels (csrc/conv_small2.cu, csrc/conv_small.cu) at the scale of the LeNet line of
the benchmark (B=4096), against float64.

Every kernel here is persistent or walks images in a per-block loop: conv_small_corr2_kernel runs units of (image
group, row band) over at most 132 blocks and prefetches the next unit's images while it computes, and the weight
gradients walk images over 528 (first generation) or 792 (wgrad2) blocks.  At the batch sizes of
tests/test_plan_gpu.py each block gets one unit or one image, so none of those loops takes a second round there.  Each
case below asks the launchers' own planning code (bb_conv_small_geometry) which route and geometry it gets and asserts
that the case reaches what it is named for: more units than blocks with a ragged last round, several images per
weight-gradient block, a channel chunk smaller than the channel count, and so on.

One-node fp32 plans are built by hand (kind 0, stride 1) and run through PASS_BB, PASS_TF and PASS_TB.  Checks:
  * correlation outputs (t_y, a_x, at_x), element by element:
        |got - ref| <= c (K + 2) 2^-23 (sum |in| |w| + |bias| + |C0|),   K = npairs CI KH KW;
  * weight gradients (a_W, at_W) and bias sums: rel-L2 and max|err| / max|ref| per tensor (K = N HO WO npairs, up to
    8e5 terms, so the a-priori bound says nothing);
  * the first-generation correlation and every corr2 variant (PX 4/5/7, 4-byte staging) sum each element in the same
    order with the same fmaf chain, so they must agree bit for bit;
  * the weight gradient is fixed-order (per-block partials added in block order): two runs return the same bits.
Outputs that are written are filled with NaN first; outputs accumulated into (beta = 1) hold known values."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from betty_b200 import _native as N
from betty_b200.plan import NODE_DTYPE, OPS, PASS_BB, PASS_TB, PASS_TF

pytestmark = pytest.mark.gpu

SM = 132
GEO_KEYS = ("route", "grid", "units", "PX", "IMGS", "RY", "bands", "CIC", "nstages", "VW", "groups", "OB", "tasks",
            "ns", "part_floats")
CORR2, CORR_V1, WGRAD2, WGRAD_V1, GENERIC = 1, 2, 3, 4, 0

# Bars, set from the worst values measured on an H100 SXM 80 GB (700 W) over every case below (DESIGN.md §4)
CORR_C = 1 / 4          # correlation outputs: worst measured ratio at c = 1 is 4.6e-2 (three_bands_40, t_y)
WGRAD_REL = 8e-6        # weight gradients and bias sums, rel-L2 and max|err| / max|ref|: worst measured 1.8e-6

# name: (N, C, H, W, O, KH, KW, ph, pw, input tangent active, expectations on the geometry)
CASES = {
    # the benchmark's own nodes: conv1 (data input: weight tangent only), conv1 with an input tangent, conv2
    "lenet_conv1": (4096, 3, 32, 32, 6, 5, 5, 0, 0, False, dict(PX=7, IMGS=8, bands=2, VW=4, wgrad=WGRAD_V1)),
    "lenet_conv1_ragged": (4099, 3, 32, 32, 6, 5, 5, 0, 0, False, dict(PX=7, IMGS=8, bands=2, wgrad=WGRAD_V1)),
    "lenet_conv1_tx": (4096, 3, 32, 32, 6, 5, 5, 0, 0, True, dict(PX=7, nstages=2, wgrad=WGRAD_V1)),
    "lenet_conv1_tx_ragged": (4099, 3, 32, 32, 6, 5, 5, 0, 0, True, dict(PX=7, nstages=2, wgrad=WGRAD_V1)),
    "lenet_conv2": (4096, 6, 14, 14, 16, 5, 5, 0, 0, True, dict(PX=5, IMGS=16, wgrad=WGRAD2)),
    "lenet_conv2_ragged": (4099, 6, 14, 14, 16, 5, 5, 0, 0, True, dict(PX=5, IMGS=16, wgrad=WGRAD2)),
    # geometry edges
    "pad2_5x5": (301, 3, 32, 32, 6, 5, 5, 2, 2, True, dict(VW=2, bands=2, RY=16)),
    "k3_pad1_16to16": (1100, 16, 20, 20, 16, 3, 3, 1, 1, True, dict(PX=5)),
    "odd_w": (1401, 3, 15, 15, 6, 3, 3, 1, 1, True, dict(VW=1)),
    "co12": (1401, 4, 12, 12, 12, 3, 3, 1, 1, True, dict()),
    "co8": (2201, 4, 12, 12, 8, 3, 3, 0, 0, True, dict()),
    "co2_wgrad2_ob2": (1401, 16, 12, 12, 2, 5, 5, 2, 2, True, dict(wgrad=WGRAD2, OB=2)),
    "k3x5_ph1_pw0": (2201, 6, 14, 18, 8, 3, 5, 1, 0, True, dict()),
    "three_bands_40": (301, 3, 40, 40, 6, 3, 3, 1, 1, True, dict(bands=3)),
    "ragged_channel_chunk": (100, 13, 64, 64, 6, 5, 5, 2, 2, True, dict(CIC=9)),
    "n_below_imgs": (3, 3, 32, 32, 6, 5, 5, 0, 0, True, dict(IMGS=3, small=True)),
}
BENCH_NODES = ("lenet_conv1", "lenet_conv1_tx", "lenet_conv2")


def geometry(which, n, c, h, w, o, kh, kw, ph, pw, npairs):
    """bb_conv_small_geometry: which 0 tangent forward, 1 data gradient, 2 weight gradient."""
    out = np.zeros(15, dtype=np.int64)
    N.call("bb_conv_small_geometry", which, n, c, h, w, o, kh, kw, ph, pw, npairs, out.ctypes.data, 15)
    return dict(zip(GEO_KEYS, (int(v) for v in out)))


def _geometries(case):
    n, c, h, w, o, kh, kw, ph, pw, act_x, _ = CASES[case]
    np_tf = 2 if act_x else 1
    return {"tf": geometry(0, n, c, h, w, o, kh, kw, ph, pw, np_tf),
            "dgrad": geometry(1, n, c, h, w, o, kh, kw, ph, pw, 2) if act_x else None,
            "wgrad": geometry(2, n, c, h, w, o, kh, kw, ph, pw, np_tf)}


def _check_geometry(case, geo):
    exp = dict(CASES[case][10])
    tf = geo["tf"]
    assert tf["route"] == CORR2, f"{case}: tangent forward not on corr2: {tf}"
    if exp.pop("small", False):
        assert tf["units"] <= tf["grid"], (case, tf)
    else:
        assert tf["units"] > tf["grid"] and tf["units"] % tf["grid"], f"{case}: no ragged second round: {tf}"
        assert tf["grid"] == SM, (case, tf)
    want_wgrad = exp.pop("wgrad", None)
    wg = geo["wgrad"]
    if want_wgrad is not None:
        assert wg["route"] == want_wgrad, f"{case}: weight gradient route {wg}"
    if want_wgrad is not None:
        assert wg["units"] > 1 and CASES[case][0] % wg["grid"], f"{case}: one image per weight-gradient block: {wg}"
    if "OB" in exp:
        assert wg["OB"] == exp.pop("OB"), (case, wg)
    for k, v in exp.items():
        assert tf[k] == v, f"{case}: {k} = {tf[k]}, expected {v}: {tf}"
    if case == "ragged_channel_chunk":
        assert tf["CIC"] < CASES[case][1] and CASES[case][1] % tf["CIC"], (case, tf)
    if geo["dgrad"] is not None:
        assert geo["dgrad"]["route"] == CORR2, f"{case}: data gradient not on corr2: {geo['dgrad']}"


def _inputs(case, seed=1234):
    n, c, h, w, o, kh, kw, ph, pw, act_x, _ = CASES[case]
    ho, wo = h + 2 * ph - kh + 1, w + 2 * pw - kw + 1
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g, device="cuda") * scale
    t = dict(x=r(n, c, h, w), W=r(o, c, kh, kw, scale=0.2), t_W=r(o, c, kh, kw, scale=0.2), t_b=r(o),
             a_y=r(n, o, ho, wo), at_y=r(n, o, ho, wo),
             a_x0=r(n, c, h, w), at_x0=r(n, c, h, w), a_W0=r(o, c, kh, kw), at_W0=r(o, c, kh, kw), a_b0=r(o), at_b0=r(o))
    if act_x:
        t["t_x"] = r(n, c, h, w)
    return t


def _offset_view(t):
    """The same values at base + 1 float (a 4-byte aligned, not 16-byte aligned view)."""
    buf = torch.empty(t.numel() + 1, device=t.device, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def run_node(case, inp, beta=1, misalign=False):
    """One fp32 conv2d node through PASS_BB, PASS_TF and PASS_TB.  Returns the outputs."""
    n, c, h, w, o, kh, kw, ph, pw, act_x, _ = CASES[case]
    ho, wo = h + 2 * ph - kh + 1, w + 2 * pw - kw + 1
    x, t_x = inp["x"], inp.get("t_x")
    if misalign:
        x = _offset_view(x)
        t_x = _offset_view(t_x) if t_x is not None else None
    nan = lambda *s: torch.full(s, float("nan"), device="cuda")
    out = {"t_y": nan(n, o, ho, wo)}
    for k in ("a_W", "at_W", "a_b", "at_b") + (("a_x", "at_x") if act_x else ()):
        out[k] = inp[k + "0"].clone() if beta else nan(*inp[k + "0"].shape)
    rec = np.zeros(1, dtype=NODE_DTYPE)
    r = rec[0]
    r["op"], r["kind"] = OPS["conv2d"], 0
    r["active"] = (1 if act_x else 0) | 2 | 4
    r["pad0"] = (1 if act_x else 0) | 2 | 4
    r["beta"][:] = (beta, beta, beta, 0)
    r["dims"][0:15] = (n, c, h, w, o, kh, kw, ho, wo, 1, 1, ph, pw, 1, 1)
    r["base"][0], r["dt"][0] = x.data_ptr(), 0
    r["base"][1], r["dt"][1] = inp["W"].data_ptr(), 0
    if act_x:
        r["t"][0], r["a"][0], r["at"][0] = t_x.data_ptr(), out["a_x"].data_ptr(), out["at_x"].data_ptr()
    r["t"][1], r["a"][1], r["at"][1] = inp["t_W"].data_ptr(), out["a_W"].data_ptr(), out["at_W"].data_ptr()
    r["t"][2], r["a"][2], r["at"][2] = inp["t_b"].data_ptr(), out["a_b"].data_ptr(), out["at_b"].data_ptr()
    r["t"][3], r["a"][3], r["at"][3] = out["t_y"].data_ptr(), inp["a_y"].data_ptr(), inp["at_y"].data_ptr()
    handle = C.c_void_p()
    N.call("bb_plan_create", rec.ctypes.data, 1, C.byref(handle))
    try:
        s = torch.cuda.current_stream().cuda_stream
        for pas in (PASS_BB, PASS_TF, PASS_TB):
            N.call("bb_plan_run", handle, pas, s)
        torch.cuda.synchronize()
    finally:
        N.lib().bb_plan_destroy(handle)
    return out


def reference(case, inp, beta=1):
    """float64 values of every output, with the magnitude sums of the correlation outputs for the elementwise bound."""
    n, c, h, w, o, kh, kw, ph, pw, act_x, _ = CASES[case]
    d = {k: v.double() for k, v in inp.items()}
    pad = (ph, pw)
    conv = lambda a, b, bias=None: F.conv2d(a, b, bias, padding=pad)
    dgrad = lambda g, wt: torch.nn.grad.conv2d_input(d["x"].shape, wt, g, padding=pad)
    wgrad = lambda a, g: torch.nn.grad.conv2d_weight(a, d["W"].shape, g, padding=pad)
    ref, mag = {}, {}
    ref["t_y"] = conv(d["x"], d["t_W"], d["t_b"])
    mag["t_y"] = conv(d["x"].abs(), d["t_W"].abs(), d["t_b"].abs())
    ref["a_W"] = wgrad(d["x"], d["a_y"])
    ref["at_W"] = wgrad(d["x"], d["at_y"])
    ref["a_b"] = d["a_y"].sum((0, 2, 3))
    ref["at_b"] = d["at_y"].sum((0, 2, 3))
    if act_x:
        ref["t_y"] = ref["t_y"] + conv(d["t_x"], d["W"])
        mag["t_y"] = mag["t_y"] + conv(d["t_x"].abs(), d["W"].abs())
        ref["at_W"] = ref["at_W"] + wgrad(d["t_x"], d["a_y"])
        ref["a_x"] = dgrad(d["a_y"], d["W"])
        mag["a_x"] = dgrad(d["a_y"].abs(), d["W"].abs())
        ref["at_x"] = dgrad(d["at_y"], d["W"]) + dgrad(d["a_y"], d["t_W"])
        mag["at_x"] = dgrad(d["at_y"].abs(), d["W"].abs()) + dgrad(d["a_y"].abs(), d["t_W"].abs())
    if beta:
        for k in ref:
            if k != "t_y":
                ref[k] = ref[k] + d[k + "0"]
                if k in mag:
                    mag[k] = mag[k] + d[k + "0"].abs()
    return ref, mag


def _k_terms(case, key):
    n, c, h, w, o, kh, kw, ph, pw, act_x, _ = CASES[case]
    npairs = 2 if act_x else 1
    return npairs * (c if key == "t_y" else o) * kh * kw


def check_against_fp64(case, got, ref, mag, what):
    """Elementwise bound on the correlation outputs, rel-L2 / max-ratio on the reductions.  Returns the worst values."""
    worst = {}
    for k, want in ref.items():
        a = got[k].double()
        assert torch.isfinite(a).all(), f"{what}: {k} has non-finite values (an element was not written)"
        err = (a - want).abs()
        if k in mag:
            ratio = float((err / ((_k_terms(case, k) + 2) * 2.0 ** -23 * mag[k]).clamp_min(1e-300)).max())
            worst[k] = ratio
            assert ratio <= CORR_C, f"{what}: {k} error {ratio:.3e} of the fp32 bound (bar {CORR_C})"
        else:
            rel = float(err.norm() / want.norm())
            mx = float(err.max() / want.abs().max())
            worst[k] = max(rel, mx)
            assert rel <= WGRAD_REL and mx <= WGRAD_REL, f"{what}: {k} rel-L2 {rel:.3e}, max ratio {mx:.3e} (bar {WGRAD_REL})"
    return worst


def _fmt(worst):
    return ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items()))


@pytest.mark.parametrize("case", sorted(CASES))
def test_small_conv_against_float64(case):
    geo = _geometries(case)
    _check_geometry(case, geo)
    inp = _inputs(case)
    got = run_node(case, inp)
    ref, mag = reference(case, inp)
    worst = check_against_fp64(case, got, ref, mag, case)
    tf, wg = geo["tf"], geo["wgrad"]
    print(f"[small conv] {case}: tf units {tf['units']} / grid {tf['grid']} (PX {tf['PX']}, IMGS {tf['IMGS']}, "
          f"bands {tf['bands']}, CIC {tf['CIC']}, stages {tf['nstages']}, VW {tf['VW']}); wgrad route {wg['route']} "
          f"grid {wg['grid']}, images/block {wg['units']}; worst: {_fmt(worst)}")


@pytest.mark.parametrize("case", BENCH_NODES)
def test_small_conv_written_outputs_beta0(case):
    """beta = 0: every output is written over NaN (the weight gradients through the memset + partial finish)."""
    inp = _inputs(case, seed=99)
    got = run_node(case, inp, beta=0)
    ref, mag = reference(case, inp, beta=0)
    worst = check_against_fp64(case, got, ref, mag, f"{case} beta=0")
    print(f"[small conv] {case} beta=0: worst: {_fmt(worst)}")


def _corr_keys(case):
    return ("t_y", "a_x", "at_x") if CASES[case][9] else ("t_y",)


ROUTE_CASES = ("lenet_conv1_tx_ragged", "lenet_conv2_ragged", "pad2_5x5", "odd_w", "co12", "k3x5_ph1_pw0",
               "three_bands_40", "ragged_channel_chunk")


@pytest.mark.parametrize("case", ROUTE_CASES)
def test_correlation_routes_bit_identical(case, monkeypatch):
    """corr2 under every PX it can take and with 4-byte staging, and the first-generation kernel, against the default
    corr2 launch: the same p -> ci -> i -> j fmaf chain per element, so the same bits.  The weight gradient on each
    route is held to the fp64 bar."""
    inp = _inputs(case)
    ref, mag = reference(case, inp)
    base = run_node(case, inp)
    g0 = _geometries(case)["tf"]
    variants = [("BB200_CORR2_VW1", "1"), ("BB200_CONV_SMALL_V1", "1")]
    for px in (4, 5, 7):
        monkeypatch.setenv("BB200_CORR2_PX", str(px))
        g = _geometries(case)["tf"]
        monkeypatch.delenv("BB200_CORR2_PX")
        if g["route"] == CORR2 and g["PX"] == px and px != g0["PX"]:
            variants.append(("BB200_CORR2_PX", str(px)))
    seen = []
    for var, val in variants:
        monkeypatch.setenv(var, val)
        g = _geometries(case)
        want_route = CORR_V1 if var == "BB200_CONV_SMALL_V1" else CORR2
        assert g["tf"]["route"] == want_route, f"{case} {var}={val}: {g['tf']}"
        if var == "BB200_CORR2_VW1":
            assert g["tf"]["VW"] == 1
        got = run_node(case, inp)
        monkeypatch.delenv(var)
        for k in _corr_keys(case):
            assert torch.equal(got[k], base[k]), \
                f"{case}: {k} under {var}={val} differs from corr2 (max {float((got[k] - base[k]).abs().max()):.3e})"
        check_against_fp64(case, got, ref, mag, f"{case} {var}={val}")
        seen.append(f"{var}={val}")
    print(f"[small conv] {case}: bit-identical correlation outputs under {', '.join(seen)}")


@pytest.mark.parametrize("case", ("lenet_conv1", "lenet_conv1_tx"))
def test_misaligned_operands_stage_4_bytes(case):
    """x and t_x at base + 1 float: the shape stages 16-byte vectors when aligned, so the launch has to fall back to
    4-byte copies; same bits as the aligned run."""
    assert _geometries(case)["tf"]["VW"] == 4
    inp = _inputs(case)
    a = run_node(case, inp)
    b = run_node(case, inp, misalign=True)
    ref, mag = reference(case, inp)
    check_against_fp64(case, b, ref, mag, f"{case} misaligned")
    for k in _corr_keys(case):
        assert torch.equal(a[k], b[k]), f"{case}: {k} from a misaligned view differs from the aligned run"


WGRAD_ROUTES = {
    # conv1: v1 by default (15 tasks), wgrad2 with BB200_WGRAD2_ALWAYS
    "lenet_conv1_ragged": ("BB200_WGRAD2_ALWAYS", WGRAD_V1, WGRAD2),
    # conv2: wgrad2 by default, v1 (TPT = 2 with 480 tasks) with BB200_CONV_SMALL_V1
    "lenet_conv2_ragged": ("BB200_CONV_SMALL_V1", WGRAD2, WGRAD_V1),
}


@pytest.mark.parametrize("case", sorted(WGRAD_ROUTES))
def test_weight_gradient_routes_and_run_to_run_identity(case, monkeypatch):
    """Both weight-gradient kernels against fp64, and each of them bit-identical from run to run (per-block partials
    added in block order, no atomics)."""
    var, r0, r1 = WGRAD_ROUTES[case]
    inp = _inputs(case)
    ref, mag = reference(case, inp)
    res = {}
    for route, env in ((r0, None), (r1, var)):
        if env:
            monkeypatch.setenv(env, "1")
        g = _geometries(case)["wgrad"]
        assert g["route"] == route, f"{case} {env}: weight gradient route {g}"
        runs = [run_node(case, inp) for _ in range(2)]
        if env:
            monkeypatch.delenv(env)
        for k in ("a_W", "at_W"):
            a, b = runs[0][k], runs[1][k]
            assert torch.equal(a, b), f"{case} route {route}: {k} differs between two runs (max {float((a - b).abs().max()):.3e})"
        res[route] = check_against_fp64(case, runs[0], ref, mag, f"{case} route {route}")
    print(f"[small conv] {case}: weight gradient bit-identical run to run on routes {r0} and {r1}; "
          f"at_W vs fp64 {res[r0]['at_W']:.2e} / {res[r1]['at_W']:.2e}")
