"""The depthwise convolution kernels (csrc/conv_dw.cu) at every (kernel, dilation, stride, channels, plane) the DARTS
search network Network(16, 10, 8) runs them at, B = 64, against float64.

One-node fp32 conv2d plans (groups = C = O, dims[15] = groups) are built by hand and run through PASS_BB, PASS_TF and
PASS_TB with every operand active.  Checks:
  * t_y, a_x, at_x element by element:  |got - ref| <= c (K + 2) 2^-23 (sum |in| |w| + |C0|),  K = npairs KH KW;
  * the weight gradients a_W, at_W: rel-L2 and max|err| / max|ref| (K = N HO WO terms);
  * the weight gradient is fixed-order (per-block partials added in block order): two runs give the same bits.
The ``ragged`` cases use a batch that leaves the last image group of the weight-gradient blocks short, so the partials
finish adds several partials of unequal extent.  ``test_depthwise_with_bias`` adds an active bias: the in-kernel t_b
term of the tangent forward and the channel sums after the depthwise launches.

Mutants these tests catch: the weight-gradient finish dropping its last partial (a_W / at_W of the ragged cases: the
last group holds 5 of 61 images), the tangent-backward kernel omitting the a_y (x) t_x term (at_W), a dropped
dwT(a_y, t_W) term (at_x), a wrong halo offset or dilation stride in the tap table (t_y, a_W)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from betty_b200 import _native as N
from betty_b200.plan import NODE_DTYPE, OPS, PASS_BB, PASS_TB, PASS_TF

pytestmark = pytest.mark.gpu

SM = 132
# Bars, set from the worst values measured on an H100 80 GB over every case below (printed per case)
CORR_C = 1 / 4          # t_y, a_x, at_x: worst measured ratio at c = 1 is 0.16 (a_x)
WGRAD_REL = 2e-6        # a_W, at_W, rel-L2 and max|err| / max|ref|: worst measured 3.5e-7
BIAS_REL = 8e-6         # a_b, at_b: conv.cu's channel sums, the bar of tests/test_conv_small_scale_gpu.py

# the depthwise ops of the DARTS cells: (k, dilation) of sep_conv_3x3 / sep_conv_5x5 / dil_conv_3x3 / dil_conv_5x5
OPS_KD = ((3, 1), (5, 1), (3, 2), (5, 2))
# (C, H, stride): normal cells at 16 x 32^2, 32 x 16^2, 64 x 8^2; the first depthwise conv of a reduction cell's edge
SHAPES = ((16, 32, 1), (32, 16, 1), (64, 8, 1), (32, 32, 2), (64, 16, 2))
CASES = {f"c{c}_h{h}_s{s}_k{k}_d{d}": (64, c, h, k, d, s) for (c, h, s) in SHAPES for (k, d) in OPS_KD}
CASES["ragged_c64_h8_k3_d1"] = (61, 64, 8, 3, 1, 1)
CASES["ragged_c32_h32_s2_k5_d2"] = (61, 32, 32, 5, 2, 2)


def images_per_block(n, c, ho, wo):
    """conv_dw.cu geom(): image groups double while a group has < 512 outputs and the grid covers every SM twice."""
    ipb = 1
    while 2 * ipb <= n and ipb * ho * wo < 512 and ((n + 2 * ipb - 1) // (2 * ipb)) * c >= 2 * SM:
        ipb *= 2
    return ipb


def _geom(case):
    n, c, h, k, d, s = CASES[case]
    p = d * (k - 1) // 2
    ho = (h + 2 * p - d * (k - 1) - 1) // s + 1
    return n, c, h, k, d, s, p, ho


def _inputs(case, seed=1234):
    n, c, h, k, d, s, p, ho = _geom(case)
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *sh, scale=1.0: torch.randn(*sh, generator=g, device="cuda") * scale
    return dict(x=r(n, c, h, h), t_x=r(n, c, h, h), W=r(c, 1, k, k, scale=0.3), t_W=r(c, 1, k, k, scale=0.3),
                a_y=r(n, c, ho, ho), at_y=r(n, c, ho, ho), a_x0=r(n, c, h, h), at_x0=r(n, c, h, h),
                a_W0=r(c, 1, k, k), at_W0=r(c, 1, k, k))


def run_node(case, inp, beta=1):
    n, c, h, k, d, s, p, ho = _geom(case)
    nan = lambda *sh: torch.full(sh, float("nan"), device="cuda")
    out = {"t_y": nan(n, c, ho, ho)}
    bias = "t_b" in inp
    for key in ("a_x", "at_x", "a_W", "at_W") + (("a_b", "at_b") if bias else ()):
        out[key] = inp[key + "0"].clone() if beta else nan(*inp[key + "0"].shape)
    rec = np.zeros(1, dtype=NODE_DTYPE)
    r = rec[0]
    r["op"], r["kind"] = OPS["conv2d"], 0
    r["active"] = r["pad0"] = 7 if bias else 3
    r["beta"][:] = (beta, beta, beta, 0)
    r["dims"][0:16] = (n, c, h, h, c, k, k, ho, ho, s, s, p, p, d, d, c)
    r["base"][0], r["base"][1] = inp["x"].data_ptr(), inp["W"].data_ptr()
    r["t"][0], r["a"][0], r["at"][0] = inp["t_x"].data_ptr(), out["a_x"].data_ptr(), out["at_x"].data_ptr()
    r["t"][1], r["a"][1], r["at"][1] = inp["t_W"].data_ptr(), out["a_W"].data_ptr(), out["at_W"].data_ptr()
    if bias:
        r["t"][2], r["a"][2], r["at"][2] = inp["t_b"].data_ptr(), out["a_b"].data_ptr(), out["at_b"].data_ptr()
    r["t"][3], r["a"][3], r["at"][3] = out["t_y"].data_ptr(), inp["a_y"].data_ptr(), inp["at_y"].data_ptr()
    handle = C.c_void_p()
    N.call("bb_plan_create", rec.ctypes.data, 1, C.byref(handle))
    try:
        st = torch.cuda.current_stream().cuda_stream
        for pas in (PASS_BB, PASS_TF, PASS_TB):
            N.call("bb_plan_run", handle, pas, st)
        torch.cuda.synchronize()
    finally:
        N.lib().bb_plan_destroy(handle)
    return out


def reference(case, inp, beta=1):
    n, c, h, k, d, s, p, ho = _geom(case)
    D = {key: v.double() for key, v in inp.items()}
    conv = lambda a, w: F.conv2d(a, w, None, s, p, d, c)
    dgrad = lambda gy, w: torch.nn.grad.conv2d_input(D["x"].shape, w, gy, s, p, d, c)
    wgrad = lambda a, gy: torch.nn.grad.conv2d_weight(a, D["W"].shape, gy, s, p, d, c)
    ref = {"t_y": conv(D["t_x"], D["W"]) + conv(D["x"], D["t_W"]),
           "a_x": dgrad(D["a_y"], D["W"]),
           "at_x": dgrad(D["at_y"], D["W"]) + dgrad(D["a_y"], D["t_W"]),
           "a_W": wgrad(D["x"], D["a_y"]),
           "at_W": wgrad(D["x"], D["at_y"]) + wgrad(D["t_x"], D["a_y"])}
    A = {key: v.abs() for key, v in D.items()}
    mag = {"t_y": F.conv2d(A["t_x"], A["W"], None, s, p, d, c) + F.conv2d(A["x"], A["t_W"], None, s, p, d, c),
           "a_x": torch.nn.grad.conv2d_input(D["x"].shape, A["W"], A["a_y"], s, p, d, c),
           "at_x": torch.nn.grad.conv2d_input(D["x"].shape, A["W"], A["at_y"], s, p, d, c)
           + torch.nn.grad.conv2d_input(D["x"].shape, A["t_W"], A["a_y"], s, p, d, c)}
    if "t_b" in D:
        ref["t_y"] = ref["t_y"] + D["t_b"].view(1, -1, 1, 1)
        mag["t_y"] = mag["t_y"] + A["t_b"].view(1, -1, 1, 1)
        ref["a_b"], ref["at_b"] = D["a_y"].sum((0, 2, 3)), D["at_y"].sum((0, 2, 3))
    if beta:
        for key in [q for q in ("a_x", "at_x", "a_W", "at_W", "a_b", "at_b") if q in ref]:
            ref[key] = ref[key] + D[key + "0"]
            if key in mag:
                mag[key] = mag[key] + A[key + "0"]
    return ref, mag


def check(case, got, ref, mag):
    n, c, h, k, *_ = _geom(case)
    worst = {}
    for key, want in ref.items():
        a = got[key].double()
        assert torch.isfinite(a).all(), f"{case}: {key} has non-finite values (an element was not written)"
        err = (a - want).abs()
        if key in mag:
            npairs = 1 if key == "a_x" else 2
            ratio = float((err / ((npairs * k * k + 2) * 2.0 ** -23 * mag[key]).clamp_min(1e-300)).max())
            worst[key] = ratio
            assert ratio <= CORR_C, f"{case}: {key} error {ratio:.3e} of the fp32 bound (bar {CORR_C})"
        else:
            rel = float(err.norm() / want.norm())
            mx = float(err.max() / want.abs().max())
            worst[key] = max(rel, mx)
            bar = BIAS_REL if key in ("a_b", "at_b") else WGRAD_REL
            assert rel <= bar and mx <= bar, f"{case}: {key} rel-L2 {rel:.3e}, max {mx:.3e} (bar {bar})"
    return worst


@pytest.mark.parametrize("case", sorted(CASES))
def test_depthwise_against_float64(case):
    n, c, h, k, d, s, p, ho = _geom(case)
    assert N.lib().bb_conv_dw_ok(c, c, c, h, h, k, k, ho, ho, p, p) == 1
    groups = -(-n // images_per_block(n, c, ho, ho))
    if case.startswith("ragged"):
        assert groups > 1 and n % images_per_block(n, c, ho, ho), f"{case}: no ragged last image group"
    inp = _inputs(case)
    got = run_node(case, inp)
    ref, mag = reference(case, inp)
    worst = check(case, got, ref, mag)
    again = run_node(case, inp)
    for key in got:
        assert torch.equal(got[key], again[key]), f"{case}: {key} differs between two runs"
    print(f"[depthwise] {case}: N {n}, image groups {groups}; worst: "
          + ", ".join(f"{key} {v:.2e}" for key, v in sorted(worst.items())))


def test_depthwise_overwrite_mode():
    """beta = 0: adjoints are overwritten (outputs start as NaN)."""
    case = "ragged_c64_h8_k3_d1"
    inp = _inputs(case, seed=7)
    got = run_node(case, inp, beta=0)
    ref, mag = reference(case, inp, beta=0)
    check(case, got, ref, mag)


@pytest.mark.parametrize("beta", (1, 0))
def test_depthwise_with_bias(beta):
    """An active bias: t_y gains t_b in the forward kernel; a_b / at_b are the channel sums of a_y / at_y."""
    case = "ragged_c32_h32_s2_k5_d2"
    inp = _inputs(case, seed=11)
    g = torch.Generator(device="cuda").manual_seed(12)
    c = CASES[case][1]
    for key in ("t_b", "a_b0", "at_b0"):
        inp[key] = torch.randn(c, generator=g, device="cuda")
    got = run_node(case, inp, beta=beta)
    ref, mag = reference(case, inp, beta=beta)
    check(case, got, ref, mag)
