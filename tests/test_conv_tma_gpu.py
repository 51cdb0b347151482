"""Unit test of the TMA-fed wgmma convolution kernels (csrc/conv_tma.cu: `gemm_tma_kernel` with TMA_CONV operands
for the forward / input-gradient products, `wgrad_tma_kernel` for the weight gradient, the im2col route of
data-input layers) through the C ABI, in the style of test_gemm_tma_gpu.py: a ONE-node plan is built by hand, every
operand holds bf16-representable values (so the kernels' bf16 operand packs are exact), and each output is compared
with the same convolution evaluated in float64.  What is left is fp32 accumulation order: 2e-5.

Rules under test (SURVEY.md App. B, Conv2d row):
    TF   t_y   = conv(t_x, W) + conv(x, t_W) + t_b
    TB   at_x  = dgrad(at_y, W) + dgrad(a_y, t_W)
         at_W += wgrad(at_y, x) + wgrad(a_y, t_x)        at_b += sum(at_y)
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from betty_b200 import _native as N
from betty_b200.plan import NODE_DTYPE, OPS, PASS_BB, PASS_TB, PASS_TF, HvpPlan

pytestmark = pytest.mark.gpu

# (N, C, H, W, O, k, pad)
SHAPES = {
    "c64_12x12": (4, 64, 12, 12, 64, 3, 1),
    "c64_21x21_odd": (3, 64, 21, 21, 64, 3, 1),
    "ragged_10x14_c32_o64": (5, 32, 10, 14, 64, 3, 1),
    "c48_o40_9x11": (4, 48, 9, 11, 40, 3, 1),          # channels not a multiple of 64 either way
    "valid_padding": (4, 64, 12, 12, 64, 3, 0),
    "one_by_one": (6, 64, 8, 8, 64, 1, 0),
    "wide_rows_42": (2, 64, 42, 42, 64, 3, 1),
    "data_input_c3": (6, 3, 20, 20, 64, 3, 1),         # x is data: im2col + plain TMA GEMMs (run_small_c)
    "data_input_c1_o32": (9, 1, 14, 14, 32, 3, 1),
}


def _bf(*shape, scale=1.0, gen=None):
    return (torch.randn(*shape, generator=gen, device="cuda") * scale).bfloat16()


def _rel(a, b):
    return float((a.double() - b).norm() / (b.norm() + 1e-300))


@pytest.mark.parametrize("case", sorted(SHAPES))
def test_conv_tma_rules_against_float64(case):
    n, c, h, w, o, k, pad = SHAPES[case]
    ho, wo = h + 2 * pad - k + 1, w + 2 * pad - k + 1
    g = torch.Generator(device="cuda").manual_seed(1234)
    data_input = c * k * k <= 64
    x, wt = _bf(n, c, h, w, gen=g), _bf(o, c, k, k, scale=0.2, gen=g)
    t_x = None if data_input else _bf(n, c, h, w, gen=g).float()
    t_w, t_b = _bf(o, c, k, k, scale=0.2, gen=g).float(), torch.randn(o, generator=g, device="cuda")
    a_y, at_y = _bf(n, o, ho, wo, gen=g).float(), _bf(n, o, ho, wo, gen=g).float()
    t_y = torch.full((n, o, ho, wo), float("nan"), device="cuda")
    a_x = torch.zeros(n, c, h, w, device="cuda")
    at_x = torch.full((n, c, h, w), float("nan"), device="cuda")
    at_w, at_b = torch.zeros(o, c, k, k, device="cuda"), torch.zeros(o, device="cuda")

    rec = np.zeros(1, dtype=NODE_DTYPE)
    r = rec[0]
    r["op"], r["kind"] = OPS["conv2d"], 1
    r["active"] = (0 if data_input else 1) | 2 | 4
    r["pad0"] = 0 if data_input else 1
    r["beta"][:] = (0, 1, 1, 0)
    r["dims"][0:15] = (n, c, h, w, o, k, k, ho, wo, 1, 1, pad, pad, 1, 1)
    r["base"][0], r["dt"][0] = x.data_ptr(), 1
    r["base"][1], r["dt"][1] = wt.data_ptr(), 1
    if not data_input:
        r["t"][0], r["a"][0], r["at"][0] = t_x.data_ptr(), a_x.data_ptr(), at_x.data_ptr()
    r["t"][1], r["at"][1] = t_w.data_ptr(), at_w.data_ptr()
    r["t"][2], r["at"][2] = t_b.data_ptr(), at_b.data_ptr()
    r["t"][3], r["a"][3], r["at"][3] = t_y.data_ptr(), a_y.data_ptr(), at_y.data_ptr()

    handle = C.c_void_p()
    N.call("bb_plan_create", rec.ctypes.data, 1, C.byref(handle))
    try:
        scratch = torch.empty(HvpPlan._tma_scratch_bytes(r) + 4096, dtype=torch.uint8, device="cuda")
        N.call("bb_plan_set_scratch", handle, scratch.data_ptr(), scratch.numel())
        pbytes = HvpPlan._tma_persistent_bytes(r)
        persist = torch.empty(max(pbytes, 1), dtype=torch.uint8, device="cuda")
        if pbytes:
            N.call("bb_plan_set_persistent", handle, persist.data_ptr(), pbytes)
        for pas in (PASS_TF, PASS_TB):
            assert N.lib().bb_plan_node_route(handle, 0, pas) == 2, f"{case}: pass {pas} does not take the TMA path"
        s = torch.cuda.current_stream().cuda_stream
        N.call("bb_plan_run", handle, PASS_BB, s)        # packs the K-loop constants (x, a_y) into the persistent arena
        N.call("bb_plan_run", handle, PASS_TF, s)
        N.call("bb_plan_run", handle, PASS_TB, s)
        torch.cuda.synchronize()
    finally:
        N.lib().bb_plan_destroy(handle)

    d = lambda t: t.double()
    X, Wt, TW, AY, ATY = d(x), d(wt), d(t_w), d(a_y), d(at_y)
    want_ty = F.conv2d(X, TW, d(t_b), padding=pad)
    want_atw = torch.nn.grad.conv2d_weight(X, Wt.shape, ATY, padding=pad)
    if not data_input:
        TX = d(t_x)
        want_ty = want_ty + F.conv2d(TX, Wt, None, padding=pad)
        want_atw = want_atw + torch.nn.grad.conv2d_weight(TX, Wt.shape, AY, padding=pad)
        want_atx = (torch.nn.grad.conv2d_input(X.shape, Wt, ATY, padding=pad)
                    + torch.nn.grad.conv2d_input(X.shape, TW, AY, padding=pad))
        assert _rel(at_x, want_atx) < 2e-5, f"{case}: at_x {_rel(at_x, want_atx):.3e}"
    assert _rel(t_y, want_ty) < 2e-5, f"{case}: t_y {_rel(t_y, want_ty):.3e}"
    assert _rel(at_w, want_atw) < 2e-5, f"{case}: at_W {_rel(at_w, want_atw):.3e}"
    assert _rel(at_b, ATY.sum((0, 2, 3))) < 2e-5, f"{case}: at_b"
