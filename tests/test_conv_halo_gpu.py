"""Unit test of the halo-resident wgmma convolution (csrc/conv_halo.cu) through the C ABI: one TMA band of
128 + 2(W+2) + 2 padded pixel rows per tile, nine taps = nine wgmma descriptors at 128-byte row offsets inside it.
Operands hold bf16 values, so the only error against the float64 convolution is fp32 accumulation order (2e-5)."""
import pytest
import torch
import torch.nn.functional as F

from betty_b200 import _native as N

pytestmark = pytest.mark.gpu

SHAPES = {"42x42_n6": (6, 42, 42), "21x21_n9": (9, 21, 21), "10x10_n40": (40, 10, 10), "5x7_n33": (33, 5, 7),
          "42x42_n800_slice": (37, 42, 42), "14x14_n25": (25, 14, 14)}


def _padded(x):
    """NCHW float -> bf16 [N][H+2][W+2][64] with a zero border"""
    n, c, h, w = x.shape
    out = torch.zeros(n, h + 2, w + 2, 64, dtype=torch.bfloat16, device=x.device)
    out[:, 1:h + 1, 1:w + 1, :c] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
    return out


@pytest.mark.parametrize("case", sorted(SHAPES))
@pytest.mark.parametrize("npairs,flip,beta", [(1, 0, 0), (2, 0, 0), (2, 1, 1), (1, 1, 0)])
def test_halo_convolution_against_float64(case, npairs, flip, beta):
    n, h, w = SHAPES[case]
    g = torch.Generator(device="cuda").manual_seed(7)
    acts = [torch.randn(n, 64, h, w, generator=g, device="cuda").bfloat16().float() for _ in range(npairs)]
    # weights as the kernel wants them: [n_out][tap][ch]
    wms = [(0.1 * torch.randn(64, 9, 64, generator=g, device="cuda")).bfloat16() for _ in range(npairs)]
    bias = torch.randn(64, generator=g, device="cuda") if not flip else None
    out0 = torch.randn(n, 64, h, w, generator=g, device="cuda")
    out = out0.clone() if beta else torch.full_like(out0, float("nan"))
    pads = [_padded(a) for a in acts]
    args = [pads[0].data_ptr(), pads[1].data_ptr() if npairs > 1 else 0, wms[0].data_ptr(), wms[1].data_ptr() if npairs > 1 else 0]
    N.call("bb_conv_halo_bf16", n, h, w, npairs, *args, flip, out.data_ptr(), beta, bias.data_ptr() if bias is not None else 0,
           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    want = out0.double() if beta else torch.zeros_like(out0, dtype=torch.float64)
    for a, wm in zip(acts, wms):
        k = wm.double().reshape(64, 3, 3, 64).permute(0, 3, 1, 2)       # [n][ch][i][j]
        if flip:
            k = k.flip(2, 3)
        want = want + F.conv2d(a.double(), k, padding=1)
    if bias is not None:
        want = want + bias.double().view(1, -1, 1, 1)
    err = float((out.double() - want).norm() / want.norm())
    assert err < 2e-5, f"{case} npairs={npairs} flip={flip}: rel {err:.3e}"


@pytest.mark.parametrize("case", sorted(SHAPES))
@pytest.mark.parametrize("npairs", [1, 2])
def test_halo_weight_gradient_against_float64(case, npairs):
    n, h, w = SHAPES[case]
    g = torch.Generator(device="cuda").manual_seed(11)
    xs = [torch.randn(n, 64, h, w, generator=g, device="cuda").bfloat16().float() for _ in range(npairs)]
    gys = [torch.randn(n, 64, h, w, generator=g, device="cuda").bfloat16().float() for _ in range(npairs)]
    out0 = torch.randn(64, 64, 3, 3, generator=g, device="cuda")
    out = out0.clone()
    xp, gp = [_padded(t) for t in xs], [_padded(t) for t in gys]
    N.call("bb_wgrad_halo_bf16", n, h, w, npairs, xp[0].data_ptr(), xp[1].data_ptr() if npairs > 1 else 0,
           gp[0].data_ptr(), gp[1].data_ptr() if npairs > 1 else 0, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    want = out0.double()
    for x, gy in zip(xs, gys):
        want = want + torch.nn.grad.conv2d_weight(x.double(), (64, 64, 3, 3), gy.double(), padding=1)
    err = float((out.double() - want).norm() / want.norm())
    assert err < 2e-5, f"{case} npairs={npairs}: rel {err:.3e}"


@pytest.mark.parametrize("case", ["42x42_n6", "21x21_n9", "5x7_n33"])
@pytest.mark.parametrize("flip", [0, 1])
def test_halo_convolution_bf16_padded_output(case, flip):
    """Output mode of the fused blocks: the product lands as bf16 in the padded NHWC layout (the next kernel's TMA
    operand), border rows written as zeros."""
    n, h, w = SHAPES[case]
    g = torch.Generator(device="cuda").manual_seed(5)
    acts = [torch.randn(n, 64, h, w, generator=g, device="cuda").bfloat16().float() for _ in range(2)]
    wms = [(0.1 * torch.randn(64, 9, 64, generator=g, device="cuda")).bfloat16() for _ in range(2)]
    bias = torch.randn(64, generator=g, device="cuda")
    pads = [_padded(a) for a in acts]
    out = torch.full((n, h + 2, w + 2, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    N.call("bb_conv_halo_bf16_nhwc", n, h, w, 2, pads[0].data_ptr(), pads[1].data_ptr(), wms[0].data_ptr(), wms[1].data_ptr(),
           flip, out.data_ptr(), bias.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    want = torch.zeros(n, 64, h, w, dtype=torch.float64, device="cuda")
    for a, wm in zip(acts, wms):
        k = wm.double().reshape(64, 3, 3, 64).permute(0, 3, 1, 2)
        want = want + F.conv2d(a.double(), k.flip(2, 3) if flip else k, padding=1)
    want = want + bias.double().view(1, -1, 1, 1)
    got = out[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2).double()
    assert float((got - want).norm() / want.norm()) < 4e-3          # bf16 rounding of the result
    border = out.clone()
    border[:, 1:-1, 1:-1, :] = 0
    assert float(border.float().abs().max()) == 0.0                 # NaN-filled border was overwritten with zeros
