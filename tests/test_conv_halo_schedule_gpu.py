"""The tile schedule of the halo convolution (csrc/conv_halo.cu, conv_halo_kernel): each CTA walks the tiles
blockIdx.x, blockIdx.x + grid, ... and its two consumer warpgroups take them in turn (local tile lt -> warpgroup lt & 1),
each accumulating all 128 rows of its tile (computed transposed: one m64n128 product per k-step).  The shapes below are chosen by their tile count against
the 132-CTA grid of an H100 SXM: fewer tiles than CTAs (warpgroup 1 never gets a tile), one and two tiles per CTA with some CTAs one
tile short, an odd number of tiles per CTA, ragged last tiles (total rows not a multiple of 128), and the three shapes
the implicit-MAML benchmark runs (N=800 at 42x42, 21x21, 10x10).  Each runs with one operand pair (four band buffers)
and two (two band buffers), both tap orders, with and without bias, into both outputs: bf16 padded NHWC and fp32 NCHW
accumulated onto existing values (beta = 1).

Reference: the float64 convolution of the bf16 operands.  The check is elementwise,
    |C - ref| <= c * (K + 2) * 2^-23 * (sum_p |A_p| * |B_p| + |bias| + |C0|)      (K = 9 * 64 * pairs)
plus, for the bf16 output, its rounding 2^-8 * (|ref| + that bound), so a lost or duplicated tile or one warpgroup's
rows gone wrong fails on its own elements instead of vanishing in a global norm.  c = C_BOUND, set from the worst
ratio measured over this file (see below); every case prints its worst ratio.  The outputs start as NaN, the padded
output's border rows must come back exactly zero, a canary past the last output element must be untouched, and two
runs must give the same bits."""
import pytest
import torch
import torch.nn.functional as F

from betty_b200 import _native as N

pytestmark = pytest.mark.gpu

# The worst ratio |C - ref| / bound measured over this file with c = 1 was 5.2e-3 (fp32 output; the bf16 output's error
# is its rounding; H100 SXM 80 GB, 700 W), so c = 1/32 leaves a factor 6, while an element never written stays NaN.
C_BOUND = 1.0 / 32
CANARY_ROWS = 128          # one tile's worth of padded rows past the output
CANARY = -7.0              # a value the kernel never writes there

# name: (N, H, W, tiles) -- tiles = ceil(N * (H+2) * (W+2) / 128), asserted below
SHAPES = {
    "91t_42x42_n6": (6, 42, 42, 91),            # < 132 tiles: one per CTA, warpgroup 1 idle; ragged
    "133t_10x10_n118": (118, 10, 10, 133),      # one tile per CTA, CTA 0 has two; ragged
    "263t_10x10_n233": (233, 10, 10, 263),      # two per CTA, one CTA a tile short; ragged
    "264t_10x10_n234": (234, 10, 10, 264),      # exactly two per CTA; ragged
    "265t_21x21_n64": (64, 21, 21, 265),        # two per CTA, CTA 0 has three; ragged
    "331t_21x21_n80": (80, 21, 21, 331),        # three tiles (odd) on 67 CTAs, two on the rest; ragged
    "605t_42x42_n40": (40, 42, 42, 605),        # five (odd) or four per CTA; last tile full
    "bench_42x42_n800": (800, 42, 42, 12100),
    "bench_21x21_n800": (800, 21, 21, 3307),    # ragged
    "bench_10x10_n800": (800, 10, 10, 900),
}
ORDER = list(SHAPES)       # small shapes first


def _padded(x):
    """NCHW float -> bf16 [N][H+2][W+2][64] with a zero border"""
    n, c, h, w = x.shape
    out = torch.zeros(n, h + 2, w + 2, 64, dtype=torch.bfloat16, device=x.device)
    out[:, 1:h + 1, 1:w + 1, :c] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
    return out


def _kernel(wm, flip):
    k = wm.double().reshape(64, 3, 3, 64).permute(0, 3, 1, 2)     # [n][ch][i][j]
    return k.flip(2, 3) if flip else k


def _check(name, got, exact, mag, bf16_out):
    """elementwise bar; returns the worst |got - exact| / bound at c = 1"""
    err = (got.double() - exact).abs()
    fp32 = mag * 2.0 ** -23
    rnd = 2.0 ** -8 * (exact.abs() + fp32) if bf16_out else torch.zeros_like(fp32)
    worst = float(((err - rnd).clamp_min(0) / fp32.clamp_min(1e-30)).max())
    ok = err <= C_BOUND * fp32 + rnd
    bad = int((~ok).sum())           # NaN (an element never written) counts as bad
    assert bad == 0, f"{name}: {bad} elements outside the bar (worst ratio {worst:.3e} at c = 1)"
    return worst


@pytest.mark.parametrize("case", ORDER)
@pytest.mark.parametrize("npairs", [1, 2])
@pytest.mark.parametrize("flip", [0, 1])
def test_halo_schedule_against_float64(case, npairs, flip):
    n, h, w, tiles = SHAPES[case]
    rows = n * (h + 2) * (w + 2)
    assert -(-rows // 128) == tiles
    g = torch.Generator(device="cuda").manual_seed(3 + 2 * npairs + flip)
    acts = [torch.randn(n, 64, h, w, generator=g, device="cuda").bfloat16().float() for _ in range(npairs)]
    wms = [(0.1 * torch.randn(64, 9, 64, generator=g, device="cuda")).bfloat16() for _ in range(npairs)]
    bias = torch.randn(64, generator=g, device="cuda")
    pads = [_padded(a) for a in acts]
    args = [pads[0].data_ptr(), pads[1].data_ptr() if npairs > 1 else 0, wms[0].data_ptr(),
            wms[1].data_ptr() if npairs > 1 else 0]
    ref = torch.zeros(n, 64, h, w, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref)
    for a, wm in zip(acts, wms):
        k = _kernel(wm, flip)
        ref += F.conv2d(a.double(), k, padding=1)
        mag += F.conv2d(a.double().abs(), k.abs(), padding=1)
    del acts
    K = 9 * 64 * npairs
    mag *= K + 2
    st = torch.cuda.current_stream().cuda_stream
    c0 = torch.randn(n, 64, h, w, generator=g, device="cuda")
    worst = []
    for with_bias in (False, True):
        bptr = bias.data_ptr() if with_bias else 0
        bb = bias.double().view(1, -1, 1, 1) if with_bias else 0.0
        babs = (K + 2) * bias.double().abs().view(1, -1, 1, 1) if with_bias else 0.0
        tag = f"{case} npairs={npairs} flip={flip} bias={int(with_bias)}"

        # bf16 padded NHWC
        runs = []
        for _ in range(2):
            buf = torch.full(((rows + CANARY_ROWS) * 64,), float("nan"), dtype=torch.bfloat16, device="cuda")
            buf[rows * 64:] = CANARY
            N.call("bb_conv_halo_bf16_nhwc", n, h, w, npairs, *args, flip, buf.data_ptr(), bptr, st)
            runs.append(buf)
        torch.cuda.synchronize()
        assert torch.equal(runs[0].view(torch.int16), runs[1].view(torch.int16)), f"{tag} nhwc: runs differ"
        buf = runs[0]
        assert bool((buf[rows * 64:] == CANARY).all()), f"{tag} nhwc: canary past the output overwritten"
        out = buf[:rows * 64].view(n, h + 2, w + 2, 64)
        border = out.clone()
        border[:, 1:-1, 1:-1, :] = 0
        assert bool((border == 0).all()), f"{tag} nhwc: border rows not zero"
        got = out[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2)
        worst.append(_check(f"{tag} nhwc", got, ref + bb, mag + babs, True))
        del runs, buf, out, border, got

        # fp32 NCHW, beta = 1
        runs = []
        for _ in range(2):
            buf = torch.full((n * 64 * h * w + 4096,), CANARY, device="cuda")
            buf[:n * 64 * h * w] = c0.reshape(-1)
            N.call("bb_conv_halo_bf16", n, h, w, npairs, *args, flip, buf.data_ptr(), 1, bptr, st)
            runs.append(buf)
        torch.cuda.synchronize()
        assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), f"{tag} nchw: runs differ"
        buf = runs[0]
        assert bool((buf[n * 64 * h * w:] == CANARY).all()), f"{tag} nchw: canary past the output overwritten"
        got = buf[:n * 64 * h * w].view(n, 64, h, w)
        worst.append(_check(f"{tag} nchw", got, c0.double() + ref + bb, mag + babs + (K + 2) * c0.double().abs(), False))
        del runs, buf, got
    print(f"{case} npairs={npairs} flip={flip}: worst ratio at c = 1: nhwc {max(worst[0::2]):.3e}, "
          f"nchw {max(worst[1::2]):.3e}")
