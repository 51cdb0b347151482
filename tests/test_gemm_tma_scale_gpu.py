"""The TMA-fed wgmma GEMM (csrc/gemm_tma.cu) at the products of one RoBERTa-base layer, as the benchmark's
bert_data_reweighting line runs them (B=16 x L=50 = 800 tokens, hidden 768, 12 heads of 64, FFN 3072, bf16 autocast).

The shapes and strides below come from the lowered IR of that workload: record_tape of
``workloads.roberta_reweight(batch=16, seq=50, precision="bf16")`` and ``ir.lower_tape`` give 98 gemm nodes, per layer
four 800x768x768 and one 800x3072x768 / 800x768x3072 Linear (A = activations, k-contiguous; B = the weight read
transposed, brs = 1, bcs = in; bias), and two batched attention products over 192 (sequence, head) slices:
Q.K^T (A = Q [192][50][64], B = K^T copied contiguous [192][64][50]) and P.V (A = P [192][50][50], B = V).  Each node
runs in the tangent pass as the two-pair product W.t_x + t_W.x and in the adjoint pass as a data gradient
(gC.B^T [+ aC.t_B^T]) and a weight gradient (A^T.gC [+ t_A^T.aC], written into the transposed weight: crs = 1); this
file builds those forms from the same layouts (gemm.cu bb_launch_gemm) and calls them through bb_gemm_bf16_tma_ex,
which reports the configuration it launched so that each case asserts the route it names.

Reference: the float64 product of the bf16-rounded operands (+ bias, + C0 when accumulating).  The check is
elementwise, |C - ref| <= c * (K + 2) * 2^-23 * (sum_p |A_p|.|B_p| + |bias| + |C0|)_ij + tiny, so one wrong tile,
a dropped k-block or a bias added by every split fails on its own elements instead of vanishing in a global norm.
c = 1/8: the worst ratio measured over this file with c = 1 was 3.4e-2 (P.V's weight gradient; H100 SXM 80 GB, 700 W),
so the bar leaves a factor 3.7, while a bias added by every split lands at ~200 and a skipped tile at NaN (the outputs
start as NaN).  Every case prints its worst ratio to the bound."""
import ctypes as C

import pytest
import torch

from betty_b200 import _native as N
from betty_b200.arena import stream_ptr

pytestmark = pytest.mark.gpu

C_BOUND = 0.125                   # see the module docstring
TOKENS, HID, FFN, SLICES, SEQ, HD = 800, 768, 3072, 192, 50, 64
FORCE_BN64, FORCE_BN128, NO_PERSIST = 1, 2, 4
SM = 132


def _ksplit(n):
    return n << 8


class Op:
    """A strided operand: storage tensor (fp32 or bf16) and (row, col, batch) strides of the logical matrix."""

    def __init__(self, t, rs, cs, bs=0):
        self.t, self.rs, self.cs, self.bs = t, rs, cs, bs

    def dt(self):
        return 1 if self.t.dtype == torch.bfloat16 else 0

    def logical(self, batch, rows, cols):
        v = torch.as_strided(self.t, (batch, rows, cols), (self.bs, self.rs, self.cs))
        return v.to(torch.bfloat16).double()


def _rand(*shape, scale=1.0, dtype=torch.float32, gen=None):
    return (torch.randn(*shape, generator=gen) * scale).to(dtype).cuda()


_SCRATCH = {}


def _scratch():
    if "s" not in _SCRATCH:
        _SCRATCH["s"] = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    return _SCRATCH["s"]


def run(M, Nn, K, pairs, out, crs, ccs, cbs=0, batch=1, beta=0, bias=None, plane_ohw=0, min_n=64, flags=0):
    """C (beta)= sum_p A_p . B_p (+ bias) through bb_gemm_bf16_tma_ex.  pairs: [(A: Op over (m, k), B: Op over
    (k, n))].  Returns the launched route {bn, ksplit, persistent, kinds}."""
    n = len(pairs)
    aptr = (C.c_void_p * 2)(*[p[0].t.data_ptr() for p in pairs], *([0] * (2 - n)))
    bptr = (C.c_void_p * 2)(*[p[1].t.data_ptr() for p in pairs], *([0] * (2 - n)))
    ad = (C.c_int64 * 8)(*sum([[a.dt(), a.rs, a.cs, a.bs] for a, _ in pairs], []), *([0] * 4 * (2 - n)))
    bd = (C.c_int64 * 8)(*sum([[b.dt(), b.rs, b.cs, b.bs] for _, b in pairs], []), *([0] * 4 * (2 - n)))
    route = (C.c_int * 7)()
    s = _scratch()
    N.call("bb_gemm_bf16_tma_ex", M, Nn, K, n, batch, aptr, ad, bptr, bd, out.data_ptr(), crs, ccs, cbs, beta,
           None if bias is None else bias.data_ptr(), 1, plane_ohw, min_n, flags, s.data_ptr(), s.numel(), route,
           stream_ptr())
    torch.cuda.synchronize()
    return dict(bn=route[0], ksplit=route[1], persistent=bool(route[2]), kinds=tuple(route[3:7]))


def reference(M, Nn, K, pairs, batch, c0=None, bias=None):
    """(float64 result, float64 magnitude sum_p |A_p|.|B_p| + |bias| + |C0|), both [batch][M][N]."""
    ref = torch.zeros(batch, M, Nn, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref)
    for a, b in pairs:
        A, B = a.logical(batch, M, K), b.logical(batch, K, Nn)
        ref += A @ B
        mag += A.abs() @ B.abs()
    if bias is not None:
        ref += bias.double()
        mag += bias.double().abs()
    if c0 is not None:
        ref += c0.double()
        mag += c0.double().abs()
    return ref, mag


def check(name, got, ref, mag, K):
    """Elementwise bound; returns the worst ratio |C - ref| / bound and prints it with its location."""
    bound = C_BOUND * (K + 2) * 2.0 ** -23 * mag + 1e-30
    err = (got.double() - ref).abs()
    ratio = err / bound
    worst = float(ratio.max())
    where = tuple(int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
    print(f"[gemm scale] {name}: worst |C-ref|/bound {worst:.3e} at {where} (bound c={C_BOUND})")
    bad = int((~(ratio <= 1)).sum())          # NaN (an element never written) counts as outside
    assert bad == 0, (f"{name}: {bad} of {ratio.numel()} elements outside the bound, worst {worst:.3e} at {where}: "
                      f"got {float(got.reshape(ratio.shape)[where]):.6e} want {float(ref[where]):.6e}")
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# one RoBERTa-base layer: the Linear products
LINEARS = {"qkvo": (HID, HID), "ffn_up": (HID, FFN), "ffn_down": (FFN, HID)}


def _linear_tensors(din, dout, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(
        x=_rand(TOKENS, din, dtype=torch.bfloat16, gen=g),         # autocast copy of the activations
        tx=_rand(TOKENS, din, gen=g),
        W=_rand(dout, din, scale=0.02, dtype=torch.bfloat16, gen=g),   # autocast copy of the weight
        tW=_rand(dout, din, scale=0.02, gen=g),
        b=_rand(dout, scale=0.5, gen=g), tb=_rand(dout, scale=0.5, gen=g),
        ay=_rand(TOKENS, dout, scale=1e-3, gen=g), aty=_rand(TOKENS, dout, scale=1e-3, gen=g),
    )


def linear_products(din, dout, T):
    """name -> (M, N, K, pairs, bias, output layout (rows, cols, crs, ccs), beta)"""
    x, tx = Op(T["x"], din, 1), Op(T["tx"], din, 1)
    Wt, tWt = Op(T["W"], 1, din), Op(T["tW"], 1, din)          # B[k = in][n = out] = W[n][k]
    W, tW = Op(T["W"], din, 1), Op(T["tW"], din, 1)            # B[k = out][n = in] = W[k][n]
    ay, aty = Op(T["ay"], dout, 1), Op(T["aty"], dout, 1)
    xT, txT = Op(T["x"], 1, din), Op(T["tx"], 1, din)          # A[m = in][k = token]
    row = (TOKENS, dout, dout, 1)
    return {
        "fwd": (TOKENS, dout, din, [(x, Wt)], T["b"], row, 0),
        "tangent_fwd": (TOKENS, dout, din, [(tx, Wt), (x, tWt)], T["tb"], row, 0),
        "data_grad": (TOKENS, din, dout, [(ay, W)], None, (TOKENS, din, din, 1), 1),
        "data_grad_tangent": (TOKENS, din, dout, [(aty, W), (ay, tW)], None, (TOKENS, din, din, 1), 1),
        # weight gradient into the transposed weight [out][in]: C[m = in][n = out] at n*din + m
        "weight_grad": (din, dout, TOKENS, [(xT, ay)], None, (din, dout, 1, din), 1),
        "weight_grad_tangent": (din, dout, TOKENS, [(xT, aty), (txT, ay)], None, (din, dout, 1, din), 1),
    }


LINEAR_CASES = [(lin, prod) for lin in LINEARS for prod in ("fwd", "tangent_fwd", "data_grad", "data_grad_tangent",
                                                              "weight_grad", "weight_grad_tangent")]


def _out(rows, cols, crs, ccs, beta, seed):
    g = torch.Generator().manual_seed(seed)
    store = (torch.randn(rows * cols, generator=g) if beta else torch.full((rows * cols,), float("nan"))).cuda()
    c0 = torch.as_strided(store, (rows, cols), (crs, ccs)).clone() if beta else None
    return store, c0


def _logical_out(store, rows, cols, crs, ccs, batch=1, cbs=0):
    return torch.as_strided(store, (batch, rows, cols), (cbs, crs, ccs))


@pytest.mark.parametrize("lin,prod", LINEAR_CASES)
def test_roberta_linear_products(lin, prod):
    din, dout = LINEARS[lin]
    T = _linear_tensors(din, dout, seed=LINEAR_CASES.index((lin, prod)))
    M, Nn, K, pairs, bias, (rows, cols, crs, ccs), beta = linear_products(din, dout, T)[prod]
    store, c0 = _out(rows, cols, crs, ccs, beta, 1)
    r = run(M, Nn, K, pairs, store, crs, ccs, beta=beta, bias=bias)
    ref, mag = reference(M, Nn, K, pairs, 1, None if c0 is None else c0[None], bias)
    print(f"[gemm scale] {lin}/{prod} {M}x{Nn}x{K} pairs={len(pairs)}: route {r}")
    assert r["kinds"][2 * len(pairs):] == (-1,) * (4 - 2 * len(pairs))
    check(f"{lin}/{prod}", _logical_out(store, rows, cols, crs, ccs), ref, mag, K)


# ---------------------------------------------------------------------------------------------------------------------
# attention: batched over 192 (sequence, head) slices, K = 50 is one ragged k-block
def _attn_tensors(seed):
    g = torch.Generator().manual_seed(seed)
    t = {}
    for nm in ("Q", "V"):
        t[nm] = _rand(SLICES, SEQ, HD, dtype=torch.bfloat16, gen=g)
        t["t" + nm] = _rand(SLICES, SEQ, HD, gen=g)
    t["Kt"] = _rand(SLICES, HD, SEQ, dtype=torch.bfloat16, gen=g)
    t["tKt"] = _rand(SLICES, HD, SEQ, gen=g)
    t["P"] = torch.softmax(_rand(SLICES, SEQ, SEQ, gen=g), -1).to(torch.bfloat16)
    t["tP"] = _rand(SLICES, SEQ, SEQ, scale=0.02, gen=g)
    for nm, shp in (("S", (SLICES, SEQ, SEQ)), ("O", (SLICES, SEQ, HD))):     # adjoints of scores / context
        t["a" + nm] = _rand(*shp, scale=1e-2, gen=g)
        t["at" + nm] = _rand(*shp, scale=1e-2, gen=g)
    return t


def attention_products(T):
    """name -> (M, N, K, pairs, output (rows, cols)).  Outputs are contiguous [192][rows][cols]."""
    sq, so, ss = SEQ * HD, SEQ * HD, SEQ * SEQ
    Q, tQ = Op(T["Q"], HD, 1, sq), Op(T["tQ"], HD, 1, sq)
    Kt, tKt = Op(T["Kt"], SEQ, 1, sq), Op(T["tKt"], SEQ, 1, sq)
    P, tP = Op(T["P"], SEQ, 1, ss), Op(T["tP"], SEQ, 1, ss)
    V, tV = Op(T["V"], HD, 1, sq), Op(T["tV"], HD, 1, sq)
    aS, atS = Op(T["aS"], SEQ, 1, ss), Op(T["atS"], SEQ, 1, ss)
    aO, atO = Op(T["aO"], HD, 1, so), Op(T["atO"], HD, 1, so)
    KtT, tKtT = Op(T["Kt"], 1, SEQ, sq), Op(T["tKt"], 1, SEQ, sq)   # B[k][n] = Kt[n][k]
    QT, tQT = Op(T["Q"], 1, HD, sq), Op(T["tQ"], 1, HD, sq)         # A[m][k] = Q[k][m]
    VT, tVT = Op(T["V"], 1, HD, sq), Op(T["tV"], 1, HD, sq)
    PT, tPT = Op(T["P"], 1, SEQ, ss), Op(T["tP"], 1, SEQ, ss)
    return {
        "qk": (SEQ, SEQ, HD, [(Q, Kt)], (SEQ, SEQ)),
        "qk_tangent": (SEQ, SEQ, HD, [(tQ, Kt), (Q, tKt)], (SEQ, SEQ)),
        "qk_grad_q": (SEQ, HD, SEQ, [(atS, KtT), (aS, tKtT)], (SEQ, HD)),
        "qk_grad_k": (HD, SEQ, SEQ, [(QT, atS), (tQT, aS)], (HD, SEQ)),
        "pv": (SEQ, HD, SEQ, [(P, V)], (SEQ, HD)),
        "pv_tangent": (SEQ, HD, SEQ, [(tP, V), (P, tV)], (SEQ, HD)),
        "pv_grad_p": (SEQ, SEQ, HD, [(atO, VT), (aO, tVT)], (SEQ, SEQ)),
        "pv_grad_v": (SEQ, HD, SEQ, [(PT, atO), (tPT, aO)], (SEQ, HD)),
    }


ATTN_CASES = ("qk", "qk_tangent", "qk_grad_q", "qk_grad_k", "pv", "pv_tangent", "pv_grad_p", "pv_grad_v")


@pytest.mark.parametrize("prod", ATTN_CASES)
def test_roberta_attention_products(prod):
    T = _attn_tensors(seed=ATTN_CASES.index(prod))
    M, Nn, K, pairs, (rows, cols) = attention_products(T)[prod]
    assert (rows, cols) == (M, Nn)
    for beta in (0, 1):
        g = torch.Generator().manual_seed(7)
        store = torch.randn(SLICES * M * Nn, generator=g).cuda()
        c0 = store.view(SLICES, M, Nn).clone() if beta else None
        r = run(M, Nn, K, pairs, store, Nn, 1, cbs=M * Nn, batch=SLICES, beta=beta, min_n=32)
        assert r["ksplit"] == 1 and not r["persistent"], r
        ref, mag = reference(M, Nn, K, pairs, SLICES, c0)
        check(f"attention/{prod} beta={beta} route {r}", store.view(SLICES, M, Nn), ref, mag, K)


# ---------------------------------------------------------------------------------------------------------------------
# routes
def _ffn_down(seed=3):
    T = _linear_tensors(FFN, HID, seed)
    return T, linear_products(FFN, HID, T)["fwd"]


@pytest.mark.parametrize("ksplit", [1, 2, 4, 8])
def test_forced_split_k_at_ffn_down(ksplit):
    """800 x 768 x 3072 (the FFN down projection, with bias) at each split count; two runs return the same bits."""
    T, (M, Nn, K, pairs, bias, _, _) = _ffn_down()
    outs = []
    for _ in range(2):
        out = torch.full((M * Nn,), float("nan"), device="cuda")
        r = run(M, Nn, K, pairs, out, Nn, 1, bias=bias, flags=_ksplit(ksplit))
        assert r["ksplit"] == ksplit, r
        outs.append(out)
    ref, mag = reference(M, Nn, K, pairs, 1, None, bias)
    check(f"ffn_down ksplit={ksplit} route {r}", outs[0].view(1, M, Nn), ref, mag, K)
    assert torch.equal(outs[0], outs[1]), f"ksplit={ksplit}: two runs differ by {float((outs[0] - outs[1]).abs().max()):.3e}"


@pytest.mark.parametrize("prod", ["weight_grad_tangent", "data_grad_tangent"])
@pytest.mark.parametrize("ksplit", [2, 4])
def test_forced_split_k_accumulating_strided(prod, ksplit):
    """Split-K into an accumulated output: the transposed weight gradient (column-major, K = 800 ragged) and the
    data gradient, two pairs each; bit-identical across runs."""
    din, dout = LINEARS["ffn_up"]
    T = _linear_tensors(din, dout, seed=11)
    M, Nn, K, pairs, bias, (rows, cols, crs, ccs), beta = linear_products(din, dout, T)[prod]
    outs = []
    for _ in range(2):
        store, c0 = _out(rows, cols, crs, ccs, beta, 5)
        r = run(M, Nn, K, pairs, store, crs, ccs, beta=beta, flags=_ksplit(ksplit))
        assert r["ksplit"] == ksplit, r
        outs.append(store)
    ref, mag = reference(M, Nn, K, pairs, 1, c0[None], None)
    check(f"ffn_up/{prod} ksplit={ksplit}", _logical_out(outs[0], rows, cols, crs, ccs), ref, mag, K)
    assert torch.equal(outs[0], outs[1]), f"{prod} ksplit={ksplit}: two runs differ"


@pytest.mark.parametrize("bn", [64, 128])
def test_forced_tile_width(bn):
    """The FFN up projection (800 x 3072 x 768) with each tile width, unsplit and split."""
    T = _linear_tensors(HID, FFN, seed=4)
    M, Nn, K, pairs, bias, _, _ = linear_products(HID, FFN, T)["tangent_fwd"]
    ref, mag = reference(M, Nn, K, pairs, 1, None, bias)
    for ks in (1, 2):
        out = torch.full((M * Nn,), float("nan"), device="cuda")
        r = run(M, Nn, K, pairs, out, Nn, 1, bias=bias,
                flags=(FORCE_BN64 if bn == 64 else FORCE_BN128) | _ksplit(ks))
        assert r["bn"] == bn and r["ksplit"] == ks, r
        check(f"ffn_up tangent bn={bn} ksplit={ks}", out.view(1, M, Nn), ref, mag, K)


@pytest.mark.parametrize("shape", [(4000, 3000, 200), (8192, 1280, 256)])
def test_persistent_kernel_matches_one_tile_per_cta(shape):
    """More than 4 x 132 CTAs: gemm_tma_persist_kernel walks several tiles per CTA.  One shape is ragged in M, N and
    K.  Each tile sees the same k-order on both kernels, so the outputs are bit-identical."""
    M, Nn, K = shape
    g = torch.Generator().manual_seed(M)
    A = Op(_rand(M, K, gen=g), K, 1)
    Bm = _rand(Nn, K, scale=0.05, dtype=torch.bfloat16, gen=g)
    B = Op(Bm, 1, K)
    bias = _rand(Nn, gen=g)
    ref, mag = reference(M, Nn, K, [(A, B)], 1, None, bias)
    outs = {}
    for persist in (True, False):
        out = torch.full((M * Nn,), float("nan"), device="cuda")
        r = run(M, Nn, K, [(A, B)], out, Nn, 1, bias=bias, flags=0 if persist else NO_PERSIST)
        tiles = -(-M // 128) * -(-Nn // r["bn"])
        assert tiles >= 600 and r["ksplit"] == 1 and r["persistent"] == persist, (r, tiles)
        check(f"{shape} persistent={persist} route {r}", out.view(1, M, Nn), ref, mag, K)
        outs[persist] = out
    assert torch.equal(outs[True], outs[False]), "persistent and one-tile-per-CTA kernels differ"


@pytest.mark.parametrize("persist", [True, False])
def test_plane_output(persist):
    """Output mode 2: rows are pixels (img, q) of planes with plane_ohw pixels, written NCHW, with bias."""
    imgs, ohw, Nn, K = 160, 441, 64, 576      # 552 m-tiles x one 64-wide n-tile: more than 4 x 132 CTAs
    M = imgs * ohw
    g = torch.Generator().manual_seed(9)
    A = Op(_rand(M, K, dtype=torch.bfloat16, gen=g), K, 1)
    B = Op(_rand(Nn, K, scale=0.05, gen=g), 1, K)
    bias = _rand(Nn, gen=g)
    out = torch.full((imgs * Nn * ohw,), float("nan"), device="cuda")
    r = run(M, Nn, K, [(A, B)], out, 0, 0, bias=bias, plane_ohw=ohw, min_n=32, flags=0 if persist else NO_PERSIST)
    assert r["persistent"] == persist, r
    ref, mag = reference(M, Nn, K, [(A, B)], 1, None, bias)
    ref = ref.view(imgs, ohw, Nn).permute(0, 2, 1).reshape(1, imgs * Nn, ohw)
    mag = mag.view(imgs, ohw, Nn).permute(0, 2, 1).reshape(1, imgs * Nn, ohw)
    check(f"plane output persistent={persist} route {r}", out.view(1, imgs * Nn, ohw), ref, mag, K)


def test_default_route_run_to_run():
    """The cost model's own choice at every Linear shape of the layer, twice: bit-identical."""
    for lin, (din, dout) in LINEARS.items():
        T = _linear_tensors(din, dout, seed=21)
        for prod, (M, Nn, K, pairs, bias, (rows, cols, crs, ccs), beta) in linear_products(din, dout, T).items():
            outs, routes = [], []
            for _ in range(2):
                store, _ = _out(rows, cols, crs, ccs, beta, 2)
                routes.append(run(M, Nn, K, pairs, store, crs, ccs, beta=beta, bias=bias))
                outs.append(store)
            assert routes[0] == routes[1]
            assert torch.equal(outs[0], outs[1]), f"{lin}/{prod} route {routes[0]}: two runs differ"
