"""``sama`` (SURVEY.md 8 f3): the plugin against what the REAL reference function ``betty.hypergradient.sama.sama``
returns on the same seeded inputs (tests/golden/sama, made by oracle/make_golden.py), with a lower Adam optimizer whose
state carries exp_avg / exp_avg_sq / last_grad the way the reference's ImplicitProblem stores them
(implicit_problem.py:50-66), and with SGD (identity preconditioner)."""
import os

import pytest
import torch

from betty_b200 import hypergradient as H
from oracle import make_golden as MG
from tests.helpers import assert_close, rel_l2

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sama")


def _golden(name, wl):
    rec = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    assert abs(MG.input_checksum(wl) - rec["checksum"]) <= 1e-6 * max(1.0, abs(rec["checksum"])), "inputs drifted"
    return rec


@pytest.mark.parametrize("case", ["logistic", "mlp", "lenet"])
@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_sama_matches_the_reference_function(case, optimizer):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    name = f"sama_{optimizer}_{case}"
    fac, kw, opt = MG.SAMA_CASES[name]
    wl = MG.sama_workload(fac, kw, opt, device="cuda")     # seeded on the CPU generator, as the golden run was
    want = [t.cuda() for t in _golden(name, wl)["hypergrad"]]
    w_before = [p.detach().clone() for p in wl.lower.parameters()]
    got = H.sama(wl.vector, wl.lower, wl.upper, False)
    # finite differences in fp32: the reference's own noise floor applies (SURVEY 8c); measured against float64 below
    assert_close(got, want, 5e-3 if case != "logistic" else 1e-3, f"sama {case}/{optimizer}")
    for a, b in zip(wl.lower.parameters(), w_before):
        assert torch.allclose(a, b, rtol=0, atol=1e-5)        # parameters restored (sama.py:49-51)
    # sync=True accumulates into .grad and returns None
    for p in wl.upper.trainable_parameters():
        p.grad = None
    assert H.sama(wl.vector, wl.lower, wl.upper, True) is None
    assert rel_l2([p.grad for p in wl.upper.trainable_parameters()], want) < 1e-2


def test_adam_preconditioner_kernel_against_the_reference_formula():
    from betty_b200.hypergradient.sama import precondition

    wl = MG.precondition_workload(device="cuda")
    rec = _golden("precondition", wl)
    got = precondition(list(wl.vector), wl.lower)
    assert_close(got, [t.cuda() for t in rec["adam"]], 1e-5, "adam preconditioner")
    # a parameter without state (never stepped): the reference substitutes zeros, so does the kernel
    p0 = next(iter(wl.lower.module.parameters()))
    wl.lower.optimizer.state[p0] = {}
    assert_close(precondition(list(wl.vector), wl.lower), [t.cuda() for t in rec["adam_empty_first"]], 1e-5, "empty state")
