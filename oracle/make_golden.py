"""TEST INFRASTRUCTURE -- generate ``tests/golden/*.pt`` by running the REAL reference.

Run where the reference sources are available (``bash oracle/fetch_ref.sh <reference checkout>`` mirrors them into
``oracle/_ref``):

    PYTHONDONTWRITEBYTECODE=1 python oracle/make_golden.py [case ...]

For every case below the seeded workload is built on CPU (fp32), the reference's own
``betty.hypergradient.{neumann,cg,darts}`` is called on it (``sync=False``) and the returned
hypergradient -- plus, for Neumann, the K-loop output of the reference's ``approx_inverse_hvp`` -- is
stored with a checksum of the inputs.  The cases are small so the fixtures stay a few hundred kB.
"""
import os
import sys

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))   # the reference mirror made by oracle/fetch_ref.sh

import torch  # noqa: E402

from betty_b200 import workloads as W  # noqa: E402

CASES = {
    "logistic_neumann": ("logistic_regression_hpo", dict(method="neumann", K=5, alpha=1.0)),
    "logistic_cg_quirk": ("logistic_regression_hpo", dict(method="cg", K=3, alpha=0.1)),
    "logistic_cg": ("logistic_regression_hpo", dict(method="cg", K=8, alpha=1.0)),
    "logistic_darts": ("logistic_regression_hpo", dict(method="darts")),
    "mlp_cg": ("mlp_reweight", dict(method="cg", K=5)),
    "mlp_neumann": ("mlp_reweight", dict(method="neumann", K=6, alpha=0.2)),
    "lenet_cg": ("learning_to_reweight", dict(method="cg", batch=8, K=5)),
    "lenet_neumann": ("learning_to_reweight", dict(method="neumann", batch=8, K=5, alpha=0.1)),
    "fourconv_neumann": ("implicit_maml", dict(method="neumann", n=10, K=5, alpha=0.01, hidden=16)),
    "fourconv_cg": ("implicit_maml", dict(method="cg", n=10, K=3, alpha=1.0, hidden=16)),
    "roberta_tiny_cg": ("bert_data_reweighting", dict(method="cg", batch=4, seq=10, K=3, tiny=True)),
    "roberta_tiny_neumann": ("bert_data_reweighting", dict(method="neumann", batch=4, seq=10, K=4, alpha=0.05, tiny=True)),
    "darts_lite": ("neural_architecture_search", dict(batch=4, c=4, cells=1)),
    # sama (reference hypergradient/sama.py): the factories attach the lower Adam state (workloads.attach_adam_state, 3 real steps)
    "logistic_sama": ("logistic_regression_hpo", dict(method="sama")),
    "mlp_sama": ("mlp_reweight", dict(method="sama")),
}


# Extra model families, used by the CPU oracle test only (tests/golden_cpu/): the GPU parity suite globs tests/golden/.
CPU_ONLY_CASES = {
    "resnet_cg": ("learning_to_reweight_resnet", dict(method="cg", batch=4, n=1, width=4, K=4)),
    "resnet_neumann": ("learning_to_reweight_resnet", dict(method="neumann", batch=4, n=1, width=4, K=5, alpha=0.05)),
    "fourconv_mini_neumann": ("implicit_maml", dict(method="neumann", n=2, K=4, alpha=0.01, hidden=4, image="miniimagenet")),
    "mlp_cg_long": ("mlp_reweight", dict(method="cg", K=12)),
}


# sama against the reference function with either lower optimizer (tests/test_sama_gpu.py, tests/golden/sama/; a
# subdirectory, so the parity suites, which glob tests/golden/*.pt, do not take these records for their own cases):
# factory, kwargs, lower optimizer ("adam": the state the factory attaches; "sgd": identity preconditioner).
SAMA_CASES = {
    f"sama_{opt}_{case}": (fac, kw, opt)
    for case, (fac, kw) in {"logistic": ("logistic_regression_hpo", dict(method="sama")),
                            "mlp": ("mlp_reweight", dict(method="sama")),
                            "lenet": ("learning_to_reweight", dict(method="sama", batch=32))}.items()
    for opt in ("adam", "sgd")
}


def sama_workload(factory, kw, opt, device="cpu"):
    wl = W.FACTORIES[factory](device=device, **kw)
    wl.lower.config.sama_adam_alpha = 1.0
    if opt == "sgd":
        wl.lower.optimizer = torch.optim.SGD(wl.lower.module.parameters(), lr=0.1)
    return wl


def precondition_workload(device="cpu"):
    """mlp_reweight with 4 Adam steps of lower state (the preconditioner fixture of tests/test_sama_gpu.py)."""
    wl = W.mlp_reweight(device=device, method="sama")
    wl.lower.optimizer = W.attach_adam_state(wl, 4, 1e-2).lower.optimizer
    return wl


def make_sama(out_dir, only):
    import importlib

    sama = importlib.import_module("betty.hypergradient.sama").sama      # the package re-exports the function
    precondition = importlib.import_module("betty.hypergradient.utils").precondition

    os.makedirs(out_dir, exist_ok=True)
    for case, (factory, kw, opt) in SAMA_CASES.items():
        if only and case not in only:
            continue
        wl = sama_workload(factory, kw, opt)
        rec = {"factory": factory, "kwargs": kw, "optimizer": opt, "checksum": input_checksum(wl), "torch": torch.__version__}
        rec["hypergrad"] = [g.detach().clone() for g in sama(wl.vector, wl.lower, wl.upper, False)]
        torch.save(rec, os.path.join(out_dir, case + ".pt"))
        print(f"{case:24s} |hg|={float(torch.cat([t.reshape(-1) for t in rec['hypergrad']]).norm()):.6e}")
    if not only or "precondition" in only:
        wl = precondition_workload()
        rec = {"checksum": input_checksum(wl), "torch": torch.__version__,
               "adam": [t.detach().clone() for t in precondition(list(wl.vector), wl.lower)]}
        p0 = next(iter(wl.lower.module.parameters()))
        wl.lower.optimizer.state[p0] = {}     # a parameter without state (never stepped)
        rec["adam_empty_first"] = [t.detach().clone() for t in precondition(list(wl.vector), wl.lower)]
        torch.save(rec, os.path.join(out_dir, "precondition.pt"))
        print("precondition")


def make_darts_network(out_path):
    """The reference's DARTS search network Network(16, 10, 8) + Architecture(4) (examples/neural_architecture_search)
    evaluated with the weights of betty_b200's restatement (seed 0) on a seeded input: its parameter shapes and logits
    (tests/test_workloads_cpu.py)."""
    import importlib
    import types

    nas = os.path.join(ROOT, "oracle", "_ref", "examples", "neural_architecture_search")
    sys.modules.setdefault("utils", types.SimpleNamespace(accuracy=None))   # model_search imports it for an unused helper
    sys.path.insert(0, nas)
    MS = importlib.import_module("model_search")
    torch.manual_seed(0)
    net, arch = W.DartsSearchNetwork(16, 10, 8), W.DartsArchitecture(4)
    ref, ref_arch = MS.Network(16, 10, 8, None), MS.Architecture(4)
    shapes = [tuple(p.shape) for p in ref.parameters()]
    with torch.no_grad():
        for a, b in zip(ref.parameters(), net.parameters()):
            a.copy_(b)
        for a, b in zip(ref_arch.parameters(), arch.parameters()):
            a.copy_(b)
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(1))
    ref.train()
    with torch.no_grad():
        logits = ref(x, ref_arch()).clone()
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    torch.save({"shapes": shapes, "logits": logits, "torch": torch.__version__}, out_path)
    print("darts_network", tuple(logits.shape))


def input_checksum(wl):
    s = 0.0
    for t in list(wl.lower.module.parameters()) + list(wl.upper.module.parameters()) + list(wl.vector):
        s += float(t.double().sum())
    for b in wl.lower.cur_batch:
        if torch.is_tensor(b):
            s += float(b.double().sum())
    return s


def main():
    import betty.hypergradient as ref  # the real thing, read-only
    from betty.hypergradient.neumann import approx_inverse_hvp

    torch.set_num_threads(1)  # deterministic reductions
    todo = [(os.path.join(ROOT, "tests", "golden"), c, f, k) for c, (f, k) in CASES.items()]
    todo += [(os.path.join(ROOT, "tests", "golden_cpu"), c, f, k) for c, (f, k) in CPU_ONLY_CASES.items()]
    only = set(sys.argv[1:])
    make_sama(os.path.join(ROOT, "tests", "golden", "sama"), only)
    if not only or "darts_network" in only:
        make_darts_network(os.path.join(ROOT, "tests", "golden", "models", "darts_network.pt"))
    for out_dir, case, factory, kw in todo:
        if only and case not in only:
            continue
        os.makedirs(out_dir, exist_ok=True)
        wl = W.FACTORIES[factory](device="cpu", **kw)
        method = wl.lower.config.type
        rec = {"factory": factory, "kwargs": kw, "method": method, "checksum": input_checksum(wl),
               "torch": torch.__version__}
        fn = ref.jvp_fn_mapping[method]
        hg = fn(wl.vector, wl.lower, wl.upper, False)
        rec["hypergrad"] = [g.detach().clone() for g in hg]
        if method == "neumann":
            loss = wl.lower.training_step_exec(wl.lower.cur_batch)
            g = torch.autograd.grad(loss, wl.lower.trainable_parameters(), create_graph=True)
            x = approx_inverse_hvp(wl.vector, g, wl.lower.trainable_parameters(),
                                   iterations=wl.lower.config.neumann_iterations,
                                   alpha=wl.lower.config.neumann_alpha)
            rec["ihvp"] = [t.detach().clone() for t in x]
        torch.save(rec, os.path.join(out_dir, case + ".pt"))
        n = sum(t.numel() for t in rec["hypergrad"])
        print(f"{case:24s} method={method:8s} |hg|={float(torch.cat([t.reshape(-1) for t in rec['hypergrad']]).norm()):.6e} n={n}")


if __name__ == "__main__":
    main()
