"""Drop-in replacements for ``betty.hypergradient.{neumann, cg, darts, sama}`` (+ the ``finite_diff`` alias
named by BASELINE.json; the reference calls the same algorithm ``darts``, SURVEY.md §0 item 1).

``install()`` rebinds the reference's plugin table in place, so ``Engine`` / ``ImplicitProblem`` and
the ``Config(type=...)`` selector are used unchanged (reference betty/hypergradient/__init__.py:13-19).
"""
from .cg import cg
from .cg_global import cg_global
from .darts import darts
from .neumann import neumann
from .sama import sama

finite_diff = darts

# "cg_global" is an ADDITION to the reference's table (global-batch CG with rank-sharded vectors, SURVEY.md 8e optional
# variant); the other keys replace the reference's entries one for one
jvp_fn_mapping = {"darts": darts, "finite_diff": darts, "sama": sama, "neumann": neumann, "cg": cg, "cg_global": cg_global}


def get_grads(loss, path, retain_graph, do_sync):
    """Mirror of reference ``betty/hypergradient/__init__.py:22-39`` over this package's table (used
    when the reference is not importable, e.g. on the GPU box)."""
    import torch

    lower = path[1].meta_trainable_parameters()
    jvp = torch.autograd.grad(loss, lower, retain_graph=retain_graph, allow_unused=True)
    jvp = tuple(torch.zeros_like(p) if g is None else g for g, p in zip(jvp, lower))
    for i in range(1, len(path) - 1):
        kind = path[i].config.type
        assert kind in jvp_fn_mapping
        sync = bool(do_sync and i == len(path) - 2)
        jvp = jvp_fn_mapping[kind](jvp, path[i], path[i + 1], sync)
    return jvp


def install(reference_module=None, callers: bool = False):
    """Rebind ``betty.hypergradient.jvp_fn_mapping`` entries to the native engine.  Returns the table.
    ``callers=True`` also rebinds the three caller-side methods of SURVEY.md §8 f4 (``betty_b200.callers``:
    flat ``Problem.synchronize_params``, arena ``ImplicitProblem.cache_states`` / ``recover_states``)."""
    if reference_module is None:
        import betty.hypergradient as reference_module  # the user's installed reference
    reference_module.jvp_fn_mapping.update(jvp_fn_mapping)
    if callers:
        import importlib

        from ..callers import install_callers

        install_callers(importlib.import_module(reference_module.__name__.split(".")[0]))
    return reference_module.jvp_fn_mapping
