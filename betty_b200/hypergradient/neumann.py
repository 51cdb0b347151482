"""``neumann`` plugin -- drop-in for reference ``betty/hypergradient/neumann.py:8-56``."""
from .. import _native as N
from .. import engine as E


def neumann(vector, curr, prev, sync):
    """Best-response-Jacobian x vector by a K-term Neumann series for H^-1 v.

    Same signature, config knobs (``neumann_iterations``, ``neumann_alpha``), return value and
    ``sync`` side effect as the reference.  The K-loop runs as sm_90a kernels.
    """
    assert len(curr.paths) == 0, "neumann method is not supported for higher order MLO!"
    call = E.HypergradientCall(curr, "neumann")
    return call.finish(prev, call.solve(vector), sync)
