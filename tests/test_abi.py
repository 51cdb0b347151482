"""CPU tests: the C-ABI library loads and exports every symbol include/betty_b200.h declares; the
plugin table mirrors the reference's and fails loudly without CUDA."""
import ctypes
import os
import re
import types

import pytest
import torch

from betty_b200 import _native as N
from betty_b200 import hypergradient as H
from betty_b200 import workloads as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "betty_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(bb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    N.build()
    lib = ctypes.CDLL(N.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/betty_b200.h but not exported"
    assert set(syms) == set(N.EXPORTS), set(syms) ^ set(N.EXPORTS)
    assert b"sm_90a" in N.lib().bb_version()
    assert N.lib().bb_kloop_ws_bytes() >= 512


def test_plugin_table_matches_reference_keys_and_alias():
    assert H.jvp_fn_mapping["finite_diff"] is H.jvp_fn_mapping["darts"]
    for k in ("neumann", "cg", "darts"):
        assert callable(H.jvp_fn_mapping[k])


# the keys of the reference's betty.hypergradient.jvp_fn_mapping (betty/hypergradient/__init__.py:33-37)
REFERENCE_TABLE_KEYS = ("cg", "darts", "neumann", "reinforce", "sama")


def test_install_rebinds_reference_table():
    ref = types.ModuleType("betty.hypergradient")          # stands in for the reference's module: same table keys
    ref.jvp_fn_mapping = {k: object() for k in REFERENCE_TABLE_KEYS}
    saved = dict(ref.jvp_fn_mapping)
    table = H.install(ref)
    assert table is ref.jvp_fn_mapping
    for k in H.jvp_fn_mapping:
        assert ref.jvp_fn_mapping[k] is H.jvp_fn_mapping[k]
    assert set(REFERENCE_TABLE_KEYS) - {"reinforce"} <= set(H.jvp_fn_mapping)
    assert ref.jvp_fn_mapping["reinforce"] is saved["reinforce"]  # untouched (out of scope)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
@pytest.mark.parametrize("method", ["neumann", "cg", "darts"])
def test_no_cpu_fallback(method):
    wl = W.logistic_hpo(method=method)
    with pytest.raises(N.NativeError):
        H.jvp_fn_mapping[method](wl.vector, wl.lower, wl.upper, False)


def test_higher_order_assert_matches_reference():
    wl = W.logistic_hpo(method="neumann")
    wl.lower.paths = [["something"]]
    with pytest.raises(AssertionError):
        H.neumann(wl.vector, wl.lower, wl.upper, False)
