"""ctypes binding of ``libbetty_b200.so`` (the C ABI declared in ``include/betty_b200.h``).

There is no CPU fallback: if the shared library has not been built (``python -c "import
__graft_entry__ as g; g.build()"`` or ``make -C betty_b200/csrc``) loading raises, and every compute
entry point raises when no CUDA device is present.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libbetty_b200.so")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")

_lock = threading.Lock()
_lib = None
launch_counter = 0  # kernels launched through this binding (bench.py reports it as gpu_launches)


class NativeError(RuntimeError):
    pass


class MtChunk(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("n", C.c_int32), ("pad", C.c_int32)]


# name -> (argtypes, kernel launches per call or None when data dependent)
_SIGS = {
    "bb_kloop_ws_bytes": ([], 0),
    "bb_neumann_update": ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_int64, C.c_void_p], 1),
    "bb_scale": ([C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p], 1),
    "bb_cg_dots": ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_int, C.c_int64, C.c_void_p, C.c_void_p], 1),
    "bb_cg_init": ([C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p], 1),
    "bb_cg_update_xr": ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p, C.c_void_p], 1),
    "bb_cg_update_p": ([C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p], 1),
    "bb_mt_copy": ([C.c_void_p, C.c_int, C.c_int, C.c_void_p], 1),
    "bb_mt_axpby": ([C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_float, C.c_void_p], 1),
    "bb_mt_sumsq": ([C.c_void_p, C.c_int, C.c_void_p, C.c_void_p], 1),
    "bb_fd_eps": ([C.c_void_p, C.c_double, C.c_void_p], 1),
    "bb_mt_fd_combine": ([C.c_void_p, C.c_int, C.c_void_p, C.c_void_p], 1),
    "bb_mt_adam_precondition": ([C.c_void_p, C.c_int, C.c_void_p], 1),
    "bb_bn_forward_splits": ([C.c_int64, C.c_int], 0),
    "bb_bn_forward": ([C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                       C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p], 3),
    "bb_gemm_bf16_tc": ([C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                         C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p], 1),
    "bb_gemm_bf16_tma": ([C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_int,
                          C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                          C.c_void_p], None),
    "bb_gemm_bf16_tma_ex": ([C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                             C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p], None),
    "bb_plan_set_scratch": ([C.c_void_p, C.c_void_p, C.c_int64], 0),
    "bb_plan_set_persistent": ([C.c_void_p, C.c_void_p, C.c_int64], 0),
    "bb_node_bytes": ([], 0),
    "bb_plan_create": ([C.c_void_p, C.c_int, C.POINTER(C.c_void_p)], 0),
    "bb_plan_destroy": ([C.c_void_p], 0),
    "bb_plan_set_zero_regions": ([C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int], 0),
    "bb_plan_run": ([C.c_void_p, C.c_int, C.c_void_p], None),
    "bb_plan_launch_count": ([C.c_void_p, C.c_int], 0),
    "bb_plan_profile": ([C.c_void_p, C.c_int, C.c_void_p, C.c_void_p], None),
    "bb_plan_hvp": ([C.c_void_p, C.c_void_p], None),
    "bb_plan_hvp_replay": ([C.c_void_p, C.c_void_p], None),
    "bb_plan_set_uniform_shift": ([C.c_void_p, C.c_int, C.c_double], 0),
    "bb_plan_invalidate_constants": ([C.c_void_p], 0),
    "bb_plan_graph_captures": ([C.c_void_p], 0),
    "bb_plan_node_route": ([C.c_void_p, C.c_int, C.c_int], 0),
    "bb_conv_halo_bf16": ([C.c_int] * 4 + [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p], 1),
    "bb_conv_halo_bf16_nhwc": ([C.c_int] * 4 + [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p], 1),
    "bb_conv_halo_phases": ([C.c_int] * 4 + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 5, None),
    "bb_conv_halo_phase_names": ([C.c_char_p, C.c_int], 0),
    "bb_wgrad_halo_bf16": ([C.c_int] * 4 + [C.c_void_p] * 6, 1),
    "bb_convblock_ws_bytes": ([C.c_int] * 9, 0),
    "bb_convblock2_ws_bytes": ([C.c_int] * 9, 0),
    "bb_plan_neumann_loop": ([C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                              C.c_int, C.c_void_p], None),
    "bb_plan_cg_loop": ([C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                         C.c_int64, C.c_void_p, C.c_int, C.c_void_p], None),
}
EXPORTS = tuple(_SIGS) + ("bb_version",)


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(verbose: bool = False) -> str:
    """Compile every ``csrc/*.cu`` for sm_90a into ``libbetty_b200.so`` (in-tree, so it travels to the
    GPU box with the snapshot).  Incremental: one object per source, rebuilt when older than its
    source or any header."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler",
             "-fPIC", "-I", INCLUDE]
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(INCLUDE, "betty_b200.h"))
    newest_hdr = max(os.path.getmtime(h) for h in hdrs)
    objs, procs = [], []
    for src in sources():
        obj = src[:-3] + ".o"
        objs.append(obj)
        if os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(src), newest_hdr):
            continue
        cmd = [nvcc, *flags, "-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise NativeError(f"nvcc failed on {src}:\n{out.decode()}")
    need_link = (not os.path.exists(LIB_PATH)) or any(os.path.getmtime(o) > os.path.getmtime(LIB_PATH) for o in objs)
    if need_link:
        cmd = [nvcc, "-shared", "-o", LIB_PATH, *objs, "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise NativeError("link failed:\n" + r.stdout.decode())
    return LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise NativeError(
                    f"{LIB_PATH} is missing: build the CUDA extension first (python -c 'import __graft_entry__ "
                    "as g; g.build()').  betty_b200 has no CPU or PyTorch fallback.")
            alt = os.environ.get("BB200_LIB")                   # A/B runs of tools/ against another build
            l = C.CDLL(alt or LIB_PATH)
            for name, (argtypes, _) in _SIGS.items():
                if alt and not hasattr(l, name):
                    continue
                fn = getattr(l, name)
                fn.argtypes = argtypes
                fn.restype = C.c_int64 if name.endswith("_bytes") and name != "bb_node_bytes" and name != "bb_kloop_ws_bytes" else C.c_int
            l.bb_version.restype = C.c_char_p
            _lib = l
    return _lib


def call(name: str, *args) -> int:
    """Call a C-ABI entry point, raise on a non-zero status, count the launches."""
    global launch_counter
    fn = getattr(lib(), name)
    rc = fn(*args)
    if rc != 0:
        raise NativeError(f"{name} failed with status {rc}" + (" (cudaError)" if rc > 0 else ""))
    n = _SIGS[name][1]
    if n:
        launch_counter += n
    return rc


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise NativeError("betty_b200 needs a CUDA device (sm_90a); there is no CPU fallback.")
