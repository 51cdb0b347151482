"""Neumann (K=20, alpha=0.01) and CG (K=10) hypergradients through the DARTS search network Network(16, 10, 8) +
Architecture(4) at B=64: the native engine against the reference's own plugin on the same GPU.

Per method, one JSON line: K-loop iterations per second (from the time of a call at 2K minus a call at K, so prologue
and epilogue cancel), whole calls per second at K, the same two rates of the reference's plugin, peak device memory of
an engine call, kernel launches per K-loop iteration, and the card's name and power limit read in the same run.
``--profile`` instead traces one engine call with torch.profiler and reports the depthwise kernels' share of the GPU
time (a separate run: tracing slows the host)."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from betty_b200 import _native as N          # noqa: E402
from betty_b200 import hypergradient as H     # noqa: E402
from betty_b200 import workloads as W         # noqa: E402
from betty_b200 import engine as E            # noqa: E402
from betty_b200.trace import op_tensors        # noqa: E402

CONFIGS = {"neumann": dict(K=20, alpha=0.01), "cg": dict(K=10, alpha=1.0)}


def card():
    """Name and power limit of the device this process runs on (nvidia-smi addressed by PCI bus id, which does not
    depend on CUDA_VISIBLE_DEVICES)."""
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    out = subprocess.run(["nvidia-smi", f"--id={bus}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    return out or torch.cuda.get_device_name()


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def memory(plan, tape):
    """Bytes of what an engine call keeps on the device: the plan's tangent / adjoint / adjoint-tangent arenas, its
    constants and scratch, and the recorded forward's tensors (bases every rule reads)."""
    seen, tape_b = set(), 0
    for op in tape.ops:
        for t in op_tensors(op):
            if t.is_cuda:
                st = t.untyped_storage()
                if st.data_ptr() not in seen:
                    seen.add(st.data_ptr())
                    tape_b += st.nbytes()
    consts = sum(t.numel() * t.element_size() for t in plan._keep)
    mulc = sum(1 for n in plan.g.nodes if n.op == "mulc")
    return {"arenas_GB": round(plan.bytes_buffers / 1e9, 3), "constants_GB": round(consts / 1e9, 3),
            "mulc_nodes": mulc, "tape_GB": round(tape_b / 1e9, 3), "root_values": plan.g.stats.get("values")}


def set_k(wl, k):
    cfg = wl.lower.config
    cfg.neumann_iterations = cfg.cg_iterations = k


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def rates(wl, method, fn, K, reps, warmup):
    def call():
        return fn(list(wl.vector), wl.lower, wl.upper, False)

    out = {}
    for k in (K, 2 * K):
        set_k(wl, k)
        for _ in range(warmup):
            call()
        out[k] = timed(call, reps)
        log(f"  {method} K={k}: {out[k] * 1e3:.1f} ms per call")
    set_k(wl, K)
    return {"kloop_it_s": K / max(out[2 * K] - out[K], 1e-9), "call_s": out[K], "calls_s": 1.0 / out[K]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--methods", default="neumann,cg")
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--profile", default=None, help="write a torch.profiler trace here and report kernel shares")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    for method in args.methods.split(","):
        cfg = CONFIGS[method]
        wl = W.darts_search_full(device=dev, batch=args.batch, method=method, K=cfg["K"], alpha=cfg["alpha"])
        engine = H.jvp_fn_mapping[method]
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            for _ in range(args.warmup):
                engine(list(wl.vector), wl.lower, wl.upper, False)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                engine(list(wl.vector), wl.lower, wl.upper, False)
                torch.cuda.synchronize()
            os.makedirs(args.profile, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.profile, f"darts_{method}.pt.trace.json"))
            kern = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
            total = sum(e.self_device_time_total for e in kern)
            dw = sum(e.self_device_time_total for e in kern if "dw_fwd_kernel" in e.key or "dw_bwd_kernel" in e.key)
            top = sorted(kern, key=lambda e: -e.self_device_time_total)[:8]
            print(json.dumps({"method": method, "card": card(), "gpu_us": total, "depthwise_us": dw,
                              "depthwise_share": dw / total if total else None,
                              "top": [(e.key[:80], e.self_device_time_total) for e in top]}), flush=True)
            continue
        E.plan_cache.clear()
        torch.cuda.reset_peak_memory_stats(dev)
        set_k(wl, cfg["K"])
        log(f"{method}: first call (builds the plan)")
        t0 = time.perf_counter()
        engine(list(wl.vector), wl.lower, wl.upper, False)
        torch.cuda.synchronize()
        first_s = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated(dev)
        entry = next(reversed(E.plan_cache.entries.values()))
        mem = memory(entry.plan, entry.plan.tape)
        hits0 = E.plan_cache.hits
        l0 = N.launch_counter
        engine(list(wl.vector), wl.lower, wl.upper, False)
        l1 = N.launch_counter
        set_k(wl, 2 * cfg["K"])
        engine(list(wl.vector), wl.lower, wl.upper, False)
        l2 = N.launch_counter
        set_k(wl, cfg["K"])
        assert E.plan_cache.hits == hits0 + 2, "later calls did not reuse the cached plan"
        res = {"method": method, "batch": args.batch, "K": cfg["K"], "alpha": cfg["alpha"], "card": card(),
               "first_call_s": round(first_s, 3),
               "engine": rates(wl, method, engine, cfg["K"], args.reps, args.warmup),
               "peak_mem_GB": round(peak / 1e9, 3), "memory": mem,
               "launches_per_iter": ((l2 - l1) - (l1 - l0)) / cfg["K"]}
        log(json.dumps(res))
        if not args.no_reference:
            from oracle import reference as R

            R.load()
            ref_fn = getattr(importlib.import_module(f"betty.hypergradient.{method}"), method)
            E.plan_cache.clear()
            torch.cuda.empty_cache()
            res["reference"] = rates(wl, method, ref_fn, cfg["K"], max(2, args.reps // 2), 1)
            res["speedup_kloop"] = res["engine"]["kloop_it_s"] / res["reference"]["kloop_it_s"]
            res["speedup_call"] = res["engine"]["calls_s"] / res["reference"]["calls_s"]
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
