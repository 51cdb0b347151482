#!/usr/bin/env python
"""HVP-iters/sec of the hypergradient K-loop (BASELINE.json metric).

    python bench.py [--gpus N --steps K --warmup W] [--workload NAME] [--impl reference] [--dump-outputs DIR]

One "step" = one full K-loop (K Hessian-vector products + the Neumann/CG vector updates) over one
synthetic batch, inputs resident in HBM; prologue (lower forward + tape) is built once, outside the
timed region, exactly as the metric is defined in SURVEY.md §8(d).  ``e2e`` times the whole plugin
call ``fn(vector, curr, prev, sync)`` with the batch and direction coming from pinned HOST memory and
the hypergradient read back to the host every step.  Under torchrun every rank solves its own local
system on its own batch (the reference's DDP semantics, SURVEY.md §0 item 5): no collective in the
K-loop, one all-reduce of the hypergradient in ``e2e``.

``--impl reference`` times the reference's own CPU autograd path (oracle/_ref, the unmodified reference mirrored by
oracle/fetch_ref.sh; the oracle port if that mirror is missing) on the host cores.  The default run reports the
config the >=60 % roofline target is quoted on (implicit_maml) and carries configs 2 and 5 as `extra` sub-records.

``--dump-outputs DIR`` writes what the last timed step of the headline workload returned (the hypergradient, one
array per parameter tensor) as ``DIR/<workload>.<index>.npy`` in float32; the workloads are seeded, so two builds run
with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

WORKLOADS = {
    # name: (factory, kwargs, method, describe)
    "learning_to_reweight": ("learning_to_reweight", dict(method="cg", batch=4096, K=20), "LeNet-5 3x32x32 B=4096, MWN-weighted CE + 0.05|w|^2, CG K=20, fp32"),
    "learning_to_reweight_b100": ("learning_to_reweight", dict(method="cg", batch=100, K=20), "LeNet-5 B=100 (reference batch), CG K=20, fp32"),
    "implicit_maml": ("implicit_maml", dict(method="neumann", n=800, image="miniimagenet", K=20, alpha=0.01, precision="bf16"), "4-conv mini-ImageNet N=800, CE + 0.5|w-theta|^2, Neumann K=20, bf16 autocast"),
    "implicit_maml_n25": ("implicit_maml", dict(method="neumann", n=25, image="miniimagenet", K=20, alpha=0.01, precision="bf16"), "4-conv mini-ImageNet N=25, Neumann K=20, bf16 autocast"),
    "bert_data_reweighting": ("bert_data_reweighting", dict(method="cg", batch=16, seq=50, K=10, precision="bf16"), "RoBERTa-base B=16xL=50, MWN-weighted CE + 5e-3|w|^2, CG K=10, bf16 autocast"),
    "logistic_regression_hpo": ("logistic_regression_hpo", dict(method="neumann", K=5), "20-dim logistic HPO, Neumann K=5, fp32"),
    "neural_architecture_search": ("neural_architecture_search_full", dict(batch=64, c=16, layers=8), "DARTS search network Network(16,10,8) + Architecture(4), P=1,930,618 in 1,399 tensors, B=64, finite-difference hypergradient (1 call = 1 iter-equivalent), fp32"),
    "neural_architecture_search_lite": ("neural_architecture_search", dict(batch=64, c=16, cells=4), "compact DARTS-style supernet c16 x 4 cells B=64, finite difference, fp32 (round-1 stand-in)"),
}
DEFAULT = "implicit_maml"      # the config BASELINE.json's ">=60 % HBM roofline on the Neumann K=20 path" is quoted on
EXTRA = ("learning_to_reweight", "bert_data_reweighting", "neural_architecture_search")   # sub-records of the default run
L2_BYTES = 50 * 1024 * 1024      # H100 SXM
DUMP_MAX_BYTES = 64 * 1024 * 1024


# -------------------------------------------------------------------------------------------------
class ClockSampler(threading.Thread):
    """Samples SM clock and throttle reasons through NVML while the timed region runs."""

    def __init__(self, index, period=0.05):
        super().__init__(daemon=True)
        self.index, self.period = index, period
        self.samples, self.reasons, self.power = [], set(), []
        self.stop_flag = threading.Event()
        self.max_mhz = None
        try:
            import pynvml as nv

            nv.nvmlInit()
            self.nv = nv
            self.h = nv.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = nv.nvmlDeviceGetMaxClockInfo(self.h, nv.NVML_CLOCK_SM)
        except Exception as e:  # pragma: no cover
            self.nv = None
            self.err = repr(e)

    _NAMES = {0x1: "gpu_idle", 0x2: "applications_clocks_setting", 0x4: "sw_power_cap", 0x8: "hw_slowdown",
              0x10: "sync_boost", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown",
              0x80: "hw_power_brake_slowdown", 0x100: "display_clock_setting"}

    def run(self):
        if self.nv is None:
            return
        nv = self.nv
        while not self.stop_flag.is_set():
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
                self.power.append(nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0)
                try:
                    r = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                for bit, name in self._NAMES.items():
                    if r & bit and name != "gpu_idle":
                        self.reasons.add(name)
            except Exception:
                pass
            time.sleep(self.period)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.max_mhz, "reasons": ["nvml_unavailable"]}
        s = sorted(self.samples)
        return {"sm_mhz": s[len(s) // 2], "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(s), "power_w_max": max(self.power) if self.power else None}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("hbm_gbs", 3350.0), d.get("bf16_tflops_sustained", 989.0), "measured"
    return 3350.0, 989.0, "datasheet"      # H100 SXM: HBM3 bandwidth, dense BF16


def flush_l2(buf):
    buf.add_(1.0)


# -------------------------------------------------------------------------------------------------
def dump_outputs(out_dir, name, tensors):
    """Write the arrays a caller of the timed path receives as float32 .npy files, at most DUMP_MAX_BYTES in all: above
    that, every tensor contributes the same fraction of its elements, picked by a fixed seed."""
    import numpy as np

    os.makedirs(out_dir, exist_ok=True)
    flat = [t.detach().reshape(-1).float().cpu() for t in tensors]
    total = sum(f.numel() for f in flat)
    keep = min(1.0, DUMP_MAX_BYTES / 4 / max(total, 1))
    gen = torch.Generator().manual_seed(0)
    for i, f in enumerate(flat):
        if keep < 1.0:
            idx = torch.randperm(f.numel(), generator=gen)[: max(1, int(f.numel() * keep))].sort().values
            f = f[idx]
        np.save(os.path.join(out_dir, f"{name}.{i:03d}.npy"), f.numpy().astype(np.float32))


def build_workload(name, device, seed=0):
    from betty_b200 import workloads as W

    factory, kw, desc = WORKLOADS[name]
    wl = W.FACTORIES[factory](device=device, seed=seed, **kw)
    return wl, kw, desc


def reference_kloop_rate(workload, budget_s, max_iters=None, calibrate=True):
    """HVP-iters/s of the reference's CPU autograd path on this host (bounded sample of `workload`).

    With ``oracle/_ref`` present (the unmodified reference, mirrored by oracle/fetch_ref.sh) the K-loop that is timed
    is the reference's own code -- ``betty.hypergradient.neumann.approx_inverse_hvp``, the loop inside
    ``betty.hypergradient.cg.cg`` (timed by difference, see oracle/reference.py), ``betty.hypergradient.darts.darts``
    -- driven through the duck-typed problems of betty_b200.shim (``kind: "reference"``); otherwise the oracle port
    (``kind: "port"``)."""
    from oracle import ref_port
    from oracle import reference as R

    wl, kw, desc = build_workload(workload, "cpu")
    method = wl.lower.config.type
    K = kw.get("K", 1)
    cores = min(os.cpu_count() or 1, 32)
    kind = "reference" if R.available() else "port"
    t_all = time.perf_counter()
    if method == "darts":
        torch.set_num_threads(cores)
        fn = (lambda: R.kloop_seconds(wl, "darts", 1)["kloop_s"]) if kind == "reference" else None
        if fn is None:
            def fn():
                t0 = time.perf_counter()
                ref_port.darts(wl.vector, wl.lower, wl.upper, False)
                return time.perf_counter() - t0
        fn()                                                   # warm-up
        n, spent = 0, 0.0
        while (n < 1 or spent < budget_s) and n < 20:
            spent += fn()
            n += 1
        return {"value": n / spent, "unit": "HVP-iters/s", "cores": cores, "kind": kind, "iters": n, "K": 1,
                "seconds": spent, "desc": desc,
                "sample": f"{n} finite-difference call(s) of the full-size workload ({spent:.1f} s), fp32, torch {torch.__version__} CPU autograd"}
    if calibrate:
        in_grad = ref_port.lower_gradient(wl.lower)
        hvp = ref_port.make_hvp(in_grad, wl.lower.trainable_parameters())
        cores = best_thread_count(hvp, list(wl.vector), budget_s=min(40.0, budget_s))
        del in_grad, hvp
    else:
        torch.set_num_threads(min(cores, 16))
        cores = min(cores, 16)
    cap = K if max_iters is None else min(K, max_iters)

    def run(k):
        if kind == "reference":
            return R.kloop_seconds(wl, method, k)["kloop_s"]
        ig = ref_port.lower_gradient(wl.lower)
        h = ref_port.make_hvp(ig, wl.lower.trainable_parameters())
        t0 = time.perf_counter()
        if method == "neumann":
            ref_port.neumann_series(list(wl.vector), h, k, wl.lower.config.neumann_alpha)
        else:
            ref_port.cg_solve(list(wl.vector), h, k, wl.lower.config.cg_alpha)
        return time.perf_counter() - t0

    t1 = run(1)                                                # also the warm-up
    k = int(max(1, min(cap, round(0.5 * budget_s / max(t1, 1e-6)))))
    iters, spent = 0, 0.0
    while iters == 0 or (spent + k * t1 < budget_s and iters < 4 * cap):
        spent += run(k)
        iters += k
    return {"value": iters / spent, "unit": "HVP-iters/s", "cores": cores, "kind": kind, "iters": iters, "K": K,
            "seconds": spent, "desc": desc, "k_per_step": k,
            "sample": f"{iters} K-loop iteration(s) ({spent:.1f} s; {k} per step of K={K}) of the full-size workload, fp32, torch {torch.__version__} CPU autograd, total {time.perf_counter() - t_all:.0f} s incl. prologue"}


def run_reference(args):
    """--impl reference: the reference's own CPU implementation of the path on this box's host cores."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    t0 = time.perf_counter()
    rec = reference_kloop_rate(args.workload, budget_s=args.ref_budget_s)
    wall = time.perf_counter() - t0
    steps = max(1, rec["iters"] // max(1, rec.get("k_per_step", 1)))
    line = {
        "impl": "reference", "metric": "HVP-iters/sec", "value": rec["value"], "unit": "HVP-iters/s",
        "n_gpus": args.gpus, "steps": steps, "warmup": 1, "ms_per_step": 1e3 * rec["seconds"] / steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": args.workload, "describe": rec["desc"], "K": rec["K"], "wall_s": wall},
        "cpu_baseline": {"value": rec["value"], "unit": "HVP-iters/s", "cores": rec["cores"], "kind": rec["kind"],
                         "sample": rec["sample"]},
        "e2e": {"value": rec["value"], "unit": "HVP-iters/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))
    return 0


# -------------------------------------------------------------------------------------------------
def measure(name, args, dev, dist, world, rank, local, steps, e2e_steps, with_cpu, dump_dir=None):
    """One workload: K-loop rate (inputs resident), e2e through the plugin call from pinned host buffers, roofline."""
    import gc

    from betty_b200 import _native as N
    from betty_b200 import engine as E
    from betty_b200 import hypergradient as H

    wl, kw, desc = build_workload(name, dev, seed=rank)
    kw = dict(kw)
    method = wl.lower.config.type
    K = kw.get("K", 1)

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- prologue once (outside the timed region) -------------------------------------------
    if method == "darts":
        # finite difference: no K-loop to isolate -- one step = one plugin call (two lower fwd/bwd passes on
        # PyTorch + the K4 kernels), reported as calls/s (SURVEY.md 8d: "1 call = 1 iter-equivalent")
        class _FdCall:
            hvp = None
            layout = type("L", (), {"n_logical": sum(p.numel() for p in wl.lower.parameters())})()

            def solve(self, vec):
                return H.darts(vec, wl.lower, wl.upper, False)

        call = _FdCall()
        K = kw["K"] = 1
    else:
        call = E.HypergradientCall(wl.lower, method)
    flush = torch.zeros(L2_BYTES // 4 * 2, device=dev)  # twice the L2, written between steps

    for _ in range(args.warmup):
        call.solve(wl.vector)
        flush_l2(flush)
    barrier()
    sampler = ClockSampler(local)
    sampler.start()
    launches0 = N.launch_counter
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    barrier()
    t0 = time.perf_counter()
    out = None
    for i in range(steps):
        ev[i][0].record()
        out = call.solve(wl.vector)
        ev[i][1].record()
        flush_l2(flush)
    barrier()
    wall = time.perf_counter() - t0
    sampler.stop_flag.set()
    sampler.join()
    if dump_dir is not None and rank == 0 and out is not None:
        dump_outputs(dump_dir, name, out)
    del out
    step_ms = [a.elapsed_time(b) for a, b in ev]
    dev_ms = sum(step_ms)  # device time of the K steps, L2 flushes excluded
    launches = N.launch_counter - launches0
    t = torch.tensor([dev_ms], device=dev, dtype=torch.float64)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms_max = float(t.item())
    ms_per_step = dev_ms_max / steps
    value = world * K * steps / (dev_ms_max / 1e3)

    # ---- roofline (before e2e: the plan of `call` is still alive) -------------------------------
    hbm, tf, which = measured_peaks()
    roof = None
    if call.hvp is not None and hasattr(call.hvp, "roofline"):
        roof = call.hvp.roofline(hbm_gbs=hbm, which=which)
        from betty_b200.roofline import survey_bytes

        sb = survey_bytes(call.hvp.g, method)
        per_gpu = value / world
        roof["plan"] = roof.pop("iteration")                       # the executed plan's own byte count / node times
        roof["iteration"] = {"alg_bytes": sb["bytes"], "formula": sb["formula"], "A_in": sb["A_in"], "A_out": sb["A_out"],
                             "P": sb["P"], "s_a": sb["s_a"], "iters_per_s_per_gpu": per_gpu,
                             "achieved_GBps": sb["bytes"] * per_gpu / 1e9, "frac": sb["bytes"] * per_gpu / 1e9 / hbm,
                             "hbm_ceiling_iters_per_s": hbm * 1e9 / sb["bytes"],
                             "note": "SURVEY 8(d) bytes x measured K-loop rate (vector kernels K1-K3 included in the time)"}
    elif method == "darts":
        roof = fd_kernel_roofline(wl, dev, hbm, which)
    n_params = call.layout.n_logical
    del call
    gc.collect()

    # ---- e2e: whole plugin call from pinned host buffers -------------------------------------
    host_batch = [b.cpu().pin_memory() if torch.is_tensor(b) else b for b in wl.lower.cur_batch]
    host_vec = [v.cpu().pin_memory() for v in wl.vector]
    h2d = sum(b.numel() * b.element_size() for b in host_batch if torch.is_tensor(b)) + sum(v.numel() * 4 for v in host_vec)
    d2h = 0
    fn = H.jvp_fn_mapping[method]

    def e2e_step():
        nonlocal d2h
        wl.lower.cur_batch = tuple(b.to(dev, non_blocking=True) if torch.is_tensor(b) else b for b in host_batch)
        vec = [v.to(dev, non_blocking=True) for v in host_vec]
        hg = fn(vec, wl.lower, wl.upper, False)
        if dist is not None:
            flat = torch.cat([g.reshape(-1) for g in hg])
            dist.all_reduce(flat, op=dist.ReduceOp.AVG)  # what the upper module's DDP reducer does
            hg = [flat]
        out = [g.cpu() for g in hg]
        d2h = sum(o.numel() * o.element_size() for o in out)
        return out

    for _ in range(2):      # warm-up: allocator pools, cuBLAS/cuDNN handles of the lower forward, plan cache
        e2e_step()
    # Python's cyclic collector: a generation-2 pass over the ~10^6 objects torch / transformers create at import takes
    # tens of ms and would land inside one of the few timed calls.  Collect now and freeze what is alive (the usual
    # serving-process idiom); garbage created by the timed calls themselves is still collected as usual.
    gc.collect()
    gc.freeze()
    barrier()
    launches1 = N.launch_counter
    t1 = time.perf_counter()
    e2e_step_ms = []
    for _ in range(e2e_steps):
        ts = time.perf_counter()
        e2e_step()          # ends with the D2H read of the result: the step's wall time is well defined
        e2e_step_ms.append(round(1e3 * (time.perf_counter() - ts), 3))
    barrier()
    e2e_wall = time.perf_counter() - t1
    gc.unfreeze()
    t = torch.tensor([e2e_wall], device=dev, dtype=torch.float64)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_value = world * K * e2e_steps / float(t.item())

    rec = {
        "value": value, "unit": "HVP-iters/s", "ms_per_step": ms_per_step, "steps": steps,
        "dtype": "f32" if wl.lower.config.precision == "fp32" else "bf16+f32",
        "config": {"workload": name, "describe": desc, "K": K, "method": method, "hvp": args.hvp,
                   "cuda_graph": E.settings.cuda_graph,
                   "l2": f"{2 * L2_BYTES >> 20} MB buffer rewritten between timed steps",
                   "parallelism": f"replicas x{world} (local solve per rank, SURVEY 8e)",
                   "n_params": n_params, "wall_s": wall},
        "clocks": sampler.summary(),
        "e2e": {"value": e2e_value, "unit": "HVP-iters/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "steps": e2e_steps, "step_ms": e2e_step_ms,
                "includes": "H2D batch+v, prologue, K-loop, epilogue, D2H hypergradient",
                "gpu_launches": N.launch_counter - launches1},
        "gpu_launches": launches,
        "roofline": roof,
    }
    del wl, flush, host_batch, host_vec
    gc.collect()
    torch.cuda.empty_cache()
    if with_cpu:
        r = reference_kloop_rate(name, budget_s=args.cpu_budget_s, max_iters=args.ref_iters)
        rec["cpu_baseline"] = {k: r[k] for k in ("value", "unit", "cores", "kind", "sample")}
    return rec


def fd_kernel_roofline(wl, dev, hbm, which):
    """Finite difference: the only kernels of ours are K4 (norm, three parameter sweeps, combine); report the
    parameter sweep `w += eps v` over this workload's own parameter tensors (12 B per element)."""
    from betty_b200 import _native as N
    from betty_b200 import engine as E
    from betty_b200.arena import ChunkTable

    ps = [p.data for p in wl.lower.parameters()]
    vs = [torch.randn_like(p) for p in ps]
    tab = ChunkTable([v.data_ptr() for v in vs], [p.data_ptr() for p in ps], [p.numel() for p in ps], dev, keep=(vs, ps))
    ws = E.Workspace.get(dev)
    s = torch.cuda.current_stream().cuda_stream
    zero = torch.zeros(1, device=dev)
    reps = 20
    for _ in range(3):
        N.call("bb_mt_axpby", tab.ptr, tab.n, 1.0, zero.data_ptr(), 1.0, s)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        N.call("bb_mt_axpby", tab.ptr, tab.n, 1.0, zero.data_ptr(), 1.0, s)   # w += 0 * v: values unchanged
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    n = sum(p.numel() for p in ps)
    ach = 12.0 * n / (ms * 1e-3) / 1e9
    return {"bound": "hbm", "kernel": f"mt_axpby (K4 parameter sweep w += eps v over {len(ps)} tensors, {n} elements; "
            "L2-resident at this size)", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm,
            "traffic": None, "peak_source": which, "kernel_ms": ms, "kernel_alg_bytes": 12 * n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default=None, choices=sorted(WORKLOADS))
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--hvp", default="native", choices=["native", "autograd"])
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extra", action="store_true", help="skip the sub-records of the other headline configs")
    ap.add_argument("--ref-iters", type=int, default=4, help="cap on K-loop iterations per CPU-baseline step")
    ap.add_argument("--ref-budget-s", type=float, default=60.0, help="--impl reference: CPU seconds of timed K-loop")
    ap.add_argument("--cpu-budget-s", type=float, default=12.0, help="cpu_baseline leg: CPU seconds of timed K-loop")
    ap.add_argument("--e2e-steps", type=int, default=5)
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the headline workload's last timed output as DIR/<workload>.<i>.npy (float32)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else args.warmup
    extras = [] if (args.workload is not None or args.no_extra) else list(EXTRA)
    args.workload = args.workload or DEFAULT

    if args.impl == "reference":
        return run_reference(args)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (no CPU fallback); use --impl reference for the CPU arm")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=dev)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False

    from betty_b200 import engine as E

    E.settings.hvp = args.hvp
    E.settings.cuda_graph = not args.no_graph
    with_cpu = rank == 0 and world == 1 and not args.no_cpu_baseline
    main_rec = measure(args.workload, args, dev, dist, world, rank, local, args.steps, args.e2e_steps, with_cpu,
                       dump_dir=args.dump_outputs)
    line = {
        "metric": "HVP-iters/sec", "value": main_rec["value"], "unit": "HVP-iters/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": main_rec["ms_per_step"], "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": main_rec["dtype"], "data": "synthetic",
        "config": main_rec["config"], "clocks": main_rec["clocks"], "e2e": main_rec["e2e"],
        "gpu_launches": main_rec["gpu_launches"] + main_rec["e2e"]["gpu_launches"], "roofline": main_rec["roofline"],
    }
    if "cpu_baseline" in main_rec:
        line["cpu_baseline"] = main_rec["cpu_baseline"]
    if extras:
        # the other headline configs of BASELINE.json (LeNet CG K=20 fp32; RoBERTa-base CG K=10 bf16; DARTS finite difference) as
        # sub-records of the same line: same timing rules, fewer steps
        line["extra"] = {}
        for name in extras:
            try:
                r = measure(name, args, dev, dist, world, rank, local, max(3, args.steps // 2), 3, with_cpu)
            except Exception as exc:      # a sub-record must never cost the headline line
                line["extra"][name] = {"error": f"{type(exc).__name__}: {exc}"[:400]}
                continue
            line["extra"][name] = r
            line["gpu_launches"] += r["gpu_launches"] + r["e2e"]["gpu_launches"]
    if rank == 0:
        print(json.dumps(line))
    if dist is not None:
        dist.destroy_process_group()
    return 0


def best_thread_count(hvp, v, budget_s: float = 40.0):
    """torch's CPU autograd is not monotone in thread count on many-core hosts (128 threads were 4x slower than 16
    on the pool's boxes): time one H.v at 8 / 16 / 32 threads (capped by the core count), stop as soon as more
    threads get slower or the calibration budget is spent, keep the fastest."""
    cores = os.cpu_count() or 1
    cands = sorted({min(cores, 8), min(cores, 16), min(cores, 32)})
    t_start = time.perf_counter()
    best, best_t = cands[0], None
    for i, nt in enumerate(cands):
        torch.set_num_threads(nt)
        if i == 0:
            hvp(v)          # warm-up (allocator, oneDNN primitive caches)
        t0 = time.perf_counter()
        hvp(v)
        dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best, best_t = nt, dt
        elif dt > 1.1 * best_t:
            break
        if time.perf_counter() - t_start > budget_s:
            break
    torch.set_num_threads(best)
    return best


if __name__ == "__main__":
    sys.exit(main())
