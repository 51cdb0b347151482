"""Per-kernel device time of the benchmark's headline K-loop (implicit_maml: 4-conv mini-ImageNet, N=800, Neumann K=20,
bf16), built the way bench.py builds it.

    python tools/kloop_kernels.py [--steps S] [--out DIR]

1. Times S solves with the K-loop captured as a CUDA graph (the benchmark's setting, profiler off): ms per iteration.
2. Profiles S more solves under torch.profiler with CUDA activities and writes the trace to DIR.  If the kernels
   launched by graph replays do not show in the trace, the profiled run uses engine.settings.cuda_graph = False.
3. Prints, per kernel name, the launches and time per iteration and the share of the summed kernel time, the two
   halo kernels' share together, and the weight gradient's TF/s from FLOPs computed from the shapes (useful pixels and
   padded 128-row tiles) against the H100 SXM data-sheet 989 dense BF16 TFLOP/s.  The kernel sum is compared with the
   graph-on iteration time.
The card's name, power limit and maximum SM clock are read in the same run."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from betty_b200 import engine as E  # noqa: E402

PEAK_TFLOPS = 989.0
HALO = ("conv_halo_kernel", "wgrad_halo_kernel")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30)
        return r.stdout.decode().strip().splitlines()[torch.cuda.current_device()]
    except Exception as exc:  # the numbers below still stand; say where the card name is missing
        return f"{torch.cuda.get_device_name()} (power limit not read: {exc})"


def halo_flops(n, hw=(42, 21, 10)):
    """FLOPs per K-loop iteration of the weight gradient: blocks 2-4 (42x42, 21x21, 10x10) each run one two-pair
    wgrad_halo_kernel, so the launch count identifies the shapes.  conv_halo_kernel runs with one and with two pairs at
    shapes the launch count does not identify; tools/halo_bench.py gives its rate per shape."""
    per_px = 2.0 * 64 * 64 * 9 * 2
    useful = sum(per_px * n * h * h for h in hw)
    padded = sum(per_px * -(-n * (h + 2) * (h + 2) // 128) * 128 for h in hw)
    return {"wgrad_halo_kernel": (useful, padded, len(hw))}


def short(name):
    name = re.sub(r"^void ", "", name).replace("(anonymous namespace)::", "")
    return name.split("(")[0][:80]


def kernel_table(trace_path):
    ev = json.load(open(trace_path))["traceEvents"]
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in ev:
        if e.get("cat") == "kernel":
            k = short(e["name"])
            tot[k] += e["dur"] * 1e-3
            cnt[k] += 1
    return tot, cnt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: a new temporary directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kloop_kernels.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    args.out = args.out or tempfile.mkdtemp(prefix="kloop_kernels_")
    os.makedirs(args.out, exist_ok=True)
    print(f"card: {card()}   library: {os.environ.get('BB200_LIB', 'in-tree')}")

    wl, kw, desc = bench.build_workload(bench.DEFAULT, dev)
    K, n = kw["K"], kw["n"]

    def make_call(graph):
        E.settings.cuda_graph = graph
        call = E.HypergradientCall(wl.lower, wl.lower.config.type)
        for _ in range(args.warmup):
            call.solve(wl.vector)
        torch.cuda.synchronize()
        return call

    call = make_call(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        call.solve(wl.vector)
    e1.record()
    torch.cuda.synchronize()
    iter_ms = e0.elapsed_time(e1) / (args.steps * K)
    print(f"{desc}\ngraph on, profiler off: {iter_ms:.3f} ms per iteration ({1e3 / iter_ms:.1f} it/s)")

    def profile(call, tag):
        from torch.profiler import ProfilerActivity, profile as prof_ctx

        with prof_ctx(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                call.solve(wl.vector)
            torch.cuda.synchronize()
        path = os.path.join(args.out, f"kloop_kernels_{tag}.pt.trace.json")
        prof.export_chrome_trace(path)
        print(f"trace: {path}")
        return kernel_table(path)

    tot, cnt = profile(call, "graph")
    mode = "graph on"
    if not any(h in k for k in tot for h in HALO):
        call.release()
        del call
        call = make_call(False)
        tot, cnt = profile(call, "nograph")
        mode = "graph off (graph replays did not show in the trace)"
    iters = args.steps * K
    ksum = sum(tot.values()) / iters
    print(f"profiled {args.steps} solves x K={K}, {mode}: kernel sum {ksum:.3f} ms per iteration = "
          f"{ksum / iter_ms:.1%} of the graph-on iteration time")
    print(f"\n| kernel | launches/iter | ms/iter | share |\n|---|---|---|---|")
    for k, t in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"| `{k}` | {cnt[k] / iters:.2f} | {t / iters:.4f} | {t / iters / ksum:.1%} |")
    fl = halo_flops(n)
    print("\n| halo kernel | ms/iter | share | TF/s useful | of 989 | TF/s padded |\n|---|---|---|---|---|---|")
    share = 0.0
    for h in HALO:
        t = sum(v for k, v in tot.items() if h in k) / iters
        share += t / ksum
        launches = sum(v for k, v in cnt.items() if h in k) / iters
        if h in fl and launches == fl[h][2]:
            u, p, _ = fl[h]
            print(f"| `{h}` | {t:.4f} | {t / ksum:.1%} | {u / t * 1e-9:.1f} | {u / t * 1e-9 / PEAK_TFLOPS:.1%} | "
                  f"{p / t * 1e-9:.1f} |")
        else:
            print(f"| `{h}` | {t:.4f} | {t / ksum:.1%} | see halo_bench.py | | |")
    print(f"\nhalo kernels together: {share:.1%} of the summed kernel time")


if __name__ == "__main__":
    main()
