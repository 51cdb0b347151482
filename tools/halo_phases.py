"""Where the time of one conv_halo_kernel tile goes, at the three shapes the implicit-MAML benchmark runs it (N=800 at
42x42, 21x21 and 10x10), with two operand pairs and with one.

A separate instantiation of the kernel (bb_conv_halo_phases; the plan and the K-loop never launch it) has thread 0 of
the consumer warpgroup that owns a tile (local tile lt of a CTA -> warpgroup lt & 1) read clock64() at fixed points of
its tile loop.  The library names the points (bb_conv_halo_phase_names) in program order; each phase below is the time
from one recorded point to the next one of the same tile, per warpgroup: the wait for the issue turn (top -> turn), the
band waits, the issue, the drain and the epilogue.  `period` is the time from one tile's `turn` (its first wgmma) to
the next tile's, i.e. the cost of a tile to the tensor pipe.  Cycles become nanoseconds at the SM clock the same run
shows (clock64 over globaltimer, per CTA).  Each warpgroup's first tile is left out (it waits for the resident
weights).  The stamps cost a few instructions per point, so the phase variant runs slightly slower than the default
one; compare it with itself across builds.
With BB200_LIB=<path> the same run measures another build of the library.
    python tools/halo_phases.py [N H W] [--reps R]"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from betty_b200 import _native as N  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=30)
        return r.stdout.decode().strip().splitlines()[torch.cuda.current_device()]
    except Exception as exc:
        return f"{torch.cuda.get_device_name()} (power limit not read: {exc})"


def phase_names():
    buf = ctypes.create_string_buffer(512)
    N.call("bb_conv_halo_phase_names", buf, len(buf))
    return buf.value.decode().split(",")


def measure(n, h, w, npairs, reps):
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    nset = 3   # rotate over operand sets larger than L2, as tools/halo_bench.py does
    acts = [[torch.randn(n, h + 2, w + 2, 64, generator=g, device=dev).bfloat16() for _ in range(2)] for _ in range(nset)]
    wms = [(0.1 * torch.randn(64, 9, 64, generator=g, device=dev)).bfloat16() for _ in range(2)]
    outp = torch.empty(n, h + 2, w + 2, 64, dtype=torch.bfloat16, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    layout = (ctypes.c_int * 3)()

    def run(i, stamps_ptr):
        a = acts[i % nset]
        N.call("bb_conv_halo_phases", n, h, w, npairs, a[0].data_ptr(), a[1].data_ptr() if npairs > 1 else 0,
               wms[0].data_ptr(), wms[1].data_ptr() if npairs > 1 else 0, 0, outp.data_ptr(), 0, stamps_ptr, layout, st)

    run(0, None)
    grid, slots, nst = layout[0], layout[1], layout[2]
    stamps = torch.zeros(4 * grid + grid * slots * 2 * nst, dtype=torch.int64, device=dev)
    samples = []
    for i in range(3 + reps):
        stamps.zero_()
        run(i, stamps.data_ptr())
        torch.cuda.synchronize()
        if i >= 3:
            samples.append(stamps.cpu().numpy().astype(np.float64))
    del acts
    torch.cuda.empty_cache()
    return grid, slots, nst, samples


def summarize(grid, slots, nst, samples, names):
    phases, periods, ghz, kernel_us = {}, [], [], []
    order = []
    turn = names.index("turn")
    for s in samples:
        hdr = s[:4 * grid].reshape(grid, 4)
        ratio = (hdr[:, 3] - hdr[:, 1]) / np.maximum(hdr[:, 2] - hdr[:, 0], 1)   # cycles per ns
        ghz.append(np.median(ratio))
        kernel_us.append((hdr[:, 2].max() - hdr[:, 0].min()) * 1e-3)
        cyc_ns = np.median(ratio)
        v = s[4 * grid:].reshape(grid, slots, 2, nst)
        for c in range(grid):
            prev_turn = None
            for sl in range(slots):
                wg = sl & 1
                row = v[c, sl, wg]
                ks = [k for k in range(nst) if row[k] != 0]
                if not ks:
                    continue
                if sl > 1:
                    for a, b in zip(ks, ks[1:]):
                        key = f"{names[a]} -> {names[b]}"
                        if key not in phases:
                            phases[key] = ([], [])
                            order.append(key)
                        phases[key][wg].append((row[b] - row[a]) / cyc_ns)
                    periods.append((row[turn] - prev_turn) / cyc_ns)
                prev_turn = row[turn]
    return order, phases, periods, float(np.median(ghz)), float(np.median(kernel_us))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("shape", nargs="*", type=int, help="N H W (default: the benchmark's three shapes)")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("halo_phases.py needs a CUDA device")
    print(f"card: {card()}   library: {os.environ.get('BB200_LIB', N.LIB_PATH)}")
    names = phase_names()
    print(f"stamp points: {', '.join(names)}")
    shapes = [tuple(args.shape)] if len(args.shape) == 3 else [(800, 42, 42), (800, 21, 21), (800, 10, 10)]
    for n, h, w in shapes:
        for npairs in (2, 1):
            grid, slots, nst, samples = measure(n, h, w, npairs, args.reps)
            order, phases, periods, ghz, kus = summarize(grid, slots, nst, samples, names)
            print(f"\nN={n} {h}x{w}, {npairs} pair{'s' if npairs > 1 else ''}: {grid} CTAs, up to {slots - 1} tiles each, "
                  f"phase kernel {kus:.1f} us, SM clock {ghz * 1e3:.0f} MHz")
            print(f"  {'phase':34s} {'wg0 median':>10s} {'p90':>7s} {'wg1 median':>10s} {'p90':>7s}   (ns)")
            for key in order:
                cols = []
                for x in phases[key]:
                    cols += [np.median(x), np.percentile(x, 90)] if x else [np.nan, np.nan]
                print(f"  {key:34s} {cols[0]:10.0f} {cols[1]:7.0f} {cols[2]:10.0f} {cols[3]:7.0f}")
            x = np.asarray(periods)
            if x.size:
                print(f"  {'period (turn to next turn)':34s} {np.median(x):10.0f} {np.percentile(x, 90):7.0f}")


if __name__ == "__main__":
    main()
