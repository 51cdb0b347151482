"""Time the halo convolution / weight-gradient kernels alone at the three shapes the implicit-MAML benchmark runs them
(N=800 at 42x42, 21x21 and 10x10; CUDA events on the launch stream, L2 flushed between launches by rotating over
operand sets larger than L2).  TF/s are given from useful FLOPs (N*H*W pixels) and from padded FLOPs (every 128-row
tile of the padded layout, which is what the tensor cores execute), with the useful rate as a fraction of the H100
SXM data-sheet 989 dense BF16 TFLOP/s.  With BB200_LIB=<path> the same run times another build of the library.
    python tools/halo_bench.py [N H W]"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from betty_b200 import _native as N

PEAK_TFLOPS = 989.0


def bench_shape(n, h, w):
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    nset = 3
    acts = [[torch.randn(n, h + 2, w + 2, 64, generator=g, device=dev).bfloat16() for _ in range(2)] for _ in range(nset)]
    wms = [(0.1 * torch.randn(64, 9, 64, generator=g, device=dev)).bfloat16() for _ in range(2)]
    outp = [torch.empty(n, h + 2, w + 2, 64, dtype=torch.bfloat16, device=dev) for _ in range(nset)]
    outf = torch.zeros(n, 64, h, w, device=dev)
    wg = torch.zeros(64, 64, 3, 3, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def timed(fn, reps=20):
        for i in range(3):
            fn(i % nset)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
        ev[0].record()
        for i in range(reps):
            fn(i % nset)
            ev[i + 1].record()
        torch.cuda.synchronize()
        ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
        return ts[len(ts) // 2] * 1e3

    def conv_nhwc(np_):
        return lambda i: N.call("bb_conv_halo_bf16_nhwc", n, h, w, np_, acts[i][0].data_ptr(), acts[i][1].data_ptr() if np_ > 1 else 0,
                                wms[0].data_ptr(), wms[1].data_ptr() if np_ > 1 else 0, 0, outp[i].data_ptr(), 0, st)

    def conv_f32(np_):
        return lambda i: N.call("bb_conv_halo_bf16", n, h, w, np_, acts[i][0].data_ptr(), acts[i][1].data_ptr() if np_ > 1 else 0,
                                wms[0].data_ptr(), wms[1].data_ptr() if np_ > 1 else 0, 1, outf.data_ptr(), 0, 0, st)

    def wgrad(np_):
        return lambda i: N.call("bb_wgrad_halo_bf16", n, h, w, np_, acts[i][0].data_ptr(), acts[i][1].data_ptr() if np_ > 1 else 0,
                                acts[(i + 1) % nset][0].data_ptr(), acts[(i + 1) % nset][1].data_ptr() if np_ > 1 else 0,
                                wg.data_ptr(), st)

    per_px = 2.0 * 64 * 64 * 9
    useful = per_px * n * h * w
    padded = per_px * -(-n * (h + 2) * (w + 2) // 128) * 128
    print(f"shape N={n} H={h} W={w}")
    runs = [("conv->nhwc bf16, 2 pairs", conv_nhwc(2), 2), ("conv->nhwc bf16, 1 pair", conv_nhwc(1), 1),
            ("conv->nchw f32,  2 pairs", conv_f32(2), 2), ("conv->nchw f32,  1 pair", conv_f32(1), 1),
            ("wgrad, 2 pairs", wgrad(2), 2)]
    for name, fn, np_ in runs:
        us = timed(fn)
        tf = np_ * useful / us * 1e-6
        print(f"  {name:26s} {us:8.1f} us   {tf:6.1f} TF/s useful ({tf / PEAK_TFLOPS:5.1%} of {PEAK_TFLOPS:.0f})"
              f"   {np_ * padded / us * 1e-6:6.1f} TF/s padded")
    del acts, outp, outf
    torch.cuda.empty_cache()


def main():
    print(f"device: {torch.cuda.get_device_name()}   library: {os.environ.get('BB200_LIB', N.LIB_PATH)}")
    shapes = [tuple(int(a) for a in sys.argv[1:4])] if len(sys.argv) >= 4 else [(800, 42, 42), (800, 21, 21), (800, 10, 10)]
    for n, h, w in shapes:
        bench_shape(n, h, w)


if __name__ == "__main__":
    main()
