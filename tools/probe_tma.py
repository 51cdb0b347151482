"""GPU probe of the TMA-fed wgmma GEMM (csrc/gemm_tma.cu): error vs a bf16-rounded fp64 matmul for every operand
layout, then throughput on large shapes next to the software-staged kernel.  Usage: python tools/probe_tma.py"""
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from betty_b200 import _native as N
from betty_b200.arena import stream_ptr


def operands(M, Nn, K, a_dt, b_dt, a_trans, b_trans, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).cuda()
    B = torch.randn(K, Nn, generator=g).cuda()
    C0 = torch.randn(M, Nn, generator=g).cuda()
    A_mem = A.t().contiguous().t() if a_trans else A.contiguous()
    B_mem = B.contiguous() if b_trans else B.t().contiguous().t()
    if a_dt == 1:
        A_mem = A.to(torch.bfloat16).t().contiguous().t() if a_trans else A.to(torch.bfloat16).contiguous()
    if b_dt == 1:
        B_mem = B.to(torch.bfloat16).contiguous() if b_trans else B.to(torch.bfloat16).t().contiguous().t()
    return A, B, C0, A_mem, B_mem


def call(entry, M, Nn, K, A_mem, a_dt, B_mem, b_dt, C, beta, scratch):
    args = [M, Nn, K, A_mem.data_ptr(), a_dt, A_mem.stride(0), A_mem.stride(1), B_mem.data_ptr(), b_dt, B_mem.stride(0),
            B_mem.stride(1), C.data_ptr(), C.stride(0), C.stride(1), beta]
    if entry == "bb_gemm_bf16_tma":
        args += [scratch.data_ptr(), scratch.numel()]
    args.append(stream_ptr())
    return getattr(N.lib(), entry)(*args)


def main():
    scratch = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    shapes = [(128, 128, 64), (128, 128, 256), (256, 384, 192), (200, 300, 100), (800, 768, 768), (768, 3072, 800),
              (65, 64, 64), (128, 128, 4096), (64, 64, 64), (100, 72, 136)]
    layouts = [(0, 1, False, False), (0, 0, True, True), (1, 0, False, True), (0, 1, True, False), (1, 1, False, False),
               (1, 1, True, True)]
    worst = 0.0
    for shape in shapes:
        for lay in layouts:
            for beta in (0, 1):
                M, Nn, K = shape
                a_dt, b_dt, a_tr, b_tr = lay
                A, B, C0, A_mem, B_mem = operands(M, Nn, K, a_dt, b_dt, a_tr, b_tr)
                C = C0.clone()
                rc = call("bb_gemm_bf16_tma", M, Nn, K, A_mem, a_dt, B_mem, b_dt, C, beta, scratch)
                torch.cuda.synchronize()
                want = A.to(torch.bfloat16).double() @ B.to(torch.bfloat16).double()
                if beta:
                    want = want + C0.double()
                err = float((C.double() - want).norm() / want.norm())
                worst = max(worst, err)
                flag = "" if err < 2e-5 and rc == 0 else "   <-- BAD"
                print(f"shape={shape} layout={lay} beta={beta} rc={rc} err={err:.2e}{flag}", flush=True)
    print("worst", worst, flush=True)
    for shape in [(800, 768, 768), (800, 3072, 768), (768, 768, 800), (4096, 4096, 4096), (8192, 8192, 1024)]:
        M, Nn, K = shape
        for lay in [(0, 1, False, False), (0, 0, True, True), (1, 1, False, False)]:
            a_dt, b_dt, a_tr, b_tr = lay
            A, B, C0, A_mem, B_mem = operands(M, Nn, K, a_dt, b_dt, a_tr, b_tr)
            C = C0.clone()
            line = f"shape={shape} layout={lay}"
            for entry in ("bb_gemm_bf16_tma", "bb_gemm_bf16_tc"):
                for _ in range(3):
                    call(entry, M, Nn, K, A_mem, a_dt, B_mem, b_dt, C, 0, scratch)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(10):
                    call(entry, M, Nn, K, A_mem, a_dt, B_mem, b_dt, C, 0, scratch)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / 10
                line += f"  {entry[-3:]}: {ms * 1e3:8.1f} us {2 * M * Nn * K / ms / 1e9:7.1f} TF"
            print(line, flush=True)


if __name__ == "__main__":
    main()
