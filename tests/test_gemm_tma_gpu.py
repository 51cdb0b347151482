"""GPU unit test of the TMA-fed wgmma GEMM (csrc/gemm_tma.cu) through the C ABI: every operand layout (k-fast /
m,n-fast storage, fp32 -> packed or bf16 -> direct tensor maps), ragged edges, split-K, beta.
Reference = matmul of the bf16-rounded operands in fp64."""
import pytest
import torch

from betty_b200 import _native as N
from betty_b200.arena import stream_ptr

pytestmark = pytest.mark.gpu


def _run(M, Nn, K, a_dt, b_dt, a_trans, b_trans, beta, seed=0):
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
    C = C0.clone()
    scratch = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    N.call("bb_gemm_bf16_tma", M, Nn, K, A_mem.data_ptr(), a_dt, A_mem.stride(0), A_mem.stride(1), B_mem.data_ptr(), b_dt,
           B_mem.stride(0), B_mem.stride(1), C.data_ptr(), C.stride(0), C.stride(1), beta, scratch.data_ptr(),
           scratch.numel(), stream_ptr())
    torch.cuda.synchronize()
    want = A.to(torch.bfloat16).double() @ B.to(torch.bfloat16).double()
    if beta:
        want = want + C0.double()
    return float((C.double() - want).norm() / want.norm())


@pytest.mark.parametrize("shape", [(128, 128, 64), (256, 384, 192), (200, 300, 100), (800, 768, 768), (768, 3072, 800),
                                    (65, 64, 64), (128, 128, 4096), (100, 72, 136)])
@pytest.mark.parametrize("layout", [(0, 1, False, False), (0, 0, True, True), (1, 0, False, True), (0, 1, True, False),
                                     (1, 1, False, False), (1, 1, True, True)])
def test_tma_gemm_matches_bf16_matmul(shape, layout):
    M, Nn, K = shape
    a_dt, b_dt, a_tr, b_tr = layout
    for beta in (0, 1):
        err = _run(M, Nn, K, a_dt, b_dt, a_tr, b_tr, beta)
        assert err < 2e-5, (shape, layout, beta, err)


def test_tma_gemm_declines_small_and_unscratched():
    A = torch.randn(32, 64, device="cuda")
    B = torch.randn(64, 64, device="cuda")
    C = torch.zeros(32, 64, device="cuda")
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    rc = N.lib().bb_gemm_bf16_tma(32, 64, 64, A.data_ptr(), 0, 64, 1, B.data_ptr(), 0, 64, 1, C.data_ptr(), 64, 1, 0,
                                  scratch.data_ptr(), scratch.numel(), stream_ptr())
    assert rc == 1
    A = torch.randn(256, 256, device="cuda")
    C = torch.zeros(256, 256, device="cuda")
    rc = N.lib().bb_gemm_bf16_tma(256, 256, 256, A.data_ptr(), 0, 256, 1, A.data_ptr(), 0, 256, 1, C.data_ptr(), 256, 1, 0,
                                  None, 0, stream_ptr())
    assert rc == 1
