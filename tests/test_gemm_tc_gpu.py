"""GPU unit test of the wgmma tensor-core GEMM building block (csrc/gemm_tc.cu) through the C ABI.
Reference = torch matmul of the bf16-rounded operands accumulated in fp32/fp64."""
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
    A_mem = (A.t().contiguous().t() if a_trans else A.contiguous())       # same values, m-fast or k-fast storage
    B_mem = (B.contiguous() if b_trans else B.t().contiguous().t())       # b_trans: n-fast storage; else k-fast
    if a_dt == 1:
        A_mem = A_mem.to(torch.bfloat16) if not a_trans else A.to(torch.bfloat16).t().contiguous().t()
    if b_dt == 1:
        B_mem = B.to(torch.bfloat16).contiguous() if b_trans else B.to(torch.bfloat16).t().contiguous().t()
    C = C0.clone()
    N.call("bb_gemm_bf16_tc", M, Nn, K, A_mem.data_ptr(), a_dt, A_mem.stride(0), A_mem.stride(1), B_mem.data_ptr(), b_dt,
           B_mem.stride(0), B_mem.stride(1), C.data_ptr(), C.stride(0), C.stride(1), beta, stream_ptr())
    torch.cuda.synchronize()
    want = A.to(torch.bfloat16).double() @ B.to(torch.bfloat16).double()
    if beta:
        want = want + C0.double()
    err = float((C.double() - want).norm() / want.norm())
    return err


@pytest.mark.parametrize("shape", [(128, 128, 64), (128, 128, 256), (256, 384, 192), (200, 300, 100), (800, 768, 768),
                                    (768, 3072, 800), (65, 64, 64), (128, 128, 4096)])
@pytest.mark.parametrize("layout", [(0, 1, False, False), (0, 0, True, True), (1, 0, False, True), (0, 1, True, False)])
def test_tc_gemm_matches_bf16_matmul(shape, layout):
    M, Nn, K = shape
    a_dt, b_dt, a_tr, b_tr = layout
    for beta in (0, 1):
        err = _run(M, Nn, K, a_dt, b_dt, a_tr, b_tr, beta)
        assert err < 2e-5, (shape, layout, beta, err)
