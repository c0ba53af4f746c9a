"""Grouped tile rasterisation (B200DDP_GEMM_GROUP_M / set_gemm_group_m): results must be bit-identical to the
default m-fastest order, since only the order in which persistent CTAs pick tiles changes.  The default stays m-fastest;
the knob is for larger-than-L2 problems.  mode 1 = single-CTA tiles, mode 2 = cluster pairs."""

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("M,N,K", [(2048, 2048, 512), (1000, 3000, 264), (4096, 768, 768)])
def test_grouped_raster_is_bit_identical(mode, M, N, K):
    from b200ddp import _ext
    C = _ext.get()
    torch.manual_seed(1)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    try:
        C.set_gemm_cta_mode(mode)
        C.set_gemm_group_m(0)
        d0 = C.gemm(a, b, None, False, False, 0, False, None)
        outs = []
        for g in (1, 4, 8):
            C.set_gemm_group_m(g)
            outs.append(C.gemm(a, b, None, False, False, 0, False, None))
    finally:
        C.set_gemm_group_m(0)
        C.set_gemm_cta_mode(0)
    ref = a.float() @ b.float().t()
    assert float((d0.float() - ref).norm() / ref.norm()) < 1e-2
    for d in outs:
        assert torch.equal(d, d0)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("M,N,K", [(2048, 2048, 512), (1000, 3000, 264), (304, 264, 72), (100352, 64, 64), (4096, 768, 768)])
def test_tma_store_epilogue_is_bit_identical(mode, a_mn, b_mn, M, N, K):
    """Opt-in staged epilogue (shared memory + TMA store): same fp32 accumulators, same rounding -> same bits,
    including ragged M / N edges (the TMA unit clips them)."""
    from b200ddp import _ext
    C = _ext.get()
    torch.manual_seed(2)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    bias = torch.randn(N, device="cuda", dtype=torch.bfloat16)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    try:
        C.set_gemm_cta_mode(mode)
        C.set_gemm_tma_store(0)
        d0 = C.gemm(a, b, None, a_mn, b_mn, 0, False, None)
        e0 = C.gemm(a, b, bias, a_mn, b_mn, 2, False, None)
        C.set_gemm_tma_store(1)
        d1 = C.gemm(a, b, None, a_mn, b_mn, 0, False, None)
        e1 = C.gemm(a, b, bias, a_mn, b_mn, 2, False, None)
        f1 = C.gemm(a, b, None, a_mn, b_mn, 0, True, None)           # fp32 output falls back to the direct epilogue
    finally:
        C.set_gemm_tma_store(0)
        C.set_gemm_cta_mode(0)
    ref = A.float() @ B.float().t()
    assert float((d0.float() - ref).norm() / ref.norm()) < 1e-2
    assert torch.equal(d1, d0)
    assert torch.equal(e1, e0)
    assert f1.dtype == torch.float32 and float((f1 - ref).norm() / ref.norm()) < 1e-2
