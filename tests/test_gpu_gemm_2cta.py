"""Cluster-pair GEMM (two CTAs of a cluster, 256x128 pair tiles, B tile shared through TMA multicast) vs fp32 matmul and
the single-CTA kernel, every operand layout, ragged shapes."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    mod = _ext.get()
    yield mod
    mod.set_gemm_cta_mode(0)


def _rel_err(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 512, 256), (1000, 1000, 2048), (4096, 3072, 768), (304, 264, 72), (8192, 768, 3072)])
def test_gemm_2cta_matches_reference_and_1cta(C, a_mn, b_mn, M, N, K):
    torch.manual_seed(0)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    ref = A.float() @ B.float().t()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    C.set_gemm_cta_mode(2)
    d2 = C.gemm(a, b, None, a_mn, b_mn, 0, False, None)
    C.set_gemm_cta_mode(1)
    d1 = C.gemm(a, b, None, a_mn, b_mn, 0, False, None)
    C.set_gemm_cta_mode(0)
    assert _rel_err(d2, ref) < 1e-2, _rel_err(d2, ref)
    assert torch.equal(d1, d2)          # same accumulation order per output element -> bit-identical


def test_gemm_2cta_epilogue_and_fp32(C):
    a = torch.randn(1024, 512, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(768, 512, device="cuda", dtype=torch.bfloat16) * 0.1
    bias = torch.randn(768, device="cuda", dtype=torch.bfloat16)
    C.set_gemm_cta_mode(2)
    d = C.gemm(a, b, bias, False, False, 2, True, None)
    C.set_gemm_cta_mode(0)
    ref = torch.relu(a.float() @ b.float().t() + bias.float())
    assert d.dtype == torch.float32 and _rel_err(d, ref) < 2e-3
