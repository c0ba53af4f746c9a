"""wgmma GEMM (fwd / dgrad / wgrad operand layouts, epilogues, ragged shapes) vs fp32 matmul."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def _rel_err(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 256), (128, 128, 8), (8, 8, 8), (200, 136, 72),
                                   (1000, 1000, 2048), (4096, 768, 768), (4096, 3072, 768), (512, 30528, 768), (8192, 768, 3072)])
def test_gemm_nt(C, M, N, K):
    torch.manual_seed(0)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d = C.gemm(a, b)
    ref = a.float() @ b.float().t()
    assert _rel_err(d, ref) < 1e-2, _rel_err(d, ref)
    d32 = C.gemm(a, b, None, False, False, 0, True, None)
    assert d32.dtype == torch.float32 and _rel_err(d32, ref) < 1e-5 + 2e-3


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (256, 384, 200), (4096, 768, 3072), (768, 3072, 4096), (1000, 2048, 32)])
def test_gemm_operand_layouts(C, a_mn, b_mn, M, N, K):
    torch.manual_seed(1)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    ref = A.float() @ B.float().t()
    a = A.t().contiguous() if a_mn else A                  # stored [K, M] when MN-major
    b = B.t().contiguous() if b_mn else B                  # stored [K, N] when MN-major
    d = C.gemm(a, b, None, a_mn, b_mn, 0, False, None)
    assert _rel_err(d, ref) < 1e-2, _rel_err(d, ref)


@pytest.mark.parametrize("epi", [1, 2, 3])
def test_gemm_epilogues(C, epi):
    torch.manual_seed(2)
    a = torch.randn(512, 256, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(384, 256, device="cuda", dtype=torch.bfloat16) * 0.1
    bias = torch.randn(384, device="cuda", dtype=torch.bfloat16)
    d = C.gemm(a, b, bias, False, False, epi, False, None)
    ref = a.float() @ b.float().t() + bias.float()
    ref = torch.relu(ref) if epi == 2 else F.gelu(ref) if epi == 3 else ref
    assert _rel_err(d, ref) < 1e-2


def test_gemm_fp32_accumulate_into(C):
    a = torch.randn(256, 128, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(128, 128, device="cuda", dtype=torch.bfloat16)
    out = torch.ones(256, 128, device="cuda")
    C.gemm(a, b, None, False, False, 0, True, out)
    assert _rel_err(out, a.float() @ b.float().t() + 1.0) < 1e-3


@pytest.mark.parametrize("act", [None, "relu", "gelu"])
@pytest.mark.parametrize("tokens,fin,fout", [(256, 256, 512), (4096, 768, 3072), (32, 2048, 1000)])
def test_linear_module_fwd_bwd(C, act, tokens, fin, fout):
    from b200ddp.ops import Linear
    torch.manual_seed(3)
    lin = Linear(fin, fout, activation=act).to("cuda", torch.bfloat16)
    x = torch.randn(tokens, fin, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    before = C.launch_count()
    y = lin(x)
    dy = torch.randn_like(y)
    y.backward(dy)
    assert C.launch_count() - before >= 3                  # fwd + dgrad + wgrad on wgmma
    xr = x.detach().float().requires_grad_()
    wr, br = lin.weight.detach().float().requires_grad_(), lin.bias.detach().float().requires_grad_()
    yr = F.linear(xr, wr, br)
    yr = torch.relu(yr) if act == "relu" else F.gelu(yr) if act == "gelu" else yr
    yr.backward(dy.float())
    assert _rel_err(y, yr) < 1.5e-2
    assert _rel_err(x.grad, xr.grad) < 2e-2
    assert _rel_err(lin.weight.grad, wr.grad) < 2e-2
    assert _rel_err(lin.bias.grad, br.grad) < 2e-2
