"""The element-wise checker in numerics.py, on the CPU: the fp64 truth rounded to the output dtype passes, and each fault a
GEMM or its column statistics could plausibly make fails, including faults the older global-norm check lets through."""
import pytest
import torch

import numerics as nm

M, N, K = 256, 256, 72


@pytest.fixture(scope="module")
def problem():
    g = torch.Generator().manual_seed(0)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16)
    b = torch.randn(N, K, generator=g).to(torch.bfloat16)
    bias = torch.randn(N, generator=g).to(torch.bfloat16)
    bias[-1] = 1.0
    return a, b, bias


def _truth(a, b, bias=None, epilogue=0, dtype=torch.bfloat16):
    ref, _ = nm.gemm_reference(a, b, bias, epilogue)
    return ref.to(dtype)


@pytest.mark.parametrize("epilogue", [0, 1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_rounded_truth_passes(problem, epilogue, dtype):
    a, b, bias = problem
    nm.check_gemm("truth", _truth(a, b, bias, epilogue, dtype), a, b, bias, epilogue)


def test_truth_through_an_fp32_accumulation_passes(problem):
    """An fp32 sum of the products in k order (what a correct kernel does) stays well inside the bound at C_ACC."""
    a, b, bias = problem
    acc = torch.zeros(M, N, dtype=torch.float32)
    for k in range(K):
        acc += a[:, k, None].float() * b[None, :, k].float()
    acc += bias.float()
    assert nm.check_gemm("fp32 k-order", acc, a, b, bias, 1) < 0.5


def _rejected(got, a, b, bias=None, epilogue=0):
    with pytest.raises(AssertionError, match="out of bound; worst at"):
        nm.check_gemm("fault", got, a, b, bias, epilogue)


def test_dropped_last_partial_k_block_fails(problem):
    a, b, _ = problem
    _rejected(_truth(a[:, :64], b[:, :64]), a, b)           # K = 72 computed as 64: the last 8-wide k-block is lost


@pytest.mark.parametrize("where", ["last_row", "last_col"])
def test_one_zeroed_element_fails_where_the_norm_check_passes(problem, where):
    a, b, _ = problem
    got = _truth(a, b)
    ref = a.double() @ b.double().t()
    if where == "last_row":
        got[-1, N // 2] = 0
    else:
        got[M // 2, -1] = 0
    assert nm.rel_err(got, ref) < 1e-2                      # invisible to the global norm
    _rejected(got, a, b)


def test_swapped_adjacent_columns_fail(problem):
    a, b, _ = problem
    got = _truth(a, b)
    got[:, [10, 11]] = got[:, [11, 10]]
    _rejected(got, a, b)


def test_missing_bias_on_the_last_column_fails_where_the_norm_check_passes(problem):
    a, b, bias = problem
    got = _truth(a, b, bias, 1)
    got[:, -1] = _truth(a, b)[:, -1]
    ref = a.double() @ b.double().t() + bias.double()
    assert nm.rel_err(got, ref) < 1e-2
    _rejected(got, a, b, bias, 1)


def test_error_message_names_the_worst_element(problem):
    a, b, _ = problem
    got = _truth(a, b)
    got[3, 7] += 100.0
    with pytest.raises(AssertionError, match=r"1 of 65536 elements out of bound; worst at \(3, 7\)"):
        nm.check_gemm("d", got, a, b)


@pytest.mark.parametrize("rows", [20, 200])
def test_column_statistics_truth_passes_and_a_misattributed_group_fails(problem, rows):
    a, b, _ = problem
    d = _truth(a[:rows], b)
    ref, bnd = nm.column_stats_reference(d)
    assert ref.shape == (2, (rows + 31) // 32, N)
    stats = ref.float()
    nm.check("stats", stats, ref, bnd)
    # summed in row order in fp32, as the kernel's butterfly reduction does in some order
    x = torch.zeros(ref.shape[1] * 32, N)
    x[:rows] = d.float()
    x = x.view(-1, 32, N)
    s, q = torch.zeros(x.shape[0], N), torch.zeros(x.shape[0], N)
    for r in range(32):
        s += x[:, r]
        q += x[:, r] * x[:, r]
    assert nm.check("stats fp32", torch.stack([s, q]), ref, bnd) < 0.5
    if ref.shape[1] > 1:
        bad = stats.clone()
        bad[:, 1] = stats[:, 0]                             # group 0's rows credited to group 1
        with pytest.raises(AssertionError, match="out of bound"):
            nm.check("stats", bad, ref, bnd)
    bad = stats.clone()
    bad[:, -1] = 0                                          # the last (partial) group lost
    with pytest.raises(AssertionError, match="out of bound"):
        nm.check("stats", bad, ref, bnd)


def test_nan_fails():
    ref = torch.ones(4, 4, dtype=torch.float64)
    got = ref.float().clone()
    got[2, 1] = float("nan")
    with pytest.raises(AssertionError, match=r"worst at \(2, 1\)"):
        nm.check("nan", got, ref, torch.full_like(ref, 1e-3))
