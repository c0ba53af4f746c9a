"""Every wgmma GEMM instantiation that `gemm` and `gemm_stats` can reach, checked element by element against fp64.

`launch_gemm_bf16` picks one of 30 kernels from the operand layout, the tile choice (cluster pair 256 x 128, single
128 x 128, single 128 x 64), the epilogue kind (direct stores, or shared memory + TMA store) and column statistics.
`dispatch` below mirrors that rule; the parameter tables are run through it, and a test asserts that together they reach
all 30.  Each call writes into a view of a larger buffer filled with a sentinel, at element offset 0 and at offset 1
(which misaligns the rows and forces the scalar stores), and every byte outside the view must survive.

Cross-checks that need no tolerance: cluster-pair and single-CTA results are bitwise equal, and so are TMA-store and
direct results, for every epilogue; an accumulating call equals the previous contents plus the same call's fp32 result,
bitwise; `gemm_nt` is `gemm` bitwise; `gemm_stats`' output is `gemm`'s, bitwise, and its statistics repeat bitwise.
"""
import contextlib
import itertools

import pytest
import torch

import numerics as nm

pytestmark = pytest.mark.gpu

LAYOUTS = [(False, False), (False, True), (True, True), (True, False)]     # (a_mn, b_mn): NT, dgrad, wgrad-like, NN
OUTS = ("bf16", "fp32", "acc")        # bf16 output, fp32 output, fp32 accumulate into the given out
GUARD = 64                            # sentinel elements after the view

# (M, N, K): why the shape is here.  MN-major layouts need a stored row of a multiple of 8 elements (gemm_shape_supported).
SMALL = {
    (1, 1, 8): "smallest problem, N = 1",
    (7, 10, 24): "a partial 32-column chunk, misaligned rows",
    (129, 65, 72): "one row past a tile, one column past 64, one k-block plus 8",
    (255, 100, 136): "misaligned bf16 and fp32 rows: scalar stores, TMA store not eligible",
    (200, 264, 520): "TMA clipping on the last slab; a pair tile whose second CTA is partly empty",
    (264, 56, 200): "at most 64 columns on every layout: the 128 x 64 tile, TMA store clipped at column 56",
}
LARGE = {
    (1000, 30522, 64): "the unpadded BERT vocabulary",
    (4096, 768, 3072): "BERT-base FFN down-projection",
    (8192, 2304, 768): "BERT-base fused qkv projection",
}
STATS = {
    (20, 56, 40): "M < 32: one partial statistics group; N <= 64",
    (129, 65, 72): "M % 32 != 0, N > 64, ragged columns (direct stores only)",
    (200, 264, 520): "M % 32 != 0, N > 64, TMA store eligible",
    (4096, 768, 768): "a model shape",
}


def supported(M, N, K, a_mn, b_mn):
    """Mirror of gemm_shape_supported: TMA needs a 16-byte row pitch on both operands."""
    return (M if a_mn else K) % 8 == 0 and (N if b_mn else K) % 8 == 0


def dispatch(layout, N, mode, tma_store, out, aligned, stats=False):
    """Mirror of launch_gemm_bf16: the (layout, tile choice, TMA-store epilogue, column statistics) kernel a call runs.
    choice 0 = cluster pair 256 x 128 (mode 2), else 2 = single 128 x 64 when N <= 64, 1 = single 128 x 128."""
    choice = 0 if mode == 2 else (2 if N <= 64 else 1)
    tma_st = bool(tma_store) and out == "bf16" and N % 8 == 0 and aligned
    return layout, choice, tma_st, stats


def configs(large):
    """(mode, tma_store, epilogue, out, offset) of every call one (shape, layout) case makes; reduced on large shapes."""
    epilogues = (1, 3) if large else (0, 1, 2, 3)
    return list(itertools.product((1, 2), (0, 1), epilogues, OUTS, (0, 1)))


CASES = [(shape, layout, False) for shape in SMALL for layout in LAYOUTS if supported(*shape, *layout)] + \
        [(shape, layout, True) for shape in LARGE for layout in LAYOUTS if supported(*shape, *layout)]
STATS_CONFIGS = list(itertools.product((1, 2), (0, 1)))


def _case_id(case):
    (M, N, K), (a_mn, b_mn), _ = case
    return f"{M}x{N}x{K}-{'A_mn' if a_mn else 'A_k'}-{'B_mn' if b_mn else 'B_k'}"


def test_parameter_tables_reach_every_instantiation():
    every = {(layout, choice, tma, False) for layout in LAYOUTS for choice in range(3) for tma in (False, True)}
    every |= {((False, False), choice, tma, True) for choice in range(3) for tma in (False, True)}
    assert len(every) == 30
    reached = {dispatch(layout, shape[1], mode, tma, out, off == 0)
               for shape, layout, large in CASES for mode, tma, _, out, off in configs(large)}
    reached |= {dispatch((False, False), shape[1], mode, tma, "bf16", True, stats=True)
                for shape in STATS for mode, tma in STATS_CONFIGS}
    assert reached == every, sorted(every - reached)


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


@contextlib.contextmanager
def switches(C, mode, tma_store):
    try:
        C.set_gemm_cta_mode(mode)
        C.set_gemm_tma_store(tma_store)
        yield
    finally:
        C.set_gemm_cta_mode(0)
        C.set_gemm_tma_store(0)


def _inputs(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    return a, b, bias


_SENTINEL = {torch.bfloat16: (torch.int16, 0x7FB5), torch.float32: (torch.int32, 0x7FB5A5A5)}


def _framed(M, N, dtype, offset):
    """A contiguous [M, N] view at element `offset` into a sentinel-filled buffer; returns (raw bits, view)."""
    itype, pattern = _SENTINEL[dtype]
    raw = torch.full((offset + M * N + GUARD,), pattern, dtype=itype, device="cuda")
    return raw, raw.view(dtype)[offset:offset + M * N].view(M, N)


def _assert_frame(raw, offset, count, what):
    _, pattern = _SENTINEL[torch.bfloat16 if raw.dtype == torch.int16 else torch.float32]
    outside = torch.cat([raw[:offset], raw[offset + count:]])
    hit = (outside != pattern).nonzero()
    assert hit.numel() == 0, f"{what}: {hit.numel()} elements written outside out, first at frame index {int(hit[0])}"


def _call(C, a, b, bias, layout, epi, out, offset, old=None):
    """One gemm into a framed out.  fp32 `out` with out_fp32=False is a plain fp32 output; with out_fp32=True it is
    accumulated into."""
    M, N = (a.shape[1] if layout[0] else a.shape[0]), (b.shape[1] if layout[1] else b.shape[0])
    dtype = torch.bfloat16 if out == "bf16" else torch.float32
    raw, view = _framed(M, N, dtype, offset)
    if old is not None:
        view.copy_(old)
    C.gemm(a, b, bias if epi else None, layout[0], layout[1], epi, out == "acc", view)
    torch.cuda.synchronize()
    _assert_frame(raw, offset, M * N, f"{out} epilogue {epi} offset {offset}")
    return view.clone()


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_gemm_matches_fp64_elementwise(C, case):
    (M, N, K), layout, large = case
    a, b, bias = _inputs(M, N, K, seed=M + N + K)
    ops = (a.t().contiguous() if layout[0] else a, b.t().contiguous() if layout[1] else b)
    old = torch.randn(M, N, device="cuda")
    refs = {}
    got = {}
    for mode, tma, epi, out, off in configs(large):
        where = f"{_case_id(case)} mode {mode} tma_store {tma} epilogue {epi} {out} offset {off}"
        with switches(C, mode, tma):
            d = _call(C, *ops, bias, layout, epi, out, off, old if out == "acc" else None)
        key = (mode, tma, epi, out)
        if off == 1:
            assert torch.equal(d, got[key]), f"{where}: differs from the aligned out"
            continue
        got[key] = d
        if out == "acc":
            assert torch.equal(d, old + got[(mode, tma, epi, "fp32")]), f"{where}: not old + the fp32 result, bitwise"
            continue
        if epi not in refs:
            refs[epi] = nm.gemm_reference(a, b, bias if epi else None, epi)
        ref, acc = refs[epi]
        nm.check(where, d, ref, nm.bound(ref, acc, d.dtype), group=f"gemm {out}")
        if mode == 2:
            assert torch.equal(d, got[(1, tma, epi, out)]), f"{where}: cluster pair differs from single CTA"
        if tma == 1:
            assert torch.equal(d, got[(mode, 0, epi, out)]), f"{where}: TMA-store epilogue differs from direct stores"


@pytest.mark.parametrize("M,N,K", [(7, 10, 24), (129, 65, 72), (264, 56, 200), (4096, 768, 768)])
def test_gemm_nt_is_gemm(C, M, N, K):
    a, b, bias = _inputs(M, N, K, seed=7)
    for epi, bb in ((0, None), (1, bias), (3, bias)):
        d = C.gemm_nt(a, b, bb, epi, None)
        assert torch.equal(d, C.gemm(a, b, bb, False, False, epi, False, None)), epi
        nm.check_gemm(f"gemm_nt epilogue {epi}", d, a, b, bb, epi, group="gemm bf16")
        out = torch.empty(M, N, device="cuda")
        d32 = C.gemm_nt(a, b, bb, epi, out)
        assert d32.data_ptr() == out.data_ptr()
        assert torch.equal(d32, C.gemm(a, b, bb, False, False, epi, True, None)), epi


@pytest.mark.parametrize("M,N,K", list(STATS), ids=[f"{m}x{n}x{k}" for m, n, k in STATS])
def test_gemm_stats_matches_fp64_per_group(C, M, N, K):
    a, b, _ = _inputs(M, N, K, seed=11)
    seen = {}
    for mode, tma in STATS_CONFIGS:
        where = f"gemm_stats {M}x{N}x{K} mode {mode} tma_store {tma}"
        with switches(C, mode, tma):
            d, stats = C.gemm_stats(a, b)
            d2, stats2 = C.gemm_stats(a, b)
            plain = C.gemm(a, b)
        assert stats.shape == (2, (M + 31) // 32, N) and stats.dtype == torch.float32, where
        assert torch.equal(d, plain), f"{where}: output differs from gemm"
        assert torch.equal(d, d2) and torch.equal(stats, stats2), f"{where}: not bitwise repeatable"
        nm.check_gemm(f"{where}: output", d, a, b, group="gemm bf16")
        ref, bnd = nm.column_stats_reference(d)
        nm.check(f"{where}: statistics [sum | sum of squares, group, column]", stats, ref, bnd, group="gemm_stats")
        seen[(mode, tma)] = stats
    for mode, tma in STATS_CONFIGS:
        assert torch.equal(seen[(mode, tma)], seen[(1, 0)]), f"statistics differ between mode {mode} tma_store {tma} and mode 1 direct"
