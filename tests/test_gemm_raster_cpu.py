"""Host mirror of the persistent GEMM's tile rasterisation (csrc/gemm.h::gemm_tile_coords).

The producer, issuer and epilogue roles of the wgmma kernels all map a linear tile id through this function, so a
bijection here is what guarantees every output tile is computed exactly once whatever the order.
"""
import pytest

from b200ddp import _ext

pytestmark = pytest.mark.skipif(not _ext.available(), reason="native extension not built")


@pytest.mark.parametrize("num_m,num_n", [(1, 1), (3, 1), (1, 7), (32, 32), (33, 5), (7, 40), (16, 3)])
@pytest.mark.parametrize("group_m", [0, 1, 4, 8, 64])
def test_tile_order_is_a_bijection(num_m, num_n, group_m):
    order = _ext.get().gemm_tile_order(num_m, num_n, group_m)
    assert len(order) == num_m * num_n
    assert sorted(order) == [(m, n) for m in range(num_m) for n in range(num_n)]


def test_default_order_is_m_fastest():
    order = _ext.get().gemm_tile_order(4, 3, 0)
    assert order[:5] == [(0, 0), (1, 0), (2, 0), (3, 0), (0, 1)]


def test_grouped_order_keeps_a_wave_in_a_compact_patch():
    # 32x32 tiles, 132 tiles in flight (one wave of single-CTA tiles, one per SM): the grouped order touches 8 m-blocks x 17
    # n-blocks, the m-fastest order 32 m-blocks x 5 n-blocks -> operand tiles fetched per wave 25 vs 37.
    C = _ext.get()
    for group_m, max_operand_tiles in ((0, 37), (8, 25)):
        wave = C.gemm_tile_order(32, 32, group_m)[:132]
        ms = {m for m, _ in wave}
        ns = {n for _, n in wave}
        assert len(ms) + len(ns) <= max_operand_tiles, (group_m, len(ms), len(ns))


def test_short_last_band():
    # 10 m-blocks with bands of 4: the last band has 2 rows and must still be swept n-major
    order = _ext.get().gemm_tile_order(10, 3, 4)
    assert order[-6:] == [(8, 0), (9, 0), (8, 1), (9, 1), (8, 2), (9, 2)]
