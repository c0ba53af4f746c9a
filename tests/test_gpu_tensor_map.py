"""The shared TMA tensor-map encoder against recorded maps.

``tests/golden/tensor_maps.json`` holds the 128-byte ``CUtensorMap`` that the per-file encoders (GEMM, convolution / attention,
BatchNorm) produced for the geometries the kernels use, before they were merged into ``encode_tensor_map``: a map is a pure
function of (pointer, element type, swizzle, dims, strides, box), so the one encoder must reproduce every byte.  Encoding only
records the pointer, so the recorded address needs no allocation behind it."""
import json
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu

CASES = json.loads((Path(__file__).parent / "golden" / "tensor_maps.json").read_text())


@pytest.fixture(scope="module")
def C():
    import torch
    from b200ddp import _ext
    torch.zeros(1, device="cuda")
    return _ext.get()


def _encode(C, case):
    return C._tensor_map_bytes(case["ptr"], case["dtype"], case["swizzle"], case["dims"], case["strides"], case["box"])


def test_golden_covers_every_kind_of_map():
    kinds = {(c["dtype"], c["swizzle"], len(c["dims"])) for c in CASES}
    assert {(9, 3, 2), (0, 3, 2), (9, 0, 2), (9, 3, 4)} <= kinds          # bf16 / 8-bit 128B-swizzled, bf16 unswizzled, rank 4


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_tensor_map_bytes_match_recorded(C, case):
    got = _encode(C, case)
    assert len(got) == 128
    assert got.hex() == case["bytes"]
    assert _encode(C, case) == got                                        # the cached map is the same map


def test_tensor_map_key_separates_dtype_swizzle_and_box(C):
    base = next(c for c in CASES if c["name"] == "batchnorm_resident")
    same_shape_swizzled = dict(base, swizzle=3)
    other_box = dict(base, box=[base["box"][0], base["box"][1] * 2])
    maps = {_encode(C, c) for c in (base, same_shape_swizzled, other_box)}
    assert len(maps) == 3


def test_tensor_map_rejects_bad_rank(C):
    with pytest.raises(RuntimeError):
        C._tensor_map_bytes(0x7F0000004000, 9, 3, [64] * 5, [128] * 4, [64] * 5)
    with pytest.raises(RuntimeError):
        C._tensor_map_bytes(0x7F0000004000, 9, 3, [64, 64], [128, 128], [64, 64])
