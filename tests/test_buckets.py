"""Bucket planner vs torch's ``_compute_bucket_assignment_by_size`` and the layouts stock DDP builds."""
import pytest
import torch
import torch.distributed as dist

from b200ddp.models import build_model
from b200ddp.parallel.buckets import MiB, assign_by_size, bucket_sizes_mib, plan_buckets


def _sizes(model):
    return [p.numel() for p in model.parameters()]


@pytest.mark.parametrize("name,expected", [
    ("foo", [0.0]),
    ("resnet50", [11.84, 30.04, 28.29, 25.77, 1.55]),
    ("resnet152", [11.84, 30.04, 32.56, 25.57, 25.57, 25.57, 25.57, 25.57, 25.78, 1.55]),
])
def test_torch_order_matches_stock_layout(name, expected):
    model = build_model(name)
    params = list(model.parameters())
    ref = dist._compute_bucket_assignment_by_size(params, [1 * MiB, 25 * MiB])[0]
    mine = assign_by_size([p.numel() * 4 for p in params], None, [1 * MiB, 25 * MiB])
    assert mine == ref
    specs = plan_buckets(_sizes(model), [4] * len(params), order="torch", max_tensors=10 ** 9)
    assert bucket_sizes_mib(specs) == expected


@pytest.mark.parametrize("cap,count", [(1, 76), (25, 14), (256, 3)])
def test_bert_bucket_counts(cap, count):
    """Layouts of the stock BERT-base tensor list (199 tensors: separate query / key / value), and the planner
    against torch's on this package's model, whose Q / K / V projection is one stored parameter (151 tensors)."""
    import torch
    model = build_model("bert-base", with_mlm_head=False)
    stock = []
    for name, p in model.named_parameters():
        if ".qkv." in name:
            stock += [torch.nn.Parameter(torch.empty_like(c)) for c in p.detach().chunk(3, dim=0)]
        else:
            stock.append(p)
    assert len(stock) == 199
    specs = plan_buckets([p.numel() for p in stock], [4] * len(stock), bucket_cap_bytes=cap * MiB, order="torch", max_tensors=10 ** 9)
    assert len(specs) == count
    ref = dist._compute_bucket_assignment_by_size(stock, [1 * MiB, cap * MiB])[0]
    assert [s.param_indices for s in reversed(specs)] == ref
    params = list(model.parameters())
    mine = plan_buckets(_sizes(model), [4] * len(params), bucket_cap_bytes=cap * MiB, order="torch", max_tensors=10 ** 9)
    ref = dist._compute_bucket_assignment_by_size(params, [1 * MiB, cap * MiB])[0]
    assert [s.param_indices for s in reversed(mine)] == ref


def test_backward_order_first_bucket_small_and_layout_aligned():
    model = build_model("resnet50")
    n = _sizes(model)
    specs = plan_buckets(n, [4] * len(n))
    assert sum(len(s.param_indices) for s in specs) == len(n)
    assert sorted(i for s in specs for i in s.param_indices) == list(range(len(n)))
    # first bucket to launch holds the LAST parameters (fc) and is the small one
    assert specs[0].param_indices[0] == len(n) - 1
    for s in specs:
        assert len(s.param_indices) <= 192
        assert all(o % 8 == 0 for o in s.offsets) and s.total_elems % 8 == 0
        assert s.flags_offset >= sum(s.numels)
        assert s.total_elems - s.flags_offset >= len(s.numels)
        for (o, m), o2 in zip(zip(s.offsets, s.numels), s.offsets[1:] + [s.flags_offset]):
            assert o + m <= o2


def test_keys_split_dtypes_and_limits_advance():
    groups = assign_by_size([10, 10, 10, 10, 50], ["a", "b", "a", "b", "a"], [15, 40])
    assert groups == [[0, 2], [1, 3], [4]]
    assert assign_by_size([5] * 6, None, [10], max_tensors=None) == [[0, 1], [2, 3], [4, 5]]
    assert assign_by_size([1] * 5, None, [100], max_tensors=2) == [[0, 1], [2, 3], [4]]


def test_native_planner_matches_python():
    from b200ddp import _ext
    C = _ext.get()
    g = torch.Generator().manual_seed(0)
    for _ in range(20):
        n = int(torch.randint(1, 60, (1,), generator=g))
        sizes = torch.randint(1, 5000, (n,), generator=g).tolist()
        keys = torch.randint(0, 2, (n,), generator=g).tolist()
        limits = [1000, 4000]
        assert C.assign_by_size(sizes, keys, limits, 7) == assign_by_size(sizes, keys, limits, max_tensors=7)


def test_ready_order_rebuild():
    n = [100, 200, 300, 400]
    order = [2, 3, 0, 1]
    specs = plan_buckets(n, [4] * 4, bucket_cap_bytes=10 ** 9, first_bucket_bytes=0, ready_order=order)
    assert specs[0].param_indices == order
