"""Distributed plumbing on CPU (gloo, world_size 2)."""
import copy
import os
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from b200ddp.models import BranchyFooModel, FooModel
from b200ddp.parallel import DistributedDataParallel


def _spawn(fn, world, port, *args):
    mp.spawn(_entry, args=(fn, world, port, args), nprocs=world, join=True)


def _entry(rank, fn, world, port, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fn(rank, world, *args)
    finally:
        dist.destroy_process_group()


def _full_batch_grads(model, x, y):
    m = copy.deepcopy(model)
    loss = nn.functional.mse_loss(m(x), y)
    loss.backward()
    return [p.grad.clone() for p in m.parameters()]


def _check_ddp(rank, world, as_view, find_unused):
    torch.manual_seed(1234 + rank)                      # different init per rank: wrap must broadcast rank 0's
    model = FooModel()
    ddp = DistributedDataParallel(model, backend="gloo", gradient_as_bucket_view=as_view,
                                  find_unused_parameters=find_unused, bucket_cap_mb=0.0001, first_bucket_mb=0.00005)
    flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    gathered = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    assert all(torch.equal(g, gathered[0]) for g in gathered), "init broadcast failed"
    assert len(ddp._specs) > 1                           # tiny caps: several buckets, exercised in order

    torch.manual_seed(99)
    X, Y = torch.randn(8 * world, 10), torch.randn(8 * world, 5)
    expect = _full_batch_grads(model, X, Y)              # mean over the global batch
    xs, ys = X[rank::world], Y[rank::world]
    loss = nn.functional.mse_loss(ddp(xs), ys)
    loss.backward()
    for p, e in zip(model.parameters(), expect):
        assert torch.allclose(p.grad, e, atol=1e-6), (p.grad - e).abs().max()
    if as_view:
        flats = ddp.reducer.flats
        assert any(p.grad.data_ptr() >= f.data_ptr() and p.grad.data_ptr() < f.data_ptr() + f.numel() * 4
                   for p in model.parameters() for f in flats)

    # no_sync: grads stay local, next synced backward reduces the accumulated sum
    model.zero_grad(set_to_none=True)
    with ddp.no_sync():
        nn.functional.mse_loss(ddp(xs), ys).backward()
    local = [p.grad.clone() for p in model.parameters()]
    nn.functional.mse_loss(ddp(xs), ys).backward()
    for p, e, l in zip(model.parameters(), expect, local):
        assert torch.allclose(p.grad, 2 * e, atol=1e-5)
    assert ddp.ddp_stats()["buckets_launched"] == 2 * len(ddp._specs)


@pytest.mark.parametrize("as_view", [False, True])
def test_ddp_gloo_grad_parity(free_port, as_view):
    _spawn(_check_ddp, 2, free_port, as_view, True)


def _check_unused(rank, world):
    torch.manual_seed(0)
    model = BranchyFooModel()
    ddp = DistributedDataParallel(model, backend="gloo", find_unused_parameters=True)
    x, y = torch.randn(4, 10), torch.randn(4, 5)
    # (a) aux unused on every rank: its grads stay None, the rest reduce normally
    nn.functional.mse_loss(ddp(x, use_aux=False), y).backward()
    assert model.aux.weight.grad is None and model.net1.weight.grad is not None
    # (b) aux used on rank 0 only: every rank receives grad/world for it
    model.zero_grad(set_to_none=True)
    out = ddp(x, use_aux=(rank == 0))
    nn.functional.mse_loss(out, y).backward()
    g = model.aux.weight.grad
    assert g is not None
    gathered = [torch.zeros_like(g) for _ in range(world)]
    dist.all_gather(gathered, g)
    assert torch.equal(gathered[0], gathered[1]) and gathered[0].abs().sum() > 0


def test_find_unused_parameters_semantics(free_port):
    _spawn(_check_unused, 2, free_port)


def _check_strict(rank, world):
    model = BranchyFooModel()
    ddp = DistributedDataParallel(model, backend="gloo", find_unused_parameters=False)
    x, y = torch.randn(4, 10), torch.randn(4, 5)
    with pytest.raises(RuntimeError, match="find_unused_parameters"):
        nn.functional.mse_loss(ddp(x, use_aux=False), y).backward()


def test_missing_grad_without_find_unused_raises(free_port):
    _spawn(_check_strict, 2, free_port)


def _check_mismatch(rank, world):
    model = FooModel(hidden=10 if rank == 0 else 12)
    with pytest.raises(RuntimeError, match="differ"):
        DistributedDataParallel(model, backend="gloo")


def test_param_shape_verification(free_port):
    _spawn(_check_mismatch, 2, free_port)


def _check_buffers_and_rebuild(rank, world):
    torch.manual_seed(rank)
    model = nn.Sequential(nn.Linear(6, 6), nn.BatchNorm1d(6), nn.Linear(6, 2))
    ddp = DistributedDataParallel(model, backend="gloo", find_unused_parameters=False)
    with torch.no_grad():
        model[1].running_mean.fill_(float(rank + 1))
    out = ddp(torch.randn(4, 6))                          # forward broadcasts rank 0's buffers first
    out.sum().backward()
    # the forward pass then updates the running mean from (different) local batches; undo that to compare
    assert ddp.rebuild_buckets()
    order = [i for s in ddp._specs for i in s.param_indices]
    assert sorted(order) == list(range(len(list(model.parameters()))))
    model.zero_grad()
    ddp(torch.randn(4, 6)).sum().backward()               # rebuilt reducer still works
    g = model[0].weight.grad
    gathered = [torch.zeros_like(g) for _ in range(world)]
    dist.all_gather(gathered, g)
    assert torch.allclose(gathered[0], gathered[1])


def test_buffer_broadcast_and_bucket_rebuild(free_port):
    _spawn(_check_buffers_and_rebuild, 2, free_port)


def test_single_process_wrap_is_transparent():
    model = FooModel()
    ddp = DistributedDataParallel(model, backend="gloo")
    x, y = torch.randn(4, 10), torch.randn(4, 5)
    nn.functional.mse_loss(ddp(x), y).backward()
    assert all(p.grad is not None for p in model.parameters())
    assert list(ddp.state_dict().keys()) == ["net1.weight", "net1.bias", "net2.weight", "net2.bias"]


def test_auto_backend_leaves_the_peer_transport_for_multi_node_jobs(monkeypatch):
    """One peer-memory arena spans one NVSwitch domain (<= 8 GPUs of one host); `auto` must not pick it beyond that."""
    from b200ddp.parallel import backend as B

    class FakeDist:
        def __init__(self, world):
            self.world = world

        def is_available(self):
            return True

        def is_initialized(self):
            return True

        def get_world_size(self, group=None):
            return self.world

    monkeypatch.setattr(B, "dist", FakeDist(8))
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "8")
    assert B.spans_one_nvswitch_domain()
    monkeypatch.setattr(B, "dist", FakeDist(16))            # 2 nodes x 8 (run.sbatch)
    assert not B.spans_one_nvswitch_domain()
    monkeypatch.setattr(B, "dist", FakeDist(8))             # 2 nodes x 4
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "4")
    assert not B.spans_one_nvswitch_domain()
    assert B.pick_backend_name("auto", torch.device("cuda", 0)) == "nccl"
    assert B.pick_backend_name("b200", torch.device("cuda", 0)) == "b200"      # explicit choice is honoured
    assert B.pick_backend_name("auto", torch.device("cpu")) == "gloo"
