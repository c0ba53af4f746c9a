"""Multi-GPU checks of the NVSwitch peer-memory transport (run with >= 2 GPUs)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _world():
    """World size for these tests: 2 by default (every box with >= 2 GPUs); B200DDP_TEST_WORLD=4|8 widens it."""
    want = int(os.environ.get("B200DDP_TEST_WORLD", "2"))
    return max(2, min(want, torch.cuda.device_count()))


def _entry(rank, fn, world, port, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), B200DDP_TIMEOUT_S="6")
    torch.cuda.set_device(rank)
    if os.environ.get("B200DDP_TEST_DUMP_AFTER"):          # debugging aid: dump every rank's Python stack if a test stalls
        import faulthandler
        import sys
        faulthandler.dump_traceback_later(float(os.environ["B200DDP_TEST_DUMP_AFTER"]), exit=True, file=sys.stderr)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        fn(rank, world, *args)
        torch.cuda.synchronize()
    except BaseException:
        # a failing rank must not wait for its peers in collective teardown (they may be blocked on it): report and leave
        import traceback
        traceback.print_exc()
        os._exit(1)
    try:
        from b200ddp.parallel.peer import PeerCollectives
        PeerCollectives.shutdown_all()
    finally:
        dist.destroy_process_group()


def _spawn(fn, port, *args, world=None):
    mp.spawn(_entry, args=(fn, world or _world(), port, args), nprocs=world or _world(), join=True)


# --------------------------------------------------------------------------------------------------
def _check_collectives(rank, world):
    from b200ddp.parallel.peer import PeerCollectives
    dev = torch.device("cuda", rank)
    comm = PeerCollectives.get(None, dev, min_bytes=64 << 20)
    algos = ["one_shot", "two_shot"] + (["nvls", "nvls_one_shot"] if comm.nvls else [])
    print(f"[rank {rank}] nvls={comm.nvls} world={world}", flush=True)

    def stage(msg):
        if rank == 0:
            print(f"[collectives] {msg}", flush=True)
    torch.manual_seed(100 + rank)
    sizes = [1, 7, 165, 4096, 100003, 1 << 20]
    for dtype in (torch.float32, torch.bfloat16):
        for wire in ("fp32", "bf16"):
            for algo in algos:
                if algo in ("one_shot", "nvls_one_shot"):
                    use = sizes[:4]
                else:
                    use = sizes
                stage(f"allreduce {dtype} wire={wire} algo={algo}")
                tensors = [torch.randn(n, device=dev).to(dtype) for n in use]
                ref = [t.float().clone() for t in tensors]
                for r in ref:
                    dist.all_reduce(r)
                comm.allreduce_(tensors, wire=wire, algo=algo, scale=1.0 / world)
                torch.cuda.synchronize()
                comm.check()
                lossy = wire == "bf16" or dtype == torch.bfloat16
                for t, r in zip(tensors, ref):
                    exp = r / world
                    tol = 3e-2 if lossy else 1e-5
                    err = (t.float() - exp).abs().max().item()
                    assert err <= tol * max(1.0, exp.abs().max().item()), (dtype, wire, algo, t.numel(), err)
                # every rank must hold bit-identical results
                flat = torch.cat([t.float().reshape(-1) for t in tensors])
                gathered = [torch.empty_like(flat) for _ in range(world)]
                dist.all_gather(gathered, flat)
                assert all(torch.equal(g, gathered[0]) for g in gathered), (dtype, wire, algo)
    stage("symmetric")
    # in-place allreduce on symmetric (arena-resident) tensors
    for dtype in (torch.float32, torch.bfloat16):
        sym = comm.symmetric_empty(40000, dtype)
        for algo in ["two_shot"] + (["nvls"] if comm.nvls else []):
            torch.manual_seed(50 + rank)
            sym.copy_(torch.randn(40000, device=dev).to(dtype))
            ref = sym.float().clone()
            dist.all_reduce(ref)
            dist.barrier(device_ids=[rank])
            comm.allreduce_symmetric_(sym, algo=algo, scale=1.0 / world)
            torch.cuda.synchronize()
            comm.check()
            tol = 1e-5 if dtype == torch.float32 else 3e-2
            assert (sym.float() - ref / world).abs().max().item() <= tol * max(1.0, ref.abs().max().item() / world), (dtype, algo)
    stage("broadcast")
    # broadcast: odd sizes, unaligned views, several dtypes, a tensor larger than one staging chunk
    torch.manual_seed(7)
    base = [torch.randn(5), torch.randn(1000, 33), torch.randint(0, 100, (77,)), torch.randn(3, 5, 7).to(torch.bfloat16),
            torch.randn(20 * 1024 * 1024)]
    mine = [(b.clone() if rank == 0 else torch.zeros_like(b)).to(dev) for b in base]
    view = torch.zeros(1001, device=dev)[1:]                 # 4-byte aligned only
    if rank == 0:
        view.copy_(torch.arange(1000.0))
    os.environ["B200DDP_SCRATCH_MB"] = "64"
    n = comm.broadcast_tensors(mine + [view], src=0)
    torch.cuda.synchronize()
    comm.check()
    assert n >= 2
    for m, b in zip(mine, base):
        assert torch.equal(m.cpu(), b), (rank, b.shape)
    assert torch.equal(view.cpu(), torch.arange(1000.0))
    stage("stress")
    # stress the barrier protocol: 1000 back-to-back collectives of odd sizes, cycling through every algorithm, checked on
    # the device against the expected sum (no host sync inside the loop, so launches of consecutive epochs overlap)
    sizes = [3, 1, 165, 4099, 7, 65537, 33, 1023]
    bad = torch.zeros((), device=dev)
    bufs = {n: torch.empty(n, device=dev) for n in sizes}
    for it in range(1000):
        n = sizes[it % len(sizes)]
        algo = algos[it % len(algos)] if n <= 4099 else ("nvls" if comm.nvls and it % 2 else "two_shot")
        t = bufs[n]
        t.fill_(float(rank + 1 + it % 5))
        comm.allreduce_([t], wire="fp32", algo=algo, scale=1.0)
        expect = float(sum(r + 1 + it % 5 for r in range(world)))
        bad += (t - expect).abs().max()
    torch.cuda.synchronize()
    comm.check()
    assert float(bad) == 0.0, float(bad)


def test_peer_collectives(free_port):
    _spawn(_check_collectives, free_port)


# --------------------------------------------------------------------------------------------------
def _train_pair(rank, world, model_fn, make_batch, steps, ddp_kwargs, dtype, graph):
    """Train the same model with our DDP (b200 transport) and with stock torch DDP (NCCL); compare."""
    from b200ddp.engine.step import TrainStep
    from b200ddp.ops import MSELoss
    from b200ddp.optim import FusedSGD
    from b200ddp.parallel import DistributedDataParallel
    dev = torch.device("cuda", rank)
    torch.manual_seed(1000 + rank)                           # rank-dependent init: wrap must broadcast rank 0's
    ours = model_fn().to(dev)
    if dtype == torch.bfloat16:
        ours = ours.to(dtype)
    torch.manual_seed(1000)                                  # rank 0's init everywhere for the stock model
    stock = model_fn().to(dev)
    if dtype == torch.bfloat16:
        stock = stock.to(dtype)
    ddp = DistributedDataParallel(ours, device_ids=[rank], backend="b200", **ddp_kwargs)
    assert ddp.backend_name == "b200"
    for a, b in zip(ours.parameters(), stock.parameters()):
        assert torch.equal(a, b), "peer broadcast did not deliver rank 0's weights"
    ref = nn.parallel.DistributedDataParallel(stock, device_ids=[rank])
    opt = FusedSGD(ours.parameters(), lr=0.05, max_grad_norm=1.0)
    ropt = torch.optim.SGD(stock.parameters(), lr=0.05)
    step = TrainStep(ddp, MSELoss(), opt, dev, use_graph=graph)
    for i in range(steps):
        x, y = make_batch(rank, i, dev, dtype)
        step(x, y)
        ropt.zero_grad(set_to_none=True)
        nn.functional.mse_loss(ref(x).float(), y.float()).backward()
        torch.nn.utils.clip_grad_norm_(stock.parameters(), 1.0)
        ropt.step()
    torch.cuda.synchronize()
    ddp.comm.check()
    tol = 1e-5 if dtype == torch.float32 else 5e-2
    for a, b in zip(ours.parameters(), stock.parameters()):
        assert torch.allclose(a.float(), b.float(), atol=tol, rtol=tol), (a.float() - b.float()).abs().max()
    # ranks agree bit-for-bit with each other
    flat = torch.cat([p.detach().float().reshape(-1) for p in ours.parameters()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    assert all(torch.equal(g, gathered[0]) for g in gathered)
    return ddp, step


def _foo_batch(rank, i, dev, dtype):
    g = torch.Generator().manual_seed(rank * 1000 + i)
    return torch.randn(32, 10, generator=g).to(dev, dtype), torch.randn(32, 5, generator=g).to(dev, dtype)


def _check_ddp_foo(rank, world):
    from b200ddp.models import FooModel
    for graph in (False, True):
        for kwargs in (dict(find_unused_parameters=True), dict(gradient_as_bucket_view=True),
                       dict(wire_dtype="fp32", bucket_cap_mb=0.0001, first_bucket_mb=0.00005)):
            ddp, step = _train_pair(rank, world, FooModel, _foo_batch, 12, kwargs, torch.float32, graph)
            stats = ddp.ddp_stats()
            assert stats["buckets_launched"] >= len(ddp._specs)
            if graph:
                assert step.graph is not None


def test_ddp_foo_matches_stock_ddp(free_port):
    _spawn(_check_ddp_foo, free_port)


def _check_ddp_mlp_bf16_and_unused(rank, world):
    from b200ddp.models import BranchyFooModel
    from b200ddp.ops import Linear
    from b200ddp.parallel import DistributedDataParallel

    def mlp():
        return nn.Sequential(Linear(256, 512, activation="relu"), Linear(512, 512, activation="relu"), Linear(512, 64))

    def batch(rank, i, dev, dtype):
        g = torch.Generator().manual_seed(rank * 77 + i)
        return torch.randn(64, 256, generator=g).to(dev, dtype), torch.randn(64, 64, generator=g).to(dev, dtype)

    _train_pair(rank, world, mlp, batch, 6, dict(bucket_cap_mb=0.5), torch.bfloat16, False)

    # unused-parameter semantics on the native reducer
    dev = torch.device("cuda", rank)
    torch.manual_seed(3)
    m = BranchyFooModel().to(dev)
    ddp = DistributedDataParallel(m, device_ids=[rank], backend="b200", find_unused_parameters=True)
    x, y = torch.randn(8, 10, device=dev), torch.randn(8, 5, device=dev)
    nn.functional.mse_loss(ddp(x, use_aux=False), y).backward()
    torch.cuda.synchronize()
    assert m.aux.weight.grad is None and m.net1.weight.grad is not None
    m.zero_grad(set_to_none=True)
    nn.functional.mse_loss(ddp(x, use_aux=(rank == 0)), y).backward()
    torch.cuda.synchronize()
    g = m.aux.weight.grad
    assert g is not None and g.abs().sum() > 0
    gathered = [torch.empty_like(g) for _ in range(world)]
    dist.all_gather(gathered, g)
    assert all(torch.equal(t, gathered[0]) for t in gathered)
    # strict mode raises
    ddp2 = DistributedDataParallel(BranchyFooModel().to(dev), device_ids=[rank], backend="b200", find_unused_parameters=False)
    with pytest.raises(RuntimeError, match="find_unused_parameters"):
        nn.functional.mse_loss(ddp2(x, use_aux=False), y).backward()


def test_ddp_bf16_and_unused_parameters(free_port):
    _spawn(_check_ddp_mlp_bf16_and_unused, free_port)


# --------------------------------------------------------------------------------------------------
def _check_one_shot_ownership(rank, world):
    """Regression for the one-shot allreduce: every phase must give a vector to the same block, else a block reads staging
    another block has not packed yet (stale gradients of the previous launch).  Geometry of the ResNet-50 fp32 BatchNorm
    bucket (208 KB: 7 blocks, slices misaligned with the block stride for every world size), block start skew provoked
    by a long-running kernel that occupies the SMs, values that change every launch so stale data cannot pass."""
    from b200ddp.parallel.peer import PeerCollectives
    dev = torch.device("cuda", rank)
    comm = PeerCollectives.get(None, dev, min_bytes=64 << 20)
    algos = ["one_shot"] + (["nvls_one_shot"] if comm.nvls else [])
    n = 53224                                                 # 207.9 KB fp32: V = 13306 vectors, not a multiple of world * 7 * 256
    hog = torch.empty(64 << 20, device=dev)
    t = torch.empty(n, device=dev)
    idx = torch.arange(n, device=dev, dtype=torch.float32)
    bad = torch.zeros((), device=dev)
    for it in range(300):
        for algo in algos:
            if it % 3 == rank % 3:
                hog.normal_()                                 # staggers this rank's comm-kernel blocks against its peers'
            t.copy_(idx * 1e-3 + float(it * world + rank))
            comm.allreduce_([t], wire="fp32", algo=algo, scale=1.0, blocks=7)
            expect = idx * 1e-3 * world + float(sum(it * world + r for r in range(world)))
            bad += (t - expect).abs().max()
    torch.cuda.synchronize()
    comm.check()
    assert float(bad) < 1e-2 * 300 * len(algos), float(bad)


def test_one_shot_allreduce_block_ownership_under_skew(free_port):
    _spawn(_check_one_shot_ownership, free_port)


# --------------------------------------------------------------------------------------------------
def _check_ddp_resnet50(rank, world):
    """ResNet-50, bf16 weights + fp32 BatchNorm (mixed bf16 / fp32 buckets, NVLS two-shot on the large ones, one-shot on the
    BatchNorm bucket, bounded tail bucket, buffer broadcast on the comm stream, whole step replayed from a CUDA graph)
    against stock torch DDP + NCCL driving the SAME model class: parameters and running statistics agree within bf16
    tolerance after 10 steps and every rank holds bit-identical state."""
    from b200ddp.engine.step import TrainStep
    from b200ddp.models import build_model
    from b200ddp.ops import MSELoss
    from b200ddp.optim import FusedSGD
    from b200ddp.parallel import DistributedDataParallel
    from b200ddp.utils import to_mixed_bf16
    dev = torch.device("cuda", rank)

    def make(seed):
        torch.manual_seed(seed)
        return to_mixed_bf16(build_model("resnet50").to(dev)).to(memory_format=torch.channels_last)
    ours, stock = make(1000 + rank), make(1000)              # rank-dependent init on our side: the wrap must broadcast rank 0's
    ddp = DistributedDataParallel(ours, device_ids=[rank], backend="b200")
    ref = nn.parallel.DistributedDataParallel(stock, device_ids=[rank])
    kinds = {str(p.dtype) for p in ours.parameters()}
    assert kinds == {"torch.bfloat16", "torch.float32"} and len(ddp._specs) >= 5
    # (a) one eager forward / backward on identical weights: the averaged gradients agree tensor by tensor (the only
    #     differences are the wire rounding order - scale-then-round here, sum-then-divide in NCCL - and kernel run order)
    g = torch.Generator().manual_seed(rank * 977 + 5)
    x = torch.randn(8, 3, 96, 96, generator=g).to(dev, torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randn(8, 1000, generator=g).to(dev, torch.bfloat16)
    crit = MSELoss()
    crit(ddp(x), y).backward()
    crit(ref(x), y).backward()
    torch.cuda.synchronize()
    ddp.comm.check()
    worst = (0.0, "")
    for (n, a), b in zip(ours.named_parameters(), stock.parameters()):
        ga, gb = a.grad.float(), b.grad.float()
        err = float((ga - gb).norm() / (gb.norm() + 1e-12))
        worst = max(worst, (err, n))
        assert err < 2e-2, ("gradient mismatch", n, err)
    # running statistics: this wrapper publishes rank 0's right after the forward, stock DDP at the start of the NEXT
    # forward - so straight after one forward only rank 0 is comparable (every rank is compared after phase (b))
    if rank == 0:
        for (n, a), b in zip(ours.named_buffers(), stock.buffers()):
            assert torch.allclose(a.float(), b.float(), atol=1e-3, rtol=1e-3), (n, float((a.float() - b.float()).abs().max()))
    ours.zero_grad(set_to_none=False)
    stock.zero_grad(set_to_none=False)

    # (b) ten optimizer steps, ours replayed from the CUDA graph: bf16 training of a randomly initialised network is
    #     chaotic at the last bit, so the trajectories are compared in norm; what must be EXACT is rank agreement
    opt = FusedSGD(ours.parameters(), lr=0.01, max_grad_norm=1000.0)
    ropt = FusedSGD(stock.parameters(), lr=0.01, max_grad_norm=1000.0)
    step = TrainStep(ddp, MSELoss(), opt, dev, use_graph=True)
    rstep = TrainStep(ref, MSELoss(), ropt, dev, use_graph=False)
    for i in range(10):
        g = torch.Generator().manual_seed(rank * 131 + i)
        x = torch.randn(8, 3, 96, 96, generator=g).to(dev, torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randn(8, 1000, generator=g).to(dev, torch.bfloat16)
        step(x, y)
        rstep(x, y)
    torch.cuda.synchronize()
    ddp.comm.check()
    assert step.graph is not None
    pa = torch.cat([p.detach().float().reshape(-1) for p in ours.parameters()])
    pb = torch.cat([p.detach().float().reshape(-1) for p in stock.parameters()])
    rel = float((pa - pb).norm() / pb.norm())
    assert rel < 1e-1, ("trajectories diverged", rel, "worst one-step gradient error", worst)
    flat = torch.cat([p.detach().float().reshape(-1) for p in list(ours.parameters()) + list(ours.buffers())])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    assert all(torch.equal(t, gathered[0]) for t in gathered), "ranks diverged"
    stats = ddp.ddp_stats()
    assert stats["buckets_launched"] >= len(ddp._specs)


def test_ddp_resnet50_matches_stock_ddp(free_port):
    _spawn(_check_ddp_resnet50, free_port)


# --------------------------------------------------------------------------------------------------
def _check_timeout(rank, world):
    """A peer that never shows up must surface as an error after the timeout, not hang the kernel forever
    (signal-pad waits need timeouts)."""
    import time
    from b200ddp.parallel.peer import PeerCollectives, PeerCommError
    dev = torch.device("cuda", rank)
    os.environ["B200DDP_TIMEOUT_S"] = "2"
    comm = PeerCollectives.get(None, dev, min_bytes=8 << 20)
    assert comm.timeout_s == 2.0
    t = torch.ones(1024, device=dev)
    comm.allreduce_([t], wire="fp32", algo="one_shot")            # healthy collective first
    torch.cuda.synchronize()
    comm.check()
    dist.barrier(device_ids=[rank])
    if rank == 0:
        t0 = time.time()
        comm.allreduce_([t], wire="fp32", algo="one_shot")        # rank 1..n never join this one
        torch.cuda.synchronize()
        assert time.time() - t0 < 15
        with pytest.raises(PeerCommError):
            comm.check()
    dist.barrier(device_ids=[rank])


def test_missing_peer_times_out_instead_of_hanging(free_port):
    _spawn(_check_timeout, free_port, world=2)
