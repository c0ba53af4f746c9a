"""FusedAdamW under the native DDP transport (run with >= 2 GPUs)."""
import pytest
import torch
import torch.distributed as dist
import torch.nn as nn

from test_gpu_multi import _spawn

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _check_ddp_bert_adamw(rank, world):
    """A small bf16 BERT under this DDP (sum-of-squares partials from the allreduce epilogue feed the clip) with FusedAdamW
    and graph replay, against stock torch DDP + NCCL driving the same optimizer: every rank ends bit-identical and the
    two trajectories agree in norm after 10 steps."""
    from b200ddp.engine.step import TrainStep
    from b200ddp.models.bert import BertConfig, BertForMaskedLM
    from b200ddp.ops import CrossEntropyLoss
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    from b200ddp.parallel import DistributedDataParallel
    from b200ddp.utils import to_mixed_bf16
    dev = torch.device("cuda", rank)
    cfg = BertConfig(vocab_size=1000, hidden=256, layers=2, heads=4, intermediate=1024, max_position=64, pad_vocab_to=64)

    def make(seed):
        torch.manual_seed(seed)
        return to_mixed_bf16(BertForMaskedLM(cfg).to(dev))
    ours, stock = make(2000 + rank), make(2000)            # rank-dependent init on our side: the wrap must broadcast rank 0's
    ddp = DistributedDataParallel(ours, device_ids=[rank], backend="b200")
    ref = nn.parallel.DistributedDataParallel(stock, device_ids=[rank])
    hyper = dict(lr=2e-3, betas=(0.9, 0.98), eps=1e-6, max_grad_norm=1.0)
    opt = FusedAdamW(weight_decay_groups(ours, 0.01), **hyper)
    ropt = FusedAdamW(weight_decay_groups(stock, 0.01), **hyper)
    step = TrainStep(ddp, CrossEntropyLoss(), opt, dev, use_graph=True)
    rstep = TrainStep(ref, CrossEntropyLoss(), ropt, dev, use_graph=False)
    for i in range(10):
        g = torch.Generator().manual_seed(rank * 131 + i)
        x = torch.randint(0, cfg.vocab_size, (8, 64), generator=g).to(dev)
        y = torch.where(torch.rand(8, 64, generator=g) < 0.15, torch.randint(0, cfg.vocab_size, (8, 64), generator=g),
                        torch.full((8, 64), -100)).to(dev)
        step(x, y)
        rstep(x, y)
    torch.cuda.synchronize()
    ddp.comm.check()
    assert step.graph is not None and int(opt._step_dev) == 10
    pa = torch.cat([p.detach().float().reshape(-1) for p in ours.parameters()])
    pb = torch.cat([p.detach().float().reshape(-1) for p in stock.parameters()])
    rel = float((pa - pb).norm() / pb.norm())
    assert rel < 1e-1, ("trajectories diverged", rel)
    flat = torch.cat([pa, opt._master, opt._exp_avg, opt._exp_avg_sq])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    assert all(torch.equal(t, gathered[0]) for t in gathered), "ranks diverged"


def test_ddp_bert_adamw_ranks_agree(free_port):
    _spawn(_check_ddp_bert_adamw, free_port)
