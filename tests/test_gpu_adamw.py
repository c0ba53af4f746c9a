"""FusedAdamW on one GPU: the multi_adamw kernel against torch.optim.AdamW on fp32 copies, the CUDA-graph step against
the eager step, bit-exact checkpoint / resume, and a short bf16 BERT-base training run."""
import copy
import math

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda", 0)


def _params(dtype):
    """More than 120 tensors (two kernel tables in the decay group), a channels_last 4-D tensor, an odd-sized one that
    ends in a scalar tail, and one that never gets a gradient."""
    torch.manual_seed(4)
    shapes = [(10, 10), (10,), (300, 77), (64, 3, 7, 7), (20001,), (5,), (33, 65), (7,)] + [(24, 40), (40,)] * 60
    params = [nn.Parameter(torch.randn(*s, device=dev()).to(dtype)) for s in shapes]
    params[3].data = params[3].data.contiguous(memory_format=torch.channels_last)
    return params, 7                                      # params[7] has no gradient


def _groups(params, wd):
    return [{"params": [p for p in params if p.dim() >= 2], "weight_decay": wd},
            {"params": [p for p in params if p.dim() < 2], "weight_decay": 0.0}]


def _master_of(opt, p):
    for g in opt._groups:
        for q, off, n in zip(g.params, g.offsets, g.numels):
            if q is p:
                return opt._master[off:off + n]
    raise KeyError


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_fused_adamw_matches_torch(dtype, wd):
    from b200ddp.optim import FusedAdamW
    from b200ddp.optim.fused import _physical_flat
    params, no_grad = _params(dtype)
    ref = [nn.Parameter(p.detach().float().clone()) for p in params]
    untouched = params[no_grad].detach().clone()
    hyper = dict(lr=0.05, betas=(0.8, 0.99), eps=1e-6)
    opt = FusedAdamW(_groups(params, wd), max_grad_norm=0.5, **hyper)
    ropt = torch.optim.AdamW(_groups(ref, wd), **hyper)
    assert sum(g.plan.total_blocks > 0 for g in opt._groups) >= 2 and len(params) > 120
    for it in range(4):
        for i, (p, r) in enumerate(zip(params, ref)):
            if i == no_grad:
                continue
            g = torch.randn_like(r) * (0.1 if it % 2 else 3.0)
            if p.dim() == 4:
                g = g.contiguous(memory_format=torch.channels_last)
            p.grad = g.to(dtype)
            r.grad = p.grad.float().clone()
        total = torch.nn.utils.clip_grad_norm_([r for r in ref if r.grad is not None], 0.5)
        assert float(total) > 0.5                          # clipping is active
        opt.step(); ropt.step()
        assert math.isclose(opt.grad_norm(), float(total), rel_tol=2e-3)
    assert torch.equal(params[no_grad].detach(), untouched)
    for i, (p, r) in enumerate(zip(params, ref)):
        if dtype == torch.float32:
            assert torch.allclose(p.detach(), r.detach(), atol=1e-5, rtol=0), (i, float((p - r).abs().max()))
        else:
            m = _master_of(opt, p)                          # storage order of p (r has p's layout)
            assert torch.allclose(m, _physical_flat(r.detach()), atol=1e-5, rtol=0), (i, float((m - _physical_flat(r)).abs().max()))
            assert torch.equal(_physical_flat(p.detach()), m.to(torch.bfloat16)), i      # p = bf16 rounding of its master
    assert int(opt._step_dev) == 4


def _run_step(accum, graph, steps=10):
    from b200ddp.engine.step import TrainStep
    from b200ddp.ops import Linear, MSELoss
    from b200ddp.optim import FusedAdamW, weight_decay_groups
    torch.manual_seed(0)
    model = nn.Sequential(Linear(64, 128, activation="relu"), Linear(128, 32)).to(dev())
    opt = FusedAdamW(weight_decay_groups(model, 0.01), lr=1e-2, max_grad_norm=1.0)
    step = TrainStep(model, MSELoss(), opt, dev(), accumulation=accum, use_graph=graph)
    g = torch.Generator().manual_seed(5)
    for i in range(steps * accum):
        x = torch.randn(16, 64, generator=g).to(dev())
        y = torch.randn(16, 32, generator=g).to(dev())
        step(x, y, boundary=(i + 1) % accum == 0)
    torch.cuda.synchronize()
    return [p.detach().clone() for p in model.parameters()], step, opt


@pytest.mark.parametrize("accum", [1, 2])
def test_fused_adamw_graph_step_equals_eager_step(accum):
    """The step count lives on the device: a graph that baked the bias correction of its capture step would drift."""
    eager, _, eopt = _run_step(accum, False)
    graphed, step, gopt = _run_step(accum, True)
    assert step.graph is not None
    assert int(eopt._step_dev) == int(gopt._step_dev) == 10
    for a, b in zip(eager, graphed):
        assert torch.allclose(a, b, atol=1e-6, rtol=1e-5), float((a - b).abs().max())


def test_fused_adamw_resume_is_bit_exact():
    """state_dict -> fresh optimizer -> continue == the uninterrupted run (bf16 + fp32 masters, channels_last), and a
    torch.optim.AdamW on fp32 copies can take over the same state dict."""
    from b200ddp.optim import FusedAdamW
    hyper = dict(lr=1e-2, betas=(0.9, 0.98), eps=1e-8)

    def grads(i, params):
        g = torch.Generator().manual_seed(100 + i)
        for p in params:
            p.grad = torch.randn(p.shape, generator=g).to(dev(), p.dtype)
            if p.dim() == 4:
                p.grad = p.grad.contiguous(memory_format=torch.channels_last)

    for dtype in (torch.bfloat16, torch.float32):
        base, _ = _params(dtype)
        base = base[:8]
        a = [nn.Parameter(p.detach().clone()) for p in base]
        opt_a = FusedAdamW(_groups(a, 0.01), max_grad_norm=1.0, **hyper)
        for i in range(6):
            grads(i, a)
            opt_a.step()
        b = [nn.Parameter(p.detach().clone()) for p in base]
        opt_b = FusedAdamW(_groups(b, 0.01), max_grad_norm=1.0, **hyper)
        for i in range(3):
            grads(i, b)
            opt_b.step()
        sd = copy.deepcopy(opt_b.state_dict())
        assert float(sd["state"][0]["step"]) == 3 and sd["state"][2]["exp_avg"].is_contiguous(memory_format=torch.channels_last)
        c = [nn.Parameter(p.detach().clone()) for p in b]
        opt_c = FusedAdamW(_groups(c, 0.01), max_grad_norm=1.0, **hyper)
        opt_c.load_state_dict(sd)
        for i in range(3, 6):
            grads(i, c)
            opt_c.step()
        for pa, pc in zip(a, c):
            assert torch.equal(pa.detach(), pc.detach())
        if dtype == torch.float32:
            r = [nn.Parameter(p.detach().clone()) for p in b]
            ropt = torch.optim.AdamW(_groups(r, 0.01), **hyper)
            ropt.load_state_dict(sd)
            for i in range(3, 6):
                grads(i, r)
                torch.nn.utils.clip_grad_norm_(r, 1.0)
                ropt.step()
            for pa, pr in zip(a, r):
                assert torch.allclose(pa.detach(), pr.detach(), atol=1e-5, rtol=0)


def test_bert_base_adamw_graph_training_lowers_the_loss(tmp_path):
    """What `python ddp.py --model bert-base --fp16 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 128` runs."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    from b200ddp.optim import FusedAdamW
    args = cli.build_parser().parse_args(["--model", "bert-base", "--fp16", "--optimizer", "adamw", "--cuda_graph",
                                          "--max_steps", "30", "--seq_len", "128", "--per_gpu_train_batch_size", "16",
                                          "--lr", "5e-4", "--warmup_steps", "5", "--weight_decay", "0.01",
                                          "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
                                          "--output_dir", str(tmp_path / "out")])
    cli.setup(args)
    trainer = Trainer(args, build_model("bert-base"), cli.log)
    assert isinstance(trainer.optimizer, FusedAdamW) and trainer.optimizer._master is not None
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)
