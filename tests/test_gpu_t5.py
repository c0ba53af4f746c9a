"""T5 on the H100: the native bf16 model (relative-bias attention kernels, cross-attention on 8 q, bias-free ReLU linears
on the wgmma GEMM) against its fp32 path (the CPU references) on right-padded and packed rows, a training step without
host synchronisation, the fused LM-head loss against the unfused one, and ``ddp.py``-style training of t5-small on
span-corruption pairs under a CUDA graph, whose losses equal the eager run's bitwise."""
import copy
import math
from dataclasses import replace

import pytest
import torch
import torch.nn.functional as F

from b200ddp.models.t5 import T5Config, T5ForConditionalGeneration
from b200ddp.utils.precision import to_mixed_bf16

pytestmark = pytest.mark.gpu

V, SK, SQ, START = 1024, 256, 128, 2


def _small(pack=False, fused=False):
    torch.manual_seed(0)
    return T5ForConditionalGeneration(T5Config(vocab_size=V, d_model=256, num_layers=2, num_decoder_layers=2, num_heads=4, d_ff=1024,
                                               pad_token_id=0, bos_token_id=START if pack else None, fused_lm_loss=fused))


def _pairs(pack, B=6, seed=1):
    """(sources [B, 256] padded with 0, labels [B, 128] padded with -100): one pair per row, or packed pairs whose
    documents start with id 2 on both sides."""
    g = torch.Generator().manual_seed(seed)
    X = torch.zeros(B, SK, dtype=torch.long)
    Y = torch.full((B, SQ), -100)
    for r in range(B):
        a = b = 0
        while True:
            s, t = int(torch.randint(20, 200, (1,), generator=g)), int(torch.randint(5, 100, (1,), generator=g))
            if a + s > SK or b + t > SQ:
                break
            X[r, a:a + s] = torch.randint(3, V, (s,), generator=g)
            Y[r, b:b + t] = torch.randint(3, V, (t,), generator=g)
            if pack:
                X[r, a], Y[r, b] = START, START
            a, b = a + s, b + t
            if not pack:
                break
    return X, Y


def _loss(model, x, y):
    logits = model(x, y)
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), y.reshape(-1))


@pytest.mark.parametrize("pack", [False, True], ids=["padded", "packed"])
def test_native_bf16_t5_matches_the_fp32_path(pack):
    """Loss within 2 % and every parameter gradient within 5 % (relative norm) of the fp32 CPU path, the tolerances of
    the BART test."""
    X, Y = _pairs(pack)
    ref = _small(pack)
    native = copy.deepcopy(ref).cuda()
    to_mixed_bf16(native)
    lr = _loss(ref, X, Y)
    ln = _loss(native, X.cuda(), Y.cuda())
    assert abs(float(ln.detach()) - float(lr.detach())) < 2e-2 * float(lr.detach())
    lr.backward()
    ln.backward()
    grads = dict(native.named_parameters())
    for n, p in ref.named_parameters():
        g = grads[n].grad.float().cpu()
        rel = float((g - p.grad).norm() / p.grad.norm().clamp(min=1e-8))
        assert rel < 5e-2, (n, rel)


def test_t5_step_has_no_host_synchronisation():
    X, Y = _pairs(True)
    model = _small(True).cuda()
    to_mixed_bf16(model)
    x, y = X.cuda(), Y.cuda()
    _loss(model, x, y).backward()
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = _loss(model, x, y)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss))


def test_fused_lm_loss_matches_the_unfused_loss():
    """The fused head's loss within 1e-2 of the unfused one (bf16 logits against the fused kernel's fp32 log-sum-exp),
    and its gradients within 2 % (relative norm)."""
    X, Y = _pairs(True)
    plain = _small(True).cuda()
    to_mixed_bf16(plain)
    fused = copy.deepcopy(plain)
    fused.config = replace(plain.config, fused_lm_loss=True)
    x, y = X.cuda(), Y.cuda()
    lp = _loss(plain, x, y)
    lf = fused.lm_head_loss()(fused(x, y).reshape(-1, 256), y.reshape(-1))
    assert abs(float(lf.detach()) - float(lp.detach())) < 1e-2, (float(lf), float(lp))
    lp.backward()
    lf.backward()
    grads = dict(fused.named_parameters())
    for n, p in plain.named_parameters():
        rel = float((grads[n].grad.float() - p.grad.float()).norm() / p.grad.float().norm().clamp(min=1e-8))
        assert rel < 2e-2, (n, rel)


def _train(tmp_path, extra):
    """What `python ddp.py --model t5-small --fp16 --optimizer adamw --per_gpu_train_batch_size 8 --seq_len 256
    --min_seq_len 64 --max_steps 20 [extra]` runs; returns every step's loss."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model, model_entry
    argv = ["--model", "t5-small", "--fp16", "--optimizer", "adamw", "--per_gpu_train_batch_size", "8", "--seq_len", "256",
            "--min_seq_len", "64", "--max_steps", "20", "--logging_steps", "1", "--dataset_size", "256", "--lr", "1e-4",
            "--warmup_steps", "2", "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": SyntheticTokens.PAD_ID}
    if args.pack:
        kwargs["bos_token_id"] = model_entry("t5-small").start_id
    if args.fused_lm_loss:
        kwargs["fused_lm_loss"] = True
    trainer = Trainer(args, build_model("t5-small", **kwargs), cli.log)
    sums = []
    read = trainer.step_fn.read_loss_sum
    trainer.step_fn.read_loss_sum = lambda: sums.append(read()) or sums[-1]
    trainer.train()
    assert (trainer.step_fn.graph is not None) == args.cuda_graph
    return [b - a for a, b in zip([0.0] + sums[:-1], sums)][:20]


@pytest.mark.parametrize("layout", [[], ["--pack"]], ids=["padded", "packed"])
def test_training_under_a_cuda_graph_equals_eager_bitwise(tmp_path, capsys, layout):
    graph = _train(tmp_path / "g", ["--cuda_graph", *layout])
    eager = _train(tmp_path / "e", layout)
    with capsys.disabled():
        print(f"\nt5-small {layout} losses on {torch.cuda.get_device_name()}: {[round(v, 4) for v in graph[::4]]}; "
              f"eager bitwise equal: {graph == eager}")
    assert all(math.isfinite(v) for v in graph)
    assert sum(graph[-4:]) / 4 < graph[0] - 0.05               # random span text: the sentinels and </s> can be learned
    assert graph == eager


def test_fused_lm_loss_training_matches_the_unfused_loss(tmp_path):
    """Under ddp.py-style training, the fused head's losses stay within 2e-2 of the unfused ones over 20 steps."""
    fused = _train(tmp_path / "f", ["--cuda_graph", "--fused_lm_loss"])
    plain = _train(tmp_path / "p", ["--cuda_graph"])
    assert max(abs(a - b) for a, b in zip(fused, plain)) < 2e-2, (fused, plain)
