"""BART on the H100: the native bf16 model against its fp32 path (the CPU references), a training step without host
synchronisation, and ``ddp.py``-style training of bart-base under a CUDA graph on right-padded and packed rows, whose
losses equal the eager run's bitwise, with the fused LM-head loss within a stated tolerance of the unfused one."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.data import SyntheticDenoising
from b200ddp.models.bart import BartConfig, BartForConditionalGeneration
from b200ddp.utils.precision import to_mixed_bf16

pytestmark = pytest.mark.gpu

V = 1000


def _small(bos_token_id=None):
    torch.manual_seed(0)
    model = BartForConditionalGeneration(BartConfig(vocab_size=V, hidden=256, encoder_layers=2, decoder_layers=2, heads=4, intermediate=1024,
                                                    max_position=512, pad_token_id=0, bos_token_id=bos_token_id))
    with torch.no_grad():                                       # away from zero biases
        for n, p in model.named_parameters():
            if n.endswith("bias"):
                p.normal_(0.0, 0.02)
    return model


def _loss(model, x, y):
    logits = model(x, y)
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), y.reshape(-1))


@pytest.mark.parametrize("pack", [False, True], ids=["padded", "packed"])
def test_native_bf16_bart_matches_the_fp32_path(pack):
    """Loss within 2 % and every parameter gradient within 5 % (relative norm) of the fp32 CPU path."""
    ds = SyntheticDenoising(samples=12, seq_len=256, vocab=V, start_id=3, mask_id=V - 1, min_len=40, pack=pack)
    ref = _small(3 if pack else None)
    native = copy.deepcopy(ref).cuda()
    to_mixed_bf16(native)
    lr = _loss(ref, ds.X, ds.Y)
    ln = _loss(native, ds.X.cuda(), ds.Y.cuda())
    assert abs(float(ln.detach()) - float(lr.detach())) < 2e-2 * float(lr.detach())
    lr.backward()
    ln.backward()
    grads = dict(native.named_parameters())
    for n, p in ref.named_parameters():
        g = grads[n].grad.float().cpu()
        rel = float((g - p.grad).norm() / p.grad.norm().clamp(min=1e-8))
        assert rel < 5e-2, (n, rel)


def test_bart_step_has_no_host_synchronisation():
    ds = SyntheticDenoising(samples=8, seq_len=256, vocab=V, start_id=3, mask_id=V - 1, min_len=40, pack=True)
    model = _small(3).cuda()
    to_mixed_bf16(model)
    x, y = ds.X.cuda(), ds.Y.cuda()
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


def _train(tmp_path, extra):
    """What `python ddp.py --model bart-base --fp16 --optimizer adamw --per_gpu_train_batch_size 8 --seq_len 256
    --min_seq_len 64 --max_steps 20 [extra]` runs; returns every step's loss."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model, model_entry
    argv = ["--model", "bart-base", "--fp16", "--optimizer", "adamw", "--per_gpu_train_batch_size", "8", "--seq_len", "256",
            "--min_seq_len", "64", "--max_steps", "20", "--logging_steps", "1", "--dataset_size", "256", "--lr", "1e-4",
            "--warmup_steps", "2", "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": SyntheticTokens.PAD_ID}
    if args.pack:
        kwargs["bos_token_id"] = model_entry("bart-base").start_id
    if args.fused_lm_loss:
        kwargs["fused_lm_loss"] = True
    trainer = Trainer(args, build_model("bart-base", **kwargs), cli.log)
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
        print(f"\nbart-base {layout} losses on {torch.cuda.get_device_name()}: {[round(v, 4) for v in graph[::4]]}; "
              f"eager bitwise equal: {graph == eager}")
    assert all(math.isfinite(v) for v in graph)
    assert sum(graph[-4:]) / 4 < graph[0] - 0.05               # random targets: only the copied tokens can be learned
    assert graph == eager


def test_fused_lm_loss_matches_the_unfused_loss(tmp_path):
    """The fused head's losses stay within 2e-2 of the unfused ones over 20 steps (bf16 logits against the fused
    kernel's fp32 log-sum-exp)."""
    fused = _train(tmp_path / "f", ["--cuda_graph", "--fused_lm_loss"])
    plain = _train(tmp_path / "p", ["--cuda_graph"])
    assert max(abs(a - b) for a, b in zip(fused, plain)) < 2e-2, (fused, plain)
