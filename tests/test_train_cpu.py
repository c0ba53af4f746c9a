"""End-to-end CPU runs of the template: CLI, checkpoint layout, resume, accumulation, gloo launcher."""
import os
import subprocess
import sys

import pytest
import torch

from b200ddp.engine import cli
from b200ddp.engine.trainer import Trainer
from b200ddp.models import FooModel
from b200ddp.ops import MSELoss, cross_entropy, layer_norm, linear, mse_loss
from b200ddp.optim import FusedSGD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(tmp_path, *flags):
    args = cli.build_parser().parse_args(["--no_cuda", "--no_tensorboard", "--output_dir", str(tmp_path / "out"),
                                          "--dataset_size", "640", *flags])
    cli.setup(args)
    trainer = Trainer(args, FooModel(), cli.log)
    return trainer, trainer.train()


def test_single_process_run_checkpoint_layout(tmp_path):
    trainer, (global_step, avg_loss) = _run(tmp_path, "--max_steps", "30", "--logging_steps", "10", "--save_steps", "20")
    assert global_step == 31                              # starts at 1, exits when > max_steps (reference ddp.py:206,280)
    assert 0.5 < avg_loss < 2.0
    ckpt = tmp_path / "out" / "checkpoint-20"
    assert sorted(os.listdir(ckpt)) == ["model.bin", "optimizer.pt", "scheduler.pt", "trainer_state.pt", "training_args.bin"]
    state = torch.load(ckpt / "model.bin")
    assert list(state.keys()) == ["net1.weight", "net1.bias", "net2.weight", "net2.bias"]
    assert tuple(state["net2.weight"].shape) == (5, 10)
    saved_args = torch.load(ckpt / "training_args.bin", weights_only=False)
    assert saved_args.max_steps == 30 and saved_args.per_gpu_train_batch_size == 32
    assert not (tmp_path / "out" / "checkpoint-40").exists()


def test_accumulation_saves_once_per_boundary(tmp_path):
    trainer, (global_step, _) = _run(tmp_path, "--max_steps", "6", "--gradient_accumulation_steps", "4", "--save_steps", "2",
                                     "--logging_steps", "2")
    assert global_step == 7
    assert sorted(os.listdir(tmp_path / "out")) == ["checkpoint-2", "checkpoint-4", "checkpoint-6"]
    assert trainer.step_fn.micro_steps == 6 * 4


def test_resume_restores_state(tmp_path):
    t1, _ = _run(tmp_path, "--max_steps", "10", "--save_steps", "10", "--seed", "3")
    w_after_10 = torch.load(tmp_path / "out" / "checkpoint-10" / "model.bin")["net1.weight"]
    t2, (gs, _) = _run(tmp_path, "--max_steps", "14", "--save_steps", "0", "--seed", "3", "--resume_from", "latest")
    assert t2._resume_state["global_step"] == 10 and gs == 15
    assert t2.scheduler.last_step == 9 + 5                # 9 steps before the save + 5 after resume
    assert not torch.equal(t2.model.net1.weight.detach(), w_after_10)   # training continued from the restored weights


def test_evaluate_returns_loss(tmp_path):
    trainer, _ = _run(tmp_path, "--max_steps", "5", "--save_steps", "0")
    res = trainer.evaluate(max_batches=3)
    assert res["eval_samples"] == 96 and res["eval_loss"] > 0


def test_fused_sgd_cpu_matches_torch_sgd_with_clip():
    torch.manual_seed(0)
    a, b = FooModel(), FooModel()
    b.load_state_dict(a.state_dict())
    oa = FusedSGD(a.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-2, nesterov=True, max_grad_norm=0.05)
    ob = torch.optim.SGD(b.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-2, nesterov=True)
    for i in range(5):
        x, y = torch.randn(16, 10), torch.randn(16, 5)
        for m, o in ((a, oa), (b, ob)):
            o.zero_grad()
            torch.nn.functional.mse_loss(m(x), y).backward()
        torch.nn.utils.clip_grad_norm_(b.parameters(), 0.05)
        oa.step(); ob.step()
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.allclose(pa, pb, atol=1e-6)


def test_cpu_ops_match_torch():
    torch.manual_seed(0)
    x, w, b = torch.randn(7, 12), torch.randn(5, 12), torch.randn(5)
    assert torch.allclose(linear(x, w, b, "relu"), torch.relu(torch.nn.functional.linear(x, w, b)))
    assert torch.allclose(mse_loss(x, x * 0.5), torch.nn.functional.mse_loss(x, x * 0.5))
    t = torch.randint(0, 12, (7,))
    assert torch.allclose(cross_entropy(x, t), torch.nn.functional.cross_entropy(x, t))
    g, be = torch.randn(12), torch.randn(12)
    assert torch.allclose(layer_norm(x, g, be), torch.nn.functional.layer_norm(x, (12,), g, be))


def test_torchrun_gloo_two_ranks(tmp_path, free_port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port), os.path.join(ROOT, "ddp.py"), "--no_cuda", "--no_tensorboard", "--max_steps", "12",
           "--save_steps", "6", "--logging_steps", "6", "--dataset_size", "512", "--output_dir", str(tmp_path / "o")]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=240, env=env, cwd=str(tmp_path))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "[Finished training.] [global_step=13]" in res.stdout
    assert sorted(os.listdir(tmp_path / "o")) == ["checkpoint-12", "checkpoint-6"]
    assert "backend='gloo'" in res.stdout and "world_size=2" in res.stdout


def test_launch_scripts_run_the_template(tmp_path, free_port):
    """The shipped launchers themselves (reference: run.sh, run.slurm.sh - L5 of the layer map): `run.sh` with two ranks on
    the CPU (gloo), and the per-node half of the SLURM launcher under a faked one-node SLURM environment."""
    common = ["--no_cuda", "--no_tensorboard", "--max_steps", "6", "--save_steps", "6", "--logging_steps", "3", "--dataset_size", "256"]
    env = dict(os.environ, OMP_NUM_THREADS="1", NGPU="2", MASTER_PORT=str(free_port))
    res = subprocess.run(["sh", os.path.join(ROOT, "run.sh"), *common, "--output_dir", str(tmp_path / "a")], capture_output=True, text=True,
                         timeout=240, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "[Finished training.] [global_step=7]" in res.stdout and "world_size=2" in res.stdout
    assert os.listdir(tmp_path / "a") == ["checkpoint-6"]
    env = dict(os.environ, OMP_NUM_THREADS="1", SLURM_JOB_NUM_NODES="1", SLURM_NODEID="0", GPUS_PER_NODE="2", MASTER_ADDR="127.0.0.1",
               MASTER_PORT=str(free_port), B200DDP_BACKEND="gloo")
    res = subprocess.run(["bash", os.path.join(ROOT, "run.slurm.sh"), *common, "--output_dir", str(tmp_path / "b")], capture_output=True, text=True,
                         timeout=240, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "[Finished training.] [global_step=7]" in res.stdout and "backend='gloo'" in res.stdout
    assert os.listdir(tmp_path / "b") == ["checkpoint-6"]


def test_default_loss_and_dataset_per_model():
    import argparse
    from b200ddp.engine.trainer import build_criterion, build_dataset, loss_kind
    from b200ddp.ops import CrossEntropyLoss
    foo = argparse.Namespace(model="foo", loss=None, dataset_size=64)
    assert loss_kind(foo) == "mse" and isinstance(build_criterion(foo), MSELoss)
    rn = argparse.Namespace(model="resnet50", loss=None, dataset_size=4, image_samples=4)
    assert loss_kind(rn) == "ce" and isinstance(build_criterion(rn), CrossEntropyLoss)
    ds = build_dataset(rn)
    x, y = ds[0]
    assert tuple(x.shape) == (3, 224, 224) and y.dtype == torch.int64
    rn.loss = "mse"
    assert tuple(build_dataset(rn)[0][1].shape) == (1000,)


def test_static_loss_scale_is_transparent():
    """--loss_scale N multiplies the loss before backward and the fused optimizer divides the gradients again: the
    trajectory is unchanged (up to rounding), clipping still sees unscaled gradients."""
    from b200ddp.engine.step import TrainStep
    torch.manual_seed(0)
    a, b = FooModel(), FooModel()
    b.load_state_dict(a.state_dict())
    sa = TrainStep(a, MSELoss(), FusedSGD(a.parameters(), lr=0.1, max_grad_norm=0.5), torch.device("cpu"))
    sb = TrainStep(b, MSELoss(), FusedSGD(b.parameters(), lr=0.1, max_grad_norm=0.5), torch.device("cpu"), loss_scale=1024.0)
    for _ in range(5):
        x, y = torch.randn(16, 10), torch.randn(16, 5)
        la, lb = sa(x, y), sb(x, y)
        assert torch.allclose(la, lb, atol=1e-6)
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.allclose(p, q, atol=1e-6)


def test_resnet_matches_torchvision_given_its_weights():
    """Same parameter names / shapes as torchvision's ResNet-50 (checkpoints and DDP bucket layouts carry over) and, on the
    stock CPU path, the same function."""
    import torch
    tv = pytest.importorskip("torchvision")
    from b200ddp.models.resnet import ResNet
    torch.manual_seed(0)
    ref = tv.models.resnet.ResNet(tv.models.resnet.Bottleneck, [1, 1, 1, 1], num_classes=10)
    ours = ResNet([1, 1, 1, 1], num_classes=10)
    ours.load_state_dict(ref.state_dict())                # identical parameter / buffer names and shapes
    x = torch.randn(2, 3, 64, 64)
    assert torch.allclose(ours(x), ref(x), atol=1e-4)


def test_bert_matches_huggingface_reference_given_its_weights():
    """Architecture parity with the stock model of the BERT config: same weights -> same logits (fp32, CPU)."""
    import torch
    transformers = pytest.importorskip("transformers")
    from b200ddp.models.bert import BertConfig, BertForMaskedLM
    torch.manual_seed(0)
    hf_cfg = transformers.BertConfig(vocab_size=120, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                                     intermediate_size=128, max_position_embeddings=32, hidden_dropout_prob=0.0,
                                     attention_probs_dropout_prob=0.0)
    hf = transformers.BertForMaskedLM(hf_cfg).eval()
    mine = BertForMaskedLM(BertConfig(vocab_size=120, hidden=64, layers=2, heads=4, intermediate=128, max_position=32,
                                      pad_vocab_to=64)).eval()
    mine.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, 120, (3, 17))
    types = torch.randint(0, 2, (3, 17))
    with torch.no_grad():
        ref = hf(input_ids=ids, token_type_ids=types).logits
        out = mine(ids, types)
    assert out.shape == (3, 17, 128)                      # vocabulary padded to a multiple of 64
    assert torch.allclose(out[..., :120], ref, atol=2e-4, rtol=1e-4)
    assert float(out[..., 120:].max()) < -1e3             # padding logits can never win


def test_resnet50_matches_torchvision_given_its_weights():
    """Same parameter names / shapes as torchvision's ResNet-50 and the same function (train and eval mode)."""
    import torch
    tv = pytest.importorskip("torchvision")
    from b200ddp.models import resnet50
    torch.manual_seed(0)
    ref = tv.models.resnet50(num_classes=10)
    mine = resnet50(num_classes=10)
    mine.load_state_dict(ref.state_dict())                 # strict: identical keys and shapes
    x = torch.randn(2, 3, 64, 64)
    for mode in ("eval", "train"):
        getattr(ref, mode)()
        getattr(mine, mode)()
        with torch.no_grad():
            a, b = ref(x), mine(x)
        assert torch.allclose(a, b, atol=1e-4, rtol=1e-4), mode
    # running statistics were updated identically by the training-mode pass
    for (k, u), (_, v) in zip(ref.state_dict().items(), mine.state_dict().items()):
        assert torch.allclose(u.float(), v.float(), atol=1e-5), k


def test_trace_dir_writes_a_chrome_trace(tmp_path):
    """--trace_dir: a torch.profiler timeline of a few optimizer steps (the reference has no tracing)."""
    import json
    trace_dir = tmp_path / "traces"
    _run(tmp_path, "--max_steps", "12", "--save_steps", "0", "--trace_dir", str(trace_dir), "--trace_steps", "2", "--trace_skip", "3")
    path = trace_dir / "trace_rank0.json"
    assert path.exists()
    events = json.loads(path.read_text())["traceEvents"]
    assert any("ProfilerStep" in str(e.get("name", "")) for e in events)
