"""ConvNeXt on the CPU: torchvision's parameter counts, state dict key for key, initialisation, logits and gradients from the
same weights, the depthwise convolution and the patch gathers against ``F.conv2d``, the DDP bucket plan, the registry, the
CLI and a short ``ddp.py`` training run."""
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.nn.functional as F

from b200ddp.models import MODEL_REGISTRY, convnext_base, convnext_small, convnext_tiny
from b200ddp.ops import cross_entropy, depthwise_conv2d, depthwise_conv2d_reference, patchify_nhwc
from b200ddp.parallel.buckets import MiB

tvm = pytest.importorskip("torchvision.models")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESETS = {"convnext_tiny": convnext_tiny, "convnext_small": convnext_small, "convnext_base": convnext_base}
PARAMS = {"convnext_tiny": 28_589_128, "convnext_small": 50_223_688, "convnext_base": 88_591_464}


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_parameter_counts(name):
    with torch.device("meta"):
        model = PRESETS[name]()
    assert sum(p.numel() for p in model.parameters()) == PARAMS[name]


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_state_dict_is_torchvisions_key_for_key(name):
    with torch.device("meta"):
        ours, theirs = PRESETS[name](), getattr(tvm, name)(stochastic_depth_prob=0.0)
    a, b = ours.state_dict(), theirs.state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape for k in a)
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in theirs.named_parameters()]


def test_loading_is_strict_both_ways():
    ours, theirs = convnext_tiny(), tvm.convnext_tiny(stochastic_depth_prob=0.0)
    ours.load_state_dict(theirs.state_dict(), strict=True)
    theirs.load_state_dict(ours.state_dict(), strict=True)
    assert all(torch.equal(p, q) for p, q in zip(ours.parameters(), theirs.parameters()))


def test_initialisation_is_torchvisions():
    """The same seed gives the same weights: the same modules are built in the same order and re-initialised alike."""
    torch.manual_seed(5)
    ours = convnext_tiny()
    torch.manual_seed(5)
    theirs = tvm.convnext_tiny(stochastic_depth_prob=0.0)
    for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
        assert torch.equal(p, q), n
    ls = ours.features[1][0].layer_scale
    assert ls.shape == (96, 1, 1) and bool((ls == 1e-6).all())
    assert float(ours.features[0][0].weight.detach().abs().max()) <= 2.0 and float(ours.classifier[2].bias.detach().abs().max()) == 0


def test_matches_torchvision_given_its_weights():
    """Forward and backward are torchvision's ops in torchvision's order: bitwise equal, or at worst 1e-5 relative."""
    torch.manual_seed(0)
    theirs = tvm.convnext_tiny(stochastic_depth_prob=0.0)
    with torch.no_grad():                                        # non-trivial layer scales, so every branch counts
        for m in theirs.modules():
            if hasattr(m, "layer_scale"):
                m.layer_scale.uniform_(0.1, 0.5)
    ours = convnext_tiny()
    ours.load_state_dict(theirs.state_dict(), strict=True)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 64, 96, generator=g)
    target = torch.randint(0, 1000, (2,), generator=g)
    a, b = ours(x), theirs(x)
    assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max())
    cross_entropy(a, target).backward()
    F.cross_entropy(b, target).backward()
    for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
        assert float((p.grad - q.grad).abs().max()) <= 1e-5 * float(q.grad.abs().max()) + 1e-30, n


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
@pytest.mark.parametrize("shape", [(1, 7, 7, 16), (2, 9, 13, 8), (1, 3, 5, 24)])
def test_depthwise_conv2d_on_cpu_is_the_reference(shape, layout):
    g = torch.Generator().manual_seed(sum(shape))
    B, H, W, C = shape
    x = torch.randn(B, H, W, C, generator=g, requires_grad=True)
    w = torch.randn(C, 1, 7, 7, generator=g)
    if layout == "channels_last":
        w = w.contiguous(memory_format=torch.channels_last)
    w.requires_grad_(True)
    b = torch.randn(C, generator=g, requires_grad=True)
    y = depthwise_conv2d(x, w, b)
    ref = F.conv2d(x.detach().permute(0, 3, 1, 2), w.detach(), b.detach(), padding=3, groups=C).permute(0, 2, 3, 1)
    assert y.shape == (B, H, W, C) and torch.equal(y, ref)
    assert torch.equal(depthwise_conv2d_reference(x, w, b), y)
    y.backward(torch.randn(y.shape, generator=g))
    assert x.grad.shape == x.shape and w.grad.shape == w.shape and b.grad.shape == b.shape


@pytest.mark.parametrize("p,layout", [(4, "nchw"), (4, "channels_last"), (2, "nhwc")])
def test_patch_gather_times_the_permuted_weight_is_the_convolution(p, layout):
    g = torch.Generator().manual_seed(p)
    C, D = (3, 16) if p == 4 else (8, 16)
    img = torch.randn(2, C, 8, 12, generator=g, dtype=torch.float64)
    w = torch.randn(D, C, p, p, generator=g, dtype=torch.float64)
    if layout == "channels_last":
        img = img.contiguous(memory_format=torch.channels_last)
    nhwc = img.permute(0, 2, 3, 1) if layout != "nhwc" else img.permute(0, 2, 3, 1).contiguous()
    rows = patchify_nhwc(nhwc, p)
    got = rows @ w.permute(0, 2, 3, 1).reshape(D, -1).t()
    ref = F.conv2d(img, w, stride=p).permute(0, 2, 3, 1).reshape(-1, D)
    assert rows.shape == (2 * (8 // p) * (12 // p), p * p * C)
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)
    with pytest.raises(ValueError, match="divisible"):
        patchify_nhwc(nhwc[:, :7], p)


def test_ddp_bucket_assignment_matches_torch():
    from b200ddp.parallel.buckets import assign_by_size, plan_buckets
    with torch.device("meta"):
        model = convnext_tiny()
    params = list(model.parameters())
    for cap in (1, 25):
        ref = dist._compute_bucket_assignment_by_size(params, [1 * MiB, cap * MiB])[0]
        assert assign_by_size([p.numel() * 4 for p in params], None, [1 * MiB, cap * MiB]) == ref
        specs = plan_buckets([p.numel() for p in params], [4] * len(params), bucket_cap_bytes=cap * MiB, order="torch",
                             max_tensors=10 ** 9)
        assert [s.param_indices for s in reversed(specs)] == ref


def test_registry_entries():
    for name in ("convnext-tiny", "convnext-small", "convnext-base"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "image" and e.config is None and e.start_id is None and not e.fp8 and not e.contrastive


def test_cli_rejects_fp8(tmp_path):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "convnext-tiny",
                                          "--no_cuda", "--fp8", "--fp16"])
    with pytest.raises(ValueError, match="--fp8"):
        cli.setup(args)


def test_ddp_py_cpu_training_run(tmp_path):
    cmd = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", "convnext-tiny", "--no_cuda", "--no_tensorboard",
           "--max_steps", "2", "--logging_steps", "1", "--save_steps", "0", "--per_gpu_train_batch_size", "2",
           "--dataset_size", "8", "--optimizer", "adamw", "--output_dir", str(tmp_path / "o")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="4"),
                         cwd=str(tmp_path))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "[Finished training.] [global_step=3]" in res.stdout
