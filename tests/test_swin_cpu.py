"""Swin on the CPU: torchvision's parameter counts, state dict key for key, initialisation, logits and gradients from the
same weights, the window-attention reference against torchvision's ``shifted_window_attention``, the relative position
index, the patch-merging gather, the DDP bucket plan, the registry, the CLI and a short ``ddp.py`` training run.

torchvision's ``swin_t()`` fixes ``stochastic_depth_prob=0.2``, so the reference models are its ``SwinTransformer`` built
with the same arguments and ``stochastic_depth_prob=0.0``."""
import copy
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from b200ddp.models import MODEL_REGISTRY, swin_b, swin_s, swin_t
from b200ddp.models.swin import merge_patches
from b200ddp.ops import cross_entropy, swin_relative_position_index, window_attention, window_attention_reference
from b200ddp.parallel.buckets import MiB

tvs = pytest.importorskip("torchvision.models.swin_transformer")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESETS = {"swin_t": swin_t, "swin_s": swin_s, "swin_b": swin_b}
PARAMS = {"swin_t": 28_288_354, "swin_s": 49_606_258, "swin_b": 87_768_224}
ARCH = {"swin_t": (96, [2, 2, 6, 2], [3, 6, 12, 24]), "swin_s": (96, [2, 2, 18, 2], [3, 6, 12, 24]),
        "swin_b": (128, [2, 2, 18, 2], [4, 8, 16, 32])}


def torchvision_swin(name):
    embed, depths, heads = ARCH[name]
    return tvs.SwinTransformer(patch_size=[4, 4], embed_dim=embed, depths=depths, num_heads=heads, window_size=[7, 7],
                               stochastic_depth_prob=0.0)


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_parameter_counts(name):
    with torch.device("meta"):
        model = PRESETS[name]()
    assert sum(p.numel() for p in model.parameters()) == PARAMS[name]


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_state_dict_is_torchvisions_key_for_key(name):
    with torch.device("meta"):
        ours, theirs = PRESETS[name](), torchvision_swin(name)
    a, b = ours.state_dict(), theirs.state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape and a[k].dtype == b[k].dtype for k in a)
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in theirs.named_parameters()]
    if name == "swin_t":
        assert len(a) == 185


def test_loading_is_strict_both_ways():
    ours, theirs = swin_t(), torchvision_swin("swin_t")
    ours.load_state_dict(theirs.state_dict(), strict=True)
    theirs.load_state_dict(ours.state_dict(), strict=True)
    assert all(torch.equal(p, q) for p, q in zip(ours.parameters(), theirs.parameters()))


def test_initialisation_is_torchvisions():
    """The same seed gives the same weights: the same modules are built in the same order and re-initialised alike."""
    torch.manual_seed(5)
    ours = swin_t()
    torch.manual_seed(5)
    theirs = torchvision_swin("swin_t")
    for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
        assert torch.equal(p, q), n
    for (n, p), q in zip(ours.named_buffers(), theirs.buffers()):
        assert torch.equal(p, q), n
    assert float(ours.head.weight.detach().abs().max()) <= 2.0 and float(ours.head.bias.detach().abs().max()) == 0
    assert float(ours.features[1][0].mlp[0].bias.detach().abs().max()) == 0


@pytest.mark.parametrize("size", [(96, 128), (60, 92)])
def test_matches_torchvision_given_its_weights(size):
    """Forward and backward are torchvision's ops in torchvision's order, padding included: bitwise equal, or at worst
    1e-5 relative."""
    torch.manual_seed(0)
    theirs = torchvision_swin("swin_t")
    with torch.no_grad():                                        # tables large enough to shape the attention
        for m in theirs.modules():
            if hasattr(m, "relative_position_bias_table"):
                m.relative_position_bias_table.normal_(0, 1)
    ours = swin_t()
    ours.load_state_dict(theirs.state_dict(), strict=True)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, *size, generator=g)
    target = torch.randint(0, 1000, (2,), generator=g)
    a, b = ours(x), theirs(x)
    assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max())
    cross_entropy(a, target).backward()
    F.cross_entropy(b, target).backward()
    for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
        assert float((p.grad - q.grad).abs().max()) <= 1e-5 * float(q.grad.abs().max()) + 1e-30, n


@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("B,H,W,heads", [(2, 14, 14, 3), (1, 21, 14, 2)])
def test_window_attention_reference_is_torchvisions(B, H, W, heads, shift):
    """qkv and proj applied outside: the reference on raster rows equals torchvision's shifted_window_attention."""
    g = torch.Generator().manual_seed(B + H + W + shift)
    C = 32 * heads
    x = torch.randn(B, H, W, C, generator=g, dtype=torch.float64)
    wqkv, bqkv = torch.randn(3 * C, C, generator=g, dtype=torch.float64) * C ** -0.5, torch.randn(3 * C, generator=g, dtype=torch.float64)
    wp, bp = torch.randn(C, C, generator=g, dtype=torch.float64) * C ** -0.5, torch.randn(C, generator=g, dtype=torch.float64)
    table = torch.randn(169, heads, generator=g, dtype=torch.float64)
    index = swin_relative_position_index()
    bias = table[index].view(49, 49, heads).permute(2, 0, 1).contiguous().unsqueeze(0)
    ref = tvs.shifted_window_attention(x, wqkv, wp, bias, [7, 7], heads, [shift, shift], qkv_bias=bqkv, proj_bias=bp)
    qkv = F.linear(x.reshape(-1, C), wqkv, bqkv)
    got = F.linear(window_attention_reference(qkv, table, B, H, W, heads, shift), wp, bp).view(B, H, W, C)
    assert torch.allclose(got, ref, rtol=1e-10, atol=1e-10)
    assert torch.equal(window_attention(qkv, table, B, H, W, heads, shift), window_attention_reference(qkv, table, B, H, W, heads, shift))


def test_relative_position_index_is_the_kernels_analytic_index():
    """Entry 49 i + j is (yi - yj + 6) 13 + (xi - xj + 6) = 13 ly_i + lx_i - (13 ly_j + lx_j) + 84, what the kernel uses."""
    tv = tvs.ShiftedWindowAttention(32, [7, 7], [0, 0], 1).relative_position_index
    ours = swin_relative_position_index()
    assert ours.dtype == torch.int64 and torch.equal(ours, tv)
    code = torch.tensor([13 * (i // 7) + i % 7 for i in range(49)])
    assert torch.equal(ours.view(49, 49), code[:, None] - code[None, :] + 84)
    assert int(ours.min()) == 0 and int(ours.max()) == 168


def test_patch_merging_gather_is_torchvisions_order():
    """(kx, ky, c): x0 = (0, 0), x1 = (1, 0), x2 = (0, 1), x3 = (1, 1) as (row, column) offsets."""
    x = torch.arange(2 * 4 * 6 * 3, dtype=torch.float32).view(2, 4, 6, 3)
    got = merge_patches(x)
    assert torch.equal(got, tvs._patch_merging_pad(x))
    assert torch.equal(got[0, 0, 0], torch.cat([x[0, 0, 0], x[0, 1, 0], x[0, 0, 1], x[0, 1, 1]]))


def test_window_attention_rejects_bad_shifts():
    qkv = torch.zeros(49, 96)
    with pytest.raises(ValueError, match="shift"):
        window_attention(qkv, torch.zeros(169, 1), 1, 7, 7, 1, 7)


def test_ddp_bucket_assignment_matches_torch():
    from b200ddp.parallel.buckets import assign_by_size, plan_buckets
    with torch.device("meta"):
        model = swin_t()
    params = list(model.parameters())
    for cap in (1, 25):
        ref = dist._compute_bucket_assignment_by_size(params, [1 * MiB, cap * MiB])[0]
        assert assign_by_size([p.numel() * 4 for p in params], None, [1 * MiB, cap * MiB]) == ref
        specs = plan_buckets([p.numel() for p in params], [4] * len(params), bucket_cap_bytes=cap * MiB, order="torch",
                             max_tensors=10 ** 9)
        assert [s.param_indices for s in reversed(specs)] == ref


def test_registry_entries():
    for name in ("swin-t", "swin-s", "swin-b"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "image" and e.config is None and e.start_id is None and not e.fp8 and not e.contrastive


def _setup(tmp_path, extra):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "swin-t",
                                          "--no_cuda", *extra])
    cli.setup(args)
    return args


def test_cli_takes_the_image_flags(tmp_path):
    args = _setup(tmp_path, ["--fp16", "--channels_last", "--cuda_graph"])
    assert args.model == "swin-t" and args.channels_last and args.cuda_graph


@pytest.mark.parametrize("extra,flag", [(["--fp8", "--fp16"], "--fp8"), (["--pack"], "--pack"), (["--min_seq_len", "8"], "--min_seq_len")])
def test_cli_rejects_fp8_and_token_flags(tmp_path, extra, flag):
    with pytest.raises(ValueError, match=flag):
        _setup(tmp_path, extra)


def test_ddp_py_cpu_training_run(tmp_path):
    cmd = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", "swin-t", "--no_cuda", "--no_tensorboard",
           "--max_steps", "2", "--logging_steps", "1", "--save_steps", "0", "--per_gpu_train_batch_size", "2",
           "--dataset_size", "8", "--optimizer", "adamw", "--output_dir", str(tmp_path / "o")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="4"),
                         cwd=str(tmp_path))
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "[Finished training.] [global_step=3]" in res.stdout


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _small_swin():
    from b200ddp.models.swin import SwinConfig, SwinTransformer
    torch.manual_seed(0)
    return SwinTransformer(SwinConfig(embed_dim=32, depths=(2, 2), heads=(1, 2), num_classes=10)).double()


def _gloo_worker(rank, world, port, path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200ddp.parallel import DistributedDataParallel
        model = _small_swin()
        g = torch.Generator().manual_seed(7)
        x, y = torch.randn(4, 3, 56, 56, generator=g, dtype=torch.float64), torch.randint(0, 10, (4,), generator=g)
        full = copy.deepcopy(model)
        cross_entropy(full(x), y).backward()                    # the mean over the global batch
        ddp = DistributedDataParallel(model, backend="gloo", bucket_cap_mb=0.05, first_bucket_mb=0.01)
        n = x.shape[0] // world
        cross_entropy(ddp(x[rank * n:(rank + 1) * n]), y[rank * n:(rank + 1) * n]).backward()
        if rank == 0:
            torch.save({"buckets": len(ddp._specs), "ddp": {k: p.grad.clone() for k, p in model.named_parameters()},
                        "full": {k: p.grad.clone() for k, p in full.named_parameters()}}, path)
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_gradients_match_the_full_batch(tmp_path):
    """The bucketed all-reduce of a small Swin's gradients (tables included) over two gloo ranks, in several buckets,
    equals the single-process gradient of the whole batch."""
    path = tmp_path / "grads.pt"
    mp.spawn(_gloo_worker, args=(2, _free_port(), str(path)), nprocs=2, join=True)
    got = torch.load(path)
    assert got["buckets"] > 1 and list(got["ddp"]) == list(got["full"])
    for k, g in got["ddp"].items():
        assert torch.allclose(g, got["full"][k], rtol=1e-9, atol=1e-15), k
