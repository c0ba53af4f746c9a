"""Swin V2 on the CPU: torchvision's parameter counts, state dict key for key, initialisation, logits and gradients from the
same weights in fp64, the cosine window-attention reference against torchvision's ``shifted_window_attention`` with
``logit_scale``, the relative position index and coordinates table, the k bias's zero gradient, the DDP bucket plan, the
registry, the CLI and a short ``ddp.py`` training run.

torchvision's ``swin_v2_t()`` fixes ``stochastic_depth_prob=0.2``, so the reference models are its ``SwinTransformer``
built with the same arguments, ``SwinTransformerBlockV2``, ``PatchMergingV2`` and ``stochastic_depth_prob=0.0``."""
import copy
import math
import os
import socket
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from b200ddp.models import MODEL_REGISTRY, swin_v2_b, swin_v2_s, swin_v2_t
from b200ddp.ops import (cross_entropy, swin_relative_position_index, swin_v2_relative_coords_table, window_attention_v2,
                         window_attention_v2_reference)
from b200ddp.parallel.buckets import MiB

tvs = pytest.importorskip("torchvision.models.swin_transformer")
tvm = pytest.importorskip("torchvision.models")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESETS = {"swin_v2_t": swin_v2_t, "swin_v2_s": swin_v2_s, "swin_v2_b": swin_v2_b}
ARCH = {"swin_v2_t": (96, [2, 2, 6, 2], [3, 6, 12, 24]), "swin_v2_s": (96, [2, 2, 18, 2], [3, 6, 12, 24]),
        "swin_v2_b": (128, [2, 2, 18, 2], [4, 8, 16, 32])}
ENTRIES = {"swin_v2_t": 233, "swin_v2_s": 449, "swin_v2_b": 449}


def torchvision_swin_v2(name):
    embed, depths, heads = ARCH[name]
    return tvs.SwinTransformer(patch_size=[4, 4], embed_dim=embed, depths=depths, num_heads=heads, window_size=[8, 8],
                               stochastic_depth_prob=0.0, block=tvs.SwinTransformerBlockV2, downsample_layer=tvs.PatchMergingV2)


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_parameter_counts_are_torchvisions(name):
    with torch.device("meta"):
        ours, theirs = PRESETS[name](), getattr(tvm, name)()
    n = sum(p.numel() for p in ours.parameters())
    assert n == sum(p.numel() for p in theirs.parameters())
    assert n == {"swin_v2_t": 28_351_570, "swin_v2_s": 49_737_442, "swin_v2_b": 87_930_848}[name]


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_state_dict_is_torchvisions_key_for_key(name):
    with torch.device("meta"):
        ours, theirs = PRESETS[name](), getattr(tvm, name)()
    a, b = ours.state_dict(), theirs.state_dict()
    assert list(a) == list(b) and len(a) == ENTRIES[name]
    assert all(a[k].shape == b[k].shape and a[k].dtype == b[k].dtype for k in a)
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in theirs.named_parameters()]
    assert [n for n, _ in ours.named_buffers()] == [n for n, _ in theirs.named_buffers()]


def test_loading_is_strict_both_ways():
    ours, theirs = swin_v2_t(), torchvision_swin_v2("swin_v2_t")
    ours.load_state_dict(theirs.state_dict(), strict=True)
    theirs.load_state_dict(ours.state_dict(), strict=True)
    assert all(torch.equal(p, q) for p, q in zip(ours.parameters(), theirs.parameters()))


def test_initialisation_is_torchvisions():
    """The same seed gives the same weights and buffers: the same modules are built in the same order and re-initialised
    alike, the k third of every qkv bias is zero and every logit_scale is log 10."""
    torch.manual_seed(5)
    ours = swin_v2_t()
    torch.manual_seed(5)
    theirs = torchvision_swin_v2("swin_v2_t")
    for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
        assert torch.equal(p, q), n
    for (n, p), q in zip(ours.named_buffers(), theirs.buffers()):
        assert p.dtype == q.dtype and torch.equal(p, q), n
    attn = ours.features[1][0].attn
    assert torch.equal(attn.logit_scale, torch.full((3, 1, 1), math.log(10.0)))
    assert float(attn.qkv.bias.detach()[96:192].abs().max()) == 0.0
    assert float(attn.cpb_mlp[0].weight.detach().abs().max()) <= 2.0


def _seeded_pair(seed=0):
    torch.manual_seed(seed)
    theirs = torchvision_swin_v2("swin_v2_t")
    with torch.no_grad():                                        # scales and tables large enough to shape the attention
        for m in theirs.modules():
            if hasattr(m, "logit_scale"):
                m.logit_scale.add_(torch.randn_like(m.logit_scale))
                m.cpb_mlp[2].weight.normal_(0, 0.5)
                m.qkv.bias.normal_(0, 0.1)
    ours = swin_v2_t()
    ours.load_state_dict(theirs.state_dict(), strict=True)
    return ours.double(), theirs.double()


@pytest.mark.parametrize("size", [(64, 96), (60, 92)])
def test_matches_torchvision_given_its_weights_in_fp64(size):
    """Forward, loss and every gradient are torchvision's ops in torchvision's order, padding included (60 x 92 is not a
    multiple of 8 at any stage): equal to 1e-12 relative in fp64."""
    ours, theirs = _seeded_pair()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, *size, generator=g, dtype=torch.float64)
    target = torch.randint(0, 1000, (2,), generator=g)
    a, b = ours(x), theirs(x)
    assert float((a - b).abs().max()) <= 1e-12 * float(b.abs().max())
    la, lb = F.cross_entropy(a, target), F.cross_entropy(b, target)          # fp64 (ops.cross_entropy takes fp32 on the CPU)
    assert abs(float(la) - float(lb)) <= 1e-12 * abs(float(lb))
    la.backward()
    lb.backward()
    for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
        assert float((p.grad - q.grad).abs().max()) <= 1e-12 * float(q.grad.abs().max()) + 1e-30, n


def test_k_bias_gets_a_zero_gradient():
    ours, _ = _seeded_pair()
    x = torch.randn(1, 3, 64, 64, dtype=torch.float64)
    ours(x).square().mean().backward()
    for m in ours.modules():
        if hasattr(m, "logit_scale"):
            C = m.qkv.weight.shape[1]
            g = m.qkv.bias.grad
            assert float(g[C:2 * C].abs().max()) == 0.0 and float(g[:C].abs().max()) > 0 and float(g[2 * C:].abs().max()) > 0


@pytest.mark.parametrize("shift", [0, 4])
@pytest.mark.parametrize("B,H,W,heads", [(2, 16, 16, 3), (1, 24, 16, 2)])
def test_window_attention_v2_reference_is_torchvisions(B, H, W, heads, shift):
    """qkv and proj applied outside: the reference on raster rows equals torchvision's shifted_window_attention with
    logit_scale, given the same table, and with a logit scale above log 100 (the clamp) on one head."""
    g = torch.Generator().manual_seed(B + H + W + shift)
    C = 32 * heads
    x = torch.randn(B, H, W, C, generator=g, dtype=torch.float64)
    wqkv, bqkv = torch.randn(3 * C, C, generator=g, dtype=torch.float64) * C ** -0.5, torch.randn(3 * C, generator=g, dtype=torch.float64)
    bqkv[C:2 * C] = 0                                              # torchvision zeroes it at every call
    wp, bp = torch.randn(C, C, generator=g, dtype=torch.float64) * C ** -0.5, torch.randn(C, generator=g, dtype=torch.float64)
    table = 16 * torch.sigmoid(torch.randn(225, heads, generator=g, dtype=torch.float64))
    logit = torch.randn(heads, 1, 1, generator=g, dtype=torch.float64) + math.log(10.0)
    logit[0] = math.log(100.0) + 0.5
    scale = torch.clamp(logit, max=math.log(100.0)).exp().view(-1)
    index = swin_relative_position_index(window=8)
    bias = table[index].view(64, 64, heads).permute(2, 0, 1).contiguous().unsqueeze(0)
    ref = tvs.shifted_window_attention(x, wqkv, wp, bias, [8, 8], heads, [shift, shift], qkv_bias=bqkv, proj_bias=bp, logit_scale=logit)
    qkv = F.linear(x.reshape(-1, C), wqkv, bqkv)
    got = F.linear(window_attention_v2_reference(qkv, table, scale, B, H, W, heads, shift), wp, bp).view(B, H, W, C)
    assert torch.allclose(got, ref, rtol=1e-10, atol=1e-10)
    assert torch.equal(window_attention_v2(qkv, table, scale, B, H, W, heads, shift),
                       window_attention_v2_reference(qkv, table, scale, B, H, W, heads, shift))


def test_relative_position_index_is_the_kernels_analytic_index():
    """Entry 64 i + j is (yi - yj + 7) 15 + (xi - xj + 7) = 15 ly_i + lx_i - (15 ly_j + lx_j) + 112, what the kernel uses,
    and torchvision's buffer; the default window is still V1's 7."""
    tv = tvs.ShiftedWindowAttentionV2(32, [8, 8], [0, 0], 1).relative_position_index
    ours = swin_relative_position_index(window=8)
    assert ours.dtype == torch.int64 and ours.shape == (4096,) and torch.equal(ours, tv)
    code = torch.tensor([15 * (i // 8) + i % 8 for i in range(64)])
    assert torch.equal(ours.view(64, 64), code[:, None] - code[None, :] + 112)
    assert int(ours.min()) == 0 and int(ours.max()) == 224
    assert torch.equal(swin_relative_position_index(), tvs.ShiftedWindowAttention(32, [7, 7], [0, 0], 1).relative_position_index)


def test_relative_coords_table_is_torchvisions():
    tv = tvs.ShiftedWindowAttentionV2(32, [8, 8], [0, 0], 1).relative_coords_table
    ours = swin_v2_relative_coords_table()
    assert ours.shape == (1, 15, 15, 2) and ours.dtype == torch.float32 and torch.equal(ours, tv)


def test_window_attention_v2_rejects_bad_shifts():
    qkv = torch.zeros(64, 96)
    with pytest.raises(ValueError, match="shift"):
        window_attention_v2(qkv, torch.zeros(225, 1), torch.ones(1), 1, 8, 8, 1, 8)


def test_logit_scale_and_cpb_mlp_stay_fp32_under_bf16():
    from b200ddp.utils import to_mixed_bf16
    model = to_mixed_bf16(swin_v2_t())
    attn = model.features[1][0].attn
    assert attn.logit_scale.dtype == attn.cpb_mlp[0].weight.dtype == attn.cpb_mlp[0].bias.dtype == attn.cpb_mlp[2].weight.dtype == torch.float32
    assert attn.qkv.weight.dtype == torch.bfloat16
    # the bf16 buffer is not what the MLP reads: it reads the exact fp32 table
    assert attn.relative_coords_table.dtype == torch.bfloat16
    ref = 16 * torch.sigmoid(attn.cpb_mlp(swin_v2_relative_coords_table()).view(-1, 3))
    assert torch.equal(attn.bias_table(), ref)


def test_ddp_bucket_assignment_matches_torch():
    from b200ddp.parallel.buckets import assign_by_size, plan_buckets
    with torch.device("meta"):
        model = swin_v2_t()
    params = list(model.parameters())
    for cap in (1, 25):
        ref = dist._compute_bucket_assignment_by_size(params, [1 * MiB, cap * MiB])[0]
        assert assign_by_size([p.numel() * 4 for p in params], None, [1 * MiB, cap * MiB]) == ref
        specs = plan_buckets([p.numel() for p in params], [4] * len(params), bucket_cap_bytes=cap * MiB, order="torch",
                             max_tensors=10 ** 9)
        assert [s.param_indices for s in reversed(specs)] == ref


def test_registry_entries():
    for name in ("swin-v2-t", "swin-v2-s", "swin-v2-b"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "image" and e.image_size == 256 and e.config is None and e.start_id is None and not e.fp8
        assert not e.contrastive and not e.own_loss
    assert all(e.image_size == 224 for n, e in MODEL_REGISTRY.items() if not n.startswith("swin-v2"))


def test_training_data_is_256_square():
    from b200ddp.engine.trainer import build_dataset
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--model", "swin-v2-t", "--no_cuda", "--dataset_size", "4"])
    x, _ = build_dataset(args)[0]
    assert tuple(x.shape) == (3, 256, 256)


def _setup(tmp_path, extra):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "swin-v2-t",
                                          "--no_cuda", *extra])
    cli.setup(args)
    return args


def test_cli_takes_the_image_flags(tmp_path):
    args = _setup(tmp_path, ["--fp16", "--channels_last", "--cuda_graph"])
    assert args.model == "swin-v2-t" and args.channels_last and args.cuda_graph


@pytest.mark.parametrize("extra,flag", [(["--fp8", "--fp16"], "--fp8"), (["--pack"], "--pack"), (["--min_seq_len", "8"], "--min_seq_len")])
def test_cli_rejects_fp8_and_token_flags(tmp_path, extra, flag):
    with pytest.raises(ValueError, match=flag):
        _setup(tmp_path, extra)


def test_ddp_py_cpu_training_run(tmp_path):
    cmd = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", "swin-v2-t", "--no_cuda", "--no_tensorboard",
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


def _small_swin_v2():
    from b200ddp.models.swin import SwinConfig, SwinTransformer
    torch.manual_seed(0)
    return SwinTransformer(SwinConfig(embed_dim=32, depths=(2, 2), heads=(1, 2), num_classes=10, window=8, v2=True)).double()


def _gloo_worker(rank, world, port, path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200ddp.parallel import DistributedDataParallel
        model = _small_swin_v2()
        g = torch.Generator().manual_seed(7)
        x, y = torch.randn(4, 3, 64, 64, generator=g, dtype=torch.float64), torch.randint(0, 10, (4,), generator=g)
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
    """The bucketed all-reduce of a small Swin V2's gradients (logit scales and cpb MLPs included) over two gloo ranks, in
    several buckets, equals the single-process gradient of the whole batch."""
    path = tmp_path / "grads.pt"
    mp.spawn(_gloo_worker, args=(2, _free_port(), str(path)), nprocs=2, join=True)
    got = torch.load(path)
    assert got["buckets"] > 1 and list(got["ddp"]) == list(got["full"])
    for k, g in got["ddp"].items():
        assert torch.allclose(g, got["full"][k], rtol=1e-9, atol=1e-15), k
