"""CLIP on the GPU: QuickGELU, the row L2 normalisation and the fused contrastive cross-entropy element by element against
fp64 (``numerics`` bounds) and bitwise repeatable, ``clip_loss`` forward and backward against fp64 transformers
arithmetic, the native bf16 CLIP-ViT-B/32 against its fp32 torch path, no host synchronisation, and
``ddp.py --model clip-vit-b-32`` training under a CUDA graph with and without channels_last."""
import copy
import math

import pytest
import torch

import numerics as nm
from b200ddp.ops import clip_loss, linear

pytestmark = pytest.mark.gpu

U = nm.U


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def dev():
    return torch.device("cuda", 0)


def _quick64(z):
    return z * torch.sigmoid(1.702 * z)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n", [8 * 3072 * 4, 1001])
def test_quick_gelu_matches_fp64(C, dtype, n):
    g = torch.Generator().manual_seed(n)
    pre = (torch.randn(n, generator=g) * 3).to(dtype).to(dev())
    dy = torch.randn(n, generator=g).to(dtype).to(dev())
    y, dx = C.clip.quick_gelu_fwd(pre), C.clip.quick_gelu_bwd(dy, pre)
    z, d = pre.double(), dy.double()
    s = torch.sigmoid(1.702 * z)
    # __expf: a relative error growing with |1.702 z| (the exponent's rounding), carried through 1 / (1 + e) and the products
    grow = 8.0 * U * (1.0 + 2.0 * z.abs())
    nm.check("quick_gelu fwd", y, _quick64(z), nm.bound(_quick64(z), grow * (z.abs() + 1e-30), dtype), "quick_gelu")
    ref = d * (s + 1.702 * z * s * (1 - s))
    nm.check("quick_gelu bwd", dx, ref, nm.bound(ref, grow * (1.0 + 2.0 * z.abs()) * d.abs(), dtype), "quick_gelu")
    assert torch.equal(y, C.clip.quick_gelu_fwd(pre)) and torch.equal(dx, C.clip.quick_gelu_bwd(dy, pre))


def test_linear_quick_gelu_uses_the_native_pass():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 512, generator=g).to(dev(), torch.bfloat16).requires_grad_(True)
    w = (torch.randn(2048, 512, generator=g) * 0.05).to(dev(), torch.bfloat16).requires_grad_(True)
    b = (torch.randn(2048, generator=g) * 0.05).to(dev(), torch.bfloat16).requires_grad_(True)
    y = linear(x, w, b, activation="quick_gelu")
    dy = torch.randn_like(y)
    y.backward(dy)
    pre = (x.double() @ w.double().t() + b.double()).detach().requires_grad_(True)
    ref = _quick64(pre)
    ref.backward(dy.double())
    assert float((y.double() - ref).norm() / ref.norm()) < 1e-2
    assert float((x.grad.double() - pre.grad @ w.double()).norm() / (pre.grad @ w.double()).norm()) < 2e-2


@pytest.mark.parametrize("B,D", [(8, 512), (256, 512), (24, 768)])
def test_l2_normalisation_matches_fp64(C, B, D):
    g = torch.Generator().manual_seed(B + D)
    x = (torch.randn(B, D, generator=g) * 3).to(dev(), torch.bfloat16)
    du = torch.randn(B, D, generator=g).to(dev(), torch.bfloat16)
    u, rnorm = C.clip.l2norm_fwd(x)
    dx = C.clip.l2norm_bwd(du, x, rnorm)
    X, G = x.double(), du.double()
    rn = 1.0 / X.norm(dim=-1, keepdim=True)
    U64 = X * rn
    eps_r = (D / 2 + 4) * U                                      # the fp32 sum of squares and the square root
    nm.check("l2norm u", u, U64, nm.bound(U64, (eps_r + 2 * U) * U64.abs(), torch.bfloat16), "l2norm")
    nm.check("l2norm rnorm", rnorm, rn[:, 0], nm.bound(rn[:, 0], eps_r * rn[:, 0], torch.float32), "l2norm")
    dot = (U64 * G).sum(-1, keepdim=True)
    ref = rn * (G - U64 * dot)
    acc = rn * ((G.abs() + U64.abs() * dot.abs()) * (3 * eps_r + 8 * U) + U64.abs() * (D + 3) * U * (U64 * G).abs().sum(-1, keepdim=True))
    nm.check("l2norm dx", dx, ref, nm.bound(ref, acc, torch.bfloat16), "l2norm")
    u2, r2 = C.clip.l2norm_fwd(x)
    assert torch.equal(u, u2) and torch.equal(rnorm, r2) and torch.equal(dx, C.clip.l2norm_bwd(du, x, rnorm))


def _contrastive64(z_img, z_txt, ls, offset):
    """fp64: loss, dz_img, dz_txt, d logit_scale and their element-wise bounds."""
    B, N = z_img.shape
    s = math.exp(ls)
    labels = torch.arange(B, device=z_img.device) + offset
    out, bnds = [], []
    loss, dscale, acc_loss, acc_ds = 0.0, 0.0, 0.0, 0.0
    for z in (z_img.double(), z_txt.double()):
        p = torch.softmax(s * z, -1)
        onehot = torch.nn.functional.one_hot(labels, N).double()
        rows = torch.logsumexp(s * z, -1) - s * z.gather(1, labels[:, None])[:, 0]
        loss += float(rows.sum()) / (2 * B)
        dz = s * (p - onehot) / (2 * B)
        rel_p = (N + 8 + 16 * s) * U                              # exp of s z - max and the row sum, in fp32
        out.append(dz)
        bnds.append(s / (2 * B) * (p * rel_p + (p - onehot).abs() * 4 * U))
        terms = s / (2 * B) * ((p * z).sum(-1) - z.gather(1, labels[:, None])[:, 0])
        dscale += float(terms.sum())
        acc_ds += float((s / (2 * B) * (2 * N + 24 + 16 * s) * U * ((p * z.abs()).sum(-1) + z.abs().max(-1).values)).sum()
                        + 2 * B * U * terms.abs().sum())
        acc_loss += float(((N + 16 + 16 * s) * U + 2 * B * U * rows.abs()).sum()) / (2 * B)
    return loss, out[0], out[1], dscale, acc_loss, bnds[0], bnds[1], acc_ds


@pytest.mark.parametrize("B,world,rank", [(8, 1, 0), (256, 1, 0), (64, 4, 0), (64, 4, 3), (256, 8, 5)])
@pytest.mark.parametrize("ls", [2.6592, math.log(100.0)])
def test_contrastive_xent_matches_fp64(C, B, world, rank, ls):
    N = world * B
    g = torch.Generator().manual_seed(B * 31 + rank)
    uf = torch.nn.functional.normalize(torch.randn(N, 64, generator=g, dtype=torch.float64), dim=-1)
    vf = torch.nn.functional.normalize(uf + 0.5 * torch.randn(N, 64, generator=g, dtype=torch.float64), dim=-1)
    sl = slice(rank * B, (rank + 1) * B)
    z_img = (uf[sl] @ vf.t()).float().to(dev())
    z_txt = (vf[sl] @ uf.t()).float().to(dev())
    scale = torch.tensor([ls], dtype=torch.float32, device=dev())
    loss, dscale, dz_img, dz_txt = C.clip.contrastive_xent(z_img, z_txt, scale, rank * B)
    r_loss, r_dzi, r_dzt, r_ds, a_loss, b_dzi, b_dzt, a_ds = _contrastive64(z_img, z_txt, float(scale), rank * B)
    f64 = lambda v: torch.tensor(v, dtype=torch.float64)
    nm.check("contrastive loss", loss.cpu(), f64(r_loss), nm.bound(f64(r_loss), f64(a_loss), torch.float32), "contrastive")
    nm.check("contrastive dz_img", dz_img, r_dzi, nm.bound(r_dzi, b_dzi, torch.bfloat16), "contrastive")
    nm.check("contrastive dz_txt", dz_txt, r_dzt, nm.bound(r_dzt, b_dzt, torch.bfloat16), "contrastive")
    nm.check("contrastive dscale", dscale.cpu(), f64(r_ds), nm.bound(f64(r_ds), f64(a_ds), torch.float32), "contrastive")
    again = C.clip.contrastive_xent(z_img, z_txt, scale, rank * B)
    assert all(torch.equal(a, b) for a, b in zip((loss, dscale, dz_img, dz_txt), again))


@pytest.mark.parametrize("B", [8, 64])
def test_clip_loss_matches_fp64_transformers_formula(B):
    g = torch.Generator().manual_seed(B)
    img = torch.randn(B, 512, generator=g).to(dev(), torch.bfloat16).requires_grad_(True)
    txt = (img.detach().float() + torch.randn(B, 512, generator=g).to(dev())).to(torch.bfloat16).requires_grad_(True)
    scale = torch.tensor(2.6592, device=dev(), requires_grad=True)
    loss = clip_loss(img, txt, scale)
    loss.backward()
    I, T, S = (t.detach().double().requires_grad_(True) for t in (img, txt, scale))
    lpt = (T / T.norm(dim=-1, keepdim=True)) @ (I / I.norm(dim=-1, keepdim=True)).t() * S.exp()   # logits_per_text
    labels = torch.arange(B, device=dev())
    ref = (torch.nn.functional.cross_entropy(lpt, labels) + torch.nn.functional.cross_entropy(lpt.t(), labels)) / 2
    ref.backward()
    # bf16 features (one rounding of u) under fp32 accumulation: relative errors of a few bf16 units
    assert abs(float(loss) - float(ref)) <= 2e-2 * abs(float(ref))
    for got, want in ((img.grad, I.grad), (txt.grad, T.grad)):
        assert float((got.double() - want).norm() / want.norm()) < 3e-2
    assert abs(float(scale.grad) - float(S.grad)) <= 3e-2 * abs(float(S.grad)) + 1e-4


def test_clip_loss_rejects_what_the_native_path_cannot_run():
    x = torch.randn(12, 512, device=dev(), dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="B % 8"):
        clip_loss(x, x, torch.zeros((), device=dev()))
    with pytest.raises(ValueError, match="bf16"):
        clip_loss(x[:8].float(), x[:8].float(), torch.zeros((), device=dev()))


def _seeded_clip():
    from b200ddp.models import clip_vit_b_32
    torch.manual_seed(0)
    model = clip_vit_b_32()
    with torch.no_grad():                       # away from zero biases and unit norms
        for n, p in model.named_parameters():
            if n.endswith("bias"):
                p.normal_(0.0, 0.02)
    return model


def _pairs(B, seed=3):
    from b200ddp.data import SyntheticImageText
    ds = SyntheticImageText(samples=B, batch=B, seed=seed)
    ids = ds.Y.clone()
    ids[-1] = torch.where(ids[-1] == SyntheticImageText.EOT_ID, torch.ones_like(ids[-1]), ids[-1])   # one caption without EOT
    ids[0, 20:] = SyntheticImageText.EOT_ID                                                        # one padded with EOT
    return ds.X, ids


def test_native_bf16_clip_matches_the_fp32_torch_path():
    ref = _seeded_clip().to(dev())
    native = copy.deepcopy(ref)
    from b200ddp.utils.precision import to_mixed_bf16
    to_mixed_bf16(native)
    assert native.logit_scale.dtype == torch.float32
    x, ids = _pairs(16)
    x, ids = x.to(dev()), ids.to(dev())
    ri, rt, rs = ref(x, ids)
    ni, nt, ns = native(x.to(torch.bfloat16), ids)
    for a, b in ((ni, ri), (nt, rt)):
        assert float((a.float() - b).norm() / b.norm()) < 5e-2
    lr = clip_loss(ri.cpu(), rt.cpu(), rs.cpu())              # fp32 features: the torch body, on the CPU
    ln = clip_loss(ni, nt, ns)
    assert abs(float(ln) - float(lr)) < 5e-2 * max(1.0, abs(float(lr)))
    lr.backward()
    ln.backward()
    rel = float((native.logit_scale.grad - ref.logit_scale.grad).abs() / ref.logit_scale.grad.abs().clamp(min=1e-6))
    assert rel < 0.1


def test_clip_step_has_no_host_synchronisation():
    model = _seeded_clip().to(dev())
    from b200ddp.utils.precision import to_mixed_bf16
    to_mixed_bf16(model)
    x, ids = _pairs(8)
    x, ids = x.to(dev(), torch.bfloat16), ids.to(dev())
    clip_loss(*model(x, ids)).backward()
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = clip_loss(*model(x, ids))
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss)) and model.logit_scale.grad is not None


def _train(tmp_path, extra):
    """What `python ddp.py --model clip-vit-b-32 --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size 32
    --max_steps 30 --logging_steps 1 [extra]` runs on 64 pairs; returns every step's loss."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "clip-vit-b-32", "--fp16", "--cuda_graph", "--optimizer", "adamw", "--per_gpu_train_batch_size", "32",
            "--max_steps", "30", "--logging_steps", "1", "--dataset_size", "64", "--lr", "1e-4", "--warmup_steps", "2",
            "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    trainer = Trainer(args, build_model("clip-vit-b-32"), cli.log)
    sums = []
    read = trainer.step_fn.read_loss_sum
    trainer.step_fn.read_loss_sum = lambda: sums.append(read()) or sums[-1]
    trainer.train()
    assert trainer.step_fn.graph is not None
    return [b - a for a, b in zip([0.0] + sums[:-1], sums)][:30]


def test_ddp_training_under_a_cuda_graph(tmp_path, capsys):
    losses = _train(tmp_path / "a", [])
    cl = _train(tmp_path / "b", ["--channels_last"])
    with capsys.disabled():
        print(f"\nclip-vit-b-32 losses on {torch.cuda.get_device_name(dev())}: {[round(v, 4) for v in losses[::5]]}; "
              f"channels_last bitwise equal: {losses == cl}")
    assert all(math.isfinite(v) for v in losses)
    assert sum(losses[-5:]) / 5 < losses[0] - 0.3
    assert losses == cl
