"""ViT-MAE on the GPU: the masked-autoencoder kernels (shuffle, masked patch embedding, unshuffle, head-dim-32 image
attention, reconstruction loss) element by element against fp64 with tests/numerics.py's bounds and bitwise repeatable, the
native bf16 vit-mae-base against its own fp32 path, no host synchronisation, CUDA-graph replay equal to eager, and
``ddp.py --model vit-mae-base`` training."""
import copy
import math

import pytest
import torch

import numerics as nm
from b200ddp.models import vit_mae_base
from b200ddp.models.vit_mae import ViTMAEConfig, ViTMAEForPreTraining
from b200ddp.ops import (image_attention, image_token_rows, mae_loss, mae_loss_reference, mae_patch_embed, mae_patchify, mae_shuffle,
                         mae_unshuffle)

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda", 0)


def stable_ranks(noise, keep):
    ids_shuffle = torch.argsort(noise, dim=1, stable=True)
    return ids_shuffle[:, :keep], torch.argsort(ids_shuffle, dim=1)


@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("keep", [1, 49, 196])
def test_shuffle_is_the_stable_argsort(B, keep):
    g = torch.Generator(device="cpu").manual_seed(B * 1000 + keep)
    noise = torch.rand(B, 196, generator=g)
    noise[:, ::7] = noise[:, 3:4]                               # forced ties, broken by patch index
    if B > 1:
        noise[1] = 0.5                                          # an image of one value
    ids_keep, ids_restore = mae_shuffle(noise.to(dev()), keep)
    ref_keep, ref_restore = stable_ranks(noise, keep)
    assert torch.equal(ids_keep.cpu().long(), ref_keep) and torch.equal(ids_restore.cpu().long(), ref_restore)


def _images(B, cl, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, 3, 224, 224, generator=g).to(dev(), torch.bfloat16)
    return x.contiguous(memory_format=torch.channels_last) if cl else x


@pytest.mark.parametrize("cl", [False, True])
def test_masked_patch_embed_against_fp64(cl):
    B, keep, D = 3, 49, 768
    g = torch.Generator(device="cpu").manual_seed(1)
    images = _images(B, cl)
    w = (torch.randn(D, 3, 16, 16, generator=g) * 0.02).to(dev(), torch.bfloat16).requires_grad_()
    b = (torch.randn(D, generator=g) * 0.02).to(dev(), torch.bfloat16).requires_grad_()
    cls = (torch.randn(1, 1, D, generator=g) * 0.02).to(dev(), torch.bfloat16).requires_grad_()
    pos = torch.randn(1, 197, D, generator=g).to(dev(), torch.bfloat16)
    ids_keep, _ = mae_shuffle(torch.rand(B, 196, generator=g).to(dev()), keep)
    out = mae_patch_embed(images, w, b, cls, pos, ids_keep)
    T = image_token_rows(B, keep + 1)
    assert out.shape == (T, D)
    # fp64: the kept patches times the weight, + bias (the GEMM output rounded to bf16), + pos
    patches = mae_patchify(images.float(), 16).view(B, 196, 16, 16, 3).permute(0, 1, 4, 2, 3).reshape(B, 196, -1)
    kept = torch.gather(patches, 1, ids_keep.long()[..., None].expand(-1, -1, 768)).reshape(-1, 768)
    y, acc = nm.gemm_reference(kept, w.detach().reshape(D, -1), b.detach(), epilogue=1)
    acc = acc * (1 + nm.rounding(torch.bfloat16)) + nm.rounding(torch.bfloat16) * y.abs()   # the GEMM's bf16 output
    posk = torch.gather(pos.double()[0, 1:].expand(B, -1, -1), 1, ids_keep.long()[..., None].expand(-1, -1, D)).reshape(-1, D)
    got = out.view(-1, D)[:B * (keep + 1)].view(B, keep + 1, D)
    ref = (y + posk).view(B, keep, D)
    nm.check("mae patch rows", got[:, 1:], ref, nm.bound(ref, acc.view(B, keep, D), torch.bfloat16))
    ref_cls = (cls.double() + pos.double()[:, :1]).expand(B, 1, D)
    nm.check("mae class rows", got[:, :1], ref_cls, nm.bound(ref_cls, torch.zeros_like(ref_cls), torch.bfloat16))
    assert torch.all(out[B * (keep + 1):] == 0)
    dy = torch.randn(T, D, generator=g).to(dev(), torch.bfloat16)
    out.backward(dy)
    d = dy.double()[:B * (keep + 1)].view(B, keep + 1, D)
    ref_dcls = d[:, 0].sum(0).view(1, 1, D)
    nm.check("mae d cls", cls.grad, ref_dcls, nm.bound(ref_dcls, B * nm.U * d[:, 0].abs().sum(0).view(1, 1, D), torch.bfloat16))
    ref_db = d[:, 1:].sum((0, 1))
    assert torch.allclose(b.grad.double(), ref_db, rtol=2 ** -6, atol=1e-2)
    # the weight gradient, element by element: sum over the kept patches of dy[its row] x the patch, so a patch row
    # routed to the wrong stream row (patchify) or a misplaced dpatch row (the backward) shows
    dyp = d[:, 1:].reshape(-1, D)
    nm.check_gemm("mae d weight", w.grad.reshape(D, -1), dyp.t().contiguous(), kept.t().contiguous())
    grads = (w.grad.clone(), b.grad.clone(), cls.grad.clone())
    w.grad = b.grad = cls.grad = None
    out2 = mae_patch_embed(images, w, b, cls, pos, ids_keep)
    out2.backward(dy)
    assert torch.equal(out, out2) and all(torch.equal(a, c) for a, c in zip(grads, (w.grad, b.grad, cls.grad)))


@pytest.mark.parametrize("B", [1, 3, 64])
def test_unshuffle_against_fp64(B):
    keep, N, E = 49, 196, 512
    g = torch.Generator(device="cpu").manual_seed(B)
    Te = image_token_rows(B, keep + 1)
    y = torch.randn(Te, E, generator=g).to(dev(), torch.bfloat16).requires_grad_()
    mask = torch.randn(1, 1, E, generator=g).to(dev(), torch.bfloat16).requires_grad_()
    pos = torch.randn(1, N + 1, E, generator=g).to(dev(), torch.bfloat16)
    ids_keep, ids_restore = mae_shuffle(torch.rand(B, N, generator=g).to(dev()), keep)
    z = mae_unshuffle(y, mask, pos, ids_keep, ids_restore)
    Td = image_token_rows(B, N + 1)
    assert z.shape == (Td, E)
    yd = y.detach().double()[:B * (keep + 1)].view(B, keep + 1, E)
    src = torch.cat([yd[:, 1:], mask.detach().double().expand(B, N - keep, E)], 1)
    src = torch.gather(src, 1, ids_restore.long()[..., None].expand(-1, -1, E))
    ref = torch.cat([yd[:, :1], src], 1) + pos.double()
    nm.check("mae unshuffle", z[:B * (N + 1)].view(B, N + 1, E), ref, nm.bound(ref, torch.zeros_like(ref), torch.bfloat16))
    assert torch.all(z[B * (N + 1):] == 0)
    dz = torch.randn(Td, E, generator=g).to(dev(), torch.bfloat16)
    z.backward(dz)
    d = dz.double()[:B * (N + 1)].view(B, N + 1, E)
    ref_dy = torch.cat([d[:, :1], torch.gather(d[:, 1:], 1, ids_keep.long()[..., None].expand(-1, -1, E))], 1)
    assert torch.equal(y.grad[:B * (keep + 1)].double().view(B, keep + 1, E), ref_dy)
    assert torch.all(y.grad[B * (keep + 1):] == 0)
    masked = (ids_restore.long() >= keep)[..., None]
    ref_dm = torch.where(masked, d[:, 1:], 0.0).sum((0, 1)).view(1, 1, E)
    acc = B * N * nm.U * torch.where(masked, d[:, 1:].abs(), 0.0).sum((0, 1)).view(1, 1, E)
    nm.check("mae d mask_token", mask.grad, ref_dm, nm.bound(ref_dm, acc, torch.bfloat16))
    gm = mask.grad.clone()
    mask.grad = None
    mae_unshuffle(y, mask, pos, ids_keep, ids_restore).backward(dz)
    assert torch.equal(gm, mask.grad)


def _attention_case(B, tokens, heads, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    T = image_token_rows(B, tokens)
    qkv = torch.randn(T, 96 * heads, generator=g).to(dev(), torch.bfloat16)
    qkv[B * tokens:] = float("nan")                              # padding rows are never read
    return qkv, torch.randn(T, 32 * heads, generator=g).to(dev(), torch.bfloat16), T


@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("tokens", [1, 50, 197, 256])
def test_image_attention_against_fp64(B, tokens):
    heads = 16 if B < 64 else 4
    qkv, dout, T = _attention_case(B, tokens, heads, B * 7 + tokens)
    x = qkv.clone().requires_grad_()
    o = image_attention(x, B, tokens, heads)
    o.backward(dout)
    assert torch.all(o[B * tokens:] == 0) and torch.all(x.grad[B * tokens:] == 0)
    S = 256                                                       # images padded to the numerics references' key tile
    C = 32 * heads

    def per_image(t, cols):                                       # [B, heads, S, 32], rows past tokens zero
        v = torch.zeros(B, S, cols, dtype=t.dtype, device=t.device)
        v[:, :tokens] = t[:B * tokens].view(B, tokens, cols)
        return v.view(B, S, cols // 32, 32).transpose(1, 2)

    q, k, v = (per_image(qkv[:, i * C:(i + 1) * C], C) for i in range(3))
    j = torch.arange(S, device=dev())
    visible = ((j[None, :] < tokens) & (j[:, None] < tokens)).expand(B, S, S).contiguous()
    ref = nm.attention_reference(q, k, v, visible, 32 ** -0.5)
    r, a = ref["o"]
    got = per_image(o.detach(), C)
    nm.check("image_attention o", got[:, :, :tokens], r[:, :, :tokens], nm.bound(r, a, torch.bfloat16)[:, :, :tokens])
    from b200ddp import _ext
    o_k, lse_k = _ext.get().mae.attention_fwd(qkv, B, tokens)
    lse4 = torch.full((B, heads, S), -math.inf, dtype=torch.float32, device=dev())
    lse4[:, :, :tokens] = lse_k[:B * tokens].view(B, tokens, heads).transpose(1, 2)
    bref = nm.attention_bwd_reference(q, k, v, per_image(o_k, C), lse4, per_image(dout, C), visible, 32 ** -0.5)
    for i, name in enumerate(("dq", "dk", "dv")):
        r, a = bref[name]
        g_ = per_image(x.grad[:, i * C:(i + 1) * C], C)
        nm.check(f"image_attention {name}", g_[:, :, :tokens], r[:, :, :tokens], nm.bound(r, a, torch.bfloat16)[:, :, :tokens])
    x2 = qkv.clone().requires_grad_()
    o2 = image_attention(x2, B, tokens, heads)
    o2.backward(dout)
    assert torch.equal(o, o2) and torch.equal(x.grad, x2.grad)


@pytest.mark.parametrize("norm_pix", [False, True])
@pytest.mark.parametrize("cl", [False, True])
def test_mae_loss_against_fp64(norm_pix, cl):
    B, N, keep = 3, 196, 49
    g = torch.Generator(device="cpu").manual_seed(int(norm_pix) * 2 + int(cl))
    images = _images(B, cl, seed=5)
    Td = image_token_rows(B, N + 1)
    pred = torch.randn(Td, 768, generator=g).to(dev(), torch.bfloat16).requires_grad_()
    _, ids_restore = mae_shuffle(torch.rand(B, N, generator=g).to(dev()), keep)
    loss = mae_loss(pred, images, ids_restore, keep, norm_pix)
    ref = mae_loss_reference(pred.detach().double(), images.double(), ids_restore.long(), keep, norm_pix)
    assert abs(float(loss) - float(ref)) <= 64 * nm.U * abs(float(ref)) + 1e-6
    gscale = torch.tensor(0.37, device=dev())
    (loss * gscale).backward()
    pd = pred.detach().double().requires_grad_()
    (mae_loss_reference(pd, images.double(), ids_restore.long(), keep, norm_pix) * 0.37).backward()
    r = pd.grad
    acc = 64 * nm.U * r.abs() + 2 ** -20 * r.abs().max()
    nm.check("mae dpred", pred.grad, r, nm.bound(r, acc, torch.bfloat16))
    rows = torch.arange(Td, device=dev())
    b, j = rows // (N + 1), rows % (N + 1)
    masked = (b < B) & (j > 0)
    masked[masked.clone()] = ids_restore.view(-1).long()[(b * N + j - 1)[masked]] >= keep
    assert torch.all(pred.grad[~masked] == 0)
    dp = pred.grad.clone()
    pred.grad = None
    loss2 = mae_loss(pred, images, ids_restore, keep, norm_pix)
    (loss2 * gscale).backward()
    assert torch.equal(loss, loss2) and torch.equal(dp, pred.grad)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.mark.parametrize("norm_pix", [False, True])
def test_native_bf16_matches_fp32_path(norm_pix):
    torch.manual_seed(0)
    ref = ViTMAEForPreTraining(ViTMAEConfig(norm_pix_loss=norm_pix)).to(dev())
    model = copy.deepcopy(ref).to(torch.bfloat16)
    images = _images(4, False, seed=3)
    noise = torch.rand(4, 196, device=dev())
    l_ref = ref(images.float(), noise)
    l_ref.backward()
    l = model(images, noise)
    l.backward()
    assert abs(float(l) - float(l_ref)) <= 0.02 * abs(float(l_ref))
    for (name, p), (_, q) in zip(model.named_parameters(), ref.named_parameters()):
        if not p.requires_grad:
            assert p.grad is None
            continue
        assert _rel(p.grad, q.grad) < 0.06, name


def test_no_host_synchronisation_and_graph_replay_is_bitwise():
    torch.manual_seed(0)
    model = vit_mae_base().to(dev(), torch.bfloat16)
    images = _images(8, True, seed=4)
    noise = torch.rand(8, 196, device=dev())

    def step():
        for p in model.parameters():
            p.grad = None
        loss = model(images, noise)
        loss.backward()
        return loss.detach().clone(), [p.grad.clone() for p in model.parameters() if p.requires_grad]

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager_loss, eager_grads = step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    for p in model.parameters():
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = model(images, noise)
        loss.backward()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, eager_loss)
    for p, g in zip([p for p in model.parameters() if p.requires_grad], eager_grads):
        assert torch.equal(p.grad, g)


def _train(tmp_path, extra):
    """What `python ddp.py --model vit-mae-base --fp16 --optimizer adamw --per_gpu_train_batch_size 16 --max_steps 16 [extra]`
    runs; returns every step's loss."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "vit-mae-base", "--fp16", "--optimizer", "adamw", "--per_gpu_train_batch_size", "16", "--max_steps", "16",
            "--logging_steps", "1", "--dataset_size", "64", "--lr", "1e-3", "--warmup_steps", "2", "--save_steps", "0",
            "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    trainer = Trainer(args, build_model("vit-mae-base"), cli.log)
    sums = []
    read = trainer.step_fn.read_loss_sum
    trainer.step_fn.read_loss_sum = lambda: sums.append(read()) or sums[-1]
    trainer.train()
    assert (trainer.step_fn.graph is not None) == args.cuda_graph
    return [b - a for a, b in zip([0.0] + sums[:-1], sums)][:16]


@pytest.mark.parametrize("extra", [["--cuda_graph"], [], ["--cuda_graph", "--channels_last"]], ids=["graph", "eager", "channels_last"])
def test_ddp_trains(tmp_path, capsys, extra):
    losses = _train(tmp_path, extra)
    with capsys.disabled():
        print(f"\nvit-mae-base {extra} losses on {torch.cuda.get_device_name()}: {[round(v, 4) for v in losses[::3]]}")
    assert len(losses) == 16 and all(math.isfinite(v) for v in losses)
    assert sum(losses[-4:]) / 4 < sum(losses[:4]) / 4, losses
