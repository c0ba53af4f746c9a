"""Vision Transformer on the GPU: the patchify kernel against torch's permutation (bitwise), ``patch_embed`` forward and
backward element by element against fp64, ``packed_attention`` on the image-as-document layout (one long row of many
short documents) against the fp64 attention reference, the native bf16 ViT-B/16 against its fp32 torch path, no host
synchronisation, and ``ddp.py --model vit-b-16`` training under a CUDA graph."""
import copy
import math

import pytest
import torch

import numerics as nm
from b200ddp.ops import cross_entropy, image_token_bounds, image_token_rows, patch_embed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    from b200ddp import _ext
    return _ext.get()


def dev():
    return torch.device("cuda", 0)


def _patch_rows(images, p):
    """[B, C, H, W] -> the patch matrix [T, C p p] in token order by torch ops: zero class and padding rows."""
    B, Cn, H, W = images.shape
    gh, gw = H // p, W // p
    patches = images.reshape(B, Cn, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B, gh * gw, Cn * p * p)
    per = gh * gw + 1
    out = torch.zeros(image_token_rows(B, per), Cn * p * p, dtype=images.dtype, device=images.device)
    out[:B * per].view(B, per, -1)[:, 1:] = patches
    return out


@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("p", [16, 32])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_patchify_is_the_torch_permutation_bitwise(C, layout, p, B):
    g = torch.Generator(device="cuda").manual_seed(B * p)
    images = torch.randn(B, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16)
    if layout == "channels_last":
        images = images.contiguous(memory_format=torch.channels_last)
    per = (224 // p) ** 2 + 1
    got = C.vit.patchify(images, p, image_token_rows(B, per))
    assert torch.equal(got, _patch_rows(images, p))


def _inputs(B, p, D=768, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    per = (224 // p) ** 2 + 1

    def rnd(*s, std=1.0):
        return (torch.randn(*s, device="cuda", generator=g) * std).to(torch.bfloat16).requires_grad_(True)
    images = torch.randn(B, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16)
    w = rnd(D, 3, p, p, std=1 / math.sqrt(3 * p * p))
    return images, w, rnd(D, std=0.1), rnd(1, 1, D, std=0.5), rnd(1, per, D, std=0.5), per


def _run(images, w, b, cls, pos, dy):
    for t in (w, b, cls, pos):
        t.grad = None
    out = patch_embed(images, w, b, cls, pos)
    out.backward(dy)
    return out.detach(), [t.grad.clone() for t in (w, b, cls, pos)]


@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("B,p", [(1, 16), (3, 16), (64, 16), (5, 32)])
def test_patch_embed_matches_fp64_elementwise(layout, B, p):
    images, w, b, cls, pos, per = _inputs(B, p, seed=B + p)
    if layout == "channels_last":
        images = images.contiguous(memory_format=torch.channels_last)
        w = w.detach().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    D = w.shape[0]
    T = image_token_rows(B, per)
    real = B * per
    g = torch.Generator(device="cuda").manual_seed(7)
    dy = torch.randn(T, D, device="cuda", generator=g).to(torch.bfloat16)
    dy[real:] = float("nan")                                     # the gradients must not read the padding rows
    out, grads = _run(images, w, b, cls, pos, dy)
    out2, grads2 = _run(images, w, b, cls, pos, dy)
    assert torch.equal(out, out2) and all(torch.equal(a, c) for a, c in zip(grads, grads2))   # bitwise repeatable
    assert all(bool(torch.isfinite(t).all()) for t in grads)

    # forward: the GEMM (bias epilogue, bf16 output), then + pos in fp32 and one bf16 rounding
    P = _patch_rows(images, p)
    w2 = w.detach().reshape(D, -1)
    y_ref, y_acc = nm.gemm_reference(P, w2, b.detach(), epilogue=1)
    y_bnd = nm.bound(y_ref, y_acc, torch.bfloat16)
    pos64, cls64 = pos.detach().double().reshape(per, D), cls.detach().double().reshape(1, D)
    ref = torch.zeros(T, D, dtype=torch.float64, device="cuda")
    acc = torch.zeros_like(ref)
    ref[:real] = (y_ref[:real].view(B, per, D) + pos64).reshape(real, D)
    acc[:real] = y_bnd[:real] + nm.U * ref[:real].abs()
    cls_rows = torch.arange(B, device="cuda") * per
    ref[cls_rows] = (cls64 + pos64[0]).expand(B, D)
    acc[cls_rows] = nm.U * ref[cls_rows].abs()
    nm.check("patch_embed tokens", out, ref, nm.bound(ref, acc, torch.bfloat16), "vit tokens")
    assert float(out[real:].abs().max()) == 0 if real < T else True

    # backward: patch-row gradient dP (dy at patch rows, 0 elsewhere); dW = dPᵀ P on the GEMM, db = Σ dP, d pos / d cls
    # fixed-order fp32 sums over the B images
    dP = torch.zeros_like(dy)
    dP[:real].view(B, per, D)[:, 1:] = dy[:real].view(B, per, D)[:, 1:]
    nm.check_gemm("patch_embed dW", grads[0].reshape(D, -1), dP.t(), P.t(), group="vit dW")
    dP64 = dP.double()
    nm.check("patch_embed db", grads[1], dP64.sum(0), nm.bound(dP64.sum(0), T * nm.U * dP64.abs().sum(0), torch.bfloat16), "vit db")
    rows = dy[:real].double().view(B, per, D)
    dpos_ref, dpos_acc = rows.sum(0), B * nm.U * rows.abs().sum(0)
    nm.check("patch_embed dpos", grads[3].reshape(per, D), dpos_ref, nm.bound(dpos_ref, dpos_acc, torch.bfloat16), "vit dpos")
    assert torch.equal(grads[2].reshape(D), grads[3].reshape(per, D)[0])


SCALE = 0.125                                                   # 1 / sqrt(64)


@pytest.mark.parametrize("B", [1, 5, 64])
@pytest.mark.parametrize("per", [197, 50])
def test_packed_attention_on_the_image_layout_matches_fp64(C, B, per):
    H, d = 12, 64
    bounds = image_token_bounds(B, per, "cuda")
    T = bounds.shape[1]
    real = B * per
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + per)
    qkv = torch.randn(T, 3 * H * d, device="cuda", generator=g).to(torch.bfloat16)
    dout = torch.randn(T, H * d, device="cuda", generator=g).to(torch.bfloat16)
    o, lse = C.packed_attention_fwd(qkv, bounds, H)
    dqkv = C.packed_attention_bwd(dout, qkv, o, lse, bounds, H)
    assert float(o[real:].abs().max()) == 0 if real < T else True
    assert float(dqkv[real:].abs().max()) == 0 if real < T else True

    def heads(t):
        return t.reshape(1, T, -1, d).transpose(1, 2)
    q, k, v = heads(qkv)[:, :H], heads(qkv)[:, H:2 * H], heads(qkv)[:, 2 * H:]
    vis = nm.attention_visible(bounds, T)
    where = f"image layout B={B} tokens={per}"
    fwd = nm.attention_reference(q, k, v, vis, SCALE)
    nm.check_attention(where, {"o": heads(o), "lse": lse}, fwd, "attn images")
    del fwd
    bwd = nm.attention_bwd_reference(q, k, v, heads(o), lse, heads(dout), vis, SCALE)
    dq, dk, dv = heads(dqkv)[:, :H], heads(dqkv)[:, H:2 * H], heads(dqkv)[:, 2 * H:]
    nm.check_attention(where, {"dq": dq, "dk": dk, "dv": dv}, bwd, "attn images")


def _seeded_vit_b_16(seed=0):
    from b200ddp.models import vit_b_16
    torch.manual_seed(seed)
    model = vit_b_16()
    with torch.no_grad():                                       # a non-zero head, so every gradient is non-trivial
        model.heads.head.weight.normal_(0.0, 0.02)
        model.heads.head.bias.normal_(0.0, 0.02)
        model.class_token.normal_(0.0, 0.02)
    return model


def test_native_bf16_vit_matches_the_fp32_torch_path():
    ref = _seeded_vit_b_16().to(dev())
    native = copy.deepcopy(ref).to(torch.bfloat16)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 3, 224, 224, generator=g).to(dev())
    target = torch.randint(0, 1000, (8,), generator=g).to(dev())
    lr = cross_entropy(ref(x), target)
    lr.backward()
    ln = cross_entropy(native(x.to(torch.bfloat16)), target)
    ln.backward()
    assert abs(float(ln) - float(lr)) < 5e-2 * max(1.0, abs(float(lr)))
    for (n, p), q in zip(native.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rel = float((p.grad.float() - q.grad).norm() / (q.grad.norm() + 1e-8))
        assert rel < 0.2, (n, rel)


def test_vit_step_has_no_host_synchronisation():
    model = _seeded_vit_b_16().to(dev(), torch.bfloat16)
    x = torch.randn(4, 3, 224, 224, device=dev()).to(torch.bfloat16)
    target = torch.randint(0, 1000, (4,), device=dev())
    cross_entropy(model(x), target).backward()
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = cross_entropy(model(x), target)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss)) and model.conv_proj.weight.grad is not None


def _train(tmp_path, extra):
    """What `python ddp.py --model vit-b-16 --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size 32
    --max_steps 30 --logging_steps 1 [extra]` runs on 64 images; returns every step's loss."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "vit-b-16", "--fp16", "--cuda_graph", "--optimizer", "adamw", "--per_gpu_train_batch_size", "32",
            "--max_steps", "30", "--logging_steps", "1", "--dataset_size", "64", "--lr", "3e-4", "--warmup_steps", "2",
            "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    trainer = Trainer(args, build_model("vit-b-16"), cli.log)
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
        print(f"\nvit-b-16 losses on {torch.cuda.get_device_name(dev())}: {[round(v, 4) for v in losses[::5]]}; "
              f"channels_last bitwise equal: {losses == cl}")
    assert abs(losses[0] - math.log(1000)) < 1e-3               # the zero-initialised head
    assert all(math.isfinite(v) for v in losses)
    assert sum(losses[-5:]) / 5 < losses[0] - 1.0
    assert max(abs(a - b) for a, b in zip(losses, cl)) <= 1e-3 * losses[0]
