"""Swin V2 on the GPU: the cosine shifted-window attention kernels (output, lse, dq, dk, dv, the table and the scale
gradients) element by element against fp64 and bitwise repeatable, the native bf16 Swin-V2-T against its fp32 torch
path, no host synchronisation, and ``ddp.py --model swin-v2-t`` training under a CUDA graph.

Bounds follow tests/numerics.py's attention section with n = 64 keys per query (one key tile, no padding rows) and the
bias add (table entry and the -100 mask) in the score error, plus the normalisation.  The kernel rounds each normalised
row x^ = x / max(||x||, 1e-12) once to bf16 after an fp32 norm of 32 squares, a square root and a division, so every
element of x^ is within eps_n = 2^-8 + 48 u of the exact one (relative), and the cosine q^ . k^ within
(2 eps_n + eps_n^2 + C_ACC 32 u (1 + eps_n)^2) sum |qn| |kn| of the exact cosine (qn, kn the exact normalised rows).  In the
backward, dcos = scale dS is rounded to bf16; dq^ = dcos k^ accumulates in fp32; the projection
(dq^ - q^ (q^ . dq^)) / max(||q||, 1e-12) adds the error of the 32-term dot product, of q^ in it and of the fp32 norm.
The scale gradient is the fp32 sum of dS cos over each window (a 32-term chain per thread, a 32-lane butterfly and 4 warp
sums), then over the windows in 32 strided chains and across the 32."""
import copy
import math

import pytest
import torch

import numerics as nm
from b200ddp import _ext
from b200ddp.ops import cross_entropy, swin_relative_position_index, window_attention_v2

pytestmark = pytest.mark.gpu

WIN, N = 8, 64
EPS = 1e-12
EPS_N = nm.BF16_U + 48 * nm.U
# (batch, height, width, heads, shift, inputs): Swin-V2-T's four stages at 256, Swin-V2-B's first and last, a non-square
# map, shift 0 on the largest map, one image, a (0, 4) shift, logit scales above log 100 (the clamp) and q / k rows with
# tiny norms, some under 1e-12
SHAPES = [(2, 64, 64, 3, 4, "plain"), (2, 32, 32, 6, 4, "plain"), (2, 16, 16, 12, 4, "plain"), (2, 8, 8, 24, 0, "plain"),
          (2, 64, 64, 4, 4, "plain"), (2, 8, 8, 32, 0, "plain"), (2, 16, 32, 3, 4, "plain"), (2, 64, 64, 3, 0, "plain"),
          (1, 64, 64, 3, 4, "plain"), (2, 8, 16, 4, (0, 4), "plain"), (2, 32, 32, 6, 4, "clamp"), (2, 32, 32, 6, 4, "tiny")]


def dev():
    return torch.device("cuda", 0)


def _regions(n, shift):
    c = torch.arange(n)
    return torch.zeros_like(c) if shift == 0 else (c >= n - WIN).long() + (c >= n - shift).long()


def _windows(B, H, W, sy, sx):
    """The raster rows [N, 64] of every window's tokens (in window order, local raster order) and their shift regions."""
    wy, wx = H // WIN, W // WIN
    yp = (torch.arange(wy)[:, None] * WIN + torch.arange(WIN)[None, :])
    xp = (torch.arange(wx)[:, None] * WIN + torch.arange(WIN)[None, :])
    y, x = (yp + sy) % H, (xp + sx) % W
    b = torch.arange(B)[:, None, None, None, None]
    rows = (b * H + y[None, :, None, :, None]) * W + x[None, None, :, None, :]
    reg = _regions(H, sy)[yp][:, None, :, None] * 3 + _regions(W, sx)[xp][None, :, None, :]
    reg = reg.expand(wy, wx, WIN, WIN).expand(B, wy, wx, WIN, WIN)
    return rows.reshape(-1, N).to(dev()), reg.reshape(-1, N).to(dev())


def _unnormalize(dxh, xn, norm, err_dxh):
    """(dx^ - xn (xn . dx^)) / max(||x||, 1e-12) (no projection where the norm is under 1e-12) and its bound, given the
    bound err_dxh of the kernel's dx^ and eps_n of its x^."""
    big = norm >= EPS
    d = norm.clamp_min(EPS)
    dot = torch.where(big, (xn * dxh).sum(-1, keepdim=True), 0.0)
    xa = xn.abs()
    err_dot = torch.where(big, (xa * err_dxh).sum(-1, keepdim=True) * (1 + EPS_N) + EPS_N * (xa * dxh.abs()).sum(-1, keepdim=True)
                          + 34 * nm.U * (xa * (dxh.abs() + err_dxh)).sum(-1, keepdim=True) * (1 + EPS_N), 0.0)
    num = dxh - xn * dot
    err_num = err_dxh + xa * (1 + EPS_N) * err_dot + EPS_N * xa * dot.abs() + 3 * nm.U * (dxh.abs() + xa * dot.abs())
    return num / d, (err_num + 48 * nm.U * num.abs()) / d


def _reference(qkv, table, scale, B, H, W, heads, sy, sx, o, lse, dout):
    """fp64 cosine window attention with element-wise bounds; the backward at the kernel's own o and lse.  Returns
    {name: (ref, acc)} in the kernels' layouts."""
    C, n, e, ca, U = 32 * heads, N, nm.EXP_ULPS, nm.C_ACC, nm.U
    rows, reg = _windows(B, H, W, sy, sx)
    Nw = rows.shape[0]

    def split(t, parts):                                           # [BHW, parts C] -> parts x [N, heads, 64, 32]
        t = t.double()[rows]
        return [t[..., k * C:(k + 1) * C].reshape(Nw, n, heads, 32).transpose(1, 2) for k in range(parts)]
    Q, K, V = split(qkv, 3)
    O, dO = split(o, 1)[0], split(dout, 1)[0]
    L = lse.double()[rows].transpose(1, 2)[..., None]
    qnorm, knorm = Q.norm(dim=-1, keepdim=True), K.norm(dim=-1, keepdim=True)
    Qn, Kn = Q / qnorm.clamp_min(EPS), K / knorm.clamp_min(EPS)
    sc = scale.double().view(1, heads, 1, 1)
    idx = swin_relative_position_index(dev(), WIN).view(n, n)
    bias = table.double()[idx].permute(2, 0, 1)[None]
    mask = torch.where(reg[:, :, None] != reg[:, None, :], -100.0, 0.0)[:, None] if sy or sx else torch.zeros(1, 1, n, n, device=dev())
    cos = Qn @ Kn.transpose(-1, -2)
    qk = sc * cos
    s = qk + bias + mask
    Qa, Ka, Va, dOa = Qn.abs(), Kn.abs(), V.abs(), dO.abs()
    err_cos = (2 * EPS_N + EPS_N ** 2 + ca * 32 * U * (1 + EPS_N) ** 2) * (Qa @ Ka.transpose(-1, -2))
    add = 2 * U * (qk.abs() + bias.abs() + mask.abs())              # the scale multiply and the two adds

    l = torch.logsumexp(s, -1, keepdim=True)
    P = torch.exp(s - l)
    smax = s.abs().amax(-1, keepdim=True)
    rho = sc * err_cos + add + U * (e + 3 + 2 * (s.abs() + smax)) + (e + 3) * U
    sum_prho = (P * rho).sum(-1, keepdim=True)
    o_ref = P @ V
    o_acc = (nm.BF16_U * P + P * rho) @ Va + ca * U * (n + 1) * (P @ Va) + o_ref.abs() * (sum_prho + (n + 2) * U)
    lse_bnd = sum_prho + (n + 2) * U + 2 * U * (l.abs() + 1)

    Pb = torch.exp(s - L)
    dP = dO @ V.transpose(-1, -2)
    err_dP = ca * 32 * U * (dOa @ Va.transpose(-1, -2))
    D = (dO * O).sum(-1, keepdim=True)
    err_D = 32 * U * (dO * O).abs().sum(-1, keepdim=True)
    dS = Pb * (dP - D)
    rho_b = sc * err_cos + add + U * (e + 3 + 2 * (s.abs() + L.abs()))
    err32 = Pb * rho_b * (dP - D).abs() + Pb * (err_dP + err_D) + 2 * U * dS.abs()
    dSa = dS.abs()
    dcos = sc * dS
    err_dcos = sc * (err32 + 2 * U * dSa) + nm.BF16_U * sc * (dSa + err32 + 2 * U * dSa)
    dcosa = dcos.abs()
    err_P = Pb * (rho_b + nm.BF16_U * (1 + rho_b))
    mult = EPS_N + ca * U * (n + 1) * (1 + EPS_N)                      # k^ (q^) against kn (qn), and the accumulation

    dqh = dcos @ Kn
    err_dqh = (err_dcos @ Ka) * (1 + EPS_N) + mult * (dcosa @ Ka)
    dkh = dcos.transpose(-1, -2) @ Qn
    err_dkh = (err_dcos.transpose(-1, -2) @ Qa) * (1 + EPS_N) + mult * (dcosa.transpose(-1, -2) @ Qa)
    dq = _unnormalize(dqh, Qn, qnorm, err_dqh)
    dk = _unnormalize(dkh, Kn, knorm, err_dkh)
    dv = (Pb.transpose(-1, -2) @ dO, err_P.transpose(-1, -2) @ dOa + ca * U * (n + 1) * (Pb.transpose(-1, -2) @ dOa))

    def rows_of(t):                                                # [N, heads, 64, X] -> [BHW, heads X]
        out = torch.empty(B * H * W, heads * t.shape[-1], dtype=torch.float64, device=dev())
        out[rows.reshape(-1)] = t.transpose(1, 2).reshape(Nw * n, -1)
        return out
    bins = idx.reshape(-1)
    depth = n + -(-Nw // 32) + 32
    dtable = torch.zeros(225, heads, dtype=torch.float64, device=dev()).index_add_(0, bins, dS.sum(0).reshape(heads, -1).t())
    dtable_mag = torch.zeros_like(dtable).index_add_(0, bins, dSa.sum(0).reshape(heads, -1).t())
    dtable_err = torch.zeros_like(dtable).index_add_(0, bins, err32.sum(0).reshape(heads, -1).t())
    dscale = (dS * cos).sum((0, 2, 3))
    dscale_err = (err32 * (cos.abs() + err_cos) + dSa * err_cos).sum((0, 2, 3))
    dscale_mag = (dSa * cos.abs()).sum((0, 2, 3))
    sdepth = 32 + 5 + 2 + -(-Nw // 32) + 32
    return {"o": (rows_of(o_ref), rows_of(o_acc)), "lse": (rows_of(l), rows_of(lse_bnd)),
            "dqkv": (torch.cat([rows_of(dq[0]), rows_of(dk[0]), rows_of(dv[0])], 1), torch.cat([rows_of(dq[1]), rows_of(dk[1]), rows_of(dv[1])], 1)),
            "dtable": (dtable, dtable_err + depth * U * dtable_mag), "dscale": (dscale, dscale_err + sdepth * U * dscale_mag)}


def _inputs(B, H, W, heads, kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows, C = B * H * W, 32 * heads
    qkv = torch.randn(rows, 3 * C, device="cuda", generator=g)
    if kind == "tiny":
        qkv[::7, :2 * C] *= 1e-7
        qkv[3::11, :C] *= 1e-14                                   # q norms under 1e-12
        qkv[5::13, C:2 * C] *= 1e-14                              # k norms under 1e-12
    qkv = qkv.to(torch.bfloat16).requires_grad_(True)
    table = (16 * torch.sigmoid(torch.randn(225, heads, device="cuda", generator=g))).requires_grad_(True)
    logit = torch.randn(heads, device="cuda", generator=g) * 0.5 + math.log(10.0)
    if kind == "clamp":
        logit[::2] = math.log(100.0) + 1.0
    scale = torch.clamp(logit, max=math.log(100.0)).exp().requires_grad_(True)
    dout = torch.randn(rows, C, device="cuda", generator=g).to(torch.bfloat16)
    return qkv, table, scale, dout


@pytest.mark.parametrize("B,H,W,heads,shift,kind", SHAPES, ids=lambda v: str(v).replace(" ", ""))
def test_window_attention_v2_matches_fp64_elementwise(B, H, W, heads, shift, kind):
    sy, sx = (shift, shift) if isinstance(shift, int) else shift
    qkv, table, scale, dout = _inputs(B, H, W, heads, kind, B * 1000 + H * 10 + W + heads)
    C = 32 * heads

    def run():
        qkv.grad = table.grad = scale.grad = None
        o = window_attention_v2(qkv, table, scale, B, H, W, heads, shift)
        o.backward(dout)
        return [o.detach().clone(), qkv.grad.clone(), table.grad.clone(), scale.grad.clone()]

    first, second = run(), run()
    assert all(torch.equal(p, q) for p, q in zip(first, second))            # bitwise repeatable
    o, dqkv, dtable, dscale = first
    o2, lse = _ext.get().swin_v2.attention_fwd(qkv.detach(), table.detach(), scale.detach(), B, H, W, sy, sx)
    assert torch.equal(o, o2)
    ref = _reference(qkv.detach(), table.detach(), scale.detach(), B, H, W, heads, sy, sx, o, lse, dout)
    where = f"{B}x{H}x{W} heads={heads} shift={shift} {kind}"
    r, a = ref["o"]
    nm.check(f"swin v2 o {where}", o, r, nm.bound(r, a, torch.bfloat16), "swin v2 fwd o")
    r, a = ref["lse"]
    nm.check(f"swin v2 lse {where}", lse, r, a + nm.FLOOR, "swin v2 fwd lse")
    r, a = ref["dqkv"]
    for k, name in enumerate(("dq", "dk", "dv")):
        sl = slice(k * C, (k + 1) * C)
        nm.check(f"swin v2 {name} {where}", dqkv[:, sl], r[:, sl], nm.bound(r[:, sl], a[:, sl], torch.bfloat16), f"swin v2 bwd {name}")
    r, a = ref["dtable"]
    nm.check(f"swin v2 dtable {where}", dtable, r, nm.bound(r, a, torch.float32), "swin v2 bwd dtable")
    r, a = ref["dscale"]
    nm.check(f"swin v2 dscale {where}", dscale, r, nm.bound(r, a, torch.float32), "swin v2 bwd dscale")


def test_window_attention_v2_rejects_unsupported_shapes():
    table, scale = torch.zeros(225, 2, device="cuda"), torch.ones(2, device="cuda")
    qkv = torch.zeros(2 * 16 * 16, 3 * 64 * 2, device="cuda", dtype=torch.bfloat16)       # head dim 64
    with pytest.raises(ValueError, match="head dim 32"):
        window_attention_v2(qkv, table, scale, 2, 16, 16, 2, 4)
    qkv = torch.zeros(2 * 12 * 16, 3 * 32 * 2, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="multiples of 8"):
        window_attention_v2(qkv, table, scale, 2, 12, 16, 2, 4)


def _seeded_swin_v2_t(seed=0):
    """Swin-V2-T with logit scales and cpb weights large enough that the attention is far from uniform (scale 15, table
    entries spread over several units), but not so sharp that the bf16 rounding of q^ and k^ (2^-8 of a cosine, times the
    scale) dominates the comparison with the fp32 path."""
    from b200ddp.models import swin_v2_t
    torch.manual_seed(seed)
    model = swin_v2_t()
    with torch.no_grad():
        for m in model.modules():
            if hasattr(m, "logit_scale"):
                m.logit_scale.fill_(math.log(15.0))
                m.cpb_mlp[2].weight.normal_(0, 0.05)
    return model


def test_native_bf16_swin_v2_matches_the_fp32_torch_path(capsys):
    from b200ddp.utils import to_mixed_bf16
    ref = _seeded_swin_v2_t().to(dev())
    native = to_mixed_bf16(copy.deepcopy(ref))
    assert native.features[1][0].attn.logit_scale.dtype == torch.float32
    assert native.features[1][0].attn.cpb_mlp[0].weight.dtype == torch.float32
    g = torch.Generator().manual_seed(3)
    x = torch.randn(8, 3, 256, 256, generator=g).to(dev())
    target = torch.randint(0, 1000, (8,), generator=g).to(dev())
    lr = cross_entropy(ref(x), target)
    lr.backward()
    ln = cross_entropy(native(x.to(torch.bfloat16)), target)
    ln.backward()
    assert abs(float(ln.detach()) - float(lr.detach())) < 5e-2 * max(1.0, abs(float(lr.detach())))
    C = native.features[1][0].attn.qkv.weight.shape[1]
    assert float(native.features[1][0].attn.qkv.bias.grad[C:2 * C].abs().max()) == 0.0
    rels = {}
    for (n, p), q in zip(native.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rels[n] = float((p.grad.float() - q.grad).norm() / (q.grad.norm() + 1e-8))
    worst = max(rels, key=rels.get)
    with capsys.disabled():
        print(f"\nswin-v2-t native bf16 against fp32: loss {float(ln):.4f} / {float(lr):.4f}, largest gradient rel. diff "
              f"{rels[worst]:.4f} ({worst}), stem {rels['features.0.0.weight']:.4f}")
    # logit_scale's and the cpb MLP's gradients are sums of dS cos and dS over every window and pair of a stage, which
    # cancel to a small fraction of their terms, so the bf16 network's different activations move them further; the
    # kernel's d scale and d table themselves are checked against fp64 element by element above
    loose = ("logit_scale", "cpb_mlp")
    assert all(r < (0.35 if any(k in n for k in loose) else 0.2) for n, r in rels.items()), sorted(rels.items(), key=lambda kv: -kv[1])[:8]


def test_native_path_rejects_sizes_off_the_window_grid():
    model = _seeded_swin_v2_t().to(dev(), torch.bfloat16)
    with pytest.raises(ValueError, match="multiples of 256"):
        model(torch.zeros(1, 3, 224, 224, device=dev(), dtype=torch.bfloat16))


def test_swin_v2_step_has_no_host_synchronisation():
    from b200ddp.utils import to_mixed_bf16
    model = to_mixed_bf16(_seeded_swin_v2_t().to(dev()))
    x = torch.randn(4, 3, 256, 256, device=dev()).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
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
    attn = model.features[1][1].attn
    assert math.isfinite(float(loss)) and attn.logit_scale.grad is not None and attn.cpb_mlp[0].weight.grad is not None


def _train(tmp_path, extra):
    """What `python ddp.py --model swin-v2-t --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size 32
    --max_steps 30 --logging_steps 1 [extra]` runs on 64 images; returns every step's loss."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "swin-v2-t", "--fp16", "--cuda_graph", "--optimizer", "adamw", "--per_gpu_train_batch_size", "32",
            "--max_steps", "30", "--logging_steps", "1", "--dataset_size", "64", "--lr", "1e-3", "--warmup_steps", "2",
            "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    torch.manual_seed(0)
    trainer = Trainer(args, build_model("swin-v2-t"), cli.log)
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
        print(f"\nswin-v2-t losses on {torch.cuda.get_device_name(dev())}: {[round(v, 4) for v in losses[::5]]}; "
              f"last 5 mean {sum(losses[-5:]) / 5:.4f}; channels_last bitwise equal: {losses == cl}")
    assert all(math.isfinite(v) for v in losses)
    assert abs(losses[0] - math.log(1000)) < 0.5
    assert sum(losses[-5:]) / 5 < 0.7 * losses[0]
    assert losses == cl
