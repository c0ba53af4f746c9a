"""Mamba-2 on the GPU: the conv over in_proj's xBC columns, the chunked SSD scan and the gated RMSNorm kernels (forward and
every gradient) element by element against float64 references computed from the kernels' own bf16 inputs, at
mamba2-130m's and mamba2-370m's layer shapes on fixed, right-padded and packed rows plus small ragged cases (S not a
multiple of the 64-row chunk, documents starting at and just after a chunk boundary, one-token documents, a document over
several chunks, strong decay); bitwise repeatable gradients; no host synchronisation; the native bf16 model against its
fp32 reference path; and ``ddp.py --model mamba2-130m`` training under a CUDA graph.

Per-element bound, for an output o against its fp64 reference r over a tensor of reference values R:
    |o - r| <= RTOL |r| + ATOL rms(R)
bf16 outputs are one bf16 rounding (2^-8 relative) of an fp32 value.  The SSD's tensor-core products add one more bf16
rounding of an operand that is not an input: (C B^T o M) and (M o dY X^T) [T-row tiles], w_j x_j and the fp32 chunk states
h_in and their gradients; each is 2^-8 relative per element, and summed over 64 or 128 terms of mixed sign it stays within
a few 2^-8 of rms(R).  So RTOL = ATOL = 2^-5 for the bf16 outputs (u, y, the norm output, dx, dB, dC, d dt, dz, dy).  The
fp32 parameter gradients (conv weight and bias, A_log, D, dt_bias, the norm weight) are fp32 sums over the B S rows of
products that carry those roundings, with RTOL = ATOL = 2^-8.  The largest error-to-bound ratio is printed; on an H100 80GB
HBM3 (700 W power limit) it was 0.731 (the SSD's dx) for the bf16 outputs and 0.714 (the norm weight) for the fp32
parameter gradients."""
import math

import pytest
import torch

from b200ddp.ops import (Mamba2GradLink, causal_conv1d_window, causal_conv1d_window_reference, document_bounds, gated_rms_norm,
                         gated_rms_norm_reference, ssd_scan, ssd_scan_reference)

pytestmark = pytest.mark.gpu

BF16_TOL = 2.0 ** -5
F32_TOL = 2.0 ** -8
N = 128


def dev():
    return torch.device("cuda", 0)


def _ids(B, S, layout, g, starts=None):
    ids = torch.randint(2, 1000, (B, S), generator=g)
    if layout in ("padded", "packed"):
        lens = torch.randint(S // 8, S + 1, (B,), generator=g)
        lens[0] = S
        for b in range(B):
            ids[b, lens[b]:] = 0
        if layout == "packed":
            for b in range(B):
                n = int(lens[b])
                st = torch.randint(1, max(2, n), (4,), generator=g)
                ids[b, st[st < n]] = 1
    if starts is not None:
        ids[0, starts] = 1
    return ids


def _inputs(B, S, H, layout, seed=0, starts=None, dt_bias=None):
    g = torch.Generator().manual_seed(seed)
    E = 64 * H
    CD, W = E + 2 * N, 2 * E + 2 * N + H
    ids = _ids(B, S, layout, g, starts)
    bounds, _ = document_bounds(ids.to(dev()), 1 if layout == "packed" else None, 0 if layout != "fixed" else None)
    bf = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dev(), torch.bfloat16)
    dtb = dt_bias if dt_bias is not None else torch.log(torch.expm1(torch.rand(H, generator=g) * 0.099 + 0.001))
    t = dict(zx=bf(B, S, W), w=bf(CD, 1, 4, scale=0.5), b=bf(CD, scale=0.5), xbc=bf(B, S, CD, scale=0.5),
             A_log=torch.log(torch.arange(1, H + 1.0)).to(dev()), D=(torch.rand(H, generator=g) + 0.5).to(dev()),
             dtb=torch.as_tensor(dtb, dtype=torch.float32).expand(H).contiguous().to(dev()), nw=bf(E, scale=0.2) + 1, y=bf(B, S, E))
    return t, bounds.to(torch.int32)


WORST = {}


def _check(name, got, ref, tol):
    got, ref = got.detach().double(), ref.detach().double()
    rms = float(ref.square().mean().sqrt()) if ref.numel() else 0.0
    bound = tol * ref.abs() + tol * rms + 1e-30
    assert torch.isfinite(got).all(), name
    ratio = float(((got - ref).abs() / bound).max())
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    assert ratio <= 1.0, f"{name}: worst error / bound = {ratio:.3f}"


def _leaf(t, double=False):
    return (t.double() if double else t).detach().clone().requires_grad_(True)


CASES = [(8, 2048, 24, "fixed"), (8, 2048, 24, "padded"), (8, 2048, 24, "packed"), (8, 2048, 32, "packed"),
         (3, 200, 8, "packed", [64, 65, 100, 101, 150]), (2, 300, 8, "fixed", None, 5.0), (2, 70, 24, "padded")]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(str(v) for v in c[:4]) + ("-starts" if len(c) > 4 and c[4] else "")
                         + ("-decay" if len(c) > 5 else ""))
def test_kernels_match_float64(case, capsys):
    B, S, H, layout = case[:4]
    starts = case[4] if len(case) > 4 else None
    t, bd = _inputs(B, S, H, layout, seed=B * S + H, starts=starts, dt_bias=case[5] if len(case) > 5 else None)
    E = 64 * H
    CD = E + 2 * N
    real = (bd[..., 0] < bd[..., 1])
    g = torch.Generator().manual_seed(1)
    rnd = lambda *s: torch.randn(*s, generator=g).to(dev(), torch.bfloat16)
    # conv over the xBC window
    zx, w, b = _leaf(t["zx"]), _leaf(t["w"]), _leaf(t["b"])
    u = causal_conv1d_window(zx, w, b, bd, col=E)
    gu = rnd(B, S, CD)
    u.backward(gu)
    zr, wr, br = _leaf(t["zx"], True), _leaf(t["w"], True), _leaf(t["b"], True)
    ur = causal_conv1d_window_reference(zr, wr, br, bd, col=E)
    ur.backward(gu.double())
    _check("conv u", u, ur, BF16_TOL)
    _check("conv dx", zx.grad[..., E:E + CD], zr.grad[..., E:E + CD], BF16_TOL)
    assert (zx.grad[..., :E] == 0).all() and (zx.grad[..., E + CD:] == 0).all()
    _check("conv dweight", w.grad, wr.grad, F32_TOL)
    _check("conv dbias", b.grad, br.grad, F32_TOL)
    assert (u[~real] == 0).all() and (zx.grad[~real] == 0).all()
    # SSD
    ins = {k: _leaf(t[k]) for k in ("xbc", "zx", "A_log", "D", "dtb")}
    y = ssd_scan(ins["xbc"], ins["zx"][..., -H:], ins["A_log"], ins["D"], ins["dtb"], bd)
    gy = rnd(B, S, E)
    y.backward(gy)
    ref = {k: _leaf(t[k], True) for k in ins}
    yr = ssd_scan_reference(ref["xbc"], ref["zx"][..., -H:], ref["A_log"], ref["D"], ref["dtb"], bd)
    yr.backward(gy.double())
    _check("ssd y", y, yr, BF16_TOL)
    _check("ssd dx", ins["xbc"].grad[..., :E], ref["xbc"].grad[..., :E], BF16_TOL)
    _check("ssd dB", ins["xbc"].grad[..., E:E + N], ref["xbc"].grad[..., E:E + N], BF16_TOL)
    _check("ssd dC", ins["xbc"].grad[..., E + N:], ref["xbc"].grad[..., E + N:], BF16_TOL)
    _check("ssd d dt", ins["zx"].grad[..., -H:], ref["zx"].grad[..., -H:], BF16_TOL)
    for k in ("A_log", "D", "dtb"):
        _check(f"ssd d{k}", ins[k].grad, ref[k].grad, F32_TOL)
    assert (y[~real] == 0).all() and (ins["xbc"].grad[~real] == 0).all() and (ins["zx"].grad[~real] == 0).all()
    # gated norm on the z columns (the wide kernels take 1024 < E <= 4096)
    if E > 1024:
        yy, zz, nw = _leaf(t["y"]), _leaf(t["zx"]), _leaf(t["nw"])
        o = gated_rms_norm(yy, zz[..., :E], nw, 1e-5)
        go = rnd(B, S, E)
        o.backward(go)
        yr_, zr_, nr = _leaf(t["y"], True), _leaf(t["zx"], True), _leaf(t["nw"], True)
        orf = gated_rms_norm_reference(yr_, zr_[..., :E], nr, 1e-5)
        orf.backward(go.double())
        _check("norm out", o, orf, BF16_TOL)
        _check("norm dy", yy.grad, yr_.grad, BF16_TOL)
        _check("norm dz", zz.grad[..., :E], zr_.grad[..., :E], BF16_TOL)
        _check("norm dweight", nw.grad, nr.grad, F32_TOL)
    with capsys.disabled():
        print(f"\n{case}: worst error / bound so far {', '.join(f'{k} {v:.3f}' for k, v in WORST.items())}")


def _chain(t, bd, H):
    """The mixer's ops with one link, as the model runs them: (output, gradients of zxbcdt, conv weight / bias, A_log, D,
    dt_bias, norm weight)."""
    E = 64 * H
    ins = {k: _leaf(t[k]) for k in ("zx", "w", "b", "A_log", "D", "dtb", "nw")}
    link = Mamba2GradLink(ins["zx"])
    xbc = causal_conv1d_window(ins["zx"], ins["w"], ins["b"], bd, col=E, link=link)
    y = ssd_scan(xbc, ins["zx"][..., -H:], ins["A_log"], ins["D"], ins["dtb"], bd, link=link)
    o = gated_rms_norm(y, ins["zx"][..., :E], ins["nw"], 1e-5, link=link)
    o.backward(torch.ones_like(o))
    return [o] + [ins[k].grad for k in sorted(ins)]


def test_linked_gradients_equal_unlinked_and_are_bitwise_repeatable():
    t, bd = _inputs(2, 300, 24, "packed", seed=5)
    a, b = _chain(t, bd, 24), _chain(t, bd, 24)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    E = 64 * 24
    ins = {k: _leaf(t[k]) for k in ("zx", "w", "b", "A_log", "D", "dtb", "nw")}
    xbc = causal_conv1d_window(ins["zx"], ins["w"], ins["b"], bd, col=E)
    y = ssd_scan(xbc, ins["zx"][..., -24:], ins["A_log"], ins["D"], ins["dtb"], bd)
    gated_rms_norm(y, ins["zx"][..., :E], ins["nw"], 1e-5).backward(torch.ones_like(y))
    assert torch.equal(ins["zx"].grad, a[1 + sorted(ins).index("zx")])


def _small_model(dtype):
    from b200ddp.models.mamba2 import Mamba2Config, Mamba2ForCausalLM
    from b200ddp.utils.precision import to_mixed_bf16
    torch.manual_seed(0)
    m = Mamba2ForCausalLM(Mamba2Config(vocab_size=1000, hidden=768, layers=2, heads=24)).to(dev())
    return to_mixed_bf16(m) if dtype == torch.bfloat16 else m


def test_native_model_matches_fp32_path():
    ids = torch.randint(1, 1000, (2, 300), device=dev())
    out = {}
    for dtype in (torch.float32, torch.bfloat16):
        m = _small_model(dtype)
        logits = m(ids[:, :-1]).float()
        loss = torch.nn.functional.cross_entropy(logits.reshape(-1, 1000), ids[:, 1:].reshape(-1))
        loss.backward()
        out[dtype] = (float(loss), {k: p.grad.float() for k, p in m.named_parameters()})
    (l32, g32), (l16, g16) = out[torch.float32], out[torch.bfloat16]
    assert abs(l16 - l32) <= 0.01 * abs(l32)
    for k in g32:
        assert float((g16[k] - g32[k]).norm()) <= 0.1 * float(g32[k].norm()), k


def test_no_host_synchronisation():
    m = _small_model(torch.bfloat16)
    m.config.pad_token_id, m.config.bos_token_id = 0, 1
    ids = torch.randint(2, 1000, (2, 256), device=dev())
    ids[1, 100:] = 0
    ids[0, 70] = 1
    m(ids).float().sum().backward()                      # warm up: module loads and workspace allocation
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m(ids).float().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def _train(tmp_path, extra):
    """What `python ddp.py --model mamba2-130m --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size 8 --seq_len 512
    --max_steps 30 --logging_steps 1 [extra]` runs; returns every step's loss."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "mamba2-130m", "--fp16", "--cuda_graph", "--optimizer", "adamw", "--per_gpu_train_batch_size", "8",
            "--seq_len", "512", "--max_steps", "30", "--logging_steps", "1", "--dataset_size", "64", "--lr", "1e-3",
            "--warmup_steps", "2", "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kw = {}
    if cli.padding_on(args):
        kw["pad_token_id"] = SyntheticTokens.PAD_ID
        if args.pack:
            kw["bos_token_id"] = 1
    if args.fused_lm_loss:
        kw["fused_lm_loss"] = True
    torch.manual_seed(0)
    trainer = Trainer(args, build_model("mamba2-130m", **kw), cli.log)
    sums = []
    read = trainer.step_fn.read_loss_sum
    trainer.step_fn.read_loss_sum = lambda: sums.append(read()) or sums[-1]
    trainer.train()
    assert trainer.step_fn.graph is not None
    return [b - a for a, b in zip([0.0] + sums[:-1], sums)][:30]


def test_ddp_training_under_a_cuda_graph(tmp_path, capsys):
    losses = _train(tmp_path / "a", [])
    padded = _train(tmp_path / "b", ["--min_seq_len", "64", "--max_steps", "5"])
    packed = _train(tmp_path / "c", ["--min_seq_len", "64", "--pack", "--max_steps", "5"])
    fused = _train(tmp_path / "d", ["--fused_lm_loss", "--max_steps", "5"])
    with capsys.disabled():
        print(f"\nmamba2-130m losses on {torch.cuda.get_device_name(dev())}: {[round(v, 4) for v in losses[::5]]}; "
              f"last 5 mean {sum(losses[-5:]) / 5:.4f}; padded {padded}; packed {packed}; fused {fused}")
    assert all(math.isfinite(v) for v in losses + padded + packed + fused)
    assert sum(losses[-5:]) / 5 < losses[0] - 1.0


def test_dtypes_and_misaligned_bounds():
    t, bounds = _inputs(2, 200, 24, "packed", seed=3)
    E, H = 64 * 24, 24
    # fp16 (or mixed) CUDA activations raise instead of falling back to the reference; fp32 runs the reference
    with pytest.raises(ValueError, match="bf16"):
        causal_conv1d_window(t["zx"].half(), t["w"], t["b"], bounds, col=E)
    with pytest.raises(ValueError, match="bf16"):
        ssd_scan(t["xbc"].half(), t["zx"][..., -H:].half(), t["A_log"], t["D"], t["dtb"], bounds)
    with pytest.raises(ValueError, match="bf16"):
        ssd_scan(t["xbc"].float(), t["zx"][..., -H:], t["A_log"], t["D"], t["dtb"], bounds)
    with pytest.raises(ValueError, match="bf16"):
        gated_rms_norm(t["y"], t["zx"][..., :E].half(), t["nw"], 1e-5)
    with pytest.raises(ValueError):
        ssd_scan(t["xbc"][..., :64 * 4 + 256], t["zx"][..., -4:], t["A_log"][:4], t["D"][:4], t["dtb"][:4], bounds)
    y32 = ssd_scan(t["xbc"].float(), t["zx"][..., -H:].float(), t["A_log"], t["D"], t["dtb"], bounds)
    assert y32.dtype == torch.float32
    odd = torch.zeros(bounds.numel() + 1, dtype=torch.int32, device=dev())[1:].view(bounds.shape)
    odd.copy_(bounds)
    a, b = _chain(t, bounds, H), _chain(t, odd, H)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
