"""ModernBERT on the GPU: sliding-window document attention (``packed_attention`` on ``window_bounds``) against an fp32
dense band reference on fixed, right-padded and packed rows up to 8192 tokens; the GeGLU kernels against fp32; the
bias-free GELU linear and LayerNorm; a tiny ModernBERT against its CPU body; a training step without host
synchronisation; and the full modernbert-base preset training under CUDA graphs at 8192 tokens."""
import math

import pytest
import torch

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu
H, D = 2, 64


def dev():
    return torch.device("cuda", 0)


def _ids(layout, S, seed=0):
    """[3, S] ids with 1 as the document start and 0 as padding: fixed rows, right-padded rows (one of them empty), or
    packed rows (documents of 1 and of odd lengths, tail padding, an empty row)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 100, (3, S), generator=g)
    if layout == "padded":
        for r, n in enumerate((S, S // 2 + 37, 0)):
            ids[r, n:] = 0
    elif layout == "packed":
        for r, docs in enumerate(([S // 3, 1, S // 4 + 5], [S], [])):
            at = 0
            for n in docs:
                ids[r, at] = 1
                at += n
            ids[r, at:] = 0
    return ids


def _bounds(layout, S):
    ids = _ids(layout, S).to(dev())
    return Fn.document_bounds(ids, 1 if layout == "packed" else None, None if layout == "fixed" else 0)[0]


def _band_reference(qkv, bounds, window, dy):
    """fp32 attention with the dense mask same-document & |i - j| <= window, built without window_bounds."""
    S = qkv.shape[1]
    i = torch.arange(S, device=qkv.device)
    keep = Fn._bounds_mask(bounds, S, qkv.device) & ((i[:, None] - i[None, :]).abs() <= window)
    x = qkv.detach().float().requires_grad_(True)
    out = Fn._masked_attention_reference(x, keep[:, None], H)
    out.backward(dy.float())
    return out.detach(), x.grad


@pytest.mark.parametrize("layout", ["fixed", "padded", "packed"])
@pytest.mark.parametrize("S", [128, 512, 8192])
@pytest.mark.parametrize("window", [1, 64, 127, 200, "S"])
def test_windowed_packed_attention_matches_dense_band_reference(layout, S, window):
    w = S if window == "S" else window
    bounds = _bounds(layout, S)
    local = Fn.window_bounds(bounds, w)
    g = torch.Generator(device="cuda").manual_seed(S + w)
    qkv = torch.randn(3, S, 3 * H * D, device=dev(), generator=g).to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn(3, S, H * D, device=dev(), generator=g).to(torch.bfloat16)
    out = Fn.packed_attention(qkv, local, H)
    (dqkv,) = torch.autograd.grad(out, qkv, dy)
    out2 = Fn.packed_attention(qkv, local, H)
    (dqkv2,) = torch.autograd.grad(out2, qkv, dy)
    assert torch.equal(out, out2) and torch.equal(dqkv, dqkv2)                     # deterministic
    real = (bounds[..., 1] > bounds[..., 0])
    assert (out[~real] == 0).all() and (dqkv[~real] == 0).all()                   # padding rows: zero output and gradient
    if w >= S - 1:
        plain = Fn.packed_attention(qkv, bounds, H)
        (dplain,) = torch.autograd.grad(plain, qkv, dy)
        assert torch.equal(out, plain) and torch.equal(dqkv, dplain)
    if S == 8192:                                    # the dense fp32 reference of three 8192 rows: check one row
        rows = [2 if layout == "fixed" else 0]
        qkv_r, bounds_r, dy_r = qkv[rows], bounds[rows], dy[rows]
        out_r, dq_r = out[rows], dqkv[rows]
    else:
        qkv_r, bounds_r, dy_r, out_r, dq_r = qkv, bounds, dy, out, dqkv
    ref, dref = _band_reference(qkv_r, bounds_r, w, dy_r)
    rel = float((out_r.float() - ref).norm() / ref.norm().clamp_min(1e-6))
    rel_g = float((dq_r.float() - dref).norm() / dref.norm().clamp_min(1e-6))
    assert rel < 1e-2 and rel_g < 2e-2, (rel, rel_g)


@pytest.mark.parametrize("rows", [16384, 999])
def test_geglu_matches_fp32_and_is_deterministic(rows):
    I = 1152
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = torch.randn(rows, 2 * I, device=dev(), generator=g).to(torch.bfloat16)
    dy = torch.randn(rows, I, device=dev(), generator=g).to(torch.bfloat16)
    xg = x.clone().requires_grad_(True)
    y = Fn.geglu(xg)
    (dx,) = torch.autograd.grad(y, xg, dy)
    xf = x.float().requires_grad_(True)
    a, gate = xf.chunk(2, -1)
    ref = torch.nn.functional.gelu(a) * gate
    (dref,) = torch.autograd.grad(ref, xf, dy.float())
    ref = ref.detach()
    assert float((y.float() - ref).abs().max()) <= 1e-2 * float(ref.abs().max())
    assert float((y.float() - ref).norm() / ref.norm()) < 4e-3
    assert float((dx.float() - dref).norm() / dref.norm()) < 4e-3
    y2 = Fn.geglu(x)
    assert torch.equal(y, y2) and torch.equal(dx, torch.autograd.grad(Fn.geglu(xg), xg, dy)[0])


def test_geglu_rejects_bad_input():
    x = torch.randn(8, 2 * 64, device=dev()).to(torch.bfloat16)
    with pytest.raises(ValueError):
        Fn.geglu(x.float())                                                     # not bf16
    with pytest.raises(ValueError):
        Fn.geglu(torch.randn(8, 2 * 12, device=dev()).to(torch.bfloat16))       # I % 8 != 0
    with pytest.raises(ValueError):
        Fn.geglu(torch.randn(8, 7, device=dev()).to(torch.bfloat16))            # odd width
    buf = torch.empty(x.numel() + 1, device=dev(), dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        Fn.geglu(buf[1:].view_as(x))                                            # 2-byte aligned
    with pytest.raises(ValueError):
        Fn.geglu(torch.randn(128, 8, device=dev()).to(torch.bfloat16).t())     # not contiguous


def test_bias_free_gelu_linear_runs_native_and_matches_torch():
    from b200ddp import _ext
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(512, 768, device=dev(), generator=g).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(768, 768, device=dev(), generator=g) * 0.03).to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn(512, 768, device=dev(), generator=g).to(torch.bfloat16)
    before = _ext.get().launch_count()
    y = Fn.linear(x, w, None, "gelu")
    dx, dw = torch.autograd.grad(y, (x, w), dy)
    assert _ext.get().launch_count() - before >= 2                  # the GEMM and the GELU pass are native launches
    xf, wf = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    ref = torch.nn.functional.gelu(xf @ wf.t())
    rdx, rdw = torch.autograd.grad(ref, (xf, wf), dy.float())
    for a, b in ((y, ref), (dx, rdx), (dw, rdw)):
        assert float((a.float() - b).norm() / b.norm()) < 1e-2


def test_bias_free_layer_norm_on_cuda_matches_torch():
    from b200ddp.ops import LayerNorm
    ln = LayerNorm(768, eps=1e-5, bias=False).to(dev(), torch.bfloat16)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5)
    x = torch.randn(4096, 768, device=dev()).to(torch.bfloat16).requires_grad_(True)
    dy = torch.randn_like(x)
    y = ln(x)
    dx, dwt = torch.autograd.grad(y, (x, ln.weight), dy)
    xf, wf = x.detach().float().requires_grad_(True), ln.weight.detach().float().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xf, (768,), wf, None, 1e-5)
    rdx, rdw = torch.autograd.grad(ref, (xf, wf), dy.float())
    for a, b in ((y, ref), (dx, rdx), (dwt, rdw)):
        assert float((a.float() - b).norm() / b.norm()) < 1e-2


def _tiny_cfg(**kw):
    from b200ddp.models.modernbert import ModernBertConfig
    return ModernBertConfig(**{**dict(vocab_size=1024, hidden=128, layers=4, heads=2, intermediate=192, max_position=512,
                                      local_attention=32), **kw})


def _batch(layout, S, seed):
    ids = _ids(layout, S, seed) * 7 % 1000 + 2
    ids = torch.where(_ids(layout, S, seed) == 0, 0, ids)
    if layout == "packed":
        ids = torch.where(_ids(layout, S, seed) == 1, 1, ids)
    g = torch.Generator().manual_seed(seed + 1)
    labels = torch.where((torch.rand(ids.shape, generator=g) < 0.3) & (ids > 1), torch.randint(2, 1024, ids.shape, generator=g), -100)
    return ids, labels


@pytest.mark.parametrize("layout", ["fixed", "padded", "packed"])
def test_modernbert_tiny_gpu_matches_cpu_body(layout):
    from b200ddp.models.modernbert import ModernBertForMaskedLM
    from b200ddp.ops import cross_entropy
    kw = {"fixed": {}, "padded": {"pad_token_id": 0}, "packed": {"pad_token_id": 0, "cls_token_id": 1}}[layout]
    torch.manual_seed(7)
    ref = ModernBertForMaskedLM(_tiny_cfg(**kw))
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if "norm" in n:
                p.uniform_(0.5, 1.5)
        ref.decoder.bias.uniform_(-0.5, 0.5)
    gpu = ModernBertForMaskedLM(_tiny_cfg(**kw))
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    assert gpu.model.global_cos_sin.dtype == torch.float32 and gpu.model.local_cos_sin.dtype == torch.float32
    ids, labels = _batch(layout, 256, seed=1)
    lr = cross_entropy(ref(ids), labels)
    lr.backward()
    lg = cross_entropy(gpu(ids.to(dev())), labels.to(dev()))
    lg.backward()
    assert abs(float(lg) - float(lr)) < 5e-2 * max(1.0, abs(float(lr)))
    for (n, p), q in zip(gpu.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rel = float((p.grad.float().cpu() - q.grad).norm() / (q.grad.norm() + 1e-8))
        assert rel < 0.2, (n, rel)


def test_modernbert_step_has_no_host_synchronisation():
    from b200ddp.models.modernbert import ModernBertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = ModernBertForMaskedLM(_tiny_cfg(pad_token_id=0, cls_token_id=1)).to(dev(), torch.bfloat16)
    ids, labels = _batch("packed", 256, seed=2)
    ids, labels = ids.to(dev()), labels.to(dev())
    cross_entropy(model(ids), labels).backward()
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = cross_entropy(model(ids), labels)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss)) and model.decoder.bias.grad is not None


@pytest.mark.parametrize("extra", [["--min_seq_len", "1024", "--pack"], ["--fp8"]])
def test_modernbert_base_graph_training_at_8192_tokens(tmp_path, extra, capsys):
    """What `python ddp.py --model modernbert-base --fp16 --optimizer adamw --cuda_graph --seq_len 8192
    --per_gpu_train_batch_size 2 --max_steps 4 [--min_seq_len 1024 --pack | --fp8]` runs."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models import build_model
    argv = ["--model", "modernbert-base", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "4", "--seq_len",
            "8192", "--per_gpu_train_batch_size", "2", "--dataset_size", "64", "--lr", "1e-4", "--warmup_steps", "1",
            "--save_steps", "0", "--logging_steps", "2", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"fp8": True} if args.fp8 else {}
    if args.pack:
        kwargs.update(pad_token_id=SyntheticTokens.PAD_ID, cls_token_id=50281)
    ds = build_dataset(args)
    assert ds.cls_token_id == (50281 if args.pack else None)
    trainer = Trainer(args, build_model("modernbert-base", **kwargs), cli.log, dataset=ds)
    trainer.train()
    loss = trainer.evaluate(max_batches=2)["eval_loss"]
    with capsys.disabled():
        print(f"\nmodernbert-base 2 x 8192 {' '.join(extra)} on {torch.cuda.get_device_name(dev())}: eval loss {loss:.4f}")
    assert trainer.step_fn.graph is not None
    assert math.isfinite(loss) and abs(loss - math.log(50368)) < 1.5
