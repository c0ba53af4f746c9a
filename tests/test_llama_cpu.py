"""Llama / SmolLM on the CPU: grouped-query causal attention against a brute-force loop and against the multi-head
reference with K / V repeated, the rotary, RMSNorm and SwiGLU bodies and gradients against fp64 formulas, a tiny GQA
model against Hugging Face's (whole rows and packed documents), the SmolLM-135M shape, the CLI, the dataset's start ids
and a short training run."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn


def _bounds(layout, S):
    b = torch.zeros(len(layout), S, 2, dtype=torch.int32)
    for r, docs in enumerate(layout):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
    return b


def _brute_force_gqa(qkv, bounds, heads, kv_heads):
    B, S, Wd = qkv.shape
    d = Wd // (heads + 2 * kv_heads)
    x = qkv.double()
    out = torch.zeros(B, S, heads * d, dtype=torch.float64)
    for b in range(B):
        for i in range(S):
            s0 = min(max(int(bounds[b, i, 0]), 0), S)
            e0 = min(max(int(bounds[b, i, 1]), s0), S)
            keys = [j for j in range(s0, e0) if j <= i]
            for h in range(heads if keys else 0):
                hk = h // (heads // kv_heads)
                q = x[b, i, h * d:(h + 1) * d]
                kc = slice((heads + hk) * d, (heads + hk + 1) * d)
                vc = slice((heads + kv_heads + hk) * d, (heads + kv_heads + hk + 1) * d)
                p = torch.softmax(torch.stack([q @ x[b, j, kc] for j in keys]) / math.sqrt(d), 0)
                out[b, i, h * d:(h + 1) * d] = sum(p[n] * x[b, j, vc] for n, j in enumerate(keys))
    return out


@pytest.mark.parametrize("heads,kv_heads", [(4, 2), (3, 1), (6, 2)])
def test_gqa_reference_matches_brute_force_and_repeated_mha(heads, kv_heads):
    torch.manual_seed(heads * 10 + kv_heads)
    S, d = 20, 8
    bounds = _bounds([[5, 1, 10], [20], []], S)
    qkv = torch.randn(3, S, (heads + 2 * kv_heads) * d, dtype=torch.float64)
    ref = Fn.causal_attention_reference(qkv, bounds, heads, kv_heads)
    assert torch.allclose(ref, _brute_force_gqa(qkv, bounds, heads, kv_heads), atol=1e-12)
    rep = Fn._repeat_kv(qkv, heads, kv_heads)
    assert rep.shape[-1] == 3 * heads * d
    assert torch.allclose(ref, Fn.causal_attention_reference(rep, bounds, heads), atol=1e-12)
    # the op's CPU body and its gradient, against the reference with repeated K / V
    x = qkv.clone().requires_grad_(True)
    y = Fn.causal_attention(x, bounds, heads, kv_heads)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = qkv.clone().requires_grad_(True)
    Fn.causal_attention_reference(Fn._repeat_kv(xr, heads, kv_heads), bounds, heads).backward(dy)
    assert torch.allclose(x.grad, xr.grad, atol=1e-10)


def test_gqa_with_equal_heads_is_the_multi_head_op():
    torch.manual_seed(0)
    qkv = torch.randn(2, 16, 3 * 2 * 8)
    bounds = _bounds([[16], [7, 9]], 16)
    a = Fn.causal_attention(qkv, bounds, 2)
    assert torch.equal(a, Fn.causal_attention(qkv, bounds, 2, 2)) and torch.equal(a, Fn.causal_attention(qkv, bounds, 2, None))
    with pytest.raises(ValueError):
        Fn.causal_attention(torch.randn(2, 16, 5 * 8), bounds, 3, 2)      # 2 does not divide 3


def _rope64(x, pos, theta=10000.0):
    """fp64 rotate_half rotation of [..., d] rows at integer positions."""
    d = x.shape[-1]
    inv = theta ** (-torch.arange(0, d, 2, dtype=torch.float64) / d)
    ang = pos.double()[..., None] * inv
    cos, sin = torch.cat([ang.cos()] * 2, -1), torch.cat([ang.sin()] * 2, -1)
    rot = torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1)
    return x * cos + rot * sin


def test_rotary_body_and_gradient_match_fp64_rotate_half():
    torch.manual_seed(1)
    heads, kv, d, S = 3, 1, 64, 12
    qkv = torch.randn(2, S, (heads + 2 * kv) * d, dtype=torch.float64)
    pos = torch.tensor([list(range(S)), [0, 1, 2, 0, 1, 2, 3, 4, 5, 6, 7, 2047]])
    table = Fn.rotary_cos_sin(2048)
    assert table.dtype == torch.float32 and table.shape == (2048, 2, 32)
    x = qkv.clone().requires_grad_(True)
    y = Fn.rotary(x, pos, table, heads, kv)
    qk = qkv[..., :(heads + kv) * d].reshape(2, S, heads + kv, d)
    expect = torch.cat([_rope64(qk, pos[:, :, None]).reshape(2, S, -1), qkv[..., (heads + kv) * d:]], -1)
    assert torch.allclose(y, expect, atol=1e-5)                   # the table is fp32
    assert torch.equal(y[..., (heads + kv) * d:], qkv[..., (heads + kv) * d:])
    dy = torch.randn_like(y)
    y.backward(dy)
    # the transpose rotation: <rope(x), dy> = <x, rope^T(dy)>
    assert torch.allclose((y.detach() * dy).sum(), (qkv * x.grad).sum(), rtol=1e-10)
    inv = Fn._rotary_reference(y.detach(), pos, table, heads, kv, inverse=True)
    assert torch.allclose(inv, qkv, atol=1e-5)


def test_rms_norm_and_swiglu_match_fp64_formulas():
    torch.manual_seed(2)
    x = torch.randn(5, 24, dtype=torch.float64, requires_grad=True)
    w = (torch.rand(24, dtype=torch.float64) + 0.5).requires_grad_(True)
    y = Fn.rms_norm(x, w, 1e-5)
    ref = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * w
    assert torch.allclose(y, ref.to(y.dtype), atol=1e-6)
    dy = torch.randn_like(ref)
    gx, gw = torch.autograd.grad(y, (x, w), dy)
    rx, rw = torch.autograd.grad(ref, (x, w), dy)
    assert torch.allclose(gx, rx, atol=1e-5) and torch.allclose(gw, rw, atol=1e-5)
    gu = torch.randn(7, 32, dtype=torch.float64, requires_grad=True)
    s = Fn.swiglu(gu)
    g, u = gu.detach().chunk(2, -1)
    assert torch.allclose(s, (g / (1 + torch.exp(-g)) * u).to(s.dtype), atol=1e-6)
    ds = torch.randn_like(s)
    (gg,) = torch.autograd.grad(s, gu, ds)
    sg = torch.sigmoid(g)
    expect = torch.cat([ds * u * sg * (1 + g * (1 - sg)), ds * g * sg], -1)
    assert torch.allclose(gg, expect.to(gg.dtype), atol=1e-5)
    from b200ddp.ops import RMSNorm
    m = RMSNorm(24)
    assert [n for n, _ in m.named_parameters()] == ["weight"]


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    return LlamaConfig(vocab_size=512, max_position=256, hidden=128, layers=2, heads=4, kv_heads=2, intermediate=256, **kw)


def _tiny_hf(seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.LlamaConfig(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                   num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256,
                                   rms_norm_eps=1e-5, rope_theta=10000.0, tie_word_embeddings=True, attention_bias=False,
                                   mlp_bias=False)
    return transformers.LlamaForCausalLM(cfg).eval()


def test_tiny_llama_matches_hugging_face_logits_and_loss():
    from b200ddp.models.llama import LlamaForCausalLM
    hf = _tiny_hf()
    ours = LlamaForCausalLM(_tiny_cfg())
    ours.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, 512, (2, 40), generator=torch.Generator().manual_seed(3))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    with torch.no_grad():
        ref = hf(ids, labels=ids)
        logits = ours(ids)
    assert logits.shape == (2, 40, 512)
    assert torch.allclose(logits, ref.logits, atol=1e-4), float((logits - ref.logits).abs().max())
    assert abs(float(Fn.cross_entropy(logits, labels)) - float(ref.loss)) < 1e-4


def test_packed_llama_row_matches_each_document_run_alone_through_hugging_face():
    from b200ddp.models.llama import LlamaForCausalLM
    BOS = 1
    hf = _tiny_hf(seed=4)
    ours = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, bos_token_id=BOS))
    ours.load_hf_state_dict(hf.state_dict())
    g = torch.Generator().manual_seed(5)
    docs = [torch.cat([torch.tensor([BOS]), torch.randint(2, 512, (n - 1,), generator=g)]) for n in (17, 1, 30)]
    row = torch.cat(docs + [torch.zeros(64 - 48, dtype=torch.long)])[None]
    with torch.no_grad():
        packed = ours(row)[0]
        at = 0
        for d in docs:
            alone = hf(d[None]).logits[0]
            assert torch.allclose(packed[at:at + len(d)], alone, atol=1e-4), float((packed[at:at + len(d)] - alone).abs().max())
            at += len(d)


def test_smollm_135m_shape_and_fp8_linears():
    from b200ddp.models import LlamaConfig, build_model
    c = LlamaConfig()
    assert (c.vocab_size, c.max_position, c.hidden, c.layers, c.heads, c.kv_heads, c.intermediate, c.eps, c.rope_theta) == \
        (49152, 2048, 576, 30, 9, 3, 1536, 1e-5, 10000.0)
    m = build_model("smollm-135m")
    assert sum(p.numel() for p in m.parameters()) == 134_515_008
    assert "model.cos_sin" not in m.state_dict()
    m8 = build_model("smollm-135m", fp8=True)
    fp8 = [n for n, x in m8.named_modules() if getattr(x, "fp8", False) is True]
    assert len(fp8) == 120 and all(n.split(".")[-1] in ("qkv", "o_proj", "gate_up", "down_proj") for n in fp8)
    assert m8.to(torch.bfloat16).model.cos_sin.dtype == torch.float32


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_smollm_cli_accepts_its_flags_and_rejects_long_rows(tmp_path):
    from b200ddp.engine import cli
    cli.setup(_args(tmp_path, "--model", "smollm-135m", "--no_cuda", "--seq_len", "2048", "--min_seq_len", "32", "--pack"))
    with pytest.raises(ValueError, match="2048"):
        cli.setup(_args(tmp_path, "--model", "smollm-135m", "--no_cuda", "--seq_len", "4096"))
    with pytest.raises(ValueError, match="CUDA device"):
        cli.setup(_args(tmp_path, "--model", "smollm-135m", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="gpt2"):
        cli.setup(_args(tmp_path, "--model", "resnet50", "--no_cuda", "--pack", "--min_seq_len", "32", "--seq_len", "64"))


def test_smollm_dataset_start_ids():
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine.trainer import build_dataset
    ds = build_dataset(types.SimpleNamespace(model="smollm-135m", dataset_size=40, seq_len=64, min_seq_len=4, pack=True))
    assert ds.bos_token_id == 1 and ds.pad_token_id == 0 and int(ds.X.max()) < 49152
    for x, y, docs in zip(ds.X, ds.Y, ds.doc_lengths):
        at = 0
        for n in docs:
            assert x[at] == 1 and (x[at + 1:at + n] > 1).all()
            assert torch.equal(y[at:at + n - 1], x[at + 1:at + n]) and y[at + n - 1] == -100
            at += n
        assert (x[at:] == 0).all()
    gpt = SyntheticTokens(samples=40, seq_len=64, vocab=50257, min_len=4, pack=True, causal=True)
    assert gpt.bos_token_id == 50256                              # GPT-2's default is unchanged
    with pytest.raises(ValueError):
        SyntheticTokens(samples=4, seq_len=64, vocab=100, min_len=4, pack=True, causal=True, bos_token_id=0)


def test_short_cpu_training_run_lowers_the_loss(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models.llama import LlamaForCausalLM
    args = _args(tmp_path, "--model", "smollm-135m", "--no_cuda", "--seq_len", "64", "--min_seq_len", "8", "--pack",
                 "--optimizer", "adamw", "--lr", "3e-3", "--max_steps", "30", "--per_gpu_train_batch_size", "4",
                 "--warmup_steps", "2", "--save_steps", "0", "--logging_steps", "10")
    cli.setup(args)
    from b200ddp.engine.trainer import build_dataset
    ds = build_dataset(args)
    ds.X = torch.where(ds.X > 1, ds.X % 16 + 2, ds.X)               # a small alphabet leaves something to learn
    ds.Y = torch.where(ds.Y > 1, ds.Y % 16 + 2, ds.Y)
    model = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, bos_token_id=1))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert math.isfinite(after) and after < before - 0.1, (before, after)
