"""Qwen3-0.6B on the CPU: a tiny Qwen3-shaped model (4 heads of dim 128 at hidden 256, so heads * head_dim != hidden,
perturbed q / k norm weights, theta 1e6, eps 1e-6) against Hugging Face's ``Qwen3ForCausalLM`` on whole rows and on packed
documents, the op's CPU body and gradients, the full preset against Hugging Face's parameter count, the FP8 linears, the
other presets left as they were, the CLI, the dataset's start id, AdamW's decay groups and a short training run."""
import math
import types

import pytest
import torch

from b200ddp.ops import functional as Fn

QWEN_BOS = 151643


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    return LlamaConfig(vocab_size=512, max_position=256, hidden=256, layers=2, heads=4, kv_heads=2, intermediate=384, eps=1e-6,
                       rope_theta=1e6, explicit_head_dim=128, qk_norm=True, **kw)


def _tiny_hf(seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.Qwen3Config(vocab_size=512, hidden_size=256, intermediate_size=384, num_hidden_layers=2,
                                   num_attention_heads=4, num_key_value_heads=2, head_dim=128, max_position_embeddings=256,
                                   rms_norm_eps=1e-6, rope_theta=1e6, tie_word_embeddings=True, attention_bias=False,
                                   use_sliding_window=False)
    hf = transformers.Qwen3ForCausalLM(cfg).eval()
    with torch.no_grad():                            # Hugging Face initialises the q / k norm weights to ones
        for n, p in hf.named_parameters():
            if n.endswith(("q_norm.weight", "k_norm.weight")):
                p.uniform_(0.5, 1.5)
    return hf


def test_tiny_qwen3_matches_hugging_face_logits_and_loss():
    from b200ddp.models.llama import LlamaForCausalLM
    hf = _tiny_hf()
    ours = LlamaForCausalLM(_tiny_cfg())
    assert ours.config.head_dim == 128
    ours.load_hf_state_dict(hf.state_dict())
    block = ours.model.layers[0]
    assert block.qkv.weight.shape == ((4 + 2 * 2) * 128, 256) and block.o_proj.weight.shape == (256, 4 * 128)
    assert torch.equal(block.q_norm.weight, hf.model.layers[0].self_attn.q_norm.weight)
    ids = torch.randint(0, 512, (2, 40), generator=torch.Generator().manual_seed(3))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    with torch.no_grad():
        ref = hf(ids, labels=ids)
        logits = ours(ids)
    assert logits.shape == (2, 40, 512)
    assert torch.allclose(logits, ref.logits, atol=1e-4), float((logits - ref.logits).abs().max())
    assert abs(float(Fn.cross_entropy(logits, labels)) - float(ref.loss)) < 1e-4


def test_packed_qwen3_row_matches_each_document_run_alone_through_hugging_face():
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


def test_qk_norm_rotary_cpu_body_is_norm_then_rope_with_its_gradients():
    H, Hkv, d, B, S = 4, 2, 128, 2, 9
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(B, S, (H + 2 * Hkv) * d, generator=g, dtype=torch.float64)
    wq, wk = (torch.rand(d, generator=g, dtype=torch.float64) + 0.5 for _ in range(2))
    pos = torch.randint(0, 64, (B, S), generator=g)
    table = Fn.rotary_cos_sin(64, d, 1e6).double()
    ins = [t.clone().requires_grad_(True) for t in (qkv, wq, wk)]
    y = Fn.qk_norm_rotary(*ins, pos, table, H, Hkv, 1e-6)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    # the same thing written out: each query / key head normalised over its d elements, times its weight, then rope
    ref_in = [t.clone().requires_grad_(True) for t in (qkv, wq, wk)]
    x = ref_in[0].reshape(B, S, H + 2 * Hkv, d)
    w = torch.cat([ref_in[1].expand(H, d), ref_in[2].expand(Hkv, d)])
    qk = x[:, :, :H + Hkv]
    qk = qk / torch.sqrt(qk.pow(2).mean(-1, keepdim=True) + 1e-6) * w
    ref = Fn._rotary_reference(torch.cat([qk, x[:, :, H + Hkv:]], 2).reshape(B, S, -1), pos, table, H, Hkv)
    ref.backward(dy)
    assert torch.allclose(y, ref, atol=1e-12)
    assert torch.equal(y[..., (H + Hkv) * d:], qkv[..., (H + Hkv) * d:])            # value heads pass through
    for a, b in zip(ins, ref_in):
        assert torch.allclose(a.grad, b.grad, atol=1e-10)
    assert torch.autograd.gradcheck(lambda a, b, c: Fn.qk_norm_rotary(a, b, c, pos[:, :3], table, H, Hkv, 1e-6),
                                    [t.detach()[:, :3].clone().requires_grad_(True) if i == 0 else t.detach().clone().requires_grad_(True)
                                     for i, t in enumerate((qkv, wq, wk))])


def test_qk_norm_rotary_rejects_bad_shapes():
    qkv = torch.randn(1, 4, 8 * 128)
    pos, table, w = torch.zeros(1, 4, dtype=torch.long), Fn.rotary_cos_sin(8, 128), torch.ones(128)
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, torch.ones(64), w, pos, table, 4, 2)                   # weight shape
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, w, w, pos, table, 3, 2)                                # width not (H + 2 Hkv) * d
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, w, w, pos.float(), table, 4, 2)                        # positions not integer
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, w, w, pos, Fn.rotary_cos_sin(8, 64), 4, 2)             # table for another head dim
    with pytest.raises(ValueError):
        Fn.qk_norm_rotary(qkv, w, w, pos, table, 4, 2, eps=0.0)


def test_qwen3_0_6b_preset_matches_hugging_face_parameter_count_and_fp8_linears():
    transformers = pytest.importorskip("transformers")
    from b200ddp.models import build_model
    with torch.device("meta"):
        m = build_model("qwen3-0.6b")
        m8 = build_model("qwen3-0.6b", fp8=True)
        hf = transformers.Qwen3ForCausalLM(transformers.Qwen3Config(
            vocab_size=151936, hidden_size=1024, intermediate_size=3072, num_hidden_layers=28, num_attention_heads=16,
            num_key_value_heads=8, head_dim=128, max_position_embeddings=40960, rms_norm_eps=1e-6, rope_theta=1e6,
            tie_word_embeddings=True, attention_bias=False))
    c = m.config
    assert (c.vocab_size, c.max_position, c.hidden, c.layers, c.heads, c.kv_heads, c.head_dim, c.intermediate, c.eps,
            c.rope_theta, c.attention_bias, c.qk_norm) == (151936, 40960, 1024, 28, 16, 8, 128, 3072, 1e-6, 1e6, False, True)
    n = sum(p.numel() for p in m.parameters())
    assert n == 596_049_920 == sum(p.numel() for p in hf.parameters())
    assert not [k for k in m.state_dict() if k.endswith(".bias")]
    norms = [k for k in m.state_dict() if k.endswith(("q_norm.weight", "k_norm.weight"))]
    assert len(norms) == 56 and all(m.state_dict()[k].shape == (128,) for k in norms)
    fp8 = [n for n, x in m8.named_modules() if getattr(x, "fp8", False) is True]
    assert len(fp8) == 112 and all(n.split(".")[-1] in ("qkv", "o_proj", "gate_up", "down_proj") for n in fp8)
    for _, x in m8.named_modules():                   # every FP8 GEMM dimension is a multiple of 16
        if getattr(x, "fp8", False) is True:
            assert x.in_features % 16 == 0 and x.out_features % 16 == 0


@pytest.mark.parametrize("name,params,head_dim", [("smollm-135m", 134_515_008, 64), ("qwen2.5-1.5b", 1_543_714_304, 128),
                                                  ("granite-3.0-1b-a400m", 1_334_690_816, 64)])
def test_other_presets_keep_their_head_dim_and_state_dict_keys(name, params, head_dim):
    from b200ddp.models import build_model
    with torch.device("meta"):
        m = build_model(name)
    c = m.config
    assert c.explicit_head_dim is None and c.qk_norm is False and c.head_dim == c.hidden // c.heads == head_dim
    assert sum(p.numel() for p in m.parameters()) == params
    keys = set(m.state_dict())
    assert not [k for k in keys if "q_norm" in k or "k_norm" in k]
    expect = {"input_layernorm.weight", "post_attention_layernorm.weight", "qkv.weight", "o_proj.weight"}
    expect |= {"moe.router.weight", "moe.w_gate_up", "moe.w_down"} if c.num_experts else {"gate_up.weight", "down_proj.weight"}
    expect |= {"qkv.bias"} if c.attention_bias else set()
    assert {k.split(".", 3)[3] for k in keys if k.startswith("model.layers.")} == expect
    assert keys - {k for k in keys if k.startswith("model.layers.")} == {"model.embed_tokens.weight", "model.norm.weight"}


def test_head_dim_must_divide_hidden_unless_given():
    from b200ddp.models.llama import LlamaConfig, LlamaModel
    with pytest.raises(ValueError, match="divide hidden"):
        LlamaModel(LlamaConfig(vocab_size=64, hidden=256, layers=1, heads=3, kv_heads=1, intermediate=64))
    m = LlamaModel(LlamaConfig(vocab_size=64, hidden=256, layers=1, heads=3, kv_heads=1, intermediate=64, explicit_head_dim=128))
    assert m.layers[0].qkv.weight.shape == (5 * 128, 256) and m.layers[0].o_proj.weight.shape == (256, 3 * 128)
    with pytest.raises(ValueError, match="query-scale"):
        LlamaModel(LlamaConfig(vocab_size=64, hidden=256, layers=1, heads=2, kv_heads=1, intermediate=64, qk_norm=True,
                               attention_multiplier=0.25))


def test_qwen3_norm_weights_fall_into_adamw_no_decay_group():
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.optim import weight_decay_groups
    m = LlamaForCausalLM(_tiny_cfg())
    decay, no_decay = weight_decay_groups(m, 0.1)
    names = {id(p): n for n, p in m.named_parameters()}
    assert all(p.ndim >= 2 for p in decay["params"]) and decay["weight_decay"] == 0.1
    assert no_decay["weight_decay"] == 0.0
    assert {names[id(p)] for p in no_decay["params"] if names[id(p)].endswith(("q_norm.weight", "k_norm.weight"))} == \
        {f"model.layers.{i}.{n}.weight" for i in range(2) for n in ("q_norm", "k_norm")}
    assert not [names[id(p)] for p in decay["params"] if "_norm" in names[id(p)]]


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_qwen3_cli_accepts_its_flags_and_rejects_long_rows(tmp_path):
    from b200ddp.engine import cli
    cli.setup(_args(tmp_path, "--model", "qwen3-0.6b", "--no_cuda", "--seq_len", "32768", "--min_seq_len", "256", "--pack"))
    cli.setup(_args(tmp_path, "--model", "qwen3-0.6b", "--no_cuda", "--fused_lm_loss"))
    with pytest.raises(ValueError, match="32768"):
        cli.setup(_args(tmp_path, "--model", "qwen3-0.6b", "--no_cuda", "--seq_len", "32896"))
    with pytest.raises(ValueError, match="CUDA device"):
        cli.setup(_args(tmp_path, "--model", "qwen3-0.6b", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="min_seq_len below"):
        cli.setup(_args(tmp_path, "--model", "qwen3-0.6b", "--no_cuda", "--pack", "--seq_len", "256"))
    with pytest.raises(ValueError, match="qwen3-0.6b"):
        cli.setup(_args(tmp_path, "--model", "resnet50", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="qwen3-0.6b"):
        cli.setup(_args(tmp_path, "--model", "resnet50", "--no_cuda", "--fused_lm_loss"))


def test_qwen3_dataset_documents_start_with_endoftext():
    from b200ddp.engine.trainer import build_dataset
    ds = build_dataset(types.SimpleNamespace(model="qwen3-0.6b", dataset_size=40, seq_len=64, min_seq_len=4, pack=True))
    assert ds.bos_token_id == QWEN_BOS and ds.pad_token_id == 0 and int(ds.X.max()) < 151936
    for x, docs in zip(ds.X, ds.doc_lengths):
        at = 0
        for n in docs:
            assert x[at] == QWEN_BOS and (x[at + 1:at + n] != QWEN_BOS).all()
            at += n
    rows = build_dataset(types.SimpleNamespace(model="qwen3-0.6b", dataset_size=8, seq_len=64, min_seq_len=None, pack=False))
    assert rows.X.shape == (8, 64) and int(rows.X.max()) < 151936 and rows.bos_token_id is None


def test_short_cpu_qwen3_training_run_lowers_the_loss(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models.llama import LlamaForCausalLM
    args = _args(tmp_path, "--model", "qwen3-0.6b", "--no_cuda", "--seq_len", "64", "--min_seq_len", "8", "--pack",
                 "--optimizer", "adamw", "--lr", "3e-3", "--max_steps", "30", "--per_gpu_train_batch_size", "4",
                 "--warmup_steps", "2", "--save_steps", "0", "--logging_steps", "10")
    cli.setup(args)
    ds = build_dataset(args)
    bos = ds.X == QWEN_BOS                                         # a small alphabet leaves something to learn
    ds.X = torch.where(bos, torch.ones_like(ds.X), torch.where(ds.X > 0, ds.X % 16 + 2, ds.X))
    ds.Y = torch.where(ds.Y > 0, ds.Y % 16 + 2, ds.Y)
    ds.bos_token_id = 1
    model = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, bos_token_id=1))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert math.isfinite(after) and after < before - 0.1, (before, after)
    assert any(float((layer.q_norm.weight - 1).abs().max()) > 0 for layer in model.model.layers)   # the norm weights train
