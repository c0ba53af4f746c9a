"""Qwen2.5-1.5B on the CPU: a tiny Qwen2-shaped model (head dim 128, q / k / v bias, theta 1e6, eps 1e-6) against
Hugging Face's ``Qwen2ForCausalLM`` on whole rows and on packed documents, the full preset's parameter count, the CLI,
the dataset's start id, AdamW's decay groups and a short training run."""
import math
import types

import pytest
import torch

from b200ddp.ops import functional as Fn

QWEN_BOS = 151643


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    return LlamaConfig(vocab_size=512, max_position=256, hidden=256, layers=2, heads=2, kv_heads=1, intermediate=384, eps=1e-6,
                       rope_theta=1e6, attention_bias=True, **kw)


def _tiny_hf(seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.Qwen2Config(vocab_size=512, hidden_size=256, intermediate_size=384, num_hidden_layers=2,
                                   num_attention_heads=2, num_key_value_heads=1, max_position_embeddings=256,
                                   rms_norm_eps=1e-6, rope_theta=1e6, tie_word_embeddings=True, use_sliding_window=False)
    hf = transformers.Qwen2ForCausalLM(cfg).eval()
    with torch.no_grad():                            # Hugging Face initialises the q / k / v biases to zero
        for n, p in hf.named_parameters():
            if n.endswith("_proj.bias"):
                p.normal_(std=0.5)
    return hf


def test_tiny_qwen_matches_hugging_face_logits_and_loss():
    from b200ddp.models.llama import LlamaForCausalLM
    hf = _tiny_hf()
    ours = LlamaForCausalLM(_tiny_cfg())
    assert ours.config.head_dim == 128
    ours.load_hf_state_dict(hf.state_dict())
    assert ours.model.layers[0].qkv.bias.shape == (4 * 128,)
    ids = torch.randint(0, 512, (2, 40), generator=torch.Generator().manual_seed(3))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    with torch.no_grad():
        ref = hf(ids, labels=ids)
        logits = ours(ids)
    assert logits.shape == (2, 40, 512)
    assert torch.allclose(logits, ref.logits, atol=1e-4), float((logits - ref.logits).abs().max())
    assert abs(float(Fn.cross_entropy(logits, labels)) - float(ref.loss)) < 1e-4


def test_packed_qwen_row_matches_each_document_run_alone_through_hugging_face():
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


def test_qwen2_5_1_5b_shape_bias_and_fp8_linears():
    from b200ddp.models import build_model
    with torch.device("meta"):
        m = build_model("qwen2.5-1.5b")
        m8 = build_model("qwen2.5-1.5b", fp8=True)
    c = m.config
    assert (c.vocab_size, c.max_position, c.hidden, c.layers, c.heads, c.kv_heads, c.intermediate, c.eps, c.rope_theta,
            c.attention_bias, c.head_dim) == (151936, 32768, 1536, 28, 12, 2, 8960, 1e-6, 1e6, True, 128)
    assert sum(p.numel() for p in m.parameters()) == 1_543_714_304
    biases = [n for n, p in m.named_parameters() if n.endswith(".bias")]
    assert len(biases) == 28 and all(n.endswith(".qkv.bias") for n in biases)
    fp8 = [n for n, x in m8.named_modules() if getattr(x, "fp8", False) is True]
    assert len(fp8) == 112 and all(n.split(".")[-1] in ("qkv", "o_proj", "gate_up", "down_proj") for n in fp8)
    for _, x in m8.named_modules():                   # every FP8 GEMM dimension is a multiple of 16
        if getattr(x, "fp8", False) is True:
            assert x.in_features % 16 == 0 and x.out_features % 16 == 0
    from b200ddp.models.llama import LlamaConfig
    assert LlamaConfig().attention_bias is False     # SmolLM is unchanged


def test_qwen_bias_parameters_fall_into_adamw_no_decay_group():
    from b200ddp.models.llama import LlamaForCausalLM
    from b200ddp.optim import weight_decay_groups
    m = LlamaForCausalLM(_tiny_cfg())
    decay, no_decay = weight_decay_groups(m, 0.1)
    names = {id(p): n for n, p in m.named_parameters()}
    assert all(p.ndim >= 2 for p in decay["params"]) and decay["weight_decay"] == 0.1
    assert no_decay["weight_decay"] == 0.0
    assert {names[id(p)] for p in no_decay["params"] if names[id(p)].endswith("qkv.bias")} == \
        {f"model.layers.{i}.qkv.bias" for i in range(2)}


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_qwen_cli_accepts_its_flags_and_rejects_long_rows(tmp_path):
    from b200ddp.engine import cli
    cli.setup(_args(tmp_path, "--model", "qwen2.5-1.5b", "--no_cuda", "--seq_len", "32768", "--min_seq_len", "256", "--pack"))
    with pytest.raises(ValueError, match="32768"):
        cli.setup(_args(tmp_path, "--model", "qwen2.5-1.5b", "--no_cuda", "--seq_len", "32896"))
    with pytest.raises(ValueError, match="CUDA device"):
        cli.setup(_args(tmp_path, "--model", "qwen2.5-1.5b", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="min_seq_len below"):
        cli.setup(_args(tmp_path, "--model", "qwen2.5-1.5b", "--no_cuda", "--pack", "--seq_len", "256"))
    with pytest.raises(ValueError, match="qwen2.5-1.5b"):
        cli.setup(_args(tmp_path, "--model", "resnet50", "--no_cuda", "--fp16", "--fp8"))


def test_qwen_dataset_start_id():
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine.trainer import build_dataset
    assert SyntheticTokens.QWEN_BOS_ID == QWEN_BOS
    ds = build_dataset(types.SimpleNamespace(model="qwen2.5-1.5b", dataset_size=40, seq_len=64, min_seq_len=4, pack=True))
    assert ds.bos_token_id == QWEN_BOS and ds.pad_token_id == 0 and int(ds.X.max()) < 151936
    for x, y, docs in zip(ds.X, ds.Y, ds.doc_lengths):
        at = 0
        for n in docs:
            assert x[at] == QWEN_BOS and (x[at + 1:at + n] != QWEN_BOS).all() and (x[at + 1:at + n] > 0).all()
            assert torch.equal(y[at:at + n - 1], x[at + 1:at + n]) and y[at + n - 1] == -100
            at += n
        assert (x[at:] == 0).all()
    rows = build_dataset(types.SimpleNamespace(model="qwen2.5-1.5b", dataset_size=8, seq_len=64, min_seq_len=None, pack=False))
    assert rows.X.shape == (8, 64) and int(rows.X.max()) < 151936 and rows.bos_token_id is None
    assert torch.equal(rows.Y[:, :-1], rows.X[:, 1:])


def test_short_cpu_training_run_lowers_the_loss(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models.llama import LlamaForCausalLM
    args = _args(tmp_path, "--model", "qwen2.5-1.5b", "--no_cuda", "--seq_len", "64", "--min_seq_len", "8", "--pack",
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
