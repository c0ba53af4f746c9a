"""Key-padding attention without a GPU: the CPU reference against fp64 SDPA, BERT padding invariance, the padded synthetic
dataset, the --min_seq_len checks, and a padded BERT training run on the CPU."""
import logging
import types

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import attention, attention_reference


def _sdpa_masked(qkv, lens, heads):
    B, S, W = qkv.shape
    q, k, v = (t.reshape(B, S, heads, -1).transpose(1, 2) for t in qkv.split(W // 3, dim=-1))
    mask = (torch.arange(S)[None, :] < lens[:, None])[:, None, None, :]
    return F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B, S, W // 3)


def test_reference_matches_fp64_sdpa_with_the_key_mask():
    torch.manual_seed(0)
    S, heads = 256, 2
    lens = torch.tensor([1, 127, 128, 129, 256, 7])
    qkv = torch.randn(len(lens), S, 3 * heads * 64, dtype=torch.float64)
    ref = _sdpa_masked(qkv, lens, heads)
    out = attention_reference(qkv.float(), lens, heads)
    assert out.dtype == torch.float32
    assert torch.allclose(out.double(), ref, rtol=1e-5, atol=1e-5)
    assert torch.allclose(attention_reference(qkv, lens, heads), ref, rtol=1e-12, atol=1e-12)


def test_length_zero_gives_zero_output_and_zero_gradient():
    torch.manual_seed(1)
    qkv = torch.randn(2, 128, 3 * 128, requires_grad=True)
    lens = torch.tensor([0, 40])
    out = attention(qkv, lens, 2)
    out.backward(torch.randn_like(out))
    assert (out[0] == 0).all() and torch.isfinite(out).all()
    assert (qkv.grad[0] == 0).all() and torch.isfinite(qkv.grad).all()
    assert (qkv.grad[1, 40:, 128:] == 0).all()                  # keys / values beyond the length get no gradient
    assert qkv.grad[1, :, :128].abs().sum() > 0


def test_cpu_op_gradient_matches_autograd_through_the_reference():
    torch.manual_seed(2)
    qkv = torch.randn(3, 128, 3 * 128, dtype=torch.float64)
    lens = torch.tensor([5, 128, 64])
    dy = torch.randn(3, 128, 128, dtype=torch.float64)
    a = qkv.clone().requires_grad_(True)
    attention(a, lens, 2).backward(dy)
    b = qkv.clone().requires_grad_(True)
    attention_reference(b, lens, 2).backward(dy)
    assert torch.allclose(a.grad, b.grad, rtol=1e-12, atol=1e-12)


def _tiny_cfg(**kw):
    from b200ddp.models.bert import BertConfig
    cfg = dict(vocab_size=1000, hidden=128, layers=2, heads=2, intermediate=256, max_position=256, pad_vocab_to=64)
    cfg.update(kw)
    return BertConfig(**cfg)


def test_bert_is_invariant_to_the_padded_length():
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(3)
    model = BertForMaskedLM(_tiny_cfg(pad_token_id=0)).eval()
    lens = [128, 77, 1, 100]
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(1, 1000, (4, 128), generator=g)
    labels = torch.randint(0, 1000, (4, 128), generator=g)
    pad = torch.arange(128)[None, :] >= torch.tensor(lens)[:, None]
    ids, labels = ids.masked_fill(pad, 0), labels.masked_fill(pad, -100)
    ids256 = torch.cat([ids, torch.zeros(4, 128, dtype=torch.long)], dim=1)
    labels256 = torch.cat([labels, torch.full((4, 128), -100)], dim=1)
    with torch.no_grad():
        a, b = model(ids), model(ids256)
        for i, n in enumerate(lens):
            assert torch.allclose(a[i, :n], b[i, :n], rtol=1e-4, atol=1e-4), i
        la, lb = cross_entropy(a, labels), cross_entropy(b, labels256)
    assert abs(float(la) - float(lb)) < 1e-4


def test_attn_mask_and_pad_token_id_are_exclusive():
    from b200ddp.models.bert import BertModel
    model = BertModel(_tiny_cfg(pad_token_id=0), with_pooler=False)
    ids = torch.randint(1, 1000, (2, 16))
    with pytest.raises(ValueError):
        model(ids, attn_mask=torch.ones(2, 1, 16, 16, dtype=torch.bool))


def test_bert_base_keeps_its_state_dict_with_a_pad_id():
    from b200ddp.models import bert_base
    a, b = bert_base(), bert_base(pad_token_id=0)
    assert {k: v.shape for k, v in a.state_dict().items()} == {k: v.shape for k, v in b.state_dict().items()}
    assert b.bert.config.pad_token_id == 0 and a.bert.config.pad_token_id is None


def test_synthetic_tokens_pad_only_the_tail():
    from b200ddp.data import SyntheticTokens
    ds = SyntheticTokens(samples=64, seq_len=128, vocab=500, min_len=20)
    assert ds.pad_token_id == 0 and ds.lengths is not None
    assert int(ds.lengths.min()) >= 20 and int(ds.lengths.max()) <= 128 and len(set(ds.lengths.tolist())) > 10
    pos = torch.arange(128)[None, :]
    tail = pos >= ds.lengths[:, None]
    assert (ds.X[tail] == 0).all() and (ds.Y[tail] == -100).all()
    assert (ds.X[~tail] >= 1).all() and (ds.X[~tail] < 500).all()
    again = SyntheticTokens(samples=64, seq_len=128, vocab=500, min_len=20)
    assert torch.equal(ds.X, again.X) and torch.equal(ds.Y, again.Y)


def test_synthetic_tokens_default_is_unchanged():
    from b200ddp.data import SyntheticTokens
    # the fixed-length recipe, spelled out: ids, then label candidates, then the mask draw, from one seeded generator
    g = torch.Generator().manual_seed(1234)
    X = torch.randint(0, 30522, (32, 64), generator=g)
    labels = torch.randint(0, 30522, (32, 64), generator=g)
    Y = torch.where(torch.rand(32, 64, generator=g) < 0.15, labels, torch.full_like(labels, -100))
    for kw in ({}, {"min_len": None}, {"min_len": 64}):
        ds = SyntheticTokens(samples=32, seq_len=64, **kw)
        assert torch.equal(ds.X, X) and torch.equal(ds.Y, Y), kw
        assert ds.lengths is None and ds.pad_token_id is None


def _args(**kw):
    base = dict(model="bert-base", seq_len=512, fp16=True, device=torch.device("cuda"), min_seq_len=128)
    base.update(kw)
    return types.SimpleNamespace(**base)


@pytest.mark.parametrize("kw", [dict(model="resnet50"), dict(model="foo"), dict(min_seq_len=0), dict(min_seq_len=513),
                                dict(fp16=False), dict(seq_len=384 + 64, min_seq_len=100)])
def test_invalid_min_seq_len_is_rejected(kw):
    from b200ddp.engine.cli import check_min_seq_len_args
    with pytest.raises(ValueError):
        check_min_seq_len_args(_args(**kw))


def test_valid_min_seq_len_is_accepted():
    from b200ddp.engine.cli import check_min_seq_len_args, padding_on
    check_min_seq_len_args(_args())
    check_min_seq_len_args(_args(min_seq_len=None, model="foo"))
    check_min_seq_len_args(_args(device=torch.device("cpu"), fp16=False, seq_len=100, min_seq_len=10))   # CPU: any length
    assert padding_on(_args()) and not padding_on(_args(min_seq_len=512)) and not padding_on(_args(min_seq_len=None))


def _cpu_args(tmp_path, **kw):
    from b200ddp.engine import cli
    argv = ["--model", "bert-base", "--no_cuda", "--max_steps", "12", "--seq_len", "64", "--min_seq_len", "16",
            "--per_gpu_train_batch_size", "8", "--optimizer", "adamw", "--lr", "2e-3", "--warmup_steps", "2",
            "--save_steps", "0", "--logging_steps", "4", "--no_tensorboard", "--output_dir", str(tmp_path / "out")]
    args = cli.build_parser().parse_args(argv)
    args.local_rank, args.n_gpu, args.world_size, args.node_rank = -1, 0, 1, 0
    args.device = torch.device("cpu")
    args.train_batch_size = 8
    for k, v in kw.items():
        setattr(args, k, v)
    return args


def test_padded_dataset_needs_a_model_that_derives_lengths(tmp_path):
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models.bert import BertForMaskedLM
    args = _cpu_args(tmp_path)
    with pytest.raises(ValueError):
        Trainer(args, BertForMaskedLM(_tiny_cfg()), logging.getLogger("test"))


def test_padded_tiny_bert_trains_on_the_cpu(tmp_path):
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models.bert import BertForMaskedLM
    torch.manual_seed(0)
    args = _cpu_args(tmp_path)
    model = BertForMaskedLM(_tiny_cfg(pad_token_id=0, vocab_size=30522))
    trainer = Trainer(args, model, logging.getLogger("test"))
    assert trainer.dataset.lengths is not None and int(trainer.dataset.lengths.min()) >= 16
    first = trainer.evaluate(max_batches=2)["eval_loss"]
    trainer.train()
    last = trainer.evaluate(max_batches=2)["eval_loss"]
    assert last < first - 0.05, (first, last)
