"""Packed-document BERT without a GPU: document_bounds, the packed reference against per-document attention, a tiny
packed BERT against each document run alone, the packed synthetic dataset, and the --pack checks."""
import logging
import types

import pytest
import torch

from b200ddp.ops import attention, attention_reference, document_bounds, packed_attention, packed_attention_reference

CLS, PAD = 101, 0


def test_document_bounds_on_hand_made_rows():
    ids = torch.tensor([[CLS, 5, 6, CLS, 7, PAD, PAD, PAD],     # a CLS in the middle, tail padding
                        [3, 4, CLS, 9, 9, 9, CLS, 2],           # no CLS at position 0
                        [PAD] * 8,                              # all padding
                        [CLS, 1, 1, 1, CLS, 1, PAD, CLS]])      # a CLS beyond the length is padding
    bounds, pos = document_bounds(ids, CLS, PAD)
    assert bounds.dtype == torch.int32 and bounds.shape == (4, 8, 2) and pos.dtype == torch.long
    assert bounds[0].tolist() == [[0, 3]] * 3 + [[3, 5]] * 2 + [[0, 0]] * 3
    assert pos[0].tolist() == [0, 1, 2, 0, 1, 0, 0, 0]
    assert bounds[1].tolist() == [[0, 2]] * 2 + [[2, 6]] * 4 + [[6, 8]] * 2
    assert pos[1].tolist() == [0, 1, 0, 1, 2, 3, 0, 1]
    assert bounds[2].tolist() == [[0, 0]] * 8 and pos[2].tolist() == [0] * 8
    # length 7 (one pad id): position 6 is inside it, position 7 (a CLS) is not
    assert bounds[3].tolist() == [[0, 4]] * 4 + [[4, 7]] * 3 + [[0, 0]]
    assert pos[3].tolist() == [0, 1, 2, 3, 0, 1, 2, 0]
    # no pad id: every position is inside the row's length
    b2, p2 = document_bounds(ids, CLS, None)
    assert b2[3].tolist() == [[0, 4]] * 4 + [[4, 7]] * 3 + [[7, 8]] and p2[3].tolist() == [0, 1, 2, 3, 0, 1, 2, 0]
    assert b2[2].tolist() == [[0, 8]] * 8 and p2[2].tolist() == list(range(8))
    for p in (pos, p2):
        assert (p >= 0).all()


def test_document_bounds_random_rows_have_nonnegative_positions_inside_their_document():
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, 120, (16, 64), generator=g)           # pad ids and CLS ids anywhere
    bounds, pos = document_bounds(ids, CLS, PAD)
    start, end = bounds[..., 0].long(), bounds[..., 1].long()
    j = torch.arange(64)
    lens = (ids != PAD).sum(1, keepdim=True)
    inside = j < lens
    assert (pos >= 0).all() and (pos < 64).all()
    assert ((start <= j) & (j < end))[inside].all()
    assert (start == end)[~inside].all()
    assert torch.equal(pos[inside], (j - start)[inside])


def _packed_row(doc_lens, S, heads, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(1, S, 3 * heads * 64, generator=g, dtype=dtype)
    ids = torch.full((1, S), PAD)
    at = 0
    for n in doc_lens:
        ids[0, at:at + n] = 7
        ids[0, at] = CLS
        at += n
    return qkv, ids


def test_packed_reference_equals_each_document_alone():
    S, heads = 256, 2
    doc_lens = [1, 63, 64, 65, 40, 3]
    qkv, ids = _packed_row(doc_lens, S, heads, seed=1)
    bounds, _ = document_bounds(ids, CLS, PAD)
    out = packed_attention_reference(qkv, bounds, heads)
    at = 0
    for n in doc_lens:
        alone = torch.zeros(1, S, qkv.shape[-1])
        alone[0, :n] = qkv[0, at:at + n]
        ref = attention_reference(alone, torch.tensor([n]), heads)
        assert torch.allclose(out[0, at:at + n], ref[0, :n], rtol=1e-5, atol=1e-5), n
        at += n
    assert (out[0, at:] == 0).all()                             # padding rows see no key


def test_packed_op_gradient_matches_the_reference_and_isolates_documents():
    S, heads = 128, 2
    qkv, ids = _packed_row([50, 30, 20], S, heads, seed=2, dtype=torch.float64)
    bounds, _ = document_bounds(ids, CLS, PAD)
    dy = torch.randn(1, S, heads * 64, dtype=torch.float64)
    a = qkv.clone().requires_grad_(True)
    packed_attention(a, bounds, heads).backward(dy)
    b = qkv.clone().requires_grad_(True)
    packed_attention_reference(b, bounds, heads).backward(dy)
    assert torch.allclose(a.grad, b.grad, rtol=1e-12, atol=1e-12)
    assert (a.grad[0, 100:] == 0).all()                         # padding gets no gradient
    dy2 = torch.zeros_like(dy)
    dy2[0, :50] = dy[0, :50]                                     # gradient of the first document's output only
    c = qkv.clone().requires_grad_(True)
    packed_attention(c, bounds, heads).backward(dy2)
    assert (c.grad[0, 50:] == 0).all()


def _tiny_cfg(**kw):
    from b200ddp.models.bert import BertConfig
    cfg = dict(vocab_size=1000, hidden=128, layers=2, heads=2, intermediate=256, max_position=128, pad_vocab_to=64)
    cfg.update(kw)
    return BertConfig(**cfg)


def test_tiny_packed_bert_equals_each_document_alone():
    """Position ids restart per document and nothing crosses a document boundary: every document's logits equal those
    of the same document alone in a right-padded row."""
    from b200ddp.models.bert import BertForMaskedLM
    torch.manual_seed(3)
    packed = BertForMaskedLM(_tiny_cfg(pad_token_id=PAD, cls_token_id=CLS)).eval()
    padded = BertForMaskedLM(_tiny_cfg(pad_token_id=PAD)).eval()
    padded.load_state_dict(packed.state_dict())
    S = 128
    rows = [[40, 1, 57, 20], [128], [64, 63]]
    g = torch.Generator().manual_seed(4)
    ids = torch.full((len(rows), S), PAD)
    docs = []
    for r, lens in enumerate(rows):
        at = 0
        for n in lens:
            doc = torch.randint(1, 1000, (n,), generator=g)
            doc[doc == CLS] = 7
            doc[0] = CLS
            ids[r, at:at + n] = doc
            docs.append((r, at, doc))
            at += n
    with torch.no_grad():
        out = packed(ids)
        for r, at, doc in docs:
            alone = torch.full((1, S), PAD)
            alone[0, :len(doc)] = doc
            ref = padded(alone)
            assert torch.allclose(out[r, at:at + len(doc)], ref[0, :len(doc)], rtol=0, atol=1e-5), (r, at, len(doc))


def test_attn_mask_and_cls_token_id_are_exclusive():
    from b200ddp.models.bert import BertModel
    model = BertModel(_tiny_cfg(cls_token_id=CLS), with_pooler=False)
    with pytest.raises(ValueError):
        model(torch.randint(1, 1000, (2, 16)), attn_mask=torch.ones(2, 1, 16, 16, dtype=torch.bool))


def test_bert_base_keeps_its_state_dict_with_a_cls_id():
    from b200ddp.models import bert_base
    a, b = bert_base(), bert_base(pad_token_id=0, cls_token_id=CLS)
    assert {k: v.shape for k, v in a.state_dict().items()} == {k: v.shape for k, v in b.state_dict().items()}
    assert b.bert.config.cls_token_id == CLS and a.bert.config.cls_token_id is None


# ---- dataset ------------------------------------------------------------------------------------------------------------
def test_packed_dataset_invariants():
    from b200ddp.data import SyntheticTokens
    ds = SyntheticTokens(samples=200, seq_len=128, vocab=500, min_len=16, pack=True)
    assert ds.cls_token_id == CLS and ds.pad_token_id == PAD and len(ds) == ds.X.shape[0] < 200
    assert sorted(i for row in ds.doc_ids for i in row) == list(range(200))      # every document exactly once
    for r in range(len(ds)):
        lens = ds.doc_lengths[r]
        fill = sum(lens)
        assert fill <= 128 and int(ds.lengths[r]) == fill
        x, y = ds.X[r], ds.Y[r]
        starts = torch.tensor([0] + lens[:-1]).cumsum(0)
        is_cls = torch.zeros(128, dtype=torch.bool)
        is_cls[starts] = True
        assert torch.equal(x == CLS, is_cls), r                  # CLS only at document starts
        assert (x[fill:] == PAD).all() and (y[fill:] == -100).all()
        assert (x[:fill] != PAD).all() and (x[:fill] < 500).all()  # padding only in the tail
        assert all(16 <= n <= 128 for n in lens)
    again = SyntheticTokens(samples=200, seq_len=128, vocab=500, min_len=16, pack=True)
    assert torch.equal(ds.X, again.X) and torch.equal(ds.Y, again.Y) and ds.doc_ids == again.doc_ids
    other = SyntheticTokens(samples=200, seq_len=128, vocab=500, min_len=16, pack=True, seed=5)
    assert not torch.equal(ds.X[:, :8], other.X[:, :8]) or ds.doc_ids != other.doc_ids


def test_packed_dataset_pads_less_than_ten_percent_at_the_defaults():
    from b200ddp.data import SyntheticTokens
    ds = SyntheticTokens(min_len=128, pack=True)
    fill = float(ds.lengths.float().mean()) / 512
    assert 1.0 - fill < 0.10, 1.0 - fill
    assert sum(len(r) for r in ds.doc_lengths) == 512


def test_default_and_padded_datasets_are_unchanged_by_packing():
    from b200ddp.data import SyntheticTokens
    for kw in ({}, {"min_len": 20}):
        a = SyntheticTokens(samples=32, seq_len=64, **kw)
        b = SyntheticTokens(samples=32, seq_len=64, pack=False, **kw)
        assert torch.equal(a.X, b.X) and torch.equal(a.Y, b.Y) and a.cls_token_id is None and a.doc_lengths is None


# ---- CLI and trainer ----------------------------------------------------------------------------------------------------
def _args(**kw):
    base = dict(model="bert-base", seq_len=512, fp16=True, device=torch.device("cuda"), min_seq_len=128, pack=True)
    base.update(kw)
    return types.SimpleNamespace(**base)


@pytest.mark.parametrize("kw", [dict(min_seq_len=None), dict(min_seq_len=512), dict(model="resnet50"), dict(model="foo"),
                                dict(fp16=False), dict(seq_len=384 + 64, min_seq_len=100)])
def test_invalid_pack_is_rejected(kw):
    from b200ddp.engine.cli import check_pack_args
    with pytest.raises(ValueError):
        check_pack_args(_args(**kw))


def test_valid_pack_is_accepted():
    from b200ddp.engine.cli import check_pack_args
    check_pack_args(_args())
    check_pack_args(_args(pack=False, min_seq_len=None, model="foo"))
    check_pack_args(_args(device=torch.device("cpu"), fp16=False, seq_len=100, min_seq_len=10))


def test_pack_flag_parses_and_without_min_seq_len_fails_setup():
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--model", "bert-base", "--no_cuda", "--pack"])
    assert args.pack
    with pytest.raises(ValueError):
        cli.check_pack_args(types.SimpleNamespace(**{**vars(args), "device": torch.device("cpu")}))


def _cpu_args(tmp_path, **kw):
    from b200ddp.engine import cli
    argv = ["--model", "bert-base", "--no_cuda", "--max_steps", "12", "--seq_len", "64", "--min_seq_len", "16", "--pack",
            "--per_gpu_train_batch_size", "8", "--optimizer", "adamw", "--lr", "2e-3", "--warmup_steps", "2",
            "--save_steps", "0", "--logging_steps", "4", "--no_tensorboard", "--output_dir", str(tmp_path / "out")]
    args = cli.build_parser().parse_args(argv)
    args.local_rank, args.n_gpu, args.world_size, args.node_rank = -1, 0, 1, 0
    args.device = torch.device("cpu")
    args.train_batch_size = 8
    for k, v in kw.items():
        setattr(args, k, v)
    return args


@pytest.mark.parametrize("cfg", [dict(), dict(pad_token_id=PAD), dict(pad_token_id=PAD, cls_token_id=5)])
def test_packed_dataset_needs_a_model_that_derives_documents(tmp_path, cfg):
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models.bert import BertForMaskedLM
    with pytest.raises(ValueError):
        Trainer(_cpu_args(tmp_path), BertForMaskedLM(_tiny_cfg(vocab_size=30522, **cfg)), logging.getLogger("test"))


def test_packed_tiny_bert_trains_on_the_cpu(tmp_path, caplog):
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models.bert import BertForMaskedLM
    torch.manual_seed(0)
    model = BertForMaskedLM(_tiny_cfg(pad_token_id=PAD, cls_token_id=CLS, vocab_size=30522))
    with caplog.at_level(logging.INFO, logger="test"):
        trainer = Trainer(_cpu_args(tmp_path), model, logging.getLogger("test"))
    assert trainer.dataset.doc_lengths is not None and trainer.count_pad_id == PAD
    assert any("Packed sequences." in r.getMessage() for r in caplog.records)
    first = trainer.evaluate(max_batches=2)["eval_loss"]
    with caplog.at_level(logging.INFO, logger="test"):
        trainer.train()
    last = trainer.evaluate(max_batches=2)["eval_loss"]
    assert last < first - 0.05, (first, last)
    done = [r for r in caplog.records if "Finished training." in r.getMessage()]
    assert done and "tokens_per_s" in done[-1].args and done[-1].args["tokens_per_s"] > 0
