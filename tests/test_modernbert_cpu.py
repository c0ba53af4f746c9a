"""ModernBERT on the CPU: a tiny ModernBERT (hidden 128, two heads of dim 64, four layers so both layer types occur, a
local window of +-8 that clips inside the rows) against Hugging Face's ``ModernBertForMaskedLM`` on fixed, right-padded
and packed rows; ``window_bounds`` against an independently built band mask; the GeGLU and bias-free LayerNorm CPU
bodies; the two presets against Hugging Face's parameter counts and names; the CLI, the dataset's start id and a short
training run."""
import math
import types

import pytest
import torch

from b200ddp.ops import functional as Fn

MODERNBERT_CLS = 50281


def _tiny_cfg(**kw):
    from b200ddp.models.modernbert import ModernBertConfig
    return ModernBertConfig(**{**dict(vocab_size=512, hidden=128, layers=4, heads=2, intermediate=192, max_position=256,
                                      local_attention=16), **kw})


def _tiny_hf(seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.ModernBertConfig(vocab_size=512, hidden_size=128, intermediate_size=192, num_hidden_layers=4,
                                        num_attention_heads=2, max_position_embeddings=256, local_attention=16,
                                        pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2)
    cfg._attn_implementation = "eager"
    hf = transformers.ModernBertForMaskedLM(cfg).eval()
    with torch.no_grad():                            # Hugging Face starts the norms at 1 and the decoder bias at 0
        for n, p in hf.named_parameters():
            if "norm" in n:
                p.uniform_(0.5, 1.5)
        hf.decoder.bias.uniform_(-0.5, 0.5)
    return hf


def _ours(hf, **kw):
    from b200ddp.models.modernbert import ModernBertForMaskedLM
    m = ModernBertForMaskedLM(_tiny_cfg(**kw))
    m.load_hf_state_dict(hf.state_dict())
    return m.eval()


def test_tiny_modernbert_matches_hugging_face_logits_and_loss():
    hf = _tiny_hf()
    assert hf.config.layer_types == ["full_attention", "sliding_attention", "sliding_attention", "full_attention"]
    ours = _ours(hf)
    assert [layer.is_global for layer in ours.model.layers] == [True, False, False, True]
    ids = torch.randint(3, 512, (2, 40), generator=torch.Generator().manual_seed(3))
    labels = torch.where(torch.rand(2, 40, generator=torch.Generator().manual_seed(4)) < 0.3, ids, -100)
    with torch.no_grad():
        ref = hf(ids, labels=labels)
        logits = ours(ids)
    assert logits.shape == (2, 40, 512)
    assert torch.allclose(logits, ref.logits, atol=1e-4), float((logits - ref.logits).abs().max())
    assert abs(float(Fn.cross_entropy(logits, labels)) - float(ref.loss)) < 1e-4


def test_right_padded_modernbert_matches_hugging_face_on_real_tokens():
    hf = _tiny_hf(seed=1)
    ours = _ours(hf, pad_token_id=0)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(3, 512, (3, 48), generator=g)
    lens = torch.tensor([48, 30, 9])
    keep = torch.arange(48)[None, :] < lens[:, None]
    ids = torch.where(keep, ids, 0)
    with torch.no_grad():
        ref = hf(ids, attention_mask=keep.long()).logits
        logits = ours(ids)
    err = (logits - ref)[keep].abs().max()
    assert float(err) < 1e-4, float(err)


def test_packed_modernbert_row_matches_each_document_run_alone_through_hugging_face():
    CLS = 1
    hf = _tiny_hf(seed=4)
    ours = _ours(hf, pad_token_id=0, cls_token_id=CLS)
    g = torch.Generator().manual_seed(5)
    docs = [torch.cat([torch.tensor([CLS]), torch.randint(3, 512, (n - 1,), generator=g)]) for n in (27, 1, 20)]
    row = torch.cat(docs + [torch.zeros(64 - 48, dtype=torch.long)])[None]
    with torch.no_grad():
        packed = ours(row)[0]
        at = 0
        for d in docs:
            alone = hf(d[None]).logits[0]
            assert torch.allclose(packed[at:at + len(d)], alone, atol=1e-4), float((packed[at:at + len(d)] - alone).abs().max())
            at += len(d)


@pytest.mark.parametrize("window", [0, 1, 3, 7, 30, 63, 64, 200])
def test_window_bounds_mask_is_the_band_inside_each_document(window):
    S = 64
    ids = torch.full((3, S), 7)
    ids[0, [0, 20, 21, 45]] = 101                    # documents 0-19, 20, 21-44, 45-63
    ids[1, 50:] = 0                                  # one document, padded from 50
    ids[2] = 0                                       # all padding
    bounds, _ = Fn.document_bounds(ids, 101, 0)
    win = Fn.window_bounds(bounds, window)
    assert win.dtype == torch.int32 and win.shape == (3, S, 2)
    # independently: same document (the same start) and both real, and |i - j| <= window
    start = bounds[..., 0].long()
    real = bounds[..., 1] > bounds[..., 0]
    i = torch.arange(S)
    same_doc = (start[:, :, None] == start[:, None, :]) & real[:, :, None] & real[:, None, :]
    expect = same_doc & ((i[:, None] - i[None, :]).abs() <= window)
    assert torch.equal(Fn._bounds_mask(win, S, "cpu"), expect)
    assert (win[2] == 0).all() and (win[1, 50:] == 0).all()             # padding rows stay empty
    if window >= S - 1:
        assert win is bounds
    else:
        assert torch.equal(Fn.window_bounds(bounds.long(), window), win)


def test_window_bounds_rejects_bad_windows():
    bounds, _ = Fn.document_bounds(torch.ones(1, 8, dtype=torch.long), None, None)
    for bad in (-1, 2.0, 1.5, True, None):
        with pytest.raises(ValueError):
            Fn.window_bounds(bounds, bad)
    with pytest.raises(ValueError):
        Fn.window_bounds(bounds.float(), 2)
    with pytest.raises(ValueError):
        Fn.window_bounds(bounds[0], 2)


def test_geglu_cpu_body_and_gradient_match_hugging_face_expression():
    transformers = pytest.importorskip("transformers")
    act = transformers.activations.ACT2FN["gelu"]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 7, 2 * 24, generator=g, dtype=torch.float64, requires_grad=True)
    y = Fn.geglu(x)
    a, gate = x.chunk(2, -1)
    ref = act(a) * gate
    assert y.shape == (5, 7, 24) and torch.allclose(y, ref, atol=1e-12)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (gx,) = torch.autograd.grad(y, x, dy)
    (rx,) = torch.autograd.grad(ref, x, dy)
    assert torch.allclose(gx, rx, atol=1e-12)
    xb = x.detach().to(torch.bfloat16)
    assert Fn.geglu(xb).dtype == torch.bfloat16
    assert torch.equal(Fn.geglu(xb), (act(xb.float()[..., :24]) * xb.float()[..., 24:]).to(torch.bfloat16))
    with pytest.raises(ValueError):
        Fn.geglu(torch.randn(4, 7))


def test_bias_free_layer_norm_matches_torch():
    from b200ddp.ops import LayerNorm
    ours = LayerNorm(48, eps=1e-5, bias=False)
    ref = torch.nn.LayerNorm(48, eps=1e-5, bias=False)
    with torch.no_grad():
        ours.weight.uniform_(0.5, 1.5)
        ref.weight.copy_(ours.weight)
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in ref.named_parameters()] == ["weight"]
    x = torch.randn(6, 48, requires_grad=True)
    y, r = ours(x), ref(x)
    assert torch.allclose(y, r, atol=1e-6)
    dy = torch.randn_like(y)
    assert torch.allclose(torch.autograd.grad(y, (x, ours.weight), dy)[1], torch.autograd.grad(r, (x, ref.weight), dy)[1], atol=1e-5)
    assert [n for n, _ in LayerNorm(48).named_parameters()] == ["weight", "bias"]


@pytest.mark.parametrize("name,hf_kw,params,tensors", [
    ("modernbert-base", {}, 149_655_232, 137),
    ("modernbert-large", dict(hidden_size=1024, intermediate_size=2624, num_hidden_layers=28, num_attention_heads=16),
     395_881_664, 173)])
def test_presets_match_hugging_face_parameters_and_names(name, hf_kw, params, tensors):
    transformers = pytest.importorskip("transformers")
    from b200ddp.models import build_model
    with torch.device("meta"):
        m = build_model(name)
        m8 = build_model(name, fp8=True)
        hf = transformers.ModernBertForMaskedLM(transformers.ModernBertConfig(**hf_kw))
    assert sum(p.numel() for p in m.parameters()) == params == sum(p.numel() for p in hf.parameters())
    assert len(list(m.parameters())) == tensors == len(list(hf.parameters()))
    assert set(m.state_dict()) == set(hf.state_dict()) - {"decoder.weight"}
    c = m.config
    assert (c.vocab_size, c.max_position, c.eps, c.local_attention, c.global_every) == (50368, 8192, 1e-5, 128, 3)
    assert sum(layer.is_global for layer in m.model.layers) == (8 if name == "modernbert-base" else 10)
    fp8 = [n for n, x in m8.named_modules() if getattr(x, "fp8", False) is True]
    assert len(fp8) == 4 * c.layers and all(n.split(".", 3)[3] in ("attn.Wqkv", "attn.Wo", "mlp.Wi", "mlp.Wo") for n in fp8)


def test_load_hf_state_dict_checks_the_tie():
    hf = _tiny_hf()
    sd = dict(hf.state_dict())
    sd["decoder.weight"] = sd["decoder.weight"] + 1
    from b200ddp.models.modernbert import ModernBertForMaskedLM
    with pytest.raises(ValueError, match="decoder.weight"):
        ModernBertForMaskedLM(_tiny_cfg()).load_hf_state_dict(sd)


def test_init_follows_hugging_face_scheme():
    from b200ddp.models.modernbert import ModernBertForMaskedLM
    torch.manual_seed(0)
    m = ModernBertForMaskedLM(_tiny_cfg(layers=8))
    out = 0.02 / math.sqrt(16)
    for w, std in ((m.model.embeddings.tok_embeddings.weight, 0.02), (m.model.layers[3].attn.Wqkv.weight, 0.02),
                   (m.model.layers[3].mlp.Wi.weight, 0.02), (m.model.layers[3].attn.Wo.weight, out),
                   (m.model.layers[3].mlp.Wo.weight, out), (m.head.dense.weight, out)):
        w = w.detach()
        assert float(w.abs().max()) <= 2 * std and 0.8 * 0.88 * std < float(w.std()) < 1.2 * 0.88 * std   # sd of N cut at 2 sigma
    assert all(float(p.detach().min()) == float(p.detach().max()) == 1.0 for n, p in m.named_parameters() if "norm" in n)
    assert float(m.decoder.bias.detach().abs().max()) == 0.0


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_modernbert_cli_accepts_8192_tokens_and_rejects_more(tmp_path):
    from b200ddp.engine import cli
    cli.setup(_args(tmp_path, "--model", "modernbert-base", "--no_cuda", "--seq_len", "8192"))
    cli.setup(_args(tmp_path, "--model", "modernbert-large", "--no_cuda", "--seq_len", "8192", "--min_seq_len", "1024", "--pack"))
    with pytest.raises(ValueError, match="8192"):
        cli.setup(_args(tmp_path, "--model", "modernbert-base", "--no_cuda", "--seq_len", "8193"))
    with pytest.raises(ValueError, match="CUDA device"):
        cli.setup(_args(tmp_path, "--model", "modernbert-base", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="causal"):
        cli.setup(_args(tmp_path, "--model", "modernbert-base", "--no_cuda", "--fused_lm_loss"))


def test_modernbert_dataset_documents_start_with_its_cls_and_bert_keeps_101():
    from b200ddp.engine.trainer import build_dataset
    for model, cls in (("modernbert-base", MODERNBERT_CLS), ("bert-base", 101)):
        ds = build_dataset(types.SimpleNamespace(model=model, dataset_size=40, seq_len=64, min_seq_len=4, pack=True))
        assert ds.cls_token_id == cls and ds.pad_token_id == 0
        for x, docs in zip(ds.X, ds.doc_lengths):
            at = 0
            for n in docs:
                assert x[at] == cls and (x[at + 1:at + n] != cls).all()
                at += n
    rows = build_dataset(types.SimpleNamespace(model="modernbert-base", dataset_size=8, seq_len=64, min_seq_len=None, pack=False))
    assert rows.X.shape == (8, 64) and int(rows.X.max()) < 50368 and rows.cls_token_id is None


def test_short_cpu_modernbert_training_run_lowers_the_loss(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models.modernbert import ModernBertForMaskedLM
    args = _args(tmp_path, "--model", "modernbert-base", "--no_cuda", "--seq_len", "64", "--min_seq_len", "8", "--pack",
                 "--optimizer", "adamw", "--lr", "3e-3", "--max_steps", "30", "--per_gpu_train_batch_size", "4",
                 "--warmup_steps", "2", "--save_steps", "0", "--logging_steps", "10")
    cli.setup(args)
    ds = build_dataset(args)
    cls = ds.X == MODERNBERT_CLS                                   # a small alphabet leaves something to learn
    ds.X = torch.where(cls, torch.ones_like(ds.X), torch.where(ds.X > 0, ds.X % 16 + 2, ds.X))
    ds.Y = torch.where(ds.Y > 0, ds.Y % 16 + 2, ds.Y)
    ds.cls_token_id = 1
    model = ModernBertForMaskedLM(_tiny_cfg(pad_token_id=0, cls_token_id=1))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert math.isfinite(after) and after < before - 0.1, (before, after)
