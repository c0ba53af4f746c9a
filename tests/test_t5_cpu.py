"""T5 on the CPU: the relative position bucket and the clamped table against transformers, the table's gradient,
``relative_attention`` against a dense-bias attention written independently of it, and ``models/t5.py`` against
``transformers.T5ForConditionalGeneration`` (parameter counts, strict loading, loss, logits and every gradient in fp32)."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import (packed_attention_reference, relative_attention, relative_attention_reference,
                         relative_position_bucket, relative_position_table)
from b200ddp.ops.functional import document_bounds

transformers = pytest.importorskip("transformers")
from transformers.models.t5.modeling_t5 import T5Attention  # noqa: E402


@pytest.mark.parametrize("bidirectional", [True, False])
def test_bucket_matches_transformers(bidirectional):
    rel = torch.arange(-4096, 4097)
    ours = relative_position_bucket(rel, bidirectional)
    ref = T5Attention._relative_position_bucket(rel, bidirectional=bidirectional, num_buckets=32, max_distance=128)
    assert torch.equal(ours, ref)
    # beyond +-128 every distance shares the bucket of +-128, which is what makes the 257-column table exact
    assert torch.equal(ours, relative_position_bucket(rel.clamp(-128, 128), bidirectional))


@pytest.mark.parametrize("bidirectional", [True, False])
@pytest.mark.parametrize("S", [1, 100, 257, 1024])
def test_table_reproduces_compute_bias(bidirectional, S):
    cfg = transformers.T5Config(num_heads=3, d_model=192, d_kv=64, relative_attention_num_buckets=32,
                                relative_attention_max_distance=128, is_decoder=not bidirectional)
    torch.manual_seed(S)
    att = T5Attention(cfg, has_relative_attention_bias=True)
    torch.nn.init.normal_(att.relative_attention_bias.weight)
    with torch.no_grad():
        dense = att.compute_bias(S, S)[0]                                  # [H, S, S]
        table = relative_position_table(att.relative_attention_bias.weight, bidirectional)
    pos = torch.arange(S)
    col = (pos[None, :] - pos[:, None]).clamp(-128, 128) + 128
    assert table.dtype == torch.float32 and table.shape == (3, 257)
    assert torch.equal(table[:, col], dense)


@pytest.mark.parametrize("bidirectional", [True, False])
def test_table_gradient_is_the_gather_gradient(bidirectional):
    torch.manual_seed(0)
    w = torch.randn(32, 4, dtype=torch.float64, requires_grad=True)
    dt = torch.randn(4, 257, dtype=torch.float64)
    relative_position_table(w, bidirectional).backward(dt)
    idx = relative_position_bucket(torch.arange(-128, 129), bidirectional)
    w2 = w.detach().clone().requires_grad_(True)
    w2[idx].t().backward(dt)
    assert torch.allclose(w.grad, w2.grad, rtol=1e-12, atol=0)


def _dense_bias_sdpa(qkv, bounds, table, heads, causal):
    """Attention with T5's bias through SDPA's float mask: unscaled scores (scale 1), bias + -inf where hidden."""
    B, S, W = qkv.shape
    hidden = W // 3
    q, k, v = (t.reshape(B, S, heads, hidden // heads).transpose(1, 2).double() for t in qkv.split(hidden, -1))
    pos = torch.arange(S)
    bias = table.double()[:, (pos[None, :] - pos[:, None]).clamp(-128, 128) + 128]      # [H, S, S]
    b = bounds.long()
    vis = (pos >= b[..., :1]) & (pos < b[..., 1:])                                       # [B, S, S]
    if causal:
        vis &= pos[None, :] <= pos[:, None]
    mask = bias[None] + torch.where(vis[:, None], 0.0, -math.inf)
    live = vis.any(-1)[:, None, :, None]
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=torch.where(live, mask, 0.0), scale=1.0)
    return torch.where(live, o, 0.0).transpose(1, 2).reshape(B, S, hidden)


@pytest.mark.parametrize("causal", [False, True])
def test_relative_attention_matches_dense_bias_sdpa(causal):
    torch.manual_seed(1)
    B, S, H = 3, 300, 3
    ids = torch.full((B, S), 7)
    ids[0, [0, 90, 200]] = 2
    ids[1, 150:] = 0                      # right padding
    ids[2] = 0                            # an all-padding row
    bounds, _ = document_bounds(ids, 2, 0)
    qkv = torch.randn(B, S, 3 * H * 64, dtype=torch.float64, requires_grad=True)
    table = torch.randn(H, 257, dtype=torch.float64, requires_grad=True)
    dy = torch.randn(B, S, H * 64, dtype=torch.float64)
    out = relative_attention(qkv, bounds, table, H, causal)
    ref = _dense_bias_sdpa(qkv, bounds, table, H, causal)
    assert torch.allclose(out, ref, rtol=1e-10, atol=1e-10)
    assert (out[2] == 0).all()
    g = torch.autograd.grad(out, (qkv, table), dy)
    g_ref = torch.autograd.grad(ref, (qkv, table), dy)
    for a, b in zip(g, g_ref):
        assert torch.allclose(a, b, rtol=1e-9, atol=1e-9)


def test_zero_table_and_prescaled_queries_give_packed_attention():
    """With a zero table the biased attention is packed attention on queries scaled by 1/sqrt(64) = 1/8."""
    torch.manual_seed(2)
    B, S, H = 2, 256, 2
    ids = torch.full((B, S), 7)
    ids[0, 100] = 2
    ids[1, 200:] = 0
    bounds, _ = document_bounds(ids, 2, 0)
    qkv = torch.randn(B, S, 3 * H * 64, dtype=torch.float64)
    scaled = qkv.clone()
    scaled[..., :H * 64] /= 8
    out = relative_attention_reference(scaled, bounds, torch.zeros(H, 257, dtype=torch.float64), H, causal=False)
    assert torch.allclose(out, packed_attention_reference(qkv, bounds, H), rtol=1e-12, atol=1e-12)


def test_packed_rows_equal_each_document_alone():
    """Distances are k - i inside a row, so a document packed after others gets the bias it gets alone."""
    torch.manual_seed(3)
    S, H = 384, 2
    docs = [130, 200, 54]
    qkv = torch.randn(1, S, 3 * H * 64, dtype=torch.float64)
    table = torch.randn(H, 257, dtype=torch.float64)
    ids = torch.full((1, S), 7)
    ids[0, [0, 130, 330]] = 2
    bounds, _ = document_bounds(ids, 2, None)
    for causal in (False, True):
        packed = relative_attention(qkv, bounds, table, H, causal)
        at = 0
        for n in docs:
            alone = relative_attention(qkv[:, at:at + n], torch.tensor([[[0, n]] * n]), table, H, causal)
            assert torch.allclose(packed[:, at:at + n], alone, rtol=1e-12, atol=1e-12)
            at += n


def test_table_rejects_a_weight_that_is_not_2d():
    with pytest.raises(ValueError):
        relative_position_table(torch.zeros(32), True)


# ---- the model against transformers.T5ForConditionalGeneration ---------------------------------------------------------
def _hf_config(**kw):
    base = dict(vocab_size=320, d_model=128, d_kv=64, num_heads=2, d_ff=256, num_layers=2, num_decoder_layers=2, dropout_rate=0.0,
                feed_forward_proj="relu", tie_word_embeddings=True, relative_attention_num_buckets=32,
                relative_attention_max_distance=128, decoder_start_token_id=0, pad_token_id=0, eos_token_id=1)
    base.update(kw)
    return transformers.T5Config(**base)


def _ours_like(hf_cfg, **kw):
    from b200ddp.models.t5 import T5Config, T5ForConditionalGeneration
    return T5ForConditionalGeneration(T5Config(vocab_size=hf_cfg.vocab_size, d_model=hf_cfg.d_model, num_layers=hf_cfg.num_layers,
                                               num_decoder_layers=hf_cfg.num_decoder_layers, num_heads=hf_cfg.num_heads,
                                               d_kv=hf_cfg.d_kv, d_ff=hf_cfg.d_ff, **kw))


@pytest.mark.parametrize("name,count", [("t5-small", 60_506_624), ("t5-base", 222_903_552)])
def test_parameter_counts_match_transformers(name, count):
    from b200ddp.models.t5 import T5_BASE, T5_SMALL, T5ForConditionalGeneration
    preset = {"t5-small": T5_SMALL, "t5-base": T5_BASE}[name]
    with torch.device("meta"):
        ours = T5ForConditionalGeneration(preset)
        hf = transformers.T5ForConditionalGeneration(transformers.T5Config(
            vocab_size=32128, d_model=preset.d_model, d_kv=64, d_ff=preset.d_ff, num_layers=preset.num_layers,
            num_decoder_layers=preset.num_decoder_layers, num_heads=preset.num_heads, feed_forward_proj="relu"))
    assert sum(p.numel() for p in ours.parameters()) == count == sum(p.numel() for p in hf.parameters())


def test_load_hf_state_dict_is_strict():
    torch.manual_seed(0)
    hf = transformers.T5ForConditionalGeneration(_hf_config())
    sd = hf.state_dict()
    ours = _ours_like(hf.config)
    ours.load_hf_state_dict(sd)
    missing = dict(sd)
    del missing["decoder.block.1.layer.1.EncDecAttention.k.weight"]
    with pytest.raises(KeyError, match="missing"):
        ours.load_hf_state_dict(missing)
    extra = dict(sd)
    extra["encoder.block.1.layer.0.SelfAttention.relative_attention_bias.weight"] = torch.zeros(32, 2)
    with pytest.raises(KeyError, match="unexpected"):
        ours.load_hf_state_dict(extra)


def _grads_as_ours(model_like, named_grads):
    """transformers' parameter gradients in our layout (through load_hf_state_dict's mapping)."""
    model_like.load_hf_state_dict(named_grads)
    return {k: v.detach() for k, v in model_like.state_dict().items()}


@pytest.mark.parametrize("src_len,tgt_len", [((300, 17), (40, 150)), ((129, 256), (1, 64)), ((200, 5), (130, 12))])
def test_fp32_model_matches_transformers(src_len, tgt_len):
    """Right-padded pairs: loss, logits at labelled positions and every parameter gradient, both relative biases included."""
    torch.manual_seed(sum(src_len) + sum(tgt_len))
    hf = transformers.T5ForConditionalGeneration(_hf_config())
    ours = _ours_like(hf.config, pad_token_id=0)
    ours.load_hf_state_dict(hf.state_dict())
    B, Sk, Sq = 2, max(src_len), max(tgt_len)
    src = torch.randint(3, 320, (B, Sk))
    labels = torch.randint(3, 320, (B, Sq))
    for b in range(B):
        src[b, src_len[b]:] = 0
        labels[b, tgt_len[b]:] = -100
    out = hf(input_ids=src, attention_mask=(src != 0).long(), labels=labels)
    out.loss.backward()
    logits = ours(src, labels)
    loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), labels.reshape(-1), ignore_index=-100)
    loss.backward()
    assert torch.allclose(loss, out.loss, rtol=1e-5, atol=1e-5)
    keep = labels != -100
    assert torch.allclose(logits[keep], out.logits[keep], rtol=1e-4, atol=1e-4)
    want = _grads_as_ours(_ours_like(hf.config), {k: p.grad for k, p in hf.named_parameters()})
    for k, p in ours.named_parameters():
        assert torch.allclose(p.grad, want[k], rtol=1e-4, atol=1e-5), k
    assert ours.encoder.relative_attention_bias.weight.grad.abs().sum() > 0
    assert ours.decoder.relative_attention_bias.weight.grad.abs().sum() > 0


def test_packed_rows_equal_each_pair_alone():
    torch.manual_seed(5)
    cfg = _hf_config()
    ours = _ours_like(cfg, pad_token_id=0, bos_token_id=2)
    alone = _ours_like(cfg, pad_token_id=0)
    alone.load_state_dict(ours.state_dict())
    pairs = [(150, 60), (90, 40), (40, 30)]
    Sk, Sq = 300, 140
    src = torch.zeros(1, Sk, dtype=torch.long)
    labels = torch.full((1, Sq), -100)
    a = b = 0
    docs = []
    for s, t in pairs:
        xs, xt = torch.randint(3, 320, (s,)), torch.randint(3, 320, (t,))
        xs[0] = xt[0] = 2
        src[0, a:a + s], labels[0, b:b + t] = xs, xt
        docs.append((xs, xt, b))
        a, b = a + s, b + t
    packed = ours(src, labels)
    for xs, xt, at in docs:
        one = alone(xs[None], xt[None])
        assert torch.allclose(packed[0, at:at + len(xt)], one[0], rtol=1e-4, atol=1e-4)


# ---- span-corruption data, registry, CLI and training -----------------------------------------------------------------
def _split_docs(row, start):
    """A row's documents (each starting with `start`), padding (0 or -100) dropped."""
    row = [int(v) for v in row if v not in (0, -100)]
    docs = []
    for v in row:
        if v == start or not docs:
            docs.append([])
        docs[-1].append(v)
    return docs


def _reassemble(src, tgt):
    """The document text from a source and its target, checking the sentinels on the way."""
    from b200ddp.data import SyntheticSpanCorruption as D
    assert src[0] == tgt[0] == 2 and src[-1] == tgt[-1] == D.EOS_ID
    spans, cur = {}, None
    for v in tgt[1:-1]:
        if v > D.FIRST_SENTINEL - 100:
            cur = v
            spans[cur] = []
        else:
            spans[cur].append(v)
    sentinels = list(spans)
    assert sentinels == list(range(D.FIRST_SENTINEL, D.FIRST_SENTINEL - len(sentinels), -1))   # descending, in order
    assert spans[sentinels[-1]] == []                                                          # the closing sentinel
    text, seen = [], []
    for v in src[1:-1]:
        if v > D.FIRST_SENTINEL - 100:
            seen.append(v)
            text += spans[v]
        else:
            text.append(v)
    assert seen == sentinels[:-1] and all(spans[s] for s in seen)
    return text, len(seen), sum(len(spans[s]) for s in seen)


@pytest.mark.parametrize("pack", [False, True])
def test_span_corruption_reassembles_and_packs(pack):
    from b200ddp.data import SyntheticSpanCorruption as D
    ds = D(samples=40, seq_len=256, min_len=8, pack=pack, seed=7)
    assert ds.Y.shape[1] == D.target_width_for(256) == 128 and D.target_width_for(512) == 128 and D.target_width_for(1024) == 256
    pairs = 0
    for x, y in zip(ds.X, ds.Y):
        srcs, tgts = _split_docs(x, 2), _split_docs(y, 2)
        assert len(srcs) == len(tgts) and (pack or len(srcs) == 1)
        assert sum(map(len, srcs)) <= 256 and sum(map(len, tgts)) <= ds.Y.shape[1]      # both fits
        for s, t in zip(srcs, tgts):
            text, spans, noise = _reassemble(s, t)
            n = len(text)
            assert all(3 <= v < D.TEXT_END for v in text)
            assert noise == min(max(round(0.15 * n), 1), n - 1) and spans == max(round(noise / 3), 1)
            pairs += 1
    assert pairs == 40
    assert ds.lengths.tolist() == (ds.X != 0).sum(1).tolist()
    if pack:
        assert ds.bos_token_id == 2 and len(ds) < 40 and sorted(i for r in ds.doc_ids for i in r) == list(range(40))
    again = D(samples=40, seq_len=256, min_len=8, pack=pack, seed=7)
    assert torch.equal(again.X, ds.X) and torch.equal(again.Y, ds.Y)
    other = D(samples=40, seq_len=256, min_len=8, pack=pack, seed=8)
    assert not torch.equal(other.X, ds.X)


def test_span_corruption_fixed_sources_fill_the_row():
    from b200ddp.data import SyntheticSpanCorruption as D
    ds = D(samples=6, seq_len=512)
    assert ds.X.shape == (6, 512) and ds.Y.shape == (6, 128)
    assert ((ds.X != 0).sum(1) >= 511).all() and ((ds.Y != -100).sum(1) <= 128).all()


def test_packing_checks_the_target_row_too():
    """Short documents have long targets for their sources: packing by source length alone would overflow the label
    columns here, so the packer must (and does) check both rows."""
    from b200ddp.data import SyntheticSpanCorruption as D
    ds = D(samples=1000, seq_len=512, min_len=4, pack=True, seed=3)
    width = ds.Y.shape[1]
    docs = [(len(s), len(t)) for x, y in zip(ds.X, ds.Y) for s, t in zip(_split_docs(x, 2), _split_docs(y, 2))]
    assert len(docs) == 1000 and width == 128
    for x, y in zip(ds.X, ds.Y):
        assert (x != 0).sum() <= 512 and (y != -100).sum() <= width
    free, fill = [], []                                         # first fit decreasing on the sources alone
    for s, t in sorted(docs, key=lambda d: -d[0]):
        r = next((r for r, f in enumerate(free) if f >= s), len(free))
        if r == len(free):
            free.append(512)
            fill.append(0)
        free[r] -= s
        fill[r] += t
    assert max(fill) > width


def _cli_args(tmp_path, model, *flags):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", model, "--no_cuda", *flags])


@pytest.mark.parametrize("flags", [[], ["--min_seq_len", "32", "--seq_len", "128"], ["--pack", "--min_seq_len", "32", "--seq_len", "128"],
                                   ["--fused_lm_loss"], ["--cuda_graph"], ["--optimizer", "adamw", "--gradient_accumulation_steps", "2"],
                                   ["--seq_len", "1024"]])
@pytest.mark.parametrize("model", ["t5-small", "t5-base"])
def test_cli_accepts(tmp_path, model, flags):
    from b200ddp.engine import cli
    cli.setup(_cli_args(tmp_path, model, *flags))


@pytest.mark.parametrize("flags,match", [(["--fp8", "--fp16"], "--fp8"), (["--sparse_prediction"], "--sparse_prediction"),
                                         (["--seq_len", "1025"], "1024")])
def test_cli_rejects(tmp_path, flags, match):
    from b200ddp.engine import cli
    with pytest.raises(ValueError, match=match):
        cli.setup(_cli_args(tmp_path, "t5-small", *flags))


def test_cli_rejects_gpu_misuse():
    import argparse
    from b200ddp.engine import cli
    for fp16, seq_len, match in ((False, 128, "--fp16"), (True, 100, "multiple of 128")):
        args = argparse.Namespace(model="t5-small", device=torch.device("cuda"), fp16=fp16, seq_len=seq_len)
        with pytest.raises(ValueError, match=match):
            cli.check_seq2seq_args(args)


def test_registry_and_dataset(tmp_path):
    from b200ddp.data import SyntheticSpanCorruption
    from b200ddp.engine.trainer import build_dataset
    from b200ddp.models import MODEL_REGISTRY
    for name in ("t5-small", "t5-base"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "causal" and e.seq2seq and e.start_id == 2 and e.config.max_position == 1024 and not e.fp8
    ds = build_dataset(_cli_args(tmp_path, "t5-small", "--pack", "--min_seq_len", "16", "--seq_len", "128"))
    assert isinstance(ds, SyntheticSpanCorruption) and ds.bos_token_id == 2 and ds.Y.shape[1] == 128


def _tiny_t5_entry(monkeypatch):
    """t5-small's registry entry with a 1-layer, d 128 model, so CPU training runs stay short."""
    from b200ddp import models
    from b200ddp.models import t5 as t5mod
    tiny = t5mod.T5Config(d_model=128, num_layers=1, num_decoder_layers=1, num_heads=2, d_ff=256)
    monkeypatch.setitem(models.MODEL_REGISTRY, "t5-small", models.ModelEntry(
        lambda **kw: t5mod._build(tiny, kw.get("pad_token_id"), kw.get("bos_token_id"), kw.get("fused_lm_loss", False)),
        "causal", tiny, start_id=2, seq2seq=True))


def test_short_cpu_training_run_resumes(tmp_path, monkeypatch):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    _tiny_t5_entry(monkeypatch)
    flags = ["--per_gpu_train_batch_size", "2", "--max_steps", "2", "--logging_steps", "1", "--save_steps", "2", "--optimizer", "adamw",
             "--lr", "1e-4", "--dataset_size", "8", "--seq_len", "64", "--min_seq_len", "16", "--pack"]
    args = _cli_args(tmp_path, "t5-small", *flags)
    cli.setup(args)
    step, loss = Trainer(args, build_model("t5-small", pad_token_id=0, bos_token_id=2), cli.log).train()
    assert step == 3 and math.isfinite(loss) and loss > 0
    args = _cli_args(tmp_path, "t5-small", *flags[:5], "4", *flags[6:], "--resume_from", "latest")
    cli.setup(args)
    step, loss = Trainer(args, build_model("t5-small", pad_token_id=0, bos_token_id=2), cli.log).train()
    assert step >= 3 and math.isfinite(loss)


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gloo_model():
    from b200ddp.models.t5 import T5Config, T5ForConditionalGeneration
    torch.manual_seed(0)
    return T5ForConditionalGeneration(T5Config(vocab_size=32128, d_model=64, num_layers=1, num_decoder_layers=1, num_heads=1,
                                               d_ff=128, pad_token_id=0)).double()


def _gloo_data():
    from b200ddp.data import SyntheticSpanCorruption
    return SyntheticSpanCorruption(samples=4, seq_len=48, min_len=12, seed=3)


def _gloo_loss(model, x, y):
    logits = model(x, y)
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]), y.reshape(-1))


def _ddp_worker(rank, world, port, path):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200ddp.parallel import DistributedDataParallel
        model = _gloo_model()
        ddp = DistributedDataParallel(model, backend="gloo")
        ds = _gloo_data()
        n = len(ds) // world
        _gloo_loss(ddp, ds.X[rank * n:(rank + 1) * n], ds.Y[rank * n:(rank + 1) * n]).backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        torch.optim.SGD(model.parameters(), lr=0.1).step()
        torch.save({"grads": grads, "params": {k: p.detach().clone() for k, p in model.named_parameters()}}, f"{path}.{rank}")
    finally:
        dist.destroy_process_group()


def test_gloo_world_2_keeps_ranks_identical_and_averages_gradients(tmp_path):
    import torch.multiprocessing as mp
    path = str(tmp_path / "rank")
    mp.spawn(_ddp_worker, args=(2, _free_port(), path), nprocs=2, join=True)
    r0, r1 = torch.load(f"{path}.0"), torch.load(f"{path}.1")
    ds = _gloo_data()
    single = []
    for half in (slice(0, 2), slice(2, 4)):
        m = _gloo_model()
        _gloo_loss(m, ds.X[half], ds.Y[half]).backward()
        single.append({k: p.grad for k, p in m.named_parameters()})
    for k in single[0]:
        want = (single[0][k] + single[1][k]) / 2
        assert torch.allclose(r0["grads"][k], want, rtol=1e-9, atol=1e-12), k
        assert torch.equal(r0["params"][k], r1["params"][k]), k
