"""Causal document attention, tanh GELU, GPT-2 and causal-LM data on the CPU: the reference against a brute-force loop,
``document_bounds`` without a document id, ``gelu_tanh`` in every linear body, a tiny GPT-2 against Hugging Face's,
the causal labels (and unchanged MLM rows), and the CLI / trainer checks."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn


def _brute_force(qkv, bounds, heads):
    """Row by row: query i softmax-attends to keys j with start_i <= j <= i and j < end_i; no such key gives zeros."""
    B, S, Wd = qkv.shape
    hidden = Wd // 3
    hd = hidden // heads
    q, k, v = qkv.double().split(hidden, dim=-1)
    out = torch.zeros(B, S, hidden, dtype=torch.float64)
    for b in range(B):
        for i in range(S):
            s0 = min(max(int(bounds[b, i, 0]), 0), S)
            e0 = min(max(int(bounds[b, i, 1]), s0), S)
            keys = [j for j in range(s0, e0) if j <= i]
            if not keys:
                continue
            for h in range(heads):
                c = slice(h * hd, (h + 1) * hd)
                sc = torch.stack([q[b, i, c] @ k[b, j, c] for j in keys]) / math.sqrt(hd)
                p = torch.softmax(sc, 0)
                out[b, i, c] = sum(p[n] * v[b, j, c] for n, j in enumerate(keys))
    return out


def _bounds(layout, S):
    b = torch.zeros(len(layout), S, 2, dtype=torch.int32)
    for r, docs in enumerate(layout):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
    return b


def test_causal_reference_matches_a_brute_force_loop():
    torch.manual_seed(0)
    S, heads = 24, 2
    bounds = _bounds([[5, 1, 10, 8], [24], [7], []], S)
    bounds[2, 3, 0] = 5                                        # malformed: start after the row itself, sees nothing
    qkv = torch.randn(4, S, 3 * 2 * 8, dtype=torch.float64)
    ref = Fn.causal_attention_reference(qkv, bounds, heads)
    assert torch.allclose(ref, _brute_force(qkv, bounds, heads), atol=1e-12)
    assert (ref[3] == 0).all() and (ref[2, 7:] == 0).all() and (ref[2, 3] == 0).all()


def test_causal_op_gradient_matches_the_reference_and_never_looks_ahead():
    torch.manual_seed(1)
    S, heads = 32, 2
    bounds = _bounds([[10, 22], [30]], S)
    x = torch.randn(2, S, 3 * 128, requires_grad=True)
    y = Fn.causal_attention(x, bounds, heads)
    (g,) = torch.autograd.grad(y[:, 15].sum(), x)
    assert (g[:, 16:] == 0).all() and (g[0, :10] == 0).all()  # later tokens and other documents get no gradient
    xr = x.detach().requires_grad_(True)
    (gr,) = torch.autograd.grad(Fn.causal_attention_reference(xr, bounds, heads)[:, 15].sum(), xr)
    assert torch.allclose(g, gr)


def test_document_bounds_without_a_document_id_gives_one_document_per_row():
    ids = torch.tensor([[5, 50256, 7, 0, 0], [1, 2, 3, 4, 5], [0, 0, 0, 0, 0]])
    bounds, pos = Fn.document_bounds(ids, None, 0)
    expect = torch.tensor([[[0, 3]] * 3 + [[0, 0]] * 2, [[0, 5]] * 5, [[0, 0]] * 5], dtype=torch.int32)
    assert torch.equal(bounds, expect)
    assert torch.equal(pos, torch.tensor([[0, 1, 2, 0, 0], [0, 1, 2, 3, 4], [0] * 5]))
    b2, _ = Fn.document_bounds(ids, None, None)
    assert (b2[..., 0] == 0).all() and (b2[..., 1] == 5).all()
    # with an id, a document still starts there (unchanged behaviour)
    b3, p3 = Fn.document_bounds(ids, 50256, 0)
    assert b3[0, :, 0].tolist() == [0, 1, 1, 0, 0] and p3[0].tolist() == [0, 0, 1, 0, 0]


@pytest.mark.parametrize("fp8", [False, True])
def test_gelu_tanh_matches_torch(fp8):
    torch.manual_seed(2)
    x = torch.randn(16, 32)
    w = torch.randn(48, 32) * 0.2
    b = torch.randn(48) * 0.1
    xa, wa, ba = (t.clone().requires_grad_(True) for t in (x, w, b))
    y = Fn.linear(xa, wa, ba, "gelu_tanh", fp8=fp8)
    if fp8:                                                    # the emulated recipe quantises x and W first
        x_in, w_in = Fn._fp8_round_trip(x, "e4m3"), Fn._fp8_round_trip(w, "e4m3")
    else:
        x_in, w_in = x, w
    pre = (x_in @ w_in.t() + b).requires_grad_(True)
    ref = F.gelu(pre, approximate="tanh")
    assert torch.allclose(y, ref, atol=1e-5)
    dy = torch.randn_like(ref)
    y.backward(dy)
    ref.backward(dy)
    if not fp8:
        (dx,) = torch.autograd.grad(F.gelu(F.linear(x.requires_grad_(True), w, b), approximate="tanh"), x, dy)
        assert torch.allclose(xa.grad, dx, atol=1e-5)
    assert torch.allclose(Fn._gelu_tanh_grad(pre.detach()) * dy, pre.grad, atol=1e-5)
    # "gelu" stays the erf form
    assert torch.allclose(Fn.linear(x, w, b, "gelu"), F.gelu(F.linear(x, w, b)))


def _tiny_hf(seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.GPT2Config(vocab_size=1000, n_positions=128, n_embd=128, n_layer=2, n_head=2)
    return transformers.GPT2LMHeadModel(cfg).eval()


def _tiny(**kw):
    from b200ddp.models.gpt import GPTConfig, GPTLMHeadModel
    return GPTLMHeadModel(GPTConfig(vocab_size=1000, max_position=128, hidden=128, layers=2, heads=2, intermediate=512, **kw))


def test_tiny_gpt2_matches_hugging_face_logits_and_loss():
    hf = _tiny_hf()
    ours = _tiny()
    ours.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, 1000, (2, 40), generator=torch.Generator().manual_seed(3))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    with torch.no_grad():
        ref = hf(ids, labels=ids)
        logits = ours(ids)
    assert logits.shape == (2, 40, 1024)
    assert torch.allclose(logits[..., :1000], ref.logits, atol=1e-4), float((logits[..., :1000] - ref.logits).abs().max())
    assert (logits[..., 1000:] < -1e3).all()                  # padded vocabulary rows never win
    loss = Fn.cross_entropy(logits, labels)
    assert abs(float(loss) - float(ref.loss)) < 1e-4
    assert abs(float(Fn.cross_entropy(logits, labels)) - float(Fn.cross_entropy(logits[..., :1000], labels))) < 1e-5


def test_packed_gpt2_row_matches_each_document_run_alone_through_hugging_face():
    BOS = 999
    hf = _tiny_hf(seed=4)
    ours = _tiny(pad_token_id=0, bos_token_id=BOS)
    ours.load_hf_state_dict(hf.state_dict())
    g = torch.Generator().manual_seed(5)
    docs = [torch.cat([torch.tensor([BOS]), torch.randint(1, BOS, (n - 1,), generator=g)]) for n in (17, 1, 30)]
    row = torch.cat(docs + [torch.zeros(64 - 48, dtype=torch.long)])[None]
    with torch.no_grad():
        packed = ours(row)[0, :, :1000]
        at = 0
        for d in docs:
            alone = hf(d[None]).logits[0]
            assert torch.allclose(packed[at:at + len(d)], alone, atol=1e-4), float((packed[at:at + len(d)] - alone).abs().max())
            at += len(d)
    # right padding alone (pad id, no BOS id): the real tokens match HF on the unpadded row
    padded = _tiny(pad_token_id=0)
    padded.load_hf_state_dict(hf.state_dict())
    ids = torch.cat([docs[2], torch.zeros(10, dtype=torch.long)])[None]
    with torch.no_grad():
        assert torch.allclose(padded(ids)[0, :30, :1000], hf(docs[2][None]).logits[0], atol=1e-4)


def test_gpt2_registry_defaults_and_fp8_linears():
    from b200ddp.models import GPTConfig, build_model
    c = GPTConfig()
    assert (c.vocab_size, c.padded_vocab, c.max_position, c.hidden, c.layers, c.heads, c.intermediate, c.eps) == \
        (50257, 50304, 1024, 768, 12, 12, 3072, 1e-5)
    m = build_model("gpt2", fp8=True)
    fp8 = [n for n, x in m.named_modules() if getattr(x, "fp8", False) is True]
    assert len(fp8) == 48 and all(n.split(".")[-1] in ("qkv", "attn_out", "ffn_in", "ffn_out") for n in fp8)
    assert "vocab_bias" not in m.state_dict()
    assert m.transformer.h[0].ffn_in.activation == "gelu_tanh"


def test_causal_token_rows():
    from b200ddp.data import SyntheticTokens
    fixed = SyntheticTokens(samples=4, seq_len=32, vocab=50257, causal=True)
    assert torch.equal(fixed.Y[:, :-1], fixed.X[:, 1:]) and (fixed.Y[:, -1] == -100).all()
    assert fixed.lengths is None and fixed.pad_token_id is None and (fixed.X > 0).all()
    padded = SyntheticTokens(samples=16, seq_len=32, vocab=50257, min_len=4, causal=True)
    for x, y, n in zip(padded.X, padded.Y, padded.lengths.tolist()):
        assert (x[:n] > 0).all() and (x[n:] == 0).all()
        assert torch.equal(y[:n - 1], x[1:n]) and (y[n - 1:] == -100).all()
    packed = SyntheticTokens(samples=40, seq_len=64, vocab=50257, min_len=4, pack=True, causal=True)
    assert packed.bos_token_id == 50256 and packed.cls_token_id is None and packed.pad_token_id == 0
    for x, y, docs in zip(packed.X, packed.Y, packed.doc_lengths):
        at = 0
        for n in docs:
            assert x[at] == 50256 and (x[at + 1:at + n] != 50256).all() and (x[at:at + n] > 0).all()
            assert torch.equal(y[at:at + n - 1], x[at + 1:at + n]) and y[at + n - 1] == -100
            at += n
        assert (x[at:] == 0).all() and (y[at:] == -100).all()


def test_mlm_rows_are_unchanged_by_the_causal_option():
    from b200ddp.data import SyntheticTokens
    for kw in ({}, {"min_len": 100}, {"min_len": 100, "pack": True}):
        a = SyntheticTokens(samples=64, seq_len=128, **kw)
        b = SyntheticTokens(samples=64, seq_len=128, causal=False, **kw)
        assert torch.equal(a.X, b.X) and torch.equal(a.Y, b.Y) and b.bos_token_id is None


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_gpt2_cli_accepts_its_flags_and_rejects_long_rows(tmp_path):
    from b200ddp.engine import cli
    args = _args(tmp_path, "--model", "gpt2", "--no_cuda", "--seq_len", "256", "--min_seq_len", "32", "--pack")
    cli.setup(args)
    with pytest.raises(ValueError, match="1024"):
        cli.setup(_args(tmp_path, "--model", "gpt2", "--no_cuda", "--seq_len", "2048"))
    with pytest.raises(ValueError, match="CUDA device"):                 # --fp8 now accepts gpt2, still needs a GPU
        cli.setup(_args(tmp_path, "--model", "gpt2", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="gpt2"):
        cli.setup(_args(tmp_path, "--model", "resnet50", "--no_cuda", "--min_seq_len", "32", "--seq_len", "64"))


def test_trainer_rejects_a_gpt_model_that_ignores_the_datasets_documents():
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine.trainer import Trainer, build_dataset
    ds = build_dataset(types.SimpleNamespace(model="gpt2", dataset_size=50, seq_len=64, min_seq_len=8, pack=True))
    assert ds.bos_token_id == SyntheticTokens.BOS_ID
    trainer = Trainer.__new__(Trainer)
    trainer.dataset = ds
    trainer.log = types.SimpleNamespace(info=lambda *a, **k: None)
    for kw in ({}, {"pad_token_id": 0}, {"pad_token_id": 0, "bos_token_id": 7}):
        with pytest.raises(ValueError):
            trainer._check_padding(_tiny(**kw))
    trainer._check_padding(_tiny(pad_token_id=0, bos_token_id=SyntheticTokens.BOS_ID))
    padded = build_dataset(types.SimpleNamespace(model="gpt2", dataset_size=50, seq_len=64, min_seq_len=8, pack=False))
    trainer.dataset = padded
    with pytest.raises(ValueError):
        trainer._check_padding(_tiny())
    trainer._check_padding(_tiny(pad_token_id=0))
