"""Packed-document attention (csrc/attention.cu, segment mode) on the GPU: accuracy against fp64 beside SDPA's own bf16
error with the block-diagonal mask, isolation between documents, padding rows, agreement with the key-padding kernels,
determinism, bounds, CUDA-graph replay with a new packing, input checks, and packed BERT training."""
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.ops import functional as Fn

pytestmark = pytest.mark.gpu

HEADS, HD = 12, 64
W = HEADS * HD
CLS, PAD = 101, 0


def dev():
    return torch.device("cuda", 0)


def C():
    from b200ddp import _ext
    return _ext.get()


def _bounds(layout, S):
    """layout: one list of document lengths per row (the rest of a row is padding) -> int32 [B, S, 2] on the GPU."""
    b = torch.zeros(len(layout), S, 2, dtype=torch.int32)
    for r, docs in enumerate(layout):
        at = 0
        for n in docs:
            b[r, at:at + n, 0], b[r, at:at + n, 1] = at, at + n
            at += n
        assert at <= S
    return b.to(dev())


def _inputs(B, S, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B * S, 3 * W, device=dev(), generator=g).to(torch.bfloat16)
    dout = torch.randn(B * S, W, device=dev(), generator=g).to(torch.bfloat16)
    return qkv, dout


def _split(t, B, S):
    return [x.reshape(B, S, HEADS, HD).transpose(1, 2) for x in t.reshape(B, S, 3 * W).split(W, dim=-1)]


def _mask(bounds, S):
    j = torch.arange(S, device=dev())
    return ((j >= bounds[..., :1].long()) & (j < bounds[..., 1:].long()))[:, None]      # [B, 1, S, S]


def _reference(qkv, dout, bounds, B, S):
    """fp64 o, lse, dqkv; rows that see no key give zeros and lse = -inf."""
    x = qkv.double().requires_grad_(True)
    q, k, v = _split(x, B, S)
    keep = _mask(bounds, S)
    s = ((q @ k.transpose(-1, -2)) / 8.0).masked_fill(~keep, -math.inf)
    lse = torch.logsumexp(s, dim=-1)
    p = torch.softmax(s.masked_fill(~keep, torch.finfo(torch.float64).min), dim=-1) * keep
    o = (p @ v).transpose(1, 2).reshape(B * S, -1)
    o.backward(dout.double())
    return o.detach(), lse.detach(), x.grad


def _sdpa(qkv, dout, bounds, B, S):
    """SDPA in bf16 with the dense block-diagonal boolean mask.  A row that sees no key would be NaN there, so it sees
    its own key instead and its output is zeroed (as its reference is): its dO is then zero, which adds nothing to any
    gradient."""
    x = qkv.detach().clone().requires_grad_(True)
    q, k, v = _split(x, B, S)
    live = bounds[..., 1] > bounds[..., 0]
    mask = _mask(bounds, S) | (~live[:, None, :, None] & torch.eye(S, dtype=torch.bool, device=dev()))
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B * S, -1)
    o = torch.where(live.reshape(B * S, 1), o, torch.zeros_like(o))
    o.backward(dout)
    return o.detach(), x.grad


def _rms(t):
    return float(t.double().pow(2).mean().sqrt())


def _random_packing(S, seed, lo=1):
    g = torch.Generator().manual_seed(seed)
    docs, at = [], 0
    while True:
        n = int(torch.randint(lo, S + 1, (1,), generator=g))
        if at + n > S:
            return docs
        docs.append(n)
        at += n


LAYOUTS = {                                                     # S -> document lengths per row
    "one_doc_per_row": lambda S: [[S], [S // 2 + 3], [S - 1]],
    "tile_edges": lambda S: ([[1, 63, 64, 65, 63], [127, 129], [128, 128]] if S == 256 else
                             [[1, 63, 64, 65, 127, 128, 64], [129, 127, 1, 128, 127], [129, 129, 129, 125]]),
    "many_one_token_docs": lambda S: [[1] * S, [1] * (S // 2) + [S // 4]],
    "docs_and_tail_padding": lambda S: [[100, 5, 40], _random_packing(S, 3, 16), [S // 2]],
    "all_padding_row": lambda S: [[], [70, 30], [S]],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("S", [256, 512])
def test_packed_attention_is_as_accurate_as_sdpa(layout, S):
    docs = LAYOUTS[layout](S)
    B = len(docs)
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(B, S, seed=S + len(layout))
    o, lse = C().packed_attention_fwd(qkv, bounds, HEADS)
    dqkv = C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    o_ref, lse_ref, d_ref = _reference(qkv, dout, bounds, B, S)
    o_lib, d_lib = _sdpa(qkv, dout, bounds, B, S)
    assert torch.isfinite(o.float()).all() and torch.isfinite(dqkv.float()).all()
    live = torch.isfinite(lse_ref)
    assert torch.equal(torch.isfinite(lse), live)
    assert torch.allclose(lse.double()[live], lse_ref[live], rtol=0, atol=2e-3), float((lse.double() - lse_ref)[live].abs().max())
    for name, ours, lib, ref in (("o", o, o_lib, o_ref), ("dq", dqkv[:, :W], d_lib[:, :W], d_ref[:, :W]),
                                 ("dk", dqkv[:, W:2 * W], d_lib[:, W:2 * W], d_ref[:, W:2 * W]),
                                 ("dv", dqkv[:, 2 * W:], d_lib[:, 2 * W:], d_ref[:, 2 * W:])):
        err, lib_err = _rms(ours.double() - ref), _rms(lib.double() - ref)
        assert err <= 1.5 * lib_err + 2e-3 * _rms(ref), (name, err, lib_err, _rms(ref))


def test_perturbing_one_document_leaves_the_others_bit_identical():
    S = 512
    docs = [[100, 130, 29, 200], [64, 64, 300]]
    B = len(docs)
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(B, S, seed=21)
    o, lse = C().packed_attention_fwd(qkv, bounds, HEADS)
    d = C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    qkv2 = qkv.clone()
    qkv2[130:259] = torch.randn_like(qkv2[130:259], dtype=torch.float32).to(torch.bfloat16)   # row 0, doc 2 + doc 3's first
    dout2 = dout.clone()
    dout2[130:259] *= -3
    o2, lse2 = C().packed_attention_fwd(qkv2, bounds, HEADS)
    d2 = C().packed_attention_bwd(dout2, qkv2, o2, lse2, bounds, HEADS)
    keep = torch.ones(B * S, dtype=torch.bool, device=dev())
    keep[100:259] = False                                       # the touched documents of row 0: [100, 230), [230, 259)
    assert torch.equal(o[keep], o2[keep]) and torch.equal(d[keep], d2[keep])
    assert torch.equal(lse.view(B, HEADS, S)[1], lse2.view(B, HEADS, S)[1])
    assert not torch.equal(o[130:259], o2[130:259])


def test_padding_rows_get_zeros_minus_inf_and_zero_gradients():
    S = 256
    docs = [[], [1, 40], [256]]
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(3, S, seed=5)
    o, lse = C().packed_attention_fwd(qkv, bounds, HEADS)
    d = C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    assert torch.isfinite(o.float()).all() and torch.isfinite(d.float()).all() and not torch.isnan(lse).any()
    o3, d3, lse3 = o.view(3, S, W), d.view(3, S, 3 * W), lse.view(3, HEADS, S)
    for r, fill in ((0, 0), (1, 41)):
        assert (o3[r, fill:] == 0).all() and (d3[r, fill:] == 0).all(), r
        assert torch.isinf(lse3[r, :, fill:]).all() and (lse3[r, :, fill:] < 0).all(), r
    assert torch.isfinite(lse3[1, :, :41]).all() and torch.isfinite(lse3[2]).all()
    assert d3[1, :41].abs().sum() > 0


def test_single_document_bounds_match_the_key_padding_kernels():
    """bounds (0, len) on every row, dO zero at rows >= len: o, lse and dqkv on rows < len are bit-identical."""
    S = 512
    lens = [512, 300, 129, 1, 128, 64]
    B = len(lens)
    qkv, dout = _inputs(B, S, seed=8)
    lt = torch.tensor(lens, dtype=torch.int32, device=dev())
    bounds = torch.zeros(B, S, 2, dtype=torch.int32, device=dev())
    bounds[..., 1] = lt[:, None]
    inside = (torch.arange(S, device=dev())[None, :] < lt[:, None]).reshape(B * S)
    dout = dout * inside[:, None]
    o_k, lse_k = C().attention_fwd(qkv, lt, HEADS)
    d_k = C().attention_bwd(dout, qkv, o_k, lse_k, lt, HEADS)
    o_p, lse_p = C().packed_attention_fwd(qkv, bounds, HEADS)
    d_p = C().packed_attention_bwd(dout, qkv, o_p, lse_p, bounds, HEADS)
    assert torch.equal(o_p[inside], o_k[inside]) and torch.equal(d_p[inside], d_k[inside])
    lin = inside.view(B, 1, S).expand(B, HEADS, S)
    assert torch.equal(lse_p[lin], lse_k[lin])


def test_packed_attention_is_deterministic():
    S = 512
    docs = [_random_packing(S, s) for s in range(8)]
    bounds = _bounds(docs, S)
    qkv, dout = _inputs(8, S, seed=9)
    runs = []
    for _ in range(2):
        o, lse = C().packed_attention_fwd(qkv, bounds, HEADS)
        runs.append((o, lse, C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_packed_attention_stays_in_bounds():
    B, S = 3, 256
    bounds = _bounds([[], [100, 56], [256]], S)
    # out-of-range bounds are clamped on the device: they may give any values, but never touch memory outside
    bounds[1, 200:, 0], bounds[1, 200:, 1] = -50, 10 ** 6
    bounds[2, :5, 0], bounds[2, :5, 1] = 300, 200
    qkv, dout = _inputs(B, S, seed=2)
    sentinel, pad = -12345.0, 64
    o_buf = torch.full((B * S * W + 2 * pad,), sentinel, device=dev(), dtype=torch.bfloat16)
    lse_buf = torch.full((B * HEADS * S + 2 * pad,), sentinel, device=dev())
    d_buf = torch.full((B * S * 3 * W + 2 * pad,), sentinel, device=dev(), dtype=torch.bfloat16)
    o = o_buf[pad:pad + B * S * W].view(B * S, W)
    lse = lse_buf[pad:pad + B * HEADS * S].view(B, HEADS, S)
    dqkv = d_buf[pad:pad + B * S * 3 * W].view(B * S, 3 * W)
    C().packed_attention_fwd(qkv, bounds, HEADS, o, lse)
    C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS, dqkv)
    o_ref, lse_ref = C().packed_attention_fwd(qkv, bounds, HEADS)
    assert torch.equal(o, o_ref) and torch.equal(lse, lse_ref)
    assert torch.equal(dqkv, C().packed_attention_bwd(dout, qkv, o_ref, lse_ref, bounds, HEADS))
    for buf in (o_buf, lse_buf, d_buf):
        assert (buf[:pad] == sentinel).all() and (buf[-pad:] == sentinel).all()


def test_graph_replay_with_a_new_packing_matches_eager():
    B, S = 4, 512
    bounds = _bounds([_random_packing(S, s, 16) for s in range(B)], S)
    qkv, dout = _inputs(B, S, seed=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                  # warm-up: tensor maps, kernel attributes
        o, lse = C().packed_attention_fwd(qkv, bounds, HEADS)
        C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o_g, lse_g = C().packed_attention_fwd(qkv, bounds, HEADS)
        d_g = C().packed_attention_bwd(dout, qkv, o_g, lse_g, bounds, HEADS)
    for layout in ([[512], [1] * 100, [], [300, 200]], [_random_packing(S, 40 + s, 8) for s in range(B)]):
        bounds.copy_(_bounds(layout, S))
        graph.replay()
        o, lse = C().packed_attention_fwd(qkv, bounds, HEADS)
        d = C().packed_attention_bwd(dout, qkv, o, lse, bounds, HEADS)
        torch.cuda.synchronize()
        assert torch.equal(o_g, o) and torch.equal(lse_g, lse) and torch.equal(d_g, d), layout


def test_packed_attention_rejects_unsupported_input():
    good = torch.randn(2, 128, 3 * 128, device=dev()).to(torch.bfloat16)
    bounds = _bounds([[100], [28, 100]], 128)
    Fn.packed_attention(good, bounds, 2)                        # head dim 64, S = 128: accepted
    with pytest.raises(ValueError):
        Fn.packed_attention(good.half(), bounds, 2)             # not bf16
    with pytest.raises(ValueError):
        Fn.packed_attention(good, bounds, 4)                    # head dim 32
    with pytest.raises(ValueError):
        Fn.packed_attention(torch.randn(2, 192, 3 * 128, device=dev()).to(torch.bfloat16), _bounds([[1], [1]], 192), 2)
    with pytest.raises(ValueError):
        Fn.packed_attention(torch.randn(2, 128, 6 * 128, device=dev()).to(torch.bfloat16)[..., :3 * 128], bounds, 2)
    with pytest.raises(ValueError):
        Fn.packed_attention(good, bounds[:, :64], 2)            # bounds not [B, S, 2]
    with pytest.raises(ValueError):
        Fn.packed_attention(good, bounds.float(), 2)            # bounds not integer


def test_packed_op_matches_its_cpu_body():
    B, S, H = 2, 128, 2
    torch.manual_seed(0)
    qkv = torch.randn(B, S, 3 * H * HD).to(torch.bfloat16)
    bounds = _bounds([[5, 60, 63], [30]], S).cpu()
    dy = torch.randn(B, S, H * HD).to(torch.bfloat16)
    xc = qkv.clone().requires_grad_(True)
    Fn.packed_attention(xc, bounds, H).backward(dy)
    yc = Fn.packed_attention_reference(qkv, bounds, H)
    xg = qkv.to(dev()).requires_grad_(True)
    yg = Fn.packed_attention(xg, bounds.to(dev()), H)
    yg.backward(dy.to(dev()))
    assert torch.allclose(yg.float().cpu(), yc.float(), rtol=2e-2, atol=2e-2)
    assert torch.allclose(xg.grad.float().cpu(), xc.grad.float(), rtol=5e-2, atol=5e-2)


# ---- BERT --------------------------------------------------------------------------------------------------------------
def _tiny_cfg(**kw):
    from b200ddp.models.bert import BertConfig
    return BertConfig(vocab_size=1000, hidden=128, layers=2, heads=2, intermediate=256, max_position=128, pad_vocab_to=64, **kw)


def _packed_batch(rows, S, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 1000, (len(rows), S), generator=g)
    ids[ids == CLS] = 7
    labels = torch.where(torch.rand(len(rows), S, generator=g) < 0.3, torch.randint(0, 1000, ids.shape, generator=g),
                         torch.full(ids.shape, -100))
    for r, docs in enumerate(rows):
        at = 0
        for n in docs:
            ids[r, at] = CLS
            at += n
        ids[r, at:], labels[r, at:] = PAD, -100
    return ids, labels


def test_packed_bert_tiny_gpu_matches_cpu_reference():
    """bf16 GPU model (native packed attention) against the fp32 CPU model with the same weights."""
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(7)
    ref = BertForMaskedLM(_tiny_cfg(pad_token_id=PAD, cls_token_id=CLS))
    gpu = BertForMaskedLM(_tiny_cfg(pad_token_id=PAD, cls_token_id=CLS))
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(dev(), torch.bfloat16)
    ids, labels = _packed_batch([[40, 1, 57, 30], [128], [64, 63], []], 128, seed=1)
    lr = cross_entropy(ref(ids), labels)
    lr.backward()
    lg = cross_entropy(gpu(ids.to(dev())), labels.to(dev()))
    lg.backward()
    lg, lr = float(lg.detach()), float(lr.detach())
    assert abs(lg - lr) < 5e-2 * max(1.0, abs(lr))
    for (n, p), q in zip(gpu.named_parameters(), ref.parameters()):
        if float(q.grad.norm()) < 1e-4:
            assert float(p.grad.float().norm()) < 5e-2, n
            continue
        rel = float((p.grad.float().cpu() - q.grad).norm() / (q.grad.norm() + 1e-8))
        assert rel < 0.2, (n, rel)


def test_packed_bert_step_has_no_host_synchronisation():
    from b200ddp.models.bert import BertForMaskedLM
    from b200ddp.ops import cross_entropy
    torch.manual_seed(1)
    model = BertForMaskedLM(_tiny_cfg(pad_token_id=PAD, cls_token_id=CLS)).to(dev(), torch.bfloat16)
    ids, labels = _packed_batch([[100, 28], [1, 1, 126], [50], [128]], 128, seed=2)
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
    assert math.isfinite(float(loss))


@pytest.mark.parametrize("fp8", [False, True])
def test_packed_bert_base_graph_training_lowers_the_loss(tmp_path, fp8):
    """What `python ddp.py --model bert-base --fp16 --optimizer adamw --cuda_graph --max_steps 30 --seq_len 128
    --min_seq_len 32 --pack [--fp8]` runs."""
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    argv = ["--model", "bert-base", "--fp16", "--optimizer", "adamw", "--cuda_graph", "--max_steps", "30", "--seq_len", "128",
            "--min_seq_len", "32", "--pack", "--per_gpu_train_batch_size", "16", "--lr", "5e-4", "--warmup_steps", "5",
            "--weight_decay", "0.01", "--save_steps", "0", "--logging_steps", "10", "--no_tensorboard",
            "--output_dir", str(tmp_path / "out")] + (["--fp8"] if fp8 else [])
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": PAD, "cls_token_id": CLS, **({"fp8": True} if fp8 else {})}
    trainer = Trainer(args, build_model("bert-base", **kwargs), cli.log)
    assert trainer.dataset.doc_lengths is not None and max(len(r) for r in trainer.dataset.doc_lengths) > 1
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.05, (before, after)
