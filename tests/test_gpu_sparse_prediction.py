"""Sparse masked-LM prediction on the H100: ``compact_rows`` against ``torch.nonzero``, ``linear_cross_entropy(sparse=True)``
against the dense fused op and an fp32 torch reference at the BERT-base and ModernBERT-base head shapes (trained bias),
exact zeros on unlabelled rows, determinism, framed outputs, no labelled rows, no host synchronisation, CUDA-graph replay
on a batch with another number of labelled rows, the memory it saves, and tiny encoders trained with
``--sparse_prediction --cuda_graph``."""
import math

import pytest
import torch

from b200ddp.ops import compact_rows, cross_entropy, linear, linear_cross_entropy

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp(min=1e-30))


@pytest.mark.parametrize("T", [1, 77, 1024, 5000, 16384 + 7])
@pytest.mark.parametrize("frac", [0.0, 0.15, 1.0])
def test_compact_rows_equals_nonzero_and_is_repeatable(T, frac):
    V = 1000
    g = torch.Generator(device=dev).manual_seed(T)
    t = torch.randint(0, V, (T,), device=dev, generator=g)
    r = torch.rand(T, device=dev, generator=g)
    t = torch.where(r < frac, t, torch.where(r < 0.5 + frac / 2, torch.full_like(t, -100), t + V))   # ignored or >= V
    index, count, out = compact_rows(t, -100, V)
    valid = (t != -100) & (t >= 0) & (t < V)
    want = torch.cat([torch.nonzero(valid)[:, 0], torch.nonzero(~valid)[:, 0]])
    n = int(valid.sum())
    assert int(count) == n and torch.equal(index.long(), want)
    assert torch.equal(out[:n], t[want[:n]]) and (out[n:] == -100).all()
    again = compact_rows(t, -100, V)
    assert all(torch.equal(a, b) for a, b in zip((index, count, out), again))


def _case(N, V, H, frac, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    h = torch.randn(N, H, device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn(V, H, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    b = (torch.randn(V, device=dev, generator=g) * 0.1).to(torch.bfloat16)
    t = torch.randint(0, V, (N,), device=dev, generator=g)
    t = torch.where(torch.rand(N, device=dev, generator=g) < frac, t, torch.full_like(t, -100))
    return h, w, t, b


def _run(h, w, t, b, sparse, scale=1.0):
    hh, ww, bb = (x.clone().requires_grad_(True) for x in (h, w, b))
    loss = linear_cross_entropy(hh, ww, t, bb, sparse=sparse)
    (loss * scale).backward()
    return loss.detach(), hh.grad, ww.grad, bb.grad


def _reference(h, w, t, b):
    """fp32 autograd over the labelled rows (the others carry no loss and no gradient), the logits rounded to bf16 in the
    forward as the native paths use them."""
    keep = torch.nonzero((t >= 0) & (t < w.shape[0]))[:, 0]
    hh, ww, bb = (x.float().requires_grad_(True) for x in (h, w, b))
    x = hh[keep] @ ww.t() + bb
    x = x + (x.to(torch.bfloat16).float() - x).detach()
    loss = (torch.logsumexp(x, -1) - x.gather(1, t[keep][:, None])[:, 0]).sum() / max(1, keep.numel())
    loss.backward()
    return loss.detach(), hh.grad, ww.grad, bb.grad


@pytest.mark.parametrize("N,V,H", [(8192, 30528, 768), (16384, 50368, 768)])
def test_sparse_op_matches_dense_fused_op_and_fp32_reference(N, V, H):
    h, w, t, b = _case(N, V, H, 0.15)
    loss, dh, dw, db = _run(h, w, t, b, True)
    dl, dhd, dwd, dbd = _run(h, w, t, b, False)
    rl, rh, rw, rb = _reference(h, w, t, b)
    for x in (dh, dw, db):
        assert torch.isfinite(x.float()).all()
    assert abs(float(loss) - float(rl)) <= 1e-3 * abs(float(rl)), (float(loss), float(rl))
    assert abs(float(loss) - float(dl)) <= 1e-3 * abs(float(dl)), (float(loss), float(dl))
    assert (dh[t < 0] == 0).all()
    assert _rel(dh, rh) < 2e-2 and _rel(dh, dhd) < 2e-2, (_rel(dh, rh), _rel(dh, dhd))
    assert _rel(dw, rw) < 1e-2 and _rel(db, rb) < 1e-2, (_rel(dw, rw), _rel(db, rb))
    assert _rel(dw, dwd) < 1e-2 and _rel(db, dbd) < 1e-2, (_rel(dw, dwd), _rel(db, dbd))
    again = _run(h, w, t, b, True)
    assert torch.equal(again[3], db) and torch.equal(again[0], loss) and torch.equal(again[1], dh)


def test_dense_fused_op_trains_the_bias_like_the_unfused_path():
    h, w, t, b = _case(1024, 4096, 128, 0.5, seed=1)
    _, _, _, db = _run(h, w, t, b, False)
    bb = b.clone().requires_grad_(True)
    cross_entropy(linear(h, w, bb), t).backward()
    assert _rel(db, bb.grad) < 1e-2
    loss = linear_cross_entropy(h, w, t, b)                        # a bias without requires_grad stays a constant
    assert not loss.requires_grad


def test_no_labelled_rows_gives_zero_loss_and_gradients():
    h, w, _, b = _case(1000, 4096, 128, 0.0)
    loss, dh, dw, db = _run(h, w, torch.full((1000,), -100, device=dev), b, True)
    assert float(loss) == 0.0 and (dh == 0).all() and (dw == 0).all() and (db == 0).all()


def test_writes_stay_inside_framed_outputs():
    from b200ddp import _ext
    C = _ext.get()
    N, V, H = 384, 2176, 128
    h, w, t, b = _case(N, V, H, 0.3, seed=5)
    index, count, tc = compact_rows(t, -100, V)
    hc = C.gather_rows(h, index, count)
    lse_f = torch.full((N + 64,), 7.0, device=dev)
    rl_f = torch.full((N + 65,), 7.0, device=dev)
    _, lse, rl = C.lm_loss_fwd(hc, w, tc, b, -100, lse_f[32:32 + N], rl_f[32:33 + N], rows=count)
    assert (lse_f[:32] == 7).all() and (lse_f[32 + N:] == 7).all() and (rl_f[:32] == 7).all() and (rl_f[33 + N:] == 7).all()
    n = int(count)
    assert (lse[n:] == 0).all() and (rl[n:N] == 0).all()
    dh_f = torch.full((N + 2, H), 3.0, device=dev, dtype=torch.bfloat16)
    dw_f = torch.full((V + 2, H), 3.0, device=dev, dtype=torch.bfloat16)
    _, _, db = C.lm_loss_bwd(hc, w, tc, b, lse, rl, torch.ones(1, device=dev), -100, 1024, True, True, dh_f[1:N + 1], dw_f[1:V + 1],
                             rows=count, need_dbias=True)
    for f in (dh_f, dw_f):
        assert (f[0] == 3).all() and (f[-1] == 3).all()
    assert (dh_f[1 + n:N + 1] == 0).all()
    _, rh, rw, rb = _reference(h, w, t, b)
    assert _rel(dh_f[1:N + 1], rh[index.long()]) < 2e-2 and _rel(dw_f[1:V + 1], rw) < 1e-2 and _rel(db, rb) < 1e-2


def test_no_host_synchronisation():
    h, w, t, b = _case(4096, 8192, 128, 0.15, seed=6)
    _run(h, w, t, b, True)                                         # first calls: module load, tensor maps
    hh, ww, bb = (x.clone().requires_grad_(True) for x in (h, w, b))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        linear_cross_entropy(hh, ww, t, bb, sparse=True).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert hh.grad is not None and ww.grad is not None and bb.grad is not None


def test_cuda_graph_replay_with_another_labelled_row_count_equals_eager_bitwise():
    N, V, H = 4096, 16384, 256
    h, w, t, b = _case(N, V, H, 0.15, seed=7)
    hh, ww, bb = (x.clone().requires_grad_(True) for x in (h, w, b))
    st = t.clone()

    def step():
        loss = linear_cross_entropy(hh, ww, st, bb, sparse=True)
        return (loss,) + torch.autograd.grad(loss, (hh, ww, bb))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for frac, seed in ((0.4, 8), (0.02, 9)):                       # more labelled rows than at capture, then fewer
        _, _, t2, _ = _case(N, V, H, frac, seed=seed)
        assert int((t2 >= 0).sum()) != int((t >= 0).sum())
        st.copy_(t2)
        graph.replay()
        ref = _run(h, w, t2, b, True)
        for a, e in zip(out, ref):
            assert torch.equal(a, e)


def test_memory_at_modernbert_head_shape_stays_below_one_logits_tensor():
    N, V, H = 16384, 50368, 768
    h, w, t, b = _case(N, V, H, 0.15, seed=10)
    logits_bytes = N * V * 2

    def rise(sparse):
        hh, ww, bb = (x.clone().requires_grad_(True) for x in (h, w, b))
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        linear_cross_entropy(hh, ww, t, bb, sparse=sparse).backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    sparse, dense = rise(True), rise(False)
    print(f"\n[sparse prediction memory] {N} x {V} x {H}: fwd+bwd rise sparse {sparse / 1e9:.2f} GB, dense fused "
          f"{dense / 1e9:.2f} GB, logits {logits_bytes / 1e9:.2f} GB")
    assert sparse < logits_bytes, (sparse, logits_bytes)


# ---- tiny encoders through the trainer: --sparse_prediction --cuda_graph (+ --pack, + --min_seq_len, + --fp8) -------------
def _tiny(family, sparse, **kw):
    if family == "bert":
        from b200ddp.models.bert import BertConfig, BertForMaskedLM
        return BertForMaskedLM(BertConfig(vocab_size=500, hidden=128, layers=2, heads=2, intermediate=256, max_position=256,
                                          pad_vocab_to=64, sparse_prediction=sparse, **kw))
    from b200ddp.models.modernbert import ModernBertConfig, ModernBertForMaskedLM
    return ModernBertForMaskedLM(ModernBertConfig(vocab_size=512, hidden=128, layers=4, heads=2, intermediate=192, max_position=256,
                                                  local_attention=32, sparse_prediction=sparse, **kw))


_MODEL = {"bert": "bert-base", "modernbert": "modernbert-base"}


@pytest.mark.parametrize("family,extra", [("bert", []), ("modernbert", []), ("bert", ["--pack"]), ("modernbert", ["--pack"]),
                                          ("bert", ["--min_seq_len"]), ("modernbert", ["--min_seq_len", "--fp8"]),
                                          ("bert", ["--pack", "--fp8"])])
def test_tiny_encoders_train_with_sparse_prediction_and_cuda_graph(tmp_path, family, extra):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.ops import CrossEntropyLoss
    from b200ddp.utils import to_mixed_bf16
    flags = ["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", _MODEL[family], "--fp16", "--cuda_graph",
             "--sparse_prediction", "--seq_len", "256", "--optimizer", "adamw", "--lr", "3e-3", "--max_steps", "40",
             "--per_gpu_train_batch_size", "8", "--warmup_steps", "2", "--save_steps", "0", "--logging_steps", "10"]
    flags += ["--min_seq_len", "32"] if ("--pack" in extra or "--min_seq_len" in extra) else []
    flags += [f for f in extra if f in ("--pack", "--fp8")]
    args = cli.build_parser().parse_args(flags)
    cli.setup(args)
    ds = build_dataset(args)
    cls = getattr(ds, "cls_token_id", None)
    is_cls = ds.X == cls if cls is not None else torch.zeros_like(ds.X, dtype=torch.bool)
    ds.X = torch.where(is_cls, torch.ones_like(ds.X), torch.where(ds.X > 0, ds.X % 16 + 2, ds.X))   # a small alphabet to learn
    ds.Y = torch.where(ds.Y > 0, ds.Y % 16 + 2, ds.Y)
    kw = dict(fp8="--fp8" in extra)
    if "--pack" in extra:
        ds.cls_token_id = 1
        kw.update(pad_token_id=0, cls_token_id=1)
    elif "--min_seq_len" in extra:
        kw.update(pad_token_id=0)
    torch.manual_seed(0)
    model = _tiny(family, True, **kw)
    plain = _tiny(family, False, **kw)
    plain.load_state_dict(model.state_dict())
    plain = to_mixed_bf16(plain.to(dev))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    x, y = ds.X[:8].to(dev), ds.Y[:8].to(dev)
    with torch.no_grad():                                          # first-step loss: sparse equals unfused
        ls = float(trainer.criterion(trainer.model(x), y))
        lp = float(CrossEntropyLoss()(plain(x), y))
    assert abs(ls - lp) < 2e-3 * abs(lp), (ls, lp)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert trainer.step_fn.graph is not None
    assert math.isfinite(after) and after < before - 0.1, (before, after)
