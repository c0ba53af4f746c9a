"""BART on the CPU: the state dict and parameter counts against ``transformers.BartForConditionalGeneration``, logits,
loss and gradients against it on fixed, right-padded and packed rows, the cross-attention op and ``cross_bounds``, the
synthetic denoising data, the CLI, short training runs and the gradient across two gloo ranks."""
import math
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from b200ddp.data import SyntheticDenoising
from b200ddp.models import MODEL_REGISTRY
from b200ddp.models.bart import BartConfig, BartForConditionalGeneration
from b200ddp.ops import cross_attention, cross_attention_reference, cross_bounds, document_bounds

transformers = pytest.importorskip("transformers")

V = 100
START = 3


def _hf_config(**kw):
    return transformers.BartConfig(vocab_size=V, d_model=128, encoder_layers=2, decoder_layers=2, encoder_attention_heads=2,
                                   decoder_attention_heads=2, encoder_ffn_dim=256, decoder_ffn_dim=256, max_position_embeddings=64,
                                   dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, pad_token_id=0, bos_token_id=START,
                                   eos_token_id=6, decoder_start_token_id=2, forced_eos_token_id=None, **kw)


def _pair(pad_token_id=0, bos_token_id=None, seed=0):
    """(transformers' tiny model in eval mode, ours loaded from its state dict), fp64."""
    torch.manual_seed(seed)
    hf = transformers.BartForConditionalGeneration(_hf_config()).double().eval()
    ours = BartForConditionalGeneration(BartConfig(vocab_size=V, hidden=128, encoder_layers=2, decoder_layers=2, heads=2, intermediate=256,
                                                   max_position=64, pad_token_id=pad_token_id, bos_token_id=bos_token_id)).double()
    ours.load_hf_state_dict(hf.state_dict())
    return hf, ours


def _rows(src_lens, tgt_lens, Sk, Sq, seed=1):
    g = torch.Generator().manual_seed(seed)
    B = len(src_lens)
    src = torch.randint(7, V, (B, Sk), generator=g)
    lab = torch.randint(7, V, (B, Sq), generator=g)
    for b in range(B):
        src[b, 0] = lab[b, 0] = START
        src[b, src_lens[b]:] = 0
        lab[b, tgt_lens[b]:] = -100
    return src, lab


def _grads(model):
    return {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}


def _hf_grad(hf, name):
    """transformers' gradient of our parameter `name`, fused and padded as ours is."""
    g = lambda k: dict(hf.named_parameters())[k].grad
    if name == "model.shared.weight":
        return g("model.shared.weight")
    side, rest = name.split(".")[1], name.split(".", 2)[2]
    if rest.startswith("layers."):
        i, field = rest.split(".")[1], rest.split(".", 2)[2]
        p = f"model.{side}.layers.{i}."
        mod, wb = field.rsplit(".", 1)
        fused = {"qkv": [f"self_attn.{x}_proj" for x in "qkv"], "cross_kv": [f"encoder_attn.{x}_proj" for x in "kv"]}
        renamed = {"out_proj": "self_attn.out_proj", "q_proj": "encoder_attn.q_proj", "cross_out_proj": "encoder_attn.out_proj"}
        if mod in fused:
            return torch.cat([g(p + m + "." + wb) for m in fused[mod]])
        return g(p + renamed.get(mod, mod) + "." + wb)
    return g(f"model.{side}.{rest}")


def test_parameter_counts_match_transformers_plus_padded_vocabulary():
    for name, hf_count, hidden in (("bart-base", 139_420_416, 768), ("bart-large", 406_291_456, 1024)):
        with torch.device("meta"):
            m = MODEL_REGISTRY[name].build()
        assert sum(p.numel() for p in m.parameters()) == hf_count + (50304 - 50265) * hidden, name
        assert m.config.padded_vocab == 50304 and "final_logits_bias" in m.state_dict()


def test_load_hf_state_dict_is_strict():
    hf, ours = _pair()
    sd = hf.state_dict()
    extra = dict(sd, **{"model.encoder.extra.weight": torch.zeros(1)})
    with pytest.raises(KeyError):
        ours.load_hf_state_dict(extra)
    missing = {k: v for k, v in sd.items() if k != "model.decoder.layers.1.encoder_attn.v_proj.bias"}
    with pytest.raises(KeyError):
        ours.load_hf_state_dict(missing)
    assert torch.equal(ours.model.shared.weight[V:], torch.zeros(ours.config.padded_vocab - V, 128, dtype=torch.float64))


@pytest.mark.parametrize("src_lens,tgt_lens", [([20, 20, 20], [24, 24, 24]), ([20, 13, 1], [24, 7, 16])], ids=["fixed", "padded"])
def test_matches_transformers(src_lens, tgt_lens):
    hf, ours = _pair()
    src, lab = _rows(src_lens, tgt_lens, 20, 24)
    out = hf(input_ids=src, attention_mask=(src != 0).long(), labels=lab)
    out.loss.backward()
    logits = ours(src, lab)
    loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), lab.reshape(-1))
    loss.backward()
    keep = lab != -100
    assert torch.allclose(logits[..., :V][keep], out.logits[keep], atol=1e-10)
    assert bool((logits[..., V:] < -1e3).all())
    assert abs(float(loss.detach()) - float(out.loss.detach())) < 1e-10
    for name, grad in _grads(ours).items():
        want = _hf_grad(hf, name)
        if name == "model.shared.weight":
            grad = grad[:V]
        assert torch.allclose(grad, want, atol=1e-9, rtol=1e-7), name


def test_packed_rows_match_each_pair_alone():
    """Two rows of packed pairs: every target document's logits equal transformers' on that pair alone."""
    hf, ours = _pair(bos_token_id=START)
    pairs = [[(9, 12), (5, 4), (1, 1)], [(14, 20), (6, 3)]]
    Sk, Sq = 24, 32
    g = torch.Generator().manual_seed(5)
    src = torch.zeros(2, Sk, dtype=torch.long)
    lab = torch.full((2, Sq), -100)
    docs = []
    for r, row in enumerate(pairs):
        a = b = 0
        for s, t in row:
            x, y = torch.randint(7, V, (s,), generator=g), torch.randint(7, V, (t,), generator=g)
            x[0] = y[0] = START
            src[r, a:a + s], lab[r, b:b + t] = x, y
            docs.append((r, b, x, y))
            a, b = a + s, b + t
    logits = ours(src, lab)
    for r, b, x, y in docs:
        alone = hf(input_ids=x[None], labels=y[None]).logits[0]
        assert torch.allclose(logits[r, b:b + len(y), :V], alone, atol=1e-10), (r, b)


def test_decoder_input_is_shift_tokens_right_on_one_document_rows():
    hf, ours = _pair()
    src, lab = _rows([20, 13, 1], [24, 7, 16], 20, 24)
    ids, _, _ = ours.model.decoder_inputs(lab)
    want = transformers.models.bart.modeling_bart.shift_tokens_right(lab, 0, 2)
    assert torch.equal(ids, want)


def test_cross_attention_matches_reference_and_dense_sdpa():
    torch.manual_seed(0)
    src = torch.tensor([[4] * 10 + [9] + [4] * 5 + [0] * 4, [4] * 20])
    tgt = torch.tensor([[4] * 7 + [9] + [4] * 8, [4] * 3 + [0] * 13])
    enc, _ = document_bounds(src, 9, 0)
    dec, _ = document_bounds(tgt, 9, 0)
    qb, kb = cross_bounds(enc, dec)
    q = torch.randn(2, 16, 128, dtype=torch.float64, requires_grad=True)
    kv = torch.randn(2, 20, 256, dtype=torch.float64, requires_grad=True)
    out = cross_attention(q, kv, qb, kb, 2)
    assert torch.equal(out, cross_attention_reference(q, kv, qb, 2))
    keep = (torch.arange(20) >= qb[..., :1].long()) & (torch.arange(20) < qb[..., 1:].long())
    qs = q.view(2, 16, 2, 64).transpose(1, 2)
    k, v = (t.reshape(2, 20, 2, 64).transpose(1, 2) for t in kv.split(128, -1))
    dense = F.scaled_dot_product_attention(qs, k, v, attn_mask=keep[:, None]).nan_to_num(0.0) * keep.any(-1)[:, None, :, None]
    assert torch.allclose(out, dense.transpose(1, 2).reshape(2, 16, 128), atol=1e-12)
    g = torch.randn_like(out)
    got = torch.autograd.grad(out, (q, kv), g)
    want = torch.autograd.grad(dense.transpose(1, 2).reshape(2, 16, 128), (q, kv), g)
    for a, b in zip(got, want):
        assert torch.allclose(a, b, atol=1e-12)


def _precondition_holds(qb, kb):
    """query i sees key j per q_bounds iff key j is seen by query i per kv_bounds, every row, every (i, j)"""
    Sq, Sk = qb.shape[1], kb.shape[1]
    i, j = torch.arange(Sq)[:, None], torch.arange(Sk)[None, :]
    a = (j >= qb[..., :1]) & (j < qb[..., 1:])
    b = ((i >= kb[..., 0][:, None, :]) & (i < kb[..., 1][:, None, :]))
    return torch.equal(a, b)


def test_cross_bounds_padded_and_packed():
    src = torch.tensor([[4, 4, 4, 0, 0, 0], [4, 4, 9, 4, 9, 4], [0] * 6])
    tgt = torch.tensor([[4, 4, 0, 0], [4, 9, 9, 4], [4, 4, 4, 4]])
    enc, _ = document_bounds(src, 9, 0)
    dec, _ = document_bounds(tgt, 9, 0)
    qb, kb = cross_bounds(enc, dec)
    assert qb.dtype == kb.dtype == torch.int32
    assert qb.tolist() == [[[0, 3], [0, 3], [0, 0], [0, 0]],
                           [[0, 2], [2, 4], [4, 6], [4, 6]],
                           [[0, 0]] * 4]
    assert kb.tolist() == [[[0, 2]] * 3 + [[0, 0]] * 3,
                           [[0, 1]] * 2 + [[1, 2]] * 2 + [[2, 4]] * 2,
                           [[0, 0]] * 6]
    assert _precondition_holds(qb, kb)


def test_cross_bounds_meet_the_precondition_exhaustively():
    """Every pair of rows of up to 3 document starts in 6 positions, with every length."""
    import itertools
    rows = []
    for n in range(0, 7):
        for starts in itertools.chain.from_iterable(itertools.combinations(range(1, n), k) for k in range(0, 3)):
            ids = [4] * n + [0] * (6 - n)
            for s in starts:
                ids[s] = 9
            rows.append(ids)
    t = torch.tensor(rows)
    bounds, _ = document_bounds(t, 9, 0)
    R = len(rows)
    enc = bounds.repeat_interleave(R, 0)
    dec = bounds.repeat(R, 1, 1)
    qb, kb = cross_bounds(enc, dec)
    assert _precondition_holds(qb, kb)
    docs = lambda b: [tuple(x) for x in b.tolist() if x[0] < x[1]]
    for r in range(0, R * R, 37):                                # the k-th target document sees the k-th source document
        e, d = sorted(set(docs(enc[r]))), sorted(set(docs(dec[r])))
        for k, (s, t) in enumerate(d):
            want = list(e[k]) if k < len(e) else [0, 0]
            assert qb[r, s].tolist() == want


def test_synthetic_denoising_data():
    a = SyntheticDenoising(samples=64, seq_len=128, vocab=V + 200, start_id=START, mask_id=V + 150, min_len=8, pack=True)
    b = SyntheticDenoising(samples=64, seq_len=128, vocab=V + 200, start_id=START, mask_id=V + 150, min_len=8, pack=True)
    assert torch.equal(a.X, b.X) and torch.equal(a.Y, b.Y)
    assert a.pad_token_id == 0 and a.bos_token_id == START
    for r in range(len(a)):
        src_docs = document_bounds(a.X[r:r + 1], START, 0)[0][0]
        tgt_docs = document_bounds(a.Y[r:r + 1].masked_fill(a.Y[r:r + 1] == -100, 0), START, 0)[0][0]
        src_starts = [int(s) for i, (s, e) in enumerate(src_docs.tolist()) if s == i and e > s]
        tgt_starts = [int(s) for i, (s, e) in enumerate(tgt_docs.tolist()) if s == i and e > s]
        assert len(src_starts) == len(tgt_starts) == len(a.doc_lengths[r])       # pairs share a row
        for (s0, s1), (t0, t1) in zip(((int(src_docs[i][0]), int(src_docs[i][1])) for i in src_starts),
                                      ((int(tgt_docs[i][0]), int(tgt_docs[i][1])) for i in tgt_starts)):
            assert s1 - s0 <= t1 - t0                                             # no source longer than its target
            assert int(a.X[r, s0]) == int(a.Y[r, t0]) == START
    fixed = SyntheticDenoising(samples=16, seq_len=64, vocab=V + 200, start_id=START, mask_id=V + 150)
    assert bool((fixed.lengths == 64).all()) and bool(((fixed.X != 0).sum(1) < 64).all())
    masked = float((fixed.Y != (V + 150)).sum() - (fixed.X[fixed.X != 0] != V + 150).sum()) / (fixed.Y.numel() - 16)
    assert 0.25 < masked < 0.35                                  # about 30 % of the tokens replaced


def _args(tmp_path, *flags):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "bart-base",
                                          "--no_cuda", *flags])


@pytest.mark.parametrize("flags", [[], ["--min_seq_len", "32", "--seq_len", "64"], ["--pack", "--min_seq_len", "32", "--seq_len", "64"],
                                   ["--fused_lm_loss"], ["--optimizer", "adamw", "--gradient_accumulation_steps", "2"]])
def test_cli_accepts(tmp_path, flags):
    from b200ddp.engine import cli
    cli.setup(_args(tmp_path, *flags))


@pytest.mark.parametrize("flags,match", [(["--fp8", "--fp16"], "--fp8"), (["--sparse_prediction"], "--sparse_prediction"),
                                         (["--seq_len", "1025"], "1024")])
def test_cli_rejects(tmp_path, flags, match):
    from b200ddp.engine import cli
    with pytest.raises(ValueError, match=match):
        cli.setup(_args(tmp_path, *flags))


def test_cli_rejects_gpu_misuse():
    import argparse
    from b200ddp.engine import cli
    for fp16, seq_len, match in ((False, 128, "--fp16"), (True, 100, "multiple of 128")):
        args = argparse.Namespace(model="bart-base", device=torch.device("cuda"), fp16=fp16, seq_len=seq_len)
        with pytest.raises(ValueError, match=match):
            cli.check_seq2seq_args(args)


def test_registry_and_dataset(tmp_path):
    from b200ddp.engine.trainer import build_dataset
    for name in ("bart-base", "bart-large"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "causal" and e.seq2seq and e.start_id not in (0, 2) and not e.fp8 and not e.contrastive
    ds = build_dataset(_args(tmp_path, "--pack", "--min_seq_len", "16", "--seq_len", "64"))
    assert isinstance(ds, SyntheticDenoising) and ds.bos_token_id == MODEL_REGISTRY["bart-base"].start_id


def test_short_cpu_training_run_resumes(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    from b200ddp.models import build_model
    flags = ["--per_gpu_train_batch_size", "2", "--max_steps", "2", "--logging_steps", "1", "--save_steps", "2", "--optimizer", "adamw",
             "--lr", "1e-4", "--dataset_size", "8", "--seq_len", "32", "--min_seq_len", "16", "--pack"]
    args = _args(tmp_path, *flags)
    cli.setup(args)
    trainer = Trainer(args, build_model("bart-base", pad_token_id=0, bos_token_id=3), cli.log)
    step, loss = trainer.train()
    assert step == 3 and math.isfinite(loss) and loss > 0
    args = _args(tmp_path, *flags[:5], "4", *flags[6:], "--resume_from", "latest")
    cli.setup(args)
    step, loss = Trainer(args, build_model("bart-base", pad_token_id=0, bos_token_id=3), cli.log).train()
    assert step >= 3 and math.isfinite(loss)                    # continues from the saved step


def _tiny(bos_token_id=None):
    torch.manual_seed(0)
    return BartForConditionalGeneration(BartConfig(vocab_size=V, hidden=128, encoder_layers=1, decoder_layers=1, heads=2, intermediate=256,
                                                   max_position=64, pad_token_id=0, bos_token_id=bos_token_id))


def test_tiny_bart_learns_to_denoise():
    ds = SyntheticDenoising(samples=8, seq_len=32, vocab=V, start_id=START, mask_id=V - 1, min_len=16)
    model = _tiny()
    opt = torch.optim.AdamW(model.parameters(), lr=3e-3)
    losses = []
    for _ in range(30):
        logits = model(ds.X, ds.Y)
        loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), ds.Y.reshape(-1))
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.5 * losses[0]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _data():
    return SyntheticDenoising(samples=4, seq_len=32, vocab=V, start_id=START, mask_id=V - 1, min_len=12, seed=3)


def _loss(model, x, y):
    logits = model(x, y)
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]), y.reshape(-1))


def _ddp_worker(rank, world, port, path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200ddp.parallel import DistributedDataParallel
        model = _tiny().double()
        ddp = DistributedDataParallel(model, backend="gloo")
        ds = _data()
        n = len(ds) // world
        _loss(ddp, ds.X[rank * n:(rank + 1) * n], ds.Y[rank * n:(rank + 1) * n]).backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        torch.optim.SGD(model.parameters(), lr=0.1).step()
        torch.save({"grads": grads, "params": {k: p.detach().clone() for k, p in model.named_parameters()}}, f"{path}.{rank}")
    finally:
        dist.destroy_process_group()


def test_gloo_world_2_keeps_ranks_identical_and_averages_gradients(tmp_path):
    path = str(tmp_path / "rank")
    mp.spawn(_ddp_worker, args=(2, _free_port(), path), nprocs=2, join=True)
    r0, r1 = torch.load(f"{path}.0"), torch.load(f"{path}.1")
    ds = _data()
    single = []
    for half in (slice(0, 2), slice(2, 4)):
        m = _tiny().double()
        _loss(m, ds.X[half], ds.Y[half]).backward()
        single.append({k: p.grad for k, p in m.named_parameters()})
    for k in single[0]:
        want = (single[0][k] + single[1][k]) / 2
        assert torch.allclose(r0["grads"][k], want, rtol=1e-9, atol=1e-12), k
        assert torch.equal(r0["params"][k], r1["params"][k]), k
