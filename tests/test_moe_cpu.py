"""Granite-3.0-1B-A400M and the mixture-of-experts op on the CPU: a tiny GraniteMoe model with all four multipliers and a
padded vocabulary against Hugging Face's ``GraniteMoeForCausalLM`` (logits, loss, loss plus the router's load-balancing
loss), the preset's parameter count, the expert-sort invariants, the CLI, and the dense presets' unchanged state dicts."""
import types

import pytest
import torch

from b200ddp.ops import functional as Fn

VOCAB = 1000                                    # padded to 1024 by pad_vocab_to=64


def _tiny_cfg(**kw):
    from b200ddp.models.llama import LlamaConfig
    base = dict(vocab_size=VOCAB, max_position=128, hidden=128, layers=2, heads=2, kv_heads=1, intermediate=64, eps=1e-6,
                num_experts=8, experts_per_token=2, router_aux_loss_coef=0.01, embedding_multiplier=12.0,
                attention_multiplier=0.015625, residual_multiplier=0.22, logits_scaling=6.0, pad_vocab_to=64)
    return LlamaConfig(**{**base, **kw})


def _tiny_hf(seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.GraniteMoeConfig(vocab_size=VOCAB, hidden_size=128, intermediate_size=64, num_hidden_layers=2,
                                        num_attention_heads=2, num_key_value_heads=1, num_local_experts=8, num_experts_per_tok=2,
                                        max_position_embeddings=128, rms_norm_eps=1e-6, rope_theta=10000.0,
                                        embedding_multiplier=12.0, attention_multiplier=0.015625, residual_multiplier=0.22,
                                        logits_scaling=6.0, tie_word_embeddings=True, router_aux_loss_coef=0.01)
    hf = transformers.GraniteMoeForCausalLM(cfg).eval()
    with torch.no_grad():                       # larger weights than the default init, so that routing and the MoE matter
        for n, p in hf.named_parameters():
            if "block_sparse_moe" in n:
                p.normal_(std=0.1)
    return hf


def _router_logits(hf, ids):
    """Each layer's router logits (fp32 [T, E]), captured with forward hooks."""
    out = []
    hooks = [layer.block_sparse_moe.router.layer.register_forward_hook(lambda m, i, o: out.append(o.float()))
             for layer in hf.model.layers]
    try:
        res = hf(ids, labels=ids)
    finally:
        for h in hooks:
            h.remove()
    return res, out


def test_tiny_granite_matches_hugging_face_logits_loss_and_aux_loss():
    from transformers.models.granitemoe.modeling_granitemoe import load_balancing_loss_func
    from b200ddp.models.llama import LlamaForCausalLM
    hf = _tiny_hf()
    ours = LlamaForCausalLM(_tiny_cfg())
    ours.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, VOCAB, (2, 40), generator=torch.Generator().manual_seed(3))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    with torch.no_grad():
        ref, router = _router_logits(hf, ids)
        logits = ours(ids)
    assert logits.shape == (2, 40, 1024)
    assert torch.allclose(logits[..., :VOCAB], ref.logits, atol=1e-4), float((logits[..., :VOCAB] - ref.logits).abs().max())
    assert (logits[..., VOCAB:] < -1e3).all()
    lm = float(Fn.cross_entropy(logits, labels))
    assert abs(lm - float(ref.loss)) < 1e-4
    aux_ref = float(load_balancing_loss_func(tuple(router), 8, 2, None))
    aux = float(ours.router_aux_loss())
    assert abs(aux - aux_ref) < 1e-5 * max(1.0, aux_ref), (aux, aux_ref)
    # the trainer's criterion: loss + coef * aux, as Hugging Face's loss with output_router_logits=True
    from b200ddp.engine.trainer import build_criterion
    crit = build_criterion(types.SimpleNamespace(loss=None, model="granite-3.0-1b-a400m"), ours)
    with torch.no_grad():
        total = float(crit(ours(ids), labels))
    assert abs(total - (float(ref.loss) + 0.01 * aux_ref)) < 1e-4


def test_fused_lm_loss_and_moe_gradients_match_the_unfused_model():
    from b200ddp.models.llama import LlamaForCausalLM
    hf = _tiny_hf(seed=1)
    plain, fused = LlamaForCausalLM(_tiny_cfg()), LlamaForCausalLM(_tiny_cfg(fused_lm_loss=True))
    plain.load_hf_state_dict(hf.state_dict())
    fused.load_hf_state_dict(hf.state_dict())
    ids = torch.randint(0, VOCAB, (2, 32), generator=torch.Generator().manual_seed(4))
    labels = torch.cat([ids[:, 1:], torch.full((2, 1), -100)], 1)
    l_plain = Fn.cross_entropy(plain(ids), labels) + 0.01 * plain.router_aux_loss()
    l_fused = fused.lm_head_loss()(fused(ids), labels) + 0.01 * fused.router_aux_loss()
    l_plain.backward()
    l_fused.backward()
    assert abs(float(l_plain.detach()) - float(l_fused.detach())) < 1e-5
    for (n, a), (_, b) in zip(plain.named_parameters(), fused.named_parameters()):
        assert torch.allclose(a.grad, b.grad, atol=1e-5, rtol=1e-4), n
    assert plain.model.layers[0].moe.router.weight.grad.abs().sum() > 0


def test_granite_preset_parameter_count_and_config():
    from b200ddp.models import build_model
    with torch.device("meta"):
        m = build_model("granite-3.0-1b-a400m")
    c = m.config
    assert (c.vocab_size, c.padded_vocab, c.hidden, c.layers, c.heads, c.kv_heads, c.head_dim, c.num_experts,
            c.experts_per_token, c.intermediate, c.max_position, c.q_scale, c.router_aux_loss_coef) == \
        (49155, 49216, 1024, 24, 16, 8, 64, 32, 8, 512, 4096, 0.125, 0.001)
    assert sum(p.numel() for p in m.parameters()) == 1_334_690_816
    assert tuple(m.model.layers[0].moe.w_gate_up.shape) == (32, 1024, 1024)
    assert tuple(m.model.layers[0].moe.w_down.shape) == (32, 1024, 512)


def test_dense_presets_build_the_same_state_dict():
    from b200ddp.models import build_model
    with torch.device("meta"):
        smol, qwen = build_model("smollm-135m"), build_model("qwen2.5-1.5b")
    sd = smol.state_dict()
    assert len(sd) == 2 + 30 * 6 and all(".moe." not in k for k in sd)
    assert sum(v.numel() for v in sd.values()) == 134_515_008
    assert smol.vocab_bias is None and qwen.vocab_bias is None
    assert sum(v.numel() for v in qwen.state_dict().values()) == 1_543_714_304
    assert set(sd) == {"model.embed_tokens.weight", "model.norm.weight"} | {
        f"model.layers.{i}.{n}.weight" for i in range(30)
        for n in ("input_layernorm", "qkv", "o_proj", "post_attention_layernorm", "gate_up", "down_proj")}


def test_attention_multiplier_must_scale_q_by_a_power_of_two():
    from b200ddp.models.llama import LlamaForCausalLM
    with pytest.raises(ValueError, match="power of two"):
        LlamaForCausalLM(_tiny_cfg(attention_multiplier=0.1))
    with pytest.raises(ValueError, match="power of two"):
        Fn.rotary(torch.zeros(1, 4, 4 * 64), torch.zeros(1, 4, dtype=torch.long), Fn.rotary_cos_sin(8), 2, 1, q_scale=0.3)


@pytest.mark.parametrize("ties", [False, True])
def test_expert_sort_invariants(ties):
    g = torch.Generator().manual_seed(7)
    T, E, k = 300, 8, 3
    logits = torch.randn(T, E, generator=g)
    if ties:                                             # every logit equal: the tie rule picks experts 0, 1, 2
        logits = torch.zeros(T, E)
    ids, gates = Fn.moe_route_reference(logits, k)
    if ties:
        assert (ids == torch.arange(k)).all() and torch.allclose(gates, torch.full((T, k), 1 / k))
    else:
        assert torch.equal(ids, torch.topk(logits, k).indices)
    counts, offsets, fwd, inv, tiles = Fn.moe_permute_reference(ids, E)
    cap = Fn.moe_capacity(T, E, k)
    assert fwd.numel() == cap and cap % 128 == 0 and cap >= T * k + E * 127
    assert int(offsets[-1]) <= cap and (offsets % 128 == 0).all()
    assert torch.equal(counts.long(), torch.bincount(ids.reshape(-1), minlength=E))
    assert ((offsets[1:] - offsets[:-1]) >= counts).all()
    flat = ids.reshape(-1)
    for e in range(E):
        seg = fwd[int(offsets[e]):int(offsets[e + 1])]
        real = seg[:int(counts[e])]
        assert (seg[int(counts[e]):] == -1).all()
        assert (flat[real.long()] == e).all() and (real[1:] > real[:-1]).all()     # stable: assignment order kept
        assert (tiles[int(offsets[e]) // 128:int(offsets[e + 1]) // 128] == e).all()
    assert (tiles[int(offsets[-1]) // 128:] == -1).all()
    assert torch.equal(fwd[inv.reshape(-1).long()].long(), torch.arange(T * k))


def test_moe_reference_matches_a_dense_per_token_loop():
    g = torch.Generator().manual_seed(2)
    T, H, I, E, k = 24, 32, 16, 4, 2
    x, wr = torch.randn(T, H, generator=g), torch.randn(E, H, generator=g)
    wgu, wd = torch.randn(E, 2 * I, H, generator=g) * 0.2, torch.randn(E, H, I, generator=g) * 0.2
    out, probsum, counts = Fn.moe(x, wr, wgu, wd, k, aux=True)
    logits = x @ wr.t()
    for t in range(T):
        top = torch.topk(logits[t], k)
        w = torch.softmax(top.values, 0)
        ref = sum(w[j] * (wd[e] @ (torch.nn.functional.silu(wgu[e, :I] @ x[t]) * (wgu[e, I:] @ x[t])))
                  for j, e in enumerate(top.indices.tolist()))
        assert torch.allclose(out[t], ref, atol=1e-4)
    assert torch.allclose(probsum, torch.softmax(logits, -1).sum(0)) and int(counts.sum()) == T * k
    with pytest.raises(ValueError, match="top_k"):
        Fn.moe(x, wr, wgu, wd, 5)


def _args(tmp_path, *extra):
    from b200ddp.engine import cli
    return cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra])


def test_granite_cli_accepts_its_flags_and_rejects_the_rest(tmp_path):
    from b200ddp.engine import cli
    args = _args(tmp_path, "--model", "granite-3.0-1b-a400m", "--no_cuda", "--seq_len", "4096", "--min_seq_len", "256", "--pack",
                 "--router_aux_loss_coef", "0")
    cli.setup(args)
    assert args.router_aux_loss_coef == 0
    with pytest.raises(ValueError, match="4096"):
        cli.setup(_args(tmp_path, "--model", "granite-3.0-1b-a400m", "--no_cuda", "--seq_len", "4224"))
    with pytest.raises(ValueError, match="mixture of experts"):
        cli.setup(_args(tmp_path, "--model", "granite-3.0-1b-a400m", "--no_cuda", "--fp16", "--fp8"))
    with pytest.raises(ValueError, match="router_aux_loss_coef"):
        cli.setup(_args(tmp_path, "--model", "smollm-135m", "--no_cuda", "--router_aux_loss_coef", "0.01"))
    with pytest.raises(ValueError, match=">= 0"):
        cli.setup(_args(tmp_path, "--model", "granite-3.0-1b-a400m", "--no_cuda", "--router_aux_loss_coef", "-1"))
    from b200ddp.engine.trainer import RouterAuxLoss, build_criterion
    on = types.SimpleNamespace(loss=None, model="granite-3.0-1b-a400m")
    from b200ddp.models.llama import LlamaForCausalLM
    assert isinstance(build_criterion(on, LlamaForCausalLM(_tiny_cfg())), RouterAuxLoss)
    assert not isinstance(build_criterion(on, LlamaForCausalLM(_tiny_cfg(router_aux_loss_coef=0.0))), RouterAuxLoss)


def test_granite_dataset_documents_start_with_id_1():
    from b200ddp.engine.trainer import build_dataset
    ds = build_dataset(types.SimpleNamespace(model="granite-3.0-1b-a400m", dataset_size=40, seq_len=64, min_seq_len=4, pack=True))
    assert ds.bos_token_id == 1 and ds.pad_token_id == 0 and int(ds.X.max()) < 49155


def test_short_cpu_training_run_lowers_the_loss(tmp_path):
    import math
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer, build_dataset
    from b200ddp.models.llama import LlamaForCausalLM
    args = _args(tmp_path, "--model", "granite-3.0-1b-a400m", "--no_cuda", "--seq_len", "64", "--min_seq_len", "8", "--pack",
                 "--optimizer", "adamw", "--lr", "3e-3", "--max_steps", "30", "--per_gpu_train_batch_size", "4",
                 "--warmup_steps", "2", "--save_steps", "0", "--logging_steps", "10")
    cli.setup(args)
    ds = build_dataset(args)
    ds.X = torch.where(ds.X > 1, ds.X % 16 + 2, ds.X)           # a small alphabet leaves something to learn
    ds.Y = torch.where(ds.Y > 1, ds.Y % 16 + 2, ds.Y)
    model = LlamaForCausalLM(_tiny_cfg(pad_token_id=0, bos_token_id=1))
    trainer = Trainer(args, model, cli.log, dataset=ds)
    before = trainer.evaluate(max_batches=4)["eval_loss"]
    trainer.train()
    after = trainer.evaluate(max_batches=4)["eval_loss"]
    assert math.isfinite(after) and after < before - 0.1, (before, after)


def test_linear_and_moe_reprs():
    from b200ddp.ops import Linear, MoE
    assert repr(Linear(4, 8)) == "Linear(in=4, out=8, bias=True, act=None)"
    r = repr(MoE(64, 32, 8, 2, aux=True))
    assert "experts=8, top_k=2, hidden=64, intermediate=32, aux=True" in r and "Linear(in=64, out=8, bias=False" in r
    assert "MoE(" in repr(_granite_tiny())


def _granite_tiny():
    from b200ddp.models.llama import LlamaForCausalLM
    return LlamaForCausalLM(_tiny_cfg())


def test_granite_aux_loss_is_rejected_under_single_process_data_parallel():
    from b200ddp.engine import cli
    dp = dict(model="granite-3.0-1b-a400m", device=torch.device("cuda"), local_rank=-1, n_gpu=2)
    with pytest.raises(ValueError, match="DataParallel"):
        cli.check_moe_args(types.SimpleNamespace(router_aux_loss_coef=None, **dp))
    with pytest.raises(ValueError, match="DataParallel"):
        cli.check_moe_args(types.SimpleNamespace(router_aux_loss_coef=0.01, **dp))
    cli.check_moe_args(types.SimpleNamespace(router_aux_loss_coef=0.0, **dp))              # no aux loss: nothing to collect
    cli.check_moe_args(types.SimpleNamespace(router_aux_loss_coef=None, **{**dp, "n_gpu": 1}))
    cli.check_moe_args(types.SimpleNamespace(router_aux_loss_coef=None, **{**dp, "local_rank": 0}))  # one process per GPU
