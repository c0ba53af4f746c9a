"""CLIP on the CPU: transformers' CLIPModel state dict loaded strictly, its parameter counts, its embeds, logits and loss
from the same weights, the caption-as-document token layout, the contrastive loss's gradient across two gloo ranks, the
CLI, a short training run and a fit to a handful of pairs."""
import math
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200ddp.models import MODEL_REGISTRY, build_model, clip_vit_b_16, clip_vit_b_32
from b200ddp.models.clip import CLIPConfig, CLIPModel, CLIPTowerConfig
from b200ddp.ops import caption_token_bounds, clip_loss, image_token_rows

transformers = pytest.importorskip("transformers")

PARAMS = {"clip_vit_b_32": 151_277_313, "clip_vit_b_16": 149_620_737}
SOT, EOT = 49406, 49407


def _hf_config(patch=32, small=False):
    c = transformers.CLIPConfig()
    c.vision_config.patch_size = patch
    if small:
        c.vision_config.update(dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
                                    image_size=64))
        c.text_config.update(dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
                                  vocab_size=EOT + 1))
        c.projection_dim = 32
    return c


def _small_ours():
    return CLIPModel(CLIPConfig(patch_size=32, image_size=64, vision=CLIPTowerConfig(64, 2, 2, 128),
                                text=CLIPTowerConfig(64, 2, 2, 128), projection_dim=32))


def _hf_model(config, seed=0):
    torch.manual_seed(seed)
    m = transformers.CLIPModel(config).eval()
    with torch.no_grad():                        # away from zero biases and unit norms, so every gradient is non-trivial
        for n, p in m.named_parameters():
            if n.endswith("bias"):
                p.normal_(0.0, 0.02)
            elif "norm" in n and n.endswith("weight"):
                p.normal_(1.0, 0.1)
    return m


def _captions(B, L=77, seed=1):
    """Captions padded with 0 and with EOT, and (the last) one without any EOT."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, SOT, (B, L), generator=g)
    ids[:, 0] = SOT
    for b in range(B - 1):
        n = int(torch.randint(3, L + 1, (1,), generator=g))
        ids[b, n - 1] = EOT
        ids[b, n:] = 0 if b % 2 == 0 else EOT
    return ids


@pytest.mark.parametrize("name,patch", [("clip_vit_b_32", 32), ("clip_vit_b_16", 16)])
def test_parameter_count_and_strict_load_of_the_presets(name, patch):
    with torch.device("meta"):
        ours = {"clip_vit_b_32": clip_vit_b_32, "clip_vit_b_16": clip_vit_b_16}[name]()
        theirs = transformers.CLIPModel(_hf_config(patch))
    assert sum(p.numel() for p in ours.parameters()) == sum(p.numel() for p in theirs.parameters()) == PARAMS[name]
    sd = theirs.state_dict()
    assert len(sd) == 398
    ours.load_hf_state_dict({k: torch.zeros(v.shape) for k, v in sd.items()})


def test_load_hf_state_dict_is_strict_both_ways():
    hf = _hf_model(_hf_config(small=True))
    sd = hf.state_dict()
    ours = _small_ours()
    ours.load_hf_state_dict(sd)
    assert float(ours.logit_scale) == float(hf.logit_scale)
    q = sd["text_model.encoder.layers.1.self_attn.q_proj.weight"]
    assert torch.equal(ours.text_model.layers[1].self_attention.in_proj_weight[:64], q)
    with pytest.raises(RuntimeError, match="unexpected keys"):
        ours.load_hf_state_dict(dict(sd, extra=torch.zeros(1)))
    with pytest.raises(RuntimeError, match="missing key"):
        ours.load_hf_state_dict({k: v for k, v in sd.items() if k != "vision_model.pre_layrnorm.bias"})


def test_matches_transformers_given_its_weights():
    hf = _hf_model(_hf_config(small=True))
    ours = _small_ours()
    ours.load_hf_state_dict(hf.state_dict())
    g = torch.Generator().manual_seed(3)
    images = torch.randn(5, 3, 64, 64, generator=g)
    ids = _captions(5)
    ref = hf(input_ids=ids, pixel_values=images, return_loss=True)
    ref.loss.backward()
    img, txt, scale = ours(images, ids)
    loss = clip_loss(img, txt, scale)
    loss.backward()
    # CLIPModel's image_embeds / text_embeds are normalised; get_*_features are not
    with torch.no_grad():
        ref_img = hf.get_image_features(pixel_values=images)
        ref_txt = hf.get_text_features(input_ids=ids)
        ref_img = getattr(ref_img, "pooler_output", ref_img)
        ref_txt = getattr(ref_txt, "pooler_output", ref_txt)
    for a, b in ((img, ref_img), (txt, ref_txt)):
        assert float((a - b).norm() / b.norm()) < 1e-5
    ui, ut = img / img.norm(dim=-1, keepdim=True), txt / txt.norm(dim=-1, keepdim=True)
    logits_per_image = scale.exp() * ui @ ut.t()
    assert float((logits_per_image - ref.logits_per_image).abs().max()) < 1e-4
    assert abs(float(loss) - float(ref.loss)) <= 1e-5 * abs(float(ref.loss))
    hf_grads = dict(hf.named_parameters())
    assert float((ours.logit_scale.grad - hf_grads["logit_scale"].grad).abs()) < 1e-5 * float(hf_grads["logit_scale"].grad.abs()) + 1e-7
    qkv = ours.vision_model.layers[0].self_attention.in_proj_weight.grad
    ref_qkv = torch.cat([hf_grads[f"vision_model.encoder.layers.0.self_attn.{p}_proj.weight"].grad for p in "qkv"])
    assert float((qkv - ref_qkv).norm() / ref_qkv.norm()) < 1e-4
    tok = ours.text_model.token_embedding.weight.grad
    ref_tok = hf_grads["text_model.embeddings.token_embedding.weight"].grad
    assert float((tok - ref_tok).norm() / ref_tok.norm()) < 1e-4


def test_initialisation_follows_transformers():
    torch.manual_seed(0)
    m = clip_vit_b_32()
    assert abs(float(m.logit_scale) - 2.6592) < 1e-6
    blk = m.text_model.layers[0]
    assert abs(float(blk.self_attention.in_proj_weight.std()) - 512 ** -0.5 * 24 ** -0.5) < 2e-4
    assert abs(float(blk.mlp[0].weight.std()) - 1024 ** -0.5) < 2e-4
    assert abs(float(m.vision_model.class_embedding.std()) - 768 ** -0.5) < 3e-3
    assert abs(float(m.visual_projection.weight.std()) - 768 ** -0.5) < 2e-4
    assert float(blk.self_attention.in_proj_bias.abs().max()) == 0 and float(blk.mlp[3].bias.abs().max()) == 0
    assert m.vision_model.patch_embedding.bias is None and m.text_projection.bias is None


@pytest.mark.parametrize("B", [1, 2, 3, 5])
def test_caption_token_bounds_match_brute_force(B):
    ids = _captions(B)
    bounds, pooled = caption_token_bounds(ids, EOT)
    T = image_token_rows(B, 77)
    assert bounds.dtype == torch.int32 and tuple(bounds.shape) == (1, T, 2)
    want = []
    for b in range(B):
        hits = (ids[b] == EOT).nonzero()
        e = int(hits[0]) if len(hits) else 0
        assert int(pooled[b]) == 77 * b + e
        want += [(77 * b, 77 * b + e + 1)] * (e + 1) + [(0, 0)] * (76 - e)
    want += [(0, 0)] * (T - 77 * B)
    assert bounds[0].tolist() == [list(w) for w in want]


def test_stream_layout_pools_what_the_dense_causal_mask_pools():
    """The causal-document reference on the caption stream gives the pooled rows of per-caption SDPA with is_causal."""
    from b200ddp.ops import causal_attention_reference
    B, H, d = 3, 2, 64
    ids = _captions(B, seed=4)
    bounds, pooled = caption_token_bounds(ids, EOT)
    T = bounds.shape[1]
    qkv = torch.randn(B * 77, 3 * H * d, dtype=torch.float64)
    stream = torch.nn.functional.pad(qkv, (0, 0, 0, T - B * 77))
    out = causal_attention_reference(stream.view(1, T, -1), bounds, H)[0]
    q, k, v = (t.view(B, 77, H, d).transpose(1, 2) for t in qkv.view(B, 77, -1).split(H * d, -1))
    dense = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B * 77, -1)
    assert torch.allclose(out[pooled], dense[pooled], atol=1e-12)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ddp_worker(rank, world, port, gather_grad, path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200ddp.ops import functional as Fn
        from b200ddp.parallel import DistributedDataParallel
        if not gather_grad:                         # the features of other ranks as constants: the gather's gradient dropped
            def plain(x, group):
                parts = [torch.empty_like(x) for _ in range(dist.get_world_size(group))]
                dist.all_gather(parts, x.detach().contiguous(), group=group)
                parts[dist.get_rank(group)] = x
                return torch.cat(parts, 0)
            Fn._gather_features = plain
        torch.manual_seed(0)
        model = _small_ours().double()
        ddp = DistributedDataParallel(model, backend="gloo")
        images, ids = _batch()
        n = images.shape[0] // world
        img, txt, scale = ddp(images[rank * n:(rank + 1) * n], ids[rank * n:(rank + 1) * n])
        clip_loss(img, txt, scale).backward()
        if rank == 0:
            torch.save({k: p.grad.clone() for k, p in model.named_parameters()}, path)
    finally:
        dist.destroy_process_group()


def _batch():
    g = torch.Generator().manual_seed(7)
    return torch.randn(8, 3, 64, 64, generator=g, dtype=torch.float64), _captions(8, seed=8)


def _ddp_grads(gather_grad, path):
    mp.spawn(_ddp_worker, args=(2, _free_port(), gather_grad, str(path)), nprocs=2, join=True)
    return torch.load(path)


def _single_process_grads():
    torch.manual_seed(0)
    model = _small_ours().double()
    images, ids = _batch()
    clip_loss(*model(images, ids)).backward()
    return {k: p.grad for k, p in model.named_parameters()}


def _max_rel(a, b):
    return max(float((a[k] - b[k]).norm() / b[k].norm().clamp(min=1e-30)) for k in b)


def test_gloo_world_2_gradients_equal_the_full_batch_gradient(tmp_path):
    want = _single_process_grads()
    got = _ddp_grads(True, tmp_path / "with_gather_grad.pt")
    assert set(got) == set(want)
    for k in want:
        assert float((got[k] - want[k]).norm()) <= 1e-9 * float(want[k].norm()) + 1e-15, k
    assert float((got["logit_scale"] - want["logit_scale"]).abs()) <= 1e-9 * float(want["logit_scale"].abs())
    # without the gather's backward the gradient is not the full batch's
    assert _max_rel(_ddp_grads(False, tmp_path / "without.pt"), want) > 1e-3


def test_registry_entries():
    for name in ("clip-vit-b-32", "clip-vit-b-16"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "image" and e.contrastive and e.config is None and e.start_id is None and not e.fp8 and not e.moe
    assert not any(e.contrastive for n, e in MODEL_REGISTRY.items() if not n.startswith("clip-"))


def test_synthetic_pairs():
    from b200ddp.data import SyntheticImageText
    ds = SyntheticImageText(samples=50, batch=16, size=32)
    assert len(ds) == 48 and tuple(ds.X.shape) == (48, 3, 32, 32) and tuple(ds.Y.shape) == (48, 77)
    for row, n in zip(ds.Y, ds.caption_lengths):
        n = int(n)
        assert 8 <= n <= 77 and int(row[0]) == SOT and int(row[n - 1]) == EOT
        assert bool(((row[1:n - 1] >= 1) & (row[1:n - 1] < SOT)).all()) and bool((row[n:] == 0).all())
    assert torch.equal(SyntheticImageText(samples=50, batch=16, size=32).Y, ds.Y)


@pytest.mark.parametrize("flags,match", [(["--pack"], "--pack"), (["--min_seq_len", "64"], "--min_seq_len"),
                                         (["--fp8", "--fp16"], "--fp8"), (["--fused_lm_loss"], "--fused_lm_loss"),
                                         (["--sparse_prediction"], "--sparse_prediction"), (["--seq_len", "512"], "--seq_len"),
                                         (["--loss", "ce"], "--loss")])
def test_cli_rejects_flags_that_do_not_apply(tmp_path, flags, match):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "clip-vit-b-32",
                                          "--no_cuda", *flags])
    with pytest.raises(ValueError, match=match):
        cli.setup(args)


@pytest.mark.parametrize("batch,n_gpu,match", [(12, 1, "multiple of 8"), (16, 2, "DataParallel")])
def test_cli_rejects_gpu_only_misuse(batch, n_gpu, match):
    import argparse
    from b200ddp.engine import cli
    args = argparse.Namespace(model="clip-vit-b-32", device=torch.device("cuda"), local_rank=-1, n_gpu=n_gpu,
                              per_gpu_train_batch_size=batch)
    with pytest.raises(ValueError, match=match):
        cli.check_contrastive_args(args)


def test_short_cpu_training_run(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "clip-vit-b-32",
                                          "--no_cuda", "--per_gpu_train_batch_size", "2", "--max_steps", "2", "--logging_steps", "1",
                                          "--save_steps", "0", "--optimizer", "adamw", "--lr", "1e-4", "--dataset_size", "8"])
    cli.setup(args)
    trainer = Trainer(args, build_model("clip-vit-b-32"), cli.log)
    step, loss = trainer.train()
    assert step == 3 and math.isfinite(loss) and loss > 0


def test_tiny_clip_fits_a_handful_of_pairs():
    """Eight pairs, trained full-batch: the loss drops well below ln(8), where a model that cannot tell pairs apart sits."""
    torch.manual_seed(0)
    model = _small_ours()
    g = torch.Generator().manual_seed(2)
    images, ids = torch.randn(8, 3, 64, 64, generator=g), _captions(8, seed=2)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    for _ in range(40):
        loss = clip_loss(*model(images, ids))
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert float(loss) < 0.25 * math.log(8)
