"""ViT-MAE on the CPU: presets and parameter counts as transformers reports them, strict state-dict loading, loss and every
gradient against ``transformers.ViTMAEForPreTraining`` with the same weights and noise, the shuffle reference's tie rule,
the registry and CLI wiring, and a tiny model's loss falling on structured images."""
import math

import pytest
import torch

from b200ddp.engine import cli
from b200ddp.engine.trainer import OwnLoss, build_criterion
from b200ddp.models import MODEL_REGISTRY, build_model, vit_mae_base, vit_mae_large
from b200ddp.models.vit_mae import ViTMAEConfig, ViTMAEForPreTraining, sincos_pos_embed
from b200ddp.ops import mae_shuffle, mae_shuffle_reference
from b200ddp.optim.adamw import weight_decay_groups

transformers = pytest.importorskip("transformers")
from transformers.models.vit_mae.modeling_vit_mae import get_2d_sincos_pos_embed  # noqa: E402

TINY = dict(hidden=64, layers=2, heads=2, intermediate=128, decoder_hidden=64, decoder_layers=2, decoder_heads=2,
            decoder_intermediate=128, image_size=32, patch_size=8)
HF_TINY = dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=2, intermediate_size=128, decoder_hidden_size=64,
               decoder_num_hidden_layers=2, decoder_num_attention_heads=2, decoder_intermediate_size=128, image_size=32, patch_size=8)


@pytest.mark.parametrize("build,total,trainable,hf_keys", [(vit_mae_base, 111_907_840, 111_655_680, 334),
                                                           (vit_mae_large, 329_541_888, 329_239_296, 526)])
def test_presets_and_parameter_counts(build, total, trainable, hf_keys):
    with torch.device("meta"):
        m = build()
    assert sum(p.numel() for p in m.parameters()) == total
    assert sum(p.numel() for p in m.parameters() if p.requires_grad) == trainable
    c = m.config
    assert (c.patch_size, c.image_size, c.mask_ratio, c.eps, c.keep, c.num_patches) == (16, 224, 0.75, 1e-12, 49, 196)
    assert (c.decoder_hidden, c.decoder_layers, c.decoder_heads, c.decoder_intermediate) == (512, 8, 16, 2048)
    assert not c.norm_pix_loss
    # each layer's 6 q / k / v keys are 2 here
    layers = c.layers + c.decoder_layers
    assert len(m.state_dict()) == hf_keys - 4 * layers


def test_position_tables_are_transformers_sincos_and_frozen():
    for dim in (512, 768, 1024):
        assert torch.allclose(sincos_pos_embed(dim, 14), torch.from_numpy(get_2d_sincos_pos_embed(dim, 14, add_cls_token=True)), atol=1e-12)
    m = ViTMAEForPreTraining(ViTMAEConfig(**TINY))
    for p in (m.vit.embeddings.position_embeddings, m.decoder.decoder_pos_embed):
        assert not p.requires_grad
    assert torch.equal(m.decoder.decoder_pos_embed[0].double(), sincos_pos_embed(64, 4).float().double())


def _pair(norm_pix, seed=0):
    cfg = transformers.ViTMAEConfig(**HF_TINY, norm_pix_loss=norm_pix)
    torch.manual_seed(seed)
    hf = transformers.ViTMAEForPreTraining(cfg).double().train()
    sd = {k: torch.randn_like(v) * 0.1 for k, v in hf.state_dict().items()}
    hf.load_state_dict(sd)
    ours = ViTMAEForPreTraining(ViTMAEConfig(**TINY, norm_pix_loss=norm_pix)).double()
    ours.load_hf_state_dict(sd)
    return hf, ours, sd


def test_load_hf_state_dict_is_strict_both_ways():
    _, ours, sd = _pair(False)
    missing = dict(sd)
    missing.pop("decoder.mask_token")
    with pytest.raises(KeyError):
        ours.load_hf_state_dict(missing)
    with pytest.raises(KeyError, match="unexpected"):
        ours.load_hf_state_dict({**sd, "vit.pooler.weight": torch.zeros(1)})


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("norm_pix", [False, True])
def test_loss_and_gradients_match_transformers(norm_pix, dtype):
    hf, ours, _ = _pair(norm_pix)
    hf, ours = hf.to(dtype), ours.to(dtype)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(3, 3, 32, 32, generator=g, dtype=torch.float64).to(dtype)
    noise = torch.rand(3, 16, generator=g)
    ref = hf(pixel_values=x, noise=noise)
    out = ours.pretraining_output(x, noise)
    ref.loss.backward()
    out.loss.backward()
    tol = 1e-12 if dtype == torch.float64 else 2e-5
    assert abs(float(ref.loss) - float(out.loss)) <= tol * abs(float(ref.loss))
    assert torch.allclose(out.logits, ref.logits, rtol=tol, atol=tol)
    assert torch.equal(out.mask, ref.mask) and torch.equal(out.ids_restore, ref.ids_restore)
    hg = dict(hf.named_parameters())
    for name, p in ours.named_parameters():
        if not p.requires_grad:
            assert p.grad is None
            continue
        if ".qkv." in name:
            stem, wb = name.rsplit(".qkv.", 1)
            r = torch.cat([hg[f"{stem}.{k}.{wb}"].grad for k in ("query", "key", "value")])
        else:
            r = hg[name].grad
        err = float((p.grad - r).abs().max() / r.abs().max().clamp_min(1e-30))
        assert err <= (1e-10 if dtype == torch.float64 else 1e-4), name


def test_shuffle_reference_is_argsort_with_ties_by_index():
    noise = torch.rand(4, 196)
    ids_keep, ids_restore = mae_shuffle(noise, 49)
    assert torch.equal(ids_keep, torch.argsort(noise, 1)[:, :49])
    assert torch.equal(ids_restore, torch.argsort(torch.argsort(noise, 1), 1))
    tied = torch.tensor([[0.5, 0.1, 0.5, 0.1, 0.0]])
    k, r = mae_shuffle_reference(tied, 2)
    assert k.tolist() == [[4, 1]] and r.tolist() == [[3, 1, 4, 2, 0]]


def _args(*argv):
    args = cli.build_parser().parse_args(["--model", "vit-mae-base", "--no_cuda", *argv])
    return args


def test_registry_and_criterion():
    for name in ("vit-mae-base", "vit-mae-large"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "image" and e.own_loss and e.config is None and not e.contrastive
    assert [n for n, e in MODEL_REGISTRY.items() if e.own_loss] == ["vit-mae-base", "vit-mae-large"]
    crit = build_criterion(_args())
    assert isinstance(crit, OwnLoss)
    loss = torch.tensor(1.5)
    assert crit(loss, torch.zeros(3, dtype=torch.long)) is loss


@pytest.mark.parametrize("argv", [["--loss", "mse"], ["--loss", "ce"], ["--seq_len", "128"], ["--fp8", "--fp16"], ["--pack", "--min_seq_len", "8"],
                                  ["--min_seq_len", "8"], ["--fused_lm_loss"], ["--sparse_prediction"]])
def test_cli_rejects_flags_that_do_not_apply(argv):
    with pytest.raises(ValueError):
        cli.setup(_args(*argv))


def test_cli_rejects_single_process_data_parallel():
    args = _args()
    args.device, args.n_gpu, args.local_rank = torch.device("cuda"), 2, -1
    with pytest.raises(ValueError, match="DataParallel"):
        cli.check_own_loss_args(args)


@pytest.mark.parametrize("argv", [[], ["--fp16", "--cuda_graph", "--channels_last"], ["--gradient_accumulation_steps", "2"],
                                  ["--optimizer", "adamw", "--eval_at_end"]])
def test_cli_accepts(argv):
    cli.setup(_args(*argv))


def test_adamw_groups_decay_the_tokens_and_skip_the_frozen_tables():
    m = ViTMAEForPreTraining(ViTMAEConfig(**TINY))
    decay, no_decay = weight_decay_groups(m, 0.05)
    ids = {id(p) for p in decay["params"]}
    assert id(m.vit.embeddings.cls_token) in ids and id(m.decoder.mask_token) in ids
    frozen = {id(m.vit.embeddings.position_embeddings), id(m.decoder.decoder_pos_embed)}
    assert not frozen & (ids | {id(p) for p in no_decay["params"]})


def test_tiny_model_loss_falls_on_structured_images():
    torch.manual_seed(0)
    m = ViTMAEForPreTraining(ViTMAEConfig(**TINY))
    yy, xx = torch.meshgrid(torch.arange(32.0), torch.arange(32.0), indexing="ij")
    images = torch.stack([torch.stack([torch.sin((xx + 3 * b) / 5), torch.cos(yy / 4), (xx + yy) / 64]) for b in range(8)])
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    g = torch.Generator().manual_seed(0)
    noise = torch.rand(8, 16, generator=g)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = m(images, noise)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses)
    assert losses[-1] < 0.5 * losses[0], losses


def test_build_on_meta_through_the_registry():
    with torch.device("meta"):
        m = build_model("vit-mae-large")
    assert m.config.hidden == 1024
