"""Vision Transformer on the CPU: torchvision's state dict key for key, its logits, loss and gradients from the same weights,
its initialisation, the image-as-document token layout, the DDP bucket plan, the CLI and a short training run."""
import math

import pytest
import torch
import torch.distributed as dist

from b200ddp.models import MODEL_REGISTRY, build_model, vit_b_16, vit_b_32, vit_l_16
from b200ddp.ops import cross_entropy, image_token_bounds, image_token_rows, patch_embed, patch_embed_reference
from b200ddp.parallel.buckets import MiB

tvm = pytest.importorskip("torchvision.models")

PRESETS = {"vit_b_16": vit_b_16, "vit_b_32": vit_b_32, "vit_l_16": vit_l_16}
PARAMS = {"vit_b_16": 86_567_656, "vit_b_32": 88_224_232, "vit_l_16": 304_326_632}


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_state_dict_is_torchvisions_key_for_key(name):
    with torch.device("meta"):
        ours, theirs = PRESETS[name](), getattr(tvm, name)()
    a, b = ours.state_dict(), theirs.state_dict()
    assert list(a) == list(b)
    assert [tuple(t.shape) for t in a.values()] == [tuple(t.shape) for t in b.values()]
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in theirs.named_parameters()]
    assert sum(p.numel() for p in ours.parameters()) == PARAMS[name]


def _seeded_torchvision(name, seed=0):
    torch.manual_seed(seed)
    tv = getattr(tvm, name)()
    with torch.no_grad():
        for n, p in tv.named_parameters():          # away from the zero head and unit norms, so every gradient is non-trivial
            if n.startswith("heads.") or n.endswith(("ln_1.weight", "ln_2.weight", "ln.weight")) or n in ("class_token",):
                p.normal_(1.0 if n.endswith("weight") and "ln" in n else 0.0, 0.1 if "ln" in n else 0.02)
            elif n.endswith("bias"):
                p.normal_(0.0, 0.02)
    return tv.eval()


@pytest.mark.parametrize("name", ["vit_b_16", "vit_b_32"])
def test_matches_torchvision_given_its_weights(name):
    tv = _seeded_torchvision(name)
    ours = PRESETS[name]()
    ours.load_state_dict(tv.state_dict(), strict=True)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(3, 3, 224, 224, generator=g)
    target = torch.randint(0, 1000, (3,), generator=g)
    ref_logits = tv(x)
    ref_loss = torch.nn.functional.cross_entropy(ref_logits, target)
    ref_loss.backward()
    logits = ours(x)
    loss = cross_entropy(logits, target)
    loss.backward()
    assert float((logits - ref_logits).norm() / ref_logits.norm()) < 1e-5
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    for (n, p), (m, q) in zip(ours.named_parameters(), tv.named_parameters()):
        assert n == m
        rel = float((p.grad - q.grad).norm() / q.grad.norm())
        assert rel < 1e-4, (n, rel)


def test_loading_is_strict_both_ways():
    tv = _seeded_torchvision("vit_b_32")
    ours = vit_b_32()
    ours.load_state_dict(tv.state_dict(), strict=True)
    fresh = tvm.vit_b_32()
    fresh.load_state_dict(ours.state_dict(), strict=True)
    assert all(torch.equal(a, b) for a, b in zip(fresh.state_dict().values(), tv.state_dict().values()))
    extra = dict(tv.state_dict(), **{"encoder.extra": torch.zeros(1)})
    with pytest.raises(RuntimeError, match="Unexpected key"):
        ours.load_state_dict(extra, strict=True)
    missing = {k: v for k, v in tv.state_dict().items() if k != "class_token"}
    with pytest.raises(RuntimeError, match="Missing key"):
        ours.load_state_dict(missing, strict=True)


def test_initialisation_is_torchvisions():
    """The same seed gives torchvision's weights exactly (the same init calls in the same order): patch weight normal cut at
    +-2 with std 1 / sqrt(768), xavier-uniform projections, biases 1e-6 / 0, position embedding std 0.02, zero head."""
    torch.manual_seed(5)
    tv = tvm.vit_b_16()
    torch.manual_seed(5)
    ours = vit_b_16()
    for (n, p), q in zip(ours.state_dict().items(), tv.state_dict().values()):
        assert torch.equal(p, q), n
    w = ours.conv_proj.weight
    assert abs(float(w.std()) - 1 / math.sqrt(768)) < 5e-4 and float(w.abs().max()) <= 2.0
    assert abs(float(ours.encoder.pos_embedding.std()) - 0.02) < 5e-4
    lim = math.sqrt(6 / (768 + 3 * 768))
    ipw = ours.encoder.layers.encoder_layer_0.self_attention.in_proj_weight
    assert float(ipw.abs().max()) <= lim and float(ipw.abs().max()) > 0.99 * lim
    assert float(ours.heads.head.weight.abs().max()) == 0 and float(ours.heads.head.bias.abs().max()) == 0
    assert float(ours.class_token.abs().max()) == 0 and float(ours.conv_proj.bias.abs().max()) == 0
    x = torch.randn(2, 3, 224, 224)
    loss = cross_entropy(ours(x), torch.tensor([3, 999]))
    assert abs(float(loss) - math.log(1000)) < 1e-6


@pytest.mark.parametrize("batch,tokens", [(1, 197), (3, 197), (64, 197), (5, 50), (7, 50), (13, 128), (2, 1)])
def test_image_token_bounds_match_brute_force(batch, tokens):
    T = image_token_rows(batch, tokens)
    assert T % 128 == 0 and batch * tokens <= T < batch * tokens + 128
    want = []
    for b in range(batch):
        want += [(b * tokens, (b + 1) * tokens)] * tokens
    want += [(0, 0)] * (T - batch * tokens)
    got = image_token_bounds(batch, tokens, "cpu")
    assert got.dtype == torch.int32 and tuple(got.shape) == (1, T, 2)
    assert got[0].tolist() == [list(w) for w in want]


def test_patch_embed_reference_is_torchvisions_input_stage():
    tv = _seeded_torchvision("vit_b_32")
    x = torch.randn(3, 3, 224, 224)
    tokens = patch_embed(x, tv.conv_proj.weight, tv.conv_proj.bias, tv.class_token, tv.encoder.pos_embedding)
    ref = torch.cat([tv.class_token.expand(3, -1, -1), tv._process_input(x)], 1) + tv.encoder.pos_embedding
    assert tuple(tokens.shape) == (256, 768)
    assert torch.equal(tokens[:150], ref.reshape(150, 768)) and float(tokens[150:].abs().max()) == 0
    assert torch.equal(patch_embed_reference(x, tv.conv_proj.weight, tv.conv_proj.bias, tv.class_token, tv.encoder.pos_embedding),
                       tokens)


def test_ddp_bucket_assignment_matches_torch():
    from b200ddp.parallel.buckets import assign_by_size, plan_buckets
    with torch.device("meta"):
        model = vit_b_16()
    params = list(model.parameters())
    for cap in (1, 25):
        ref = dist._compute_bucket_assignment_by_size(params, [1 * MiB, cap * MiB])[0]
        assert assign_by_size([p.numel() * 4 for p in params], None, [1 * MiB, cap * MiB]) == ref
        specs = plan_buckets([p.numel() for p in params], [4] * len(params), bucket_cap_bytes=cap * MiB, order="torch",
                             max_tensors=10 ** 9)
        assert [s.param_indices for s in reversed(specs)] == ref


def test_registry_entries():
    for name in ("vit-b-16", "vit-b-32", "vit-l-16"):
        e = MODEL_REGISTRY[name]
        assert e.kind == "image" and e.config is None and e.start_id is None and not e.fp8


@pytest.mark.parametrize("flags,match", [(["--pack"], "--pack"), (["--min_seq_len", "64"], "--min_seq_len"),
                                         (["--fp8", "--fp16"], "--fp8"), (["--fused_lm_loss"], "--fused_lm_loss"),
                                         (["--sparse_prediction"], "--sparse_prediction")])
def test_cli_rejects_token_only_flags(tmp_path, flags, match):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "vit-b-16",
                                          "--no_cuda", *flags])
    with pytest.raises(ValueError, match=match):
        cli.setup(args)


def test_short_cpu_training_run(tmp_path):
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "vit-b-32",
                                          "--no_cuda", "--per_gpu_train_batch_size", "2", "--max_steps", "2", "--logging_steps", "1",
                                          "--save_steps", "0", "--optimizer", "adamw", "--lr", "1e-3", "--dataset_size", "8"])
    cli.setup(args)
    trainer = Trainer(args, build_model("vit-b-32"), cli.log)
    step, loss = trainer.train()
    assert step == 3 and math.isfinite(loss) and loss > 0
