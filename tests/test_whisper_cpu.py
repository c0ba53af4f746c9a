"""Whisper on the CPU: the state dict, parameter counts, logits and gradients against
``transformers.WhisperForConditionalGeneration``, the mel filterbank and log-mel features against ``WhisperFeatureExtractor``,
the stem gathers against ``F.conv1d``, the synthetic speech data and the CLI."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from b200ddp.data import SyntheticSpeech
from b200ddp.models import MODEL_REGISTRY
from b200ddp.models.whisper import WhisperConfig, WhisperForConditionalGeneration
from b200ddp.ops import (encoder_rows, frame_patches, frame_patches_reference, log_mel_spectrogram, log_mel_spectrogram_reference, mel_patches,
                         whisper_mel_filters)

transformers = pytest.importorskip("transformers")

ROOT = Path(__file__).resolve().parents[1]
SRC = 64                      # max_source_positions of the tiny model: 128 mel frames


def _pair(seed=0):
    """(transformers' tiny model in eval mode, ours loaded from its state dict), fp64."""
    torch.manual_seed(seed)
    hf = transformers.WhisperForConditionalGeneration(transformers.WhisperConfig(
        d_model=128, encoder_layers=2, decoder_layers=2, encoder_attention_heads=2, decoder_attention_heads=2, encoder_ffn_dim=256,
        decoder_ffn_dim=256, max_source_positions=SRC, max_target_positions=64, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
        attn_implementation="eager")).double().eval()
    with torch.no_grad():                                       # away from zero biases
        for n, p in hf.named_parameters():
            if n.endswith("bias") and "layer_norm" not in n:
                p.normal_(0.0, 0.02)
    ours = WhisperForConditionalGeneration(WhisperConfig(hidden=128, encoder_layers=2, decoder_layers=2, heads=2, intermediate=256,
                                                         max_source_positions=SRC, max_position=64)).double()
    ours.load_hf_state_dict(hf.state_dict())
    return hf, ours


def _hf_grad(hf, name):
    """transformers' gradient of our parameter `name`, fused and padded as ours is."""
    g = lambda k: dict(hf.named_parameters())[k].grad
    if name.endswith("qkv.weight") or name.endswith(".kv.weight"):
        p = name.rsplit(".", 2)[0]
        return torch.cat([g(f"{p}.{x}_proj.weight") for x in ("qkv" if name.endswith("qkv.weight") else "kv")])
    if name.endswith("q_bias") or name.endswith("v_bias"):
        return g(f"{name.rsplit('.', 2)[0]}.{name[-6]}_proj.bias")
    if name.endswith("embed_tokens.weight"):
        return F.pad(g(name), (0, 0, 0, 51904 - 51865))
    return g(name)


def _labels(lens, Sq, seed=1):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, 50256, (len(lens), Sq), generator=g)
    for b, n in enumerate(lens):
        lab[b, n - 1] = 50256
        lab[b, n:] = -100
    return lab


@pytest.mark.parametrize("lens", [[24, 24], [24, 9]], ids=["fixed", "right-padded"])
def test_logits_and_gradients_match_transformers(lens):
    hf, ours = _pair()
    feats = torch.randn(2, 80, 2 * SRC, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    lab = _labels(lens, 24)
    ref = hf(input_features=feats, labels=lab).logits
    got = ours(feats, lab)
    keep = lab != -100
    assert got.shape[-1] == 51904 and torch.allclose(got[..., :51865][keep], ref[keep], rtol=1e-9, atol=1e-9)
    F.cross_entropy(ref.reshape(-1, ref.shape[-1]), lab.reshape(-1)).backward()
    F.cross_entropy(got.reshape(-1, got.shape[-1]), lab.reshape(-1)).backward()
    grads = {n: p.grad for n, p in ours.named_parameters() if p.requires_grad}
    assert len(grads) == sum(1 for p in ours.parameters() if p.requires_grad)
    for n, g in grads.items():
        want = _hf_grad(hf, n)
        assert torch.allclose(g, want, rtol=1e-7, atol=1e-10), (n, float((g - want).abs().max()))
    assert ours.model.encoder.embed_positions.weight.grad is None


def test_state_dict_loads_strictly_and_k_biases_stay_zero():
    hf, ours = _pair()
    sd = hf.state_dict()
    with pytest.raises(KeyError):
        ours.load_hf_state_dict({**sd, "extra.weight": torch.zeros(1)})
    layer = ours.model.decoder.layers[0]
    zero = torch.zeros(1, 128, dtype=torch.float64)
    k = layer.self_attn.qkv(zero)[:, 128:256]
    assert torch.equal(k, torch.zeros_like(k)) and torch.equal(layer.encoder_attn.kv(zero)[:, :128], torch.zeros(1, 128, dtype=torch.float64))
    assert torch.equal(ours.model.encoder.embed_positions.weight, sd["model.encoder.embed_positions.weight"])


def test_parameter_counts_match_transformers_plus_padded_vocabulary():
    for name, total, trainable, d in (("whisper-tiny", 37_760_640, 37_184_640, 384), ("whisper-base", 72_593_920, 71_825_920, 512),
                                      ("whisper-small", 241_734_912, 240_582_912, 768)):
        with torch.device("meta"):
            m = MODEL_REGISTRY[name].build()
        assert sum(p.numel() for p in m.parameters()) == total + 39 * d, name
        assert sum(p.numel() for p in m.parameters() if p.requires_grad) == trainable + 39 * d, name


def test_mel_filters_match_the_feature_extractor():
    want = torch.from_numpy(transformers.WhisperFeatureExtractor().mel_filters)
    got = whisper_mel_filters()
    assert got.dtype == torch.float64 and got.shape == (201, 80)
    assert float((got - want).abs().max()) < 1e-10


def _clips():
    """Tone-plus-noise clips with silent tails of different lengths."""
    g = torch.Generator().manual_seed(3)
    t = torch.arange(480000, dtype=torch.float64) / 16000
    out = []
    for f, amp, end in ((440.0, 3000.0, 300000), (1234.5, 12000.0, 479000), (97.0, 500.0, 80000)):
        w = amp * torch.sin(2 * np.pi * f * t) + 0.1 * amp * torch.randn(480000, generator=g, dtype=torch.float64)
        w[end:] = 0
        out.append(w.round().clamp(-32768, 32767).to(torch.int16))
    return torch.stack(out)


def test_log_mel_reference_matches_the_feature_extractor():
    fe = transformers.WhisperFeatureExtractor()
    wave = _clips()
    want = fe(list((wave.numpy() / 32768.0).astype(np.float32)), sampling_rate=16000, return_tensors="np").input_features
    got = log_mel_spectrogram_reference(wave, whisper_mel_filters())
    assert got.shape == (3, 80, 3000)
    assert float(np.abs(got.numpy() - want).max()) < 4e-5
    cpu = log_mel_spectrogram(wave, whisper_mel_filters(), torch.float32)
    assert cpu.dtype == torch.float32 and float((cpu.double() - got).abs().max()) < 1e-4


@pytest.mark.parametrize("bad", [torch.zeros(2, 480000, dtype=torch.int32), torch.zeros(2, 479999, dtype=torch.int16),
                                 torch.zeros(480000, dtype=torch.int16), torch.zeros(2, 960000, dtype=torch.int16)[:, ::2]],
                         ids=["int32", "short", "1d", "strided"])
def test_log_mel_rejects_other_waveforms(bad):
    with pytest.raises(ValueError, match="int16"):
        log_mel_spectrogram(bad, whisper_mel_filters())


def test_stem_gathers_composed_with_linear_match_conv1d():
    g = torch.Generator().manual_seed(4)
    B, T, d = 2, 26, 16
    feats = torch.randn(B, 80, T, dtype=torch.float64, generator=g)
    w1, b1 = torch.randn(d, 80, 3, dtype=torch.float64, generator=g), torch.randn(d, dtype=torch.float64, generator=g)
    w2, b2 = torch.randn(d, d, 3, dtype=torch.float64, generator=g), torch.randn(d, dtype=torch.float64, generator=g)
    h1 = mel_patches(feats) @ w1.permute(0, 2, 1).reshape(d, -1).T + b1
    assert torch.allclose(h1.view(B, T, d), F.conv1d(feats, w1, b1, padding=1).transpose(1, 2), rtol=1e-12, atol=1e-12)
    S = encoder_rows(T)
    assert S == 128
    h1 = h1.requires_grad_(True)
    p2 = frame_patches(h1, T, S)
    y = (p2 @ w2.permute(0, 2, 1).reshape(d, -1).T + b2).view(B, S, d)
    want = F.conv1d(h1.detach().view(B, T, d).transpose(1, 2), w2, b2, stride=2, padding=1).transpose(1, 2)
    assert torch.allclose(y[:, :T // 2], want, rtol=1e-12, atol=1e-12)
    assert torch.equal(p2.view(B, S, -1)[:, T // 2:], torch.zeros(B, S - T // 2, 3 * d, dtype=torch.float64))
    dp2 = torch.randn(B * S, 3 * d, dtype=torch.float64, generator=g)
    p2.backward(dp2)
    want = torch.zeros(B, T, d, dtype=torch.float64)               # the col2im: each h1 row sums its taps
    taps = dp2.view(B, S, 3, d)
    for s in range(T):
        for j in range(3):
            if (s + 1 - j) % 2 == 0 and 0 <= (s + 1 - j) // 2 < T // 2:
                want[:, s] += taps[:, (s + 1 - j) // 2, j]
    assert torch.equal(h1.grad.view(B, T, d), want)
    assert encoder_rows(3000) == 1536


def test_synthetic_speech():
    ds = SyntheticSpeech(samples=4, seq_len=64, min_len=8)
    assert ds.X.dtype == torch.int16 and ds.X.shape == (4, 480000) and ds.Y.shape == (4, 64)
    assert not hasattr(ds, "pad_token_id") and not hasattr(ds, "lengths")
    seg = 480000 // 64
    for x, y in zip(ds.X, ds.Y):
        n = int((y != -100).sum()) - 1
        assert 7 <= n <= 63 and int(y[n]) == 50256 and bool((y[:n] < 50256).all()) and bool((y[:n] >= 0).all())
        assert bool((x[n * seg:] == 0).all()) and (n == 0 or int(x[:n * seg].abs().max()) > 1000)
    fixed = SyntheticSpeech(samples=2, seq_len=16)
    assert bool((fixed.Y[:, -1] == 50256).all()) and bool((fixed.Y != -100).all())


def _cli(*extra, tmp_path):
    return subprocess.run([sys.executable, str(ROOT / "ddp.py"), "--no_cuda", "--model", "whisper-tiny", "--no_tensorboard", "--output_dir",
                           str(tmp_path / "out"), "--save_steps", "0", "--logging_steps", "1", "--per_gpu_train_batch_size", "2",
                           "--dataset_size", "8", *extra], capture_output=True, text=True, cwd=tmp_path, timeout=900)


@pytest.mark.parametrize("flags,message", [(["--pack", "--min_seq_len", "8", "--seq_len", "64"], "--pack does not apply"),
                                           (["--seq_len", "512"], "at most 448")], ids=["pack", "seq_len"])
def test_cli_rejects(tmp_path, flags, message):
    from b200ddp.engine import cli
    args = cli.build_parser().parse_args(["--no_tensorboard", "--output_dir", str(tmp_path / "out"), "--model", "whisper-tiny", "--no_cuda",
                                          *flags])
    with pytest.raises(ValueError, match=message):
        cli.setup(args)


def test_ddp_py_trains_whisper_tiny_on_the_cpu(tmp_path):
    proc = _cli("--seq_len", "64", "--max_steps", "3", "--min_seq_len", "16", tmp_path=tmp_path)
    assert proc.returncode == 0, proc.stderr[-3000:]
    assert "Finished training." in proc.stdout + proc.stderr
