"""Whisper on the H100: the native log-mel front end against the fp64 reference element by element, the stem gathers
bitwise against their references, whisper-tiny in bf16 against its fp32 path (the CPU references), and ``ddp.py``-style
training of whisper-tiny under a CUDA graph, whose losses fall, equal the eager run's bitwise, and stay close with the fused
LM-head loss."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from b200ddp.data import SyntheticSpeech
from b200ddp.models import build_model
from b200ddp.ops import (encoder_rows, frame_patches, frame_patches_reference, log_mel_spectrogram, log_mel_spectrogram_reference, mel_patches,
                         mel_patches_reference, whisper_mel_filters)
from b200ddp.utils.precision import to_mixed_bf16

pytestmark = pytest.mark.gpu


def _clips():
    """Silent, full-scale, nonzero first and last samples, and speech-like tones with a silent tail."""
    g = torch.Generator().manual_seed(0)
    t = torch.arange(480000, dtype=torch.float64) / 16000
    silent = torch.zeros(480000, dtype=torch.int16)
    full = torch.where(torch.rand(480000, generator=g) < 0.5, -32768, 32767).to(torch.int16)
    edges = (3000 * torch.sin(2 * math.pi * 440 * t)).round().to(torch.int16)
    edges[0], edges[-1] = 20000, -20000
    speech = (6000 * torch.sin(2 * math.pi * (200 + 50 * (t * 4).floor()) * t) + 300 * torch.randn(480000, generator=g, dtype=torch.float64))
    speech[250000:] = 0
    return torch.stack([silent, full, edges, speech.round().clamp(-32768, 32767).to(torch.int16)])


def test_log_mel_matches_the_fp64_reference():
    wave = _clips()
    filters = whisper_mel_filters()
    want = log_mel_spectrogram_reference(wave, filters)
    w = wave.cuda()
    f32 = log_mel_spectrogram(w, filters, torch.float32)
    err = (f32.double().cpu() - want).abs()
    print(f"\nlog-mel fp32 max |err| vs fp64 per clip: {[float(e.max()) for e in err]}")
    assert float(err.max()) <= 1e-4
    assert bool((f32[0] == -1.5).all())                              # silence: L = -10 everywhere
    bf = log_mel_spectrogram(w, filters, torch.bfloat16)
    assert bf.dtype == torch.bfloat16 and torch.equal(bf, f32.to(torch.bfloat16))
    assert torch.equal(log_mel_spectrogram(w, filters, torch.float32), f32)
    out = torch.empty(4, 80, 3000, dtype=torch.bfloat16, device="cuda")
    assert log_mel_spectrogram(w, filters, torch.bfloat16, out=out).data_ptr() == out.data_ptr() and torch.equal(out, bf)


def test_stem_gathers_are_exact():
    g = torch.Generator().manual_seed(1)
    B, T, d = 3, 3000, 384
    S = encoder_rows(T)
    feats = torch.randn(B, 80, T, generator=g).to(torch.bfloat16).cuda()
    p1 = mel_patches(feats)
    assert torch.equal(p1, mel_patches_reference(feats)) and torch.equal(mel_patches(feats), p1)
    h1 = torch.randn(B * T, d, generator=g).to(torch.bfloat16).cuda().requires_grad_(True)
    p2 = frame_patches(h1, T, S)
    assert torch.equal(p2, frame_patches_reference(h1.detach(), T, S)) and torch.equal(frame_patches(h1, T, S), p2)
    dp2 = torch.randn(B * S, 3 * d, generator=g).to(torch.bfloat16).cuda()
    dp2.view(B, S, 3 * d)[:, T // 2:] = float("nan")                 # the padding rows are never read
    p2.backward(dp2)
    taps = dp2.double().view(B, S, 3, d)
    want = torch.zeros(B, T, d, dtype=torch.float64, device="cuda")
    s = torch.arange(T, device="cuda")
    for j in range(3):
        l2 = s + 1 - j
        ok = (l2 >= 0) & (l2 % 2 == 0) & (l2 // 2 < T // 2)
        want[:, ok] += taps[:, (l2[ok] // 2), j]
    assert torch.equal(h1.grad, want.to(torch.bfloat16).view(B * T, d))
    first = h1.grad.clone()
    h1.grad = None
    frame_patches(h1, T, S).backward(dp2)
    assert torch.equal(h1.grad, first)


def test_native_bf16_whisper_tiny_matches_the_fp32_path():
    """Loss within 2 % and every parameter gradient within 5 % (relative norm) of the fp32 CPU path, on the same features."""
    torch.manual_seed(0)
    ref = build_model("whisper-tiny")
    with torch.no_grad():                                            # away from zero biases
        for n, p in ref.named_parameters():
            if n.endswith("bias") and "layer_norm" not in n:
                p.normal_(0.0, 0.02)
    native = to_mixed_bf16(copy.deepcopy(ref).cuda())
    ds = SyntheticSpeech(samples=2, seq_len=128, min_len=40)
    feats = log_mel_spectrogram(ds.X.cuda(), whisper_mel_filters(), torch.bfloat16)

    def loss(model, x, y):
        logits = model(x, y)
        return F.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), y.reshape(-1))
    lr = loss(ref, feats.float().cpu(), ds.Y)
    ln = loss(native, feats, ds.Y.cuda())
    assert abs(float(ln.detach()) - float(lr.detach())) < 2e-2 * float(lr.detach())
    lr.backward()
    ln.backward()
    # q_bias and v_bias are compared as the one fused bias q | 0 | v they form, as BART's qkv.bias is
    grads = dict(native.named_parameters())
    pairs = {}
    for n, p in ref.named_parameters():
        if p.requires_grad:
            key = n[:-len("q_bias")] + "bias" if n.endswith(("q_bias", "v_bias")) else n
            pairs.setdefault(key, []).append((grads[n].grad.float().cpu().flatten(), p.grad.flatten()))
    for n, gs in pairs.items():
        g, want = torch.cat([a for a, _ in gs]), torch.cat([b for _, b in gs])
        rel = float((g - want).norm() / want.norm().clamp(min=1e-8))
        assert rel < 5e-2, (n, rel)


def _train(tmp_path, extra):
    """What `python ddp.py --model whisper-tiny --fp16 --optimizer adamw --per_gpu_train_batch_size 8 --seq_len 256
    --min_seq_len 32 --max_steps 20 [extra]` runs; returns every step's loss."""
    from b200ddp.data import SyntheticTokens
    from b200ddp.engine import cli
    from b200ddp.engine.trainer import Trainer
    argv = ["--model", "whisper-tiny", "--fp16", "--optimizer", "adamw", "--per_gpu_train_batch_size", "8", "--seq_len", "256",
            "--min_seq_len", "32", "--max_steps", "20", "--logging_steps", "1", "--dataset_size", "64", "--lr", "1e-3",
            "--warmup_steps", "2", "--save_steps", "0", "--no_tensorboard", "--output_dir", str(tmp_path / "out"), *extra]
    args = cli.build_parser().parse_args(argv)
    cli.setup(args)
    kwargs = {"pad_token_id": SyntheticTokens.PAD_ID}
    if args.fused_lm_loss:
        kwargs["fused_lm_loss"] = True
    trainer = Trainer(args, build_model("whisper-tiny", **kwargs), cli.log)
    sums = []
    read = trainer.step_fn.read_loss_sum
    trainer.step_fn.read_loss_sum = lambda: sums.append(read()) or sums[-1]
    trainer.train()
    assert (trainer.step_fn.graph is not None) == args.cuda_graph
    return [b - a for a, b in zip([0.0] + sums[:-1], sums)][:20]


def test_training_under_a_cuda_graph_falls_and_equals_eager_bitwise(tmp_path, capsys):
    graph = _train(tmp_path / "g", ["--cuda_graph"])
    eager = _train(tmp_path / "e", [])
    with capsys.disabled():
        print(f"\nwhisper-tiny losses on {torch.cuda.get_device_name()}: {[round(v, 4) for v in graph[::4]]}; "
              f"eager bitwise equal: {graph == eager}")
    assert all(math.isfinite(v) for v in graph)
    assert sum(graph[-4:]) / 4 < graph[0]
    assert graph == eager


def test_fused_lm_loss_matches_the_unfused_loss(tmp_path):
    """The fused head's losses stay within 2e-2 of the unfused ones over 20 steps (bf16 logits against the fused
    kernel's fp32 log-sum-exp)."""
    fused = _train(tmp_path / "f", ["--cuda_graph", "--fused_lm_loss"])
    plain = _train(tmp_path / "p", ["--cuda_graph"])
    assert max(abs(a - b) for a, b in zip(fused, plain)) < 2e-2, (fused, plain)
