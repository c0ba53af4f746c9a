#!/usr/bin/env python
"""A model's training step: this package against torchvision or transformers, alternated in one call.

  python bench/model_step.py --model M[,M...] [--batch B] [--seq_len S] [--min_seq_len N] [--steps T] [--rounds R]
                             [--baseline_batch B] [--baseline_seq_len S] [--baseline_steps T] [--clips C] [--out rows.json]

Every run is a fresh process.  A native run is
  python ddp.py --model M --fp16 --optimizer adamw --per_gpu_train_batch_size B [--seq_len S] --max_steps T
  --logging_steps T/2 --save_steps 0 --no_tensorboard --output_dir TMP/out --lr 1e-4 [--min_seq_len N] [flags]
(bf16 weights, fp32 masters, the native kernels; --cuda_graph captures one CUDA graph per step), fed from pinned host
memory.  A baseline run trains the same preset under bf16 autocast with torch.optim.AdamW(fused=True) on one
device-resident batch of the same kind of data, so it pays no host-to-device copy.  ms/step is the mean over the second
half of the steps, from CUDA events (the trainer's own timer for ddp.py).  Peak memory is torch's max_memory_allocated.
The losses are not comparable: ddp.py reports the average over its steps on the synthetic set, a baseline its last loss
on its one batch.  Models run in the order given, each one's rows complete before the next; the defaults are each
model's own, and --batch, --seq_len, --steps and --rounds override them.  The card's name and power limit are read in
the same call.  Writes only under a temporary directory (and --out).

What each model runs per round, in this order (image models pass no --seq_len):
  vit-b-16        native graph, native eager, torchvision.models.vit_b_16; TFLOP/s from torchvision's count
  swin-t          the same with torchvision's SwinTransformer on swin_t's arguments and stochastic_depth_prob=0.0
                  (swin_t() itself fixes 0.2), channels_last input
  convnext-tiny   the same with torchvision.models.convnext_tiny(stochastic_depth_prob=0.0), channels_last model and input
  clip-vit-b-*    native graph, native eager, transformers.CLIPModel with return_loss=True; one GPU, so the features'
                  all-gather of a multi-GPU run is not measured
  bart-*          native graph, native eager, transformers.BartForConditionalGeneration (dropout 0) with attention_mask
                  and labels; targets are --seq_len tokens (or uniform in [--min_seq_len, --seq_len]) and sources about
                  80 % of that, right-padded, so both sides hold padding
  t5-*            the same with transformers.T5ForConditionalGeneration on span-corruption pairs; sources are --seq_len
                  tokens (or uniform in [--min_seq_len, --seq_len]), targets about a fifth of that, right-padded to a
                  multiple of 128
  mamba*          native fixed rows, --min_seq_len 256, --min_seq_len 256 --pack and --fused_lm_loss, each graph then
                  eager; tokens/s counts every row position, padding included.  mamba-130m adds a native fixed graph
                  run and transformers' MambaForCausalLM at --baseline_batch x --baseline_seq_len: without mamba_ssm and
                  causal_conv1d that runs ``slow_forward``, a Python loop over the sequence, so it is measured small
  whisper-*       first the log-mel front end alone (below), then native graph, native eager and
                  transformers.WhisperForConditionalGeneration (dropout 0) on features computed once beforehand, so its
                  step excludes the front end that the native steps include
Whisper's front end alone, on --clips clips in one batch: ops.log_mel_spectrogram (bf16 out) against the feature
extractor's _torch_extract_fbank_features on the same GPU (its host-to-device copy of the fp32 waveforms and copy back
included, as that is how it is called), both from CUDA-synchronised host clocks over 10 calls after warm-up, and the
numpy feature extractor per clip on the host."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASELINE = "baseline"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unknown"


# ------------------------------------------------------------------------------------------------ baselines
# Each returns the model on ``dev`` and a closure computing one step's loss on its one device-resident batch.

def _image_loss(model, batch, dev, channels_last, size=224):
    import torch
    import torch.nn.functional as F
    x = torch.randn(batch, 3, size, size, device=dev)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device=dev)
    return model, lambda: F.cross_entropy(model(x), y)


def vit_baseline(name, batch, seq_len, min_len, dev):
    import torchvision
    return _image_loss(torchvision.models.vit_b_16().to(dev), batch, dev, channels_last=False)


def swin_baseline(name, batch, seq_len, min_len, dev):
    from torchvision.models.swin_transformer import SwinTransformer
    model = SwinTransformer(patch_size=[4, 4], embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=[7, 7],
                            stochastic_depth_prob=0.0).to(dev)
    return _image_loss(model, batch, dev, channels_last=True)


def convnext_baseline(name, batch, seq_len, min_len, dev):
    import torch
    import torchvision
    model = torchvision.models.convnext_tiny(stochastic_depth_prob=0.0).to(dev, memory_format=torch.channels_last)
    return _image_loss(model, batch, dev, channels_last=True)


def clip_baseline(name, batch, seq_len, min_len, dev):
    import transformers
    from b200ddp.data import SyntheticImageText
    config = transformers.CLIPConfig()
    config.vision_config.patch_size = int(name.rsplit("-", 1)[1])
    model = transformers.CLIPModel(config).to(dev)
    pairs = SyntheticImageText(samples=batch, batch=batch)
    x, ids = pairs.X.to(dev), pairs.Y.to(dev)
    return model, lambda: model(input_ids=ids, pixel_values=x, return_loss=True).loss


def _seq2seq_loss(model, pairs, dev):
    x, y = pairs.X.to(dev), pairs.Y.to(dev)
    return model, lambda: model(input_ids=x, attention_mask=(x != 0).long(), labels=y).loss


def bart_baseline(name, batch, seq_len, min_len, dev):
    import transformers
    from b200ddp.data import SyntheticDenoising
    kw = dict(dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, pad_token_id=0)
    if name == "bart-large":
        kw.update(d_model=1024, encoder_layers=12, decoder_layers=12, encoder_attention_heads=16, decoder_attention_heads=16,
                  encoder_ffn_dim=4096, decoder_ffn_dim=4096)
    model = transformers.BartForConditionalGeneration(transformers.BartConfig(**kw)).to(dev)
    return _seq2seq_loss(model, SyntheticDenoising(samples=batch, seq_len=seq_len, min_len=min_len), dev)


def t5_baseline(name, batch, seq_len, min_len, dev):
    import transformers
    from b200ddp.data import SyntheticSpanCorruption
    from b200ddp.models.t5 import T5_BASE, T5_SMALL
    c = {"t5-small": T5_SMALL, "t5-base": T5_BASE}[name]
    cfg = transformers.T5Config(vocab_size=c.vocab_size, d_model=c.d_model, d_kv=c.d_kv, d_ff=c.d_ff, num_layers=c.num_layers,
                                num_decoder_layers=c.num_decoder_layers, num_heads=c.num_heads, feed_forward_proj="relu",
                                dropout_rate=0.0, pad_token_id=0, decoder_start_token_id=0, eos_token_id=1)
    model = transformers.T5ForConditionalGeneration(cfg).to(dev)
    return _seq2seq_loss(model, SyntheticSpanCorruption(samples=batch, seq_len=seq_len, min_len=min_len), dev)


def mamba_baseline(name, batch, seq_len, min_len, dev):
    import torch
    import torch.nn.functional as F
    import transformers
    cfg = transformers.MambaConfig(hidden_size=768, num_hidden_layers=24, vocab_size=50280, layer_norm_epsilon=1e-5)
    model = transformers.MambaForCausalLM(cfg).to(dev).train()
    ids = torch.randint(1, 50280, (batch, seq_len + 1), device=dev)
    # each step's fp32 logits stay referenced until the next step's forward returns, so the peak memory counts one
    # stale [B, S, V] logits tensor, as the README's recorded baseline numbers do
    last = []

    def loss():
        logits = model(ids[:, :-1]).logits
        last[:] = [logits]
        return F.cross_entropy(logits.float().reshape(-1, logits.shape[-1]), ids[:, 1:].reshape(-1))
    return model, loss


WHISPER_PRESETS = {"whisper-tiny": (384, 4, 6, 1536), "whisper-base": (512, 6, 8, 2048), "whisper-small": (768, 12, 12, 3072)}


def whisper_baseline(name, batch, seq_len, min_len, dev):
    import numpy as np
    import torch
    import transformers
    from b200ddp.data import SyntheticSpeech
    d, layers, heads, ffn = WHISPER_PRESETS[name]
    cfg = transformers.WhisperConfig(d_model=d, encoder_layers=layers, decoder_layers=layers, encoder_attention_heads=heads,
                                     decoder_attention_heads=heads, encoder_ffn_dim=ffn, decoder_ffn_dim=ffn, dropout=0.0,
                                     attention_dropout=0.0, activation_dropout=0.0)
    model = transformers.WhisperForConditionalGeneration(cfg).to(dev)
    pairs = SyntheticSpeech(samples=batch, seq_len=seq_len, min_len=min_len)
    fe = transformers.WhisperFeatureExtractor()
    x = torch.from_numpy(fe._torch_extract_fbank_features((pairs.X.numpy() / 32768.0).astype(np.float32), "cuda")).to(dev)
    y = pairs.Y.to(dev)
    return model, lambda: model(input_features=x, labels=y).loss


def frontend_run(clips):
    import time

    import numpy as np
    import torch
    import transformers
    sys.path.insert(0, ROOT)
    from b200ddp.data import SyntheticSpeech
    from b200ddp.ops import log_mel_spectrogram, whisper_mel_filters
    dev = torch.device("cuda", 0)
    wave = SyntheticSpeech(samples=clips, seq_len=64, min_len=16).X
    host = (wave.numpy() / 32768.0).astype(np.float32)
    fe = transformers.WhisperFeatureExtractor()
    wave_d, filters = wave.to(dev), whisper_mel_filters().to(dev, torch.float32)

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps * 1e3
    native = timed(lambda: log_mel_spectrogram(wave_d, filters, torch.bfloat16), 10)
    hf_gpu = timed(lambda: fe._torch_extract_fbank_features(host, "cuda"), 10)
    t0 = time.perf_counter()
    per = min(clips, 4)
    for i in range(per):
        fe(host[i], sampling_rate=16000, return_tensors="np")
    numpy_ms = (time.perf_counter() - t0) / per * 1e3
    return {"clips": clips, "native_ms": native, "transformers_torch_gpu_ms": hf_gpu, "numpy_host_ms_per_clip": numpy_ms}


# ------------------------------------------------------------------------------------------------ the table

GRAPH_EAGER = [("native graph", ["--cuda_graph"]), ("native eager", [])]
VS_TRANSFORMERS = GRAPH_EAGER + [("transformers", BASELINE)]
IMAGE = dict(batch=64, seq_len=None, steps=40, rounds=2, rate="images_per_s", runs=GRAPH_EAGER + [("torchvision", BASELINE)])
CLIP = dict(batch=256, seq_len=None, steps=40, rounds=2, rate="pairs_per_s", baseline=clip_baseline, runs=VS_TRANSFORMERS)
BART = dict(batch=16, seq_len=512, steps=40, rounds=2, rate="pairs_per_s", baseline=bart_baseline, runs=VS_TRANSFORMERS)
T5 = dict(BART, batch=32, baseline=t5_baseline)
WHISPER = dict(batch=16, seq_len=256, steps=30, rounds=2, rate="pairs_per_s", baseline=whisper_baseline, frontend=True,
               runs=VS_TRANSFORMERS)


def mamba_entry(name, **kw):
    runs = [(f"native {name} {mode} {graph}", flags + (["--cuda_graph"] if graph == "graph" else []))
            for mode, flags in (("fixed", []), ("min_seq_len 256", ["--min_seq_len", "256"]),
                                ("pack", ["--min_seq_len", "256", "--pack"]), ("fused_lm_loss", ["--fused_lm_loss"]))
            for graph in ("graph", "eager")]
    return dict(batch=8, seq_len=2048, steps=30, rounds=1, rate="tokens_per_s", runs=runs, **kw)


MODELS = {
    # 6.7 TFLOP per step at batch 64: 3 (forward + backward) x 2 x 17.56 G multiply-adds per image (torchvision's count)
    "vit-b-16": dict(IMAGE, flop=3 * 2 * 17.56e9, baseline=vit_baseline),
    # 1.72 TFLOP per step at batch 64: 3 (forward + backward) x 2 x 4.491 G multiply-adds per image (torchvision's count)
    "swin-t": dict(IMAGE, flop=3 * 2 * 4.491e9, baseline=swin_baseline),
    # 1.71 TFLOP per step at batch 64: 3 (forward + backward) x 2 x 4.456 G multiply-adds per image (torchvision's count)
    "convnext-tiny": dict(IMAGE, flop=3 * 2 * 4.456e9, baseline=convnext_baseline),
    "clip-vit-b-32": CLIP,
    "clip-vit-b-16": CLIP,
    "bart-base": BART,
    "bart-large": BART,
    "t5-small": T5,
    "t5-base": T5,
    # the native runs at the slow baseline's size keep --steps; only the baseline takes --baseline_steps
    "mamba-130m": mamba_entry("mamba-130m", baseline=mamba_baseline, baseline_size=(8, 256, 6), baseline_runs=[
        ("native fixed graph", ["--cuda_graph"]),
        ("transformers MambaForCausalLM slow_forward, bf16 autocast, fused AdamW", BASELINE)]),
    "mamba-370m": mamba_entry("mamba-370m"),
    "mamba2-130m": mamba_entry("mamba2-130m"),
    "mamba2-370m": mamba_entry("mamba2-370m"),
    "whisper-tiny": WHISPER,
    "whisper-base": WHISPER,
    "whisper-small": WHISPER,
}


# ------------------------------------------------------------------------------------------------ the runs

def per_step(rate, batch, seq_len):
    """What one step processes in the units of ``rate``."""
    return batch * seq_len if rate == "tokens_per_s" else batch


def native_argv(model, batch, seq_len, min_seq_len, steps, flags, tmp):
    argv = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", model, "--fp16", "--optimizer", "adamw",
            "--per_gpu_train_batch_size", str(batch)]
    if seq_len is not None:
        argv += ["--seq_len", str(seq_len)]
    argv += ["--max_steps", str(steps), "--logging_steps", str(steps // 2), "--save_steps", "0", "--no_tensorboard",
             "--output_dir", os.path.join(tmp, "out"), "--lr", "1e-4"]
    if min_seq_len is not None:
        argv += ["--min_seq_len", str(min_seq_len)]
    return argv + flags


def parse_finished(line, rate, batch, seq_len):
    """The trainer's ``Finished training.`` log line as a row; None for a value the line lacks."""
    def num(key):
        m = re.search(rf"{key}=([-\d.e]+)", line)
        return float(m.group(1)) if m else None
    ms = num("ms_per_step")
    if rate == "tokens_per_s":
        per_s = per_step(rate, batch, seq_len) / ms * 1e3 if ms else None
    else:
        per_s = num("samples_per_s")
    return {"ms_per_step": ms, rate: per_s, "peak_mem_gb": num("peak_mem_gb"), "average_loss": num("average_loss")}


def native_run(argv, tmp):
    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
    text = proc.stdout + proc.stderr
    line = next((ln for ln in text.splitlines() if "Finished training." in ln), None)
    if proc.returncode != 0 or line is None:
        raise RuntimeError(f"ddp.py failed ({proc.returncode}):\n{text[-4000:]}")
    return line


def baseline_run(model, batch, seq_len, min_len, steps):
    import torch
    sys.path.insert(0, ROOT)
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    rate = MODELS[model]["rate"]
    net, step_loss = MODELS[model]["baseline"](model, batch, seq_len, min_len, dev)
    opt = torch.optim.AdamW(net.parameters(), lr=1e-4, fused=True)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            loss = step_loss()
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    half = steps // 2
    ms = events[half - 1].elapsed_time(events[-1]) / (steps - half)
    return {"ms_per_step": ms, rate: per_step(rate, batch, seq_len) / ms * 1e3,
            "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "last_loss": float(loss)}


def baseline_subprocess(model, batch, seq_len, min_len, steps, tmp):
    """``baseline_run`` in a fresh process, so it shares no allocator or compiled state with the call."""
    argv = [sys.executable, os.path.abspath(__file__), "--baseline_only", "--model", model, "--batch", str(batch),
            "--steps", str(steps)]
    if seq_len is not None:
        argv += ["--seq_len", str(seq_len)]
    if min_len is not None:
        argv += ["--min_seq_len", str(min_len)]
    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
    if proc.returncode != 0:
        raise RuntimeError(f"baseline run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
    return json.loads(proc.stdout.strip().splitlines()[-1])


def sizes(model, args):
    """batch, seq_len, steps and rounds: the model's defaults unless the command line sets them."""
    e = MODELS[model]
    return [e[k] if getattr(args, k) is None else getattr(args, k) for k in ("batch", "seq_len", "steps", "rounds")]


def plan(model, args, tmp):
    """Every run of ``model``, in order: dicts of round, run label, batch, seq_len, steps and the ddp.py argv, or
    BASELINE for a baseline run."""
    e = MODELS[model]
    batch, seq_len, steps, rounds = sizes(model, args)
    groups = [(batch, seq_len, steps, e["runs"])]
    if "baseline_size" in e:
        given = (args.baseline_batch, args.baseline_seq_len, args.baseline_steps)
        groups.append((*(d if a is None else a for d, a in zip(e["baseline_size"], given)), e["baseline_runs"]))
    return [dict(round=r, run=label, batch=b, seq_len=s,
                 steps=t if flags == BASELINE else steps,
                 argv=BASELINE if flags == BASELINE else native_argv(model, b, s, args.min_seq_len, steps, flags, tmp))
            for r in range(rounds) for b, s, t, runs in groups for label, flags in runs]


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="A model's training step: this package against torchvision or transformers.")
    ap.add_argument("--model", type=str, required=True, help="comma-separated: " + ", ".join(MODELS))
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--seq_len", type=int, default=None)
    ap.add_argument("--min_seq_len", type=int, default=None)
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--rounds", type=int, default=None)
    ap.add_argument("--baseline_batch", type=int, default=None, help="mamba-130m's transformers run")
    ap.add_argument("--baseline_seq_len", type=int, default=None, help="mamba-130m's transformers run")
    ap.add_argument("--baseline_steps", type=int, default=None, help="mamba-130m's transformers run")
    ap.add_argument("--clips", type=int, default=64, help="Whisper's front end")
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--baseline_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args(argv)
    unknown = [m for m in args.model.split(",") if m not in MODELS]
    if unknown:
        ap.error(f"unknown --model {unknown}; choose from {', '.join(MODELS)}")
    return args


def main():
    args = parse_args()
    if args.baseline_only:
        print(json.dumps(baseline_run(args.model, args.batch, args.seq_len, args.min_seq_len, args.steps)), flush=True)
        return
    gpu = card()
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for model in args.model.split(","):
            e = MODELS[model]
            if e.get("frontend"):
                rows.append(dict(frontend_run(args.clips), run="front end", card=gpu))
                print(json.dumps(rows[-1]), flush=True)
            batch, seq_len, steps, _ = sizes(model, args)
            print(f"{model} batch {batch}, seq_len {seq_len}, min_seq_len {args.min_seq_len}, {steps} steps, on {gpu}",
                  flush=True)
            for p in plan(model, args, tmp):
                if p["argv"] == BASELINE:
                    res = baseline_subprocess(model, p["batch"], p["seq_len"], args.min_seq_len, p["steps"], tmp)
                else:
                    res = parse_finished(native_run(p["argv"], tmp), e["rate"], p["batch"], p["seq_len"])
                res.update(run=p["run"], round=p["round"], model=model, batch=p["batch"], seq_len=p["seq_len"],
                           min_seq_len=args.min_seq_len, card=gpu)
                if "flop" in e:
                    res["tflops"] = e["flop"] * p["batch"] / res["ms_per_step"] / 1e9 if res["ms_per_step"] else None
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
