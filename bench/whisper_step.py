#!/usr/bin/env python
"""Whisper training step: this package against transformers' WhisperForConditionalGeneration, alternated in one call, and
the log-mel front end alone.

  python bench/whisper_step.py [--model whisper-small] [--batch 16] [--seq_len 256] [--min_seq_len N] [--steps 30]
                               [--rounds 2] [--clips 64] [--out whisper_step.json]

Per round, three runs in fresh processes, in this order:
  native graph   python ddp.py --model whisper-small --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size B
                 --seq_len S [--min_seq_len N] --max_steps T --logging_steps T/2   (int16 clips in, the native log-mel front
                 end, bf16 weights, fp32 masters, one CUDA graph per step)
  native eager   the same without --cuda_graph
  transformers   transformers.WhisperForConditionalGeneration (the same preset, dropout 0) under bf16 autocast,
                 torch.optim.AdamW(fused=True), on the same kind of clip / transcript pairs, its features computed once
                 beforehand (so its step excludes the front end that the native steps include)
ms/step is the mean over the second half of the steps, from CUDA events (the trainer's own timer for ddp.py).  ddp.py
feeds its clips from pinned host memory; the transformers run trains on one device-resident batch.  Peak memory is
torch's max_memory_allocated.  The losses are not comparable.

The front end alone, on --clips clips in one batch: ops.log_mel_spectrogram (bf16 out) against the feature extractor's
_torch_extract_fbank_features on the same GPU (its host-to-device copy of the fp32 waveforms and copy back included, as
that is how it is called), both from CUDA-synchronised host clocks over 10 calls after warm-up, and the numpy feature
extractor per clip on the host.  The card's name and power limit are read in the same call.  Writes only under a
temporary directory (and --out)."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unknown"


PRESETS = {"whisper-tiny": (384, 4, 6, 1536), "whisper-base": (512, 6, 8, 2048), "whisper-small": (768, 12, 12, 3072)}


def transformers_run(model_name, batch, seq_len, min_len, steps):
    import numpy as np
    import torch
    import transformers
    sys.path.insert(0, ROOT)
    from b200ddp.data import SyntheticSpeech
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    d, layers, heads, ffn = PRESETS[model_name]
    cfg = transformers.WhisperConfig(d_model=d, encoder_layers=layers, decoder_layers=layers, encoder_attention_heads=heads,
                                     decoder_attention_heads=heads, encoder_ffn_dim=ffn, decoder_ffn_dim=ffn, dropout=0.0,
                                     attention_dropout=0.0, activation_dropout=0.0)
    model = transformers.WhisperForConditionalGeneration(cfg).to(dev)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    pairs = SyntheticSpeech(samples=batch, seq_len=seq_len, min_len=min_len)
    fe = transformers.WhisperFeatureExtractor()
    x = torch.from_numpy(fe._torch_extract_fbank_features((pairs.X.numpy() / 32768.0).astype(np.float32), "cuda")).to(dev)
    y = pairs.Y.to(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            loss = model(input_features=x, labels=y).loss
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    half = steps // 2
    ms = events[half - 1].elapsed_time(events[-1]) / (steps - half)
    return {"ms_per_step": ms, "pairs_per_s": batch / ms * 1e3,
            "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "last_loss": float(loss)}


def native_run(model_name, batch, seq_len, min_len, steps, graph, tmp):
    argv = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", model_name, "--fp16", "--optimizer", "adamw",
            "--per_gpu_train_batch_size", str(batch), "--seq_len", str(seq_len), "--max_steps", str(steps), "--logging_steps",
            str(steps // 2), "--save_steps", "0", "--no_tensorboard", "--output_dir", os.path.join(tmp, "out"), "--lr", "1e-4"]
    if min_len is not None:
        argv += ["--min_seq_len", str(min_len)]
    if graph:
        argv.append("--cuda_graph")
    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
    text = proc.stdout + proc.stderr
    line = next((ln for ln in text.splitlines() if "Finished training." in ln), None)
    if proc.returncode != 0 or line is None:
        raise RuntimeError(f"ddp.py failed ({proc.returncode}):\n{text[-4000:]}")

    def num(key):
        m = re.search(rf"{key}=([-\d.e]+)", line)
        return float(m.group(1)) if m else None
    return {"ms_per_step": num("ms_per_step"), "pairs_per_s": num("samples_per_s"), "peak_mem_gb": num("peak_mem_gb"),
            "average_loss": num("average_loss")}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", type=str, default="whisper-small", choices=sorted(PRESETS))
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seq_len", type=int, default=256)
    ap.add_argument("--min_seq_len", type=int, default=None)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--transformers_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.transformers_only:
        print(json.dumps(transformers_run(args.model, args.batch, args.seq_len, args.min_seq_len, args.steps)), flush=True)
        return
    gpu = card()
    front = frontend_run(args.clips)
    front.update(run="front end", card=gpu)
    print(json.dumps(front), flush=True)
    print(f"{args.model} batch {args.batch}, seq_len {args.seq_len}, min_seq_len {args.min_seq_len}, {args.steps} steps, on {gpu}",
          flush=True)
    rows = [front]
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for name in ("native graph", "native eager", "transformers"):
                if name == "transformers":
                    extra = [] if args.min_seq_len is None else ["--min_seq_len", str(args.min_seq_len)]
                    proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--transformers_only", "--model", args.model,
                                           "--batch", str(args.batch), "--seq_len", str(args.seq_len), "--steps", str(args.steps),
                                           *extra], capture_output=True, text=True, cwd=tmp)
                    if proc.returncode != 0:
                        raise RuntimeError(f"transformers run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
                    res = json.loads(proc.stdout.strip().splitlines()[-1])
                else:
                    res = native_run(args.model, args.batch, args.seq_len, args.min_seq_len, args.steps, name == "native graph", tmp)
                res.update(run=name, round=r, model=args.model, batch=args.batch, seq_len=args.seq_len, min_seq_len=args.min_seq_len,
                           card=gpu)
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
