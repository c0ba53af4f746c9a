#!/usr/bin/env python
"""Mamba training step (mamba-130m by default, or --model mamba-370m, mamba2-130m, mamba2-370m, several in one call):
ms/step, tokens/s and peak memory of this package, and for mamba-130m a row for transformers' slow path.

  python bench/mamba_step.py [--model mamba-130m[,mamba2-130m]] [--batch 8] [--seq_len 2048] [--steps 30] [--out mamba_step.json]

Native runs, each a fresh process:
  python ddp.py --model MODEL --fp16 --optimizer adamw --per_gpu_train_batch_size B --seq_len S --max_steps N
  --logging_steps N/2 [--cuda_graph] with fixed rows, --min_seq_len 256, --min_seq_len 256 --pack and --fused_lm_loss
  (bf16 weights, fp32 masters, the native kernels).  ms/step is the mean over the second half of the steps (the trainer's
  own CUDA-event timer); tokens/s counts every row position, padding included.
transformers: MambaForCausalLM with mamba-130m's config under bf16 autocast, torch.optim.AdamW(fused=True), on one
device-resident batch of --hf_batch x --hf_seq_len.  Without mamba_ssm and causal_conv1d it runs ``slow_forward``, a
Python loop over the sequence, so it is measured at that smaller size, beside a native run at the same size.
Peak memory is torch's max_memory_allocated.  The card's name and power limit are read in the same call.  Writes only under
a temporary directory (and --out)."""
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


def transformers_run(batch, seq_len, steps):
    import torch
    import torch.nn.functional as F
    import transformers
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    cfg = transformers.MambaConfig(hidden_size=768, num_hidden_layers=24, vocab_size=50280, layer_norm_epsilon=1e-5)
    model = transformers.MambaForCausalLM(cfg).to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    ids = torch.randint(1, 50280, (batch, seq_len + 1), device=dev)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            logits = model(ids[:, :-1]).logits
            loss = F.cross_entropy(logits.float().reshape(-1, logits.shape[-1]), ids[:, 1:].reshape(-1))
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    half = steps // 2
    ms = events[half - 1].elapsed_time(events[-1]) / (steps - half)
    return {"ms_per_step": ms, "tokens_per_s": batch * seq_len / ms * 1e3,
            "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "last_loss": float(loss)}


def native_run(batch, seq_len, steps, flags, tmp, model="mamba-130m"):
    argv = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", model, "--fp16", "--optimizer", "adamw",
            "--per_gpu_train_batch_size", str(batch), "--seq_len", str(seq_len), "--max_steps", str(steps),
            "--logging_steps", str(steps // 2), "--save_steps", "0", "--no_tensorboard", "--output_dir", os.path.join(tmp, "out"),
            "--lr", "1e-4", *flags]
    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
    text = proc.stdout + proc.stderr
    line = next((ln for ln in text.splitlines() if "Finished training." in ln), None)
    if proc.returncode != 0 or line is None:
        raise RuntimeError(f"ddp.py failed ({proc.returncode}):\n{text[-4000:]}")

    def num(key):
        m = re.search(rf"{key}=([-\d.e]+)", line)
        return float(m.group(1)) if m else None
    ms = num("ms_per_step")
    return {"ms_per_step": ms, "tokens_per_s": batch * seq_len / ms * 1e3 if ms else None, "peak_mem_gb": num("peak_mem_gb"),
            "average_loss": num("average_loss")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", type=str, default="mamba-130m", help="comma-separated: mamba-130m, mamba-370m, mamba2-130m, mamba2-370m")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seq_len", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--hf_batch", type=int, default=8)
    ap.add_argument("--hf_seq_len", type=int, default=256)
    ap.add_argument("--hf_steps", type=int, default=6)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--transformers_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.transformers_only:
        print(json.dumps(transformers_run(args.hf_batch, args.hf_seq_len, args.hf_steps)), flush=True)
        return
    gpu = card()
    models = args.model.split(",")
    unknown = set(models) - {"mamba-130m", "mamba-370m", "mamba2-130m", "mamba2-370m"}
    if unknown:
        raise SystemExit(f"unknown --model {sorted(unknown)}")
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for model in models:
            print(f"{model} {args.batch} x {args.seq_len}, {args.steps} steps, on {gpu}", flush=True)
            runs = [(f"{mode} {graph}", flags + (["--cuda_graph"] if graph == "graph" else []))
                    for mode, flags in (("fixed", []), ("min_seq_len 256", ["--min_seq_len", "256"]),
                                        ("pack", ["--min_seq_len", "256", "--pack"]), ("fused_lm_loss", ["--fused_lm_loss"]))
                    for graph in ("graph", "eager")]
            for name, flags in runs:
                res = native_run(args.batch, args.seq_len, args.steps, flags, tmp, model)
                res.update(run=f"native {model} {name}", batch=args.batch, seq_len=args.seq_len, card=gpu)
                rows.append(res)
                print(json.dumps(res), flush=True)
        if "mamba-130m" in models:
            res = native_run(args.hf_batch, args.hf_seq_len, args.steps, ["--cuda_graph"], tmp)
            res.update(run="native fixed graph", batch=args.hf_batch, seq_len=args.hf_seq_len, card=gpu)
            rows.append(res)
            print(json.dumps(res), flush=True)
            proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--transformers_only", "--hf_batch", str(args.hf_batch),
                                   "--hf_seq_len", str(args.hf_seq_len), "--hf_steps", str(args.hf_steps)], capture_output=True, text=True,
                                  cwd=tmp)
            if proc.returncode != 0:
                raise RuntimeError(f"transformers run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
            res = json.loads(proc.stdout.strip().splitlines()[-1])
            res.update(run="transformers MambaForCausalLM slow_forward, bf16 autocast, fused AdamW", batch=args.hf_batch,
                       seq_len=args.hf_seq_len, card=gpu)
            rows.append(res)
            print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
