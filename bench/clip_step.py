#!/usr/bin/env python
"""CLIP-ViT-B/32 training step: this package against transformers' CLIPModel, alternated in one call.

  python bench/clip_step.py [--model clip-vit-b-32] [--batch 256] [--steps 40] [--rounds 2] [--out clip_step.json]

Per round, three runs in fresh processes, in this order:
  native graph   python ddp.py --model clip-vit-b-32 --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size B
                 --max_steps S --logging_steps S/2   (bf16 weights, fp32 masters, the native kernels, one CUDA graph per step)
  native eager   the same without --cuda_graph
  transformers   transformers.CLIPModel (the same preset) under bf16 autocast, torch.optim.AdamW(fused=True),
                 return_loss=True
ms/step is the mean over the second half of the steps, from CUDA events (the trainer's own timer for ddp.py).  ddp.py
feeds its synthetic image-caption pairs from pinned host memory through the one-kernel input transform; the transformers
run trains on one device-resident batch of the same kind of pairs, so it pays no host-to-device copy.  Peak memory is
torch's max_memory_allocated.  One process, one GPU: the features' all-gather of a multi-GPU run is not measured.  The
losses are not comparable: ddp.py reports the average over its steps on the synthetic set, the transformers run its last
loss on its one batch.  The card's name and power limit are read in the same call.  Writes only under a temporary
directory (and --out)."""
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


def transformers_run(model_name, batch, steps):
    import torch
    import transformers
    sys.path.insert(0, ROOT)
    from b200ddp.data import SyntheticImageText
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    config = transformers.CLIPConfig()
    config.vision_config.patch_size = int(model_name.rsplit("-", 1)[1])
    model = transformers.CLIPModel(config).to(dev)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    pairs = SyntheticImageText(samples=batch, batch=batch)
    x, ids = pairs.X.to(dev), pairs.Y.to(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            loss = model(input_ids=ids, pixel_values=x, return_loss=True).loss
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


def native_run(model_name, batch, steps, graph, tmp):
    argv = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", model_name, "--fp16", "--optimizer", "adamw",
            "--per_gpu_train_batch_size", str(batch), "--max_steps", str(steps), "--logging_steps", str(steps // 2),
            "--save_steps", "0", "--no_tensorboard", "--output_dir", os.path.join(tmp, "out"), "--lr", "1e-4"]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", type=str, default="clip-vit-b-32", choices=["clip-vit-b-32", "clip-vit-b-16"])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--transformers_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.transformers_only:
        print(json.dumps(transformers_run(args.model, args.batch, args.steps)), flush=True)
        return
    gpu = card()
    print(f"{args.model} batch {args.batch}, {args.steps} steps, on {gpu}", flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for name in ("native graph", "native eager", "transformers"):
                if name == "transformers":
                    proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--transformers_only", "--model", args.model,
                                           "--batch", str(args.batch), "--steps", str(args.steps)], capture_output=True, text=True,
                                          cwd=tmp)
                    if proc.returncode != 0:
                        raise RuntimeError(f"transformers run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
                    res = json.loads(proc.stdout.strip().splitlines()[-1])
                else:
                    res = native_run(args.model, args.batch, args.steps, name == "native graph", tmp)
                res.update(run=name, round=r, model=args.model, batch=args.batch, card=gpu)
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
