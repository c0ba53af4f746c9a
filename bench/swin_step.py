#!/usr/bin/env python
"""Swin-T training step: this package against torchvision, alternated in one call.

  python bench/swin_step.py [--batch 64] [--steps 40] [--rounds 2] [--out swin_step.json]

Per round, three runs in fresh processes, in this order:
  native graph   python ddp.py --model swin-t --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size B
                 --max_steps S --logging_steps S/2   (bf16 weights, fp32 masters, the native kernels, one CUDA graph per step)
  native eager   the same without --cuda_graph
  torchvision    torchvision's SwinTransformer with swin_t's arguments and stochastic_depth_prob=0.0 (swin_t() itself fixes
                 0.2) under bf16 autocast, channels_last input, torch.optim.AdamW(fused=True), F.cross_entropy
ms/step is the mean over the second half of the steps, from CUDA events (the trainer's own timer for ddp.py).  ddp.py
feeds its synthetic ImageNet batches from pinned host memory through the one-kernel input transform; the torchvision run
trains on one device-resident batch, so it pays no host-to-device copy.  Peak memory is torch's max_memory_allocated.
The losses are not comparable: ddp.py reports the average over its steps on the synthetic set, the torchvision run its
last loss on its one batch.  The card's name and power limit are read in the same call.  Writes only under a temporary directory (and --out)."""
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


def torchvision_run(batch, steps):
    import torch
    import torch.nn.functional as F
    from torchvision.models.swin_transformer import SwinTransformer
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    model = SwinTransformer(patch_size=[4, 4], embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=[7, 7],
                            stochastic_depth_prob=0.0).to(dev)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    x = torch.randn(batch, 3, 224, 224, device=dev).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device=dev)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            loss = F.cross_entropy(model(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    half = steps // 2
    ms = events[half - 1].elapsed_time(events[-1]) / (steps - half)
    return {"ms_per_step": ms, "images_per_s": batch / ms * 1e3,
            "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "last_loss": float(loss)}


def native_run(batch, steps, graph, tmp):
    argv = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", "swin-t", "--fp16", "--optimizer", "adamw",
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
    return {"ms_per_step": num("ms_per_step"), "images_per_s": num("samples_per_s"), "peak_mem_gb": num("peak_mem_gb"),
            "average_loss": num("average_loss")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--torchvision_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.torchvision_only:
        print(json.dumps(torchvision_run(args.batch, args.steps)), flush=True)
        return
    # 1.72 TFLOP per step at batch 64: 3 (forward + backward) x 2 x 4.491 G multiply-adds per image (torchvision's count)
    flop = 3 * 2 * 4.491e9 * args.batch
    gpu = card()
    print(f"Swin-T batch {args.batch}, {args.steps} steps, on {gpu}", flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for name in ("native graph", "native eager", "torchvision"):
                if name == "torchvision":
                    proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--torchvision_only", "--batch", str(args.batch),
                                           "--steps", str(args.steps)], capture_output=True, text=True, cwd=tmp)
                    if proc.returncode != 0:
                        raise RuntimeError(f"torchvision run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
                    res = json.loads(proc.stdout.strip().splitlines()[-1])
                else:
                    res = native_run(args.batch, args.steps, name == "native graph", tmp)
                res.update(run=name, round=r, batch=args.batch, card=gpu,
                           tflops=flop / res["ms_per_step"] / 1e9 if res["ms_per_step"] else None)
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
