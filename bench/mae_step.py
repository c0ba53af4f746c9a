#!/usr/bin/env python
"""ViT-MAE's training step: this package against transformers, and against the native ViT-B/16 step, alternated in one call.

  python bench/mae_step.py [--model vit-mae-base] [--batch 64] [--steps 30] [--rounds 2] [--out rows.json]

Every run is a fresh process.  Per round, in this order:
  native graph    ddp.py --model M --fp16 --optimizer adamw --cuda_graph (``bench/model_step.py``'s command line)
  native eager    the same without --cuda_graph
  transformers    ViTMAEForPreTraining (ViTMAEConfig defaults, SDPA attention) under bf16 autocast with
                  torch.optim.AdamW(fused=True), on one device-resident batch of random images, fresh noise every step
  vit-b-16 graph  the native ViT-B/16 step at the same batch: every patch through a 12-layer encoder, so MAE's encoder on a
                  quarter of the patches plus its 8-layer decoder can be read against it
ms/step is the mean over the second half of the steps (CUDA events; the trainer's own timer for ddp.py), peak memory
torch's max_memory_allocated.  The card's name and power limit are read in the same call.  Writes only under a temporary
directory (and --out)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from model_step import card, native_argv, native_run, parse_finished  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def baseline_run(model, batch, steps):
    import torch
    import transformers
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    config = transformers.ViTMAEConfig() if model == "vit-mae-base" else transformers.ViTMAEConfig(
        hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096)
    config._attn_implementation = "sdpa"
    net = transformers.ViTMAEForPreTraining(config).to(dev)
    opt = torch.optim.AdamW(net.parameters(), lr=1e-4, fused=True)
    x = torch.randn(batch, 3, 224, 224, device=dev)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            loss = net(pixel_values=x).loss
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    half = steps // 2
    ms = events[half - 1].elapsed_time(events[-1]) / (steps - half)
    return {"ms_per_step": ms, "samples_per_s": batch / ms * 1e3, "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30,
            "last_loss": float(loss)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--model", default="vit-mae-base", choices=["vit-mae-base", "vit-mae-large"])
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--baseline_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.baseline_only:
        print(json.dumps(baseline_run(args.model, args.batch, args.steps)), flush=True)
        return
    gpu = card()
    print(f"{args.model} batch {args.batch}, {args.steps} steps, on {gpu}", flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        runs = [("native graph", args.model, ["--cuda_graph"]), ("native eager", args.model, []),
                ("transformers ViTMAEForPreTraining, SDPA, bf16 autocast, fused AdamW", None, None),
                ("native vit-b-16 graph", "vit-b-16", ["--cuda_graph"])]
        for r in range(args.rounds):
            for label, model, flags in runs:
                if model is None:
                    argv = [sys.executable, os.path.abspath(__file__), "--baseline_only", "--model", args.model, "--batch",
                            str(args.batch), "--steps", str(args.steps)]
                    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
                    if proc.returncode != 0:
                        raise RuntimeError(f"baseline run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
                    res = json.loads(proc.stdout.strip().splitlines()[-1])
                else:
                    argv = native_argv(model, args.batch, None, None, args.steps, flags, tmp)
                    res = parse_finished(native_run(argv, tmp), "samples_per_s", args.batch, None)
                res.update(run=label, round=r, model=model or args.model, batch=args.batch, card=gpu)
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
