#!/usr/bin/env python
"""Swin-V2-T's training step at 256 x 256: this package against torchvision, alternated in one call.

  python bench/swin_v2_step.py [--model swin-v2-t] [--batch 64] [--steps 40] [--rounds 2] [--out rows.json]

Every run is a fresh process.  Per round, in this order:
  native graph    ddp.py --model M --fp16 --optimizer adamw --cuda_graph (``bench/model_step.py``'s command line), which
                  trains on 256 x 256 images (the registry's image_size)
  native eager    the same without --cuda_graph
  torchvision     SwinTransformer with swin_v2_t's arguments, SwinTransformerBlockV2, PatchMergingV2 and
                  stochastic_depth_prob=0.0 (swin_v2_t() itself fixes 0.2), channels_last, under bf16 autocast with
                  torch.optim.AdamW(fused=True), on one device-resident batch of random 256 x 256 images
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
from model_step import _image_loss, card, native_argv, native_run, parse_finished  # noqa: E402

ARCH = {"swin-v2-t": (96, [2, 2, 6, 2], [3, 6, 12, 24]), "swin-v2-s": (96, [2, 2, 18, 2], [3, 6, 12, 24]),
        "swin-v2-b": (128, [2, 2, 18, 2], [4, 8, 16, 32])}


def torchvision_swin_v2(name):
    from torchvision.models import swin_transformer as tvs
    embed, depths, heads = ARCH[name]
    return tvs.SwinTransformer(patch_size=[4, 4], embed_dim=embed, depths=depths, num_heads=heads, window_size=[8, 8],
                               stochastic_depth_prob=0.0, block=tvs.SwinTransformerBlockV2, downsample_layer=tvs.PatchMergingV2)


def baseline_run(model, batch, steps):
    import torch
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    net, step_loss = _image_loss(torchvision_swin_v2(model).to(dev, memory_format=torch.channels_last), batch, dev, channels_last=True,
                                 size=256)
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
    return {"ms_per_step": ms, "samples_per_s": batch / ms * 1e3, "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30,
            "last_loss": float(loss)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--model", default="swin-v2-t", choices=sorted(ARCH))
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--baseline_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.baseline_only:
        print(json.dumps(baseline_run(args.model, args.batch, args.steps)), flush=True)
        return
    gpu = card()
    print(f"{args.model} batch {args.batch} at 256 x 256, {args.steps} steps, on {gpu}", flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        runs = [("native graph", ["--cuda_graph"]), ("native eager", []),
                ("torchvision SwinTransformer V2, channels_last, bf16 autocast, fused AdamW", None)]
        for r in range(args.rounds):
            for label, flags in runs:
                if flags is None:
                    argv = [sys.executable, os.path.abspath(__file__), "--baseline_only", "--model", args.model, "--batch",
                            str(args.batch), "--steps", str(args.steps)]
                    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
                    if proc.returncode != 0:
                        raise RuntimeError(f"baseline run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
                    res = json.loads(proc.stdout.strip().splitlines()[-1])
                else:
                    argv = native_argv(args.model, args.batch, None, None, args.steps, flags, tmp)
                    res = parse_finished(native_run(argv, tmp), "samples_per_s", args.batch, None)
                res.update(run=label, round=r, model=args.model, batch=args.batch, card=gpu)
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
