#!/usr/bin/env python
"""Experimental wgmma 3x3 convolution forward vs cuDNN on the ResNet-50 (batch 32) 3x3 shapes.

  python bench/conv_bench.py [--iters 20]

CUDA events, 3 warm-up launches, a 256 MB write between timed launches (L2 flush), median of `iters`."""
import argparse
import statistics

import torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from b200ddp import _ext
    C = _ext.get()
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = True
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timeit(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(args.iters):
            flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return statistics.median(ts)

    for (n, c, h, w, k) in [(32, 64, 56, 56, 64), (32, 128, 28, 28, 128), (32, 256, 14, 14, 256), (32, 512, 7, 7, 512)]:
        x = torch.randn(n, c, h, w, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        wt = (torch.randn(k, c, 3, 3, device=dev) * 0.05).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        ours = timeit(lambda: C.conv3x3_fwd(x, wt))
        lib = timeit(lambda: torch.nn.functional.conv2d(x, wt, padding=1))
        err = float((C.conv3x3_fwd(x, wt).float() - torch.nn.functional.conv2d(x, wt, padding=1).float()).norm())
        flops = 2.0 * n * h * w * k * 9 * c
        print(f"conv3x3 {n}x{c}x{h}x{w} -> {k}: ours {ours * 1e3:8.1f} us ({flops / ours / 1e9:7.1f} TFLOP/s) | cuDNN {lib * 1e3:8.1f} us "
              f"({flops / lib / 1e9:7.1f} TFLOP/s) | ours/lib {ours / lib:5.2f} | abs diff {err:.3f}", flush=True)


if __name__ == "__main__":
    main()
