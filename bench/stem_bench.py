#!/usr/bin/env python
"""The strided 7x7 stem of ResNet-50 (batch 32, 224x224, bf16, channels_last): library forward / weight gradient against
this framework's wgmma path (csrc/conv_stem.cu packing + conv_wgmma.cu / conv_wgrad_wgmma.cu through the
overlapping-window tensor map).  Timing as in bench/conv_layers.py: CUDA events around the replay of a CUDA graph of
`reps` launches rotating over > 192 MB of operands, best of 3.
  python bench/stem_bench.py [--batch 32] [--reps 20] [--out stem_bench.json]"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    from b200ddp import _ext
    C = _ext.get()
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda", 0)
    n, h, w = args.batch, 224, 224
    nsets = 6      # 6 x (9.6 MB x + 51 MB dy/y) > 192 MB
    xs = [torch.randn(n, 3, h, w, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last) for _ in range(nsets)]
    dys = [torch.randn(n, 64, h // 2, w // 2, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last) for _ in range(nsets)]
    wt = (torch.randn(64, 3, 7, 7, device=dev) / 147 ** 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

    def time_rot(fn):
        for i in range(nsets):
            fn(i)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(args.reps):
                fn(i)
        g.replay(); torch.cuda.synchronize()
        best = float("inf")
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / args.reps)
        return best

    def rel(a, b):
        return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))

    res = {"batch": n}
    y_ref = F.conv2d(xs[0], wt, None, 2, 3)
    dw_ref = torch.ops.aten.convolution_backward(dys[0], xs[0], wt, None, [2, 2], [3, 3], [1, 1], False, [0, 0], 1, [False, True, False])[1]
    y, part, xp = C.stem_conv_fprop(xs[0], wt, True, True)
    torch.cuda.synchronize()
    res["relerr_fprop_vs_lib"] = rel(y, y_ref)
    for v in (0, 1):
        res[f"relerr_wgrad_variant{v}_vs_lib"] = rel(C.stem_conv_wgrad(dys[0], xp, h, w, v), dw_ref)
    xps = [C.stem_pack_input(x) for x in xs]
    w2 = C.stem_pack_weight(wt)
    res["lib_fprop_us"] = time_rot(lambda i: F.conv2d(xs[i % nsets], wt, None, 2, 3))
    res["lib_wgrad_us"] = time_rot(lambda i: torch.ops.aten.convolution_backward(dys[i % nsets], xs[i % nsets], wt, None, [2, 2], [3, 3], [1, 1], False,
                                                                               [0, 0], 1, [False, True, False]))
    res["ours_fprop_total_us (pack x + pack w + conv, resident filter)"] = time_rot(lambda i: C.stem_conv_fprop(xs[i % nsets], wt, False, True))
    res["ours_fprop_stats_total_us (+ BatchNorm statistics epilogue)"] = time_rot(lambda i: C.stem_conv_fprop(xs[i % nsets], wt, True, True))
    res["  pack_input_us"] = time_rot(lambda i: C.stem_pack_input(xs[i % nsets]))
    res["  pack_weight_us"] = time_rot(lambda i: C.stem_pack_weight(wt))
    res["  conv_kernel_resident_us"] = time_rot(lambda i: C.stem_conv_fprop_packed(xps[i % nsets], w2, h, w, False, True, False))
    res["  conv_kernel_streamed_filter_us"] = time_rot(lambda i: C.stem_conv_fprop_packed(xps[i % nsets], w2, h, w, False, False, False))
    res["  conv_kernel_resident_stats_us"] = time_rot(lambda i: C.stem_conv_fprop_packed(xps[i % nsets], w2, h, w, True, True, False))
    for v in (0, 1):
        name = "dedicated" if v == 0 else "generic"
        res[f"ours_wgrad_{name}_total_us (GEMM + reduce + unpack)"] = time_rot(lambda i: C.stem_conv_wgrad(dys[i % nsets], xps[i % nsets], h, w, v))
        res[f"  wgrad_{name}_gemm_plus_reduce_us"] = time_rot(lambda i: C.stem_conv_wgrad(dys[i % nsets], xps[i % nsets], h, w, v, False))
    for resident in (True, False):
        dbg = C.stem_conv_fprop_packed(xps[0], w2, h, w, False, resident, True)[2]
        torch.cuda.synchronize()
        c = [int(v) for v in dbg.tolist()]
        res[f"fprop_cta0_cycles_{'resident' if resident else 'streamed'}"] = {
            "a_producer_wait": c[0], "a_producer_issue": c[1], "b_producer_wait": c[2], "b_producer_issue": c[3],
            "issuer_wait_tmem": c[4], "issuer_wait_full": c[5], "issuer_mma": c[6], "issuer_commit": c[7],
            "epilogue_wait": c[8], "epilogue_work": c[9], "kernel": c[10]}
    for k, v in res.items():
        print(f"{k:58s} {v:10.4f}" if isinstance(v, float) else f"{k:58s} {v}", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
