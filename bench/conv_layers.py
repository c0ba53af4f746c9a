#!/usr/bin/env python
"""Per-layer convolution table for ResNet-50 (batch 32, bf16, channels_last): cuDNN fprop / dgrad / wgrad time per
distinct layer shape (the bar), next to this framework's wgmma kernels (``csrc/conv_wgmma.cu``,
``csrc/conv_wgrad_wgmma.cu``), with an optional sweep over their tiling knobs.

  python bench/conv_layers.py [--reps 40] [--batch 32] [--sweep] [--only l3] [--out conv_layers.json]

Timing: CUDA events around the replay of a CUDA graph holding `reps` back-to-back launches that rotate over enough
distinct input sets to exceed the 50 MB L2 (>= 192 MB of operands in rotation), after warm-up rounds; best of 3 replays,
reported per launch.  (Single eager launches are host-bound at ~10 us through the Python bindings and event timing is
quantised at ~2 us, which hides kernels of 5-15 us.)
The reference's hot path these replace: the model's forward / backward at the reference ddp.py:221,231."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, C_in, C_out, kernel, stride, H_in, count in ResNet-50)
LAYERS = [
    ("stem7x7s2", 3, 64, 7, 2, 224, 1),
    ("l1.c1a 1x1", 64, 64, 1, 1, 56, 1),
    ("l1.c1 1x1", 256, 64, 1, 1, 56, 2),
    ("l1.c2 3x3", 64, 64, 3, 1, 56, 3),
    ("l1.c3 1x1", 64, 256, 1, 1, 56, 4),      # 3 x conv3 + the stride-1 downsample
    ("l2.c1a 1x1", 256, 128, 1, 1, 56, 1),
    ("l2.c2a 3x3s2", 128, 128, 3, 2, 56, 1),
    ("l2.ds 1x1s2", 256, 512, 1, 2, 56, 1),
    ("l2.c1 1x1", 512, 128, 1, 1, 28, 3),
    ("l2.c2 3x3", 128, 128, 3, 1, 28, 3),
    ("l2.c3 1x1", 128, 512, 1, 1, 28, 4),
    ("l3.c1a 1x1", 512, 256, 1, 1, 28, 1),
    ("l3.c2a 3x3s2", 256, 256, 3, 2, 28, 1),
    ("l3.ds 1x1s2", 512, 1024, 1, 2, 28, 1),
    ("l3.c1 1x1", 1024, 256, 1, 1, 14, 5),
    ("l3.c2 3x3", 256, 256, 3, 1, 14, 5),
    ("l3.c3 1x1", 256, 1024, 1, 1, 14, 6),
    ("l4.c1a 1x1", 1024, 512, 1, 1, 14, 1),
    ("l4.c2a 3x3s2", 512, 512, 3, 2, 14, 1),
    ("l4.ds 1x1s2", 1024, 2048, 1, 2, 14, 1),
    ("l4.c1 1x1", 2048, 512, 1, 1, 7, 2),
    ("l4.c2 3x3", 512, 512, 3, 1, 7, 2),
    ("l4.c3 1x1", 512, 2048, 1, 1, 7, 3),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--only", type=str, default="")
    ap.add_argument("--sweep", action="store_true", help="sweep tiling knobs of our kernels and report the best per layer / pass")
    ap.add_argument("--skip_lib", action="store_true")
    args = ap.parse_args()
    from b200ddp import _ext
    C = _ext.get()
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = True

    def time_rot(fn, nsets):
        """fn(i) launches on input set i % nsets; returns microseconds per launch.  The `reps` launches are captured into
        one CUDA graph and the graph replay is timed (best of 3): per-launch host overhead (~10 us through the Python
        bindings) would otherwise hide kernels of 5-15 us, and a captured graph is how the training step runs them."""
        for i in range(2 * nsets if nsets < 8 else nsets):
            fn(i)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(args.reps):
                fn(i)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        best = float("inf")
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / args.reps)
        del g
        return best

    def rel(a, b):
        return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))

    rows = []
    tot = {"lib": 0.0, "ours": 0.0}
    n = args.batch
    print(f"{'layer':14s} {'x':>3s} | {'fprop lib':>9s} {'ours':>7s} | {'dgrad lib':>9s} {'ours':>7s} | {'wgrad lib':>9s} {'ours':>7s} | best cfg / relerr f/d/w", flush=True)
    for (name, ci, co, k, s, h, cnt) in LAYERS:
        if args.only and args.only not in name:
            continue
        pad = k // 2
        ho = (h + 2 * pad - k) // s + 1
        bytes_per_set = 2 * n * (ci * h * h + co * ho * ho)
        nsets = max(2, min(48, -(-(192 << 20) // bytes_per_set)))
        xs = [torch.randn(n, ci, h, h, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last) for _ in range(nsets)]
        dys = [torch.randn(n, co, ho, ho, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last) for _ in range(nsets)]
        w = (torch.randn(co, ci, k, k, device=dev) * (1.0 / (ci * k * k) ** 0.5)).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

        def bwd(i, mask):
            return torch.ops.aten.convolution_backward(dys[i % nsets], xs[i % nsets], w, None, [s, s], [pad, pad], [1, 1], False, [0, 0], 1, mask)

        nan = float("nan")
        lib_f = lib_d = lib_w = nan
        if not args.skip_lib:
            lib_f = time_rot(lambda i: F.conv2d(xs[i % nsets], w, None, s, pad), nsets)
            lib_d = time_rot(lambda i: bwd(i, [True, False, False]), nsets) if ci > 3 else nan
            lib_w = time_rot(lambda i: bwd(i, [False, True, False]), nsets)
        row = {"layer": name, "count": cnt, "cin": ci, "cout": co, "k": k, "stride": s, "h": h, "nsets": nsets,
               "lib_fprop_us": lib_f, "lib_dgrad_us": lib_d, "lib_wgrad_us": lib_w}
        our = {"f": nan, "d": nan, "w": nan}
        best = {}
        errs = {}
        if s == 1 and k in (1, 3) and ci % 64 == 0 and co % 64 == 0:
            y_ref = F.conv2d(xs[0], w, None, 1, pad)
            g_ref = torch.ops.aten.convolution_backward(dys[0], xs[0], w, None, [1, 1], [pad, pad], [1, 1], False, [0, 0], 1, [True, True, False])
            # --- fprop / dgrad configs
            modes = [-1]
            if args.sweep and k == 3:
                modes = [1, 2]
            bns = [0] if not args.sweep else [64, 128, 256]
            for which in ("f", "d"):
                ncout = co if which == "f" else ci
                for mode in modes:
                    for bn in bns:
                        if bn and ncout % bn != 0:
                            continue
                        for bo in (0,):
                            try:
                                if which == "f":
                                    call = lambda i, mode=mode, bn=bn, bo=bo: C.conv_fprop(xs[i % nsets], w, 1, pad, mode, bn, bo, False)[0]   # noqa: E731
                                    e = rel(call(0), y_ref)
                                else:
                                    call = lambda i, mode=mode, bn=bn, bo=bo: C.conv_dgrad(dys[i % nsets], w, 1, pad, mode, bn, bo)[0]   # noqa: E731
                                    e = rel(call(0), g_ref[0])
                                torch.cuda.synchronize()
                                if not (e < 2e-2):
                                    print(f"   WRONG {name} {which} mode={mode} bn={bn} bo={bo}: relerr {e:.3e}", flush=True)
                                    continue
                                t = time_rot(call, nsets)
                                if args.sweep:
                                    print(f"   {name} {which} mode={mode} bn={bn} bo={bo}: {t:7.1f} us  relerr {e:.1e}", flush=True)
                                if not (our[which] <= t):
                                    our[which] = t; best[which] = (mode, bn, bo); errs[which] = e
                            except Exception as exc:
                                print(f"   FAIL {name} {which} mode={mode} bn={bn} bo={bo}: {type(exc).__name__}: {str(exc)[:120]}", flush=True)
            # --- wgrad configs
            wcfgs = [(0, 0, 0)]
            if args.sweep:
                wcfgs = [(0, 0, 0)] + [(0, tm, tn) for tm in (128, 256) for tn in (64, 128, 256) if tn <= ci and (tm // 128) * tn <= 512]
            for (sp, tm, tn) in wcfgs:
                try:
                    call = lambda i, sp=sp, tm=tm, tn=tn: C.conv_wgrad(dys[i % nsets], xs[i % nsets], k, 1, pad, sp, tm, tn)   # noqa: E731
                    e = rel(call(0), g_ref[1])
                    torch.cuda.synchronize()
                    if not (e < 2e-2):
                        print(f"   WRONG {name} w split={sp} tile={tm}x{tn}: relerr {e:.3e}", flush=True)
                        continue
                    t = time_rot(call, nsets)
                    if args.sweep:
                        print(f"   {name} w split={sp} tile={tm}x{tn}: {t:7.1f} us  relerr {e:.1e}", flush=True)
                    if not (our["w"] <= t):
                        our["w"] = t; best["w"] = (sp, tm, tn); errs["w"] = e
                except Exception as exc:
                    print(f"   FAIL {name} w split={sp} tile={tm}x{tn}: {type(exc).__name__}: {str(exc)[:120]}", flush=True)
        row.update({"ours_fprop_us": our["f"], "ours_dgrad_us": our["d"], "ours_wgrad_us": our["w"], "best": {k2: list(v) for k2, v in best.items()},
                    "relerr": errs})
        rows.append(row)
        for lib, ours in ((lib_f, our["f"]), (lib_d, our["d"]), (lib_w, our["w"])):
            if lib == lib:
                tot["lib"] += lib * cnt
                tot["ours"] += (ours if ours == ours else lib) * cnt
        es = "/".join(f"{errs[q]:.0e}" if q in errs else "-" for q in "fdw")
        print(f"{name:14s} {cnt:3d} | {lib_f:9.1f} {our['f']:7.1f} | {lib_d:9.1f} {our['d']:7.1f} | {lib_w:9.1f} {our['w']:7.1f} | {best} {es}", flush=True)
        del xs, dys
        torch.cuda.empty_cache()
    print(f"sum over the network (count-weighted, library time where we have no kernel): cuDNN {tot['lib']:.0f} us, ours {tot['ours']:.0f} us", flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"batch": n, "reps": args.reps, "rows": rows, "total_us": tot}, f, indent=1)


if __name__ == "__main__":
    main()
