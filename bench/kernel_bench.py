#!/usr/bin/env python
"""Per-kernel timings against the measured roofline (MEASURED_PEAKS.json: HBM copy GB/s, cuBLAS bf16 TFLOP/s).

  python bench/kernel_bench.py [--only gemm,conv,bn,sgd,ln,xent,mse,input] [--out kernels.json] [--iters 20]

Timing hygiene: >= 3 warm-up launches, CUDA events on the launching stream, a 256 MB write
between timed launches to flush the 50 MB L2, median of `iters`.  Each entry reports algorithmic bytes / FLOPs,
achieved rate and the fraction of the peak (MEASURED_PEAKS.json if present, else the H100 SXM data sheet); cuBLAS / torch timings of the same op are printed beside
ours as the library baseline.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(path):
        d = json.load(open(path))
        return d.get("hbm_gbs", 3350.0), d.get("bf16_tflops", 989.0), d.get("bf16_tflops_sustained", 989.0), "measured"
    # without a measurement: NVIDIA's H100 SXM data sheet (3.35 TB/s HBM3, 989 dense bf16 TFLOP/s at up to 700 W)
    return 3350.0, 989.0, 989.0, "H100 SXM data sheet"


_flush = None


def timeit(fn, iters=20, flush=True):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        if flush:
            _flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", type=str, default="gemm,conv,bn,sgd,ln,xent,mse,input,h2d")
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from b200ddp import _ext
    from b200ddp.ops import functional as Fn
    from b200ddp.optim import FusedSGD
    C = _ext.get()
    hbm, tf_burst, tf_sust, src = peaks()
    dev = torch.device("cuda", 0)
    want = set(args.only.split(","))
    rows = []

    def record(name, ms, flops=None, bytes_=None, lib_ms=None, note=""):
        row = {"kernel": name, "ms": ms, "lib_ms": lib_ms, "note": note}
        if flops:
            row["tflops"] = flops / ms / 1e9
            row["frac_of_peak"] = row["tflops"] / tf_burst
            row["peak"] = f"{tf_burst} TFLOP/s cuBLAS bf16 burst ({src})"
        if bytes_:
            row["gbs"] = bytes_ / ms / 1e6
            row["frac_of_peak"] = row["gbs"] / hbm
            row["peak"] = f"{hbm} GB/s copy ({src})"
        rows.append(row)
        lib = f" | lib {lib_ms:8.3f} ms ({ms / lib_ms:4.2f}x lib time)" if lib_ms else ""
        rate = f"{row.get('tflops', 0):8.1f} TFLOP/s" if flops else f"{row.get('gbs', 0):8.1f} GB/s"
        print(f"{name:44s} {ms:8.3f} ms {rate} {100 * row.get('frac_of_peak', 0):5.1f}% of peak{lib} {note}", flush=True)

    if "gemm" in want:
        shapes = [(8192, 8192, 8192), (16384, 768, 768), (16384, 3072, 768), (16384, 768, 3072), (16384, 2304, 768),
                  (4096, 30528, 768), (32, 1000, 2048),
                  # ResNet-50 1x1 convolutions at batch 32 as GEMMs [N*H*W, C_out, C_in] (memory-bound: the epilogue matters)
                  (100352, 256, 64), (100352, 64, 256), (25088, 512, 128), (6272, 1024, 256), (1568, 2048, 512)]
        for M, N, K in shapes:
            a = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            b = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            lib = timeit(lambda: torch.matmul(a, b.t(), out=out), args.iters)
            for mode, tag in ((1, "1cta"), (2, "2cta")):
                if mode == 2 and (M <= 128 or N <= 128):
                    continue
                C.set_gemm_cta_mode(mode)
                ms = timeit(lambda: C.gemm(a, b, None, False, False, 0, False, out), args.iters)
                record(f"gemm_nt[{tag}] {M}x{N}x{K}", ms, flops=2.0 * M * N * K, lib_ms=lib)
                if mode == 2 and M >= 2048:
                    for g in (4, 8, 16):       # grouped rasterisation (opt-in): L2 reuse of both operands
                        C.set_gemm_group_m(g)
                        ms = timeit(lambda: C.gemm(a, b, None, False, False, 0, False, out), args.iters)
                        record(f"gemm_nt[{tag},group_m={g}] {M}x{N}x{K}", ms, flops=2.0 * M * N * K, lib_ms=lib)
                    C.set_gemm_group_m(0)
                C.set_gemm_tma_store(1)            # staged epilogue (opt-in): smem + TMA store
                ms = timeit(lambda: C.gemm(a, b, None, False, False, 0, False, out), args.iters)
                record(f"gemm_nt[{tag},tma_store] {M}x{N}x{K}", ms, flops=2.0 * M * N * K, lib_ms=lib)
                C.set_gemm_tma_store(0)
            C.set_gemm_cta_mode(0)
        # backward layouts on the BERT FFN shape
        M, N, K = 16384, 3072, 768
        dy = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: C.gemm(dy, w, None, False, True, 0, False, None), args.iters)
        lib = timeit(lambda: torch.matmul(dy, w), args.iters)
        record(f"gemm dgrad {M}x{K}x{N}", ms, flops=2.0 * M * N * K, lib_ms=lib)
        ms = timeit(lambda: C.gemm(dy, x, None, True, True, 0, False, None), args.iters)
        lib = timeit(lambda: torch.matmul(dy.t(), x), args.iters)
        record(f"gemm wgrad {N}x{K}x{M}", ms, flops=2.0 * M * N * K, lib_ms=lib)
        bias = torch.randn(N, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: C.gemm(x, w, bias, False, False, 3, False, None), args.iters)
        lib = timeit(lambda: torch.nn.functional.gelu(torch.nn.functional.linear(x, w, bias)), args.iters)
        record(f"gemm+bias+gelu {M}x{N}x{K}", ms, flops=2.0 * M * N * K, lib_ms=lib, note="lib = cuBLAS linear + gelu kernel")

    if "conv" in want:
        import torch.nn.functional as F
        torch.backends.cudnn.benchmark = True
        n = 32
        # the stem (default ON) and one layer of each kind of the stride-1 set (default OFF); full table: bench/conv_layers.py
        x = torch.randn(n, 3, 224, 224, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        wt = (torch.randn(64, 3, 7, 7, device=dev) / 147 ** 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dy = torch.randn(n, 64, 112, 112, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        xp = C.stem_pack_input(x)
        fl = 2.0 * n * 112 * 112 * 64 * 147
        lib = timeit(lambda: F.conv2d(x, wt, None, 2, 3), args.iters)
        record("stem 7x7s2 fprop (pack + wgmma tap-GEMM) b32", timeit(lambda: C.stem_conv_fprop(x, wt, False, True), args.iters), flops=fl, lib_ms=lib)
        lib = timeit(lambda: torch.ops.aten.convolution_backward(dy, x, wt, None, [2, 2], [3, 3], [1, 1], False, [0, 0], 1, [False, True, False]), args.iters)
        record("stem 7x7s2 wgrad (split-pixel wgmma + reduce) b32", timeit(lambda: C.stem_conv_wgrad(dy, xp, 224, 224, 0), args.iters), flops=fl, lib_ms=lib)
        for (ci, co, k, hw) in [(64, 256, 1, 56), (256, 64, 1, 56), (64, 64, 3, 56), (128, 128, 3, 28), (256, 1024, 1, 14), (512, 512, 3, 7)]:
            pad = k // 2
            xa = torch.randn(n, ci, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            wa = (torch.randn(co, ci, k, k, device=dev) / (ci * k * k) ** 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            da = torch.randn(n, co, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            fl = 2.0 * n * hw * hw * ci * co * k * k
            tag = f"{k}x{k} {ci}->{co} @{hw}"

            def bwd(mask):
                return torch.ops.aten.convolution_backward(da, xa, wa, None, [1, 1], [pad, pad], [1, 1], False, [0, 0], 1, mask)
            record(f"conv fprop {tag}", timeit(lambda: C.conv_fprop(xa, wa, 1, pad, -1, 0, 0, False), args.iters), flops=fl,
                   lib_ms=timeit(lambda: F.conv2d(xa, wa, None, 1, pad), args.iters))
            record(f"conv dgrad {tag}", timeit(lambda: C.conv_dgrad(da, wa, 1, pad, -1, 0, 0), args.iters), flops=fl,
                   lib_ms=timeit(lambda: bwd([True, False, False]), args.iters))
            record(f"conv wgrad {tag}", timeit(lambda: C.conv_wgrad(da, xa, k, 1, pad, 0, 0, 0), args.iters), flops=fl,
                   lib_ms=timeit(lambda: bwd([False, True, False]), args.iters))

    if "bn" in want:
        from b200ddp.ops import FusedBatchNormAct2d
        for shape in [(32, 64, 112, 112), (32, 256, 56, 56), (32, 64, 56, 56), (32, 512, 28, 28), (32, 1024, 14, 14), (32, 2048, 7, 7)]:
            x = torch.randn(*shape, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            res = torch.randn_like(x)
            nbytes = x.numel() * 2
            bn = FusedBatchNormAct2d(shape[1], relu=True).to(dev)
            ref = torch.nn.BatchNorm2d(shape[1]).to(dev)
            ws = bn._workspace(x)
            fwd = lambda: C.bn_forward(x, res, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked, 1e-5, 0.1, True, ws[0], ws[1])
            ms = timeit(fwd, args.iters)
            lib = timeit(lambda: torch.relu(ref(x) + res), args.iters)
            record(f"bn+add+relu fwd {shape}", ms, bytes_=nbytes * 4, lib_ms=lib, note="min traffic: x read twice (2nd from L2), res, y")
            y, stats, mask = fwd()
            dy = torch.randn_like(x)
            ms = timeit(lambda: C.bn_backward(dy, x, mask, bn.weight, stats, True, True, ws[2], ws[3]), args.iters)
            xr = x.clone().requires_grad_()
            rr = res.clone().requires_grad_()
            yl = torch.relu(ref(xr) + rr)
            lib = timeit(lambda: torch.autograd.grad(yl, (xr, rr), dy, retain_graph=True), args.iters)
            record(f"bn+add+relu bwd {shape}", ms, bytes_=nbytes * 8, lib_ms=lib, note="reads dy,x,y twice; writes dx,dres")

    if "sgd" in want:
        for dtype, label in ((torch.float32, "fp32"), (torch.bfloat16, "bf16+master")):
            import torchvision
            shapes = [tuple(p.shape) for p in torchvision.models.resnet50().parameters()]
            params = [torch.nn.Parameter(torch.randn(*s, device=dev).to(dtype)) for s in shapes]
            n = sum(p.numel() for p in params)
            for p in params:
                p.grad = torch.randn_like(p)
            opt = FusedSGD(params, lr=1e-3, max_grad_norm=1000.0)
            ms = timeit(lambda: opt.step(), args.iters)
            es = 4 if dtype == torch.float32 else 2
            # norm pass reads g; update reads g + master/param, writes master (+ param)
            byt = n * (es + es + (4 + 4 if dtype == torch.float32 else 4 + 4 + 2))
            ref = [torch.nn.Parameter(p.detach().float().clone()) for p in params]
            for r, p in zip(ref, params):
                r.grad = p.grad.float()
            ropt = torch.optim.SGD(ref, lr=1e-3)

            def lib_step():
                torch.nn.utils.clip_grad_norm_(ref, 1000.0)
                ropt.step()
            lib = timeit(lib_step, args.iters)
            record(f"clip+sgd resnet50 161 tensors {label}", ms, bytes_=byt, lib_ms=lib, note="lib = clip_grad_norm_ + foreach SGD (fp32)")

    if "ln" in want:
        rows_, cols = 16384, 768
        x = torch.randn(rows_, cols, device=dev, dtype=torch.bfloat16, requires_grad=True)
        g = torch.randn(cols, device=dev, dtype=torch.bfloat16)
        b = torch.randn(cols, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: C.layernorm_fwd(x, g, b, 1e-5), args.iters)
        lib = timeit(lambda: torch.nn.functional.layer_norm(x, (cols,), g, b), args.iters)
        record(f"layernorm fwd {rows_}x{cols} bf16", ms, bytes_=rows_ * cols * 2 * 2, lib_ms=lib)
        y, mean, rstd = C.layernorm_fwd(x, g, b, 1e-5)
        dy = torch.randn_like(y)
        ms = timeit(lambda: C.layernorm_bwd(dy, x, g, mean, rstd), args.iters)
        yl = torch.nn.functional.layer_norm(x, (cols,), g.clone().requires_grad_(), b.clone().requires_grad_())
        lib = timeit(lambda: torch.autograd.grad(yl, x, dy, retain_graph=True), args.iters)
        record(f"layernorm bwd {rows_}x{cols} bf16", ms, bytes_=rows_ * cols * 2 * 3, lib_ms=lib, note="lib computes dx only")

    if "xent" in want:
        rows_, cols = 4096, 30522
        x = torch.randn(rows_, cols, device=dev, dtype=torch.bfloat16)
        t = torch.randint(0, cols, (rows_,), device=dev)
        ms = timeit(lambda: C.xent_fwd_bwd(x, t, -100, 1.0), args.iters)
        xr = x.clone().requires_grad_()

        def lib_xent():
            loss = torch.nn.functional.cross_entropy(xr.float(), t)
            torch.autograd.grad(loss, xr)
        lib = timeit(lib_xent, args.iters)
        record(f"xent fwd+bwd {rows_}x{cols} bf16", ms, bytes_=rows_ * cols * 2 * 2, lib_ms=lib, note="min traffic = read logits + write dlogits")

    if "mse" in want:
        n = 64 * 1024 * 1024
        o = torch.randn(n, device=dev, dtype=torch.bfloat16)
        t = torch.randn(n, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: C.mse_fwd_bwd(o, t, 1.0), args.iters)
        record(f"mse fwd+bwd {n} bf16", ms, bytes_=n * 2 * 3)

    if "input" in want:
        x = torch.randn(256, 3, 224, 224, device=dev)
        dst = torch.empty(x.shape, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        mean, istd = torch.zeros(3, device=dev), torch.ones(3, device=dev)
        ms = timeit(lambda: C.normalize_to_channels_last(x, dst, mean, istd, 1.0), args.iters)
        lib = timeit(lambda: x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last), args.iters)
        record("normalize+cast+NHWC 256x3x224x224", ms, bytes_=x.numel() * 6, lib_ms=lib)

    if "h2d" in want:
        for nbytes, label in ((32 * 3 * 224 * 224 * 4, "fp32 batch 19.3 MB"), (32 * 3 * 224 * 224, "uint8 batch 4.8 MB"), (256 << 20, "256 MB")):
            host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
            devb = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            ms = timeit(lambda: devb.copy_(host, non_blocking=True), args.iters, flush=False)
            rows.append({"kernel": f"H2D pinned {label}", "ms": ms, "gbs": nbytes / ms / 1e6})
            print(f"H2D pinned {label:32s} {ms:8.3f} ms {nbytes / ms / 1e6:8.1f} GB/s", flush=True)
            ms = timeit(lambda: host.copy_(devb, non_blocking=True), args.iters, flush=False)
            print(f"D2H pinned {label:32s} {ms:8.3f} ms {nbytes / ms / 1e6:8.1f} GB/s", flush=True)

    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump({"peaks": {"hbm_gbs": hbm, "bf16_tflops_burst": tf_burst, "bf16_tflops_sustained": tf_sust, "source": src},
                   "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
