#!/usr/bin/env python
"""Per-kernel timings against the measured roofline (MEASURED_PEAKS.json: HBM copy GB/s, cuBLAS bf16 TFLOP/s).

  python bench/kernel_bench.py [--only gemm,fp8,attn,llama,qwen,qwen3,modernbert,vit,clip,cross,t5,convnext,swin,mamba,mamba2,mae,conv,bn,sgd,adamw,ln,xent,lmloss,sparse,moe,mse,input] [--out kernels.json] [--iters 20]

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
    ap.add_argument("--only", type=str, default="gemm,fp8,attn,llama,qwen,conv,bn,sgd,adamw,ln,xent,mse,input,h2d")
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from b200ddp import _ext
    from b200ddp.ops import functional as Fn
    from b200ddp.optim import FusedAdamW, FusedSGD
    C = _ext.get()
    hbm, tf_burst, tf_sust, src = peaks()
    dev = torch.device("cuda", 0)
    want = set(args.only.split(","))
    rows = []

    def record(name, ms, flops=None, bytes_=None, lib_ms=None, note="", fp8=False):
        row = {"kernel": name, "ms": ms, "lib_ms": lib_ms, "note": note}
        if flops:
            row["tflops"] = flops / ms / 1e9
            if fp8:     # dense FP8 rate of the H100 SXM data sheet (700 W); there is no measured FP8 peak
                row["frac_of_peak"] = row["tflops"] / 1979.0
                row["peak"] = "1979 TFLOP/s dense FP8 (H100 SXM data sheet)"
            else:
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

    if "fp8" in want:
        # The four BERT-base encoder linears at batch 16 x seq 512 (M = 8192), FP8 (E4M3 x / W, E5M2 dy) against our bf16
        # GEMM and torch._scaled_mm (cuBLASLt, use_fast_accum=False) on the same FP8 bytes; then the two quantisation passes.
        M = 16 * 512
        bf16 = torch.bfloat16

        def scaled_mm(a, b, sa, sb):
            return torch._scaled_mm(a, b.t(), scale_a=sa, scale_b=sb, out_dtype=bf16, use_fast_accum=False)

        for N, K in ((2304, 768), (768, 768), (3072, 768), (768, 3072)):
            x = torch.randn(M, K, device=dev, dtype=bf16)
            w = (torch.randn(N, K, device=dev) * 0.05).to(bf16)
            dy = (torch.randn(M, N, device=dev) * 1e-3).to(bf16)
            xq, xqt, xs, _ = C.fp8_quantize(x, "e4m3", True, False)
            wq, wqt, ws, _ = C.fp8_quantize(w, "e4m3", True, False)
            dq, dqt, ds, _ = C.fp8_quantize(dy, "e5m2", True, False)
            flops = 2.0 * M * N * K
            for tag, fp8_call, bf16_call, ops in (
                    (f"fwd {M}x{N}x{K}", lambda: C.gemm_fp8(xq, wq, xs, ws, None, 0),
                     lambda: C.gemm(x, w, None, False, False, 0, False, None), (xq, wq, xs, ws)),
                    (f"dgrad {M}x{K}x{N}", lambda: C.gemm_fp8(dq, wqt, ds, ws, None, 0),
                     lambda: C.gemm(dy, w, None, False, True, 0, False, None), (dq, wqt, ds, ws)),
                    (f"wgrad {N}x{K}x{M}", lambda: C.gemm_fp8(dqt, xqt, ds, xs, None, 0),
                     lambda: C.gemm(dy, x, None, True, True, 0, False, None), (dqt, xqt, ds, xs))):
                try:
                    lib = timeit(lambda: scaled_mm(*ops), args.iters)
                except RuntimeError as e:          # a layout / type pair cuBLASLt does not take
                    lib, tag = None, tag + f" (_scaled_mm: {str(e).splitlines()[0][:60]})"
                ms_bf16 = timeit(bf16_call, args.iters)
                record(f"gemm bf16 {tag}", ms_bf16, flops=flops)
                ms = timeit(fp8_call, args.iters)
                record(f"gemm_fp8 {tag}", ms, flops=flops, lib_ms=lib, fp8=True,
                       note=f"lib = torch._scaled_mm; {ms_bf16 / ms:4.2f}x our bf16 GEMM's speed")
        for rows_, cols_, fmt, colsum in ((M, 768, "e4m3", False), (M, 3072, "e4m3", False), (M, 768, "e5m2", True),
                                          (M, 2304, "e5m2", True), (M, 3072, "e5m2", True)):
            t = torch.randn(rows_, cols_, device=dev, dtype=bf16)
            amax = C.fp8_amax(t)
            ms = timeit(lambda: C.fp8_amax(t), args.iters)
            record(f"fp8_amax {rows_}x{cols_}", ms, bytes_=2.0 * rows_ * cols_)
            ms = timeit(lambda: C.fp8_cast_transpose(t, amax, fmt, True, colsum), args.iters)
            # bf16 in, q and q^T out (the column-sum workspace is one fp32 row per 64 input rows)
            record(f"fp8_cast_transpose[{fmt}{',colsum' if colsum else ''}] {rows_}x{cols_}", ms, bytes_=4.0 * rows_ * cols_,
                   note="L2 flushed before each launch")

    if "attn" in want:
        # BERT-base attention at batch 16 x seq 512 (12 heads, d 64) from one fused qkv [B*S, 3*768] tensor.  Native
        # kernels against SDPA on the views BertLayer makes (flash with every key visible, the boolean key mask
        # otherwise).  The SDPA backward is timed through autograd into qkv, as in training (it includes the copy of
        # dq / dk / dv into the fused gradient).  Algorithmic FLOPs from the lengths: forward 4 sum_b S len_b d H,
        # backward 2.5x that; the native backward's recomputation of P is not counted.
        import torch.nn.functional as F
        B, S, H, d = 16, 512, 12, 64
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(B * S, 3 * H * d, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(B * S, H * d, device=dev, generator=g).to(torch.bfloat16)
        lens_random = torch.randint(128, S + 1, (B,), generator=torch.Generator().manual_seed(0))
        for label, lens in (("full length", torch.full((B,), S)), ("lengths U[128,512]", lens_random)):
            lt = lens.to(dev, torch.int32)
            fwd_flops = 4.0 * S * float(lens.sum()) * d * H
            x = qkv.view(B, S, 3 * H * d).detach().clone().requires_grad_(True)
            q, k, v = (t.reshape(B, S, H, d).transpose(1, 2) for t in x.split(H * d, dim=-1))
            mask = None if bool((lens == S).all()) else (torch.arange(S, device=dev)[None, :] < lt[:, None])[:, None, None, :]
            lib_name = "SDPA flash" if mask is None else "SDPA bool mask"

            def sdpa():
                return F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B, S, H * d)
            lib = timeit(lambda: sdpa().detach(), args.iters)
            record(f"attention fwd {label} B{B} S{S} H{H}", timeit(lambda: C.attention_fwd(qkv, lt, H), args.iters),
                   flops=fwd_flops, lib_ms=lib, note=f"lib = {lib_name} + output transpose")
            o, lse = C.attention_fwd(qkv, lt, H)
            y = sdpa()
            dy = dout.view(B, S, H * d)
            lib = timeit(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), args.iters)
            record(f"attention bwd {label} B{B} S{S} H{H}", timeit(lambda: C.attention_bwd(dout, qkv, o, lse, lt, H), args.iters),
                   flops=2.5 * fwd_flops, lib_ms=lib, note=f"lib = {lib_name} backward into qkv")
            del x, q, k, v, y
        # Packed documents: B evenly spaced rows of the training set's packing (documents U[128, 512], first-fit
        # decreasing, which fills its first rows with the longest documents alone), native segment-mode kernels against
        # SDPA with the dense block-diagonal boolean mask [B, 1, S, S].  FLOPs count only the block-diagonal: forward
        # 4 sum_docs len^2 d H, backward 2.5x that.
        from b200ddp.data import SyntheticTokens
        from b200ddp.ops import document_bounds
        packed = SyntheticTokens(seq_len=S, min_len=128, pack=True)
        rows = torch.linspace(0, len(packed) - 1, B).long().tolist()
        bounds, _ = document_bounds(packed.X[rows].to(dev), packed.cls_token_id, packed.pad_token_id)
        docs = [n for r in rows for n in packed.doc_lengths[r]]
        fwd_flops = 4.0 * sum(n * n for n in docs) * d * H
        label = f"packed {len(docs)} docs U[128,512]"
        x = qkv.view(B, S, 3 * H * d).detach().clone().requires_grad_(True)
        q, k, v = (t.reshape(B, S, H, d).transpose(1, 2) for t in x.split(H * d, dim=-1))
        j = torch.arange(S, device=dev)
        mask = ((j >= bounds[..., :1]) & (j < bounds[..., 1:]))[:, None]
        mask |= torch.eye(S, dtype=torch.bool, device=dev)          # tail padding rows: their own key, not a NaN row

        def sdpa():
            return F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B, S, H * d)
        lib = timeit(lambda: sdpa().detach(), args.iters)
        record(f"attention fwd {label} B{B} S{S} H{H}", timeit(lambda: C.packed_attention_fwd(qkv, bounds, H), args.iters),
               flops=fwd_flops, lib_ms=lib, note="lib = SDPA block-diagonal bool mask + output transpose")
        o, lse = C.packed_attention_fwd(qkv, bounds, H)
        y = sdpa()
        dy = dout.view(B, S, H * d)
        lib = timeit(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), args.iters)
        record(f"attention bwd {label} B{B} S{S} H{H}",
               timeit(lambda: C.packed_attention_bwd(dout, qkv, o, lse, bounds, H), args.iters),
               flops=2.5 * fwd_flops, lib_ms=lib, note="lib = SDPA block-diagonal bool mask backward into qkv")
        del x, q, k, v, y
        # Causal documents (GPT-2 at batch 8 x seq 1024, 12 heads): the native causal kernels against SDPA with
        # is_causal (flash) on full and right-padded rows, and against SDPA with the dense causal block-diagonal mask on
        # packed rows.  FLOPs count only the causal part of each document: forward 2 d H sum_docs len (len + 1),
        # backward 2.5x that.
        from b200ddp.data import SyntheticTokens as _Tok
        B, S = 8, 1024
        qkv = torch.randn(B * S, 3 * H * d, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(B * S, H * d, device=dev, generator=g).to(torch.bfloat16)
        j = torch.arange(S, device=dev)
        lens_random = torch.randint(128, S + 1, (B,), generator=torch.Generator().manual_seed(0))
        packed = _Tok(seq_len=S, min_len=128, vocab=50257, pack=True, causal=True)
        rows = torch.linspace(0, len(packed) - 1, B).long().tolist()
        cases = [("full length", [[S]] * B, None), ("lengths U[128,1024]", [[int(n)] for n in lens_random], None),
                 (None, [packed.doc_lengths[r] for r in rows], packed.X[rows])]
        for label, docs, ids in cases:
            if ids is None:
                lt = torch.tensor([sum(r) for r in docs], device=dev)
                bounds, _ = document_bounds(torch.where(j[None, :] < lt[:, None], 1, 0), None, 0)
            else:
                bounds, _ = document_bounds(ids.to(dev), packed.bos_token_id, packed.pad_token_id)
                label = f"packed {sum(len(r) for r in docs)} docs U[128,1024]"
            flat = [n for r in docs for n in r]
            fwd_flops = 2.0 * sum(n * (n + 1) for n in flat) * d * H
            x = qkv.view(B, S, 3 * H * d).detach().clone().requires_grad_(True)
            q, k, v = (t.reshape(B, S, H, d).transpose(1, 2) for t in x.split(H * d, dim=-1))
            if ids is None:
                mask, lib_name = None, "SDPA is_causal (flash)"
            else:
                mask = ((j >= bounds[..., :1]) & (j < bounds[..., 1:]) & (j[None, :] <= j[:, None]))[:, None]
                mask |= torch.eye(S, dtype=torch.bool, device=dev)   # tail padding rows: their own key, not a NaN row
                lib_name = "SDPA causal block-diagonal bool mask"

            def sdpa():
                return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, is_causal=mask is None) \
                    .transpose(1, 2).reshape(B, S, H * d)
            lib = timeit(lambda: sdpa().detach(), args.iters)
            record(f"causal attention fwd {label} B{B} S{S} H{H}",
                   timeit(lambda: C.causal_attention_fwd(qkv, bounds, H), args.iters),
                   flops=fwd_flops, lib_ms=lib, note=f"lib = {lib_name} + output transpose")
            o, lse = C.causal_attention_fwd(qkv, bounds, H)
            y = sdpa()
            dy = dout.view(B, S, H * d)
            lib = timeit(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), args.iters)
            record(f"causal attention bwd {label} B{B} S{S} H{H}",
                   timeit(lambda: C.causal_attention_bwd(dout, qkv, o, lse, bounds, H), args.iters),
                   flops=2.5 * fwd_flops, lib_ms=lib, note=f"lib = {lib_name} backward into qkv")
            del x, q, k, v, y

    def card():
        import subprocess
        try:
            limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                                   capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            limit = "unknown"
        return f"{torch.cuda.get_device_name(dev)}, power limit {limit or 'unknown'}"

    def causal_lm_attention(tag, B, S, H, Hkv, d, vocab, bos_id, fwd, bwd):
        # Grouped-query causal attention: the native kernels against SDPA (enable_gqa) with is_causal on full and
        # right-padded rows (SDPA computes the padding too) and with the dense causal block-diagonal mask on packed rows.
        # FLOPs count only the causal part of each document: forward 2 d H sum_docs len (len + 1), backward 2.5x that.
        import torch.nn.functional as F
        from b200ddp.data import SyntheticTokens
        from b200ddp.ops import document_bounds
        g = torch.Generator(device="cuda").manual_seed(1)
        qkv = torch.randn(B * S, (H + 2 * Hkv) * d, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(B * S, H * d, device=dev, generator=g).to(torch.bfloat16)
        j = torch.arange(S, device=dev)
        lens_random = torch.randint(256, S + 1, (B,), generator=torch.Generator().manual_seed(0))
        packed = SyntheticTokens(samples=64, seq_len=S, min_len=256, vocab=vocab, pack=True, causal=True, bos_token_id=bos_id)
        prow = torch.linspace(0, len(packed) - 1, B).long().tolist()
        cases = [("full length", [[S]] * B, None), (f"lengths U[256,{S}]", [[int(n)] for n in lens_random], None),
                 (None, [packed.doc_lengths[r] for r in prow], packed.X[prow])]
        for label, docs, ids in cases:
            if ids is None:
                lt = torch.tensor([sum(r) for r in docs], device=dev)
                bounds, _ = document_bounds(torch.where(j[None, :] < lt[:, None], 1, 0), None, 0)
            else:
                bounds, _ = document_bounds(ids.to(dev), packed.bos_token_id, packed.pad_token_id)
                label = f"packed {sum(len(r) for r in docs)} docs U[256,{S}]"
            fwd_flops = 2.0 * sum(n * (n + 1) for r in docs for n in r) * d * H
            x = qkv.view(B, S, -1).detach().clone().requires_grad_(True)
            q, k, v = (t.reshape(B, S, -1, d).transpose(1, 2) for t in x.split([H * d, Hkv * d, Hkv * d], dim=-1))
            if ids is None:
                mask, lib_name = None, "SDPA is_causal enable_gqa"
            else:
                mask = ((j >= bounds[..., :1]) & (j < bounds[..., 1:]) & (j[None, :] <= j[:, None]))[:, None]
                mask |= torch.eye(S, dtype=torch.bool, device=dev)   # tail padding rows: their own key, not a NaN row
                lib_name = "SDPA enable_gqa causal block-diagonal bool mask"

            def sdpa():
                return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, is_causal=mask is None, enable_gqa=True) \
                    .transpose(1, 2).reshape(B, S, H * d)
            lib = timeit(lambda: sdpa().detach(), args.iters)
            record(f"{tag} attention fwd {label} B{B} S{S} H{H}/{Hkv}", timeit(lambda: fwd(qkv, bounds, H, Hkv), args.iters),
                   flops=fwd_flops, lib_ms=lib, note=f"lib = {lib_name} + output transpose")
            o, lse = fwd(qkv, bounds, H, Hkv)
            y = sdpa()
            dy = dout.view(B, S, H * d)
            lib = timeit(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), args.iters)
            record(f"{tag} attention bwd {label} B{B} S{S} H{H}/{Hkv}",
                   timeit(lambda: bwd(dout, qkv, o, lse, bounds, H, Hkv), args.iters),
                   flops=2.5 * fwd_flops, lib_ms=lib, note=f"lib = {lib_name} backward into qkv")
            del x, q, k, v, y, mask
        return qkv

    def rmsnorm_rows(M, hidden, eps):
        # RMSNorm [M, hidden] bf16 against F.rms_norm (bytes: x, y; backward x, dy, dx)
        import torch.nn.functional as F
        xr = torch.randn(M, hidden, device=dev).to(torch.bfloat16)
        wr = (torch.rand(hidden, device=dev) + 0.5).to(torch.bfloat16)
        dyr = torch.randn_like(xr)
        lib = timeit(lambda: F.rms_norm(xr, (hidden,), wr, eps), args.iters)
        record(f"rmsnorm fwd {M}x{hidden} bf16", timeit(lambda: C.rmsnorm_fwd(xr, wr, eps), args.iters),
               bytes_=M * hidden * 2 * 2, lib_ms=lib, note="lib = F.rms_norm")
        _, rstd = C.rmsnorm_fwd(xr, wr, eps)
        xg, wg = xr.clone().requires_grad_(True), wr.clone().requires_grad_(True)
        yr = F.rms_norm(xg, (hidden,), wg, eps)
        lib = timeit(lambda: torch.autograd.grad(yr, (xg, wg), dyr, retain_graph=True), args.iters)
        record(f"rmsnorm bwd {M}x{hidden} bf16", timeit(lambda: C.rmsnorm_bwd(dyr, xr, wr, rstd), args.iters),
               bytes_=M * hidden * 2 * 3, lib_ms=lib, note="lib = F.rms_norm autograd (dx, dgamma)")

    def rotary_rows(qkv, H, Hkv, d, max_pos, theta):
        # Rotary on the q and k blocks of qkv (v copied) against the rotate_half expression (bytes: qkv in, out)
        M = qkv.shape[0]
        pos = torch.randint(0, max_pos, (M,), device=dev, dtype=torch.int32)
        table = Fn.rotary_cos_sin(max_pos, d, theta).to(dev)
        cos = torch.cat([table[pos.long(), 0]] * 2, -1)[:, None].to(torch.bfloat16)
        sin = torch.cat([table[pos.long(), 1]] * 2, -1)[:, None].to(torch.bfloat16)

        def rope_lib():
            qk = qkv[:, :(H + Hkv) * d].view(M, H + Hkv, d)
            rot = torch.cat([-qk[..., d // 2:], qk[..., :d // 2]], -1)
            return torch.cat([(qk * cos + rot * sin).view(M, -1), qkv[:, (H + Hkv) * d:]], -1)
        record(f"rotary fwd {M}x{(H + 2 * Hkv) * d} bf16", timeit(lambda: C.rotary(qkv, pos, table, H, Hkv, False), args.iters),
               bytes_=qkv.numel() * 2 * 2, lib_ms=timeit(rope_lib, args.iters), note="lib = rotate_half expression (bf16 cos/sin)")

    if "llama" in want:
        # SmolLM-135M's hot ops at batch 8 x 2048 (9 query heads over 3 K/V heads, d 64, hidden 576, SwiGLU 1536), each
        # against its torch equivalent.  The card and its power limit are part of every number below.
        import torch.nn.functional as F
        from b200ddp.models import MODEL_REGISTRY
        print(f"llama kernels on {card()}", flush=True)
        B, S, H, Hkv, d, hidden, inter = 8, 2048, 9, 3, 64, 576, 1536
        M = B * S
        smollm = MODEL_REGISTRY["smollm-135m"]
        qkv = causal_lm_attention("gqa", B, S, H, Hkv, d, smollm.config.vocab_size, smollm.start_id, C.causal_gqa_attention_fwd,
                                  C.causal_gqa_attention_bwd)
        rmsnorm_rows(M, hidden, 1e-5)
        rotary_rows(qkv, H, Hkv, d, S, 10000.0)
        # SwiGLU [B*S, 2 x 1536] against F.silu(g) * u (bytes: gate_up, out; backward gate_up, dy, d[gate | up])
        gu = torch.randn(M, 2 * inter, device=dev).to(torch.bfloat16)
        dys = torch.randn(M, inter, device=dev).to(torch.bfloat16)

        def swiglu_lib(t):
            a, b = t.chunk(2, -1)
            return F.silu(a) * b
        record(f"swiglu fwd {M}x{inter} bf16", timeit(lambda: C.swiglu_fwd(gu), args.iters), bytes_=M * inter * 3 * 2,
               lib_ms=timeit(lambda: swiglu_lib(gu), args.iters), note="lib = F.silu(g) * u")
        gg = gu.clone().requires_grad_(True)
        ys = swiglu_lib(gg)
        record(f"swiglu bwd {M}x{inter} bf16", timeit(lambda: C.swiglu_bwd(dys, gu), args.iters), bytes_=M * inter * 5 * 2,
               lib_ms=timeit(lambda: torch.autograd.grad(ys, gg, dys, retain_graph=True), args.iters),
               note="lib = F.silu(g) * u autograd")
        del gg, ys

    if "qwen" in want:
        # Qwen2.5-1.5B's head-dim-128 ops at batch 4 x 2048 (12 query heads over 2 K/V heads, hidden 1536), each against
        # its torch equivalent.  The card and its power limit are part of every number below.
        from b200ddp.models import MODEL_REGISTRY
        print(f"qwen kernels on {card()}", flush=True)
        B, S, H, Hkv, d, hidden = 4, 2048, 12, 2, 128, 1536
        qwen = MODEL_REGISTRY["qwen2.5-1.5b"]
        qkv = causal_lm_attention("d128", B, S, H, Hkv, d, qwen.config.vocab_size, qwen.start_id, C.causal_attention_d128_fwd,
                                  C.causal_attention_d128_bwd)
        rmsnorm_rows(8192, hidden, 1e-6)
        rotary_rows(qkv, H, Hkv, d, S, 1e6)

    if "qwen3" in want:
        # Qwen3-0.6B's per-head q / k RMSNorm + rotary at batch 8 x 2048: qkv [16384, (16 + 2 * 8) * 128] bf16.  Baselines:
        # the torch expression (F.rms_norm on the head views, then rotate_half with bf16 cos / sin, autograd for the
        # backward) and our rotary kernel alone, the floor the fusion should approach.  Algorithmic bytes: forward qkv in,
        # out and rstd out; backward dy, qkv, rstd in and dqkv out (weights and the [2, parts, 128] partials are noise).
        import torch.nn.functional as F
        print(f"qwen3 kernels on {card()}", flush=True)
        M, H, Hkv, d, eps = 16384, 16, 8, 128, 1e-6
        W, normed = (H + 2 * Hkv) * d, H + Hkv
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(M, W, device=dev, generator=g).to(torch.bfloat16)
        dy = torch.randn(M, W, device=dev, generator=g).to(torch.bfloat16)
        wq, wk = ((torch.rand(d, device=dev, generator=g) + 0.5).to(torch.bfloat16) for _ in range(2))
        pos = (torch.arange(M, device=dev, dtype=torch.int32) % 2048).contiguous()
        table = Fn.rotary_cos_sin(2048, d, 1e6).to(dev)
        cos = torch.cat([table[pos.long(), 0]] * 2, -1)[:, None].to(torch.bfloat16)
        sin = torch.cat([table[pos.long(), 1]] * 2, -1)[:, None].to(torch.bfloat16)

        def torch_fwd(t, a, b):
            h = t.view(M, H + 2 * Hkv, d)
            qk = torch.cat([F.rms_norm(h[:, :H], (d,), a, eps), F.rms_norm(h[:, H:normed], (d,), b, eps)], 1)
            rot = torch.cat([-qk[..., d // 2:], qk[..., :d // 2]], -1)
            return torch.cat([(qk * cos + rot * sin).view(M, -1), t[:, normed * d:]], -1)
        io = M * W * 2
        y, rstd = C.qk_norm_rotary_fwd(x, wq, wk, pos, table, H, Hkv, eps)
        record(f"qk_norm_rotary fwd {M}x{W} bf16", timeit(lambda: C.qk_norm_rotary_fwd(x, wq, wk, pos, table, H, Hkv, eps), args.iters),
               bytes_=2 * io + M * normed * 4, lib_ms=timeit(lambda: torch_fwd(x, wq, wk), args.iters),
               note="lib = F.rms_norm per head view + rotate_half")
        record(f"rotary alone fwd {M}x{W} bf16", timeit(lambda: C.rotary(x, pos, table, H, Hkv, False), args.iters), bytes_=2 * io,
               note="the floor: rotation without the norm")
        xg, ag, bg = (t.clone().requires_grad_(True) for t in (x, wq, wk))
        yt = torch_fwd(xg, ag, bg)
        record(f"qk_norm_rotary bwd {M}x{W} bf16",
               timeit(lambda: C.qk_norm_rotary_bwd(dy, x, rstd, wq, wk, pos, table, H, Hkv), args.iters),
               bytes_=3 * io + M * normed * 4,
               lib_ms=timeit(lambda: torch.autograd.grad(yt, (xg, ag, bg), dy, retain_graph=True), args.iters),
               note="lib = the torch expression's autograd (dqkv, dw_q, dw_k)")
        record(f"rotary alone bwd {M}x{W} bf16", timeit(lambda: C.rotary(dy, pos, table, H, Hkv, True), args.iters), bytes_=2 * io,
               note="the floor: rotation without the norm")
        del xg, ag, bg, yt

    if "modernbert" in want:
        # ModernBERT-base's attention at 2 x 8192 tokens (12 heads, d 64): local layers (window_bounds, +-64) and global
        # layers on the native document-bounds kernels, against SDPA with the dense [B, 1, S, S] mask each would need
        # (flash for global attention on fixed rows).  Fixed rows, right-padded rows (lengths U[1024, 8192]) and packed
        # documents (the CLI's packing, U[1024, 8192]).  FLOPs count the visible pairs only: forward 4 d H sum(end - start),
        # backward 2.5x that.  Then GeGLU at [16384, 2 x 1152] against F.gelu(a) * g.  The card and its power limit are
        # part of every number below.
        import torch.nn.functional as F
        from b200ddp.data import SyntheticTokens
        from b200ddp.models import MODEL_REGISTRY
        from b200ddp.ops import document_bounds, window_bounds
        print(f"modernbert kernels on {card()}", flush=True)
        entry = MODEL_REGISTRY["modernbert-base"]
        B, S, H, d, inter = 2, 8192, 12, 64, entry.config.intermediate
        w = entry.config.local_attention // 2
        g = torch.Generator(device="cuda").manual_seed(2)
        qkv = torch.randn(B * S, 3 * H * d, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(B * S, H * d, device=dev, generator=g).to(torch.bfloat16)
        j = torch.arange(S, device=dev)
        lens = torch.randint(1024, S + 1, (B,), generator=torch.Generator().manual_seed(0)).to(dev)
        packed = SyntheticTokens(samples=64, seq_len=S, min_len=1024, vocab=entry.config.vocab_size, pack=True,
                                 cls_token_id=entry.start_id)
        prow = torch.linspace(0, len(packed) - 1, B).long().tolist()
        layouts = [("fixed", document_bounds(torch.ones(B, S, dtype=torch.long, device=dev), None, None)[0]),
                   ("padded U[1024,8192]", document_bounds(torch.where(j[None, :] < lens[:, None], 1, 0), None, 0)[0]),
                   (f"packed {sum(len(packed.doc_lengths[r]) for r in prow)} docs U[1024,8192]",
                    document_bounds(packed.X[prow].to(dev), packed.cls_token_id, packed.pad_token_id)[0])]
        for label, bounds in layouts:
            for kind, bnd in (("local", window_bounds(bounds, w)), ("global", bounds)):
                fwd_flops = 4.0 * float((bnd[..., 1] - bnd[..., 0]).sum()) * d * H
                x = qkv.view(B, S, -1).detach().clone().requires_grad_(True)
                q, k, v = (t.reshape(B, S, H, d).transpose(1, 2) for t in x.split(H * d, dim=-1))
                if kind == "global" and label == "fixed":
                    mask, lib_name = None, "SDPA flash"
                else:
                    mask = ((j >= bnd[..., :1]) & (j < bnd[..., 1:]))[:, None]
                    mask |= torch.eye(S, dtype=torch.bool, device=dev)     # padding rows: their own key, not a NaN row
                    lib_name = f"SDPA dense {'band' if kind == 'local' else 'block-diagonal'} bool mask"

                def sdpa():
                    return F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B, S, H * d)
                lib = timeit(lambda: sdpa().detach(), args.iters)
                record(f"modernbert {kind} attention fwd {label} B{B} S{S}",
                       timeit(lambda: C.packed_attention_fwd(qkv, bnd, H), args.iters), flops=fwd_flops, lib_ms=lib,
                       note=f"lib = {lib_name} + output transpose")
                o, lse = C.packed_attention_fwd(qkv, bnd, H)
                y = sdpa()
                dy = dout.view(B, S, H * d)
                lib = timeit(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), args.iters)
                record(f"modernbert {kind} attention bwd {label} B{B} S{S}",
                       timeit(lambda: C.packed_attention_bwd(dout, qkv, o, lse, bnd, H), args.iters),
                       flops=2.5 * fwd_flops, lib_ms=lib, note=f"lib = {lib_name} backward into qkv")
                del x, q, k, v, y, mask
        # GeGLU [16384, 2 x 1152] (bytes: input_gate, out; backward input_gate, dy, d[input | gate])
        M = B * S
        ig = torch.randn(M, 2 * inter, device=dev).to(torch.bfloat16)
        dyg = torch.randn(M, inter, device=dev).to(torch.bfloat16)

        def geglu_lib(t):
            a, b = t.chunk(2, -1)
            return F.gelu(a) * b
        record(f"geglu fwd {M}x{inter} bf16", timeit(lambda: C.geglu_fwd(ig), args.iters), bytes_=M * inter * 3 * 2,
               lib_ms=timeit(lambda: geglu_lib(ig), args.iters), note="lib = F.gelu(a) * g")
        gg = ig.clone().requires_grad_(True)
        yg = geglu_lib(gg)
        record(f"geglu bwd {M}x{inter} bf16", timeit(lambda: C.geglu_bwd(dyg, ig), args.iters), bytes_=M * inter * 5 * 2,
               lib_ms=timeit(lambda: torch.autograd.grad(yg, gg, dyg, retain_graph=True), args.iters),
               note="lib = F.gelu(a) * g autograd")
        del gg, yg

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
        # Each shape runs the default kernels (resident: one launch per direction, activations read once, where the shape fits
        # the CTAs' shared memory) and the two-pass kernels (set_bn_two_pass).  Algorithmic bytes per path, bf16 [R, C] with
        # the 1-bit ReLU mask (R*C/8 bytes): forward resident x + res + y + mask, two-pass 2x + res + y + mask; backward
        # resident dy + x + mask + dx + dres, two-pass 2 (dy + x + mask) + dx + dres.
        # (32, 512, 28, 28) is also run without ReLU / residual (the downsample BatchNorm): x + y only.
        for shape in [(32, 64, 112, 112), (32, 256, 56, 56), (32, 64, 56, 56), (32, 512, 28, 28), (32, 1024, 14, 14), (32, 2048, 7, 7),
                      (32, 128, 56, 56), (32, 512, 28, 28, "plain")]:
            relu = len(shape) == 4
            shape = shape[:4]
            x = torch.randn(*shape, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            res = torch.randn_like(x) if relu else None
            nbytes = x.numel() * 2
            mbytes = x.numel() // 8 if relu else 0
            bn = FusedBatchNormAct2d(shape[1], relu=relu).to(dev)
            ref = torch.nn.BatchNorm2d(shape[1]).to(dev)
            ws = bn._workspace(x)
            fwd = lambda: C.bn_forward(x, res, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked, 1e-5, 0.1, relu, ws[0], ws[1])
            dy = torch.randn_like(x)
            tag = "bn+add+relu" if relu else "bn"
            lib_f = timeit((lambda: torch.relu(ref(x) + res)) if relu else (lambda: ref(x)), args.iters)
            xr = x.clone().requires_grad_()
            rr = res.clone().requires_grad_() if relu else None
            yl = torch.relu(ref(xr) + rr) if relu else ref(xr)
            lib_b = timeit(lambda: torch.autograd.grad(yl, (xr, rr) if relu else (xr,), dy, retain_graph=True), args.iters)
            streams_f = 2 if relu else 1               # x + res (read once) ... + y
            streams_b = 4 if relu else 3               # dy, x, dx (+ dres)
            for two_pass in (0, 1):
                C.set_bn_two_pass(two_pass)
                n0 = C.launch_count()
                y, stats, mask = fwd()
                path = "two-pass" if two_pass or C.launch_count() - n0 > 1 else "resident"
                if two_pass == 0 and path == "two-pass":
                    path = "default=two-pass"
                ms = timeit(fwd, args.iters)
                fb = nbytes * (streams_f + 1 + (1 if "two-pass" in path else 0)) + mbytes
                record(f"{tag} fwd {shape} [{path}]", ms, bytes_=fb, lib_ms=lib_f,
                       note=("x, res, y, mask" if relu else "x, y") + (" + 2nd x read" if "two-pass" in path else ""))
                bwd = lambda: C.bn_backward(dy, x, mask if relu else None, bn.weight, stats, relu, relu, ws[2], ws[3])
                n0 = C.launch_count()
                bwd()
                bpath = "two-pass" if two_pass or C.launch_count() - n0 > 1 else "resident"
                if two_pass == 0 and bpath == "two-pass":
                    bpath = "default=two-pass"
                ms = timeit(bwd, args.iters)
                reads = 2 * nbytes * (2 if "two-pass" in bpath else 1)
                bb = reads + nbytes * (streams_b - 2) + mbytes * (2 if "two-pass" in bpath else 1)
                record(f"{tag} bwd {shape} [{bpath}]", ms, bytes_=bb, lib_ms=lib_b,
                       note="dy, x, dx" + (", dres" if relu else "") + (" + 2nd dy, x read" if "two-pass" in bpath else ""))
            C.set_bn_two_pass(0)
        if C.bn_resident_error():
            raise RuntimeError("resident BatchNorm grid barrier timed out")

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

    if "adamw" in want:
        from b200ddp.models import build_model
        # BERT-base MLM: 154 tensors, so the decay group spans two 120-tensor tables
        shapes = [tuple(p.shape) for p in build_model("bert-base").parameters()]
        for dtype, label in ((torch.float32, "fp32"), (torch.bfloat16, "bf16+master")):
            params = [torch.nn.Parameter(torch.randn(*s, device=dev).to(dtype)) for s in shapes]
            n = sum(p.numel() for p in params)
            for p in params:
                p.grad = torch.randn_like(p) * 1e-3
            groups = [{"params": [p for p in params if p.ndim >= 2], "weight_decay": 0.01},
                      {"params": [p for p in params if p.ndim < 2], "weight_decay": 0.0}]
            opt = FusedAdamW(groups, lr=1e-4, max_grad_norm=1000.0)
            ms = timeit(lambda: opt.step(), args.iters)
            # fp32: norm pass reads g (4 B); update reads g, p, m, v (16 B) and writes p, m, v (12 B) = 32 B/element.
            # bf16+master: norm reads g (2 B); update reads g, master, m, v (14 B) and writes p, master, m, v (14 B) = 30 B.
            byt = n * (32 if dtype == torch.float32 else 30)
            ref = [torch.nn.Parameter(p.detach().float().clone()) for p in params]
            for r, p in zip(ref, params):
                r.grad = p.grad.float()
            ropt = torch.optim.AdamW([{"params": [r for r in ref if r.ndim >= 2], "weight_decay": 0.01},
                                      {"params": [r for r in ref if r.ndim < 2], "weight_decay": 0.0}], lr=1e-4, fused=True)

            def lib_step():
                torch.nn.utils.clip_grad_norm_(ref, 1000.0)
                ropt.step()
            lib = timeit(lib_step, args.iters)
            record(f"clip+adamw bert-base {len(params)} tensors {label}", ms, bytes_=byt, lib_ms=lib,
                   note="lib = clip_grad_norm_ + AdamW(fused=True) (fp32)")
            del params, ref, opt, ropt

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

    if "lmloss" in want:
        # Fused LM-head cross-entropy (forward + backward, no logits) against cross_entropy(linear(h, E, b)) at the head
        # shapes of the README's GPT-2 (8 x 1024, padded vocabulary with its bias), SmolLM (8 x 2048) and Qwen2.5 (4 x 2048)
        # runs.  FLOPs: 4 head GEMMs fused (the forward is recomputed), 3 unfused.  Memory: rise of the peak over fwd+bwd.
        print(f"lm-head loss on {card()}", flush=True)
        for label, N, V, H, with_bias in (("gpt2", 8192, 50304, 768, True), ("smollm", 16384, 49152, 576, False),
                                          ("qwen", 8192, 151936, 1536, False)):
            h = torch.randn(N, H, device=dev).to(torch.bfloat16).requires_grad_(True)
            w = (torch.randn(V, H, device=dev) * 0.02).to(torch.bfloat16).requires_grad_(True)
            t = torch.randint(0, V, (N,), device=dev)
            b = None
            if with_bias:
                b = torch.zeros(V, device=dev, dtype=torch.bfloat16)
                b[50257:] = -1e4

            def fused():
                torch.autograd.grad(Fn.linear_cross_entropy(h, w, t, b), (h, w))

            def unfused():
                torch.autograd.grad(Fn.cross_entropy(Fn.linear(h, w, b), t), (h, w))

            def peak_rise(fn):
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                fn()
                torch.cuda.synchronize()
                return (torch.cuda.max_memory_allocated() - base) / 1e9
            gemm = 2.0 * N * V * H
            mf, mu = peak_rise(fused), peak_rise(unfused)
            lib = timeit(unfused, args.iters)
            record(f"lm-loss {label} fwd+bwd {N}x{V}x{H}", timeit(fused, args.iters), flops=4 * gemm, lib_ms=lib,
                   note=f"lib = unfused native linear + cross_entropy ({3 * gemm / lib / 1e9:.0f} TFLOP/s); peak rise "
                        f"fused {mf:.2f} GB, unfused {mu:.2f} GB")
            if label == "qwen":                                        # backward slice width
                C_ = _ext.get()
                tt = t.clone()
                loss, lse, rl = C_.lm_loss_fwd(h.detach(), w.detach(), tt, None, -100)
                g1 = torch.ones(1, device=dev)
                for sl in (4096, 8192, 16384, 32768):
                    ms = timeit(lambda: C_.lm_loss_bwd(h.detach(), w.detach(), tt, None, lse, rl, g1, -100, sl), args.iters)
                    record(f"lm-loss qwen bwd slice {sl}", ms, flops=3 * gemm, note=f"dlogits buffer {N * sl * 2 / 1e6:.0f} MB")
            del h, w

    if "sparse" in want:
        # Sparse masked-LM prediction: the decoder + cross-entropy on the labelled rows only, at the BERT-base (16 x 512,
        # padded vocabulary 30528) and ModernBERT-base (2 x 8192, 50368) head shapes with 15 % and 30 % of the rows labelled,
        # against the unfused linear + cross_entropy and the dense fused op, all with the decoder bias trained.  FLOPs count
        # the useful work: 3 head GEMMs over the labelled rows.  Then compaction + gather + scatter alone, and the rise of
        # the peak memory over fwd+bwd of each.
        print(f"sparse prediction on {card()}", flush=True)
        for label, N, V, H in (("bert", 8192, 30528, 768), ("modernbert", 16384, 50368, 768)):
            h = torch.randn(N, H, device=dev).to(torch.bfloat16).requires_grad_(True)
            w = (torch.randn(V, H, device=dev) * 0.02).to(torch.bfloat16).requires_grad_(True)
            b = torch.zeros(V, device=dev, dtype=torch.bfloat16).requires_grad_(True)
            for frac in (0.15, 0.30):
                g = torch.Generator(device=dev).manual_seed(0)
                t = torch.randint(0, V, (N,), device=dev, generator=g)
                t = torch.where(torch.rand(N, device=dev, generator=g) < frac, t, torch.full_like(t, -100))
                labelled = int((t >= 0).sum())

                def unfused():
                    torch.autograd.grad(Fn.cross_entropy(Fn.linear(h, w, b), t), (h, w, b))

                def dense():
                    torch.autograd.grad(Fn.linear_cross_entropy(h, w, t, b), (h, w, b))

                def sparse():
                    torch.autograd.grad(Fn.linear_cross_entropy(h, w, t, b, sparse=True), (h, w, b))

                def compaction():
                    index, count, _ = Fn.compact_rows(t, -100, V)
                    C.scatter_rows(C.gather_rows(h.detach(), index, count), index, count)

                def peak_rise(fn):
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    fn()
                    torch.cuda.synchronize()
                    return (torch.cuda.max_memory_allocated() - base) / 1e9
                useful = 3 * 2.0 * labelled * V * H
                rise = {n: peak_rise(f) for n, f in (("unfused", unfused), ("dense", dense), ("sparse", sparse))}
                tag = f"{label} {N}x{V}x{H} {int(frac * 100)}% ({labelled} rows)"
                lib = timeit(unfused, args.iters)
                dense_ms = timeit(dense, args.iters)
                record(f"sparse lm-loss {tag}", timeit(sparse, args.iters), flops=useful, lib_ms=lib,
                       note=f"lib = unfused linear + cross_entropy; dense fused {dense_ms:.3f} ms; peak rise sparse "
                            f"{rise['sparse']:.2f} GB, dense {rise['dense']:.2f} GB, unfused {rise['unfused']:.2f} GB")
                record(f"compact+gather+scatter {tag}", timeit(compaction, args.iters), bytes_=N * 8 + 4 * N * H * 2,
                       note="bytes: targets, and the [T, H] gather and scatter (read + write each)")
            del h, w, b

    if "moe" in want:
        # Granite-3.0-1B-A400M's MoE layer at batch 8 x 2048: T = 16384 tokens, k = 8 of E = 32 experts, H = 1024, I = 512.
        # TFLOP/s count the routed rows only (T * k), not the padding of the 128-aligned segments.  Baselines: torch._grouped_mm
        # on the same permuted rows and offsets, and our dense GEMM over the same total M with one weight.  Uniform routing
        # (random logits) and skewed routing (a bias falling by 0.25 per expert index).
        print(f"moe on {card()}", flush=True)
        T, k, E, H, I = 16384, 8, 32, 1024, 512
        R = T * k
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(T, H, device=dev, generator=gen).to(torch.bfloat16)
        wgu = (torch.randn(E, 2 * I, H, device=dev, generator=gen) * 0.02).to(torch.bfloat16)
        wd = (torch.randn(E, H, I, device=dev, generator=gen) * 0.02).to(torch.bfloat16)
        for routing in ("uniform", "skewed"):
            logits = torch.randn(T, E, device=dev, generator=gen)
            if routing == "skewed":
                logits = logits - 0.25 * torch.arange(E, device=dev)
            logits = logits.to(torch.bfloat16)
            ids, gates, _ = C.moe_route(logits, k, True)
            counts, offsets, fwd, inv, tiles = C.moe_permute(ids, E)
            cap = fwd.numel()
            c = counts.tolist()
            print(f"  {routing}: rows per expert min {min(c)} max {max(c)}, {int(offsets[-1])} of {cap} permuted rows used", flush=True)
            xp = C.moe_gather(x, fwd, k)
            gu = C.moe_gemm(xp, wgu, tiles, False)
            h = C.swiglu_fwd(gu)
            y = C.moe_gemm(h, wd, tiles, False)
            dy = torch.randn(cap, H, device=dev, generator=gen).to(torch.bfloat16)
            dgu = torch.randn(cap, 2 * I, device=dev, generator=gen).to(torch.bfloat16)
            ends = offsets[1:].contiguous()

            def grouped(tag, ours, flops, lib, lib_note):
                lib_ms = None
                note = ""
                try:
                    lib_ms = timeit(lib, args.iters)
                    note = f"lib = {lib_note}"
                except Exception as err:                          # report the baseline as missing, never substitute it
                    note = f"{lib_note} did not run: {type(err).__name__}: {str(err).splitlines()[0][:120]}"
                record(f"moe {routing} {tag}", timeit(ours, args.iters), flops=flops, lib_ms=lib_ms, note=note)

            f_gu, f_dn = 2.0 * R * 2 * I * H, 2.0 * R * H * I
            grouped("fwd gate_up", lambda: C.moe_gemm(xp, wgu, tiles, False), f_gu,
                    lambda: torch._grouped_mm(xp, wgu.transpose(1, 2), offs=ends), "torch._grouped_mm")
            grouped("fwd down", lambda: C.moe_gemm(h, wd, tiles, False), f_dn,
                    lambda: torch._grouped_mm(h, wd.transpose(1, 2), offs=ends), "torch._grouped_mm")
            grouped("dgrad gate_up", lambda: C.moe_gemm(dgu, wgu, tiles, True), f_gu,
                    lambda: torch._grouped_mm(dgu, wgu, offs=ends), "torch._grouped_mm")
            grouped("dgrad down", lambda: C.moe_gemm(dy, wd, tiles, True), f_dn,
                    lambda: torch._grouped_mm(dy, wd, offs=ends), "torch._grouped_mm")
            grouped("wgrad gate_up", lambda: C.moe_gemm_wgrad(dgu, xp, offsets), f_gu,
                    lambda: torch._grouped_mm(dgu.t(), xp, offs=ends), "torch._grouped_mm")
            grouped("wgrad down", lambda: C.moe_gemm_wgrad(dy, h, offsets), f_dn,
                    lambda: torch._grouped_mm(dy.t(), h, offs=ends), "torch._grouped_mm")
            if routing == "uniform":                              # our dense GEMM over the same total M, one weight
                a, b = xp[:R].contiguous(), wgu[0].contiguous()
                record(f"moe dense gemm_nt {R}x{2 * I}x{H}", timeit(lambda: C.gemm(a, b, None, False, False, 0, False, None),
                                                                     args.iters), flops=f_gu, note="dense reference at equal M")
            # memory-bound passes: bytes each kernel must move
            dout = torch.randn(T, H, device=dev, generator=gen).to(torch.bfloat16)
            dgates = torch.randn(T, k, device=dev, generator=gen)
            dprob = torch.randn(E, device=dev, generator=gen)
            record(f"moe {routing} router fwd (+aux sums)", timeit(lambda: C.moe_route(logits, k, True), args.iters),
                   bytes_=T * E * 2 + T * k * (4 + 2))
            record(f"moe {routing} router bwd", timeit(lambda: C.moe_router_bwd(logits, ids, dgates, dprob), args.iters),
                   bytes_=T * E * 2 * 2 + T * k * (4 + 4))
            record(f"moe {routing} permute (3 kernels + memset)", timeit(lambda: C.moe_permute(ids, E), args.iters),
                   bytes_=R * 4 * 2 + cap * 4 + R * 4, note="bytes: ids read twice, both row maps written")
            record(f"moe {routing} gather", timeit(lambda: C.moe_gather(x, fwd, k), args.iters),
                   bytes_=R * H * 2 + cap * H * 2 + cap * 4)
            record(f"moe {routing} combine", timeit(lambda: C.moe_combine(y, inv, gates), args.iters),
                   bytes_=R * H * 2 + T * H * 2 + R * (4 + 2))
            record(f"moe {routing} combine bwd", timeit(lambda: C.moe_combine_bwd(dout, y, fwd, gates), args.iters),
                   bytes_=R * H * 2 * 2 + cap * H * 2 + R * (4 + 2 + 4), note="dout read once per routed row")
            del xp, gu, h, y, dy, dgu

    if "vit" in want:
        # ViT-B/16 at batch 64: the patch embedding (patchify + wgmma linear + assembly, and its backward) against torchvision's
        # conv_proj + flatten + cat + position add in bf16, and attention on the image-as-document stream against SDPA flash
        # per image on [64, 12, 197, 64]
        import torch.nn.functional as F
        print(f"vit kernels on {card()}", flush=True)
        B, p, D, H, d, per = 64, 16, 768, 12, 64, 197
        T = Fn.image_token_rows(B, per)
        g = torch.Generator(device="cuda").manual_seed(4)
        images = torch.randn(B, 3, 224, 224, device=dev, generator=g).to(torch.bfloat16)
        w = (torch.randn(D, 3, p, p, device=dev, generator=g) / 28).to(torch.bfloat16).requires_grad_(True)
        bias, cls, pos = (torch.randn(*s, device=dev, generator=g).to(torch.bfloat16).requires_grad_(True)
                          for s in ((D,), (1, 1, D), (1, per, D)))
        K = 3 * p * p

        def tv_embed():
            x = F.conv2d(images, w, bias, stride=p).flatten(2).transpose(1, 2)
            return torch.cat([cls.expand(B, -1, -1), x], 1) + pos
        # bytes: image read, patch matrix write + read, GEMM output write + read, tokens write (weights are small)
        fwd_bytes = 2 * (B * 3 * 224 * 224 + 2 * T * K + 3 * T * D)
        with torch.no_grad():
            record(f"vit patch_embed fwd B{B} p{p}", timeit(lambda: Fn.patch_embed(images, w, bias, cls, pos), args.iters),
                   bytes_=fwd_bytes, lib_ms=timeit(tv_embed, args.iters), note="lib = conv2d + flatten + cat + pos add")
        y = Fn.patch_embed(images, w, bias, cls, pos)
        dy = torch.randn(T, D, device=dev, generator=g).to(torch.bfloat16)
        yl = tv_embed()
        dyl = dy[:B * per].view(B, per, D)
        # bytes: dy read, patch-row gradient write + read, patch matrix read (the wgrad GEMM), d pos write
        bwd_bytes = 2 * (3 * T * D + T * K + per * D)
        record(f"vit patch_embed bwd B{B} p{p}", timeit(lambda: torch.autograd.grad(y, (w, bias, cls, pos), dy, retain_graph=True),
                                                          args.iters),
               bytes_=bwd_bytes, lib_ms=timeit(lambda: torch.autograd.grad(yl, (w, bias, cls, pos), dyl, retain_graph=True), args.iters),
               note="lib = the same through conv2d's backward")
        bounds = Fn.image_token_bounds(B, per, dev)
        qkv = torch.randn(T, 3 * H * d, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(T, H * d, device=dev, generator=g).to(torch.bfloat16)
        fwd_flops = 4.0 * d * H * B * per * per                   # the visible pairs only
        x = qkv[:B * per].view(B, per, -1).detach().clone().requires_grad_(True)
        q, k, v = (t.reshape(B, per, H, d).transpose(1, 2) for t in x.split(H * d, dim=-1))

        def sdpa():
            return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, per, H * d)
        with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.FLASH_ATTENTION):
            lib = timeit(lambda: sdpa().detach(), args.iters)
            record(f"vit attention fwd B{B} {per} tokens/image", timeit(lambda: C.packed_attention_fwd(qkv, bounds, H), args.iters),
                   flops=fwd_flops, lib_ms=lib, note=f"stream of {T} rows; lib = SDPA flash [{B}, {H}, {per}, {d}] + output transpose")
            o, lse = C.packed_attention_fwd(qkv, bounds, H)
            ya = sdpa()
            lib = timeit(lambda: torch.autograd.grad(ya, x, dout[:B * per].view(B, per, -1), retain_graph=True), args.iters)
            record(f"vit attention bwd B{B} {per} tokens/image",
                   timeit(lambda: C.packed_attention_bwd(dout, qkv, o, lse, bounds, H), args.iters), flops=2.5 * fwd_flops,
                   lib_ms=lib, note="lib = SDPA flash backward into qkv")
        del x, q, k, v, ya, y, yl

    if "clip" in want:
        # CLIP's contrastive loss at B = 256 pairs per rank, 512-wide features: clip_loss forward and backward against the
        # torch expression in bf16 (normalise, two logit matrices, two cross-entropies); N = 2048 stands for 8 ranks through
        # the label offset (the gathered features are inputs here, no collective).  And QuickGELU at CLIP-B's MLP width.
        import torch.nn.functional as F
        print(f"clip kernels on {card()}", flush=True)
        B, D = 256, 512
        g = torch.Generator(device="cuda").manual_seed(5)
        for N in (256, 2048):
            rank = N // B - 1
            u_img = torch.nn.functional.normalize(torch.randn(B, D, device=dev, generator=g), dim=-1).to(torch.bfloat16).requires_grad_(True)
            u_txt = torch.nn.functional.normalize(torch.randn(B, D, device=dev, generator=g), dim=-1).to(torch.bfloat16).requires_grad_(True)
            others = [torch.nn.functional.normalize(torch.randn(N - B, D, device=dev, generator=g), dim=-1).to(torch.bfloat16) for _ in range(2)]
            scale = torch.tensor(2.6592, device=dev, requires_grad=True)

            def gathered():
                return (torch.cat([others[0][:rank * B], u_img, others[0][rank * B:]]),
                        torch.cat([others[1][:rank * B], u_txt, others[1][rank * B:]]))

            def native():
                U_img, U_txt = gathered()
                return Fn._ContrastiveLoss.apply(u_img, u_txt, U_img, U_txt, scale, rank * B)

            labels = torch.arange(B, device=dev) + rank * B

            def torch_expr():
                U_img, U_txt = gathered()
                s = scale.exp()
                return (F.cross_entropy((u_img @ U_txt.t()).float() * s, labels) +
                        F.cross_entropy((u_txt @ U_img.t()).float() * s, labels)) / 2
            flops = 2 * 2.0 * B * N * D                             # the two similarity GEMMs
            with torch.no_grad():
                record(f"clip loss fwd B{B} N{N}", timeit(native, args.iters), flops=flops, lib_ms=timeit(torch_expr, args.iters),
                       note="fused cross-entropy on wgmma similarities; lib = bf16 matmuls + F.cross_entropy")
            ln, lt = native(), torch_expr()
            record(f"clip loss bwd B{B} N{N}",
                   timeit(lambda: torch.autograd.grad(ln, (u_img, u_txt, scale), retain_graph=True), args.iters), flops=2 * flops,
                   lib_ms=timeit(lambda: torch.autograd.grad(lt, (u_img, u_txt, scale), retain_graph=True), args.iters),
                   note="four GEMMs from the forward's dz; lib = autograd through the torch expression")
            del ln, lt
        x = torch.randn(256 * 50, 3072, device=dev, generator=g).to(torch.bfloat16)
        dy = torch.randn_like(x)
        n = x.numel()
        record("quick_gelu fwd 12800x3072 bf16", timeit(lambda: C.clip.quick_gelu_fwd(x), args.iters), bytes_=n * 4,
               lib_ms=timeit(lambda: x * torch.sigmoid(1.702 * x), args.iters), note="lib = x * torch.sigmoid(1.702 * x)")
        xr = x.detach().clone().requires_grad_(True)
        yl = xr * torch.sigmoid(1.702 * xr)
        record("quick_gelu bwd 12800x3072 bf16", timeit(lambda: C.clip.quick_gelu_bwd(dy, x), args.iters), bytes_=n * 6,
               lib_ms=timeit(lambda: torch.autograd.grad(yl, xr, dy, retain_graph=True), args.iters), note="lib = autograd of the same")
        del x, dy, xr, yl

    if "cross" in want:
        # Cross-attention at bart-base's shape (12 heads, batch 16): Sq = Sk = 512, and Sq 128 over Sk 1024.  Full rows
        # against SDPA (flash); right-padded rows (source / target lengths U[S/4, S]) and packed rows (the denoising data's
        # pairs, documents U[64, S]) against SDPA with the dense [B, 1, Sq, Sk] mask.  FLOPs count the visible pairs only:
        # forward 4 d H sum(q_end - q_start), backward 2.5x that.
        import torch.nn.functional as F
        from b200ddp.data import SyntheticDenoising
        from b200ddp.ops import cross_bounds, document_bounds
        H, d, B = 12, 64, 16
        g = torch.Generator(device=dev).manual_seed(0)
        for Sq, Sk in ((512, 512), (128, 1024)):
            q = torch.randn(B * Sq, H * d, device=dev, generator=g).to(torch.bfloat16)
            kv = torch.randn(B * Sk, 2 * H * d, device=dev, generator=g).to(torch.bfloat16)
            dout = torch.randn(B * Sq, H * d, device=dev, generator=g).to(torch.bfloat16)
            rng = torch.Generator().manual_seed(1)
            src_l = torch.randint(Sk // 4, Sk + 1, (B,), generator=rng)
            tgt_l = torch.randint(Sq // 4, Sq + 1, (B,), generator=rng)
            pad = lambda n, S: (torch.arange(S)[None, :] < n[:, None]).long()
            packed = SyntheticDenoising(samples=4 * B, seq_len=min(Sq, Sk), min_len=64, pack=True)
            pick = torch.linspace(0, len(packed) - 1, B).long()
            ids = lambda t, S: torch.nn.functional.pad(t, (0, S - t.shape[1]))
            cases = [("full", torch.ones(B, Sk, dtype=torch.long), torch.ones(B, Sq, dtype=torch.long), None),
                     ("padded", pad(src_l, Sk), pad(tgt_l, Sq), None),
                     ("packed", ids(packed.X[pick], Sk), ids(packed.Y[pick].clamp(min=0), Sq), packed.bos_token_id)]
            for label, src, tgt, bos in cases:
                enc, _ = document_bounds(src.to(dev), bos, 0)
                dec, _ = document_bounds(tgt.to(dev), bos, 0)
                qb, kb = cross_bounds(enc, dec)
                vis = float((qb[..., 1] - qb[..., 0]).sum())
                fwd_flops = 4.0 * d * H * vis
                xq = q.view(B, Sq, H * d).detach().clone().requires_grad_(True)
                xkv = kv.view(B, Sk, 2 * H * d).detach().clone().requires_grad_(True)
                qh = xq.view(B, Sq, H, d).transpose(1, 2)
                kh, vh = (t.reshape(B, Sk, H, d).transpose(1, 2) for t in xkv.split(H * d, -1))
                j = torch.arange(Sk, device=dev)
                mask = None if label == "full" else ((j >= qb[..., :1]) & (j < qb[..., 1:]))[:, None]
                if mask is not None:
                    mask |= ~mask.any(-1, keepdim=True) & (j == 0)      # a query that sees nothing: one key, not a NaN row

                def sdpa():
                    return F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask).transpose(1, 2).reshape(B, Sq, H * d)
                lib_name = "SDPA flash" if mask is None else "SDPA dense bool mask"
                name = f"cross {label} B{B} Sq{Sq} Sk{Sk} H{H}"
                lib = timeit(lambda: sdpa().detach(), args.iters)
                record(f"{name} fwd", timeit(lambda: C.cross.cross_attention_fwd(q, kv, qb, H), args.iters), flops=fwd_flops,
                       lib_ms=lib, note=f"lib = {lib_name} + output transpose")
                o, lse = C.cross.cross_attention_fwd(q, kv, qb, H)
                y = sdpa()
                dy = dout.view(B, Sq, H * d)
                lib = timeit(lambda: torch.autograd.grad(y, (xq, xkv), dy, retain_graph=True), args.iters)
                record(f"{name} bwd", timeit(lambda: C.cross.cross_attention_bwd(dout, q, kv, o, lse, qb, kb, H), args.iters),
                       flops=2.5 * fwd_flops, lib_ms=lib, note=f"lib = {lib_name} backward into q and kv")
                del xq, xkv, y
    if "t5" in want:
        # T5's relative position bias at t5-base's attention shape (12 heads, batch 32 x 512), encoder (segment) and
        # decoder (causal), on full, right-padded (lengths U[S/4, S]) and packed rows (documents U[64, S], first fit).
        # Three things per case: the bias kernels (forward with the table gather, backward with the dtable finish and the
        # fold into the embedding), the same kernels without bias (the price of the bias), and SDPA with the float
        # [1, H, S, S] bias (requiring grad) plus the document mask, which is what transformers' T5 attention amounts to.
        # FLOPs count the visible pairs only: forward 4 d H pairs, backward 2.5x that.
        import torch.nn.functional as F
        H, d, B, S = 12, 64, 32, 512
        g = torch.Generator(device=dev).manual_seed(0)
        qkv = torch.randn(B * S, 3 * H * d, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(B * S, H * d, device=dev, generator=g).to(torch.bfloat16)
        weight = (torch.randn(32, H, device=dev, generator=g) * 2).to(torch.bfloat16)
        rng = torch.Generator().manual_seed(1)
        lens = torch.randint(S // 4, S + 1, (B,), generator=rng)
        packed = torch.zeros(B, S, 2, dtype=torch.int32)
        for r in range(B):
            at = 0
            while at < S:
                n = min(int(torch.randint(64, S + 1, (1,), generator=rng)), S - at)
                packed[r, at:at + n, 0], packed[r, at:at + n, 1] = at, at + n
                at += n
        pos = torch.arange(S)
        layouts = [("full", torch.stack([torch.zeros(B, S, dtype=torch.int32), torch.full((B, S), S, dtype=torch.int32)], -1)),
                   ("padded", torch.stack([torch.zeros(B, S, dtype=torch.int32), torch.where(pos < lens[:, None], lens[:, None], 0).int()], -1)
                    * (pos < lens[:, None])[..., None]),
                   ("packed", packed)]
        for causal in (False, True):
            plain = "causal_attention" if causal else "packed_attention"
            for label, bounds in layouts:
                bounds = bounds.to(dev).contiguous()
                vis = Fn._causal_mask(bounds, S, dev) if causal else Fn._bounds_mask(bounds, S, dev)
                fwd_flops = 4.0 * d * H * float(vis.sum())
                name = f"t5 {'decoder causal' if causal else 'encoder segment'} {label} B{B} S{S} H{H}"

                def bias_fwd():
                    table = C.t5.relative_table_fwd(weight, Fn._relative_buckets(not causal, 32, dev))
                    return C.t5.relative_attention_fwd(qkv, bounds, table, H, causal)
                table = C.t5.relative_table_fwd(weight, Fn._relative_buckets(not causal, 32, dev))
                o, lse = C.t5.relative_attention_fwd(qkv, bounds, table, H, causal)

                def bias_bwd():
                    dqkv, dtable = C.t5.relative_attention_bwd(dout, qkv, o, lse, bounds, table, H, causal)
                    return C.t5.relative_table_bwd(dtable, Fn._relative_buckets(not causal, 32, dev), weight)
                po, plse = getattr(C, plain + "_fwd")(qkv, bounds, H)
                # SDPA: q k^T (scale 1) + bias[h, i, j] + the mask; a row that sees nothing keeps key 0 (not a NaN row)
                x = qkv.view(B, S, 3 * H * d).detach().clone().requires_grad_(True)
                qh, kh, vh = (t.reshape(B, S, H, d).transpose(1, 2) for t in x.split(H * d, -1))
                dense = table[:, (pos[None, :] - pos[:, None]).clamp(-128, 128).to(dev) + 128].to(torch.bfloat16)[None]
                dense = dense.detach().requires_grad_(True)
                keep = vis | (~vis.any(-1, keepdim=True) & (torch.arange(S, device=dev) == 0))
                mask = torch.zeros(B, 1, S, S, device=dev, dtype=torch.bfloat16).masked_fill(~keep[:, None], float("-inf"))

                def sdpa():
                    return F.scaled_dot_product_attention(qh, kh, vh, attn_mask=dense + mask, scale=1.0).transpose(1, 2).reshape(B, S, H * d)
                record(f"{name} fwd", timeit(bias_fwd, args.iters), flops=fwd_flops, lib_ms=timeit(lambda: sdpa().detach(), args.iters),
                       note="lib = SDPA with the float bias + mask")
                record(f"{name} fwd no bias", timeit(lambda: getattr(C, plain + "_fwd")(qkv, bounds, H), args.iters), flops=fwd_flops,
                       note=f"{plain}_fwd: the same kernel without the bias")
                y = sdpa()
                dy = dout.view(B, S, H * d)
                record(f"{name} bwd", timeit(bias_bwd, args.iters), flops=2.5 * fwd_flops,
                       lib_ms=timeit(lambda: torch.autograd.grad(y, (x, dense), dy, retain_graph=True), args.iters),
                       note="incl. dtable finish and fold; lib = SDPA backward into qkv and the bias")
                record(f"{name} bwd no bias", timeit(lambda: getattr(C, plain + "_bwd")(dout, qkv, po, plse, bounds, H), args.iters),
                       flops=2.5 * fwd_flops, note=f"{plain}_bwd: the same kernels without the bias")
                del x, y, dense, mask
    if "convnext" in want:
        # ConvNeXt-T's depthwise 7x7 at batch 64, its four stage shapes: forward, data gradient, and weight + bias gradient
        # against cuDNN's F.conv2d(groups=C) on channels_last bf16.  Bytes: 4 per element (read one tensor, write one) for
        # the forward and the data gradient; for the weight gradient 4 per element (dy and x) plus the fp32 partials
        # written and read once.
        import torch.nn.functional as F
        print(f"convnext kernels on {card()}", flush=True)
        for B, H, W, Cn in ((64, 56, 56, 96), (64, 28, 28, 192), (64, 14, 14, 384), (64, 7, 7, 768)):
            g = torch.Generator(device="cuda").manual_seed(Cn)
            x = torch.randn(B, H, W, Cn, device=dev, generator=g).to(torch.bfloat16)
            dy = torch.randn(B, H, W, Cn, device=dev, generator=g).to(torch.bfloat16)
            w = (torch.randn(Cn, 1, 7, 7, device=dev, generator=g) / 7).to(torch.bfloat16)
            b = torch.randn(Cn, device=dev, generator=g).to(torch.bfloat16)
            w2 = w.reshape(Cn, 49)
            xl, dyl = x.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2)          # the same memory as channels_last NCHW
            n = x.numel()
            tag = f"[{B},{H},{W},{Cn}]"
            record(f"dwconv7x7 fwd {tag}", timeit(lambda: C.convnext.dwconv_fwd(x, w2, b), args.iters), bytes_=4 * n,
                   lib_ms=timeit(lambda: F.conv2d(xl, w, b, padding=3, groups=Cn), args.iters), note="lib = cuDNN channels_last")
            record(f"dwconv7x7 dgrad {tag}", timeit(lambda: C.convnext.dwconv_dgrad(dy, w2), args.iters), bytes_=4 * n,
                   lib_ms=timeit(lambda: torch.ops.aten.convolution_backward(dyl, xl, w, [Cn], [1, 1], [3, 3], [1, 1], False, [0, 0], Cn,
                                                                              [True, False, False]), args.iters),
                   note="lib = cuDNN channels_last data gradient")
            slots = B * -(-H // min(H, 16 if min(W, 56) <= 28 else 8)) * -(-W // min(W, 56))
            record(f"dwconv7x7 wgrad {tag}", timeit(lambda: C.convnext.dwconv_wgrad(dy, x), args.iters),
                   bytes_=4 * n + 2 * 4 * slots * 50 * Cn,
                   lib_ms=timeit(lambda: torch.ops.aten.convolution_backward(dyl, xl, w, [Cn], [1, 1], [3, 3], [1, 1], False, [0, 0], Cn,
                                                                              [False, True, True]), args.iters),
                   note=f"{slots} partial slots; lib = cuDNN channels_last weight + bias gradient")
            del x, dy, xl, dyl

    if "swin" in want:
        # Swin's shifted-window attention at Swin-T's four stage shapes (batch 64) and Swin-B's first, forward and backward
        # against torchvision's arithmetic under bf16 (roll, window partition, dense scores with the gathered bias and the
        # mask, softmax, reverse partition and roll) and against SDPA with the per-window float bias + mask, both around
        # the same qkv.  Bytes, from shapes: forward reads qkv and writes o and lse; backward reads qkv, o, dO and lse,
        # writes dqkv, and writes and reads the fp32 table partials.
        import torch.nn.functional as F
        from b200ddp.ops import swin_relative_position_index
        print(f"swin kernels on {card()}", flush=True)
        index = swin_relative_position_index(dev)

        def partition(t, B, Hs, Ws, sy, sx):                  # [B H W, X] -> [B nW, 49, X] in torchvision's order
            X = t.shape[-1]
            t = torch.roll(t.view(B, Hs, Ws, X), shifts=(-sy, -sx), dims=(1, 2)) if sy or sx else t.view(B, Hs, Ws, X)
            return t.view(B, Hs // 7, 7, Ws // 7, 7, X).permute(0, 1, 3, 2, 4, 5).reshape(-1, 49, X)

        def unpartition(t, B, Hs, Ws, sy, sx):
            X = t.shape[-1]
            t = t.view(B, Hs // 7, Ws // 7, 7, 7, X).permute(0, 1, 3, 2, 4, 5).reshape(B, Hs, Ws, X)
            return (torch.roll(t, shifts=(sy, sx), dims=(1, 2)) if sy or sx else t).reshape(B * Hs * Ws, X)

        def window_mask(Hs, Ws, s):
            c = torch.arange(Hs, device=dev)
            ry = (c >= Hs - 7).long() + (c >= Hs - s).long() if s else torch.zeros_like(c)
            c = torch.arange(Ws, device=dev)
            rx = (c >= Ws - 7).long() + (c >= Ws - s).long() if s else torch.zeros_like(c)
            reg = (ry[:, None] * 3 + rx[None, :]).view(Hs // 7, 7, Ws // 7, 7).permute(0, 2, 1, 3).reshape(-1, 49)
            return torch.where(reg[:, :, None] != reg[:, None, :], -100.0, 0.0).to(torch.bfloat16)

        for name, B, Hs, heads, s in (("swin-t stage 1", 64, 56, 3, 3), ("swin-t stage 2", 64, 28, 6, 3), ("swin-t stage 3", 64, 14, 12, 3),
                                      ("swin-t stage 4", 64, 7, 24, 0), ("swin-b stage 1", 64, 56, 4, 3)):
            Cn, nrows = 32 * heads, B * Hs * Hs
            g = torch.Generator(device="cuda").manual_seed(heads)
            qkv = torch.randn(nrows, 3 * Cn, device=dev, generator=g).to(torch.bfloat16)
            table = (torch.randn(169, heads, device=dev, generator=g) * 0.02).to(torch.bfloat16)
            dout = torch.randn(nrows, Cn, device=dev, generator=g).to(torch.bfloat16)
            t32 = table.float()
            o, lse = C.swin.attention_fwd(qkv, t32, B, Hs, Hs, s, s)
            nw = B * (Hs // 7) ** 2
            mask = window_mask(Hs, Hs, s) if s else None

            def torchvision_fwd(qkv, table):
                x = partition(qkv, B, Hs, Hs, s, s).reshape(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
                q, k, v = x[0] * 32 ** -0.5, x[1], x[2]
                attn = q.matmul(k.transpose(-2, -1)) + table[index].view(49, 49, heads).permute(2, 0, 1).unsqueeze(0)
                if mask is not None:
                    attn = (attn.view(B, -1, heads, 49, 49) + mask[None, :, None]).view(-1, heads, 49, 49)
                y = F.softmax(attn, dim=-1).matmul(v).transpose(1, 2).reshape(-1, 49, Cn)
                return unpartition(y, B, Hs, Hs, s, s)

            def sdpa_fwd(qkv, table):
                x = partition(qkv, B, Hs, Hs, s, s).reshape(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
                bias = table[index].view(49, 49, heads).permute(2, 0, 1).unsqueeze(0)
                if mask is not None:
                    bias = (bias.unsqueeze(0) + mask[None, :, None]).reshape(-1, heads, 49, 49)
                    bias = bias.expand(B, -1, heads, 49, 49).reshape(-1, heads, 49, 49)
                y = F.scaled_dot_product_attention(x[0], x[1], x[2], attn_mask=bias).transpose(1, 2).reshape(-1, 49, Cn)
                return unpartition(y, B, Hs, Hs, s, s)

            fwd_bytes = nrows * (3 * Cn * 2 + Cn * 2 + heads * 4)
            bwd_bytes = nrows * (3 * Cn * 2 + 2 * Cn * 2 + heads * 4 + 3 * Cn * 2) + 2 * heads * nw * 169 * 4
            tag = f"{name} [{B}, {Hs}x{Hs}, {heads} heads, shift {s}]"
            lib = {}
            for lname, fn in (("torchvision", torchvision_fwd), ("sdpa", sdpa_fwd)):
                qg, tg = qkv.clone().requires_grad_(True), table.clone().requires_grad_(True)
                lib[lname + " fwd"] = timeit(lambda: fn(qg, tg), args.iters)
                y = fn(qg, tg)
                lib[lname + " bwd"] = timeit(lambda: torch.autograd.grad(y, (qg, tg), dout, retain_graph=True), args.iters)
                del y
            record(f"window attention fwd {tag}", timeit(lambda: C.swin.attention_fwd(qkv, t32, B, Hs, Hs, s, s), args.iters),
                   bytes_=fwd_bytes, lib_ms=lib["torchvision fwd"], note=f"lib = torchvision's arithmetic; sdpa {lib['sdpa fwd']:.4f} ms")
            record(f"window attention bwd {tag}", timeit(lambda: C.swin.attention_bwd(dout, qkv, o, lse, t32, B, Hs, Hs, s, s), args.iters),
                   bytes_=bwd_bytes, lib_ms=lib["torchvision bwd"],
                   note=f"incl. the table-gradient finish; lib = torchvision's arithmetic; sdpa {lib['sdpa bwd']:.4f} ms")
            del qkv, dout, o, lse

        # Swin V2's cosine window attention (window 8) at Swin-V2-T's four stage shapes at 256 x 256 (batch 64) and
        # Swin-V2-B's first, forward and backward against the attention part of torchvision's shifted_window_attention
        # with logit_scale under bf16 (roll, window partition, F.normalize of q and k, cosine scores times the scale, the
        # gathered bias and the mask, softmax, reverse partition and roll), around the same qkv, table and scale.  Bytes as
        # above, with 226 partial columns per window.
        index8 = swin_relative_position_index(dev, 8)

        def partition8(t, B, Hs, sy):
            X = t.shape[-1]
            t = torch.roll(t.view(B, Hs, Hs, X), shifts=(-sy, -sy), dims=(1, 2)) if sy else t.view(B, Hs, Hs, X)
            return t.view(B, Hs // 8, 8, Hs // 8, 8, X).permute(0, 1, 3, 2, 4, 5).reshape(-1, 64, X)

        def unpartition8(t, B, Hs, sy):
            X = t.shape[-1]
            t = t.view(B, Hs // 8, Hs // 8, 8, 8, X).permute(0, 1, 3, 2, 4, 5).reshape(B, Hs, Hs, X)
            return (torch.roll(t, shifts=(sy, sy), dims=(1, 2)) if sy else t).reshape(B * Hs * Hs, X)

        def window_mask8(Hs, s):
            c = torch.arange(Hs, device=dev)
            r = (c >= Hs - 8).long() + (c >= Hs - s).long()
            reg = (r[:, None] * 3 + r[None, :]).view(Hs // 8, 8, Hs // 8, 8).permute(0, 2, 1, 3).reshape(-1, 64)
            return torch.where(reg[:, :, None] != reg[:, None, :], -100.0, 0.0).to(torch.bfloat16)

        for name, B, Hs, heads, s in (("swin-v2-t stage 1", 64, 64, 3, 4), ("swin-v2-t stage 2", 64, 32, 6, 4),
                                      ("swin-v2-t stage 3", 64, 16, 12, 4), ("swin-v2-t stage 4", 64, 8, 24, 0),
                                      ("swin-v2-b stage 1", 64, 64, 4, 4)):
            Cn, nrows = 32 * heads, B * Hs * Hs
            g = torch.Generator(device="cuda").manual_seed(heads)
            qkv = torch.randn(nrows, 3 * Cn, device=dev, generator=g).to(torch.bfloat16)
            t32 = 16 * torch.sigmoid(torch.randn(225, heads, device=dev, generator=g))
            sc32 = torch.full((heads,), 10.0, device=dev)
            table, scale = t32.to(torch.bfloat16), sc32.to(torch.bfloat16)
            dout = torch.randn(nrows, Cn, device=dev, generator=g).to(torch.bfloat16)
            o, lse = C.swin_v2.attention_fwd(qkv, t32, sc32, B, Hs, Hs, s, s)
            nw = B * (Hs // 8) ** 2
            mask = window_mask8(Hs, s) if s else None

            def torchvision_fwd(qkv, table, scale):
                x = partition8(qkv, B, Hs, s).reshape(-1, 64, 3, heads, 32).permute(2, 0, 3, 1, 4)
                attn = F.normalize(x[0], dim=-1) @ F.normalize(x[1], dim=-1).transpose(-2, -1)
                attn = attn * scale.view(heads, 1, 1) + table[index8].view(64, 64, heads).permute(2, 0, 1).unsqueeze(0)
                if mask is not None:
                    attn = (attn.view(B, -1, heads, 64, 64) + mask[None, :, None]).view(-1, heads, 64, 64)
                y = F.softmax(attn, dim=-1).matmul(x[2]).transpose(1, 2).reshape(-1, 64, Cn)
                return unpartition8(y, B, Hs, s)

            fwd_bytes = nrows * (3 * Cn * 2 + Cn * 2 + heads * 4)
            bwd_bytes = nrows * (3 * Cn * 2 + 2 * Cn * 2 + heads * 4 + 3 * Cn * 2) + 2 * heads * nw * 226 * 4
            tag = f"{name} [{B}, {Hs}x{Hs}, {heads} heads, shift {s}]"
            qg, tg, sg = qkv.clone().requires_grad_(True), table.clone().requires_grad_(True), scale.clone().requires_grad_(True)
            lib_fwd = timeit(lambda: torchvision_fwd(qg, tg, sg), args.iters)
            y = torchvision_fwd(qg, tg, sg)
            lib_bwd = timeit(lambda: torch.autograd.grad(y, (qg, tg, sg), dout, retain_graph=True), args.iters)
            del y
            record(f"cosine window attention fwd {tag}", timeit(lambda: C.swin_v2.attention_fwd(qkv, t32, sc32, B, Hs, Hs, s, s), args.iters),
                   bytes_=fwd_bytes, lib_ms=lib_fwd, note="lib = torchvision's shifted_window_attention arithmetic with logit_scale")
            record(f"cosine window attention bwd {tag}",
                   timeit(lambda: C.swin_v2.attention_bwd(dout, qkv, o, lse, t32, sc32, B, Hs, Hs, s, s), args.iters),
                   bytes_=bwd_bytes, lib_ms=lib_bwd,
                   note="incl. the table / scale gradient finish; lib = torchvision's arithmetic with logit_scale")
            del qkv, dout, o, lse, qg, tg, sg

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

    if "mamba" in want:
        # Mamba's causal conv1d + SiLU and selective scan at mamba-130m's and mamba-370m's layer shapes (8 x 2048 rows, E 1536 /
        # 2048, dt rank 48 / 64) on fixed, right-padded (lengths U[256, 2048]) and packed rows.  Algorithmic bytes, from shapes:
        # conv forward reads x and writes u; its backward reads du and x, writes dx and the fp32 weight partials.  Scan
        # forward reads u, delta_raw, z, B and C, writes y and the fp32 chunk start states; its backward reads dy, u,
        # delta_raw, z, B and C (4 E + 32 columns per row) and the start states, writes du, d delta_raw, dz (3 E) and the
        # x_proj-output gradient (R + 32), and writes and reads the fp32 chunk carries (one start-state size each way).  The torch reference (fp32 arithmetic, a loop over
        # the sequence like transformers' slow_forward) is the baseline: the conv forward, and the scan forward timed
        # over 2 calls.
        from b200ddp.ops import causal_conv1d, causal_conv1d_reference, document_bounds, selective_scan, selective_scan_reference
        print(f"mamba kernels on {card()}", flush=True)
        Bm, Sm = 8, 2048
        for label, E, R in (("mamba-130m", 1536, 48), ("mamba-370m", 2048, 64)):
            g = torch.Generator(device="cuda").manual_seed(E)
            for layout in ("fixed", "padded", "packed"):
                ids = torch.randint(2, 1000, (Bm, Sm), device=dev, generator=g)
                if layout != "fixed":
                    lens = torch.randint(256, Sm + 1, (Bm, 1), device=dev, generator=g)
                    ids = torch.where(torch.arange(Sm, device=dev) < lens, ids, 0)
                    if layout == "packed":
                        ids = torch.where(torch.rand(Bm, Sm, device=dev, generator=g) < 1 / 512, 1, ids) * (ids != 0)
                bounds = document_bounds(ids, 1 if layout == "packed" else None, None if layout == "fixed" else 0)[0].to(torch.int32)
                xz = torch.randn(Bm, Sm, 2 * E, device=dev, generator=g).to(torch.bfloat16)
                w = (torch.randn(E, 1, 4, device=dev, generator=g) * 0.5).to(torch.bfloat16)
                cb = torch.zeros(E, device=dev, dtype=torch.bfloat16)
                dr = torch.randn(Bm, Sm, E, device=dev, generator=g).to(torch.bfloat16)
                xbc = torch.randn(Bm, Sm, R + 32, device=dev, generator=g).to(torch.bfloat16)
                A_log = torch.log(torch.arange(1, 17.0, device=dev)).repeat(E, 1)
                D, dtb = torch.ones(E, device=dev), torch.full((E,), -4.0, device=dev)
                T = Bm * Sm
                w32, b32, x2 = w.reshape(E, 4).float(), cb.float(), xz.view(T, 2 * E)
                u2 = C.mamba.conv_fwd(x2, w32, b32, bounds)
                ms = timeit(lambda: C.mamba.conv_fwd(x2, w32, b32, bounds), args.iters)
                lib = timeit(lambda: causal_conv1d_reference(xz, w, cb, bounds), args.iters)
                record(f"{label} conv fwd {layout}", ms, bytes_=T * E * 2 * 2, lib_ms=lib, note="lib: torch reference")
                du = torch.randn(T, E, device=dev, generator=g).to(torch.bfloat16)
                ms = timeit(lambda: C.mamba.conv_bwd(du, x2, w32, b32, bounds), args.iters)
                record(f"{label} conv bwd {layout}", ms, bytes_=T * E * 2 * 3 + 2 * 5 * E * 4 * Bm * Sm // 32)
                sargs = (u2, dr.view(T, E), xbc.view(T, R + 32), x2, A_log, D, dtb, bounds)
                y, hst, sumd = C.mamba.scan_fwd(*sargs)
                state_bytes = hst.numel() * 4
                ms = timeit(lambda: C.mamba.scan_fwd(*sargs), args.iters)
                u3 = u2.view(Bm, Sm, E)
                lib = timeit(lambda: selective_scan_reference(u3, dr, xbc, xz, A_log, D, dtb, bounds), 2, flush=False)
                record(f"{label} scan fwd {layout}", ms, bytes_=T * (4 * E * 2 + 32 * 2) + state_bytes, lib_ms=lib,
                       note="lib: torch reference")
                dy = torch.randn(T, E, device=dev, generator=g).to(torch.bfloat16)
                ms = timeit(lambda: C.mamba.scan_bwd(dy, *sargs, hst, sumd), args.iters)
                record(f"{label} scan bwd {layout}", ms, bytes_=T * (7 * E * 2 + (32 + R + 32) * 2) + 3 * state_bytes)

    if "mamba2" in want:
        # Mamba-2's conv over in_proj's xBC columns, chunked SSD scan and gated RMSNorm at mamba2-130m's and mamba2-370m's layer
        # shapes (8 x 2048 rows, 24 / 32 heads of 64, state 128, W = 2E + 256 + H) on fixed, right-padded (lengths U[256, 2048])
        # and packed rows.  Algorithmic counts, from shapes (ssd_counts): the SSD's matrix products per (chunk, head), each
        # counted once and over full 64 x 64 tiles, and the bytes each pass must move: bf16 rows read and written once, the
        # fp32 chunk states [B, chunks, H, 128, 64] written by the state kernel, read and written by the pass, and read by the
        # output (forward) or gradient (backward) kernel, two such buffers in the backward.
        from b200ddp.ops import document_bounds
        print(f"mamba2 kernels on {card()}", flush=True)
        Bm, Sm, L, N, P = 8, 2048, 64, 128, 64

        def ssd_counts(T, H, nc):
            E = H * P
            CD = E + 2 * N
            state = Bm * nc * H * N * P * 4
            f_fwd = Bm * nc * (2 * L * L * N + H * 2 * L * P * (L + 2 * N))
            f_bwd = Bm * nc * (2 * L * L * N + H * (2 * L * N * P * 2 + 2 * L * L * P * 2 + 2 * L * P * N * 5 + 2 * L * L * N * 2))
            b_fwd = T * (CD + H + E) * 2 + 4 * state
            b_bwd = T * (E + CD + H + CD + H) * 2 + 8 * state
            return f_fwd, b_fwd, f_bwd, b_bwd

        for label, H in (("mamba2-130m", 24), ("mamba2-370m", 32)):
            E = H * P
            CD, W = E + 2 * N, 2 * E + 2 * N + H
            g = torch.Generator(device="cuda").manual_seed(E)
            for layout in ("fixed", "padded", "packed"):
                ids = torch.randint(2, 1000, (Bm, Sm), device=dev, generator=g)
                if layout != "fixed":
                    lens = torch.randint(256, Sm + 1, (Bm, 1), device=dev, generator=g)
                    ids = torch.where(torch.arange(Sm, device=dev) < lens, ids, 0)
                    if layout == "packed":
                        ids = torch.where(torch.rand(Bm, Sm, device=dev, generator=g) < 1 / 512, 1, ids) * (ids != 0)
                bounds = document_bounds(ids, 1 if layout == "packed" else None, None if layout == "fixed" else 0)[0].to(torch.int32)
                T = Bm * Sm
                zx = torch.randn(T, W, device=dev, generator=g).to(torch.bfloat16)
                w32 = torch.randn(CD, 4, device=dev, generator=g) * 0.5
                b32 = torch.zeros(CD, device=dev)
                xw, z, dt = zx[:, E:E + CD], zx[:, :E], zx[:, W - H:]
                u = C.mamba2.conv_fwd(xw, w32, b32, bounds)
                ms = timeit(lambda: C.mamba2.conv_fwd(xw, w32, b32, bounds), args.iters)
                record(f"{label} conv fwd {layout}", ms, bytes_=T * CD * 2 * 2)
                du = torch.randn(T, CD, device=dev, generator=g).to(torch.bfloat16)
                dzx = torch.empty_like(zx)
                ms = timeit(lambda: C.mamba2.conv_bwd(du, xw, w32, b32, bounds, dzx[:, E:E + CD]), args.iters)
                record(f"{label} conv bwd {layout}", ms, bytes_=T * CD * 2 * 3 + 2 * 5 * CD * 4 * Bm * Sm // 32)
                A_log = torch.log(torch.arange(1, H + 1.0, device=dev))
                D, dtb = torch.ones(H, device=dev), torch.full((H,), -4.0, device=dev)
                f_fwd, b_fwd, f_bwd, b_bwd = ssd_counts(T, H, (Sm + L - 1) // L)
                ms = timeit(lambda: C.mamba2.ssd_fwd(u, dt, A_log, D, dtb, bounds), args.iters)
                record(f"{label} ssd fwd {layout}", ms, flops=f_fwd, bytes_=b_fwd)
                dy = torch.randn(T, E, device=dev, generator=g).to(torch.bfloat16)
                ms = timeit(lambda: C.mamba2.ssd_bwd(dy, u, dt, A_log, D, dtb, bounds, dzx[:, W - H:]), args.iters)
                record(f"{label} ssd bwd {layout}", ms, flops=f_bwd, bytes_=b_bwd)
                y = torch.randn(T, E, device=dev, generator=g).to(torch.bfloat16)
                nw = torch.ones(E, device=dev, dtype=torch.bfloat16)
                out, rstd = C.mamba2.gated_norm_fwd(y, z, nw, 1e-5)
                ms = timeit(lambda: C.mamba2.gated_norm_fwd(y, z, nw, 1e-5), args.iters)
                record(f"{label} gated norm fwd {layout}", ms, bytes_=T * E * 2 * 3)
                ms = timeit(lambda: C.mamba2.gated_norm_bwd(dy, y, z, nw, rstd, dzx[:, :E]), args.iters)
                record(f"{label} gated norm bwd {layout}", ms, bytes_=T * E * 2 * 5)

    if "mae" in want:
        # The masked autoencoder's kernels at ViT-MAE-base's shapes (196 patches, 49 kept, encoder 768 wide, decoder 512 wide
        # with 16 heads of 32 over 197 rows per image), batch 64 and 256.  image_attention forward and backward against SDPA
        # on [B, 16, 197, 32] around the same qkv; mae_loss forward and backward against the torch expression under bf16; the
        # shuffle, the masked patch embedding's gather / assemble and the unshuffle against their torch expressions.  Bytes,
        # from shapes: what each kernel must read and write once (attention: qkv, o, lse; backward also dO and dqkv).
        import torch.nn.functional as F
        from b200ddp.ops import image_token_rows, mae_patchify
        print(f"mae kernels on {card()}", flush=True)
        N, keep, D, E, H, P = 196, 49, 768, 512, 16, 768
        for B in (64, 256):
            g = torch.Generator(device="cuda").manual_seed(B)
            S = N + 1
            Td, Te = image_token_rows(B, S), image_token_rows(B, keep + 1)
            # image attention
            qkv = torch.randn(Td, 3 * E, device=dev, generator=g).to(torch.bfloat16)
            dout = torch.randn(Td, E, device=dev, generator=g).to(torch.bfloat16)
            o, lse = C.mae.attention_fwd(qkv, B, S)

            def sdpa(qkv):
                x = qkv[:B * S].view(B, S, 3, H, 32).permute(2, 0, 3, 1, 4)
                return F.scaled_dot_product_attention(x[0], x[1], x[2]).transpose(1, 2).reshape(B * S, E)

            qg = qkv.clone().requires_grad_(True)
            lib_f = timeit(lambda: sdpa(qg), args.iters)
            y = sdpa(qg)
            lib_b = timeit(lambda: torch.autograd.grad(y, qg, dout[:B * S], retain_graph=True), args.iters)
            del y
            rows_ = B * S
            fwd_bytes = rows_ * (3 * E * 2 + E * 2 + H * 4)
            bwd_bytes = rows_ * (3 * E * 2 + 2 * E * 2 + H * 4 + 3 * E * 2)
            attn_flops = 4.0 * 32 * H * B * S * S
            tag = f"[{B}, {H}, {S}, 32]"
            record(f"image_attention fwd {tag}", timeit(lambda: C.mae.attention_fwd(qkv, B, S), args.iters), flops=attn_flops,
                   lib_ms=lib_f, note=f"{fwd_bytes / 1e6:.1f} MB; lib = SDPA")
            record(f"image_attention bwd {tag}", timeit(lambda: C.mae.attention_bwd(dout, qkv, o, lse, B, S), args.iters),
                   flops=2.5 * attn_flops, lib_ms=lib_b, note=f"{bwd_bytes / 1e6:.1f} MB; lib = SDPA")
            del qkv, dout, o, lse, qg
            # loss
            images = torch.randn(B, 3, 224, 224, device=dev, generator=g).to(torch.bfloat16)
            noise = torch.rand(B, N, device=dev, generator=g)
            ids_keep, ids_restore = C.mae.shuffle(noise, keep)
            pred = torch.randn(Td, P, device=dev, generator=g).to(torch.bfloat16)
            dloss = torch.ones(1, device=dev)
            mask = (ids_restore >= keep).to(torch.bfloat16)

            def torch_loss(pred):
                t = mae_patchify(images, 16)
                return ((((pred[:B * S].view(B, S, P)[:, 1:] - t) ** 2).mean(-1) * mask).sum() / mask.sum()).float()

            pg = pred.clone().requires_grad_(True)
            lib_f = timeit(lambda: torch_loss(pg), args.iters)
            lt = torch_loss(pg)
            lib_b = timeit(lambda: torch.autograd.grad(lt, pg, retain_graph=True), args.iters)
            del lt
            loss_bytes = B * (N - keep) * P * 2 * 2 + B * N * 4
            record(f"mae_loss fwd B={B}", timeit(lambda: C.mae.loss(pred, images, ids_restore, keep, False), args.iters),
                   bytes_=loss_bytes, lib_ms=lib_f, note="lib = torch expression, bf16")
            record(f"mae_loss bwd B={B}", timeit(lambda: C.mae.loss_bwd(dloss, pred, images, ids_restore, keep, False), args.iters),
                   bytes_=loss_bytes + Td * P * 2, lib_ms=lib_b, note="lib = torch expression, bf16")
            del pred, pg
            # shuffle, masked patch embedding, unshuffle
            record(f"mae_shuffle B={B}", timeit(lambda: C.mae.shuffle(noise, keep), args.iters), bytes_=B * N * 4 + B * (N + keep) * 4,
                   lib_ms=timeit(lambda: torch.argsort(torch.argsort(noise, 1), 1), args.iters), note="lib = two torch.argsort")
            record(f"mae_patchify B={B}", timeit(lambda: C.mae.patchify(images, ids_keep, 16, Te), args.iters),
                   bytes_=2 * B * keep * P * 2,
                   lib_ms=timeit(lambda: torch.gather(mae_patchify(images, 16), 1, ids_keep.long()[..., None].expand(-1, -1, P)), args.iters),
                   note="lib = patchify + gather")
            yd = torch.randn(Te, D, device=dev, generator=g).to(torch.bfloat16)
            cls = torch.randn(D, device=dev, generator=g).to(torch.bfloat16)
            pos = torch.randn(S, D, device=dev, generator=g).to(torch.bfloat16)
            record(f"mae_patch_assemble B={B}", timeit(lambda: C.mae.patch_assemble(yd, cls, pos, ids_keep), args.iters),
                   bytes_=2 * Te * D * 2 + B * keep * D * 2,
                   lib_ms=timeit(lambda: yd[:B * (keep + 1)].view(B, keep + 1, D)[:, 1:] + pos[1:][ids_keep.long()], args.iters),
                   note="lib = gather + add")
            ye = torch.randn(Te, E, device=dev, generator=g).to(torch.bfloat16)
            mtok = torch.randn(E, device=dev, generator=g).to(torch.bfloat16)
            dpos = torch.randn(S, E, device=dev, generator=g).to(torch.bfloat16)
            dz = torch.randn(Td, E, device=dev, generator=g).to(torch.bfloat16)

            def torch_unshuffle():
                x = ye[:B * (keep + 1)].view(B, keep + 1, E)
                x_ = torch.cat([x[:, 1:], mtok.view(1, 1, E).expand(B, N - keep, E)], 1)
                x_ = torch.gather(x_, 1, ids_restore.long()[..., None].expand(-1, -1, E))
                return torch.cat([x[:, :1], x_], 1) + dpos

            record(f"mae_unshuffle B={B}", timeit(lambda: C.mae.unshuffle(ye, mtok, dpos, ids_restore, keep, Td), args.iters),
                   bytes_=B * keep * E * 2 + Td * E * 2, lib_ms=timeit(torch_unshuffle, args.iters), note="lib = cat, gather, cat, add")
            record(f"mae_unshuffle bwd B={B}", timeit(lambda: C.mae.unshuffle_bwd(dz, ids_keep, ids_restore, Te), args.iters),
                   bytes_=B * S * E * 2 + Te * E * 2)
            del images, yd, ye, dz

    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump({"peaks": {"hbm_gbs": hbm, "bf16_tflops_burst": tf_burst, "bf16_tflops_sustained": tf_sust, "source": src},
                   "rows": rows}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
