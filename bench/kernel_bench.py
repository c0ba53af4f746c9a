#!/usr/bin/env python
"""Per-kernel timings against the measured roofline (MEASURED_PEAKS.json: HBM copy GB/s, cuBLAS bf16 TFLOP/s).

  python bench/kernel_bench.py [--only gemm,fp8,attn,llama,qwen,conv,bn,sgd,adamw,ln,xent,mse,input] [--out kernels.json] [--iters 20]

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
        from b200ddp.data import SyntheticTokens
        print(f"llama kernels on {card()}", flush=True)
        B, S, H, Hkv, d, hidden, inter = 8, 2048, 9, 3, 64, 576, 1536
        M = B * S
        qkv = causal_lm_attention("gqa", B, S, H, Hkv, d, 49152, SyntheticTokens.LLAMA_BOS_ID, C.causal_gqa_attention_fwd,
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
        from b200ddp.data import SyntheticTokens
        print(f"qwen kernels on {card()}", flush=True)
        B, S, H, Hkv, d, hidden = 4, 2048, 12, 2, 128, 1536
        qkv = causal_lm_attention("d128", B, S, H, Hkv, d, 151936, SyntheticTokens.QWEN_BOS_ID, C.causal_attention_d128_fwd,
                                  C.causal_attention_d128_bwd)
        rmsnorm_rows(8192, hidden, 1e-6)
        rotary_rows(qkv, H, Hkv, d, S, 1e6)

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
