#!/usr/bin/env python
"""Allreduce bus-bandwidth sweep 1 KB - 1 GB at 2/4/8 GPUs, peer-memory kernels vs NCCL.

  torchrun --nproc-per-node N bench/allreduce_sweep.py [--max_mb 1024] [--out sweep_N.json]

busbw = (S / t) * 2 (P-1) / P with S the payload bytes per rank (what nccl-tests prints); device-timed with
CUDA events, max over ranks, 5 warm-up + 20 timed launches per point, buffers rotated so each launch reads
memory that is not L2-resident from the previous one when the payload is below L2 size.
Roofline: bytes per direction per GPU = S (P-1)/P for two-shot / one-shot pull, ~S/P + S/P for NVLS.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, iters, world, dev, graph=True):
    """Device time per call.  The `iters` calls are captured into one CUDA graph and replayed, so the number
    is the collective itself (kernel + inter-GPU latency), not Python / launch overhead of either stack."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = None
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
        g.replay()
    dist.barrier(device_ids=[dev.index])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if g is not None:
        g.replay()
    else:
        for _ in range(iters):
            fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max_mb", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--blocks", type=str, default=None, help="CTA counts to try (default: 8,32,128 and the largest the kernels accept)")
    args = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    os.environ.setdefault("B200DDP_SCRATCH_MB", str(args.max_mb + 8))
    from b200ddp import _ext
    from b200ddp.parallel.peer import PeerCollectives
    max_blocks = int(_ext.get().MAX_COMM_BLOCKS)
    block_list = args.blocks or f"8,32,128,{max_blocks}"
    comm = PeerCollectives.get(None, dev, min_bytes=(args.max_mb + 16) << 20)
    sym_all = comm.symmetric_empty(args.max_mb * 1024 * 1024 // 4, torch.float32)
    results = {"world": world, "nvls": comm.nvls, "points": []}
    size = 1024
    while size <= args.max_mb * 1024 * 1024:
        n = size // 4
        rot = max(1, min(8, (256 << 20) // max(size, 1)))
        bufs = [torch.randn(n, device=dev) for _ in range(rot)]
        point = {"bytes": size}
        state = {"i": 0}

        def nccl():
            dist.all_reduce(bufs[state["i"] % rot]); state["i"] += 1
        ms = timed(nccl, args.iters, world, dev)
        point["nccl_us"] = ms * 1e3
        point["nccl_busbw"] = size / (ms * 1e-3) * 2 * (world - 1) / world / 1e9
        best = None
        algos = (["one_shot"] if size <= (1 << 20) else []) + ["two_shot"] + (["nvls"] if comm.nvls else []) + \
                (["nvls_one_shot"] if comm.nvls and size <= (4 << 20) else [])
        for wire in ("fp32", "bf16"):
            for algo in algos:
                cand = sorted({int(b) for b in block_list.split(",") if 0 < int(b) <= max_blocks})
                keep = [b for b in cand if not ((size < 65536 and b > 8) or (size >= (16 << 20) and b < 32))] or \
                       ([cand[0]] if size < 65536 else [cand[-1]])
                for blocks in keep:

                    def ours():
                        comm.allreduce_([bufs[state["i"] % rot]], wire=wire, algo=algo, blocks=blocks); state["i"] += 1
                    ms = timed(ours, args.iters, world, dev)
                    comm.check()
                    key = f"{algo}_{wire}_b{blocks}"
                    point[key + "_us"] = ms * 1e3
                    bw = size / (ms * 1e-3) * 2 * (world - 1) / world / 1e9
                    if wire == "fp32" and (best is None or bw > best[1]):
                        best = (key, bw)
                    if wire == "bf16":
                        point.setdefault("best_bf16wire_busbw", 0.0)
                        point["best_bf16wire_busbw"] = max(point["best_bf16wire_busbw"], bw)
        # in-place on symmetric memory (no staging copies): the like-for-like comparison with NCCL's in-place allreduce
        sym = sym_all[:n]
        sym.normal_()
        sbest = None
        for algo in ["two_shot"] + (["nvls"] if comm.nvls else []):
            for blocks in (8, 32, 64, 128, max_blocks):
                if (size < 65536 and blocks > 8) or (size >= (16 << 20) and blocks < 64):
                    continue
                ms = timed(lambda: comm.allreduce_symmetric_(sym, algo=algo, blocks=blocks), args.iters, world, dev)
                comm.check()
                bw = size / (ms * 1e-3) * 2 * (world - 1) / world / 1e9
                point[f"sym_{algo}_b{blocks}_us"] = ms * 1e3
                if sbest is None or bw > sbest[1]:
                    sbest = (f"sym_{algo}_b{blocks}", bw, ms * 1e3)
        point["best_symmetric"] = sbest[0]
        point["best_symmetric_busbw"] = sbest[1]
        point["best_symmetric_us"] = sbest[2]
        point["best_fp32wire"] = best[0]
        point["best_fp32wire_busbw"] = best[1]
        results["points"].append(point)
        if rank == 0:
            print(f"{size:>12d} B  nccl {point['nccl_us']:9.1f} us {point['nccl_busbw']:7.1f} GB/s | ours(fp32 wire) "
                  f"{best[0]:>22s} {best[1]:7.1f} GB/s | ours(bf16 wire) {point['best_bf16wire_busbw']:7.1f} GB/s | ours(symmetric in-place) "
                  f"{sbest[0]:>18s} {sbest[2]:8.1f} us {sbest[1]:7.1f} GB/s", flush=True)
        del bufs
        size *= 4
    if rank == 0 and args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    PeerCollectives.shutdown_all()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
