"""Command line + process lifecycle (reference ``ddp.py:80-121`` ``setup``/``cleanup`` and ``ddp.py:291-314`` ``main``).

All 16 reference flags keep their names and defaults; ``--local-rank`` is accepted as an
alias because ``torch.distributed.launch`` on torch >= 2 passes that spelling.  New flags
select the model, the DDP transport and its knobs, resume, and the CUDA-graph step.

Mode selection mirrors the reference: CPU (``--no_cuda`` / no GPU), single GPU, single-process multi-GPU
``DataParallel`` (no launcher, several GPUs), DDP (launcher present).  Unlike the reference, a launcher
with ``--no_cuda`` (or no GPU) gives a working gloo DDP run instead of a crash.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch
import torch.distributed as dist

from ..models import MODEL_REGISTRY, build_model
from ..utils import (get_logger_with_rank, redirect_warnings_to_logger, resolve_local_rank, env_int, set_seed)

log = None


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="H100-native DDP training template")
    # ---- reference flags (ddp.py:293-308), same names and defaults -----------------------------
    p.add_argument("--global-step", type=int, default=0, help="(reference flag; resume uses --resume_from)")
    p.add_argument("--no_cuda", action="store_true")
    p.add_argument("--output_dir", type=str, default="outputs")
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--gradient_accumulation_steps", type=int, default=1)
    p.add_argument("--per_gpu_train_batch_size", type=int, default=32)
    p.add_argument("--max_steps", type=int, default=0)
    p.add_argument("--logging_steps", type=int, default=100)
    p.add_argument("--save_steps", type=int, default=1000)
    p.add_argument("--num_train_epochs", type=int, default=10)
    p.add_argument("--warmup_steps", type=int, default=100)
    p.add_argument("--max_grad_norm", type=float, default=1000.0)
    p.add_argument("--local_rank", "--local-rank", dest="local_rank", type=int, default=-1)
    p.add_argument("--fp16", action="store_true", help="bf16 weights + fp32 master weights (the reference's apex O2 intent)")
    p.add_argument("--loss_scale", type=int, default=0, help="accepted for parity; bf16 needs no loss scaling")
    p.add_argument("--fp16_opt_level", type=str, default="O2", help="accepted for parity")
    # ---- new flags --------------------------------------------------------------------------------
    p.add_argument("--model", type=str, default="foo", choices=sorted(MODEL_REGISTRY))
    p.add_argument("--loss", type=str, default=None, choices=[None, "mse", "ce"])
    p.add_argument("--lr", type=float, default=1e-3)
    p.add_argument("--momentum", type=float, default=0.0)
    p.add_argument("--weight_decay", type=float, default=0.0)
    p.add_argument("--dataset_size", type=int, default=100000)
    p.add_argument("--seq_len", type=int, default=512)
    p.add_argument("--backend", type=str, default="auto", choices=["auto", "b200", "nccl", "gloo"])
    p.add_argument("--bucket_cap_mb", type=float, default=None)
    p.add_argument("--gradient_as_bucket_view", action="store_true")
    p.add_argument("--find_unused_parameters", type=lambda s: s.lower() not in ("0", "false", "no"), default=True)
    p.add_argument("--no_broadcast_buffers", dest="broadcast_buffers", action="store_false")
    p.add_argument("--wire_dtype", type=str, default=None, choices=[None, "fp32", "bf16"])
    p.add_argument("--channels_last", action="store_true")
    p.add_argument("--cuda_graph", action="store_true", help="capture the whole optimizer step in a CUDA graph")
    p.add_argument("--resume_from", type=str, default=None, help="checkpoint dir, or 'latest' under --output_dir")
    p.add_argument("--log_file", type=str, default=None, help="also log to this file ({rank} is substituted)")
    p.add_argument("--no_tensorboard", action="store_true")
    p.add_argument("--tb_dir", type=str, default=None)
    p.add_argument("--eval_at_end", action="store_true")
    p.add_argument("--trace_dir", type=str, default=None,
                   help="write a torch.profiler chrome trace (trace_rank<r>.json) of --trace_steps optimizer steps here")
    p.add_argument("--trace_steps", type=int, default=3)
    p.add_argument("--trace_skip", type=int, default=10, help="optimizer steps to skip before tracing (warm-up, graph capture)")
    return p


def setup(args):
    """Device + mode selection, logger, process group, seeding; mutates ``args`` like the reference does."""
    global log
    if sys.platform == "win32":
        raise NotImplementedError("Unsupported Platform")
    args.local_rank = resolve_local_rank(args.local_rank)
    log = get_logger_with_rank("b200ddp", env_int("RANK", -1), args.local_rank, log_file=args.log_file)
    redirect_warnings_to_logger(log)
    have_cuda = torch.cuda.is_available() and not args.no_cuda
    if args.local_rank == -1:
        if have_cuda:
            device = torch.device("cuda")
            args.n_gpu = torch.cuda.device_count()
        else:
            log.critical("!!!! Using CPU for training !!!!")
            device = torch.device("cpu")
            args.n_gpu = 0
        args.world_size = 1
        args.node_rank = 0
        log.info("Using single-process training.", dict(n_gpu=args.n_gpu))
    else:
        if have_cuda:
            torch.cuda.set_device(args.local_rank)
            device = torch.device("cuda", args.local_rank)
            pg_backend = "nccl"       # bootstrap + baseline path; the data path is args.backend
            if args.backend == "gloo":
                pg_backend = "gloo"
        else:
            log.critical("!!!! Using CPU for training !!!!")
            device = torch.device("cpu")
            pg_backend = "gloo"
            args.backend = "gloo"
        log.warning("Initializing process group.")
        if pg_backend == "nccl":
            dist.init_process_group(backend="nccl", device_id=device)
        else:
            dist.init_process_group(backend=pg_backend)
        args.node_rank = dist.get_rank()      # (sic) the reference stores the GLOBAL rank here, ddp.py:104
        args.world_size = dist.get_world_size()
        log.info("Initialized distributed training process group.", dict(backend=dist.get_backend(), world_size=args.world_size,
                                                                        transport=args.backend))
        args.n_gpu = 1 if have_cuda else 0
    args.device = device
    args.train_batch_size = args.per_gpu_train_batch_size * max(1, args.n_gpu)
    set_seed(args.seed, args.n_gpu)
    log.warning("Finish setup.", dict(device=args.device, n_gpu=args.n_gpu, distributed_training=bool(args.local_rank != -1)))
    return log


def cleanup(args) -> None:
    if args.local_rank != -1:
        log.warning("Destroying process group.")
        try:
            from ..parallel.peer import PeerCollectives
            PeerCollectives.shutdown_all()
        except Exception:
            pass
        dist.destroy_process_group()


def evaluate(args, trainer):
    return trainer.evaluate()


def main(argv=None) -> int:
    from .trainer import Trainer
    args = build_parser().parse_args(argv)
    setup(args)
    model = build_model(args.model)
    trainer = Trainer(args, model, log)
    trainer.train()
    if args.eval_at_end:
        log.info("Evaluation.", evaluate(args, trainer))
    cleanup(args)
    log.warning("Process exited.")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
