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

from ..models import MODEL_REGISTRY, build_model, model_entry
from ..utils import (get_logger_with_rank, redirect_warnings_to_logger, resolve_local_rank, env_int, set_seed)

log = None


class _StoreGiven(argparse.Action):
    """Stores the value and records that the flag was given (``args.<dest>_given``), so a check can reject a flag that
    was passed even when its value equals the default."""

    def __call__(self, parser, namespace, values, option_string=None):
        setattr(namespace, self.dest, values)
        setattr(namespace, self.dest + "_given", True)


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
    p.add_argument("--optimizer", type=str, default="sgd", choices=["sgd", "adamw"],
                   help="fused SGD, or fused AdamW with fp32 masters (weight decay on ndim >= 2 parameters only)")
    p.add_argument("--adam_beta1", type=float, default=0.9)
    p.add_argument("--adam_beta2", type=float, default=0.999)
    p.add_argument("--adam_epsilon", type=float, default=1e-8)
    p.add_argument("--dataset_size", type=int, default=100000)
    p.add_argument("--seq_len", type=int, default=512, action=_StoreGiven,
                   help="token models: tokens per row (CLIP's captions are always 77 tokens and take no --seq_len)")
    p.add_argument("--backend", type=str, default="auto", choices=["auto", "b200", "nccl", "gloo"])
    p.add_argument("--bucket_cap_mb", type=float, default=None)
    p.add_argument("--gradient_as_bucket_view", action="store_true")
    p.add_argument("--find_unused_parameters", type=lambda s: s.lower() not in ("0", "false", "no"), default=True)
    p.add_argument("--no_broadcast_buffers", dest="broadcast_buffers", action="store_false")
    p.add_argument("--wire_dtype", type=str, default=None, choices=[None, "fp32", "bf16"])
    p.add_argument("--channels_last", action="store_true")
    p.add_argument("--cuda_graph", action="store_true", help="capture the whole optimizer step in a CUDA graph")
    p.add_argument("--fp8", action="store_true",
                   help="block linears on FP8 tensor cores (E4M3 x / W, E5M2 gradients); needs --model "
                        f"{_names(lambda e: e.fp8)}, --fp16 and a GPU")
    p.add_argument("--min_seq_len", type=int, default=None,
                   help="token models on right-padded rows: each row's length is uniform in [min_seq_len, --seq_len], padded "
                        "keys are hidden from attention (native key-padding or causal kernel on the GPU; needs --fp16 and "
                        f"--seq_len %% 128 == 0 there).  Needs --model {_names(lambda e: e.token_model)}.  Default: "
                        "fixed-length rows")
    p.add_argument("--pack", action="store_true",
                   help="token models on packed documents: documents with lengths uniform in [--min_seq_len, --seq_len], each "
                        "starting with the model's start id ([CLS] for BERT), packed first-fit decreasing into rows; "
                        "attention stays inside a document (native document-boundary or causal kernel on the GPU).  Needs "
                        f"--model {_names(lambda e: e.token_model)} and --min_seq_len < --seq_len")
    p.add_argument("--fused_lm_loss", action="store_true",
                   help="LM head and cross-entropy in one op that never builds the [tokens, vocab] logits (the head GEMM runs "
                        f"once more in the backward); needs --model {_names(lambda e: e.kind == 'causal')}, --loss ce, and "
                        "--fp16 on a GPU")
    p.add_argument("--sparse_prediction", action="store_true",
                   help="masked-LM encoders: run the vocabulary decoder and its cross-entropy on the labelled (masked) rows "
                        f"only, compacted on the device; needs --model {_names(lambda e: e.kind == 'encoder')}, --loss ce, and "
                        "--fp16 on a GPU")
    p.add_argument("--router_aux_loss_coef", type=float, default=None,
                   help=f"mixture-of-experts models ({_names(lambda e: e.moe)}): weight of the router load-balancing loss "
                        "added to the training loss (default: the preset's, 0.001); 0 turns it off and skips its statistics")
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
    check_seq_len_args(args)
    check_fp8_args(args)
    check_min_seq_len_args(args)
    check_pack_args(args)
    check_fused_lm_loss_args(args)
    check_sparse_prediction_args(args)
    check_moe_args(args)
    check_contrastive_args(args)
    check_seq2seq_args(args)
    check_speech_args(args)
    check_own_loss_args(args)
    args.train_batch_size = args.per_gpu_train_batch_size * max(1, args.n_gpu)
    set_seed(args.seed, args.n_gpu)
    log.warning("Finish setup.", dict(device=args.device, n_gpu=args.n_gpu, distributed_training=bool(args.local_rank != -1)))
    return log


def _names(pick) -> str:
    """The registered models whose entries ``pick`` selects, as "a, b or c"."""
    names = [n for n, e in MODEL_REGISTRY.items() if pick(e)]
    return " or ".join([", ".join(names[:-1]), names[-1]]) if len(names) > 1 else names[0]


def check_seq_len_args(args) -> None:
    """A token model trains on at most its position table's rows (or its entry's lower ``max_seq_len``): reject a longer
    ``--seq_len`` up front instead of indexing past the table."""
    entry = model_entry(args.model)
    if not entry.token_model:
        return
    limit = entry.max_seq_len or entry.config.max_position
    if args.seq_len > limit:
        raise ValueError(f"--model {args.model} trains on up to {limit} positions; --seq_len must be at most {limit} "
                         f"(got {args.seq_len})")


def check_fp8_args(args) -> None:
    """``--fp8`` runs a dense token model's block linears on FP8 tensor cores, on top of bf16 weights on a GPU: reject
    every other combination up front."""
    if not getattr(args, "fp8", False):
        return
    entry = model_entry(args.model)
    if entry.moe:
        raise ValueError(f"--fp8 covers dense block linears; --model {args.model} is a mixture of experts, whose expert GEMMs "
                         f"have no FP8 path")
    if not entry.fp8:
        raise ValueError(f"--fp8 covers the block linears of the token models; it needs --model {_names(lambda e: e.fp8)} "
                         f"(got --model {args.model})")
    if not args.fp16:
        raise ValueError("--fp8 needs --fp16: the FP8 GEMMs read bf16 activations and weights")
    if getattr(args, "device", None) is None or args.device.type != "cuda":
        raise ValueError("--fp8 needs a CUDA device (it runs on FP8 tensor cores); drop --no_cuda")


def check_min_seq_len_args(args) -> None:
    """``--min_seq_len`` pads a token model's rows; on the GPU their attention runs on the bf16 key-padding or causal
    kernels (sequence length a multiple of 128): reject every other combination up front."""
    n = getattr(args, "min_seq_len", None)
    if n is None:
        return
    if not model_entry(args.model).token_model:
        raise ValueError(f"--min_seq_len pads token rows; it needs --model {_names(lambda e: e.token_model)} "
                         f"(got --model {args.model})")
    if not 1 <= n <= args.seq_len:
        raise ValueError(f"--min_seq_len must lie in [1, --seq_len = {args.seq_len}], got {n}")
    if getattr(args, "device", None) is not None and args.device.type == "cuda":
        if not args.fp16:
            raise ValueError("--min_seq_len on a GPU needs --fp16: the key-padding attention kernel reads bf16 activations")
        if args.seq_len % 128:
            raise ValueError(f"--min_seq_len on a GPU needs --seq_len to be a multiple of 128 (got {args.seq_len})")


def check_pack_args(args) -> None:
    """``--pack`` packs documents into a token model's padded rows, so it needs everything ``--min_seq_len`` needs (on
    the GPU: ``--fp16``, ``--seq_len`` % 128 == 0) and a ``--min_seq_len`` below ``--seq_len``."""
    if not getattr(args, "pack", False):
        return
    if not model_entry(args.model).token_model:
        raise ValueError(f"--pack packs token documents; it needs --model {_names(lambda e: e.token_model)} "
                         f"(got --model {args.model})")
    if not padding_on(args):
        raise ValueError("--pack needs --min_seq_len below --seq_len (documents have lengths in [--min_seq_len, --seq_len])")
    check_min_seq_len_args(args)


def check_fused_lm_loss_args(args) -> None:
    """``--fused_lm_loss`` moves a causal LM's head into a cross-entropy criterion: it needs such a model and ``--loss ce``,
    bf16 weights on a GPU (the native op is bf16), and a process per GPU (``DataParallel`` would split the hidden states
    across GPUs and gather them back to one)."""
    if not getattr(args, "fused_lm_loss", False):
        return
    if model_entry(args.model).kind != "causal":
        raise ValueError(f"--fused_lm_loss fuses a causal LM's head into its loss; it needs --model "
                         f"{_names(lambda e: e.kind == 'causal')} (got --model {args.model}); masked-LM encoders decode "
                         f"their labelled rows only with --sparse_prediction")
    if getattr(args, "loss", None) not in (None, "ce"):
        raise ValueError(f"--fused_lm_loss computes cross-entropy; it needs --loss ce (got --loss {args.loss})")
    if getattr(args, "device", None) is not None and args.device.type == "cuda":
        if not args.fp16:
            raise ValueError("--fused_lm_loss on a GPU needs --fp16: the fused head reads bf16 hidden states and weights")
        if args.local_rank == -1 and getattr(args, "n_gpu", 1) > 1:
            raise ValueError("--fused_lm_loss does not run under single-process multi-GPU DataParallel; launch one process "
                             "per GPU (torchrun) or make one GPU visible")


def check_sparse_prediction_args(args) -> None:
    """``--sparse_prediction`` moves a masked-LM encoder's decoder into a criterion that scores the labelled rows alone: it
    needs such a model and ``--loss ce``, bf16 weights on a GPU (the native op is bf16), and a process per GPU
    (``DataParallel`` would split the head's output across GPUs and gather it back to one)."""
    if not getattr(args, "sparse_prediction", False):
        return
    if model_entry(args.model).kind != "encoder":
        raise ValueError(f"--sparse_prediction decodes a masked-LM encoder's labelled rows only; it needs --model "
                         f"{_names(lambda e: e.kind == 'encoder')} (got --model {args.model})")
    if getattr(args, "loss", None) not in (None, "ce"):
        raise ValueError(f"--sparse_prediction computes cross-entropy; it needs --loss ce (got --loss {args.loss})")
    if getattr(args, "device", None) is not None and args.device.type == "cuda":
        if not args.fp16:
            raise ValueError("--sparse_prediction on a GPU needs --fp16: the fused decoder reads bf16 hidden states and weights")
        if args.local_rank == -1 and getattr(args, "n_gpu", 1) > 1:
            raise ValueError("--sparse_prediction does not run under single-process multi-GPU DataParallel; launch one process "
                             "per GPU (torchrun) or make one GPU visible")


def check_moe_args(args) -> None:
    """``--router_aux_loss_coef`` weights a mixture-of-experts model's load-balancing loss: it needs such a model and a
    non-negative value.  The loss (on by default) reads statistics the MoE layers keep from their forward, which
    single-process multi-GPU ``DataParallel`` leaves on its per-GPU replicas: that mode needs the loss turned off."""
    coef = getattr(args, "router_aux_loss_coef", None)
    moe = model_entry(args.model).moe
    if coef is not None and not moe:
        raise ValueError(f"--router_aux_loss_coef weights a mixture-of-experts router's loss; it needs --model "
                         f"{_names(lambda e: e.moe)} (got --model {args.model})")
    if coef is not None and not coef >= 0:
        raise ValueError(f"--router_aux_loss_coef must be >= 0, got {coef}")
    if moe and coef != 0 and getattr(args, "device", None) is not None and args.device.type == "cuda" \
            and args.local_rank == -1 and getattr(args, "n_gpu", 1) > 1:
        raise ValueError(f"--model {args.model} with its router load-balancing loss does not run under single-process "
                         f"multi-GPU DataParallel; launch one process per GPU (torchrun), make one GPU visible, or pass "
                         f"--router_aux_loss_coef 0")


def check_contrastive_args(args) -> None:
    """A contrastive model (CLIP) trains on image-caption pairs with its own loss over the global batch: the token-row
    flags, ``--fp8`` and an explicit ``--loss`` do not apply, single-process multi-GPU ``DataParallel`` would split the
    pairs across GPUs without gathering their features, and on a GPU the native loss needs a batch that is a multiple of 8."""
    if not model_entry(args.model).contrastive:
        return
    for flag, given in (("--fp8", getattr(args, "fp8", False)), ("--pack", getattr(args, "pack", False)),
                        ("--min_seq_len", getattr(args, "min_seq_len", None) is not None),
                        ("--fused_lm_loss", getattr(args, "fused_lm_loss", False)),
                        ("--sparse_prediction", getattr(args, "sparse_prediction", False)),
                        ("--seq_len", getattr(args, "seq_len_given", False)), ("--loss", getattr(args, "loss", None) is not None)):
        if given:
            raise ValueError(f"{flag} does not apply to --model {args.model}: CLIP trains on image-caption pairs (77-token "
                             f"captions) with its own contrastive loss")
    if getattr(args, "device", None) is not None and args.device.type == "cuda":
        if args.local_rank == -1 and getattr(args, "n_gpu", 1) > 1:
            raise ValueError(f"--model {args.model} does not run under single-process multi-GPU DataParallel (its loss gathers "
                             f"every rank's features); launch one process per GPU (torchrun) or make one GPU visible")
        if args.per_gpu_train_batch_size % 8:
            raise ValueError(f"--model {args.model} on a GPU needs --per_gpu_train_batch_size to be a multiple of 8 (the native "
                             f"contrastive loss), got {args.per_gpu_train_batch_size}")


def check_seq2seq_args(args) -> None:
    """An encoder-decoder (BART, T5) trains on source / target pairs whose sources are always right-padded, so on the GPU its
    attention always runs on the bf16 document kernels: it needs ``--fp16`` and ``--seq_len`` a multiple of 128 there.
    ``--seq_len`` bounds both sides (the position table's check covers it)."""
    if not model_entry(args.model).seq2seq:
        return
    if getattr(args, "device", None) is not None and args.device.type == "cuda":
        if not args.fp16:
            raise ValueError(f"--model {args.model} on a GPU needs --fp16: its attention kernels read bf16 activations")
        if args.seq_len % 128:
            raise ValueError(f"--model {args.model} on a GPU needs --seq_len to be a multiple of 128 (got {args.seq_len})")


def check_speech_args(args) -> None:
    """A speech model (Whisper) trains on rows that each hold one 30-second clip and its transcript: ``--pack`` does not
    apply.  ``--seq_len`` is the transcript row length."""
    if not model_entry(args.model).speech:
        return
    if getattr(args, "pack", False):
        raise ValueError(f"--pack does not apply to --model {args.model}: each row holds one 30-second clip and its transcript")


def check_own_loss_args(args) -> None:
    """A model that returns its own loss (MAE pretraining) trains on images alone: ``--loss`` and ``--seq_len`` do not
    apply, and single-process multi-GPU ``DataParallel`` would return one scalar loss per replica.  (``--fp8``, ``--pack``,
    ``--min_seq_len``, ``--fused_lm_loss`` and ``--sparse_prediction`` are rejected for every image model already.)"""
    if not model_entry(args.model).own_loss:
        return
    for flag, given in (("--loss", getattr(args, "loss", None) is not None), ("--seq_len", getattr(args, "seq_len_given", False))):
        if given:
            raise ValueError(f"{flag} does not apply to --model {args.model}: it trains on images with its own reconstruction loss")
    if getattr(args, "device", None) is not None and args.device.type == "cuda" and args.local_rank == -1 \
            and getattr(args, "n_gpu", 1) > 1:
        raise ValueError(f"--model {args.model} does not run under single-process multi-GPU DataParallel (each replica would "
                         f"return its own loss); launch one process per GPU (torchrun) or make one GPU visible")


def padding_on(args) -> bool:
    """Rows are padded (and the model must hide padded keys) when some row can be shorter than --seq_len."""
    n = getattr(args, "min_seq_len", None)
    return n is not None and n < args.seq_len


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
    kwargs = {"fp8": True} if args.fp8 else {}
    if args.fused_lm_loss:
        kwargs["fused_lm_loss"] = True
    if args.sparse_prediction:
        kwargs["sparse_prediction"] = True
    if args.router_aux_loss_coef is not None:
        kwargs["router_aux_loss_coef"] = args.router_aux_loss_coef
    if padding_on(args) or model_entry(args.model).seq2seq:      # an encoder-decoder's sources are always padded
        from ..data import SyntheticTokens
        kwargs["pad_token_id"] = SyntheticTokens.PAD_ID
        if args.pack:
            entry = model_entry(args.model)
            kwargs["cls_token_id" if entry.kind == "encoder" else "bos_token_id"] = entry.start_id
    model = build_model(args.model, **kwargs)
    trainer = Trainer(args, model, log)
    trainer.train()
    if args.eval_at_end:
        log.info("Evaluation.", evaluate(args, trainer))
    cleanup(args)
    log.warning("Process exited.")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
