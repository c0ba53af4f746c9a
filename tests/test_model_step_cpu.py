"""``bench/model_step.py`` without a GPU: its table covers the models it should, it launches exactly the ``ddp.py`` runs
the per-model step scripts it replaced launched, it reads the trainer's ``Finished training.`` line as they did, and
every baseline builds."""
import importlib.util
import os
import shlex
import sys

import numpy as np
import pytest
import torch

from b200ddp.models import MODEL_REGISTRY
from b200ddp.utils import get_logger_with_rank

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("model_step", os.path.join(ROOT, "bench", "model_step.py"))
ms = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(ms)

MODELS = ["vit-b-16", "swin-t", "convnext-tiny", "clip-vit-b-32", "clip-vit-b-16", "bart-base", "bart-large", "t5-small",
          "t5-base", "mamba-130m", "mamba-370m", "mamba2-130m", "mamba2-370m", "whisper-tiny", "whisper-base", "whisper-small"]

# What the per-model scripts launched, recorded with subprocess.run patched, for each model's defaults, each command the
# README quotes and the optional flags.  A ddp.py run is its argv joined by spaces; a baseline run is the batch, seq_len,
# steps and min_seq_len it was given.
DDP = "{python} {root}/ddp.py"
OPT = "--fp16 --optimizer adamw"
FIXED = "--save_steps 0 --no_tensorboard --output_dir {tmp}/out --lr 1e-4"
PLANS = {
    "--model vit-b-16 --rounds 2": [
        f"{DDP} --model vit-b-16 {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model vit-b-16 {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 64 None 40 None",
        f"{DDP} --model vit-b-16 {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model vit-b-16 {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 64 None 40 None",
    ],
    "--model swin-t --rounds 2": [
        f"{DDP} --model swin-t {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model swin-t {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 64 None 40 None",
        f"{DDP} --model swin-t {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model swin-t {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 64 None 40 None",
    ],
    "--model convnext-tiny --rounds 2": [
        f"{DDP} --model convnext-tiny {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model convnext-tiny {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 64 None 40 None",
        f"{DDP} --model convnext-tiny {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model convnext-tiny {OPT} --per_gpu_train_batch_size 64 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 64 None 40 None",
    ],
    "--model clip-vit-b-32 --rounds 2 --batch 256 --steps 40": [
        f"{DDP} --model clip-vit-b-32 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model clip-vit-b-32 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 256 None 40 None",
        f"{DDP} --model clip-vit-b-32 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model clip-vit-b-32 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 256 None 40 None",
    ],
    "--model clip-vit-b-16": [
        f"{DDP} --model clip-vit-b-16 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model clip-vit-b-16 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 256 None 40 None",
        f"{DDP} --model clip-vit-b-16 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model clip-vit-b-16 {OPT} --per_gpu_train_batch_size 256 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 256 None 40 None",
    ],
    "--model bart-base": [
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 16 512 40 None",
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 16 512 40 None",
    ],
    "--model bart-large": [
        f"{DDP} --model bart-large {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model bart-large {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 16 512 40 None",
        f"{DDP} --model bart-large {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model bart-large {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 16 512 40 None",
    ],
    "--model t5-small": [
        f"{DDP} --model t5-small {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model t5-small {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 32 512 40 None",
        f"{DDP} --model t5-small {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model t5-small {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 32 512 40 None",
    ],
    "--model t5-base": [
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 32 512 40 None",
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --cuda_graph",
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED}",
        "baseline 32 512 40 None",
    ],
    "--model mamba-130m": [
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED}",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        "baseline 8 256 6 None",
    ],
    "--model mamba-370m": [
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED}",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss",
    ],
    "--model mamba2-130m": [
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED}",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss",
    ],
    "--model mamba2-370m": [
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED}",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba2-370m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 30 --logging_steps 15 {FIXED} --fused_lm_loss",
    ],
    "--model whisper-tiny": [
        f"{DDP} --model whisper-tiny {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model whisper-tiny {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 256 30 None",
        f"{DDP} --model whisper-tiny {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model whisper-tiny {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 256 30 None",
    ],
    "--model whisper-base": [
        f"{DDP} --model whisper-base {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model whisper-base {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 256 30 None",
        f"{DDP} --model whisper-base {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model whisper-base {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 256 30 None",
    ],
    "--model whisper-small": [
        f"{DDP} --model whisper-small {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model whisper-small {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 256 30 None",
        f"{DDP} --model whisper-small {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model whisper-small {OPT} --per_gpu_train_batch_size 16 --seq_len 256 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 256 30 None",
    ],
    "--model mamba-130m --steps 20": [
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED}",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 20 --logging_steps 10 {FIXED} --fused_lm_loss",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 256 --max_steps 20 --logging_steps 10 {FIXED} --cuda_graph",
        "baseline 8 256 6 None",
    ],
    "--model mamba2-130m,mamba-130m --steps 16": [
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED}",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba2-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --fused_lm_loss",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED}",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 16 --logging_steps 8 {FIXED} --fused_lm_loss",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 256 --max_steps 16 --logging_steps 8 {FIXED} --cuda_graph",
        "baseline 8 256 6 None",
    ],
    "--model bart-base --rounds 2 --steps 30": [
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 512 30 None",
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model bart-base {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 16 512 30 None",
    ],
    "--model t5-base --batch 32 --seq_len 512 --steps 30 --rounds 2": [
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 32 512 30 None",
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED} --cuda_graph",
        f"{DDP} --model t5-base {OPT} --per_gpu_train_batch_size 32 --seq_len 512 --max_steps 30 --logging_steps 15 {FIXED}",
        "baseline 32 512 30 None",
    ],
    "--model bart-large --min_seq_len 128 --rounds 1": [
        f"{DDP} --model bart-large {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --min_seq_len 128 --cuda_graph",
        f"{DDP} --model bart-large {OPT} --per_gpu_train_batch_size 16 --seq_len 512 --max_steps 40 --logging_steps 20 {FIXED} --min_seq_len 128",
        "baseline 16 512 40 128",
    ],
    "--model whisper-tiny --batch 4 --seq_len 128 --min_seq_len 32 --steps 10 --rounds 1": [
        f"{DDP} --model whisper-tiny {OPT} --per_gpu_train_batch_size 4 --seq_len 128 --max_steps 10 --logging_steps 5 {FIXED} --min_seq_len 32 --cuda_graph",
        f"{DDP} --model whisper-tiny {OPT} --per_gpu_train_batch_size 4 --seq_len 128 --max_steps 10 --logging_steps 5 {FIXED} --min_seq_len 32",
        "baseline 4 128 10 32",
    ],
    "--model mamba-130m --baseline_batch 4 --baseline_seq_len 128 --baseline_steps 4 --steps 12": [
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED}",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --min_seq_len 256 --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --min_seq_len 256",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --min_seq_len 256 --pack --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --min_seq_len 256 --pack",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --fused_lm_loss --cuda_graph",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 8 --seq_len 2048 --max_steps 12 --logging_steps 6 {FIXED} --fused_lm_loss",
        f"{DDP} --model mamba-130m {OPT} --per_gpu_train_batch_size 4 --seq_len 128 --max_steps 12 --logging_steps 6 {FIXED} --cuda_graph",
        "baseline 4 128 4 None",
    ],
}
SAME_PLAN = {
    "--model vit-b-16": "--model vit-b-16 --rounds 2",
    "--model convnext-tiny": "--model convnext-tiny --rounds 2",
    "--model swin-t": "--model swin-t --rounds 2",
    "--model clip-vit-b-32": "--model clip-vit-b-32 --rounds 2 --batch 256 --steps 40",
}


def _launches(command):
    args = ms.parse_args(shlex.split(command))
    out = []
    for model in args.model.split(","):
        for p in ms.plan(model, args, "{tmp}"):
            if p["argv"] == ms.BASELINE:
                out.append(f"baseline {p['batch']} {p['seq_len']} {p['steps']} {args.min_seq_len}")
            else:
                assert not any(" " in a for a in p["argv"][2:]), p["argv"]
                out.append(" ".join([p["argv"][0].replace(sys.executable, "{python}"),
                                     p["argv"][1].replace(ms.ROOT, "{root}"), *p["argv"][2:]]))
    return out


def test_the_table_holds_the_benchmarked_models():
    assert sorted(ms.MODELS) == sorted(MODELS)
    assert all(m in MODEL_REGISTRY for m in MODELS)


@pytest.mark.parametrize("command", sorted(PLANS))
def test_plan_launches_what_the_per_model_scripts_launched(command):
    assert _launches(command) == PLANS[command]


@pytest.mark.parametrize("command", sorted(SAME_PLAN))
def test_default_plan_matches_the_readme_command(command):
    assert _launches(command) == PLANS[SAME_PLAN[command]]


def test_every_model_has_a_recorded_default_plan():
    assert {f"--model {m}" for m in MODELS} <= set(PLANS) | set(SAME_PLAN)


def _finished_line(capsys, **values):
    log = get_logger_with_rank("b200ddp.engine.trainer", 0, -1)
    log.info("Finished training.", dict(global_step=40, average_loss=6.9123, seconds=12.5, **values))
    return capsys.readouterr().out.strip()


def test_parse_finished_reads_the_trainer_line(capsys):
    line = _finished_line(capsys, peak_mem_gb=13.704, ms_per_step=110.3125, samples_per_s=145.1)
    assert ms.parse_finished(line, "pairs_per_s", 16, 256) == {
        "ms_per_step": 110.3125, "pairs_per_s": 145.1, "peak_mem_gb": 13.704, "average_loss": 6.9123}
    assert ms.parse_finished(line, "tokens_per_s", 8, 2048) == {
        "ms_per_step": 110.3125, "tokens_per_s": 8 * 2048 / 110.3125 * 1e3, "peak_mem_gb": 13.704, "average_loss": 6.9123}
    # a CPU run logs no peak memory, and a run too short to time no throughput
    line = _finished_line(capsys)
    assert ms.parse_finished(line, "images_per_s", 64, None) == {
        "ms_per_step": None, "images_per_s": None, "peak_mem_gb": None, "average_loss": 6.9123}
    assert ms.parse_finished(line, "tokens_per_s", 8, 2048)["tokens_per_s"] is None


@pytest.mark.parametrize("name", sorted(m for m in MODELS if "baseline" in ms.MODELS[m]))
def test_baseline_builds_on_meta(name, monkeypatch):
    if ms.MODELS[name]["rate"] == "images_per_s":
        pytest.importorskip("torchvision", reason="the image baselines are torchvision's")
    else:
        transformers = pytest.importorskip("transformers", reason="the other baselines are transformers'")
        # the feature extractor's torch path needs a GPU; the features' shape is all the model sees here
        monkeypatch.setattr(transformers.WhisperFeatureExtractor, "_torch_extract_fbank_features",
                            lambda self, wave, device: np.zeros((len(wave), 80, 3000), np.float32))
    seq_len = None if ms.MODELS[name]["seq_len"] is None else 64
    model, step_loss = ms.MODELS[name]["baseline"](name, 2, seq_len, None, torch.device("meta"))
    assert all(p.is_meta for p in model.parameters())
    assert callable(step_loss)
