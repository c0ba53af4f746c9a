"""Checkpoint save / load.

Save layout is the reference's (``ddp.py:64-77,255-277``): ``<output_dir>/checkpoint-<global_step>/`` with
``model.bin`` (state_dict of the *unwrapped* module - no ``module.`` prefix), ``training_args.bin`` (pickled
Namespace), ``optimizer.pt``, ``scheduler.pt``; written by the main process only.  The reference has no
load path (``--global-step`` is parsed and ignored); ``load_checkpoint`` + ``trainer_state.pt``
(global step, epoch, batches consumed in the epoch, RNG state, running loss) add resume.
"""
from __future__ import annotations

import os
import re
from typing import Optional

import torch

MODEL_FILE = "model.bin"
ARGS_FILE = "training_args.bin"
OPTIMIZER_FILE = "optimizer.pt"
SCHEDULER_FILE = "scheduler.pt"
STATE_FILE = "trainer_state.pt"


def unwrap(model):
    return model.module if hasattr(model, "module") else model


def save_model(model, save_directory: str, log=None) -> Optional[str]:
    if os.path.isfile(save_directory):
        if log is not None:
            log.error("Provided path should be a directory, not a file", dict(save_directory=save_directory))
        return None
    os.makedirs(save_directory, exist_ok=True)
    path = os.path.join(save_directory, MODEL_FILE)
    state = {k: v.detach().cpu() for k, v in unwrap(model).state_dict().items()}
    torch.save(state, path)
    if log is not None:
        log.info("Saved model weights.", dict(path=path))
    return path


def save_checkpoint(output_dir: str, global_step: int, model, optimizer, scheduler, args, trainer_state: dict, log=None) -> str:
    ckpt_dir = os.path.join(output_dir, f"checkpoint-{global_step}")
    save_model(model, ckpt_dir, log)
    plain = _picklable_args(args)
    torch.save(plain, os.path.join(ckpt_dir, ARGS_FILE))
    if log is not None:
        log.info("Saved training args.", dict(path=os.path.join(ckpt_dir, ARGS_FILE)))
    torch.save(optimizer.state_dict(), os.path.join(ckpt_dir, OPTIMIZER_FILE))
    if log is not None:
        log.info("Saved optimizer states.", dict(path=os.path.join(ckpt_dir, OPTIMIZER_FILE)))
    torch.save(scheduler.state_dict(), os.path.join(ckpt_dir, SCHEDULER_FILE))
    if log is not None:
        log.info("Saved scheduler states.", dict(path=os.path.join(ckpt_dir, SCHEDULER_FILE)))
    torch.save(trainer_state, os.path.join(ckpt_dir, STATE_FILE))
    return ckpt_dir


def _picklable_args(args):
    import argparse
    import copy
    ns = argparse.Namespace()
    for k, v in vars(args).items():
        try:
            setattr(ns, k, copy.deepcopy(v))
        except Exception:
            setattr(ns, k, repr(v))
    return ns


def latest_checkpoint(output_dir: str) -> Optional[str]:
    if not os.path.isdir(output_dir):
        return None
    best, best_step = None, -1
    for name in os.listdir(output_dir):
        m = re.fullmatch(r"checkpoint-(\d+)", name)
        if m and os.path.isfile(os.path.join(output_dir, name, MODEL_FILE)) and int(m.group(1)) > best_step:
            best, best_step = os.path.join(output_dir, name), int(m.group(1))
    return best


def load_checkpoint(ckpt_dir: str, model, optimizer=None, scheduler=None, map_location="cpu") -> dict:
    """Restore what exists in ``ckpt_dir``; returns the trainer state dict ({} for reference-made
    checkpoints, which carry none)."""
    if model is not None:
        state = torch.load(os.path.join(ckpt_dir, MODEL_FILE), map_location=map_location, weights_only=True)
        unwrap(model).load_state_dict(state)
    opt_path = os.path.join(ckpt_dir, OPTIMIZER_FILE)
    if optimizer is not None and os.path.isfile(opt_path):
        optimizer.load_state_dict(torch.load(opt_path, map_location=map_location, weights_only=False))
    sch_path = os.path.join(ckpt_dir, SCHEDULER_FILE)
    if scheduler is not None and os.path.isfile(sch_path):
        sd = torch.load(sch_path, map_location=map_location, weights_only=False)
        if "last_step" in sd:
            scheduler.load_state_dict(sd)
        elif "last_epoch" in sd:      # a torch LambdaLR state written by the reference
            scheduler.load_state_dict({"last_step": int(sd["last_epoch"])})
    st_path = os.path.join(ckpt_dir, STATE_FILE)
    if os.path.isfile(st_path):
        return torch.load(st_path, map_location="cpu", weights_only=False)
    m = re.search(r"checkpoint-(\d+)$", ckpt_dir.rstrip("/"))
    return {"global_step": int(m.group(1))} if m else {}
