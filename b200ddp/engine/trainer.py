"""Training runtime: the reference's ``train(args, model)`` (``ddp.py:126-288``) rebuilt around
``TrainStep`` / ``BatchLoader`` / ``DevicePrefetcher`` / the native DDP wrapper.

Kept from the reference: flag names/defaults, sampler choice and ``set_epoch``, total-step
arithmetic (``ddp.py:155-161``), ``global_step`` starting at 1 and exiting when it exceeds ``max_steps``
(``ddp.py:206,280``), TensorBoard scalars ``lr`` / ``loss`` on the main process, checkpoint layout, tqdm only
on local rank -1/0, banner log lines.
Deliberately fixed (documented in README): logging/saving only at optimizer-step boundaries (Q4), no
allreduce on non-boundary accumulation micro-steps (Q5), no per-step ``loss.item()`` syncs and
non-blocking H2D (Q9), a working ``--fp16`` (bf16 weights + fp32 master, Q1), resume (Q2), an ``evaluate``
that evaluates (Q3), CPU/gloo distributed mode (Q6).
"""
from __future__ import annotations

import math
import os
import time
from typing import Callable, Optional

import torch
import torch.distributed as dist
from tqdm import tqdm
from tqdm.auto import trange

from ..data import BatchLoader, DevicePrefetcher, FooDataset, SyntheticImageNet, SyntheticTokens
from ..ops import CrossEntropyLoss, MSELoss
from ..optim import FusedSGD, get_linear_schedule_with_warmup
from ..parallel import DataParallel, DistributedDataParallel, ShardedSampler
from ..utils import StepTimer, is_main_process, nvtx_range, rng_state, restore_rng_state, to_mixed_bf16
from ..utils.checkpoint import latest_checkpoint, load_checkpoint, save_checkpoint
from .step import TrainStep


def _summary_writer():
    try:
        from torch.utils.tensorboard import SummaryWriter
    except Exception:
        try:
            from tensorboardX import SummaryWriter
        except Exception:
            return None
    return SummaryWriter


def build_dataset(args):
    # (loss_kind is defined below; resolved at call time)
    name = getattr(args, "model", "foo")
    n = int(getattr(args, "dataset_size", 100000))
    if name == "foo":
        return FooDataset(n)
    if name.startswith("resnet"):
        dense = loss_kind(args) == "mse"
        return SyntheticImageNet(samples=min(n, int(getattr(args, "image_samples", 1024))), dense_target=dense)
    if name.startswith("bert"):
        return SyntheticTokens(samples=min(n, 512), seq_len=int(getattr(args, "seq_len", 512)))
    raise ValueError(f"no default dataset for model {name!r}")


def loss_kind(args) -> str:
    """``--loss`` or the model's default: MSE for the reference's FooModel (``ddp.py:164``), cross-entropy otherwise."""
    return getattr(args, "loss", None) or ("mse" if getattr(args, "model", "foo") == "foo" else "ce")


def build_criterion(args):
    return CrossEntropyLoss() if loss_kind(args) == "ce" else MSELoss()


class Trainer:
    def __init__(self, args, model: torch.nn.Module, log, dataset=None, criterion=None,
                 input_transform: Optional[Callable] = None):
        self.args = args
        self.log = log
        self.device = args.device
        self.distributed = args.local_rank != -1
        self.is_main = is_main_process()
        self.show_bars = args.local_rank in (-1, 0)
        self.tb_writer = None
        if self.is_main and not getattr(args, "no_tensorboard", False):
            SW = _summary_writer()
            if SW is not None:
                self.tb_writer = SW(log_dir=getattr(args, "tb_dir", None))

        # ---- model placement / precision --------------------------------------------------------
        self.compute_dtype = torch.float32
        if getattr(args, "fp16", False) and self.device.type == "cuda":
            # the reference's --fp16 asks apex for O2 (half model + fp32 master weights + dynamic loss
            # scaling, ddp.py:174-180); here that is bf16 weights + fp32 masters, no loss scaling needed
            self.compute_dtype = torch.bfloat16
        model = model.to(self.device)
        if self.compute_dtype != torch.float32:
            model = to_mixed_bf16(model)
        if getattr(args, "channels_last", False):
            model = model.to(memory_format=torch.channels_last)

        # ---- optional resume: rank 0's weights reach everyone through the wrap-time broadcast -----
        self.resume_dir = getattr(args, "resume_from", None)
        if self.resume_dir == "latest":
            self.resume_dir = latest_checkpoint(args.output_dir)
        self._resume_state = {}

        # ---- data ---------------------------------------------------------------------------------
        self.dataset = dataset if dataset is not None else build_dataset(args)
        # one seedable, skippable sampler in every mode (single process = 1 replica), so mid-epoch resume replays nothing
        if self.distributed:
            self.sampler = ShardedSampler(self.dataset, seed=getattr(args, "sampler_seed", 0))
        else:
            self.sampler = ShardedSampler(self.dataset, num_replicas=1, rank=0, seed=getattr(args, "sampler_seed", 0))
        self.loader = BatchLoader(self.dataset, batch_size=args.train_batch_size, sampler=self.sampler,
                                  pin_memory=self.device.type == "cuda")
        steps_per_epoch = len(self.loader) // args.gradient_accumulation_steps
        if args.max_steps > 0:
            self.t_total = args.max_steps
            args.num_train_epochs = args.max_steps // max(1, steps_per_epoch) + 1
        else:
            self.t_total = steps_per_epoch * args.num_train_epochs

        # ---- resume (weights first: rank 0's reach every rank through the wrap-time broadcast) -----
        self.criterion = criterion if criterion is not None else build_criterion(args)
        if self.resume_dir:
            load_checkpoint(self.resume_dir, model)

        # ---- parallel wrapper ---------------------------------------------------------------------
        inner = model
        if args.n_gpu > 1:
            model = DataParallel(model)
        elif self.distributed:
            model = DistributedDataParallel(
                model, device_ids=[args.local_rank] if self.device.type == "cuda" else None,
                output_device=args.local_rank if self.device.type == "cuda" else None,
                find_unused_parameters=getattr(args, "find_unused_parameters", True),
                gradient_as_bucket_view=getattr(args, "gradient_as_bucket_view", False),
                bucket_cap_mb=getattr(args, "bucket_cap_mb", None), backend=getattr(args, "backend", "auto"),
                wire_dtype=getattr(args, "wire_dtype", None), broadcast_buffers=getattr(args, "broadcast_buffers", True))

        # ---- optimizer / schedule: built AFTER the broadcast so fp32 master weights start identical --
        self.optimizer = FusedSGD(inner.parameters(), lr=getattr(args, "lr", 1e-3), momentum=getattr(args, "momentum", 0.0),
                                  weight_decay=getattr(args, "weight_decay", 0.0), max_grad_norm=args.max_grad_norm)
        self.scheduler = get_linear_schedule_with_warmup(self.optimizer, num_warmup_steps=args.warmup_steps,
                                                         num_training_steps=self.t_total)
        if self.resume_dir:
            self._resume_state = load_checkpoint(self.resume_dir, None, self.optimizer, self.scheduler)
            log.info("Resumed from checkpoint.", dict(path=self.resume_dir, global_step=self._resume_state.get("global_step")))
        self.model = model
        if input_transform is None and self.device.type == "cuda" and getattr(args, "model", "foo").startswith("resnet"):
            input_transform = self._make_image_transform()
        self.step_fn = TrainStep(model, self.criterion, self.optimizer, self.device,
                                 accumulation=args.gradient_accumulation_steps, use_graph=getattr(args, "cuda_graph", False),
                                 input_transform=input_transform,
                                 loss_scale=float(getattr(args, "loss_scale", 0) or 0) if getattr(args, "fp16", False) else 1.0)
        self.global_step = 1
        self.tr_loss_host = 0.0
        self.timer = StepTimer(self.device, samples_per_step=args.train_batch_size * args.gradient_accumulation_steps * self._world())
        self.last_throughput = None

    # ------------------------------------------------------------------------------------------
    def _make_image_transform(self):
        """Raw NCHW batch (fp32 or uint8) -> compute dtype, channels_last when the model is, in ONE kernel
        (``csrc/input.cu``); writes into the CUDA graph's static input once that exists."""
        from .. import _ext
        C = _ext.get()
        mean = torch.zeros(3, device=self.device)
        inv_std = torch.ones(3, device=self.device)
        scratch = {}
        cl = bool(getattr(self.args, "channels_last", False))

        def transform(x):
            if x.dim() != 4 or x.dtype not in (torch.float32, torch.uint8) or not x.is_contiguous():
                return x
            shape = tuple(x.shape)
            dst = self.step_fn.static_inputs()[0]
            if dst is None or tuple(dst.shape) != shape or dst.dtype != self.compute_dtype:
                dst = scratch.get(shape)
                if dst is None:
                    dst = torch.empty(shape, dtype=self.compute_dtype, device=self.device)
                    dst = dst.contiguous(memory_format=torch.channels_last) if cl else dst
                    scratch[shape] = dst
            if not dst.is_contiguous(memory_format=torch.channels_last):
                return x.to(self.compute_dtype)
            C.normalize_to_channels_last(x, dst, mean, inv_std, 1.0 / 255.0 if x.dtype == torch.uint8 else 1.0)
            return dst
        return transform

    def _world(self) -> int:
        return dist.get_world_size() if self.distributed else 1

    def _to_compute(self, x: torch.Tensor) -> torch.Tensor:
        if x.dim() == 4 and self.step_fn.input_transform is not None:
            return x                       # the fused input kernel casts
        if x.is_floating_point() and x.dtype != self.compute_dtype:
            x = x.to(self.compute_dtype)
        return x

    def train(self):
        args, log = self.args, self.log
        log.info("Finish setting up args.", dict(args={k: v for k, v in vars(args).items()}))
        log.info("Begin training.", dict(num_examples=len(self.dataset),
                                         total_batch_size=args.train_batch_size * args.gradient_accumulation_steps * self._world(),
                                         total_optimization_steps=self.t_total,
                                         gradient_accumulation_steps=args.gradient_accumulation_steps))
        accum = args.gradient_accumulation_steps
        logging_loss = 0.0
        start_epoch, skip_batches = 0, 0
        if self._resume_state:
            self.global_step = int(self._resume_state.get("global_step", 1))
            start_epoch = int(self._resume_state.get("epoch", 0))
            skip_batches = int(self._resume_state.get("batches_in_epoch", 0))
            self.tr_loss_host = float(self._resume_state.get("tr_loss", 0.0))
            logging_loss = self.tr_loss_host
            if "rng" in self._resume_state:
                restore_rng_state(self._resume_state["rng"])
        self.optimizer.zero_grad(set_to_none=True)
        t_start = time.time()
        done = False
        tracer = self._make_tracer()
        if self.device.type == "cuda":
            torch.cuda.reset_peak_memory_stats(self.device)
        for epoch in trange(start_epoch, int(args.num_train_epochs), desc="Epoch", disable=not self.show_bars, leave=False):
            self.sampler.set_epoch(epoch)
            if skip_batches:
                self.sampler.set_start_index(skip_batches * args.train_batch_size)
            feed = DevicePrefetcher(self.loader, self.device)
            with tqdm(feed, desc=f"Epoch {epoch}", disable=not self.show_bars, leave=False,
                      total=len(self.loader) - skip_batches) as bar:
                for step, (x, y) in enumerate(bar):
                    self.model.train()
                    if x.device != self.device:
                        x, y = x.to(self.device, non_blocking=True), y.to(self.device, non_blocking=True)
                    x, y = self._to_compute(x), self._to_compute(y)
                    boundary = (step + 1) % accum == 0
                    with nvtx_range("train_step"):
                        self.step_fn(x, y, boundary=boundary)
                    if not boundary:
                        continue
                    self.scheduler.step()
                    self.global_step += 1
                    self.timer.tick()
                    if tracer is not None:
                        tracer.step()

                    if args.logging_steps > 0 and self.global_step % args.logging_steps == 0:
                        total = self.step_fn.read_loss_sum() + self.tr_loss_host   # the only host sync, every logging_steps
                        window = (total - logging_loss) / args.logging_steps
                        logging_loss = total
                        if self.show_bars:
                            bar.set_postfix(loss=window)
                        perf = self.timer.summary()
                        if perf is not None:
                            self.last_throughput = perf
                        if self.tb_writer is not None:
                            self.tb_writer.add_scalar("lr", self.scheduler.get_last_lr()[0], self.global_step)
                            self.tb_writer.add_scalar("loss", window, self.global_step)
                            if perf is not None and "samples_per_s" in perf:
                                self.tb_writer.add_scalar("samples_per_s", perf["samples_per_s"], self.global_step)

                    if args.save_steps > 0 and self.global_step % args.save_steps == 0:
                        self.save(epoch, step + 1 + skip_batches)

                    if args.max_steps > 0 and self.global_step > args.max_steps:
                        done = True
                        break
            skip_batches = 0
            if done:
                break
        total_loss = self.step_fn.read_loss_sum() + self.tr_loss_host
        elapsed = time.time() - t_start
        if tracer is not None:
            tracer.stop()
        extra = {}
        if self.device.type == "cuda":
            extra["peak_mem_gb"] = round(torch.cuda.max_memory_allocated(self.device) / 2 ** 30, 3)
        if self.last_throughput:
            extra.update({"ms_per_step": round(self.last_throughput["ms_per_step"], 4),
                          "samples_per_s": round(self.last_throughput.get("samples_per_s", 0.0), 1)})
        if hasattr(self.model, "ddp_stats"):
            extra["ddp"] = self.model.ddp_stats()
        log.info("Finished training.", dict(global_step=self.global_step, average_loss=total_loss / self.global_step,
                                            seconds=round(elapsed, 3), **extra))
        if self.tb_writer is not None:
            self.tb_writer.flush()
            self.tb_writer.close()
        return self.global_step, total_loss / self.global_step

    # ------------------------------------------------------------------------------------------
    def _make_tracer(self):
        """``--trace_dir``: torch.profiler timeline (CPU ops, CUDA kernels, the NVTX-style ranges of ``nvtx_range``) of a
        few optimizer steps per rank.  The reference has no tracing at all; numbers are never taken from a
        traced run (``StepTimer`` reports the untraced steps)."""
        trace_dir = getattr(self.args, "trace_dir", None)
        steps = int(getattr(self.args, "trace_steps", 0) or 0)
        if not trace_dir or steps <= 0:
            return None
        from torch.profiler import ProfilerActivity, profile, schedule
        os.makedirs(trace_dir, exist_ok=True)
        rank = dist.get_rank() if self.distributed else 0
        path = os.path.join(trace_dir, f"trace_rank{rank}.json")
        acts = [ProfilerActivity.CPU] + ([ProfilerActivity.CUDA] if self.device.type == "cuda" else [])

        def on_ready(prof):
            prof.export_chrome_trace(path)
            self.log.info("Wrote profiler trace.", dict(path=path, steps=steps))

        prof = profile(activities=acts, schedule=schedule(wait=int(getattr(self.args, "trace_skip", 10)), warmup=1, active=steps, repeat=1),
                       on_trace_ready=on_ready)
        prof.start()
        return prof

    # ------------------------------------------------------------------------------------------
    def save(self, epoch: int, batches_in_epoch: int) -> Optional[str]:
        """Main process writes; a barrier keeps other ranks from racing ahead into a half-written dir
        (the reference has no barrier)."""
        path = None
        if self.is_main:
            state = {"global_step": self.global_step, "epoch": epoch, "batches_in_epoch": batches_in_epoch,
                     "tr_loss": self.step_fn.read_loss_sum() + self.tr_loss_host, "rng": rng_state(),
                     "world_size": self._world()}
            path = save_checkpoint(self.args.output_dir, self.global_step, self.model, self.optimizer, self.scheduler,
                                   self.args, state, self.log)
        if self.distributed and getattr(self.args, "save_barrier", True):
            dist.barrier()
        return path

    @torch.no_grad()
    def evaluate(self, dataset=None, max_batches: Optional[int] = None) -> dict:
        """Mean loss over a dataset shard, all-reduced across ranks (the reference's ``evaluate`` is an empty
        stub that is never called, ``ddp.py:123-124``)."""
        ds = dataset if dataset is not None else self.dataset
        sampler = ShardedSampler(ds, shuffle=False) if self.distributed else torch.utils.data.SequentialSampler(ds)
        loader = BatchLoader(ds, batch_size=self.args.train_batch_size, sampler=sampler, pin_memory=self.device.type == "cuda")
        was_training = self.model.training
        self.model.eval()
        total = torch.zeros(2, dtype=torch.float64, device=self.device)
        inner = self.model.module if hasattr(self.model, "module") else self.model
        for i, (x, y) in enumerate(DevicePrefetcher(loader, self.device)):
            if max_batches is not None and i >= max_batches:
                break
            if x.device != self.device:
                x, y = x.to(self.device), y.to(self.device)
            x, y = self._to_compute(x), self._to_compute(y)
            if self.step_fn.input_transform is not None:
                x = self.step_fn.input_transform(x)
            loss = self.criterion(inner(x), y)
            total[0] += loss.double() * x.shape[0]
            total[1] += x.shape[0]
        if self.distributed:
            dist.all_reduce(total)
        self.model.train(was_training)
        n = max(1.0, float(total[1]))
        return {"eval_loss": float(total[0]) / n, "eval_samples": int(total[1])}
