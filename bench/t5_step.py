#!/usr/bin/env python
"""t5-base training step: this package against transformers' T5ForConditionalGeneration, alternated in one call.

  python bench/t5_step.py [--model t5-base] [--batch 32] [--seq_len 512] [--min_seq_len N] [--steps 40] [--rounds 2]
                          [--out t5_step.json]

Per round, three runs in fresh processes, in this order:
  native graph   python ddp.py --model t5-base --fp16 --cuda_graph --optimizer adamw --per_gpu_train_batch_size B
                 --seq_len S [--min_seq_len N] --max_steps T --logging_steps T/2   (bf16 weights, fp32 masters, the native
                 kernels, one CUDA graph per step)
  native eager   the same without --cuda_graph
  transformers   transformers.T5ForConditionalGeneration (the same preset, dropout 0) under bf16 autocast,
                 torch.optim.AdamW(fused=True), on the same span-corruption pairs with attention_mask and labels
ms/step is the mean over the second half of the steps, from CUDA events (the trainer's own timer for ddp.py).  ddp.py
feeds its synthetic pairs from pinned host memory; the transformers run trains on one device-resident batch, so it pays
no host-to-device copy.  Sources are --seq_len tokens (or uniform in [--min_seq_len, --seq_len]); targets, about a
fifth of that, are right-padded to a multiple of 128, so the target side always holds padding.  Peak memory is torch's max_memory_allocated.  The losses are not
comparable: ddp.py reports the average over its steps on the synthetic set, the transformers run its last loss on its
one batch.  The card's name and power limit are read in the same call.  Writes only under a temporary directory (and
--out)."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "unknown"


def transformers_run(model_name, batch, seq_len, min_len, steps):
    import torch
    import transformers
    sys.path.insert(0, ROOT)
    from b200ddp.data import SyntheticSpanCorruption
    from b200ddp.models.t5 import T5_BASE, T5_SMALL
    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    c = {"t5-small": T5_SMALL, "t5-base": T5_BASE}[model_name]
    cfg = transformers.T5Config(vocab_size=c.vocab_size, d_model=c.d_model, d_kv=c.d_kv, d_ff=c.d_ff, num_layers=c.num_layers,
                                num_decoder_layers=c.num_decoder_layers, num_heads=c.num_heads, feed_forward_proj="relu",
                                dropout_rate=0.0, pad_token_id=0, decoder_start_token_id=0, eos_token_id=1)
    model = transformers.T5ForConditionalGeneration(cfg).to(dev)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    pairs = SyntheticSpanCorruption(samples=batch, seq_len=seq_len, min_len=min_len)
    x, y = pairs.X.to(dev), pairs.Y.to(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    events = []
    for _ in range(steps):
        with torch.autocast("cuda", torch.bfloat16):
            loss = model(input_ids=x, attention_mask=(x != 0).long(), labels=y).loss
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)
    torch.cuda.synchronize()
    half = steps // 2
    ms = events[half - 1].elapsed_time(events[-1]) / (steps - half)
    return {"ms_per_step": ms, "pairs_per_s": batch / ms * 1e3,
            "peak_mem_gb": torch.cuda.max_memory_allocated(dev) / 2 ** 30, "last_loss": float(loss)}


def native_run(model_name, batch, seq_len, min_len, steps, graph, tmp):
    argv = [sys.executable, os.path.join(ROOT, "ddp.py"), "--model", model_name, "--fp16", "--optimizer", "adamw",
            "--per_gpu_train_batch_size", str(batch), "--seq_len", str(seq_len), "--max_steps", str(steps), "--logging_steps",
            str(steps // 2), "--save_steps", "0", "--no_tensorboard", "--output_dir", os.path.join(tmp, "out"), "--lr", "1e-4"]
    if min_len is not None:
        argv += ["--min_seq_len", str(min_len)]
    if graph:
        argv.append("--cuda_graph")
    proc = subprocess.run(argv, capture_output=True, text=True, cwd=tmp)
    text = proc.stdout + proc.stderr
    line = next((ln for ln in text.splitlines() if "Finished training." in ln), None)
    if proc.returncode != 0 or line is None:
        raise RuntimeError(f"ddp.py failed ({proc.returncode}):\n{text[-4000:]}")

    def num(key):
        m = re.search(rf"{key}=([-\d.e]+)", line)
        return float(m.group(1)) if m else None
    return {"ms_per_step": num("ms_per_step"), "pairs_per_s": num("samples_per_s"), "peak_mem_gb": num("peak_mem_gb"),
            "average_loss": num("average_loss")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", type=str, default="t5-base", choices=["t5-small", "t5-base"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq_len", type=int, default=512)
    ap.add_argument("--min_seq_len", type=int, default=None)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    ap.add_argument("--transformers_only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.transformers_only:
        print(json.dumps(transformers_run(args.model, args.batch, args.seq_len, args.min_seq_len, args.steps)), flush=True)
        return
    gpu = card()
    print(f"{args.model} batch {args.batch}, seq_len {args.seq_len}, min_seq_len {args.min_seq_len}, {args.steps} steps, on {gpu}",
          flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for name in ("native graph", "native eager", "transformers"):
                if name == "transformers":
                    extra = [] if args.min_seq_len is None else ["--min_seq_len", str(args.min_seq_len)]
                    proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--transformers_only", "--model", args.model,
                                           "--batch", str(args.batch), "--seq_len", str(args.seq_len), "--steps", str(args.steps),
                                           *extra], capture_output=True, text=True, cwd=tmp)
                    if proc.returncode != 0:
                        raise RuntimeError(f"transformers run failed:\n{proc.stdout[-2000:]}{proc.stderr[-4000:]}")
                    res = json.loads(proc.stdout.strip().splitlines()[-1])
                else:
                    res = native_run(args.model, args.batch, args.seq_len, args.min_seq_len, args.steps, name == "native graph", tmp)
                res.update(run=name, round=r, model=args.model, batch=args.batch, seq_len=args.seq_len, min_seq_len=args.min_seq_len,
                           card=gpu)
                rows.append(res)
                print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
