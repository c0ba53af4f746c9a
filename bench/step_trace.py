#!/usr/bin/env python
"""Per-kernel totals of one training step from a chrome trace written by ``bench.py --trace_dir DIR``.

  python bench/step_trace.py DIR/rank0.json [--steps 4] [--top 25]

``bench.py`` traces 4 replayed steps; every device kernel's duration is summed by kernel name and divided by the number of
steps.  The BatchNorm kernels of ``csrc/batchnorm.cu`` are also reported as one group, as a share of the summed kernel time
and of the device span of the traced steps (first kernel start to last kernel end, over the steps)."""
import argparse
import collections
import json
import re

BN_KERNELS = ("bn_stats_kernel", "bn_apply_kernel", "bn_apply_pdl_kernel", "bn_bwd_reduce_kernel", "bn_bwd_apply_kernel",
              "bn_bwd_apply_pdl_kernel", "bn_apply_partials_kernel", "bn_bwd_apply_partials_kernel", "bn_resident_fwd_kernel",
              "bn_resident_bwd_kernel")


def short_name(name: str) -> str:
    """Kernel name without namespaces, template arguments or the parameter list."""
    base = name.replace("(anonymous namespace)::", "")
    base = re.sub(r"^void\s+", "", base).split("(")[0]
    base = re.sub(r"<.*>", "", base)
    return base.split("::")[-1].strip() or name[:60]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trace")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--top", type=int, default=25)
    args = ap.parse_args()
    events = json.load(open(args.trace))
    events = events["traceEvents"] if isinstance(events, dict) else events
    kernels = [e for e in events if e.get("ph") == "X" and e.get("cat") == "kernel"]
    if not kernels:
        raise SystemExit("no device kernels in the trace")
    total = collections.Counter()
    count = collections.Counter()
    for e in kernels:
        n = short_name(e["name"])
        total[n] += float(e["dur"])
        count[n] += 1
    summed = sum(total.values()) / args.steps
    span = (max(e["ts"] + e["dur"] for e in kernels) - min(e["ts"] for e in kernels)) / args.steps
    print(f"kernels per step {len(kernels) / args.steps:.0f}, summed kernel time {summed / 1e3:.3f} ms/step, "
          f"device span {span / 1e3:.3f} ms/step")
    print(f"{'kernel':44s} {'us/step':>10s} {'launches':>9s} {'share':>7s}")
    for n, us in total.most_common(args.top):
        print(f"{n[:44]:44s} {us / args.steps:10.1f} {count[n] / args.steps:9.0f} {100 * us / args.steps / summed:6.1f}%")
    bn_us = sum(us for n, us in total.items() if n in BN_KERNELS) / args.steps
    bn_n = sum(c for n, c in count.items() if n in BN_KERNELS) / args.steps
    print(f"BatchNorm kernels: {bn_us / 1e3:.3f} ms/step in {bn_n:.0f} launches = {100 * bn_us / summed:.1f}% of summed kernel time, "
          f"{100 * bn_us / span:.1f}% of the device span")
    print(json.dumps({"summed_kernel_ms": summed / 1e3, "span_ms": span / 1e3, "bn_ms": bn_us / 1e3, "bn_launches": bn_n,
                      "bn_share_of_kernel_time": bn_us / summed,
                      "bn_by_kernel_us": {n: total[n] / args.steps for n in BN_KERNELS if n in total}}))


if __name__ == "__main__":
    main()
