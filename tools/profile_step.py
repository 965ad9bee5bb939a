#!/usr/bin/env python
"""Where a training step's GPU time goes: runs a few eager steps of bench.py (--profile --no-graph) under torch.profiler
with CUDA activities and prints the device time per kernel name and per kernel family, per step and as a share.

    python tools/profile_step.py [--workload visual_bert] [--steps 4] [--json out.json]

Tracing slows the host, so the per-step wall time of this run is not a benchmark result; the kernel durations are the
device's own.  The card's name and power limit are printed with the table, since they are part of every number in it.
"""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WARMUP = 3      # bench.py runs at least three untimed steps; they are profiled too and counted as steps

# kernel-name substring -> family, first match wins
FAMILIES = (
    ("attn_fwd_kernel", "attention fwd"),
    ("attn_bwd_dq_kernel", "attention bwd dq"),
    ("attn_bwd_dkv_kernel", "attention bwd dk/dv"),
    ("attn_delta_kernel", "attention delta"),
    ("dropout_bits", "dropout bits (attention + hidden)"),
    ("gemm", "gemm"),
    ("mmfb", "row / element-wise kernels"),
)


def family(name):
    for key, fam in FAMILIES:
        if key in name:
            return fam
    return "other (framework)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="visual_bert")
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("profile_step: no CUDA device; kernel times can only be measured on the GPU")
    from torch.profiler import ProfilerActivity, profile
    import bench
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          stdout=subprocess.PIPE, text=True).stdout.strip()
    sys.argv = ["bench.py", "--gpus", "1", "--workload", args.workload, "--steps", str(args.steps), "--warmup", str(WARMUP),
                "--profile", "--no-graph", "--no-cpu-baseline"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bench.main()
        torch.cuda.synchronize()
    steps = WARMUP + args.steps
    per_kernel = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = per_kernel[ev.name]
            k[0] += 1
            k[1] += ev.device_time
    total = sum(v[1] for v in per_kernel.values())
    fams = collections.defaultdict(float)
    for name, (_, us) in per_kernel.items():
        fams[family(name)] += us
    print("card: %s   workload: %s   profiled steps: %d (eager, traced)" % (card, args.workload, steps))
    print("%-40s %12s %7s" % ("family", "us / step", "share"))
    for fam, us in sorted(fams.items(), key=lambda kv: -kv[1]):
        print("%-40s %12.1f %6.1f%%" % (fam, us / steps, 100.0 * us / total))
    print("%-40s %12.1f" % ("all kernels", total / steps))
    print()
    print("%-100s %8s %12s %7s" % ("kernel", "launches", "us / step", "share"))
    for name, (n, us) in sorted(per_kernel.items(), key=lambda kv: -kv[1][1])[:40]:
        print("%-100s %8.1f %12.1f %6.1f%%" % (name[:100], n / steps, us / steps, 100.0 * us / total))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": card, "workload": args.workload, "steps": steps,
                       "families_us_per_step": {f: us / steps for f, us in fams.items()},
                       "kernels": {n: {"launches_per_step": c / steps, "us_per_step": us / steps}
                                   for n, (c, us) in per_kernel.items()}}, fh, indent=1)


if __name__ == "__main__":
    main()
