#!/usr/bin/env python
"""MMF's fp16 update with a learning-rate schedule, graphed, three ways over a capturable B200AdamW (the four
workloads of tools/bench_amp_step.py: autocast forward, scaled backward, clip at 1.0 times the loss scale,
scaler.step, scaler.update, then the scheduler's step):
  host        GraphedStep(..., scaler=) with a host LambdaLR (MMF's warmup_linear) stepped between replays, its lr
              staged to the device before every replay; GradScaler's own foreach non-finite check in the graph;
  device      the same with DeviceLRScheduler(opt, "warmup_linear") stepped inside the graph;
  fused       the device schedule and B200AdamW(..., fused_inf_check=True): the non-finite check in the clip launch
              (clip_grad_norm(1.0, scaler=)), no foreach pass over the gradients.

    python tools/bench_device_update.py [--models mmbt visual_bert lxmert m4c] [--steps 10] [--warmup 3]

The arms are alternated three times in one process; each time is the median of --steps updates timed one by one with
CUDA events; the median of the three is reported, with the spread.  One JSON line per model with the card's name,
power limit and SM clock read in the same run.  It fails without a GPU.
"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def sm_clock():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        cur, top = (int(x) for x in out.split(","))
        return cur, top
    except Exception:
        return None, None


def median_update_ms(fn, steps, warmup):
    """median over `steps` updates of the device time of one update (CUDA events around each call)"""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in ev)[steps // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["mmbt", "visual_bert", "lxmert", "m4c"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_update needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_graph_train_step import workloads
    from bench_lxmert import card
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW, DeviceLRScheduler
    name, limit = card()
    head = {"metric": "graphed fp16 update with warmup_linear: autocast fwd + scaled bwd + clip + scaler.step + "
                      "update + scheduler step", "unit": "ms/update", "gpu": name, "power_limit_w": limit,
            "steps": args.steps, "warmup": args.warmup, "dtype": "fp16 autocast", "data": "synthetic"}
    table = workloads(dev)
    sched_kw = dict(num_warmup_steps=1000, num_training_steps=100000)
    for key in args.models:
        torch.manual_seed(0)
        model, batch, loss_of, groups, hp, static, B = table[key]()
        arms = ("host", "device", "fused")
        models = {a: (model if a == "host" else copy.deepcopy(model)) for a in arms}
        opts = {a: B200AdamW(groups(m), capturable=True, fused_inf_check=(a == "fused"), **hp)
                for a, m in models.items()}
        scheds = {"host": torch.optim.lr_scheduler.LambdaLR(
            opts["host"], lambda s: s / 1000 if s < 1000 else max(0.0, (100000 - s) / 99000))}
        for a in ("device", "fused"):
            scheds[a] = DeviceLRScheduler(opts[a], "warmup_linear", **sched_kw)
        scalers = {a: torch.amp.GradScaler("cuda") for a in arms}
        steps = {}
        for a in arms:
            m = models[a]

            def graph_loss(b, m=m):
                with torch.autocast("cuda", dtype=torch.float16, cache_enabled=False):
                    return loss_of(m)(b)
            steps[a] = GraphedStep(m, graph_loss, batch, static_rows=static, optimizer=opts[a], max_grad_norm=1.0,
                                   scaler=scalers[a], lr_scheduler=None if a == "host" else scheds[a])

        def host():
            steps["host"](batch)
            scheds["host"].step()

        fns = {"host": host, "device": lambda: steps["device"](batch), "fused": lambda: steps["fused"](batch)}
        times = {a: [] for a in arms}
        for _ in range(3):
            for a in arms:
                times[a].append(median_update_ms(fns[a], args.steps, args.warmup))
        med = {a: sorted(v)[1] for a, v in times.items()}
        spread = {a: max(v) - min(v) for a, v in times.items()}
        cur, top = sm_clock()
        print(json.dumps(dict(head, model=key, batch=B, ms_per_update=times, median_ms=med, spread_ms=spread,
                              sm_clock_mhz=cur, max_sm_clock_mhz=top,
                              device_vs_host=med["host"] / med["device"], fused_vs_host=med["host"] / med["fused"],
                              last_lr={"host": scheds["host"].get_last_lr()[0],
                                       "device": scheds["device"].get_last_lr()[0]},
                              final_scale={a: s.get_scale() for a, s in scalers.items()})), flush=True)
        del steps, models, opts, scalers, scheds, model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
