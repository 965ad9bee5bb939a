#!/usr/bin/env python
"""Skip-padding captured in a CUDA graph, on the VisualBERT trunk of BASELINE.json configs[1]: 12 L / 768 / 12 h / 3072,
128 text tokens + 100 regions x 2048, bf16 compute, dropout 0.1, forward + backward.  Three arms, alternated `--rounds`
times in one process, median reported:

  dense_graphed   - GraphedStep over the dense path (every padded row computed);
  packed_eager    - today's skip-padding: packing planned on the host, eager launches;
  packed_graphed  - GraphedStep(..., static_rows=True): packing planned on the device at capacity B*S, every layer kernel
                    bounded by the device token count.

    python tools/bench_graph_skip_padding.py [--batches 32,166] [--steps 10] [--warmup 3] [--rounds 3]

The length distributions are those of tools/bench_varlen.py: bench.py's own (text U{64..128}, regions U{50..100}) and a
short-text one (text U{8..24}, regions U{10..100}).  The loss ignores padded positions, (sequence_output * aux *
valid).sum().  Before timing, the arms are checked to agree with dropout off, as bench_varlen.py checks them: the loss
within 1e-2 of sum |terms|, every parameter gradient within 2e-2 relative L2 of the dense path's.  Prints one JSON line per
(batch, distribution) with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_varlen import DISTS, batch, config, rel  # noqa: E402


def card():
    import torch
    name, limit, clock = torch.cuda.get_device_name(0), None, None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        f = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        limit, clock = float(f[0]), float(f[1])
    except Exception:
        pass
    return name, limit, clock


def loss_fn(model, aux):
    def run(b):
        out = model(b)
        valid = (out["attention_mask"] != 0).unsqueeze(-1)
        return (out["sequence_output"].float() * aux * valid).sum()
    return run


def grads(model):
    return {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}


def check_agreement(model, b, aux, set_skip_padding):
    """loss and gradients of the three arms' computations with dropout off (eager, one step each)"""
    from mmf_b200.graphs import static_rows
    model.eval()
    res = {}
    for arm in ("dense", "packed", "static"):
        set_skip_padding(model, arm != "dense")
        model.zero_grad(set_to_none=True)
        out = model(b) if arm != "static" else None
        if arm == "static":
            with static_rows():
                out = model(b)
        valid = (out["attention_mask"] != 0).unsqueeze(-1)
        terms = out["sequence_output"].float() * aux * valid
        terms.sum().backward()
        res[arm] = (float(terms.sum()), float(terms.detach().abs().sum()), grads(model))
    model.train()
    set_skip_padding(model, False)
    ld, mag, gd = res["dense"]
    worst, dl = 0.0, 0.0
    for arm in ("packed", "static"):
        lp, _, gp = res[arm]
        worst = max([worst] + [rel(gp[k], gd[k]) for k in gd if gd[k].norm() > 1e-6 and ".key.bias" not in k])
        dl = max(dl, abs(lp - ld) / mag)
    return dl, worst, dl < 1e-2 and worst < 2e-2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,166")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.visual_bert import B200VisualBERT
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_skip_padding needs an H100")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = B200VisualBERT(config(0.1)).to(dev).train()
    ok_all = True
    for B in [int(x) for x in a.batches.split(",")]:
        for dist, (text, regions) in DISTS.items():
            b, aux = batch(B, text, regions, dev, seed=1)
            dl, worst, ok = check_agreement(model, b, aux, set_skip_padding)
            ok_all &= ok
            set_skip_padding(model, False)
            dense_graph = GraphedStep(model, loss_fn(model, aux), b, warmup=a.warmup)
            set_skip_padding(model, True)
            packed_graph = GraphedStep(model, loss_fn(model, aux), b, warmup=a.warmup, static_rows=True)

            def eager():
                model.zero_grad(set_to_none=True)
                loss_fn(model, aux)(b).backward()

            arms = {"dense_graphed": (False, lambda: dense_graph(b)), "packed_eager": (True, eager),
                    "packed_graphed": (True, lambda: packed_graph(b))}
            times = {k: [] for k in arms}
            for _ in range(a.rounds):
                for arm, (skip, fn) in arms.items():
                    set_skip_padding(model, skip)
                    for _ in range(a.warmup):
                        fn()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(a.steps):
                        fn()
                    torch.cuda.synchronize()
                    times[arm].append((time.perf_counter() - t0) / a.steps)
            set_skip_padding(model, False)
            del dense_graph, packed_graph
            name, limit, clock = card()
            res = {"batch": B, "distribution": dist, "text": list(text), "regions": list(regions), "card": name,
                   "power_limit_w": limit, "sm_clock_mhz": clock, "agree": ok, "loss_rel_diff": dl,
                   "worst_grad_rel_l2": worst}
            for arm, ts in times.items():
                res[arm] = {"ms_per_step": round(statistics.median(ts) * 1e3, 2),
                            "ms_per_step_all": [round(t * 1e3, 2) for t in ts]}
            res["packed_graphed_vs_dense_graphed"] = round(res["dense_graphed"]["ms_per_step"] /
                                                           res["packed_graphed"]["ms_per_step"], 3)
            res["packed_graphed_vs_packed_eager"] = round(res["packed_eager"]["ms_per_step"] /
                                                          res["packed_graphed"]["ms_per_step"], 3)
            print(json.dumps(res), flush=True)
    return 0 if ok_all else 1


if __name__ == "__main__":
    sys.exit(main())
