#!/usr/bin/env python
"""The registered UNITER model's pretraining step (forward + backward) eager and captured, per task and for the mixed
task draw the model makes, on one GPU.

    python tools/bench_graph_uniter.py [--batches 64 256] [--steps 10] [--warmup 3]

Workload: the shapes of tools/bench_uniter.py - bert-base trunk (12 layers of 768/12h/3072), 60 tokens + 100 regions x
2048, dropout 0.1, bf16 compute, synthetic inputs resident in HBM.  Eager is today's step (the forward draws its task and
region masks and gathers the masked rows on the host); graphed is mmf_b200.graphs.GraphedTaskSteps (the same draws on
the host, then one CUDA-graph replay of that task's step, the batch copied into the static inputs first).  Per task the
draw is pinned to it; "mixed" draws among all five as the registered model does.  The two modes alternate three times in
one process and the median is reported, with the peak memory allocated while each mode runs.  CUDA events; one JSON line
with the card's name and power limit, read in the same run.  It fails without a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

TASKS = ["mlm", "itm", "mrc", "mrfr", "wra"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dropout", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_uniter needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    import mmf_b200.mmft  # noqa: F401
    from bench_lxmert import card, timed
    from bench_uniter import R_REG, sample_list
    from mmf_b200 import models as MD
    from mmf_b200.graphs import GraphedTaskSteps
    from mmf_b200.sample import SampleList
    torch.manual_seed(0)
    bert = dict(hidden_dropout_prob=args.dropout, attention_probs_dropout_prob=args.dropout)
    cfg = MD.load_model_config("uniter", overrides=dict(
        do_pretraining=True, tasks=",".join(TASKS), mask_probability=0.15, hidden_dropout_prob=args.dropout, encoder=bert,
        text_embeddings=bert, heads={t: {"type": t} for t in TASKS}))
    model = MD.build_model(cfg).to(dev).train()
    name, limit = card()
    rows = []
    for B in args.batches:
        g = torch.Generator().manual_seed(4321 + B)
        base = sample_list(B, dev, g)
        info = dict(base["image_info_0"])          # every input a device tensor: the captured step reads no host value
        info["image_width"] = torch.full((B,), 640.0, device=dev)
        info["image_height"] = torch.full((B,), 480.0, device=dev)
        base["image_info_0"] = info
        batch = {k: v for k, v in base.items() if torch.is_tensor(v) or isinstance(v, dict)}
        meta = {k: v for k, v in base.items() if k not in batch}

        def loss_fn(b):
            return sum(model(SampleList(dict(b, **meta)))["losses"].values())

        def eager():
            model.zero_grad(set_to_none=True)
            loss_fn(batch).backward()

        model.zero_grad(set_to_none=True)
        torch.cuda.reset_peak_memory_stats(dev)
        graphed = GraphedTaskSteps(model, loss_fn, batch, warmup=args.warmup)
        torch.cuda.synchronize(dev)
        capture_peak = torch.cuda.max_memory_allocated(dev)
        row = {"batch": B, "capture_peak_gib": capture_peak / 2 ** 30}
        for which in TASKS + ["mixed"]:
            model.tasks = list(TASKS) if which == "mixed" else [which]
            ms = {"eager": [], "graphed": []}
            peak = {}
            for _ in range(3):
                for mode, fn in (("eager", eager), ("graphed", lambda: graphed(batch))):
                    torch.cuda.synchronize(dev)
                    torch.cuda.reset_peak_memory_stats(dev)
                    ms[mode].append(timed(fn, args.steps, args.warmup))
                    peak[mode] = max(peak.get(mode, 0), torch.cuda.max_memory_allocated(dev))
            med = {m: statistics.median(v) for m, v in ms.items()}
            row[which] = {"eager_ms": ms["eager"], "graphed_ms": ms["graphed"], "eager_median_ms": med["eager"],
                          "graphed_median_ms": med["graphed"], "speedup": med["eager"] / med["graphed"],
                          "eager_peak_gib": peak["eager"] / 2 ** 30, "graphed_peak_gib": peak["graphed"] / 2 ** 30}
            print(json.dumps({"batch": B, which: row[which]}), file=sys.stderr)
        model.tasks = list(TASKS)
        del graphed
        torch.cuda.empty_cache()
        rows.append(row)
    print(json.dumps({
        "metric": "UNITER pretraining step (fwd+bwd), eager vs GraphedTaskSteps, per task and mixed", "unit": "ms/step",
        "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup, "runs": 3, "dtype": "bf16",
        "data": "synthetic", "config": {"layers": 12, "hidden": 768, "tokens": 60, "regions": R_REG, "feature_dim": 2048,
                                        "dropout": args.dropout, "mask_probability": 0.15},
        "results": rows}))


if __name__ == "__main__":
    main()
