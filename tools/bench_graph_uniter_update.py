#!/usr/bin/env python
"""The registered UNITER model's whole pretraining update with MMF's training.update_frequency, eager and captured, for
the mixed task draw, on one GPU.

    python tools/bench_graph_uniter_update.py [--batches 64 256] [--k 4] [--updates 5] [--warmup 2]

Workload: the shapes of tools/bench_graph_uniter.py - bert-base trunk (12 layers of 768/12h/3072), 60 tokens + 100
regions x 2048, dropout 0.1, bf16 compute, synthetic inputs resident in HBM - with a capturable B200AdamW (two weight-decay
groups), clipping at 1.0 and K micro-batches per update, each drawing its task among all five.  Eager is MMF's loop
(zero_grad, K x (forward, backward), clip, step); graphed is GraphedTaskSteps(..., update_frequency=K): K micro-batch
replays and one update replay.  Two precisions: "bf16" (no loss scaling) and "scaler" (a torch.amp.GradScaler: the loss
is scaled, the clip is at max_norm times the device scale, scaler.step and scaler.update; the fused kernels compute in
bf16 either way).  Each side has its own optimizer over the same model.  The two modes alternate three times in one
process and the median ms per update is reported.  CUDA events; one JSON line with the card's name and power limit, read
in the same run.  It fails without a GPU.
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
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--updates", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_uniter_update needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    import mmf_b200.mmft  # noqa: F401
    from bench_lxmert import card, timed
    from bench_uniter import R_REG, sample_list
    from mmf_b200 import models as MD
    from mmf_b200.graphs import GraphedTaskSteps
    from mmf_b200.optim import B200AdamW
    from mmf_b200.sample import SampleList
    torch.manual_seed(0)
    bert = dict(hidden_dropout_prob=args.dropout, attention_probs_dropout_prob=args.dropout)
    cfg = MD.load_model_config("uniter", overrides=dict(
        do_pretraining=True, tasks=",".join(TASKS), mask_probability=0.15, hidden_dropout_prob=args.dropout, encoder=bert,
        text_embeddings=bert, heads={t: {"type": t} for t in TASKS}))
    model = MD.build_model(cfg).to(dev).train()

    def opt_of():
        decay = [p for n, p in model.named_parameters() if not n.endswith("bias") and "LayerNorm" not in n]
        rest = [p for n, p in model.named_parameters() if n.endswith("bias") or "LayerNorm" in n]
        return B200AdamW([{"params": decay, "weight_decay": 0.01}, {"params": rest, "weight_decay": 0.0}], lr=1e-5,
                         capturable=True)
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
        row = {"batch": B}
        for prec in ("bf16", "scaler"):
            opt_e, opt_g = opt_of(), opt_of()
            sc_e = torch.amp.GradScaler("cuda") if prec == "scaler" else None
            sc_g = torch.amp.GradScaler("cuda") if prec == "scaler" else None

            def eager():
                model.zero_grad(set_to_none=True)
                for _ in range(args.k):
                    loss = loss_fn(batch)
                    (loss if sc_e is None else sc_e.scale(loss)).backward()
                if sc_e is None:
                    opt_e.clip_grad_norm(1.0)
                    opt_e.step()
                else:
                    opt_e.clip_grad_norm(1.0, scale=sc_e._get_scale_async())
                    sc_e.step(opt_e)
                    sc_e.update()

            model.zero_grad(set_to_none=True)
            graphed = GraphedTaskSteps(model, loss_fn, batch, warmup=args.warmup, optimizer=opt_g, max_grad_norm=1.0,
                                       scaler=sc_g, update_frequency=args.k)

            def replayed():
                for _ in range(args.k):
                    graphed(batch)
            ms = {"eager": [], "graphed": []}
            for _ in range(3):
                for mode, fn in (("eager", eager), ("graphed", replayed)):
                    torch.cuda.synchronize(dev)
                    ms[mode].append(timed(fn, args.updates, args.warmup))
            med = {m: statistics.median(v) for m, v in ms.items()}
            row[prec] = {"eager_ms": ms["eager"], "graphed_ms": ms["graphed"], "eager_median_ms": med["eager"],
                         "graphed_median_ms": med["graphed"], "speedup": med["eager"] / med["graphed"]}
            print(json.dumps({"batch": B, prec: row[prec]}), file=sys.stderr)
            del graphed, opt_e, opt_g
            model.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
        rows.append(row)
    print(json.dumps({
        "metric": "UNITER pretraining update with update_frequency, eager loop vs GraphedTaskSteps, mixed task draw",
        "unit": "ms/update", "gpu": name, "power_limit_w": limit, "k": args.k, "updates": args.updates,
        "warmup": args.warmup, "runs": 3, "data": "synthetic",
        "config": {"layers": 12, "hidden": 768, "tokens": 60, "regions": R_REG, "feature_dim": 2048,
                   "dropout": args.dropout, "mask_probability": 0.15, "max_grad_norm": 1.0},
        "results": rows}))


if __name__ == "__main__":
    main()
