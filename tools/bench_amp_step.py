#!/usr/bin/env python
"""MMF's fp16 training update (training.fp16: autocast forward, scaler.scale(loss).backward(), clip at 1.0 times the
loss scale, scaler.step, scaler.update) on one GPU, three ways, over a capturable B200AdamW:
  unscale     today's path: the same optimizer with `_step_supports_amp_scaling` set False, so GradScaler runs its
              unscale_ pass over every gradient and reads found_inf on the host before step(); the clip threshold is
              `1.0 * scaler.get_scale()`, as mmf/utils/general.py clip_gradients computes it (a host read as well);
  fused       the eager fused update: clip_grad_norm(1.0, scale=<device scale>), scaler.step, scaler.update - the
              optimizer's kernels unscale and skip on the device, nothing is read on the host;
  graph       GraphedStep(..., optimizer=, max_grad_norm=1.0, scaler=): the whole step replayed as one CUDA graph.

    python tools/bench_amp_step.py [--models mmbt visual_bert lxmert m4c] [--steps 10] [--warmup 3]

Workloads as tools/bench_graph_train_step.py: MMBT configs[0] (batch 2), the VisualBERT trunk at B = 32, LXMERT
pretraining at B = 64 with static rows and M4C at TextVQA shapes.  The arms are alternated three times in one process
(median reported), CUDA events, one JSON line per model with the card's name and power limit read in the same run.  It
fails without a GPU.
"""
import argparse
import copy
import contextlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["mmbt", "visual_bert", "lxmert", "m4c"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_amp_step needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_graph_train_step import workloads
    from bench_lxmert import card, timed
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.optim import B200AdamW
    name, limit = card()
    head = {"metric": "fp16 training step: autocast fwd + scaled bwd + clip_grad_norm(1.0 * scale) + scaler.step + update",
            "unit": "ms/step", "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup,
            "dtype": "fp16 autocast", "data": "synthetic"}
    table = workloads(dev)
    for key in args.models:
        torch.manual_seed(0)
        model, batch, loss_of, groups, hp, static, B = table[key]()
        ctx = static_rows if static else contextlib.nullcontext
        models = {a: (model if a == "unscale" else copy.deepcopy(model)) for a in ("unscale", "fused", "graph")}
        opts = {a: B200AdamW(groups(m), capturable=True, **hp) for a, m in models.items()}
        opts["unscale"]._step_supports_amp_scaling = False
        scalers = {a: torch.amp.GradScaler("cuda") for a in models}

        def fwd_bwd(a):
            m, s = models[a], scalers[a]
            m.zero_grad(set_to_none=True)
            with ctx(), torch.autocast("cuda", dtype=torch.float16):
                loss = loss_of(m)(batch)
            s.scale(loss).backward()

        def unscale():
            fwd_bwd("unscale")
            o, s = opts["unscale"], scalers["unscale"]
            o.clip_grad_norm(1.0 * s.get_scale())
            s.step(o)
            s.update()

        def fused():
            fwd_bwd("fused")
            o, s = opts["fused"], scalers["fused"]
            o.clip_grad_norm(1.0, scale=s._get_scale_async())
            s.step(o)
            s.update()

        m_g = models["graph"]

        def graph_loss(b):
            with torch.autocast("cuda", dtype=torch.float16, cache_enabled=False):
                return loss_of(m_g)(b)
        g = GraphedStep(m_g, graph_loss, batch, static_rows=static, optimizer=opts["graph"], max_grad_norm=1.0,
                        scaler=scalers["graph"])

        def graph():
            g(batch)

        arms = (("unscale", unscale), ("fused", fused), ("graph", graph))
        times = {a: [] for a, _ in arms}
        for _ in range(3):
            for a, fn in arms:
                times[a].append(timed(fn, args.steps, args.warmup))
        med = {a: sorted(v)[1] for a, v in times.items()}
        print(json.dumps(dict(head, model=key, batch=B, ms_per_step=times, median_ms=med,
                              fused_vs_unscale=med["unscale"] / med["fused"],
                              graph_vs_unscale=med["unscale"] / med["graph"],
                              final_scale={a: s.get_scale() for a, s in scalers.items()})), flush=True)
        del g, models, opts, scalers, model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
