#!/usr/bin/env python
"""MMF's gradient accumulation (training.update_frequency: K) on one GPU, two ways, over a capturable B200AdamW:
  eager   MMF's loop: zero_grad(set_to_none=True), K x (forward, backward - scaled with a scaler), then
          clip_grad_norm(1.0) and step(), or with a scaler clip_grad_norm(1.0, scale=<device scale>), scaler.step,
          scaler.update - the eager fused update;
  graph   GraphedStep(..., optimizer=, max_grad_norm=1.0, update_frequency=K[, scaler=]): K calls, each copying the
          batch into the static inputs and replaying the micro-batch graph, the K-th replaying the update graph too.
Both arms use the same optimizer class, so the difference is the launches the graphs save.

    python tools/bench_graph_accumulate.py [--cases mmbt visual_bert lxmert] [--steps 10] [--warmup 3]

Cases, as tools/bench_graph_train_step.py builds them (dropout as each configuration sets it): MMBT configs[0] (batch 2)
at K = 8, the VisualBERT configs[1] trunk at B = 32 and K = 4, LXMERT pretraining at B = 64 and K = 4 with static rows;
each without a scaler (bf16) and with a GradScaler (fp16 autocast).  Every micro-batch feeds the same batch.  The arms
are alternated three times in one process (median reported), CUDA events over `--steps` updates, one JSON line per case
with the card's name and power limit read in the same run.  It fails without a GPU.
"""
import argparse
import contextlib
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

UPDATE_FREQUENCY = {"mmbt": 8, "visual_bert": 4, "lxmert": 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["mmbt", "visual_bert", "lxmert"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_accumulate needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_graph_train_step import workloads
    from bench_lxmert import card, timed
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.optim import B200AdamW
    name, limit = card()
    head = {"metric": "accumulated update: K x (fwd + bwd) + clip_grad_norm(1.0) + AdamW", "unit": "ms/update",
            "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup, "data": "synthetic"}
    table = workloads(dev)
    for key in args.cases:
        K = UPDATE_FREQUENCY[key]
        for amp in (False, True):
            torch.manual_seed(0)
            model, batch, loss_of, groups, hp, static, B = table[key]()
            ctx = static_rows if static else contextlib.nullcontext
            cast = (lambda: torch.autocast("cuda", dtype=torch.float16, cache_enabled=False)) if amp else \
                contextlib.nullcontext
            m_e, m_g = model, copy.deepcopy(model)
            o_e, o_g = B200AdamW(groups(m_e), capturable=True, **hp), B200AdamW(groups(m_g), capturable=True, **hp)
            s_e, s_g = (torch.amp.GradScaler("cuda"), torch.amp.GradScaler("cuda")) if amp else (None, None)
            run_e, run_g = loss_of(m_e), loss_of(m_g)

            def eager():
                m_e.zero_grad(set_to_none=True)
                for _ in range(K):
                    with ctx(), cast():
                        loss = run_e(batch)
                    (loss if s_e is None else s_e.scale(loss)).backward()
                if s_e is None:
                    o_e.clip_grad_norm(1.0)
                    o_e.step()
                else:
                    o_e.clip_grad_norm(1.0, scale=s_e._get_scale_async())
                    s_e.step(o_e)
                    s_e.update()

            def graph_loss(b):
                with cast():
                    return run_g(b)
            g = GraphedStep(m_g, graph_loss, batch, static_rows=static, optimizer=o_g, max_grad_norm=1.0, scaler=s_g,
                            update_frequency=K)

            def graph():
                for _ in range(K):
                    g(batch)

            arms = (("eager", eager), ("graph", graph))
            times = {a: [] for a, _ in arms}
            for _ in range(3):
                for a, fn in arms:
                    times[a].append(timed(fn, args.steps, args.warmup))
            med = {a: sorted(v)[1] for a, v in times.items()}
            print(json.dumps(dict(head, model=key, batch=B, update_frequency=K, static_rows=static,
                                  dtype="fp16 autocast + GradScaler" if amp else "bf16", ms_per_update=times,
                                  median_ms=med, median_ms_per_micro_batch={a: v / K for a, v in med.items()},
                                  graph_vs_eager=med["eager"] / med["graph"],
                                  final_scale=None if not amp else {"eager": s_e.get_scale(), "graph": s_g.get_scale()})),
                  flush=True)
            del g, m_e, m_g, o_e, o_g, model, run_e, run_g
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
