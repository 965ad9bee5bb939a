#!/usr/bin/env python
"""Whole training steps (zero grads, forward, backward, gradient clipping, AdamW) on one GPU, three ways:
  eager       model.zero_grad(); loss.backward(); opt.clip_grad_norm(1.0); opt.step() with today's B200AdamW;
  graph_fb    today's best: GraphedStep replays forward + backward, then the same eager clip + step;
  graph_step  GraphedStep(..., optimizer=B200AdamW(..., capturable=True), max_grad_norm=1.0): the whole step is one replay
              (the groups' hyper-parameters are staged by one host-to-device copy before it).
Also timed alone: `opt_eager`, today's eager clip + step on the gradients of a step (what `eager` and `graph_fb` pay on
top of forward + backward), and for every model the new segment kernel over its loose parameters (the ones outside the
engine's parameter packs), against the 28 bytes per parameter it moves (4 fp32 streams read, 3 written).

    python tools/bench_graph_train_step.py [--models mmbt visual_bert lxmert m4c] [--steps 10] [--warmup 3]

Models: MMBT (BASELINE.json configs[0], batch 2), the VisualBERT trunk (configs[1]) at B = 32 with bench.py's loss,
LXMERT pretraining at B = 64 (tools/bench_lxmert.py's inputs, static rows, its four losses) and M4C at the TextVQA shapes
of tools/bench_m4c.py (B = 128, Adam groups from get_optimizer_parameters).  Dropout as each configuration sets it.  The
arms are alternated three times in one process (median reported), CUDA events, one JSON line per model with the card's
name and power limit read in the same run.  It fails without a GPU.
"""
import argparse
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def workloads(dev):
    import torch

    def bench_wl(name, B):
        def make():
            import bench
            wl = bench.WORKLOADS[name]()
            model = wl.build(0.1).to(dev).train()
            batch = bench.to_device(wl.host_batch(B, 1), dev)
            aux = wl.aux(B, dev)
            return (model, batch, lambda m: (lambda b: wl.loss(m, b, aux)), lambda m: list(m.parameters()),
                    dict(lr=1e-4, weight_decay=0.01), False, B)
        return make

    def lxmert():
        import bench_lxmert as BL
        from mmf_b200 import models as MD
        from mmf_b200.sample import SampleList
        B = 64
        model = MD.build_model(MD.load_model_config("lxmert")).to(dev).train()
        sl = BL.sample_list(B, dev, torch.Generator().manual_seed(71))
        if "cls_prob" in sl["image_info_0"]:
            sl["image_info_0"]["cls_prob"] = torch.as_tensor(sl["image_info_0"]["cls_prob"]).to(dev)
        batch = {k: v for k, v in sl.items() if torch.is_tensor(v) or isinstance(v, dict)}
        meta = {k: v for k, v in sl.items() if k not in batch}

        def loss_of(m):
            return lambda b: sum(v.sum() for v in m(SampleList(dict(b, **meta)))["losses"].values())
        return model, batch, loss_of, lambda m: list(m.parameters()), dict(lr=1e-4, weight_decay=0.01), True, B

    def m4c():
        import bench_m4c as BM
        from mmf_b200 import models as MD
        from mmf_b200.registry import registry
        from mmf_b200.sample import SampleList
        B = 128
        registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
        registry.register("textvqa_num_final_outputs", BM.ANS + BM.OCR_MAX)
        registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1}))
        model = MD.build_model(MD.load_model_config("m4c")).to(dev).train()
        sl = BM.sample_list(B, dev, torch.Generator().manual_seed(182))
        batch = {k: v for k, v in sl.items() if torch.is_tensor(v) or isinstance(v, dict)}
        meta = {k: v for k, v in sl.items() if k not in batch}
        cfg = MD.ConfigNode({"optimizer": {"type": "Adam", "params": {"lr": 1e-4, "eps": 1e-8, "weight_decay": 0}}})

        def loss_of(m):
            return lambda b: sum(v.sum() for v in m(SampleList(dict(b, **meta)))["losses"].values())
        return (model, batch, loss_of, lambda m: m.get_optimizer_parameters(cfg),
                dict(lr=1e-4, eps=1e-8, weight_decay=0.0, arithmetic="torch"), False, B)
    return {"mmbt": bench_wl("mmbt", 2), "visual_bert": bench_wl("visual_bert", 32), "lxmert": lxmert, "m4c": m4c}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["mmbt", "visual_bert", "lxmert", "m4c"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_train_step needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200 import functional as F
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW
    name, limit = card()
    head = {"metric": "training step: zero_grad + fwd + bwd + clip_grad_norm(1.0) + AdamW", "unit": "ms/step",
            "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup, "dtype": "bf16",
            "data": "synthetic"}
    table = workloads(dev)
    for key in args.models:
        torch.manual_seed(0)
        model, batch, loss_of, groups, hp, static, B = table[key]()
        m_eager, m_fb, m_step = model, copy.deepcopy(model), copy.deepcopy(model)
        o_eager, o_fb = B200AdamW(groups(m_eager), **hp), B200AdamW(groups(m_fb), **hp)
        o_step = B200AdamW(groups(m_step), capturable=True, **hp)

        def eager():
            m_eager.zero_grad(set_to_none=True)
            loss_of(m_eager)(batch).backward()
            o_eager.clip_grad_norm(1.0)
            o_eager.step()

        def opt_eager():
            o_eager.clip_grad_norm(1.0)
            o_eager.step()

        g_fb = GraphedStep(m_fb, loss_of(m_fb), batch, static_rows=static)

        def graph_fb():
            g_fb(batch)
            o_fb.clip_grad_norm(1.0)
            o_fb.step()

        g_step = GraphedStep(m_step, loss_of(m_step), batch, static_rows=static, optimizer=o_step, max_grad_norm=1.0)

        def graph_step():
            g_step(batch)

        plan = o_step._cap
        seg_table = plan.table

        def segments():
            F.adamw_segments(seg_table, plan.hp, mode=plan.mode)

        arms = (("eager", eager), ("graph_fb", graph_fb), ("graph_step", graph_step), ("opt_eager", opt_eager)) + \
            ((("segment_kernel", segments),) if seg_table is not None else ())
        times = {a: [] for a, _ in arms}
        for _ in range(3):
            for a, fn in arms:
                times[a].append(timed(fn, args.steps if a != "segment_kernel" else 100, args.warmup))
        med = {a: sorted(v)[1] for a, v in times.items()}
        n_loose = sum(r[4] for r in seg_table.rows) if seg_table is not None else 0
        n_all = sum(p.numel() for g in o_step.param_groups for p in g["params"] if p.grad is not None)
        print(json.dumps(dict(head, model=key, batch=B, ms_per_step=times, median_ms=med,
                              graph_step_vs_eager=med["eager"] / med["graph_step"],
                              graph_step_vs_graph_fb=med["graph_fb"] / med["graph_step"],
                              opt_share_of_eager=med["opt_eager"] / med["eager"],
                              params=n_all, packs=len(plan.packs), loose_tensors=len(plan.loose),
                              loose_params=n_loose,
                              segment_kernel_gbps=28 * n_loose / (med["segment_kernel"] * 1e6) if n_loose else None)),
              flush=True)
        del g_fb, g_step, m_eager, m_fb, m_step, model, o_eager, o_fb, o_step, plan
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
