#!/usr/bin/env python
"""Gradient clipping + optimizer step on one GPU: torch.nn.utils.clip_grad_norm_ followed by B200AdamW.step() against
B200AdamW.clip_grad_norm (device-side norm, coefficient read by the AdamW kernel) followed by step().

    python tools/bench_clip.py [--iters 50] [--warmup 5]

Parameter sets: the registered m4c model (default configuration, bert-base text BERT + 4-layer MMT + 5050-way output,
with its learning-rate groups) and the VisualBERT trunk of BASELINE.json configs[1] (12 layers, 768 wide).  One backward
at a small batch installs the gradients (the packs' .grad become views of their flat buffers); the timed loop is
clip + step alone, max_norm 0.25, so every iteration clips.  The two alternatives alternate in one process, each figure
is the median of three runs of --iters iterations timed with CUDA events (device time including any gap the host
leaves).  One JSON line with the card's name and power limit.  It fails without a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

MAX_NORM = 0.25


def _events_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def m4c_model(dev):
    import torch
    from bench_m4c import ANS, OCR_MAX, sample_list
    from mmf_b200 import models as MD
    from mmf_b200.registry import registry
    registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
    registry.register("textvqa_num_final_outputs", ANS + OCR_MAX)
    registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1}))
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).to(dev).train()
    sl = sample_list(8, dev, torch.Generator().manual_seed(182))
    sum(v.sum() for v in model(sl)["losses"].values()).backward()
    cfg = MD.ConfigNode({"optimizer": {"params": {"lr": 1e-4}}})
    return model, model.get_optimizer_parameters(cfg), dict(lr=1e-4, eps=1e-8, weight_decay=0.0)


def visual_bert_model(dev):
    import torch
    import bench
    wl = bench.WORKLOADS["visual_bert"]()
    torch.manual_seed(0)
    model = wl.build(0.1).to(dev).train()
    batch = bench.to_device(wl.host_batch(8, 1234), dev)
    aux = wl.aux(8, dev)
    wl.loss(model, batch, aux).backward()
    return model, list(model.parameters()), dict(lr=5e-5, eps=1e-6, weight_decay=0.01)


def measure(name, build, dev, iters, warmup):
    import torch
    from mmf_b200 import lib
    from mmf_b200.optim import B200AdamW
    model, groups, hp = build(dev)
    opt = B200AdamW(groups, arithmetic="torch", **hp)
    params = [p for g in opt.param_groups for p in g["params"]]
    grads = [p.grad for p in params if p.grad is not None]
    n_grad = sum(g.numel() for g in grads)

    def torch_clip():
        torch.nn.utils.clip_grad_norm_(params, MAX_NORM)
        opt.step()

    def fused_clip():
        opt.clip_grad_norm(MAX_NORM)
        opt.step()

    runs = {"torch_clip_grad_norm_": torch_clip, "fused_clip_grad_norm": fused_clip}
    launches = {}
    for k, fn in runs.items():
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        c0 = lib.launch_count()
        fn()
        launches[k] = lib.launch_count() - c0
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    for _ in range(3):
        for k, fn in runs.items():
            ms[k].append(_events_ms(fn, iters))
    med = {k: statistics.median(v) for k, v in ms.items()}
    # step() alone, for scale: the part both alternatives share
    for _ in range(warmup):
        opt.step()
    step_ms = statistics.median(_events_ms(opt.step, iters) for _ in range(3))
    return {"params": name, "tensors_with_grad": len(grads), "grad_elements": n_grad,
            "fp32_grad_mb": round(4 * n_grad / 1e6, 1), "ms": ms, "median_ms": med, "step_only_ms": step_ms,
            "library_launches_per_iter": launches,
            "speedup": med["torch_clip_grad_norm_"] / med["fused_clip_grad_norm"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip needs an H100: the fusion path has no CPU fallback")
    from bench_lxmert import card
    dev = torch.device("cuda", 0)
    name, limit = card()
    res = [measure("m4c", m4c_model, dev, args.iters, args.warmup),
           measure("visual_bert_configs1_trunk", visual_bert_model, dev, args.iters, args.warmup)]
    print(json.dumps({"metric": "clip_grad_norm + AdamW step, torch clip vs fused device-side clip (ms per iteration)",
                      "gpu": name, "power_limit_w": limit, "max_norm": MAX_NORM, "iters": args.iters, "results": res}))


if __name__ == "__main__":
    main()
