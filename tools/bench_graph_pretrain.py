#!/usr/bin/env python
"""Pretraining steps of the registered LXMERT, VinVL and ViLT models (forward + backward), eager against CUDA-graph
replay in static-rows mode, on one GPU.

    python tools/bench_graph_pretrain.py [--batches 64 256] [--steps 10] [--warmup 3]

Shapes and seeded inputs are those of tools/bench_lxmert.py (20 tokens + 36 regions, masked_vqa2, the four losses),
tools/bench_vinvl.py (35 tokens + 50 regions, masked LM + three-way contrastive, two trunk passes) and tools/bench_vilt.py
(masked COCO: 40 tokens + 145 image positions, mlm_multi + itm, two trunk passes); about 15 % of the valid tokens carry a
masked-LM label.  Dropout 0.1 as configured.  Three variants of each step, alternated in one process, three timings each
(median reported):
  eager         today's step: the masked-LM head gathers its labelled rows with a host read of their count;
  eager_static  the same step inside mmf_b200.graphs.static_rows(): rows selected and counted on the device, the
                vocabulary-sized kernels bounded by that count, no host read;
  graphed       GraphedStep(model, loss, batch, static_rows=True) replays.
CUDA events.  One JSON line per (model, batch), with the card's name and power limit read in the same run, the labelled
row count and the capacity (rows of the labels tensor).  It fails without a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def workloads(dev):
    import bench_lxmert as BL
    import bench_vilt as BT
    import bench_vinvl as BV
    from mmf_b200 import models as MD

    def lxmert():
        cfg = MD.load_model_config("lxmert", overrides={"hidden_dropout_prob": 0.1, "attention_probs_dropout_prob": 0.1})
        return MD.build_model(cfg), lambda B, g: BL.sample_list(B, dev, g)

    def vinvl():
        bert = dict(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
        cfg = MD.load_model_config("vinvl", overrides=dict(do_pretraining=True, bert_overrides=bert, heads={
            "mlm": {"hidden_dropout_prob": 0.1}, "contrast": {"hidden_dropout_prob": 0.1}}))
        return MD.build_model(cfg), lambda B, g: BV.sample_list(B, BV.PRE_TOK, dev, g)

    def vilt():
        return (MD.build_model(MD.load_model_config("vilt", overrides=BT.PRETRAIN)),
                lambda B, g: BT.sample_list(B, "masked_coco", dev, g))
    return {"lxmert": lxmert, "vinvl": vinvl, "vilt": vilt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["lxmert", "vinvl", "vilt"])
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_pretrain needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.sample import SampleList
    torch.manual_seed(0)
    name, limit = card()
    head = {"metric": "pretraining step (fwd+bwd, registered model)", "unit": "ms/step", "gpu": name,
            "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup, "dtype": "bf16", "data": "synthetic"}
    table = workloads(dev)
    for key in args.models:
        model, make = table[key]()
        model = model.to(dev).train()
        for B in args.batches:
            sl = make(B, torch.Generator().manual_seed(7 + B))
            if "image_info_0" in sl and "cls_prob" in sl["image_info_0"]:
                sl["image_info_0"]["cls_prob"] = torch.as_tensor(sl["image_info_0"]["cls_prob"]).to(dev)
            batch = {k: v for k, v in sl.items() if torch.is_tensor(v) or isinstance(v, dict)}
            meta = {k: v for k, v in sl.items() if k not in batch}

            def loss_of(b):
                return sum(v.sum() for v in model(SampleList(dict(b, **meta)))["losses"].values())

            def eager():
                model.zero_grad(set_to_none=True)
                loss_of(batch).backward()

            def eager_static():
                model.zero_grad(set_to_none=True)
                with static_rows():
                    loss = loss_of(batch)
                loss.backward()

            model.zero_grad(set_to_none=True)
            graphed = GraphedStep(model, loss_of, batch, static_rows=True)
            times = {"eager": [], "eager_static": [], "graphed": []}
            for _ in range(3):
                for mode, fn in (("eager", eager), ("eager_static", eager_static), ("graphed", graphed)):
                    times[mode].append(timed(fn, args.steps, args.warmup))
            med = {m: sorted(v)[1] for m, v in times.items()}
            lm = sl["lm_label_ids"]
            print(json.dumps(dict(head, model=key, batch=B, labelled_rows=int((lm != -1).sum()), label_rows=lm.numel(),
                                  ms_per_step=times, median_ms=med,
                                  graphed_speedup=med["eager"] / med["graphed"])), flush=True)
            del graphed
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
