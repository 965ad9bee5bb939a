#!/usr/bin/env python
"""The registered `albef_vit_encoder`'s forward + backward, on one GPU.

    python tools/bench_albef_vit.py [--batches 64 256] [--steps 10] [--warmup 3]

Workload: the encoder's default configuration (ViT-B/16: 12 blocks of 768 / 12 heads / 3072, 224 x 224 images, 197
positions) with drop_path_rate 0.1 and drop_rate = attn_drop_rate = 0 (ALBEF's fine-tuning setting), bf16 compute, train
mode, synthetic images resident in HBM, loss sum(out * w).  Each batch is timed eagerly and as a GraphedStep replay,
alternating, three times each.  CUDA events.  One JSON line per case, with the card's name and power limit read in the
same run.  It fails without a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_albef_vit needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200.encoders import build_encoder
    from mmf_b200.graphs import GraphedStep
    torch.manual_seed(0)
    name, limit = card()
    head = {"metric": "ALBEF ViT-B/16 encoder fwd+bwd (albef_vit_encoder)", "unit": "ms/step", "gpu": name,
            "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup, "dtype": "bf16", "data": "synthetic",
            "image_size": 224, "positions": 197, "drop_path_rate": 0.1}
    enc = build_encoder({"type": "albef_vit_encoder", "params": {"params": {"drop_path_rate": 0.1}}}).to(dev).train()
    for B in args.batches:
        g = torch.Generator(device=dev).manual_seed(B)
        batch = {"images": torch.randn(B, 3, 224, 224, device=dev, generator=g),
                 "w": torch.randn(B, 197, 768, device=dev, generator=g)}

        def loss_of(b):
            return (enc(b["images"]) * b["w"]).sum()

        def eager():
            enc.zero_grad(set_to_none=True)
            loss_of(batch).backward()

        graphed = GraphedStep(enc, loss_of, batch)
        times = {"eager": [], "graphed": []}
        for _ in range(3):
            times["eager"].append(timed(eager, args.steps, args.warmup))
            times["graphed"].append(timed(graphed, args.steps, args.warmup))
        for mode in ("eager", "graphed"):
            ms = times[mode]
            median = sorted(ms)[len(ms) // 2]
            print(json.dumps(dict(head, mode=mode, batch=B, ms_per_step=ms, median_ms=median,
                                  images_per_s=B / (median / 1e3))), flush=True)
        del graphed
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
