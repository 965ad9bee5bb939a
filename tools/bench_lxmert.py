#!/usr/bin/env python
"""The registered LXMERT model's pretraining step (forward + backward of the four losses), samples/s on one GPU.

    python tools/bench_lxmert.py [--batches 64 256] [--steps 10] [--warmup 3]

Workload: mmf/configs/models/lxmert/defaults.yaml - l/r/x = 9/5/5 layers of 768/12h/3072, 20 tokens + 36 regions x 2048
(+ 4 box coordinates), dropout 0.1, bf16 compute, the masked-LM, matched, visual (obj + feat) and answer losses,
synthetic inputs resident in HBM.  In the same call it times the trunk alone (B200LXMERTBase forward + backward of a
random projection of both streams) so that the heads' share of the step is visible.  CUDA events; one JSON line with the
card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T_TOK, R_REG, FEAT, VOCAB, NCLS = 20, 36, 2048, 30522, 1600


def card():
    import torch
    name, limit = torch.cuda.get_device_name(0), None
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        limit = float(q.stdout.strip().splitlines()[0]) if q.returncode == 0 else None
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pass
    return name, limit


def sample_list(B, dev, g):
    import torch
    from mmf_b200.sample import SampleList
    lens = torch.randint(T_TOK // 2, T_TOK + 1, (B,), generator=g)
    mask = (torch.arange(T_TOK)[None] < lens[:, None]).long()
    seg = ((torch.arange(T_TOK)[None] >= lens[:, None] // 2) & (mask == 1)).long()
    labels = torch.full((B, T_TOK), -1, dtype=torch.long)
    pick = (torch.rand(B, T_TOK, generator=g) < 0.15) & (mask == 1)
    labels[pick] = torch.randint(0, VOCAB, (B, T_TOK), generator=g)[pick]
    sl = SampleList(
        input_ids=torch.randint(1, VOCAB, (B, T_TOK), generator=g), input_mask=mask, segment_ids=seg, lm_label_ids=labels,
        image_feature_0=torch.randn(B, R_REG, FEAT, generator=g).abs(),
        image_info_0={"max_features": torch.randint(R_REG // 2, R_REG + 1, (B,), generator=g),
                      "bbox": torch.rand(B, R_REG, 4, generator=g),
                      "cls_prob": torch.softmax(torch.randn(B, R_REG, NCLS, generator=g), -1)},
        image_labels=(torch.rand(B, R_REG, generator=g) < 0.15).long(),
        targets=torch.softmax(torch.randn(B, 3129, generator=g) * 3.0, -1), is_correct=torch.randint(0, 2, (B,), generator=g),
        dataset_name="masked_vqa2", dataset_type="train")
    return sl.to(dev)


def timed(step, steps, warmup):
    import torch
    for _ in range(max(3, warmup)):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dropout", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lxmert needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from mmf_b200 import lib, models as MD
    torch.manual_seed(0)
    cfg = MD.load_model_config("lxmert", overrides={"hidden_dropout_prob": args.dropout,
                                                    "attention_probs_dropout_prob": args.dropout})
    model = MD.build_model(cfg).to(dev).train()
    trunk = model.model.bert
    name, limit = card()
    rows = []
    for B in args.batches:
        g = torch.Generator().manual_seed(1234 + B)
        sl = sample_list(B, dev, g)

        def step():
            model.zero_grad(set_to_none=True)
            sum(model(sl)["losses"].values()).backward()

        vmask = (torch.arange(R_REG, device=dev)[None] < sl["image_info_0"]["max_features"][:, None]).long()
        wl, wv = torch.randn(B, T_TOK, 768, device=dev), torch.randn(B, R_REG, 768, device=dev)

        def trunk_step():
            trunk.zero_grad(set_to_none=True)
            (lang, visn), pooled = trunk(sl["input_ids"], sl["input_mask"], sl["segment_ids"], sl["image_feature_0"],
                                         sl["image_info_0"]["bbox"], vmask)
            ((lang * wl).sum() + (visn * wv).sum() + pooled.sum()).backward()

        l0 = lib.launch_count()
        ms = timed(step, args.steps, args.warmup)
        launches = (lib.launch_count() - l0) // (args.steps + max(3, args.warmup))
        ms_trunk = timed(trunk_step, args.steps, args.warmup)
        rows.append({"batch": B, "samples_per_s": B / (ms / 1e3), "ms_per_step": ms, "trunk_ms_per_step": ms_trunk,
                     "heads_share": 1.0 - ms_trunk / ms, "library_launches_per_step": launches})
    print(json.dumps({
        "metric": "LXMERT pretraining samples/sec (fwd+bwd, registered model)", "unit": "samples/s",
        "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": max(3, args.warmup), "dtype": "bf16",
        "data": "synthetic", "config": {"layers_l_r_x": [9, 5, 5], "hidden": 768, "tokens": T_TOK, "regions": R_REG,
                                        "feature_dim": FEAT, "dropout": args.dropout},
        "results": rows}))


if __name__ == "__main__":
    main()
