#!/usr/bin/env python
"""The registered VinVL model's training step (forward + backward), on one GPU.

    python tools/bench_vinvl.py [--pretrain-batches 64 256] [--classify-batches 32 256] [--steps 10] [--warmup 3]

Workloads: bert-base trunk (12 layers of 768/12h/3072), region features 2054 wide (VinVL's 2048 + 6 box values), dropout
0.1, bf16 compute, synthetic inputs resident in HBM:
  pretraining     35 tokens + 50 regions; two trunk passes per step (masked captions, corrupt captions), masked LM on
                  ~15 % of the valid tokens plus the three-way contrastive loss;
  classification  128 tokens + 50 regions; heads.mlp with 3129 labels (the VQA2 answer space), cross-entropy.
Text and regions are padded (per-sample lengths drawn between half and the full width), and each step is timed with the
dense encoder path and with skip-padding (mmf_b200.patch.set_skip_padding) in the same run, alternating, three times each.
CUDA events; one JSON line with the card's name and power limit and the library's launches per step.  It fails without
a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

PRE_TOK, CLS_TOK, R_REG, FEAT, VOCAB, NUM_LABELS = 35, 128, 50, 2054, 30522, 3129


def _padded(B, n, g):
    import torch
    lens = torch.randint(n // 2, n + 1, (B,), generator=g)
    return lens, (torch.arange(n)[None] < lens[:, None]).long()


def sample_list(B, T, dev, g):
    import torch
    from mmf_b200.sample import SampleList
    _, mask = _padded(B, T, g)
    _, mask_corrupt = _padded(B, T, g)
    nreg, _ = _padded(B, R_REG, g)
    ids = torch.randint(1, VOCAB, (B, T), generator=g)
    labels = torch.full((B, T), -1, dtype=torch.long)
    pick = (torch.rand(B, T, generator=g) < 0.15) & (mask == 1)
    labels[pick] = ids[pick]
    sl = SampleList(
        input_ids=ids, input_ids_masked=torch.where(pick, torch.full_like(ids, 103), ids),
        input_ids_corrupt=torch.randint(1, VOCAB, (B, T), generator=g), lm_label_ids=labels, input_mask=mask,
        input_mask_corrupt=mask_corrupt, segment_ids=torch.zeros(B, T, dtype=torch.long),
        segment_ids_corrupt=torch.zeros(B, T, dtype=torch.long), image_feature_0=torch.randn(B, R_REG, FEAT, generator=g),
        image_info_0={"max_features": nreg}, contrastive_labels=torch.randint(0, 3, (B, 1), generator=g),
        labels=torch.randint(0, NUM_LABELS, (B,), generator=g), dataset_name="vqa2", dataset_type="train")
    return sl.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pretrain-batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--classify-batches", type=int, nargs="+", default=[32, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dropout", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_vinvl needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200 import lib, models as MD
    from mmf_b200.patch import set_skip_padding
    torch.manual_seed(0)
    bert = dict(hidden_dropout_prob=args.dropout, attention_probs_dropout_prob=args.dropout)
    models = {
        "pretraining": MD.build_model(MD.load_model_config("vinvl", overrides=dict(
            do_pretraining=True, bert_overrides=bert,
            heads={"mlm": {"hidden_dropout_prob": args.dropout}, "contrast": {"hidden_dropout_prob": args.dropout}}))),
        "classification": MD.build_model(MD.load_model_config("vinvl", overrides=dict(
            bert_overrides=bert, heads={"mlp": {"num_labels": NUM_LABELS, "hidden_dropout_prob": args.dropout}}))),
    }
    name, limit = card()
    warm = max(3, args.warmup)
    rows = []
    for kind, batches, T in (("pretraining", args.pretrain_batches, PRE_TOK),
                             ("classification", args.classify_batches, CLS_TOK)):
        model = models[kind].to(dev).train()
        for B in batches:
            sl = sample_list(B, T, dev, torch.Generator().manual_seed(2054 + B))
            valid = float(sl["input_mask"].sum() + sl["image_info_0"]["max_features"].sum()) / (B * (T + R_REG))

            def step():
                model.zero_grad(set_to_none=True)
                sum(v.sum() for v in model(sl)["losses"].values()).backward()

            row = {"workload": kind, "batch": B, "tokens": T, "regions": R_REG, "valid_fraction": round(valid, 3)}
            dense, packed = [], []
            for _ in range(3):
                set_skip_padding(model, False)
                dense.append(timed(step, args.steps, args.warmup))
                set_skip_padding(model, True)
                packed.append(timed(step, args.steps, args.warmup))
            for mode, ms in (("dense", dense), ("skip_padding", packed)):
                set_skip_padding(model, mode == "skip_padding")
                l0 = lib.launch_count()
                step()
                torch.cuda.synchronize()
                median = sorted(ms)[len(ms) // 2]
                row[mode] = {"ms_per_step": ms, "samples_per_s_at_median": B / (median / 1e3),
                             "library_launches_per_step": lib.launch_count() - l0}
            set_skip_padding(model, False)
            rows.append(row)
    print(json.dumps({
        "metric": "VinVL training step (fwd+bwd, registered model), dense and skip-padding", "unit": "ms/step",
        "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": warm, "dtype": "bf16", "data": "synthetic",
        "config": {"layers": 12, "hidden": 768, "feature_dim": FEAT, "dropout": args.dropout,
                   "classification_labels": NUM_LABELS},
        "results": rows}))


if __name__ == "__main__":
    main()
