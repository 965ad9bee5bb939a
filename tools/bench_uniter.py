#!/usr/bin/env python
"""The registered UNITER model's pretraining step (forward + backward), per task, on one GPU.

    python tools/bench_uniter.py [--batches 64 256] [--steps 10] [--warmup 3]

Workload: the reference's shapes - bert-base trunk (12 layers of 768/12h/3072), 60 tokens + 100 regions x 2048, dropout
0.1, bf16 compute, synthetic inputs resident in HBM; one timing per task (mlm, itm, mrc, mrfr, wra) with the task draw
pinned to it, and the library's kernel launches per step.  For word-region alignment the step is timed twice in the same
run, alternating: with the fused optimal-transport kernels and with the plain-torch restatement of mmf/modules/ot.py
(oracle/ot_oracle.optimal_transport_dist, fp32, on the same GPU tensors) in their place; the two kernels are also
timed alone.  CUDA events; one JSON line with the card's name and power limit.  It fails without a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

T_TOK, R_REG, FEAT, VOCAB, NCLS = 60, 100, 2048, 30522, 1601
TASKS = ["mlm", "itm", "mrc", "mrfr", "wra"]


def sample_list(B, dev, g):
    import torch
    from mmf_b200.sample import SampleList
    lens = torch.randint(T_TOK // 2, T_TOK + 1, (B,), generator=g)
    mask = (torch.arange(T_TOK)[None] < lens[:, None]).long()
    ids = torch.randint(1, VOCAB, (B, T_TOK), generator=g)
    labels = torch.full((B, T_TOK), -1, dtype=torch.long)
    pick = (torch.rand(B, T_TOK, generator=g) < 0.15) & (mask == 1)
    labels[pick] = ids[pick]
    lo = torch.rand(B, R_REG, 2, generator=g) * 0.5
    sl = SampleList(
        input_ids=ids, input_ids_masked=torch.where(pick, torch.full_like(ids, 103), ids), input_mask=mask,
        lm_label_ids=labels, image_feature_0=torch.randn(B, R_REG, FEAT, generator=g).abs(),
        image_info_0={"max_features": torch.randint(R_REG // 2, R_REG + 1, (B,), generator=g),
                      "bbox": torch.cat([lo + 1.0, lo + 1.2 + torch.rand(B, R_REG, 2, generator=g)], -1),
                      "cls_prob": torch.softmax(torch.randn(B, R_REG, NCLS, generator=g), -1)},
        is_correct=torch.randint(0, 2, (B,), generator=g), dataset_name="coco", dataset_type="train")
    return sl.to(dev)


def torch_ot(seq, T_len, R_len, x_len, y_len, beta=0.5, iteration=50, k=1):
    """what the reference's WRA head runs: mmf/modules/ot.py in fp32 torch ops"""
    import torch
    from oracle import ot_oracle as FO
    xp = torch.arange(T_len, device=seq.device)[None] >= torch.as_tensor(x_len, device=seq.device)[:, None]
    yp = torch.arange(R_len, device=seq.device)[None] >= torch.as_tensor(y_len, device=seq.device)[:, None]
    return FO.optimal_transport_dist(seq[:, :T_len].float(), seq[:, T_len:T_len + R_len].float(), xp, yp, beta, iteration, k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dropout", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_uniter needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    import mmf_b200.mmft  # noqa: F401
    from bench_lxmert import card, timed
    from mmf_b200 import functional as F, lib, models as MD, ops
    torch.manual_seed(0)
    bert = dict(hidden_dropout_prob=args.dropout, attention_probs_dropout_prob=args.dropout)
    cfg = MD.load_model_config("uniter", overrides=dict(
        do_pretraining=True, tasks=",".join(TASKS), mask_probability=0.15, hidden_dropout_prob=args.dropout, encoder=bert,
        text_embeddings=bert, heads={t: {"type": t} for t in TASKS}))
    model = MD.build_model(cfg).to(dev).train()
    name, limit = card()
    warm = max(3, args.warmup)
    fused_ot = ops.optimal_transport_dist
    rows = []
    for B in args.batches:
        g = torch.Generator().manual_seed(4321 + B)
        base = sample_list(B, dev, g)

        def step():
            model.zero_grad(set_to_none=True)
            sum(model(type(base)(base))["losses"].values()).backward()      # the forward edits its sample list: a fresh one

        row = {"batch": B}
        for task in TASKS:
            model.tasks = [task]
            l0 = lib.launch_count()
            ms = timed(step, args.steps, args.warmup)
            row[task] = {"ms_per_step": ms, "samples_per_s": B / (ms / 1e3),
                         "library_launches_per_step": (lib.launch_count() - l0) // (args.steps + warm)}
        # word-region alignment with the fused kernels and with torch ops in their place, alternating
        model.tasks = ["wra"]
        ms_f, ms_t = [], []
        for _ in range(3):
            ops.optimal_transport_dist = fused_ot
            ms_f.append(timed(step, args.steps, args.warmup))
            ops.optimal_transport_dist = torch_ot
            ms_t.append(timed(step, args.steps, args.warmup))
        ops.optimal_transport_dist = fused_ot
        row["wra_fused_ms_per_step"], row["wra_torch_ot_ms_per_step"] = ms_f, ms_t
        # the two kernels alone
        seq = torch.randn(B, T_TOK + R_REG, 768, device=dev).to(torch.bfloat16)
        xl, yl = [T_TOK] * B, [R_REG] * B
        x, y = seq[:, :T_TOK], seq[:, T_TOK:]
        dist, plan, saved = F.ot_fwd(x, y, xl, yl)
        dseq, gout = torch.empty_like(seq), torch.ones(B, device=dev)
        row["ot_fwd_kernel_ms"] = timed(lambda: F.ot_fwd(x, y, xl, yl), 50, 5)
        row["ot_bwd_kernel_ms"] = timed(lambda: F.ot_bwd(gout, plan, saved, x, y, xl, yl, dseq[:, :T_TOK], dseq[:, T_TOK:]), 50, 5)
        seqf = seq.float().requires_grad_(True)

        def torch_ot_alone():
            seqf.grad = None
            torch_ot(seqf, T_TOK, R_REG, xl, yl).sum().backward()
        row["torch_ot_fwd_bwd_ms"] = timed(torch_ot_alone, 10, 3)
        rows.append(row)
    print(json.dumps({
        "metric": "UNITER pretraining step per task (fwd+bwd, registered model)", "unit": "ms/step",
        "gpu": name, "power_limit_w": limit, "steps": args.steps, "warmup": warm, "dtype": "bf16", "data": "synthetic",
        "config": {"layers": 12, "hidden": 768, "tokens": T_TOK, "regions": R_REG, "feature_dim": FEAT,
                   "region_classes": NCLS, "dropout": args.dropout, "ot": {"beta": 0.5, "iterations": 50, "k": 1}},
        "results": rows}))


if __name__ == "__main__":
    main()
