#!/usr/bin/env python
"""Skip-padding (packed rows + variable-length attention) against the dense path on the VisualBERT trunk of
BASELINE.json configs[1]: 12 L / 768 / 12 h / 3072, 128 text tokens + 100 regions x 2048, batch 166, bf16 compute,
dropout 0.1, forward + backward, eager in both arms.

    python tools/bench_varlen.py [--batch 166] [--steps 10] [--warmup 3] [--rounds 5]

Both arms use one loss that ignores padded positions, (sequence_output * aux * valid).sum(), and run in one process,
alternating `--rounds` times.  Two length distributions: bench.py's own (text U{64..128}, regions U{50..100}) and a
short-text one (text U{8..24}, regions U{10..100}).  Before timing, the arms are checked to agree on the loss and every
parameter gradient with dropout off (the masks the arms draw differ, so the check cannot run with dropout on): the loss
difference within 1e-2 of sum |seq * aux * valid| (the loss sums terms of random sign, so |loss| itself is no scale),
gradients within 2e-2 relative L2.  Prints one JSON line per distribution.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, R, FEAT, H, VOCAB = 128, 100, 2048, 768, 30522
DISTS = {"bench": ((64, 128), (50, 100)), "short_text": ((8, 24), (10, 100))}


def config(p):
    return types.SimpleNamespace(hidden_size=H, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12,
                                 vocab_size=VOCAB, max_position_embeddings=512, type_vocab_size=2, hidden_dropout_prob=p,
                                 attention_probs_dropout_prob=p, layer_norm_eps=1e-12, hidden_act="gelu",
                                 initializer_range=0.02, pad_token_id=0, visual_embedding_dim=FEAT)


def batch(B, text, regions, dev, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(text[0], text[1] + 1, (B,), generator=g)
    nreg = torch.randint(regions[0], regions[1] + 1, (B,), generator=g)
    b = {"input_ids": torch.randint(0, VOCAB, (B, T), generator=g),
         "input_mask": (torch.arange(T)[None, :] < lens[:, None]).long(),
         "segment_ids": torch.zeros(B, T, dtype=torch.long),
         "image_feature_0": torch.randn(B, R, FEAT, generator=g).abs(),
         "image_info_0": {"max_features": nreg}}
    aux = torch.randn(B, T + R, H, generator=g)
    to = lambda x: {k: to(v) for k, v in x.items()} if isinstance(x, dict) else x.to(dev)
    return to(b), aux.to(dev)


def step(model, b, aux):
    out = model(b)
    valid = (out["attention_mask"] != 0).unsqueeze(-1)
    terms = out["sequence_output"].float() * aux * valid
    loss = terms.sum()
    loss.backward()
    return loss, terms.detach().abs().sum()


def card():
    import torch
    name, limit = torch.cuda.get_device_name(0), None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        limit = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return name, limit


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()


def check_agreement(model, b, aux, set_skip_padding):
    model.eval()
    out = {}
    for skip in (False, True):
        set_skip_padding(model, skip)
        model.zero_grad(set_to_none=True)
        loss, mag = step(model, b, aux)
        out[skip] = (float(loss), float(mag), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    model.train()
    (ld, mag, gd), (lp, _, gp) = out[False], out[True]
    worst = max(rel(gp[k], gd[k]) for k in gd if gd[k].norm() > 1e-6 and ".key.bias" not in k)
    dl = abs(lp - ld) / mag          # the loss sums terms of random sign: its difference is relative to their magnitude
    return dl, worst, dl < 1e-2 and worst < 2e-2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=166)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import torch
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.visual_bert import B200VisualBERT
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = B200VisualBERT(config(0.1)).to(dev).train()
    name, limit = card()
    ok_all = True
    for dist, (text, regions) in DISTS.items():
        b, aux = batch(a.batch, text, regions, dev, seed=1)
        with torch.no_grad():
            model.eval()
            valid = (model(b)["attention_mask"] != 0).float()
            model.train()
        lens = valid.sum(1)
        S = valid.shape[1]
        frac = float(lens.sum() / (a.batch * S))
        attn_frac = float((lens ** 2).sum() / (a.batch * S * S))
        dl, worst, ok = check_agreement(model, b, aux, set_skip_padding)
        ok_all &= ok
        times = {"dense": [], "skip_padding": []}
        for _ in range(a.rounds):
            for arm in times:
                set_skip_padding(model, arm == "skip_padding")
                for _ in range(a.warmup):
                    model.zero_grad(set_to_none=True)
                    step(model, b, aux)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    model.zero_grad(set_to_none=True)
                    step(model, b, aux)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) / a.steps)
        set_skip_padding(model, False)
        res = {"distribution": dist, "text": list(text), "regions": list(regions), "batch": a.batch,
               "valid_row_fraction": round(frac, 4), "sum_len2_over_BS2": round(attn_frac, 4), "card": name,
               "power_limit_w": limit, "agree": ok, "loss_rel_diff": dl, "worst_grad_rel_l2": worst}
        for arm, ts in times.items():
            ms = statistics.median(ts) * 1e3
            res[arm] = {"ms_per_step": round(ms, 2), "samples_per_s": round(a.batch / (ms / 1e3), 1),
                        "ms_per_step_all": [round(t * 1e3, 2) for t in ts]}
        res["speedup"] = round(res["dense"]["ms_per_step"] / res["skip_padding"]["ms_per_step"], 3)
        print(json.dumps(res), flush=True)
    return 0 if ok_all else 1


if __name__ == "__main__":
    sys.exit(main())
