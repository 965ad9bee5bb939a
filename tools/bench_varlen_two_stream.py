#!/usr/bin/env python
"""Two-stream skip-padding (both streams packed, variable-length self- and cross-attention) against the dense path,
forward + backward, eager in both arms, bf16 compute, dropout 0.1.

    python tools/bench_varlen_two_stream.py --workload vilbert|lxmert [--batch N] [--steps 10] [--warmup 3] [--rounds 5]

Workloads:
  vilbert - tools/bench_vilbert.py's model and inputs (BASELINE.json configs[2]: 12 t / 6 v / 6 c, 36 tokens + 36 regions x
            2048, batch 512).  Distributions: the bench's own (text U{18..36}, regions U{18..36}) and a short-text one
            (text U{4..12}, regions U{18..36}).
  lxmert  - the LXMERT encoder of BASELINE.json configs[4]: 9 l / 5 r / 5 x, 768 / 12 h / 3072, 20 tokens + 100 regions x
            2048 (+ 4 box coordinates), batch 256.  Distribution: text U{5..20}, regions U{10..100}.
Both arms use one loss that ignores padded positions and run in one process, alternating `--rounds` times.  Before timing
the arms are checked to agree with dropout off (the masks the arms draw differ, so the check cannot run with dropout on):
the loss difference within 1e-2 of the sum of |terms|, every parameter gradient within 2e-2 relative L2 (key biases, which
are analytically zero, excepted).  Prints one JSON line per distribution, with the card name and its power limit.
"""
import argparse
import json
import os
import statistics
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_varlen import card, rel          # noqa: E402

VOCAB, FEAT = 30522, 2048
WORKLOADS = {
    "vilbert": dict(T=36, R=36, batch=512, dists={"bench": ((18, 36), (18, 36)), "short_text": ((4, 12), (18, 36))}),
    "lxmert": dict(T=20, R=100, batch=256, dists={"bench": ((5, 20), (10, 100))}),
}


def lxmert_config(p):
    return types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, hidden_dropout_prob=p,
                                 attention_probs_dropout_prob=p, visual_feat_dim=FEAT, visual_pos_dim=4, l_layers=9,
                                 x_layers=5, r_layers=5, initializer_range=0.02)


def build(workload, dev):
    import torch
    torch.manual_seed(0)
    if workload == "vilbert":
        from bench_vilbert import vilbert_config
        from mmf_b200.vilbert import B200ViLBERTBase
        return B200ViLBERTBase(vilbert_config(0.1)).to(dev).train()
    from mmf_b200.lxmert import B200LXMERTEncoder
    return B200LXMERTEncoder(lxmert_config(0.1)).to(dev).train()


def batch(workload, B, T, R, text, regions, dev, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(text[0], text[1] + 1, (B,), generator=g)
    nreg = torch.randint(regions[0], regions[1] + 1, (B,), generator=g)
    vt = torch.arange(T)[None, :] < lens[:, None]
    vi = torch.arange(R)[None, :] < nreg[:, None]
    Hv = 1024 if workload == "vilbert" else 768
    b = {"vt": vt, "vi": vi, "feats": torch.randn(B, R, FEAT, generator=g).abs(),
         "wt": torch.randn(B, T, 768, generator=g) * vt[..., None], "wi": torch.randn(B, R, Hv, generator=g) * vi[..., None]}
    if workload == "vilbert":
        b["ids"] = torch.randint(0, VOCAB, (B, T), generator=g)
        b["loc"] = torch.rand(B, R, 5, generator=g)
    else:
        b["lang"] = torch.randn(B, T, 768, generator=g)
        b["boxes"] = torch.rand(B, R, 4, generator=g)
    return {k: v.to(dev) for k, v in b.items()}


def step(workload, model, b):
    if workload == "vilbert":
        t, v, _ = model(b["ids"], b["feats"], b["loc"], attention_mask=b["vt"].long(), image_attention_mask=b["vi"].long())
    else:
        add = lambda valid: ((~valid).float() * -10000.0)[:, None, None, :]
        t, v = model(b["lang"], add(b["vt"]), (b["feats"], b["boxes"]), add(b["vi"]))
    terms = [t.float() * b["wt"], v.float() * b["wi"]]
    loss = sum(x.sum() for x in terms)
    loss.backward()
    return loss, sum(x.detach().abs().sum() for x in terms)


def check_agreement(workload, model, b, set_skip_padding):
    model.eval()
    out = {}
    for skip in (False, True):
        set_skip_padding(model, skip, two_stream=True)
        model.zero_grad(set_to_none=True)
        loss, mag = step(workload, model, b)
        out[skip] = (float(loss.detach()), float(mag), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    model.train()
    (ld, mag, gd), (lp, _, gp) = out[False], out[True]
    worst = max(rel(gp[k], gd[k]) for k in gd if gd[k].norm() > 1e-6 and not (".key" in k and k.endswith("bias")))
    dl = abs(lp - ld) / mag
    return dl, worst, dl < 1e-2 and worst < 2e-2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="vilbert")
    ap.add_argument("--batch", type=int, default=0, help="0 = the workload's default")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import torch
    from mmf_b200 import functional as F
    from mmf_b200.patch import set_skip_padding
    if not torch.cuda.is_available():
        raise SystemExit("bench_varlen_two_stream needs an H100: the fusion path has no CPU fallback")
    w = WORKLOADS[a.workload]
    B, T, R = a.batch or w["batch"], w["T"], w["R"]
    dev = torch.device("cuda", 0)
    model = build(a.workload, dev)
    name, limit = card()
    calls = [0]
    cross = F.attention_varlen_cross_fwd

    def counted(*args, **kw):
        calls[0] += 1
        return cross(*args, **kw)
    F.attention_varlen_cross_fwd = counted
    ok_all = True
    for dist, (text, regions) in w["dists"].items():
        b = batch(a.workload, B, T, R, text, regions, dev, seed=1)
        dl, worst, ok = check_agreement(a.workload, model, b, set_skip_padding)
        ok_all &= ok
        times = {"dense": [], "skip_padding": []}
        for _ in range(a.rounds):
            for arm in times:
                set_skip_padding(model, arm == "skip_padding", two_stream=True)
                for _ in range(a.warmup):
                    model.zero_grad(set_to_none=True)
                    step(a.workload, model, b)
                torch.cuda.synchronize()
                calls[0] = 0
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    model.zero_grad(set_to_none=True)
                    step(a.workload, model, b)
                torch.cuda.synchronize()
                times[arm].append((time.perf_counter() - t0) / a.steps)
                if arm == "skip_padding" and calls[0] == 0:
                    raise SystemExit("the skip_padding arm did not run packed cross-attention")
        set_skip_padding(model, False, two_stream=True)
        res = {"workload": a.workload, "distribution": dist, "text": list(text), "regions": list(regions), "batch": B,
               "T": T, "R": R, "text_valid_fraction": round(float(b["vt"].float().mean()), 4),
               "region_valid_fraction": round(float(b["vi"].float().mean()), 4), "card": name, "power_limit_w": limit,
               "agree": ok, "loss_rel_diff": dl, "worst_grad_rel_l2": worst}
        for arm, ts in times.items():
            ms = statistics.median(ts) * 1e3
            res[arm] = {"ms_per_step": round(ms, 2), "samples_per_s": round(B / (ms / 1e3), 1),
                        "ms_per_step_all": [round(t * 1e3, 2) for t in ts]}
        res["speedup"] = round(res["dense"]["ms_per_step"] / res["skip_padding"]["ms_per_step"], 3)
        print(json.dumps(res), flush=True)
    F.attention_varlen_cross_fwd = cross
    return 0 if ok_all else 1


if __name__ == "__main__":
    sys.exit(main())
