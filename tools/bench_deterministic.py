#!/usr/bin/env python
"""Cost of deterministic mode (torch.use_deterministic_algorithms(True)): training steps and the ordered reduction
kernels against their atomic counterparts, on one GPU.

    python tools/bench_deterministic.py [--steps 10] [--warmup 3]

Workloads (bench.py's, default batches): visual_bert (BASELINE.json configs[1], 166 x (128 tokens + 100 regions) =
37 848 rows) as a CUDA-graphed step - one graph captured with the flag off and one with it on - then vilbert and
uniter_large as eager steps.  Off and on alternate in one process; each figure is the median of three timed runs of
--steps steps.  Kernels: each ordered reduction against the atomic one at the visual_bert shapes (37 848 rows, hidden 768,
FFN 3072; wgrad split factors from engine.best_splits; the LayerNorm backward also at H = 2048, its register kernel),
CUDA events over 50 launches.  One JSON line with the card's name and power limit.  It fails without a GPU.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _events_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _with_flag(on, fn):
    import torch
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        return fn()
    finally:
        torch.use_deterministic_algorithms(prev)


def step_times(name, steps, warmup):
    import torch
    import bench
    from mmf_b200.graphs import GraphedStep
    dev = torch.device("cuda", 0)
    wl = bench.WORKLOADS[name]()
    torch.manual_seed(0)
    model = wl.build(0.1).to(dev).train()
    B = wl.default_batch
    batch = bench.to_device(wl.host_batch(B, 1234), dev)
    aux = wl.aux(B, dev)
    if name == "visual_bert":
        graphs = {on: _with_flag(on, lambda: GraphedStep(model, lambda b: wl.loss(model, b, aux), batch, warmup=3))
                  for on in (False, True)}
        runs = {on: (lambda g=graphs[on]: g()) for on in (False, True)}
    else:
        def eager(on):
            def step():
                model.zero_grad(set_to_none=True)
                wl.loss(model, batch, aux).backward()
            return lambda: _with_flag(on, step)
        runs = {on: eager(on) for on in (False, True)}
    for on in (False, True):
        for _ in range(warmup):
            runs[on]()
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    for _ in range(3):
        for on in (False, True):
            ms[on].append(_events_ms(runs[on], steps))
    off, on = statistics.median(ms[False]), statistics.median(ms[True])
    return {"workload": name, "batch": B, "graphed": name == "visual_bert", "ms_off": ms[False], "ms_on": ms[True],
            "median_ms_off": off, "median_ms_on": on, "overhead": on / off - 1.0}


def kernel_times(reps=50):
    import torch
    from mmf_b200 import engine, functional as F, lib
    dev = torch.device("cuda", 0)
    M, H, I = 37848, 768, 3072
    g = torch.Generator().manual_seed(0)
    rows = []

    def pair(label, fn):
        t = {on: [] for on in (False, True)}
        for on in (False, True):
            _with_flag(on, fn)
        torch.cuda.synchronize()
        for _ in range(3):
            for on in (False, True):
                t[on].append(_with_flag(on, lambda: _events_ms(fn, reps)))
        off, on = statistics.median(t[False]), statistics.median(t[True])
        rows.append({"kernel": label, "us_atomic": off * 1e3, "us_ordered": on * 1e3, "ratio": on / off})

    x = {n: torch.randn(M, n, generator=g).to(torch.bfloat16).to(dev) for n in (H, 3 * H, I)}
    for m_out, n_in in ((3 * H, H), (H, H), (I, H), (H, I)):
        s = engine.best_splits(m_out, n_in, M)
        dw = torch.zeros(m_out, n_in, device=dev)
        pair("wgrad %dx%d K=%d splits=%d" % (m_out, n_in, M, s),
             lambda a=x[m_out], b=x[n_in], dw=dw, s=s: F.gemm(a, b, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                                                             splits=s))
    for n in (3 * H, I, H):
        out = torch.zeros(n, device=dev)
        pair("colsum %dx%d" % (M, n), lambda xx=x[n], out=out: F.colsum(xx, out))
    # H = 768: the streaming kernel at the bench shape; H = 2048: the register kernel (1024 < H <= 2048)
    for h in (H, 2048):
        y = x[H] if h == H else torch.randn(M, h, generator=g).to(torch.bfloat16).to(dev)
        gam, bet = torch.ones(h, dtype=torch.bfloat16, device=dev), torch.zeros(h, dtype=torch.bfloat16, device=dev)
        _, mean, rstd = F.layernorm_fwd(y, gam, bet)
        dg, db, dbias = (torch.zeros(h, device=dev) for _ in range(3))
        keep = F.dropout_bits((M,), h, 0.1, 1, 0, dev)
        pair("layernorm_bwd %dx%d (+dropout, dbias)" % (M, h),
             lambda y=y, gam=gam, mean=mean, rstd=rstd, dg=dg, db=db, dbias=dbias, keep=keep:
             F.layernorm_bwd(y, y, mean, rstd, gam, dg, db, dbias=dbias, drop_mask=keep, drop_scale=1 / 0.9))
    S = 128
    for kind, idx in (("type", torch.zeros(M, dtype=torch.int32)),
                      ("position", (torch.arange(M) % S).to(torch.int32)),
                      ("word", torch.randint(0, 30522, (M,), generator=g).to(torch.int32))):
        srt, order = F.sort_indices(idx.to(dev))
        tab = torch.zeros(int(idx.max()) + 1, H, device=dev)
        pair("embed_scatter_sorted %s %dx%d" % (kind, M, H), lambda srt=srt, order=order, tab=tab:
             F.embed_scatter_sorted(x[H], tab, srt, order))
    logits = torch.randn(8192, 30528, generator=g).to(torch.bfloat16).to(dev)
    labels = torch.randint(0, 30528, (8192,), generator=g).to(dev)
    loss = torch.zeros(1, device=dev)
    pair("ce_rows 8192x30528", lambda: F.ce_rows(logits, labels, -1, 1.0, loss))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=["visual_bert", "vilbert", "uniter_large"])
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic needs an H100: the fusion path has no CPU fallback")
    from bench_lxmert import card
    name, limit = card()
    steps = [step_times(w, args.steps, max(1, args.warmup)) for w in args.workloads]
    print(json.dumps({"metric": "deterministic-mode cost (flag off vs on, alternated, median of 3)", "gpu": name,
                      "power_limit_w": limit, "steps": args.steps, "dtype": "bf16", "data": "synthetic",
                      "steps_ms": steps, "kernels_us": kernel_times()}))


if __name__ == "__main__":
    main()
