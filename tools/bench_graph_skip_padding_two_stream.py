#!/usr/bin/env python
"""Skip-padding of M4C's causal tail and of the two-stream encoders captured in CUDA graphs, with the packing planned by one
device kernel (patch.set_skip_padding(..., device_plan=True) inside static_rows()).  Three arms, alternated `--rounds` times
in one process, median reported:

  dense_graphed   - GraphedStep / GraphedForward over the dense path;
  packed_eager    - today's skip-padding: packing planned on the host, eager launches;
  packed_graphed  - GraphedStep(..., static_rows=True) / GraphedForward(..., static_rows=True) with device_plan: packing
                    planned on the device at capacity B*S, every layer kernel bounded by its stream's device count.

    python tools/bench_graph_skip_padding_two_stream.py [--steps 10] [--warmup 3] [--rounds 3] [--only vilbert,m4c,...]

Configurations:
  vilbert        - the ViLBERT trunk of tools/bench_vilbert.py (12 t / 6 v / 6 c, 36 tokens + 36 regions x 2048, dropout
                   0.1), forward + backward of a loss over the valid positions, at B = 32 and 256, with the bench's
                   lengths (text U{18..36}) and short text (U{4..12}), regions U{18..36} (tools/bench_varlen_two_stream.py);
  m4c            - the registered m4c training step at TextVQA shapes (tools/bench_m4c.py's batch), B = 128;
  m4c_captioner  - the registered m4c_captioner greedy decode (12 steps, one forward) on the same inputs, B = 64.
Before timing, the arms are checked to agree with dropout off: the losses within 1e-2 of the sum of |terms| (ViLBERT) or
relatively (M4C), the decode's first-step scores within 2e-2 of their largest magnitude.  Also times the planning kernel alone.  Prints one JSON line per
configuration with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_graph_skip_padding import card  # noqa: E402


def _timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def _arms_times(arms, a):
    """arms: {name: (setup, fn)}; alternated a.rounds times, median ms"""
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, (setup, fn) in arms.items():
            setup()
            times[name].append(_timed(fn, a.steps, a.warmup))
    res = {}
    for name, ts in times.items():
        res[name] = {"ms": round(statistics.median(ts) * 1e3, 2), "ms_all": [round(t * 1e3, 2) for t in ts]}
    res["packed_graphed_vs_dense_graphed"] = round(res["dense_graphed"]["ms"] / res["packed_graphed"]["ms"], 3)
    res["packed_graphed_vs_packed_eager"] = round(res["packed_eager"]["ms"] / res["packed_graphed"]["ms"], 3)
    return res


def _header(what, **kw):
    name, limit, clock = card()
    return dict({"config": what, "card": name, "power_limit_w": limit, "sm_clock_mhz": clock}, **kw)


def planner(a):
    """the planning kernel alone (CUDA events, median of 200 launches)"""
    import torch
    from mmf_b200 import functional as F
    out = []
    g = torch.Generator().manual_seed(0)
    for shapes in ([(166, 228)], [(128, 182)], [(166, 228), (166, 182)]):
        B = shapes[0][0]
        masks = [(((torch.rand(B, S, generator=g) < 0.6).float() - 1) * 10000.0).cuda() for _, S in shapes]
        lens = [S for _, S in shapes]
        for _ in range(20):
            F.plan_packing(masks, B, lens)
        ts = []
        for _ in range(200):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            F.plan_packing(masks, B, lens)
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        out.append({"streams": ["%dx%d" % s for s in shapes], "us_median": round(statistics.median(ts), 2)})
    print(json.dumps(_header("plan_packing kernel", runs=out)), flush=True)


def vilbert(a):
    import torch
    from bench_varlen_two_stream import WORKLOADS, batch, build, step
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.patch import set_skip_padding
    dev = torch.device("cuda", 0)
    model = build("vilbert", dev)
    w = WORKLOADS["vilbert"]
    ok_all = True
    for B in (32, 256):
        for dist, (text, regions) in w["dists"].items():
            b = batch("vilbert", B, w["T"], w["R"], text, regions, dev, seed=1)
            loss = lambda bb: step_loss(model, bb)
            dl = _vilbert_agreement(model, b)
            ok = dl < 1e-2
            ok_all &= ok
            set_skip_padding(model, False, two_stream=True)
            dense = GraphedStep(model, loss, b, warmup=a.warmup)
            set_skip_padding(model, True, two_stream=True, device_plan=True)
            packed = GraphedStep(model, loss, b, warmup=a.warmup, static_rows=True)

            def eager():
                model.zero_grad(set_to_none=True)
                step("vilbert", model, b)

            arms = {"dense_graphed": (lambda: set_skip_padding(model, False, two_stream=True), lambda: dense(b)),
                    "packed_eager": (lambda: set_skip_padding(model, True, two_stream=True), eager),
                    "packed_graphed": (lambda: set_skip_padding(model, True, two_stream=True, device_plan=True),
                                       lambda: packed(b))}
            res = _arms_times(arms, a)
            set_skip_padding(model, False, two_stream=True)
            del dense, packed
            print(json.dumps(_header("vilbert trunk train step", batch=B, distribution=dist, text=list(text),
                                     regions=list(regions), agree=ok, loss_rel_diff=dl, **res)), flush=True)
    return ok_all


def _vilbert_agreement(model, b):
    """relative loss difference of the host- and device-planned packed arms from the dense one, dropout off (a function of
    its own, so no autograd graph of these eager steps outlives it: a capture after them binds the gradients afresh)"""
    from bench_varlen_two_stream import step
    from mmf_b200.graphs import static_rows
    from mmf_b200.patch import set_skip_padding
    model.eval()
    vals = {}
    for arm in ("dense", "packed", "static"):
        set_skip_padding(model, arm != "dense", two_stream=True, device_plan=arm == "static")
        model.zero_grad(set_to_none=True)
        with static_rows() if arm == "static" else _null():
            loss, mag = step("vilbert", model, b)
        vals[arm] = (float(loss.detach()), float(mag))
    model.train()
    model.zero_grad(set_to_none=True)
    return max(abs(vals[k][0] - vals["dense"][0]) / vals["dense"][1] for k in ("packed", "static"))


def step_loss(model, b):
    t, v, _ = model(b["ids"], b["feats"], b["loc"], attention_mask=b["vt"].long(), image_attention_mask=b["vi"].long())
    return (t.float() * b["wt"]).sum() + (v.float() * b["wi"]).sum()


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *e):
        return False


def _m4c_model(name, dev):
    import torch
    from bench_m4c import ANS, OCR_MAX
    from mmf_b200 import models as MD
    from mmf_b200.registry import registry
    registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
    registry.register("textvqa_num_final_outputs", ANS + OCR_MAX)
    registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1, "UNK_IDX": 0}))   # the captioner masks UNK
    torch.manual_seed(0)
    return MD.build_model(MD.load_model_config(name)).to(dev)


def m4c_train(a):
    import torch
    from bench_m4c import sample_list
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.patch import set_skip_padding
    dev = torch.device("cuda", 0)
    model = _m4c_model("m4c", dev).train()
    B = 128
    sl = sample_list(B, dev, torch.Generator().manual_seed(182))
    loss = lambda b: sum(v.sum() for v in model(b)["losses"].values())
    model.eval()
    vals = {}
    for arm in ("dense", "packed", "static"):
        set_skip_padding(model, arm != "dense", causal=True, device_plan=arm == "static")
        with torch.no_grad(), static_rows() if arm == "static" else _null():
            vals[arm] = float(loss(sl))
    model.train()
    dl = max(abs(vals[k] - vals["dense"]) / max(abs(vals["dense"]), 1e-6) for k in ("packed", "static"))
    ok = dl < 1e-2
    set_skip_padding(model, False, causal=True)
    dense = GraphedStep(model, loss, sl, warmup=a.warmup)
    set_skip_padding(model, True, causal=True, device_plan=True)
    packed = GraphedStep(model, loss, sl, warmup=a.warmup, static_rows=True)

    def eager():
        model.zero_grad(set_to_none=True)
        loss(sl).backward()

    arms = {"dense_graphed": (lambda: set_skip_padding(model, False, causal=True), lambda: dense(sl)),
            "packed_eager": (lambda: set_skip_padding(model, True, causal=True), eager),
            "packed_graphed": (lambda: set_skip_padding(model, True, causal=True, device_plan=True), lambda: packed(sl))}
    res = _arms_times(arms, a)
    print(json.dumps(_header("m4c train step (TextVQA shapes)", batch=B, agree=ok, loss_rel_diff=dl, **res)), flush=True)
    return ok


def captioner_decode(a):
    import torch
    from bench_m4c import sample_list
    from mmf_b200.graphs import GraphedForward, static_rows
    from mmf_b200.patch import set_skip_padding
    dev = torch.device("cuda", 0)
    model = _m4c_model("m4c_captioner", dev).eval()
    B = 64
    sl = sample_list(B, dev, torch.Generator().manual_seed(182))
    sl["dataset_type"] = "val"
    fwd = lambda b: model(b)
    scores = {}
    for arm in ("dense", "packed", "static"):
        set_skip_padding(model, arm != "dense", causal=True, device_plan=arm == "static")
        with torch.no_grad(), static_rows() if arm == "static" else _null():
            scores[arm] = fwd(sl)["scores"].float()
    # greedy decoding feeds each step's argmax back, so a near-tie decided differently by rounding changes every later step:
    # the first step's scores are compared, relative to their largest magnitude, and the agreeing argmaxes are counted
    ref = scores["dense"]
    diff = max((scores[k][:, 0] - ref[:, 0]).abs().max().item() for k in ("packed", "static")) / ref[:, 0].abs().max().item()
    same = min((scores[k].argmax(-1) == ref.argmax(-1)).float().mean().item() for k in ("packed", "static"))
    ok = diff < 2e-2
    set_skip_padding(model, False, causal=True)
    dense = GraphedForward(model, sl, warmup=a.warmup)
    set_skip_padding(model, True, causal=True, device_plan=True)
    packed = GraphedForward(model, sl, warmup=a.warmup, static_rows=True)

    def eager():
        with torch.no_grad():
            fwd(sl)

    arms = {"dense_graphed": (lambda: set_skip_padding(model, False, causal=True), lambda: dense(sl)),
            "packed_eager": (lambda: set_skip_padding(model, True, causal=True), eager),
            "packed_graphed": (lambda: set_skip_padding(model, True, causal=True, device_plan=True), lambda: packed(sl))}
    res = _arms_times(arms, a)
    print(json.dumps(_header("m4c_captioner greedy decode", batch=B, agree=ok, step0_score_rel_diff=diff,
                             argmax_agree_frac=same, **res)), flush=True)
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="planner,vilbert,m4c,m4c_captioner")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_skip_padding_two_stream needs an H100")
    runs = {"planner": planner, "vilbert": vilbert, "m4c": m4c_train, "m4c_captioner": captioner_decode}
    ok = True
    for name in a.only.split(","):
        ok &= runs[name](a) is not False
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
