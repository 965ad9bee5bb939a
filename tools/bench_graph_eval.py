#!/usr/bin/env python
"""Evaluation forwards, eager against GraphedForward (one CUDA graph replay per batch), on one GPU.

    python tools/bench_graph_eval.py [--steps 10] [--warmup 3] [--only m4c m4c_captioner vilt visual_bert]

Each workload is the eval forward an evaluation loop runs: model.eval() under torch.no_grad(), `model(batch)` with the
batch's targets, so the scores and the loss.  bf16 compute, synthetic seeded inputs resident in HBM.  Workloads:
  m4c            default m4c configuration at TextVQA shapes (tools/bench_m4c.py's batch): 20 question tokens, 100
                 objects, 50 OCR tokens, 5000 answers + 50 OCR copies, greedy decoding over 12 steps; B = 128;
  m4c_captioner  the same model with remove_unk_in_pred at TextCaps shapes (mmf/configs/datasets/textcaps: 3 caption-
                 prompt tokens, 100 objects, 50 OCR tokens, 30 decoding steps), 5000 words + 50 OCR copies; B = 64, 128;
  vilt           vqa2/vit_b32_384 (tools/bench_vilt.py's batch): 40 tokens + 145 image positions, 3129 answers,
                 logit_bce; B = 32, 256;
  visual_bert    BASELINE.json configs[1]: the VisualBERT trunk (12L/768/12h/3072, 128 tokens + 100 regions), its
                 sequence output; B = 32, 166.
For each: eager and graphed alternated three times in one process (CUDA events over `steps` calls after `warmup`), the
median ms per batch of each and their ratio, the peak allocated memory of one call of each mode (after
reset_peak_memory_stats), the size of the graph's private memory pool right after capture, the library's launches per
eager forward (a replay launches nothing from the host), and whether the replay's scores equal the eager ones bit for
bit on the timed batch.  The card's name and power limit are read in the same run.  One JSON line per case; it fails
without a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

TEXTCAPS_TXT, TEXTCAPS_DEC = 3, 30


def _pool_bytes(graph):
    """bytes of the allocator segments that belong to the graph's private pool"""
    import torch
    return sum(s["total_size"] for s in torch.cuda.memory_snapshot(mempool_id=graph.pool(), include_traces=False))


def _m4c(captioner, B, dev):
    import torch
    import bench_m4c as BM
    from mmf_b200 import models as MD
    from mmf_b200.registry import registry
    registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
    registry.register("textvqa_num_final_outputs", BM.ANS + BM.OCR_MAX)
    registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1, "UNK_IDX": 3}))
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c_captioner" if captioner else "m4c")).to(dev)
    sl = BM.sample_list(B, dev, torch.Generator().manual_seed(182))
    if captioner:                           # TextCaps: a 3-token prompt and 30 decoding steps
        g = torch.Generator().manual_seed(183)
        sl["text"] = sl["text"][:, :TEXTCAPS_TXT].contiguous()
        sl["text_len"] = torch.randint(1, TEXTCAPS_TXT + 1, (B,), generator=g).to(dev)
        sl["train_prev_inds"] = torch.randint(0, BM.ANS + BM.OCR_MAX, (B, TEXTCAPS_DEC), generator=g).to(dev)
        sl["targets"] = (torch.rand(B, TEXTCAPS_DEC, BM.ANS + BM.OCR_MAX, generator=g) < 0.001).float().to(dev)
        sl["train_loss_mask"] = (torch.rand(B, TEXTCAPS_DEC, generator=g) < 0.7).float().to(dev)
    sl["dataset_type"] = "val"
    return model, sl


def _vilt(B, dev):
    import torch
    import bench_vilt as BV
    from mmf_b200 import models as MD
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("vilt", overrides=BV.VQA)).to(dev)
    sl = BV.sample_list(B, "vqa2", dev, torch.Generator().manual_seed(384 + B))
    sl["dataset_type"] = "val"
    return model, sl


def _visual_bert(B, dev):
    import torch
    import bench
    wl = bench.VisualBertWL()
    torch.manual_seed(0)
    return wl.build(0.1).to(dev), bench.to_device(wl.host_batch(B, 17), dev)


WORKLOADS = {
    "m4c": ([128], lambda B, dev: _m4c(False, B, dev), "TextVQA shapes, 12 decoding steps"),
    "m4c_captioner": ([64, 128], lambda B, dev: _m4c(True, B, dev), "TextCaps shapes, 30 decoding steps"),
    "vilt": ([32, 256], _vilt, "vqa2/vit_b32_384, 40 tokens + 145 image positions"),
    "visual_bert": ([32, 166], _visual_bert, "BASELINE.json configs[1] trunk, 128 tokens + 100 regions"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", nargs="+", choices=sorted(WORKLOADS), default=list(WORKLOADS))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_eval needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200 import lib
    from mmf_b200.graphs import GraphedForward, _map_keep
    name, limit = card()

    for wl in args.only:
        batches, make, shape = WORKLOADS[wl]
        for B in batches:
            model, batch = make(B, dev)
            model.eval()

            def eager():
                with torch.no_grad():
                    return model(_map_keep(lambda t: t, batch))

            def peak(fn):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                out = fn()
                torch.cuda.synchronize()
                return out, torch.cuda.max_memory_allocated()

            key = "scores" if "scores" in eager() else "sequence_output"
            ref, eager_peak = peak(eager)
            ref = ref[key].clone()
            l0 = lib.launch_count()
            eager()
            torch.cuda.synchronize()
            launches = lib.launch_count() - l0
            torch.cuda.empty_cache()
            fwd = GraphedForward(model, batch, warmup=args.warmup)
            pool = _pool_bytes(fwd.graph)
            out, graphed_peak = peak(lambda: fwd(batch))
            same = bool(torch.equal(out[key], ref))
            times = {"eager": [], "graphed": []}
            for _ in range(3):
                times["eager"].append(timed(eager, args.steps, args.warmup))
                times["graphed"].append(timed(lambda: fwd(batch), args.steps, args.warmup))
            med = {k: sorted(v)[1] for k, v in times.items()}
            print(json.dumps({
                "metric": "eval forward (no_grad, scores + loss): eager vs GraphedForward", "unit": "ms/batch",
                "gpu": name, "power_limit_w": limit, "workload": wl, "shape": shape, "batch": B, "steps": args.steps,
                "warmup": args.warmup, "dtype": "bf16", "data": "synthetic",
                "ms_per_batch": times, "median_ms": med, "speedup": med["eager"] / med["graphed"],
                "peak_allocated_mib": {"eager": eager_peak / 2 ** 20, "graphed": graphed_peak / 2 ** 20},
                "graph_pool_mib": pool / 2 ** 20, "library_launches_per_eager_forward": launches,
                "replay_equals_eager": same}), flush=True)
            del fwd, out, model, batch, ref
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
