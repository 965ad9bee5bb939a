#!/usr/bin/env python
"""The registered M4C model at TextVQA shapes, on one GPU, and what the causal tail costs its attention.

    python tools/bench_m4c.py [--batch 128] [--steps 10] [--warmup 3] [--skip-padding]

Workload: the default m4c configuration (3-layer bert-base text BERT, 4-layer 768-wide MMT, dropout 0.1), 20 question
tokens + 100 objects (2048-wide features) + 50 OCR tokens + 12 decoding steps = 182 MMT positions, 5000 fixed answers +
50 OCR copies, bf16 compute, synthetic padded inputs resident in HBM.  Reported, one JSON line with the card's name and
power limit:
  train   - training step (forward, m4c_decoding_bce_with_mask, backward), three alternated repeats of `steps` steps:
            median ms, samples/s at the median, and the library's launches per step (lib.launch_count);
  decode  - the eval forward: greedy decoding over the 12 steps, ms per batch;
  attn    - the MMT's attention core alone at its shape (B x 12 heads x 182 x 182, d = 64, its key mask), forward and
            backward (with delta), causal_len = 12 and 0 alternated in one process: the tail's cost.
With --skip-padding it reports instead, for the training step and greedy decoding, the dense path against
set_skip_padding(model, causal=True) (the text BERT and the MMT run on their valid rows, the MMT with the packed causal
tail kernels), alternated three times in one process, on two batches: the seeded padded one above (its per-sample text,
object and OCR counts are printed) and one with nothing padded, where packing takes the dense path.  For each it gives the
rows per MMT call and the library's launches per training step of both modes.
CUDA events throughout.  It fails without a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

T_TXT, R_OBJ, O_OCR, D_DEC, ANS, OCR_MAX = 20, 100, 50, 12, 5000, 50


def sample_list(B, dev, g):
    import torch
    from mmf_b200.sample import SampleList

    def lens(n, lo):
        return torch.randint(lo, n + 1, (B,), generator=g)
    sl = SampleList(text=torch.randint(1, 30522, (B, T_TXT), generator=g), text_len=lens(T_TXT, 4),
                    image_feature_0=torch.randn(B, R_OBJ, 2048, generator=g).relu(),
                    obj_bbox_coordinates=torch.rand(B, R_OBJ, 4, generator=g), image_info_0={"max_features": lens(R_OBJ, 10)},
                    context_feature_0=torch.randn(B, O_OCR, 300, generator=g),
                    context_feature_1=torch.rand(B, O_OCR, 604, generator=g),
                    image_feature_1=torch.randn(B, O_OCR, 2048, generator=g).relu(),
                    order_vectors=torch.zeros(B, O_OCR, 50), ocr_bbox_coordinates=torch.rand(B, O_OCR, 4, generator=g),
                    context_info_0={"max_features": lens(O_OCR, 0)},
                    train_prev_inds=torch.randint(0, ANS + OCR_MAX, (B, D_DEC), generator=g),
                    targets=(torch.rand(B, D_DEC, ANS + OCR_MAX, generator=g) < 0.001).float(),
                    train_loss_mask=(torch.rand(B, D_DEC, generator=g) < 0.7).float(), dataset_name="textvqa",
                    dataset_type="train")
    return sl.to(dev)


def full_sample_list(B, dev, g):
    """sample_list with every question token, object and OCR slot valid"""
    import torch
    sl = sample_list(B, dev, g)
    sl["text_len"] = torch.full((B,), T_TXT, device=dev)
    sl["image_info_0"]["max_features"] = torch.full((B,), R_OBJ, device=dev)
    sl["context_info_0"]["max_features"] = torch.full((B,), O_OCR, device=dev)
    return sl


def skip_padding_times(model, batches, steps, warmup, timed):
    """training step and greedy decoding, dense and packed alternated three times per batch"""
    import torch
    from mmf_b200 import lib
    from mmf_b200.patch import set_skip_padding
    res = {}
    for name, sl in batches.items():
        counts = [sl["text_len"], sl["image_info_0"]["max_features"], sl["context_info_0"]["max_features"]]
        B = counts[0].numel()

        def train_step():
            model.zero_grad(set_to_none=True)
            sum(v.sum() for v in model(sl)["losses"].values()).backward()

        def decode():
            with torch.no_grad():
                model(sl)

        r = {"valid_counts": {"text": counts[0].tolist(), "obj": counts[1].tolist(), "ocr": counts[2].tolist()},
             "mmt_rows_per_call": {"dense": B * (T_TXT + R_OBJ + O_OCR + D_DEC),
                                   "packed": int(sum(c.sum() for c in counts)) + B * D_DEC}}
        for mode in ("dense", "packed"):
            r[mode] = {"train_ms": [], "decode_ms": []}
        for _ in range(3):
            for mode in ("dense", "packed"):
                set_skip_padding(model, mode == "packed", causal=True)
                model.train()
                r[mode]["train_ms"].append(timed(train_step, steps, warmup))
                model.eval()
                r[mode]["decode_ms"].append(timed(decode, steps, warmup))
        for mode in ("dense", "packed"):
            set_skip_padding(model, mode == "packed", causal=True)
            model.train()
            l0 = lib.launch_count()
            train_step()
            torch.cuda.synchronize()
            r[mode]["library_launches_per_step"] = lib.launch_count() - l0
            r[mode]["train_median_ms"] = sorted(r[mode]["train_ms"])[1]
            r[mode]["decode_median_ms"] = sorted(r[mode]["decode_ms"])[1]
        r["train_speedup"] = r["dense"]["train_median_ms"] / r["packed"]["train_median_ms"]
        r["decode_speedup"] = r["dense"]["decode_median_ms"] / r["packed"]["decode_median_ms"]
        res[name] = r
    set_skip_padding(model, False, causal=True)
    return res


def attention_times(B, dev, steps, warmup, timed):
    """fwd and bwd of the MMT attention core alone, causal_len 12 vs 0, alternated three times"""
    import torch
    from mmf_b200 import functional as F
    S, heads, d = T_TXT + R_OBJ + O_OCR + D_DEC, 12, 64
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = (torch.randn(B * S, 3 * heads * d, generator=g, device=dev) * 0.8).to(torch.bfloat16)
    q, k, v = qkv[:, :heads * d], qkv[:, heads * d:2 * heads * d], qkv[:, 2 * heads * d:]
    valid = torch.rand(B, S, generator=g, device=dev) < 0.7
    mask = torch.where(valid, 0.0, -10000.0).float().contiguous()
    dctx = torch.randn(B * S, heads * d, generator=g, device=dev).to(torch.bfloat16)
    out = {}
    for T in (D_DEC, 0):
        out[T] = {"fwd": [], "bwd": []}
    for _ in range(3):
        for T in (D_DEC, 0):
            ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, S, S, mask=mask, save_lo=True, causal_len=T)
            out[T]["fwd"].append(timed(lambda: F.attention_fwd(q, k, v, B, heads, S, S, mask=mask, save_lo=True,
                                                               causal_len=T), steps, warmup) * 1e3)
            out[T]["bwd"].append(timed(lambda: F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, S, S, mask=mask,
                                                               ctx_lo=lo, causal_len=T), steps, warmup) * 1e3)
    return {("causal_len_%d" % T): {kind: {"us": v, "median_us": sorted(v)[1]} for kind, v in r.items()}
            for T, r in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-padding", action="store_true",
                    help="dense against set_skip_padding(model, causal=True), on a padded and an unpadded batch")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_m4c needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200 import lib, models as MD
    from mmf_b200.registry import registry
    name, limit = card()
    registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
    registry.register("textvqa_num_final_outputs", ANS + OCR_MAX)
    registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1}))
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).to(dev)
    B = args.batch
    sl = sample_list(B, dev, torch.Generator().manual_seed(182))
    if args.skip_padding:
        batches = {"padded": sl, "unpadded": full_sample_list(B, dev, torch.Generator().manual_seed(182))}
        print(json.dumps({
            "metric": "M4C at TextVQA shapes (registered model): dense vs skip-padding with the packed causal tail",
            "gpu": name, "power_limit_w": limit, "batch": B, "steps": args.steps, "warmup": max(3, args.warmup),
            "dtype": "bf16", "data": "synthetic", "seed": 182,
            "shape": {"txt": T_TXT, "obj": R_OBJ, "ocr": O_OCR, "dec": D_DEC, "answers": ANS, "ocr_copies": OCR_MAX},
            "runs": skip_padding_times(model, batches, args.steps, args.warmup, timed)}))
        return

    def train_step():
        model.zero_grad(set_to_none=True)
        sum(v.sum() for v in model(sl)["losses"].values()).backward()

    def decode():
        with torch.no_grad():
            model(sl)

    train, dec = [], []
    for _ in range(3):
        model.train()
        train.append(timed(train_step, args.steps, args.warmup))
        model.eval()
        dec.append(timed(decode, args.steps, args.warmup))
    model.train()
    l0 = lib.launch_count()
    train_step()
    torch.cuda.synchronize()
    launches = lib.launch_count() - l0
    med = sorted(train)[1]
    print(json.dumps({
        "metric": "M4C at TextVQA shapes (registered model): training step, greedy decoding, MMT attention causal tail",
        "gpu": name, "power_limit_w": limit, "batch": B, "steps": args.steps, "warmup": max(3, args.warmup),
        "dtype": "bf16", "data": "synthetic",
        "shape": {"txt": T_TXT, "obj": R_OBJ, "ocr": O_OCR, "dec": D_DEC, "answers": ANS, "ocr_copies": OCR_MAX},
        "train": {"ms_per_step": train, "median_ms": med, "samples_per_s_at_median": B / (med / 1e3),
                  "library_launches_per_step": launches},
        "decode": {"ms_per_batch": dec, "median_ms": sorted(dec)[1]},
        "attn": attention_times(B, dev, max(args.steps, 20), args.warmup, timed)}))


if __name__ == "__main__":
    main()
