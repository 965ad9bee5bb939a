#!/usr/bin/env python
"""The registered ViLT model's training step (forward + backward), on one GPU.

    python tools/bench_vilt.py [--vqa-batches 32 256] [--pretrain-batches 64 256] [--steps 10] [--warmup 3]

Workloads, at the shapes of the reference's configurations (projects/vilt/configs): bert-base text embeddings, ViT-B/32
trunk (12 layers of 768/12h/3072) over 384 x 384 images, 40 tokens + 145 image positions, dropout as configured (0.1 in
the embeddings and the trunk's hidden states), bf16 compute, synthetic inputs resident in HBM, text padded (per-sample
lengths between 4 and 40):
  vqa        vqa2/vit_b32_384: heads.vqa2 = mlp with 3129 answers, logit_bce.  Each batch is timed eagerly and as a
             GraphedStep replay, alternating, three times each.  B = 32 is the per-GPU share of the configuration's 256 on
             8 GPUs;
  pretrain   masked_coco/pretrain: mlm_multi (~15 % of the valid tokens labelled) + itm, two trunk passes per step; eager
             only (the masked-LM head gathers a data-dependent number of rows, so the step cannot be captured).
CUDA events.  One JSON line per case, with the card's name and power limit read in the same run and the library's
launches per step (lib.launch_count(); a graph replay launches nothing from the host).  It fails without a GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

T, IMG, VOCAB, NUM_LABELS = 40, 384, 30522, 3129

# model_config.vilt of projects/vilt/configs/vqa2/vit_b32_384.yaml (with vqa2/defaults.yaml) and masked_coco/pretrain.yaml,
# over the model's default YAML; `tasks` is the trainer's dataset list
_IMAGE = dict(pretrained_model_name="google/vit-base-patch32-384", gradient_checkpointing=False, hidden_dropout_prob=0.1,
              add_pooling_layer=False, do_patch_embeddings=False, image_size=[IMG, IMG])
VQA = dict(tasks="vqa2", heads=dict(vqa2=[dict(type="mlp", num_layers=1, loss="vqa2_mlp", in_dim=768, hidden_size=1536,
                                               num_labels=NUM_LABELS, pooler_name="bert_pooler")]),
           losses=dict(vqa2_mlp="logit_bce"), image_encoder=dict(params=dict(_IMAGE, random_init=False)),
           text_embeddings=dict(max_position_embeddings=512, random_init=False))
PRETRAIN = dict(tasks="masked_coco", heads=dict(masked_coco=[
    dict(type="mlm_multi", hidden_size=768, vocab_size=VOCAB), dict(type="itm", hidden_size=768, label_key="is_correct")]),
    image_encoder=dict(params=dict(_IMAGE, random_init=True)), text_embeddings=dict(max_position_embeddings=40))


def sample_list(B, dataset, dev, g):
    import torch
    from mmf_b200.sample import SampleList
    lens = torch.randint(4, T + 1, (B,), generator=g)
    mask = (torch.arange(T)[None] < lens[:, None]).long()
    ids = torch.randint(1, VOCAB, (B, T), generator=g)
    sl = SampleList(input_ids=ids, segment_ids=torch.zeros(B, T, dtype=torch.long), input_mask=mask,
                    image=torch.randn(B, 3, IMG, IMG, generator=g), dataset_name=dataset, dataset_type="train")
    if dataset == "vqa2":
        sl["targets"] = (torch.rand(B, NUM_LABELS, generator=g) < 0.002).float()
    else:
        labels = torch.full((B, T), -1, dtype=torch.long)
        pick = (torch.rand(B, T, generator=g) < 0.15) & (mask == 1)
        pick[:, 1] = True
        labels[pick] = ids[pick]
        sl.update(input_ids_masked=torch.where(pick, torch.full_like(ids, 103), ids), lm_label_ids=labels,
                  is_correct=torch.randint(0, 2, (B,), generator=g))
    return sl.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vqa-batches", type=int, nargs="+", default=[32, 256])
    ap.add_argument("--pretrain-batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_vilt needs an H100: the fusion path has no CPU fallback")
    dev = torch.device("cuda", 0)
    from bench_lxmert import card, timed
    from mmf_b200 import lib, models as MD
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.sample import SampleList
    torch.manual_seed(0)
    name, limit = card()
    head = {"metric": "ViLT training step (fwd+bwd, registered model)", "unit": "ms/step", "gpu": name,
            "power_limit_w": limit, "steps": args.steps, "warmup": args.warmup, "dtype": "bf16", "data": "synthetic",
            "tokens": T, "image_positions": 145, "image_size": IMG}

    def launches(fn):
        l0 = lib.launch_count()
        fn()
        torch.cuda.synchronize()
        return lib.launch_count() - l0

    def row(**kw):
        ms = kw.pop("ms")
        median = sorted(ms)[len(ms) // 2]
        print(json.dumps(dict(head, **kw, ms_per_step=ms, median_ms=median, samples_per_s=kw["batch"] / (median / 1e3))),
              flush=True)

    model = MD.build_model(MD.load_model_config("vilt", overrides=VQA)).to(dev).train()
    for B in args.vqa_batches:
        sl = sample_list(B, "vqa2", dev, torch.Generator().manual_seed(384 + B))
        batch = {k: v for k, v in sl.items() if torch.is_tensor(v)}

        def loss_of(b):
            out = model(SampleList(dict(b), dataset_name="vqa2", dataset_type="train"))
            return sum(v.sum() for v in out["losses"].values())

        def eager():
            model.zero_grad(set_to_none=True)
            loss_of(batch).backward()

        n_eager = launches(eager)
        model.zero_grad(set_to_none=True)
        graphed = GraphedStep(model, loss_of, batch)
        n_graph = launches(graphed)
        times = {"eager": [], "graphed": []}
        for _ in range(3):
            times["eager"].append(timed(eager, args.steps, args.warmup))
            times["graphed"].append(timed(graphed, args.steps, args.warmup))
        for mode, n in (("eager", n_eager), ("graphed", n_graph)):
            row(workload="vqa2/vit_b32_384", mode=mode, batch=B, ms=times[mode], library_launches_per_step=n)
        del graphed
    del model
    torch.cuda.empty_cache()

    model = MD.build_model(MD.load_model_config("vilt", overrides=PRETRAIN)).to(dev).train()
    for B in args.pretrain_batches:
        sl = sample_list(B, "masked_coco", dev, torch.Generator().manual_seed(145 + B))

        def step():
            model.zero_grad(set_to_none=True)
            sum(v.sum() for v in model(SampleList(sl))["losses"].values()).backward()

        n = launches(step)
        ms = [timed(step, args.steps, args.warmup) for _ in range(3)]
        row(workload="masked_coco/pretrain", mode="eager", batch=B, ms=ms, library_launches_per_step=n)


if __name__ == "__main__":
    main()
