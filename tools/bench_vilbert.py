#!/usr/bin/env python
"""ViLBERT two-stream fusion block (BASELINE.json configs[2]) forward + backward samples/s, 1..8 GPUs.

    python tools/bench_vilbert.py [--batch 512] [--steps 10] [--warmup 3]
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 tools/bench_vilbert.py --gpus 8

Not the driver's bench (that is bench.py on configs[1]); this reports the second model family the north star names,
with the same timing rules: CUDA events, max over ranks, W >= 3 warm-up steps, inputs resident in HBM, one JSON line.
Workload: mmf/configs/models/vilbert/defaults.yaml - text 12L/768/12h/3072, image 6L/1024/8h/1024, 6 connection layers
1024/8h (d = 128), 36 tokens + 36 regions x 2048 (+ 5 location features), dropout 0.1, bf16 compute, synthetic inputs.
Algorithmic FLOPs per sample (SURVEY.md 8d): 15.24 GF forward, 45.7 GF forward + backward.
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T_TOK, R_REG, FEAT, VOCAB = 36, 36, 2048, 30522


def vilbert_config(p):
    # mmf/configs/models/vilbert/defaults.yaml:11-49
    return types.SimpleNamespace(
        hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12, vocab_size=VOCAB,
        max_position_embeddings=512, type_vocab_size=2, hidden_dropout_prob=p, attention_probs_dropout_prob=p,
        v_feature_size=FEAT, v_target_size=1601, v_hidden_size=1024, v_num_hidden_layers=6, v_num_attention_heads=8,
        v_intermediate_size=1024, bi_hidden_size=1024, bi_num_attention_heads=8, bi_intermediate_size=1024,
        v_attention_probs_dropout_prob=p, v_hidden_dropout_prob=p, v_biattention_id=[0, 1, 2, 3, 4, 5],
        t_biattention_id=[6, 7, 8, 9, 10, 11], layer_norm_eps=1e-12, hidden_act="gelu", v_hidden_act="gelu",
        initializer_range=0.02, fast_mode=False, with_coattention=True, dynamic_attention=False,
        fixed_t_layer=0, fixed_v_layer=0, in_batch_pairs=False)


def fwd_flops_per_sample():
    def layer(S, H, I, Skv=None, Hkv=None):
        Skv = S if Skv is None else Skv
        return 8 * S * H * H + 4 * S * Skv * H + 4 * S * H * I
    t = 12 * layer(T_TOK, 768, 3072)
    v = 6 * layer(R_REG, 1024, 1024)
    # connection layer: 6 projections into the 1024-wide co-attention space, 2 cross attentions, 2 output projections
    # back to each stream, then one FFN per stream (vilbert.py:388-556)
    bi = 2 * T_TOK * 768 * 1024 * 3 + 2 * R_REG * 1024 * 1024 * 3 + 2 * (4 * T_TOK * R_REG * 1024) \
        + 2 * T_TOK * 1024 * 768 + 2 * R_REG * 1024 * 1024 + 4 * T_TOK * 768 * 3072 + 4 * R_REG * 1024 * 1024
    img_proj = 2 * R_REG * FEAT * 1024 + 2 * R_REG * 5 * 1024
    return t + v + 6 * bi + img_proj


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=512, help="samples per GPU")
    ap.add_argument("--dropout", type=float, default=0.1)
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench_vilbert needs an H100: the fusion path has no CPU fallback")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl")
    from mmf_b200 import lib
    from mmf_b200.vilbert import B200ViLBERTBase
    torch.manual_seed(0)
    model = B200ViLBERTBase(vilbert_config(args.dropout)).to(dev).train()
    ddp = None
    if world > 1:
        from mmf_b200.ddp import B200DataParallel
        ddp = B200DataParallel(model)
    B = args.batch
    g = torch.Generator().manual_seed(1234 + rank)
    ids = torch.randint(0, VOCAB, (B, T_TOK), generator=g).to(dev)
    lens = torch.randint(T_TOK // 2, T_TOK + 1, (B,), generator=g)
    tmask = (torch.arange(T_TOK)[None, :] < lens[:, None]).long().to(dev)
    feats = torch.randn(B, R_REG, FEAT, generator=g).abs().to(dev)
    loc = torch.rand(B, R_REG, 5, generator=g).to(dev)
    nreg = torch.randint(R_REG // 2, R_REG + 1, (B,), generator=g)
    imask = (torch.arange(R_REG)[None, :] < nreg[:, None]).long().to(dev)      # vilbert.py:1432-1440
    wt = torch.randn(B, T_TOK, 768, device=dev)
    wv = torch.randn(B, R_REG, 1024, device=dev)
    net = ddp if ddp is not None else model

    def step():
        model.zero_grad(set_to_none=True)
        t_out, v_out, _ = net(ids, feats, loc, attention_mask=tmask, image_attention_mask=imask)
        ((t_out * wt).sum() + (v_out * wv).sum()).backward()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(max(3, args.warmup)):
        step()
    barrier()
    l0 = lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_step = ms.item() / args.steps
    if rank == 0:
        flops = 3 * fwd_flops_per_sample()
        value = B * world / (ms_step / 1e3)
        print(json.dumps({
            "metric": "multimodal-fusion samples/sec (fwd+bwd)", "value": value, "unit": "samples/s", "n_gpus": world,
            "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms_step, "higher_is_better": True,
            "scaling": "weak", "dtype": "bf16", "data": "synthetic",
            "config": {"workload": "ViLBERT two-stream 12t+6v+6c, 36 regions x 2048 + 36 tokens (BASELINE.json configs[2])",
                       "batch_per_gpu": B, "dropout": args.dropout, "inputs": "resident in HBM, larger than L2"},
            "gflop_per_sample": flops / 1e9, "tflops_algorithmic": value * flops / 1e12,
            "gpu_launches": (lib.launch_count() - l0)}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
