"""Cost of returning attention probabilities (output_attentions) on the H100.

    python tools/bench_attention_probs.py [--batch 166] [--seq 228] [--iters 20] [--warmup 5]

Reports, at the VisualBERT bench shape (12 layers / 768 / 12 heads, B = 166, S = 228, eval under no_grad):
  * the encoder forward time with output_attentions off and on;
  * the probs kernel alone (mmfb_attention_probs, fp32 and bf16 output): time per call and the achieved write
    bandwidth, B * heads * S^2 * element size / time.
Times are CUDA-event medians over --iters runs after --warmup runs.  Prints one JSON line.  Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=166)
    ap.add_argument("--seq", type=int, default=228)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from mmf_b200 import functional as F
    from mmf_b200.modules import B200BertEncoder
    B, S, H, heads, L = args.batch, args.seq, 768, 12, 12
    cfg = types.SimpleNamespace(hidden_size=H, num_attention_heads=heads, intermediate_size=3072, num_hidden_layers=L,
                                hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, layer_norm_eps=1e-12,
                                hidden_act="gelu", initializer_range=0.02)
    torch.manual_seed(0)
    enc = B200BertEncoder(cfg).cuda().eval()
    x = torch.randn(B, S, H, device="cuda")
    lens = torch.randint(S // 2, S + 1, (B,), device="cuda")
    add = ((torch.arange(S, device="cuda")[None] >= lens[:, None]).float() * -10000.0)
    res = {"gpu": torch.cuda.get_device_name(), "B": B, "S": S, "heads": heads, "layers": L}
    try:                                         # the card's power limit and max SM clock are part of every number here
        import subprocess
        res["power_limit_and_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["power_limit_and_max_sm_clock"] = "unknown"
    with torch.no_grad():
        res["encoder_fwd_ms_flag_off"] = _median_ms(lambda: enc(x, add), args.iters, args.warmup)
        res["encoder_fwd_ms_flag_on"] = _median_ms(lambda: enc(x, add, output_attentions=True), args.iters, args.warmup)
    res["encoder_fwd_overhead_pct"] = 100.0 * (res["encoder_fwd_ms_flag_on"] / res["encoder_fwd_ms_flag_off"] - 1.0)
    # the kernel alone, on one layer's q / k slices of a fused projection buffer
    W = H
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(B * S, 3 * W, generator=g, device="cuda").to(torch.bfloat16)
    q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    mask = add.contiguous()
    _, lse2 = F.attention_fwd(q, k, v, B, heads, S, S, mask)
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        out = torch.empty(B, heads, S, S, dtype=dt, device="cuda")
        ms = _median_ms(lambda: F.attention_probs(q, k, lse2, B, heads, S, S, mask, dtype=dt, out=out), args.iters * 5,
                        args.warmup)
        res["probs_kernel_ms_" + name] = ms
        res["probs_write_GBps_" + name] = out.numel() * out.element_size() / (ms * 1e-3) / 1e9
    fwd_ms = _median_ms(lambda: F.attention_fwd(q, k, v, B, heads, S, S, mask), args.iters * 5, args.warmup)
    res["attention_fwd_kernel_ms"] = fwd_ms
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
