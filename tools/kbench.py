#!/usr/bin/env python
"""Kernel-level timings at the bench shapes (BASELINE.json configs[1], batch 166): every kernel of one fusion layer timed
ALONE with CUDA events on the launching stream, L2 flushed between launches (a 160 MB buffer is zeroed), mean of N after
warm-up.  Another build of the library is timed in a process of its own:  MMFB_LIB=<path> python tools/kbench.py --only ln

    python tools/kbench.py [--batch 166] [--iters 20] [--only attn,ln,gemm,rows] [--json out.json]

Algorithmic FLOPs / bytes per launch are printed with each kernel so the roofline fraction is on the same line (against
the H100 SXM data-sheet peaks, 989 TFLOP/s dense bf16 and 3350 GB/s).
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=166)
    ap.add_argument("--seq", type=int, default=228)
    ap.add_argument("--hidden", type=int, default=768)
    ap.add_argument("--heads", type=int, default=12)
    ap.add_argument("--inter", type=int, default=3072)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", default="attn,ln,gemm,rows")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from mmf_b200 import functional as F, lib
    from mmf_b200.engine import best_splits
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    B, S, H, heads, I = args.batch, args.seq, args.hidden, args.heads, args.inter
    M = B * S
    # H100 SXM data-sheet peaks (dense bf16, HBM3), as in bench.py: the fractions printed are of these, not of measured peaks
    PF, HBM = 989.0, 3350.0
    flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)
    rows = []

    def timeit(name, fn, flops=None, nbytes=None):
        try:
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ts = []
            for _ in range(args.iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
        except Exception as e:      # a kernel that fails must not end the whole run
            print("%-58s FAILED: %s" % (name, str(e)[:120]))
            rows.append({"kernel": name, "failed": str(e)[:200]})
            return None
        us = statistics.mean(ts)
        extra = ""
        row = {"kernel": name, "us": us, "us_min": min(ts)}
        if flops:
            row["tflops"] = flops / us / 1e6
            row["frac_tensor"] = row["tflops"] / PF
            extra += "  %7.1f TFLOP/s (%.3f of data-sheet %.0f)" % (row["tflops"], row["frac_tensor"], PF)
        if nbytes:
            row["gbs"] = nbytes / us / 1e3
            row["frac_hbm"] = row["gbs"] / HBM
            extra += "  %7.1f GB/s (%.3f of data-sheet %.0f)" % (row["gbs"], row["frac_hbm"], HBM)
        print("%-58s %8.1f us (min %7.1f)%s" % (name, us, min(ts), extra))
        rows.append(row)
        return us

    bf = torch.bfloat16
    only = set(args.only.split(","))
    print("lib: %s   shapes: B=%d S=%d H=%d heads=%d I=%d (M=%d)" % (lib.LIB_PATH, B, S, H, heads, I, M))

    def attn_rows(tag, B, S, heads, d):
        """attention forward and backward of B samples of S tokens (self-attention shapes: Sq = Skv = S), padding mask
        and dropout keep bits as in training"""
        H, M = heads * d, B * S
        qkv = torch.randn(M, 3 * H, device=dev).to(bf)
        q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
        lens = torch.randint(S // 2, S + 1, (B,), device=dev)
        mask = ((torch.arange(S, device=dev)[None] >= lens[:, None]).float() * -10000.0).contiguous()
        bits = F.dropout_bits((B, heads, S), S, 0.1, 7, 0, dev)
        dctx = torch.randn(M, H, device=dev).to(bf)
        f_fwd, f_bwd = 4.0 * B * heads * S * S * d, 10.0 * B * heads * S * S * d
        b_fwd = M * 3 * H * 2 + M * H * 2 + M * H * 4 + bits.numel() * 4
        b_bwd = M * 3 * H * 2 * 2 + M * H * 2 + bits.numel() * 4
        timeit("attention_fwd" + tag, lambda: F.attention_fwd(q, k, v, B, heads, S, S, mask, bits, 1 / 0.9, save_lo=True),
               f_fwd, b_fwd)
        ctx, lse2, c32 = F.attention_fwd(q, k, v, B, heads, S, S, mask, bits, 1 / 0.9, save_lo=True)
        dq = torch.empty_like(qkv)
        timeit("attention_bwd (+delta)" + tag,
               lambda: F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, S, S, mask, bits, 1 / 0.9, dq=dq[:, :H],
                                       dk=dq[:, H:2 * H], dv=dq[:, 2 * H:], ctx_lo=c32), f_bwd, b_bwd)
        return bits

    if "attn" in only:
        bits = attn_rows("", B, S, heads, H // heads)
        timeit("dropout_bits attention [B,h,S,S]", lambda: F.dropout_bits((B, heads, S), S, 0.1, 7, 0, dev), None, bits.numel() * 4)
        # the other head size and the tile edges: one 36-row tile of d = 128 (32-row query blocks in the dk/dv kernel),
        # and S = 120 = 64 + 56 at d = 64
        attn_rows("  ViLBERT co-attention d=128 h=8 S=36 B=512", 512, 36, 8, 128)
        attn_rows("  UNITER-large d=64 h=16 S=120 B=256", 256, 120, 16, 64)
        del bits

    if "ln" in only:
        dx = torch.randn(M, H, device=dev).to(bf)
        y = torch.randn(M, H, device=dev).to(bf)
        g = torch.ones(H, device=dev, dtype=bf)
        _, mean, rstd = F.layernorm_fwd(y, g, torch.zeros_like(g))
        bits = F.dropout_bits((M,), H, 0.1, 1, 0, dev)
        dg, db_, dbias = (torch.zeros(H, device=dev) for _ in range(3))
        nb = M * (8.0 * H + H / 8.0 + 8.0)
        timeit("layernorm_bwd +dropout +dgamma/dbeta/dbias",
               lambda: F.layernorm_bwd(dx, y, mean, rstd, g, dg, db_, dbias=dbias, drop_mask=bits, drop_scale=1 / 0.9), None, nb)
        timeit("layernorm_fwd", lambda: F.layernorm_fwd(y, g, torch.zeros_like(g)), None, M * (4.0 * H + 8))
        big = torch.randn(M, 3 * H, device=dev).to(bf)
        acc = torch.zeros(3 * H, device=dev)
        timeit("colsum [M,2304]", lambda: F.colsum(big, acc), None, M * 3 * H * 2.0)
        timeit("dropout_bits hidden [M,H]", lambda: F.dropout_bits((M,), H, 0.1, 1, 0, dev), None, M * H / 8.0)
        del big

    if "gemm" in only:
        x = torch.randn(M, H, device=dev).to(bf)
        x3 = torch.randn(M, 3 * H, device=dev).to(bf)
        xi = torch.randn(M, I, device=dev).to(bf)
        w_qkv = (torch.randn(3 * H, H, device=dev) * 0.02).to(bf)
        w_o = (torch.randn(H, H, device=dev) * 0.02).to(bf)
        w_1 = (torch.randn(I, H, device=dev) * 0.02).to(bf)
        w_2 = (torch.randn(H, I, device=dev) * 0.02).to(bf)
        b3, b1, bh = (torch.zeros(n, device=dev, dtype=bf) for n in (3 * H, I, H))
        bits = F.dropout_bits((M,), H, 0.1, 1, 0, dev)
        o3, oh, oi, oi2 = torch.empty_like(x3), torch.empty_like(x), torch.empty_like(xi), torch.empty_like(xi)
        timeit("gemm QKV fwd        [M,768]x[2304,768]^T +bias", lambda: F.gemm(x, w_qkv, epi=lib.EPI_BIAS, bias=b3, out=o3), 2.0 * M * H * 3 * H)
        timeit("gemm O-proj fwd     [M,768]x[768,768]^T +bias+drop+resid", lambda: F.gemm(x, w_o, epi=lib.EPI_BIAS_DROP_RESID, bias=bh, aux=x, drop_mask=bits, drop_scale=1 / 0.9, out=oh), 2.0 * M * H * H)
        timeit("gemm FFN-up fwd     [M,768]x[3072,768]^T +bias+GELU (2 outputs)", lambda: F.gemm(x, w_1, epi=lib.EPI_BIAS_GELU, bias=b1, out=oi, out2=oi2), 2.0 * M * H * I)
        timeit("gemm FFN-down fwd   [M,3072]x[768,3072]^T +bias+drop+resid", lambda: F.gemm(xi, w_2, epi=lib.EPI_BIAS_DROP_RESID, bias=bh, aux=x, drop_mask=bits, drop_scale=1 / 0.9, out=oh), 2.0 * M * H * I)
        timeit("gemm FFN-down dgrad [M,768]x[768,3072] xGELU'(u)", lambda: F.gemm(x, w_2, b_mn=True, epi=lib.EPI_GELU_BWD, aux=xi, out=oi), 2.0 * M * H * I)
        timeit("gemm FFN-up dgrad   [M,3072]x[3072,768] +resid-grad", lambda: F.gemm(xi, w_1, b_mn=True, epi=lib.EPI_ADD_AUX, aux=x, out=oh), 2.0 * M * H * I)
        timeit("gemm O-proj dgrad   [M,768]x[768,768]", lambda: F.gemm(x, w_o, b_mn=True, epi=lib.EPI_BIAS, out=oh), 2.0 * M * H * H)
        timeit("gemm QKV dgrad      [M,2304]x[2304,768] +resid-grad", lambda: F.gemm(x3, w_qkv, b_mn=True, epi=lib.EPI_ADD_AUX, aux=x, out=oh), 2.0 * M * H * 3 * H)
        for nm, dyv, xv, n_out, k_in in (("QKV", x3, x, 3 * H, H), ("O-proj", x, x, H, H), ("FFN-up", xi, x, I, H), ("FFN-down", x, xi, H, I)):
            gw = torch.zeros(n_out, k_in, device=dev)
            sp = best_splits(n_out, k_in, M)
            timeit("gemm wgrad %-8s [%d,%d] += dY^T X (split-K %d, fp32 red)" % (nm, n_out, k_in, sp),
                   lambda: F.gemm(dyv, xv, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=gw, splits=sp), 2.0 * M * n_out * k_in)
        del x3, xi, o3, oi, oi2

    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"lib": lib.LIB_PATH, "shapes": {"B": B, "S": S, "H": H, "heads": heads, "I": I}, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
