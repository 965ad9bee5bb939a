#!/usr/bin/env python
"""What the per-element epilogue operands cost the GEMMs of one BERT layer at the bench shapes (37848 tokens).

Every GEMM whose epilogue reads `aux` (residual, pre-activation or residual gradient) is timed twice, as the training
step runs it and with aux = None (and drop_mask = None for the dropout + residual epilogue).  Without aux the kernel
skips the operand reads (and for EPI_GELU_BWD the GELU' arithmetic), so the difference bounds what faster aux reads can
win.  The O-proj dgrad reads no aux and is timed as a control.  Cold L2 and CUDA events, as in tools/kbench.py.  Another
build of the library is timed in a process of its own:  MMFB_LIB=<path> python tools/bench_gemm_epilogue.py

    python tools/bench_gemm_epilogue.py [--iters 30] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """name, power limit and max SM clock of GPU 0, as nvidia-smi reports them"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=166)
    ap.add_argument("--seq", type=int, default=228)
    ap.add_argument("--hidden", type=int, default=768)
    ap.add_argument("--inter", type=int, default=3072)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from mmf_b200 import functional as F, lib
    if not torch.cuda.is_available():
        raise RuntimeError("bench_gemm_epilogue needs an H100")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    M, H, I = args.batch * args.seq, args.hidden, args.inter
    flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)

    def timeit(fn):
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
        return statistics.mean(ts), min(ts)

    bf = torch.bfloat16
    x = torch.randn(M, H, device=dev).to(bf)
    x3 = torch.randn(M, 3 * H, device=dev).to(bf)
    xi = torch.randn(M, I, device=dev).to(bf)
    w_qkv = (torch.randn(3 * H, H, device=dev) * 0.02).to(bf)
    w_o = (torch.randn(H, H, device=dev) * 0.02).to(bf)
    w_1 = (torch.randn(I, H, device=dev) * 0.02).to(bf)
    w_2 = (torch.randn(H, I, device=dev) * 0.02).to(bf)
    bh = torch.zeros(H, device=dev, dtype=bf)
    bits = F.dropout_bits((M,), H, 0.1, 1, 0, dev)
    oh, oi = torch.empty_like(x), torch.empty_like(xi)

    # (name, flops, fn(with_aux))
    cases = [
        ("O-proj fwd +bias+drop+resid", 2.0 * M * H * H,
         lambda w: F.gemm(x, w_o, epi=lib.EPI_BIAS_DROP_RESID, bias=bh, aux=x if w else None, drop_mask=bits if w else None,
                          drop_scale=1 / 0.9, out=oh)),
        ("FFN-down fwd +bias+drop+resid", 2.0 * M * H * I,
         lambda w: F.gemm(xi, w_2, epi=lib.EPI_BIAS_DROP_RESID, bias=bh, aux=x if w else None,
                          drop_mask=bits if w else None, drop_scale=1 / 0.9, out=oh)),
        ("FFN-down dgrad xGELU'(u)", 2.0 * M * H * I,
         lambda w: F.gemm(x, w_2, b_mn=True, epi=lib.EPI_GELU_BWD, aux=xi if w else None, out=oi)),
        ("FFN-up dgrad +resid-grad", 2.0 * M * H * I,
         lambda w: F.gemm(xi, w_1, b_mn=True, epi=lib.EPI_ADD_AUX, aux=x if w else None, out=oh)),
        ("QKV dgrad +resid-grad", 2.0 * M * H * 3 * H,
         lambda w: F.gemm(x3, w_qkv, b_mn=True, epi=lib.EPI_ADD_AUX, aux=x if w else None, out=oh)),
        ("O-proj dgrad (control, no aux)", 2.0 * M * H * H,
         lambda w: F.gemm(x, w_o, b_mn=True, epi=lib.EPI_BIAS, out=oh)),
    ]
    info = {"card": card(), "lib": lib.LIB_PATH, "M": M, "H": H, "I": I, "iters": args.iters}
    print("card: %s\nlib: %s   M=%d H=%d I=%d" % (info["card"], info["lib"], M, H, I))
    print("%-32s %10s %10s %8s %9s" % ("gemm", "aux us", "no-aux us", "gap", "TFLOP/s"))
    rows = []
    for name, flops, fn in cases:
        us_aux, min_aux = timeit(lambda: fn(True))
        us_no, min_no = timeit(lambda: fn(False))
        gap = (us_aux - us_no) / us_aux
        print("%-32s %10.1f %10.1f %7.1f%% %9.1f" % (name, us_aux, us_no, 100 * gap, flops / us_aux / 1e6))
        rows.append({"gemm": name, "us": us_aux, "us_min": min_aux, "us_no_aux": us_no, "us_no_aux_min": min_no,
                     "gap": gap, "tflops": flops / us_aux / 1e6})
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
