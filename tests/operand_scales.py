"""Operand generators for the large- and degenerate-scale kernel checks (a plain module, imported by
test_operand_scales_gpu.py, which runs the kernels on them, and test_operand_scales_cpu.py, which checks in fp64 that each
generator produces the regime it claims).

The edge tests draw q, k from N(0, 0.8^2) and LayerNorm rows from N(0.5, 2^2): every softmax row is close to uniform and
every row variance is about 4, so the error terms that grow with the operand (|Z| in the score error, the row mean, the
eps of the LayerNorm) never dominate a bound.  The inputs here are the regimes of trained models:

  attention (q, k, v [S, heads * d] bf16 for one sample; every head gets the same construction)
    peaked    q, k ~ N(0, 20): scores q.k / sqrt(d) of std 20 (natural units), rows spanning more than 60 log2 units
    planted   one key per head `gap` log2 units above every other score of every query row, at a chosen key
    tie       two keys with identical rows (one in the first 64-key block, one in the last) share the row max, the rest
              lie >= TIE_GAP log2 units below: each of the two p is exactly 1/2 in fp32
    delta     planted with a gap of DELTA_GAP: p of the planted key is close to 1; dctx = that key's v, so the backward's
              dP - delta cancels

  LayerNorm rows (bf16 [M, H])
    offset    c + N(0, 1) per row, c in {16, 64}: the mean dominates the spread
    outlier   N(0, 1) with 2-6 columns of magnitude 50-200
    constant  every element of a row equal (per-row constants, zero included): var = 0, rstd = 1 / sqrt(eps)
    near      +-a around an offset 0 or 4a, exactly balanced, scaled by 2^{-1,0,1} per row, with a = 2^round(log2 sqrt(eps)):
              row variances within [eps / 10, 10 eps], every value exact in bf16
"""
import math

import torch

LOG2E = 1.0 / math.log(2.0)
QK_STD = math.sqrt(20.0)        # q, k ~ N(0, 20): score std = 20 natural units (29 log2 units)
BASE = 0.8                      # the non-planted part of q / k of the planted cases: the edge tests' distribution
LEAD = 8.0                      # coordinate 0 of every q head: the planted key's lever
ONEHOT_GAP = 200.0              # > 150 log2 units: every other p flushes to exactly 0 in fp32
TIE_GAP = 200.0
DELTA_GAP = 12.0


def _normal(shape, std, g, device):
    return torch.randn(*shape, generator=g, device=device) * std


def block_of(S, where, g):
    """a key index in the first or the last 64-key block of S keys"""
    lo, hi = (0, min(S, 64)) if where == "first" else (64 * ((S - 1) // 64), S)
    return int(torch.randint(lo, hi, (1,), generator=g).item())


def _planted_lever(gap, d):
    """coordinate 0 of the planted key: LEAD * K / sqrt(d) puts it `gap` log2 units (+ 8 natural units of margin for the
    N(0, 0.8^2) part of every score) above the others; rounded to bf16"""
    K = (gap / LOG2E + 8.0) * math.sqrt(d) / LEAD
    return float(torch.tensor(K).to(torch.bfloat16))


def attention_sample(kind, Sq, Skv, heads, d, g, device="cpu", gap=None, where="last"):
    """q [Sq, W], k / v [Skv, W] bf16 (W = heads * d) and the planted key indices (None for peaked; two for tie)"""
    W = heads * d
    cpu = torch.Generator().manual_seed(int(torch.randint(0, 2 ** 31, (1,), generator=g, device=g.device).item()))
    v = _normal((Skv, W), 1.0, g, device)
    if kind == "peaked":
        q, k = _normal((Sq, W), QK_STD, g, device), _normal((Skv, W), QK_STD, g, device)
        return q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16), None
    if kind == "tie":
        gap, where = TIE_GAP, "last"
    elif kind == "onehot":
        gap = ONEHOT_GAP
    elif kind == "delta":
        gap = DELTA_GAP
    q = _normal((Sq, W), BASE, g, device).reshape(Sq, heads, d)
    k = _normal((Skv, W), BASE, g, device).reshape(Skv, heads, d)
    q[:, :, 0] = LEAD
    k[:, :, 0] = 0.0
    j = block_of(Skv, where, cpu)
    k[j, :, 0] = _planted_lever(gap, d)
    keys = [j]
    if kind == "tie":
        j0 = block_of(Skv, "first", cpu)
        if j0 == j:                      # Skv <= 64: one block; take another key of it
            j0 = (j + 1) % Skv
        if j0 != j:
            k[j0] = k[j]
            keys = [j0, j]
    return (q.reshape(Sq, W).to(torch.bfloat16), k.reshape(Skv, W).to(torch.bfloat16), v.to(torch.bfloat16),
            keys)


def dctx_for(kind, q_rows, v, keys, g, device="cpu"):
    """dctx [q_rows, W] bf16: the planted key's v on every row for `delta` (dP - delta cancels), else N(0, 1)"""
    if kind == "delta":
        return v[keys[0]].expand(q_rows, -1).contiguous()
    return _normal((q_rows, v.shape[1]), 1.0, g, device).to(torch.bfloat16)


def scores_log2(q, k, heads):
    """fp64 log2-domain scores [heads, Sq, Skv] of one sample (no mask)"""
    d = q.shape[1] // heads
    Q = q.double().reshape(-1, heads, d).permute(1, 0, 2)
    K = k.double().reshape(-1, heads, d).permute(1, 0, 2)
    return (Q @ K.transpose(-1, -2)) * (LOG2E / math.sqrt(d))


# ----------------------------------------------------------------------------------------------------------------------
# LayerNorm rows
# ----------------------------------------------------------------------------------------------------------------------
def ln_rows(kind, M, H, g, device="cpu", c=None, eps=None):
    if kind == "offset":
        return (c + _normal((M, H), 1.0, g, device)).to(torch.bfloat16)
    if kind == "outlier":
        y = _normal((M, H), 1.0, g, device)
        for r in range(M):
            n = int(torch.randint(2, 7, (1,), generator=g, device=device).item())
            cols = torch.randperm(H, generator=g, device=device)[:n]
            mag = 50.0 + 150.0 * torch.rand(n, generator=g, device=device)
            sign = torch.where(torch.rand(n, generator=g, device=device) < 0.5, -1.0, 1.0)
            y[r, cols] = mag * sign
        return y.to(torch.bfloat16)
    if kind == "constant":
        c = (_normal((M, 1), 8.0, g, device)).to(torch.bfloat16).float()
        c[0] = 0.0
        return c.expand(M, H).to(torch.bfloat16).contiguous()
    if kind == "near":
        a = near_unit(eps)
        s = torch.ones(M, H, device=device)
        s[:, H // 2:] = -1.0
        perm = torch.argsort(torch.rand(M, H, generator=g, device=device), dim=1)
        s = torch.gather(s, 1, perm)
        f = 2.0 ** torch.randint(-1, 2, (M, 1), generator=g, device=device).float()
        off = torch.where(torch.arange(M, device=device)[:, None] % 2 == 0, 0.0, 4.0)
        return (a * f * (s + off)).to(torch.bfloat16)
    raise ValueError(kind)


def near_unit(eps):
    return 2.0 ** round(math.log2(math.sqrt(eps)))
