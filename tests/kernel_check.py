"""Per-element checks of the CUDA kernels against fp64 references (a plain module, imported by the edge tests).

A whole-tensor relative L2 norm averages a local error away: one 128 x 256 GEMM tile that lost its last k-block, or one
wrong attention row among thousands, moves it by far less than 1e-2.  The checks here compare every element instead:

    |out - ref| <= SAFETY * bound        elementwise, with ref computed in fp64 from the bf16 inputs the kernel sees

Each `bound` is built from the rounding steps the kernel actually performs (bf16 rounding u = 2^-8 relative, fp32
u = 2^-24 relative) and is written next to its formula.  SAFETY = 4 is one factor for every kernel: the bounds take
each rounding at its first-order worst case, so 4 only absorbs the second-order terms and the few constant factors
(exp2 / rsqrt / log approximations of up to 2 ulp) that are not spelled out; it is not a tolerance to tune.  A kernel
that needs more than SAFETY x its bound is a finding, not a reason to raise the factor.

One exception to "worst case": the fp32 accumulation of the tensor-core products (U_ACC, in the GEMM and attention
bounds) assumes operands of random sign, whose per-step roundings partly cancel.  The worst case grows with K / 16
steps instead (about 2^-16.4 of sum |a||b| at K = 3072).  Inputs with one sign (all-positive operands, for example)
can exceed these terms without any kernel bug; use sign-random inputs with this helper.

On failure the message names the worst element in the kernel's own coordinates (`*_layout` below), so a broken tile,
row, head or slab is visible at once.
"""
import math

import torch

SAFETY = 4.0

U_BF16 = 2.0 ** -8      # bf16 round-to-nearest: relative error <= 2^-8
U_F32 = 2.0 ** -24      # fp32 round-to-nearest
# fp32 accumulation of a dot product on the tensor cores: the running sum is rounded once per k16 step; for sign-random
# operands those errors add up like a random walk, so 16 steps' worth of worst-case rounding (2^-20 of sum |a||b|)
# covers sqrt(K/16) <= 16, i.e. K <= 4096, with room to spare
U_ACC = 2.0 ** -20
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)


def bf16_round(t):
    """fp64 tensor rounded to the nearest bf16 value, back in fp64"""
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def assert_within(out, ref, bound, layout, what="output"):
    """Fails if any element has |out - ref| > SAFETY * bound (a non-finite output always fails).  `layout(index)` turns
    the multi-index of the worst element into kernel coordinates.  Returns the worst |err| / bound (for reports)."""
    out = out.detach().to(torch.float64)
    ref = ref.detach().to(device=out.device, dtype=torch.float64)
    bound = bound.detach().to(device=out.device, dtype=torch.float64).expand_as(ref)
    assert out.shape == ref.shape, (what, tuple(out.shape), tuple(ref.shape))
    err = (out - ref).abs()
    ratio = err / bound.clamp_min(1e-300)
    ratio = torch.where(torch.isfinite(out), ratio, torch.full_like(ratio, math.inf))
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    worst = ratio.max().item() if ratio.numel() else 0.0
    if not worst <= SAFETY:
        flat = int(torch.argmax(torch.nan_to_num(ratio, nan=math.inf, posinf=1e308)).item())
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ratio.shape))
        n_bad = int((ratio > SAFETY).sum().item())
        raise AssertionError(
            "%s: %d element(s) beyond %.0f x bound; worst |err|/bound = %.3g at %s: got %r, fp64 ref %r, bound %.3g"
            % (what, n_bad, SAFETY, worst, layout(idx), out[idx].item(), ref[idx].item(), bound[idx].item()))
    return worst


# ------------------------------------------------------------------------------------------------------------------
# kernel coordinates of an element
# ------------------------------------------------------------------------------------------------------------------
def gemm_layout(block_n, splits=1, bm=128):
    """C [M, N]: (m-tile, n-tile, row in tile, column in tile, split count).  Every split adds into every element of its
    tile, so the split count of the launch is named rather than one split."""
    def f(idx):
        m, n = idx
        return "m-tile %d, n-tile %d, row %d / col %d in the %dx%d tile (element [%d, %d]), splits=%d" % (
            m // bm, n // block_n, m % bm, n % block_n, bm, block_n, m, n, splits)
    return f


def attn_layout(B, heads, S, d, rows="query"):
    """[B*S, heads*d] (ctx, dq: rows are queries; dk, dv: rows are keys) or [B, heads, S] (lse2):
    (batch, head, row, 64-row block of that sequence)."""
    def f(idx):
        if len(idx) == 3:
            b, h, r = idx
            c = None
        else:
            b, r = divmod(idx[0], S)
            h, c = divmod(idx[1], d)
        s = "batch %d, head %d, %s row %d (%s block %d)" % (b, h, rows, r, "key" if rows == "key" else "query", r // 64)
        return s + (", column %d of the head" % c if c is not None else "")
    return f


def row_layout():
    """[M, H] or [M] or [H]: (row, 256-column slab, column) of the one-warp-per-row kernels."""
    def f(idx):
        if len(idx) == 2:
            return "row %d, slab %d (column %d)" % (idx[0], idx[1] // 256, idx[1])
        return "index %d (row, or slab %d of the column vector)" % (idx[0], idx[0] // 256)
    return f


def flat_layout():
    return lambda idx: "element %s" % (idx,)


# ------------------------------------------------------------------------------------------------------------------
# GEMM:  C = epi(A B^T)
# ------------------------------------------------------------------------------------------------------------------
def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def gemm_ref(a, b):
    """a [M, K], b [N, K] (logical, bf16 values): fp64 A B^T and sum_k |a||b| (the scale of the accumulation error)."""
    a64, b64 = a.to(torch.float64), b.to(torch.float64)
    return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def gemm_bound(ref, absab, extra=0.0, bf16_out=True):
    """|c - ref| <= 2^-8 |ref| (bf16 output rounding) + 2^-20 (|A||B|^T + extra) (fp32 accumulation and epilogue
    arithmetic on terms of that size).  fp32 outputs (split-K) drop the first term."""
    b = U_ACC * (absab + extra)
    if bf16_out:
        b = b + U_BF16 * ref.abs()
    return b


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
def _heads(t, B, S, heads, d):
    return t.to(torch.float64).reshape(B, S, heads, d).permute(0, 2, 1, 3)       # [B, h, S, d]


def _merge(t):
    B, h, S, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * S, h * d)


def attention_ref(q, k, v, B, heads, Sq, Skv, mask=None, keep=None, p_drop=0.0, dctx=None, lo_used=False, p_exact=False):
    """fp64 forward (and backward when dctx is given) of softmax(Q K^T / sqrt(d) + mask) V with explicit keep bits, and
    per-element bounds for every output.  `mask` is the additive fp32 [B, Skv] mask as the kernel stages it (the caller
    applies the clamp to -10000 when it wants the kernel's effective mask).  Returns a dict of [B*S, h*d] / [B, h, Sq]
    tensors: ctx, lse2, dq, dk, dv and b_ctx, b_lo, b_lse2, b_dq, b_dk, b_dv.

    p_exact: every forward probability the kernel packs to bf16 is exactly representable (q = 0 and no mask: every
    staged p is 2^0 = 1), so the forward's bf16 packing term drops out of the bounds of O.  Only then is the fp32 O, and
    with it ctx + ctx_lo and the backward's delta, bounded at the 2^-16 level; with general P the packing error
    (2^-8 P|V|) of O itself dominates every comparison with fp64."""
    d = q.shape[1] // heads
    Q, K, V = _heads(q, B, Sq, heads, d), _heads(k, B, Skv, heads, d), _heads(v, B, Skv, heads, d)
    scale2 = LOG2E / math.sqrt(d)
    m2 = torch.zeros(B, 1, 1, Skv, dtype=torch.float64, device=Q.device)
    if mask is not None:
        m2 = mask.to(torch.float64).reshape(B, 1, 1, Skv) * LOG2E
    Z = (Q @ K.transpose(-1, -2)) * scale2 + m2                                    # log2-domain scores [B, h, Sq, Skv]
    zmax = Z.amax(-1, keepdim=True)
    lse2 = zmax + torch.log2(torch.exp2(Z - zmax).sum(-1, keepdim=True))
    P = torch.exp2(Z - lse2)
    dsc = 1.0 / (1.0 - p_drop)
    Kp = torch.ones_like(P) if keep is None else keep.to(torch.float64) * dsc     # keep * dscale
    Pd = P * Kp
    O = Pd @ V
    # exponent error of every staged score (log2 units): fmaf rounding and the mask * log2e product (2^-23 (|Z| + |M|)),
    # the fp32 accumulation of q.k (2^-20 scale2 |q||k|), ex2.approx (2^-22)
    E = 2.0 ** -23 * (Z.abs() + m2.abs()) + U_ACC * scale2 * (Q.abs() @ K.abs().transpose(-1, -2)) + 2.0 ** -22
    E = torch.where(torch.isinf(Z), torch.zeros_like(E), E)                       # keys at -inf: p = 0 exactly
    E_max = torch.gather(E, -1, Z.argmax(-1, keepdim=True))                       # the row maximum carries its own error
    r_f = LN2 * (E + E_max)                                                        # relative error of each forward p
    aV = V.abs()
    PaV = Pd @ aV
    # fp32 O = sum_j p_j v_j / l:  P packed to bf16 before the PV product (2^-8 P|V|), its fp32 accumulation (2^-20 P|V|),
    # p errors r_j in the numerator ((P r)|V|) and in the normaliser l ((P r) 1 |O|)
    b_O = ((0.0 if p_exact else U_BF16) + U_ACC) * PaV + (Pd * r_f) @ aV + (P * r_f).sum(-1, keepdim=True) * O.abs()
    res = {"ctx": _merge(O), "lse2": lse2.squeeze(-1),
           "b_ctx": _merge(b_O + U_BF16 * O.abs()),                                # + bf16 output rounding
           "b_lo": _merge(b_O + 2.0 ** -16 * O.abs())}                             # ctx + ctx_lo: hi + lo of the fp32 O
    # lse2 = max + log2(l): score errors (P E + E_max), fp32 sum of l over Skv/4 + 2 sequential adds (1.5 (Skv/4 + 2)
    # 2^-24 in log2 units), log2f (2^-20 absolute for l <= 2^9) and the final add (2^-23 |lse2|)
    e_lse = (P * E).sum(-1, keepdim=True) + E_max + 1.5 * (Skv / 4 + 2) * U_F32 + 2.0 ** -20 + 2.0 ** -23 * lse2.abs()
    res["b_lse2"] = e_lse.squeeze(-1)
    if dctx is None:
        return res
    dO = _heads(dctx, B, Sq, heads, d)
    adO = dO.abs()
    dP = dO @ V.transpose(-1, -2)
    dPd = dP * Kp
    delta = (dO * O).sum(-1, keepdim=True)
    dS = P * (dPd - delta)
    # the backward recomputes p = 2^(z - lse2) from the saved lse2: relative error ln2 (E + e_lse)
    r_b = LN2 * (E + e_lse)
    # delta = rowsum(dO * O_used): O_used is ctx (+ ctx_lo), whose error is the bound just derived, plus fp32 sums
    b_Oused = b_O + (2.0 ** -16 if lo_used else U_BF16) * O.abs()
    e_delta = (adO * b_Oused).sum(-1, keepdim=True) + U_ACC * (adO * O.abs()).sum(-1, keepdim=True)
    # dS = p (dPd - delta): dP accumulated in fp32 (2^-20 |dO||V|^T), delta error, p error; dS is then packed to bf16
    e_dS = P * (U_ACC * Kp * (adO @ aV.transpose(-1, -2)) + e_delta) + P * r_b * (dPd - delta).abs()
    adS = dS.abs()
    w_dS = e_dS + (U_BF16 + U_ACC) * adS                                           # error of the bf16 dS operand
    sc = 1.0 / math.sqrt(d)
    dQ = (dS @ K) * sc
    dK = (dS.transpose(-1, -2) @ Q) * sc
    dV = Pd.transpose(-1, -2) @ dO
    res["dq"], res["dk"], res["dv"] = _merge(dQ), _merge(dK), _merge(dV)
    res["b_dq"] = _merge(sc * (w_dS @ K.abs()) + U_BF16 * dQ.abs())
    res["b_dk"] = _merge(sc * (w_dS.transpose(-1, -2) @ Q.abs()) + U_BF16 * dK.abs())
    # dV = (P keep dscale)^T dO with P packed to bf16 and recomputed with error r_b
    res["b_dv"] = _merge(((U_BF16 + U_ACC) * Pd + Pd * r_b).transpose(-1, -2) @ adO + U_BF16 * dV.abs())
    return res


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
def layernorm_ref(y, g, b, eps=1e-12):
    """fp64 LayerNorm forward of bf16 y [M, H] with bf16 gamma / beta; bounds of mean, rstd and x."""
    M, H = y.shape
    NV = (H + 255) // 256
    y64, g64, b64 = y.to(torch.float64), g.to(torch.float64), b.to(torch.float64)
    mu = y64.mean(1)
    var = ((y64 - mu[:, None]) ** 2).mean(1)
    rs = 1.0 / torch.sqrt(var + eps)
    xh = (y64 - mu[:, None]) * rs[:, None]
    x = xh * g64 + b64
    # mean: fp32 sum of 8 NV terms per lane and a 5-level warp tree (depth 8 NV + 6), then / H
    b_mu = U_F32 * (8 * NV + 6) * y64.abs().mean(1)
    # rstd: the variance is a sum of positive terms (depth 8 NV + 6, plus the squares' rounding); rsqrtf <= 2 ulp;
    # the sqrt halves the relative error of the variance
    rho = 0.5 * U_F32 * (8 * NV + 8) + 2.0 ** -22
    b_rs = rho * rs
    # xhat = (y - mu) rstd: relative rstd error and the mean's error; x = xhat g + b rounded to bf16
    e_xh = (y64 - mu[:, None]).abs() * b_rs[:, None] + rs[:, None] * b_mu[:, None]
    b_x = U_BF16 * x.abs() + g64.abs() * e_xh + 2.0 ** -22 * (xh.abs() * g64.abs() + b64.abs())
    return {"x": x, "mean": mu, "rstd": rs, "xh": xh, "e_xh": e_xh, "b_x": b_x, "b_mean": b_mu, "b_rstd": b_rs}


def layernorm_bwd_ref(fw, dx, g, dx2=None, keep=None, dscale=1.0, n_sum_terms=1):
    """fp64 LayerNorm backward from the forward dict `fw`; bounds of dy, dz and of the column sums.  `n_sum_terms` is the
    depth of the fp32 column-sum chain (rows per warp + the block tree + one atomic per block)."""
    xh, e_xh, rs = fw["xh"], fw["e_xh"], fw["rstd"][:, None]
    H = xh.shape[1]
    NV = (H + 255) // 256
    d = dx.to(torch.float64) + (dx2.to(torch.float64) if dx2 is not None else 0.0)
    g64 = g.to(torch.float64)
    dg = d * g64
    m1 = dg.mean(1, keepdim=True)
    m2 = (dg * xh).mean(1, keepdim=True)
    dy = rs * (dg - m1 - xh * m2)
    # dy = rstd (d g - m1 - xhat m2): fp32 products / fmas (2^-20 of the terms), the row sums m1, m2 (depth 8 NV + 6),
    # the relative rstd error (rho |dy|) and xhat's error through xhat m2 and through m2 itself; then bf16 rounding
    e_m = U_F32 * (8 * NV + 6)
    terms = dg.abs() + m1.abs() + xh.abs() * m2.abs()
    e_dy_f32 = (U_ACC * rs * terms + e_m * rs * (dg.abs().mean(1, keepdim=True) + xh.abs() * (dg * xh).abs().mean(1, keepdim=True))
                + (fw["b_rstd"][:, None] / fw["rstd"][:, None]) * dy.abs()
                + rs * (e_xh * m2.abs() + xh.abs() * (dg.abs() * e_xh).mean(1, keepdim=True)))
    res = {"dy": dy, "b_dy": e_dy_f32 + U_BF16 * dy.abs()}
    kd = torch.ones_like(dy) if keep is None else keep.to(torch.float64) * dscale
    dz = dy * kd
    e_dz_f32 = e_dy_f32 * kd + U_F32 * dz.abs()
    res["dz"], res["b_dz"], res["e_dz_f32"] = dz, e_dz_f32 + U_BF16 * dz.abs(), e_dz_f32
    # column sums: products d * xhat in fp32 (xhat error e_xh), then n_sum_terms sequential fp32 adds
    res["dgamma"] = (d * xh).sum(0)
    res["b_dgamma"] = (d.abs() * e_xh).sum(0) + U_F32 * (n_sum_terms + 1) * (d * xh).abs().sum(0)
    res["dbeta"] = d.sum(0)
    res["b_dbeta"] = U_F32 * n_sum_terms * d.abs().sum(0)
    return res
