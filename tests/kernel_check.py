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

Kernels that only sum are also run on small-integer inputs and must then equal the fp64 result exactly (`exact_ints`,
`assert_equal`); the element-wise kernels are compared bit for bit (`assert_bits_equal`); the dropout keep-bits are
compared with a numpy model of the Philox stream (`dropout_uniforms`, `assert_keep_bits`).
"""
import math

import numpy as np
import torch

SAFETY = 4.0

U_BF16 = 2.0 ** -8      # bf16 round-to-nearest: relative error <= 2^-8
U_F32 = 2.0 ** -24      # fp32 round-to-nearest
# fp32 accumulation of a dot product on the tensor cores: the running sum is rounded once per k16 step; for sign-random
# operands those errors add up like a random walk, so 16 steps' worth of worst-case rounding (2^-20 of sum |a||b|)
# covers sqrt(K/16) <= 16, i.e. K <= 4096, with room to spare
U_ACC = 2.0 ** -20
# ex2.approx.ftz returns 0 for results below fp32's normal range: every probability the attention kernels compute carries,
# besides its relative error, an absolute error of at most 2^-126 (a p of 2^-150 is stored as 0).  Rows whose max lies
# more than 126 log2 units above other keys (one-hot rows of trained models) are where this term is the whole error.
U_FTZ = 2.0 ** -126
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
    """[M, H] or [M] or [H]: (row, 256-column slab, lane, column) of the one-warp-per-row kernels."""
    def f(idx):
        if len(idx) == 2:
            return "row %d, slab %d, lane %d (column %d)" % (idx[0], idx[1] // 256, (idx[1] % 256) // 8, idx[1])
        return "index %d (row, or slab %d of the column vector)" % (idx[0], idx[0] // 256)
    return f


def flat_layout():
    return lambda idx: "element %s" % (idx,)


def flat8_layout(n):
    """flat [n] buffers of the element-wise kernels (relu_bwd, add_bf16, gelu_bwd, cast_f32_bf16): each thread of a
    256-thread block owns one 8-element vector; the last n % 8 elements are the scalar tail loop of one thread."""
    def f(idx):
        i = idx[0]
        t = i // 8
        if i >= n - n % 8:
            return "tail element %d of %d (scalar loop of thread %d, block %d; element %d)" % (i % 8, n % 8, t % 256, t // 256, i)
        return "8-element vector %d (block %d, thread %d), element %d of the vector (element %d)" % (t, t // 256, t % 256, i % 8, i)
    return f


def colsum_layout():
    """[N] column sums: (256-column block = blockIdx.x, lane of the 8-column vector, column)."""
    return lambda idx: "column block %d, lane %d (column %d)" % (idx[0] // 256, (idx[0] % 256) // 8, idx[0])


def scatter_sorted_layout(sorted_idx):
    """[V, H] table gradient of the sorted scatter: the table row, its slab and lane, and the sorted positions of the
    row's run with the warps (32 positions each) and blocks (256 positions) it spans; a run is flushed at every warp
    end, so a run that spans several warps is where a lost or doubled row shows."""
    s = sorted_idx.detach().cpu().to(torch.int64)

    def f(idx):
        v, c = idx
        pos = torch.nonzero(s == v).flatten()
        head = "table row %d, slab %d, lane %d (column %d)" % (v, c // 256, (c % 256) // 8, c)
        if pos.numel() == 0:
            return head + ": no sorted position has this index"
        p0, p1 = int(pos[0]), int(pos[-1])
        return head + ": run of %d at sorted positions %d..%d, warps %d..%d, blocks %d..%d" % (
            p1 - p0 + 1, p0, p1, p0 // 32, p1 // 32, p0 // 256, p1 // 256)
    return f


def adamw_layout(group_of_block):
    """flat [n] AdamW buffers: (8-element block, its hyper-parameter group, CUDA block and thread)."""
    gid = None if group_of_block is None else group_of_block.detach().cpu().to(torch.int64)

    def f(idx):
        b = idx[0] // 8
        g = 0 if gid is None else int(gid[b])
        return "8-element block %d (CUDA block %d, thread %d), group %d, element %d" % (b, b // 256, b % 256, g, idx[0])
    return f


# ------------------------------------------------------------------------------------------------------------------
# exact comparisons: exact-sum inputs and the bit-exact element-wise kernels
# ------------------------------------------------------------------------------------------------------------------
# A worst-case bound on a long fp32 sum is about U_F32 x depth x sum |x|; on random-sign data that exceeds one row's
# contribution, so a sum that dropped or repeated a row would pass it.  The summing kernels (column sums, the scatter
# atomics, the sorted scatter, compose) therefore also run on small integers: every partial sum is then an integer far
# below 2^24 (exact in fp32; compose's |y| <= 5 x 16 = 80 is also exact in bf16), so whatever the summation or atomic
# order, the output must EQUAL the fp64 sum.
def exact_ints(*shape, gen, device="cpu", lo=-16, hi=16):
    """bf16 integers in [lo, hi]"""
    return torch.randint(lo, hi + 1, shape, generator=gen, device=device).to(torch.bfloat16)


def assert_equal(out, ref, layout, what="output"):
    """Exact-input check: torch.equal of the output (widened to fp64, which is exact) and the fp64 reference.  On failure
    the message names the element with the largest |err| in kernel coordinates and how many elements differ."""
    out64 = out.detach().to(torch.float64)
    ref = ref.detach().to(device=out64.device, dtype=torch.float64)
    assert out64.shape == ref.shape, (what, tuple(out64.shape), tuple(ref.shape))
    if torch.equal(out64, ref):
        return
    err = torch.nan_to_num((out64 - ref).abs(), nan=math.inf, posinf=math.inf)
    flat = int(torch.argmax(torch.nan_to_num(err, posinf=1e308)).item())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), err.shape))
    n_bad = int((out64 != ref).sum().item())
    raise AssertionError("%s: %d element(s) differ from the exact result; largest |err| at %s: got %r, exact %r"
                         % (what, n_bad, layout(idx), out64[idx].item(), ref[idx].item()))


_INT_VIEW = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32}


def assert_bits_equal(out, ref, layout, what="output"):
    """Bit-exact check of an element-wise kernel: NaN exactly where the reference is NaN (any payload), and the same bit
    pattern everywhere else (the sign of zero, denormals and infinities included)."""
    out, ref = out.detach(), ref.detach().to(out.device)
    assert out.dtype == ref.dtype and out.shape == ref.shape, (what, out.dtype, ref.dtype, tuple(out.shape), tuple(ref.shape))
    iv = _INT_VIEW[out.dtype]
    on, rn = torch.isnan(out), torch.isnan(ref)
    bad = (on != rn) | (~rn & (out.view(iv) != ref.view(iv)))
    if not bool(bad.any()):
        return
    flat = int(torch.nonzero(bad.flatten())[0].item())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), out.shape))
    mask = (1 << (8 * out.element_size())) - 1
    raise AssertionError("%s: %d element(s) not bit-exact; first at %s: got %r (0x%x), expected %r (0x%x)" % (
        what, int(bad.sum().item()), layout(idx), out[idx].item(), out.view(iv)[idx].item() & mask, ref[idx].item(),
        ref.view(iv)[idx].item() & mask))


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
    # + the flush of p below 2^-126 (U_FTZ per key, in the numerator and in l)
    b_O = b_O + U_FTZ * (Kp @ aV + Skv * O.abs())
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
    # the recomputed p flushed below 2^-126 (U_FTZ |dPd - delta|), and the bf16 dS operand below the normal range (U_FTZ)
    e_dS = e_dS + U_FTZ * ((dPd - delta).abs() + 1.0)
    adS = dS.abs()
    w_dS = e_dS + (U_BF16 + U_ACC) * adS                                           # error of the bf16 dS operand
    sc = 1.0 / math.sqrt(d)
    dQ = (dS @ K) * sc
    dK = (dS.transpose(-1, -2) @ Q) * sc
    dV = Pd.transpose(-1, -2) @ dO
    res["dq"], res["dk"], res["dv"] = _merge(dQ), _merge(dK), _merge(dV)
    res["b_dq"] = _merge(sc * (w_dS @ K.abs()) + U_BF16 * dQ.abs())
    res["b_dk"] = _merge(sc * (w_dS.transpose(-1, -2) @ Q.abs()) + U_BF16 * dK.abs())
    # dV = (P keep dscale)^T dO with P packed to bf16 and recomputed with error r_b (+ its flush below 2^-126, twice: the
    # fp32 p and the bf16 operand)
    res["b_dv"] = _merge(((U_BF16 + U_ACC) * Pd + Pd * r_b + 2 * U_FTZ * Kp).transpose(-1, -2) @ adO + U_BF16 * dV.abs())
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


# ------------------------------------------------------------------------------------------------------------------
# column sums, embedding compose and scatter
# ------------------------------------------------------------------------------------------------------------------
def colsum_grid_y(M, N, sms):
    """row blocks of the column-sum launch: one per 64 rows, capped so that the grid holds about 4 blocks per SM"""
    gx = (N + 255) // 256
    cap = (4 * sms + gx - 1) // gx
    return max(1, min((M + 63) // 64, cap))


def colsum_ref(x, out0, sms):
    """out0 + sum_m x[m] in fp64 and its bound.  The fp32 chain of one column is the rows one warp adds
    (ceil(M / (8 grid.y))), the 8-warp block sum and one atomic per row block (grid.y), each add rounding at most
    U_F32 of the sum of the |terms|."""
    M, N = x.shape
    gy = colsum_grid_y(M, N, sms)
    depth = -(-M // (8 * gy)) + 8 + gy
    x64, o64 = x.to(torch.float64), out0.to(torch.float64)
    return o64 + x64.sum(0), U_F32 * depth * (o64.abs() + x64.abs().sum(0))


def _gather_terms(M, H, terms, device):
    """sum and sum of |.| of the rows t[i[r]] (i < 0: no term) of (buffer, index) pairs, in fp64"""
    y = torch.zeros(M, H, dtype=torch.float64, device=device)
    a = torch.zeros_like(y)
    for t, i in terms:
        i = i.to(device=device, dtype=torch.int64)
        rows = t.to(torch.float64)[i.clamp_min(0)] * (i >= 0).to(torch.float64)[:, None]
        y += rows
        a += rows.abs()
    return y, a


def compose_ref(M, H, srcs, tabs, device):
    """y[r] = sum_k src_k[row_k[r]] + sum_k tab_k[idx_k[r]] in fp64 and its bound: up to 5 terms added in fp32 (at most
    4 roundings of U_F32 sum |terms|), then the bf16 output rounding"""
    y, a = _gather_terms(M, H, list(srcs) + list(tabs), device)
    return y, U_BF16 * y.abs() + 4 * U_F32 * a


def scatter_table_ref(dtab0, dy, idx):
    """dtab0[v] + sum_{r: idx[r] = v} dy[r] in fp64 and its bound.  Both scatters add n_v terms into row v in fp32 in an
    order that is not fixed (atomics; the sorted scatter first sums each run in registers, with one atomic per run):
    n_v roundings of at most U_F32 (|dtab0[v]| + sum |dy[r]|)."""
    V = dtab0.shape[0]
    i = idx.to(device=dy.device, dtype=torch.int64)
    ok = i >= 0
    d64 = dy.to(torch.float64)[ok]
    ref, a = dtab0.to(torch.float64).clone(), dtab0.to(torch.float64).abs()
    ref.index_add_(0, i[ok], d64)
    a.index_add_(0, i[ok], d64.abs())
    n = torch.bincount(i[ok], minlength=V).to(torch.float64)
    return ref, U_F32 * n[:, None] * a


# ------------------------------------------------------------------------------------------------------------------
# dropout keep-bits: a numpy model of the Philox stream, stated per element
# ------------------------------------------------------------------------------------------------------------------
_M32 = 0xFFFFFFFF


def philox4x32_7(seed, ctr):
    """Philox4x32 with 7 rounds as common.cuh defines it: key = (seed low, seed high), counter = (ctr low, ctr high,
    0x243F6A88, 0x85A308D3).  ctr: uint64 array.  Returns the four uint32 outputs (uint64 arrays holding 32-bit values)."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    m32, s32 = np.uint64(_M32), np.uint64(32)
    c0, c1 = ctr & m32, ctr >> s32
    c2, c3 = np.full_like(ctr, 0x243F6A88), np.full_like(ctr, 0x85A308D3)
    k0, k1 = seed & _M32, (seed >> 32) & _M32
    for _ in range(7):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)      # < 2^64: exact
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ np.uint64(k0), p1 & m32, (p0 >> s32) ^ c3 ^ np.uint64(k1), p0 & m32
        k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
    return c0, c1, c2, c3


def dropout_thresh16(p):
    """the kernel's 16-bit threshold, evaluated in fp32 like the host code: min(65535, floor(p 65536 + 0.5))"""
    t = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    return min(65535, int(np.floor(t)))


def dropout_planes(nwords, seed, offset, epoch=0):
    """[16, nwords] uint32: row b holds bit b of the 32 uniforms of each word (bit e of the row = uniform e).  Word w
    draws the Philox counters offset + (epoch << 40) + 4 w + i, i = 0..3 (mod 2^64), and output k of draw i is the
    plane of bit 15 - (4 i + k)."""
    base = np.uint64((offset + (epoch << 40)) % 2 ** 64)
    w4 = np.arange(nwords, dtype=np.uint64) * np.uint64(4)
    planes = np.empty((16, nwords), dtype=np.uint32)
    for i in range(4):
        out = philox4x32_7(seed, base + w4 + np.uint64(i))
        for k in range(4):
            planes[15 - (4 * i + k)] = out[k].astype(np.uint32)
    return planes


def uniforms_from_planes(planes):
    """[16, W] bit-planes -> [W, 32] uint32 sixteen-bit uniforms r_e (bit b of r_e = bit e of plane b)"""
    e = np.arange(32, dtype=np.uint32)
    r = np.zeros((planes.shape[1], 32), dtype=np.uint32)
    for b in range(16):
        r |= ((planes[b][:, None] >> e) & np.uint32(1)) << np.uint32(b)
    return r


def dropout_uniforms(nwords, seed, offset, epoch=0):
    """[nwords, 32] uniforms of the keep-bit words; element 32 w + e is kept where uniforms[w, e] >= thresh16"""
    return uniforms_from_planes(dropout_planes(nwords, seed, offset, epoch))


def assert_keep_bits(words, uniforms, p, what="keep bits"):
    """words (int32, any shape, flat = word index) against the model: bit e of word w = (uniforms[w, e] >= thresh16)"""
    t = dropout_thresh16(p)
    got = np.ascontiguousarray(words.detach().cpu().numpy()).view(np.uint32).reshape(-1)
    assert got.shape[0] == uniforms.shape[0], (what, got.shape, uniforms.shape)
    gk = ((got[:, None] >> np.arange(32, dtype=np.uint32)) & np.uint32(1)).astype(bool)
    bad = gk != (uniforms >= t)
    if bad.any():
        w, e = (int(v) for v in np.argwhere(bad)[0])
        raise AssertionError("%s: %d keep bit(s) in %d word(s) differ from the model; first: word %d, bit %d at p = %r "
                             "(thresh16 %d): kernel %d, uniform %d" % (what, int(bad.sum()), int(bad.any(1).sum()), w, e,
                                                                       p, t, int(gk[w, e]), int(uniforms[w, e])))


# ------------------------------------------------------------------------------------------------------------------
# AdamW (include/mmfb200.h: mmfb_adamw), one step in fp64 with the error bound carried across steps
# ------------------------------------------------------------------------------------------------------------------
def _f32(x):
    return float(np.float32(x))


def adamw_step_ref(st, g, groups, gid, *, beta1, beta2, eps, mode, grad_scale):
    """Advances st = {p, m, v, e_p, e_m, e_v} (fp64 [n]; e_* the error bounds of the kernel's fp32 state) by one step
    with gradient g (fp32 [n]), the operation order of the kernel, and hyper-parameters rounded to fp32 as the C ABI
    passes them.  Each fp32 operation adds U_F32 of its result (first order); errors already in p, m and v propagate
    through the update."""
    U = U_F32
    dev = st["p"].device
    grp = (torch.zeros(st["p"].numel() // 8, dtype=torch.int64, device=dev) if gid is None
           else gid.to(device=dev, dtype=torch.int64)).repeat_interleave(8)

    def per(key):           # the hyper-parameter of each element's group
        return torch.tensor([_f32(gr[key]) for gr in groups], dtype=torch.float64, device=dev)[grp]
    lr, wd, step, bc2s = per("lr"), per("weight_decay"), per("step_size"), per("bc2_sqrt")
    b1, b2, eps, gs = _f32(beta1), _f32(beta2), _f32(eps), _f32(grad_scale)
    c1, c2 = float(np.float32(1) - np.float32(b1)), float(np.float32(1) - np.float32(b2))
    p, m, v, e_p, e_m, e_v = (st[k] for k in ("p", "m", "v", "e_p", "e_m", "e_v"))
    gr = g.to(torch.float64) * gs
    e_gr = U * gr.abs()
    lw = lr * wd
    if mode == 1:
        p1 = p * (1 - lw)                                               # lr*wd, 1 - lr*wd and the product: 3 roundings
        e_p = e_p * (1 - lw) + p.abs() * U * (lw + (1 - lw)) + U * p1.abs()
        p = p1
        d = gr - m                                                      # m.lerp_(g, 1 - b1) = fma(g - m, 1 - b1, m)
        m_new = m + c1 * d
        e_m = (1 - c1) * e_m + c1 * (e_gr + U * d.abs()) + U * m_new.abs()
    else:
        m_new = b1 * m + c1 * gr                                        # fma(g, 1 - b1, m * b1)
        e_m = b1 * e_m + c1 * e_gr + U * b1 * m.abs() + U * m_new.abs()
    v_new = b2 * v + c2 * gr * gr                                       # fma(g * g, 1 - b2, v * b2)
    e_v = b2 * e_v + c2 * (2 * gr.abs() * e_gr + U * gr * gr) + U * b2 * v + U * v_new
    s = v_new.sqrt()
    e_s = e_v / (2 * s) + U * s
    if mode == 1:
        s, e_s = s / bc2s, e_s / bc2s + U * s / bc2s
    den = s + eps
    e_den = e_s + U * den
    q = m_new / den
    e_q = e_m / den + q.abs() * e_den / den + U * q.abs()
    p1 = p - step * q                                                   # fma(-step, m / denom, p)
    e_p = e_p + step * e_q + U * p1.abs()
    if mode == 0:
        dec = wd > 0                                                    # fma(p, -lr * wd, p)
        p2 = torch.where(dec, p1 * (1 - lw), p1)
        e_p = torch.where(dec, e_p * (1 + lw) + U * lw * p1.abs() + U * p2.abs(), e_p)
        p1 = p2
    st.update(p=p1, m=m_new, v=v_new, e_p=e_p, e_m=e_m, e_v=e_v)
    return st


def adamw_state(p, m, v):
    """fp64 copy of the fp32 optimizer state with zero error bounds, for adamw_step_ref"""
    st = {k: t.detach().to(torch.float64).clone() for k, t in (("p", p), ("m", m), ("v", v))}
    st.update({"e_" + k: torch.zeros_like(st[k]) for k in ("p", "m", "v")})
    return st


# ------------------------------------------------------------------------------------------------------------------
# element-wise GELU backward
# ------------------------------------------------------------------------------------------------------------------
def gelu_bwd_ref(dh, u):
    """du = dh GELU'(u) in fp64 and its bound: GELU' in fp32 with the erf / ex2 approximations (|err| <= 2^-21 (1 + |u|),
    as in the GEMM's gelu_bwd epilogue), the fp32 product and the bf16 output rounding"""
    dh64, u64 = dh.to(torch.float64), u.to(torch.float64)
    ref = dh64 * gelu_grad64(u64)
    return ref, U_BF16 * ref.abs() + U_F32 * ref.abs() + dh64.abs() * 2.0 ** -21 * (1 + u64.abs())
