"""Fused attention at its edges, every element of ctx, lse2, dq, dk and dv against fp64 (tests/kernel_check.py):
sequence lengths around the 64-row tiles and at the 384 / 256 limits, cross-attention far from square, odd head counts,
dropout word boundaries, ragged key lengths down to one key, fused q/k/v slices, the backward with and without ctx_lo,
and additive masks down to finfo.min and -inf."""
import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu

MASK_FLOOR = -10000.0       # the kernels treat every mask value below this as this (include/mmfb200.h)


def _inputs(B, heads, Sq, Skv, d, g):
    W = heads * d
    if Sq == Skv:                       # q / k / v as column slices of one fused projection buffer
        qkv = (torch.randn(B * Sq, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
        return qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    q = (torch.randn(B * Sq, W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    kv = (torch.randn(B * Skv, 2 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    return q, kv[:, :W], kv[:, W:]


def _check_all(out, ref, B, heads, Sq, Skv, d, tag, samples=None):
    """per-element checks of the kernel outputs `out` (dict) against the fp64 `ref`; `samples` restricts the check to
    those batch entries.  Returns {output: worst |err| / bound}."""
    sel_q = sel_k = slice(None)
    bsel = slice(None)
    if samples is not None:
        idx = torch.tensor(samples, device="cuda")
        rows_q = (idx[:, None] * Sq + torch.arange(Sq, device="cuda")).reshape(-1)
        rows_k = (idx[:, None] * Skv + torch.arange(Skv, device="cuda")).reshape(-1)
        sel_q, sel_k, bsel = rows_q, rows_k, idx
    nb = B if samples is None else len(samples)
    lq = kc.attn_layout(nb, heads, Sq, d, "query")
    lk = kc.attn_layout(nb, heads, Skv, d, "key")
    worst = {}
    worst["ctx"] = kc.assert_within(out["ctx"][sel_q], ref["ctx"][sel_q], ref["b_ctx"][sel_q], lq, tag + " ctx")
    worst["lse2"] = kc.assert_within(out["lse2"][bsel], ref["lse2"][bsel], ref["b_lse2"][bsel], lq, tag + " lse2")
    if "ctx_lo" in out:
        hi_lo = out["ctx"].double() + out["ctx_lo"].double()
        worst["ctx+lo"] = kc.assert_within(hi_lo[sel_q], ref["ctx"][sel_q], ref["b_lo"][sel_q], lq, tag + " ctx+ctx_lo")
    for name, lay, sel in (("dq", lq, sel_q), ("dk", lk, sel_k), ("dv", lk, sel_k)):
        if name in out:
            worst[name] = kc.assert_within(out[name][sel], ref[name][sel], ref["b_" + name][sel], lay, tag + " " + name)
    return worst


def run_case(B, heads, Sq, Skv, d, lens=None, p_drop=0.0, seed=0, mask_value=MASK_FLOOR, use_lo=True, mask=None):
    """forward (with ctx_lo) and backward through functional.attention_*; returns (outputs, inputs for the reference)"""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = _inputs(B, heads, Sq, Skv, d, g)
    if mask is None and lens is not None:
        lens_t = torch.tensor(lens, device="cuda")
        mask = torch.where(torch.arange(Skv, device="cuda")[None, :] < lens_t[:, None], 0.0, mask_value).float().contiguous()
    keep = dm = None
    if p_drop > 0:
        keep = torch.rand(B, heads, Sq, Skv, generator=g, device="cuda") >= p_drop
        dm = F.pack_keep_bits(keep)
    dsc = 1.0 / (1.0 - p_drop)
    ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, Sq, Skv, mask=mask, drop_mask=dm, drop_scale=dsc, save_lo=True)
    dctx = torch.randn(B * Sq, heads * d, generator=g, device="cuda").to(torch.bfloat16)
    dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, Sq, Skv, mask=mask, drop_mask=dm, drop_scale=dsc,
                                 ctx_lo=lo if use_lo else None)
    torch.cuda.synchronize()
    out = {"ctx": ctx, "lse2": lse2, "ctx_lo": lo, "dq": dq, "dk": dk, "dv": dv}
    inp = {"q": q, "k": k, "v": v, "mask": mask, "keep": keep, "p_drop": p_drop, "dctx": dctx, "lo_used": use_lo}
    return out, inp


def reference(inp, B, heads, Sq, Skv, mask=None):
    m = inp["mask"] if mask is None else mask
    return kc.attention_ref(inp["q"], inp["k"], inp["v"], B, heads, Sq, Skv, mask=m, keep=inp["keep"],
                            p_drop=inp["p_drop"], dctx=inp["dctx"], lo_used=inp["lo_used"])


def _ragged(B, Skv, g_seed):
    """key lengths: the first sample sees every key (so a single-sample case checks every key block), the second one
    key, the rest random"""
    g = torch.Generator().manual_seed(g_seed)
    lens = [Skv, 1] + torch.randint(1, Skv + 1, (max(B - 2, 0),), generator=g).tolist()
    return lens[:B]


SELF = [  # (B, heads, S, d)
    (2, 3, 1, 64), (2, 1, 2, 128), (3, 3, 63, 64), (2, 12, 64, 64), (2, 3, 65, 128), (2, 1, 127, 64), (2, 3, 128, 128),
    (2, 12, 129, 64), (2, 3, 255, 64), (2, 1, 256, 128), (2, 3, 257, 64), (2, 3, 383, 64), (1, 12, 384, 64),
    (2, 3, 129, 128), (2, 1, 1, 128),
]


@pytest.mark.parametrize("B,heads,S,d", SELF)
def test_self_attention_edges(B, heads, S, d):
    lens = _ragged(B, S, S)
    worst = {}
    for use_lo in (True, False):
        out, inp = run_case(B, heads, S, S, d, lens=lens, seed=S + d, use_lo=use_lo)
        w = _check_all(out, reference(inp, B, heads, S, S), B, heads, S, S, d,
                       "self B%d h%d S%d d%d lo=%d" % (B, heads, S, d, use_lo))
        worst = {k_: max(worst.get(k_, 0.0), v_) for k_, v_ in w.items()}
    print("attn self B%d h%d S%d d%d: %s" % (B, heads, S, d, " ".join("%s=%.3f" % kv for kv in worst.items())))


CROSS = [  # (B, heads, Sq, Skv, d)
    (2, 3, 1, 36, 64), (2, 3, 65, 1, 128), (2, 12, 36, 384, 64), (2, 3, 1000, 36, 128), (1, 3, 2048, 64, 64),
    (2, 1, 36, 256, 128),
]


@pytest.mark.parametrize("B,heads,Sq,Skv,d", CROSS)
def test_cross_attention_edges(B, heads, Sq, Skv, d):
    out, inp = run_case(B, heads, Sq, Skv, d, lens=_ragged(B, Skv, Sq), seed=Sq + Skv)
    w = _check_all(out, reference(inp, B, heads, Sq, Skv), B, heads, Sq, Skv, d, "cross Sq%d Skv%d d%d" % (Sq, Skv, d))
    print("attn cross B%d h%d Sq%d Skv%d d%d: %s" % (B, heads, Sq, Skv, d, " ".join("%s=%.3f" % kv for kv in w.items())))


@pytest.mark.parametrize("Skv", [31, 32, 33, 63, 65])
@pytest.mark.parametrize("d", [64, 128])
def test_attention_dropout_word_edges(Skv, d):
    Sq = 40 if d == 64 else 70
    for use_lo in (True, False):
        out, inp = run_case(3, 3, Sq, Skv, d, lens=_ragged(3, Skv, Skv), p_drop=0.1, seed=Skv, use_lo=use_lo)
        w = _check_all(out, reference(inp, 3, 3, Sq, Skv), 3, 3, Sq, Skv, d, "dropout Skv%d d%d" % (Skv, d))
    print("attn dropout Skv%d d%d: %s" % (Skv, d, " ".join("%s=%.3f" % kv for kv in w.items())))


MASK_VALUES = [-10000.0, -1e9, float(torch.finfo(torch.bfloat16).min), float(torch.finfo(torch.float32).min),
               float("-inf")]


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("mask_value", MASK_VALUES, ids=["-1e4", "-1e9", "bf16min", "fp32min", "-inf"])
def test_attention_masks_down_to_dtype_min(mask_value, d):
    """HF's extended attention mask uses finfo(dtype).min (or -inf): sample 0 is right-padded, sample 1 left-padded (its
    first key block is fully masked, so the online softmax starts on masked keys), sample 2 fully masked.  Every output
    is finite; below -10000 the outputs are bit-identical to the -10000 run; samples with an unmasked key match fp64
    computed with the original mask, and the -10000 run matches fp64 everywhere."""
    B, heads, S = 3, 2, 100
    mask = torch.zeros(B, S, device="cuda")
    mask[0, 60:] = mask_value
    mask[1, :70] = mask_value
    mask[2, :] = mask_value
    out, inp = run_case(B, heads, S, S, d, seed=d, mask=mask.contiguous())
    for name, t in out.items():
        assert torch.isfinite(t.float()).all(), "%s has non-finite values with mask value %r" % (name, mask_value)
    if mask_value < MASK_FLOOR:
        base, _ = run_case(B, heads, S, S, d, seed=d, mask=torch.where(mask < MASK_FLOOR, MASK_FLOOR, mask).contiguous())
        for name in out:
            assert torch.equal(out[name], base[name]), "%s differs from the -10000 run" % name
        _check_all(out, reference(inp, B, heads, S, S), B, heads, S, S, d, "mask %r d%d" % (mask_value, d), samples=[0, 1])
    else:
        _check_all(out, reference(inp, B, heads, S, S), B, heads, S, S, d, "mask %r d%d" % (mask_value, d))


@pytest.mark.parametrize("Skv", [36, 64])
def test_ctx_lo_carries_the_fp32_output(Skv):
    """With general inputs the bf16 packing of P (2^-8 P|V|) dominates the error of the fp32 output O, so no comparison
    with fp64 can see ctx_lo.  Here q = 0 and there is no mask: every staged p is exactly 1, and O = mean_j v_j has only
    fp32 error.  So ctx + ctx_lo must match fp64 to ~2^-16, while ctx alone is only good to 2^-9.
    v_j = v + -1 ulp puts O between bf16 values.  Identical key rows make dq = scale k sum_j dS_j, which is 0 in exact
    arithmetic, so dq shows the error of the backward's delta = rowsum(dO (ctx + ctx_lo)) directly; dO takes the sign of
    O - ctx, so a delta that leaves ctx_lo out errs coherently.  Both omissions are shown to fail the check."""
    from mmf_b200 import functional as F
    B, heads, Sq, d = 2, 3, 65, 64
    W = heads * d
    g = torch.Generator(device="cuda").manual_seed(Skv)
    q = torch.zeros(B * Sq, W, device="cuda", dtype=torch.bfloat16)
    kbar = torch.randn(B, 1, W, generator=g, device="cuda")
    k = kbar.expand(B, Skv, W).reshape(B * Skv, W).to(torch.bfloat16).contiguous()
    vbar = (torch.randn(B, 1, W, generator=g, device="cuda") * 0.8).to(torch.bfloat16).float()
    s = torch.randint(-1, 2, (B, Skv, W), generator=g, device="cuda").float()
    v = (vbar * (1 + s * 2.0 ** -7)).reshape(B * Skv, W).to(torch.bfloat16)
    ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, Sq, Skv, save_lo=True)
    fw = kc.attention_ref(q, k, v, B, heads, Sq, Skv, p_exact=True)
    lay = kc.attn_layout(B, heads, Sq, d)
    w_lo = kc.assert_within(ctx.double() + lo.double(), fw["ctx"], fw["b_lo"], lay, "ctx + ctx_lo")
    with pytest.raises(AssertionError):          # ctx alone misses the 2^-16 bound
        kc.assert_within(ctx, fw["ctx"], fw["b_lo"], lay, "ctx without ctx_lo")
    with pytest.raises(AssertionError):          # and so does the low part with the wrong sign
        kc.assert_within(ctx.double() - lo.double(), fw["ctx"], fw["b_lo"], lay, "ctx - ctx_lo")
    sign = torch.where(fw["ctx"] >= ctx.double(), 1.0, -1.0)
    dctx = (sign * (1 + 0.5 * torch.rand(B * Sq, W, generator=g, device="cuda", dtype=torch.float64))).to(torch.bfloat16)
    dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, Sq, Skv, ctx_lo=lo)
    dq_nolo, _, _ = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, Sq, Skv)
    torch.cuda.synchronize()
    ref_lo = kc.attention_ref(q, k, v, B, heads, Sq, Skv, dctx=dctx, lo_used=True, p_exact=True)
    w = _check_all({"ctx": ctx, "lse2": lse2, "ctx_lo": lo, "dq": dq, "dk": dk, "dv": dv}, ref_lo, B, heads, Sq, Skv, d,
                   "exact-P Skv%d" % Skv)
    with pytest.raises(AssertionError):          # a delta without ctx_lo misses the bound that ctx_lo earns
        kc.assert_within(dq_nolo, ref_lo["dq"], ref_lo["b_dq"], lay, "dq, delta without ctx_lo")
    ref_nolo = kc.attention_ref(q, k, v, B, heads, Sq, Skv, dctx=dctx, lo_used=False, p_exact=True)
    w_nolo = kc.assert_within(dq_nolo, ref_nolo["dq"], ref_nolo["b_dq"], lay, "dq without ctx_lo, its own bound")
    print("attn exact-P Skv%d: ctx+lo=%.3f %s dq(no lo)=%.3f" % (Skv, w_lo, " ".join("%s=%.3f" % kv for kv in w.items()),
                                                                 w_nolo))
