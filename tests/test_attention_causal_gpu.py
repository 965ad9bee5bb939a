"""Dense self-attention with a causal tail (causal_len, M4C's prefix-LM mask): every element of ctx, lse2, dq, dk and dv
against fp64 of the reference's own mask construction (mmf/models/m4c.py:427-437), through tests/kernel_check.py; the
argument refusals; causal_len = 0 as the call without a tail.

kernel_check.attention_ref takes a [B, Skv] key mask.  A per-query mask is the same computation with every query row as
its own batch entry (Sq = 1) over a copy of its sample's keys: ctx, lse2 and dq are that entry's, dk and dv the sum over
the entries of a sample, and so are their bounds (the sum of the per-entry bounds bounds the sum)."""
import ctypes

import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu


def reference_mask(enc_mask, T):
    """m4c.py:427-437: the [B, S, S] additive prefix-LM mask from the 0/1 mask of the encoding keys [B, S - T]"""
    B, P = enc_mask.shape
    S = P + T
    attention_mask = torch.cat([enc_mask.float(), torch.zeros(B, T, device=enc_mask.device)], dim=1)
    ext = attention_mask.unsqueeze(1).unsqueeze(2).repeat(1, 1, S, 1)
    causal = torch.zeros(T, T, device=enc_mask.device)
    for i in range(T):
        causal[i, :i + 1] = 1.0
    ext[:, :, -T:, -T:] = causal
    return ((1.0 - ext) * -10000.0)[:, 0]


def _enc_mask(B, P, seed):
    """0/1 encoding-key mask: sample 0 fully valid, sample 1 all padding (when B > 2), the others random prefixes"""
    g = torch.Generator().manual_seed(seed)
    m = torch.zeros(B, P)
    for b in range(B):
        n = P if b == 0 else (0 if b == 1 and B > 2 else int(torch.randint(0, P + 1, (1,), generator=g)))
        m[b, :n] = 1.0
    return m.cuda()


def run(B, heads, S, d, T, p_drop, seed):
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = heads * d
    qkv = (torch.randn(B * S, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    enc = _enc_mask(B, S - T, seed)
    mask = torch.cat([(1.0 - enc) * -10000.0, torch.full((B, T), float("nan"), device="cuda")], 1).contiguous()  # tail unread
    keep = dm = None
    if p_drop > 0:
        keep = torch.rand(B, heads, S, S, generator=g, device="cuda") >= p_drop
        dm = F.pack_keep_bits(keep)
    dsc = 1.0 / (1.0 - p_drop)
    ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, S, S, mask=mask, drop_mask=dm, drop_scale=dsc, save_lo=True,
                                    causal_len=T)
    dctx = torch.randn(B * S, W, generator=g, device="cuda").to(torch.bfloat16)
    dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, S, S, mask=mask, drop_mask=dm, drop_scale=dsc,
                                 ctx_lo=lo, causal_len=T)
    torch.cuda.synchronize()
    out = {"ctx": ctx, "lse2": lse2, "dq": dq, "dk": dk, "dv": dv}
    return out, (q, k, v, reference_mask(enc, T), keep, p_drop, dctx)


def per_query_reference(q, k, v, B, heads, S, mask3, keep, p_drop, dctx):
    """kc.attention_ref with each query row as its own batch entry"""
    W = q.shape[1]
    rows = torch.arange(B * S, device=q.device)
    b_of = rows // S
    kr = k.reshape(B, S, W)[b_of].reshape(B * S * S, W)
    vr = v.reshape(B, S, W)[b_of].reshape(B * S * S, W)
    keep_r = None if keep is None else keep.permute(0, 2, 1, 3).reshape(B * S, heads, 1, S)
    ref = kc.attention_ref(q, kr, vr, B * S, heads, 1, S, mask=mask3.reshape(B * S, S).contiguous(), keep=keep_r,
                           p_drop=p_drop, dctx=dctx, lo_used=True)
    out = {n: ref[n] for n in ("ctx", "b_ctx", "dq", "b_dq")}
    out["lse2"] = ref["lse2"].reshape(B, S, heads).permute(0, 2, 1)
    out["b_lse2"] = ref["b_lse2"].reshape(B, S, heads).permute(0, 2, 1)
    for n in ("dk", "b_dk", "dv", "b_dv"):
        out[n] = ref[n].reshape(B, S, S, W).sum(1).reshape(B * S, W)
    return out


def check(out, ref, B, heads, S, d, tag):
    lq = kc.attn_layout(B, heads, S, d, "query")
    lk = kc.attn_layout(B, heads, S, d, "key")
    worst = {}
    for name, lay in (("ctx", lq), ("lse2", lq), ("dq", lq), ("dk", lk), ("dv", lk)):
        worst[name] = kc.assert_within(out[name], ref[name], ref["b_" + name], lay, tag + " " + name)
    return worst


CASES = [(S, 64) for S in (13, 64, 65, 182, 200, 384)] + [(S, 128) for S in (13, 64, 65, 182, 200)]


@pytest.mark.parametrize("S,d", CASES)
def test_causal_tail_vs_fp64(S, d):
    B, heads = (3, 2) if S <= 200 else (3, 1)
    worst = {}
    for T in sorted({t for t in (1, 12, 30, 64, S) if t <= S}):
        for p_drop in (0.0, 0.1):
            out, (q, k, v, mask3, keep, p, dctx) = run(B, heads, S, d, T, p_drop, seed=S * 7 + T + d)
            for n in ("ctx", "lse2", "dq", "dk", "dv"):
                assert torch.isfinite(out[n].float()).all(), (n, S, T)
            ref = per_query_reference(q, k, v, B, heads, S, mask3, keep, p, dctx)
            w = check(out, ref, B, heads, S, d, "causal S%d d%d T%d p%.1f" % (S, d, T, p_drop))
            worst = {n: max(worst.get(n, 0.0), x) for n, x in w.items()}
    print("attn causal S%d d%d: %s" % (S, d, " ".join("%s=%.3f" % kv for kv in worst.items())))


def test_causal_len_zero_is_the_call_without_a_tail():
    from mmf_b200 import functional as F
    B, heads, S, d = 2, 3, 77, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = (torch.randn(B * S, 3 * heads * d, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    q, k, v = qkv[:, :heads * d], qkv[:, heads * d:2 * heads * d], qkv[:, 2 * heads * d:]
    mask = torch.where(torch.arange(S, device="cuda")[None] < torch.tensor([[S], [40]], device="cuda"), 0.0, -10000.0)
    dctx = torch.randn(B * S, heads * d, generator=g, device="cuda").to(torch.bfloat16)
    res = []
    for kw in ({}, {"causal_len": 0}):
        ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, S, S, mask=mask, save_lo=True, **kw)
        grads = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, S, S, mask=mask, ctx_lo=lo, **kw)
        res.append((ctx, lse2, lo) + tuple(grads))
    torch.cuda.synchronize()
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_refused_arguments_launch_nothing():
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    B, heads, S, d = 2, 2, 16, 64
    W = heads * d
    t = torch.zeros(B * S, 3 * W, dtype=torch.bfloat16, device="cuda")
    q, k, v = t[:, :W], t[:, W:2 * W], t[:, 2 * W:]
    out = torch.zeros(B * S, W, dtype=torch.bfloat16, device="cuda")
    lse2 = torch.zeros(B, heads, S, device="cuda")
    delta = torch.zeros(B, heads, S, device="cuda")
    cu = torch.tensor([0, S, 2 * S], dtype=torch.int32, device="cuda")
    probs = torch.zeros(B, heads, S, S, device="cuda")
    stream = lib._stream_ptr()

    def dense(causal_len, Sq=S, Skv=S):
        a = F._attn_args(q[:B * Sq], k[:B * Skv], v[:B * Skv], B, heads, Sq, Skv, None, None, 1.0, causal_len)
        a.ctx, a.ldo, a.lse2 = out.data_ptr(), out.stride(0), lse2.data_ptr()
        a.dctx, a.ld_dctx, a.delta = out.data_ptr(), out.stride(0), delta.data_ptr()
        for n in ("dq", "dk", "dv"):
            setattr(a, n, out.data_ptr())
            setattr(a, "ld_" + n, out.stride(0))
        return a

    calls = []
    for T in (-1, S + 1):
        calls += [("fwd T=%d" % T, lambda a=dense(T): lib.LIB.mmfb_attention_fwd(ctypes.byref(a), stream)),
                  ("bwd T=%d" % T, lambda a=dense(T): lib.LIB.mmfb_attention_bwd(ctypes.byref(a), stream))]
    calls += [("fwd Sq != Skv", lambda a=dense(2, Sq=8): lib.LIB.mmfb_attention_fwd(ctypes.byref(a), stream)),
              ("bwd Sq != Skv", lambda a=dense(2, Sq=8): lib.LIB.mmfb_attention_bwd(ctypes.byref(a), stream)),
              ("probs", lambda a=dense(2): lib.LIB.mmfb_attention_probs(ctypes.byref(a), probs.data_ptr(), 0, stream))]
    for name in ("mmfb_attention_varlen_fwd", "mmfb_attention_varlen_bwd"):
        calls.append((name, lambda a=dense(2), n=name: getattr(lib.LIB, n)(ctypes.byref(a), cu.data_ptr(), B * S, stream)))
    for name in ("mmfb_attention_varlen_cross_fwd", "mmfb_attention_varlen_cross_bwd"):
        calls.append((name, lambda a=dense(2), n=name: getattr(lib.LIB, n)(ctypes.byref(a), cu.data_ptr(), B * S,
                                                                         cu.data_ptr(), B * S, stream)))
    for what, call in calls:
        before = lib.launch_count()
        assert call() == lib.MMFB_ERR_ARG, what
        assert lib.launch_count() == before, what
        assert "causal" in lib.last_error(), (what, lib.last_error())
    torch.cuda.synchronize()
