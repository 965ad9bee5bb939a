"""Packed self-attention with a causal tail (mmfb_attention_varlen_causal_fwd / _bwd, M4C's prefix-LM mask on packed
rows): every element of ctx, lse2, dq, dk and dv of every sample against fp64 of the reference's own mask construction
(tests/test_attention_causal_gpu.py: each query row its own batch entry), with dropout fed the kernels' own keep bits;
each sample bit for bit against the dense causal kernels run on that sample alone; the argument refusals.

Sample b's tail is its last T rows, from P_b = max(len_b - T, 0) on, so alone it is the dense causal problem with B = 1,
S = len_b, no mask and causal_len = min(T, len_b): a sample shorter than T is all tail."""
import ctypes

import pytest
import torch

import kernel_check as kc
from test_attention_causal_gpu import per_query_reference, reference_mask

pytestmark = pytest.mark.gpu

LIMIT = {64: 384, 128: 256}


def lens_for(d, T):
    """0 (empty), the tail alone, a sample shorter than the tail, 64-row block edges, and max_len at the limit"""
    lens = [0, T, 63, 64, 65, 129, LIMIT[d]]
    if T > 1:
        lens.insert(2, T // 2)
    return lens


def run(lens, heads, d, T, p_drop, seed):
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(seed)
    max_len, total, W = max(lens), sum(lens), heads * d
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    qkv = (torch.randn(total, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    keep = dm = None
    if p_drop > 0:
        keep = torch.rand(heads, total, max_len, generator=g, device="cuda") >= p_drop
        dm = F.pack_keep_bits(keep)
    dsc = 1.0 / (1.0 - p_drop)
    nan = lambda: torch.full((total, W), float("nan"), device="cuda").to(torch.bfloat16)
    ctx, lse2, lo = F.attention_varlen_fwd(q, k, v, cu, max_len, heads, dm, dsc, out=nan(), save_lo=True, causal_len=T)
    dctx = torch.randn(total, W, generator=g, device="cuda").to(torch.bfloat16)
    dq, dk, dv = F.attention_varlen_bwd(dctx, q, k, v, ctx, lse2, cu, max_len, heads, dm, dsc, dq=nan(), dk=nan(), dv=nan(),
                                        ctx_lo=lo, causal_len=T)
    torch.cuda.synchronize()
    return dict(ctx=ctx, lse2=lse2, ctx_lo=lo, dq=dq, dk=dk, dv=dv), dict(q=q, k=k, v=v, keep=keep, dctx=dctx, p=p_drop,
                                                                           dsc=dsc)


def _samples(lens):
    s = 0
    for n in lens:
        yield s, s + n
        s += n


CASES = [(d, T) for d in (64, 128) for T in (1, 12, 30, 64, 65)]


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("d,T", CASES)
def test_varlen_causal_vs_fp64(d, T, p_drop):
    heads = 2
    lens = lens_for(d, T)
    out, a = run(lens, heads, d, T, p_drop, seed=d * 100 + T)
    worst = {}
    for s, e in _samples(lens):
        n = e - s
        if n == 0:
            continue
        Tb = min(T, n)
        mask3 = reference_mask(torch.ones(1, n - Tb, device="cuda"), Tb)
        keep = None if a["keep"] is None else a["keep"][:, s:e, :n].unsqueeze(0)
        ref = per_query_reference(a["q"][s:e], a["k"][s:e], a["v"][s:e], 1, heads, n, mask3, keep, a["p"], a["dctx"][s:e])
        lq, lk = kc.attn_layout(1, heads, n, d, "query"), kc.attn_layout(1, heads, n, d, "key")
        got = {"ctx": out["ctx"][s:e], "lse2": out["lse2"][:, s:e].unsqueeze(0), "dq": out["dq"][s:e], "dk": out["dk"][s:e],
               "dv": out["dv"][s:e]}
        for name, lay in (("ctx", lq), ("lse2", lq), ("dq", lq), ("dk", lk), ("dv", lk)):
            tag = "varlen causal d%d T%d p%.1f sample rows [%d, %d) %s" % (d, T, p_drop, s, e, name)
            w = kc.assert_within(got[name], ref[name], ref["b_" + name], lay, tag)
            worst[name] = max(worst.get(name, 0.0), w)
    print("attn varlen causal d%d T%d p%.1f: %s" % (d, T, p_drop, " ".join("%s=%.3f" % kv for kv in worst.items())))


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("d,T", CASES)
def test_each_sample_is_the_dense_causal_call_bit_for_bit(d, T, p_drop):
    """each packed sample equals mmfb_attention_fwd / _bwd on that sample alone (B = 1, S = len_b, no mask,
    causal_len = min(T, len_b)), with its keep bits moved into the dense layout [1, heads, len_b, ceil(len_b/32)]"""
    from mmf_b200 import functional as F
    heads = 2
    lens = lens_for(d, T)
    out, a = run(lens, heads, d, T, p_drop, seed=d * 100 + T + 1)
    for s, e in _samples(lens):
        n = e - s
        if n == 0:
            continue
        dm = None if a["keep"] is None else F.pack_keep_bits(a["keep"][:, s:e, :n].unsqueeze(0).contiguous())
        q, k, v = a["q"][s:e], a["k"][s:e], a["v"][s:e]
        ctx, lse2, lo = F.attention_fwd(q, k, v, 1, heads, n, n, None, dm, a["dsc"], save_lo=True, causal_len=min(T, n))
        dq, dk, dv = F.attention_bwd(a["dctx"][s:e], q, k, v, ctx, lse2, 1, heads, n, n, None, dm, a["dsc"], ctx_lo=lo,
                                     causal_len=min(T, n))
        torch.cuda.synchronize()
        tag = "d%d T%d p%.1f rows [%d, %d)" % (d, T, p_drop, s, e)
        assert torch.equal(out["ctx"][s:e], ctx), tag + " ctx"
        assert torch.equal(out["ctx_lo"][s:e], lo), tag + " ctx_lo"
        assert torch.equal(out["lse2"][:, s:e], lse2[0]), tag + " lse2"
        for name, t in (("dq", dq), ("dk", dk), ("dv", dv)):
            assert torch.equal(out[name][s:e], t), tag + " " + name


def test_refused_arguments_launch_nothing():
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    heads, d, lens = 2, 64, [20, 30]
    total, max_len, W = sum(lens), max(lens), heads * d
    t = torch.zeros(total, 3 * W, dtype=torch.bfloat16, device="cuda")
    q, k, v = t[:, :W], t[:, W:2 * W], t[:, 2 * W:]
    buf = torch.zeros(total, W, dtype=torch.bfloat16, device="cuda")
    stats = torch.zeros(2, heads, total, device="cuda")
    mask = torch.zeros(len(lens), max_len, device="cuda")
    cu = torch.tensor([0, 20, 50], dtype=torch.int32, device="cuda")
    stream = lib._stream_ptr()

    def args(T, Sq=max_len, with_mask=False):
        a, _, _ = F._varlen_args(q, k, v, cu, max_len, heads, None, 1.0, T)
        a.Sq = Sq
        a.ctx, a.ldo, a.lse2 = buf.data_ptr(), buf.stride(0), stats[0].data_ptr()
        a.dctx, a.ld_dctx, a.delta = buf.data_ptr(), buf.stride(0), stats[1].data_ptr()
        for n in ("dq", "dk", "dv"):
            setattr(a, n, buf.data_ptr())
            setattr(a, "ld_" + n, buf.stride(0))
        if with_mask:
            a.mask = mask.data_ptr()
        return a

    fwd, bwd = lib.LIB.mmfb_attention_varlen_causal_fwd, lib.LIB.mmfb_attention_varlen_causal_bwd
    calls = []
    for fn in (fwd, bwd):
        for T in (0, -1, max_len + 1):
            calls.append(("T=%d" % T, lambda a=args(T), fn=fn: fn(ctypes.byref(a), cu.data_ptr(), total, stream)))
        calls += [("Sq != Skv", lambda a=args(4, Sq=max_len - 1), fn=fn: fn(ctypes.byref(a), cu.data_ptr(), total, stream)),
                  ("mask", lambda a=args(4, with_mask=True), fn=fn: fn(ctypes.byref(a), cu.data_ptr(), total, stream)),
                  ("null cu", lambda a=args(4), fn=fn: fn(ctypes.byref(a), None, total, stream)),
                  ("negative total", lambda a=args(4), fn=fn: fn(ctypes.byref(a), cu.data_ptr(), -1, stream))]
    for what, call in calls:
        before = lib.launch_count()
        assert call() == lib.MMFB_ERR_ARG, what
        assert lib.launch_count() == before, what
    # total = 0: nothing to compute, no launch
    for fn in (fwd, bwd):
        before = lib.launch_count()
        assert fn(ctypes.byref(args(4)), cu.data_ptr(), 0, stream) == lib.MMFB_OK
        assert lib.launch_count() == before
    torch.cuda.synchronize()
