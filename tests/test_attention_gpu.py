"""Fused attention (fwd + recompute bwd) vs the oracle's attention_core on the same bf16 inputs.
Tolerance: 1e-2 relative L2 (bf16 bar of BASELINE.md 5); the oracle runs in fp32 on the GPU."""
import pytest
import torch

from oracle import fusion_oracle as O

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


def _case(B, heads, Sq, Skv, d, p_drop=0.0, masked=True, seed=0, full_mask_row=False):
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = heads * d
    # fused projection buffers, q/k/v are column slices (as in the layer)
    if Sq == Skv:
        qkv = (torch.randn(B * Sq, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
        q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    else:
        q = (torch.randn(B * Sq, W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
        kv = (torch.randn(B * Skv, 2 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
        k, v = kv[:, :W], kv[:, W:]
    mask01 = torch.ones(B, Skv, dtype=torch.long, device="cuda")
    if masked:
        lens = torch.randint(max(1, Skv // 2), Skv + 1, (B,), generator=g, device="cuda")
        mask01 = (torch.arange(Skv, device="cuda")[None, :] < lens[:, None]).long()
        if full_mask_row:
            mask01[0] = 0
    add = ((1.0 - mask01.float()) * -10000.0).contiguous()
    keep = dm = None
    if p_drop > 0:
        keep = torch.rand(B, heads, Sq, Skv, generator=g, device="cuda") >= p_drop
        dm = F.pack_keep_bits(keep)
    scale = 1.0 / (1.0 - p_drop)
    ctx, lse2, ctx32 = F.attention_fwd(q, k, v, B, heads, Sq, Skv, mask=add, drop_mask=dm, drop_scale=scale,
                                       save_lo=True)
    assert ctx32.dtype == torch.bfloat16 and ctx32.abs().max() <= ctx.abs().max() * 2.0 ** -7   # the low part is a rounding residual
    dctx = (torch.randn(B * Sq, W, generator=g, device="cuda")).to(torch.bfloat16)
    dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, Sq, Skv, mask=add, drop_mask=dm,
                                 drop_scale=scale, ctx_lo=ctx32 if seed % 2 == 0 else None)
    torch.cuda.synchronize()
    # oracle (fp32, same bf16-rounded inputs)
    qf = q.float().view(B, Sq, W).clone().requires_grad_(True)
    kf = k.float().view(B, Skv, W).clone().requires_grad_(True)
    vf = v.float().view(B, Skv, W).clone().requires_grad_(True)
    ref, _ = O.attention_core(qf, kf, vf, add[:, None, None, :], heads, keep, p_drop)
    ref.backward(dctx.float().view(B, Sq, W))
    errs = {
        "ctx": rel(ctx.view(B, Sq, W), ref),
        "dq": rel(dq.view(B, Sq, W), qf.grad),
        "dk": rel(dk.view(B, Skv, W), kf.grad),
        "dv": rel(dv.view(B, Skv, W), vf.grad),
    }
    print("attn B%d h%d Sq%d Skv%d d%d p%.1f: %s" % (B, heads, Sq, Skv, d, p_drop,
                                                     " ".join("%s=%.2e" % kv_ for kv_ in errs.items())))
    assert torch.isfinite(ctx.float()).all()
    return errs


@pytest.mark.parametrize("B,heads,S,d", [(2, 12, 228, 64), (3, 4, 122, 64), (2, 2, 36, 64), (2, 12, 324, 64),
                                         (2, 8, 100, 128), (1, 16, 120, 64), (2, 2, 17, 64), (1, 1, 384, 64),
                                         (1, 2, 256, 128)])
def test_self_attention(B, heads, S, d):
    errs = _case(B, heads, S, S, d)
    assert max(errs.values()) < 1e-2


@pytest.mark.parametrize("B,heads,Sq,Skv,d", [(2, 8, 36, 36, 128), (2, 8, 36, 100, 128), (2, 8, 128, 36, 128),
                                              (2, 4, 200, 50, 64), (2, 4, 50, 300, 64)])
def test_cross_attention(B, heads, Sq, Skv, d):
    errs = _case(B, heads, Sq, Skv, d, seed=3)
    assert max(errs.values()) < 1e-2


def test_fully_masked_sample_is_finite():
    # additive -10000 on every key: fp32 does not absorb it, so the reference gives the softmax of the raw scores, never NaN
    errs = _case(2, 4, 40, 40, 64, full_mask_row=True, seed=5)
    assert max(errs.values()) < 1e-2


@pytest.mark.parametrize("S,d", [(228, 64), (36, 128), (300, 64)])
def test_attention_dropout_explicit_mask(S, d):
    errs = _case(2, 4, S, S, d, p_drop=0.1, seed=7)
    assert max(errs.values()) < 1e-2


@pytest.mark.parametrize("B,heads,Sq,Skv,p_drop", [(40, 12, 228, 228, 0.1), (70, 8, 100, 256, 0.0), (64, 6, 256, 36, 0.1),
                                                   (13, 12, 128, 128, 0.0)])
def test_attention_many_items_per_cta(B, heads, Sq, Skv, p_drop):
    """d = 64, many (batch, head) items of 64-row tiles: one to four blocks per side through the two-stage ring (odd and
    even counts), with ragged key padding and one sample without any attendable key"""
    errs = _case(B, heads, Sq, Skv, 64, p_drop=p_drop, seed=11, full_mask_row=True)
    assert max(errs.values()) < 1e-2


def test_attention_repeated_launches_are_identical_under_ragged_padding():
    """Race / hang regression for the staged rings (stage refills, barrier phases): 25 forward + backward launches over 1152
    items with ragged key padding.  Every repetition must reproduce the first one bit for bit, and none may trap."""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(21)
    B, heads, S, d = 96, 12, 228, 64
    W = heads * d
    qkv = (torch.randn(B * S, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    lens = torch.randint(20, S + 1, (B,), generator=g, device="cuda")
    add = ((torch.arange(S, device="cuda")[None, :] >= lens[:, None]).float() * -10000.0).contiguous()
    bits = F.dropout_bits((B, heads, S), S, 0.1, 3, 0, "cuda")
    dctx = torch.randn(B * S, W, generator=g, device="cuda").to(torch.bfloat16)
    first = None
    for rep in range(25):
        ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, S, S, mask=add, drop_mask=bits, drop_scale=1 / 0.9, save_lo=True)
        dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, S, S, mask=add, drop_mask=bits, drop_scale=1 / 0.9,
                                     ctx_lo=lo)
        torch.cuda.synchronize()
        cur = [ctx, lse2, lo, dq, dk, dv]
        if first is None:
            first = [t.clone() for t in cur]
            assert all(torch.isfinite(t.float()).all() for t in cur)
        else:
            for name, a, b in zip(("ctx", "lse2", "ctx_lo", "dq", "dk", "dv"), first, cur):
                assert torch.equal(a, b), (name, rep)


def test_attention_limits_raise():
    from mmf_b200 import functional as F
    q = torch.zeros(500, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        F.attention_fwd(q, q, q, 1, 1, 500, 500)
    with pytest.raises(ValueError):  # hidden not divisible by heads (vilbert.py:49-53)
        F.attention_fwd(q[:, :60], q[:, :60], q[:, :60], 1, 7, 500, 500)
