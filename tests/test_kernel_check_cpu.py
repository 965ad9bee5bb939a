"""The per-element check of tests/kernel_check.py catches the local errors that a whole-tensor relative L2 < 1e-2 lets
through.  Runs on the CPU: a bf16-rounded fp64 reference stands for a correct kernel and must pass; each mutation
stands for one kind of kernel bug and must fail."""
import math

import pytest
import torch

import kernel_check as kc


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _bf16(*shape, gen, scale=1.0):
    return (torch.randn(*shape, generator=gen, dtype=torch.float64) * scale).to(torch.bfloat16)


def test_gemm_tile_missing_its_last_k_block():
    g = torch.Generator().manual_seed(1)
    M, N, K, BN = 2560, 2560, 3072, 128
    a, b = _bf16(M, K, gen=g, scale=0.5), _bf16(N, K, gen=g, scale=0.5)
    ref, absab = kc.gemm_ref(a, b)
    bound = kc.gemm_bound(ref, absab)
    lay = kc.gemm_layout(BN)
    good = kc.bf16_round(ref)
    kc.assert_within(good, ref, bound, lay)
    # m-tile 7, n-tile 11 summed k-blocks 0 .. 46 of 48 only
    bad = good.clone()
    r0, c0 = 7 * 128, 11 * BN
    a64, b64 = a[r0:r0 + 128].double(), b[c0:c0 + BN].double()
    bad[r0:r0 + 128, c0:c0 + BN] = kc.bf16_round(a64[:, :K - 64] @ b64[:, :K - 64].t())
    assert rel(bad, ref) < 1e-2                      # the whole-tensor metric misses it
    with pytest.raises(AssertionError, match=r"m-tile 7, n-tile 11"):
        kc.assert_within(bad, ref, bound, lay)


def _attn_inputs(B, heads, S, d, g):
    W = heads * d
    qkv = _bf16(B * S, 3 * W, gen=g, scale=0.8)
    return qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]


def test_attention_row_of_the_partial_tile_missing_one_key():
    g = torch.Generator().manual_seed(2)
    B, heads, S, d = 16, 12, 129, 64                 # query row 128 is alone in the last, partial 64-row tile
    q, k, v = _attn_inputs(B, heads, S, d, g)
    b0, h0, r0 = 9, 5, 128
    k = k.clone()
    # give the last key a visible weight in that row (about 0.1), as a real input may
    kcol = slice(h0 * d, (h0 + 1) * d)
    k[b0 * S + S - 1, kcol] = (q[b0 * S + r0, kcol].double() * 0.5).to(torch.bfloat16)
    ref = kc.attention_ref(q, k, v, B, heads, S, S)
    lay = kc.attn_layout(B, heads, S, d)
    good = kc.bf16_round(ref["ctx"])
    kc.assert_within(good, ref["ctx"], ref["b_ctx"], lay)
    # the row recomputed over keys 0 .. S-2
    qr = q[b0 * S + r0, kcol].double()
    kk, vv = k[b0 * S:(b0 + 1) * S - 1, kcol].double(), v[b0 * S:(b0 + 1) * S - 1, kcol].double()
    p = torch.softmax(kk @ qr / math.sqrt(d), 0)
    bad = good.clone()
    bad[b0 * S + r0, kcol] = kc.bf16_round(p @ vv)
    assert rel(bad, ref["ctx"]) < 1e-2
    with pytest.raises(AssertionError, match=r"batch 9, head 5, query row 128 \(query block 2\)"):
        kc.assert_within(bad, ref["ctx"], ref["b_ctx"], lay)


def test_attention_head_replaced_by_its_neighbour():
    g = torch.Generator().manual_seed(3)
    B, heads, S, d = 2, 4, 40, 64
    q, k, v = _attn_inputs(B, heads, S, d, g)
    ref = kc.attention_ref(q, k, v, B, heads, S, S)
    bad = kc.bf16_round(ref["ctx"])
    bad[S:2 * S, 2 * d:3 * d] = bad[S:2 * S, 3 * d:4 * d]          # batch 1: head 2 <- head 3
    with pytest.raises(AssertionError, match=r"batch 1, head 2"):
        kc.assert_within(bad, ref["ctx"], ref["b_ctx"], kc.attn_layout(B, heads, S, d))


def test_gemm_column_pair_swapped():
    g = torch.Generator().manual_seed(4)
    M, N, K = 300, 264, 72
    a, b = _bf16(M, K, gen=g), _bf16(N, K, gen=g)
    ref, absab = kc.gemm_ref(a, b)
    bad = kc.bf16_round(ref)
    bad[:, [130, 131]] = bad[:, [131, 130]]                          # one bf16x2 pair stored the wrong way round
    with pytest.raises(AssertionError, match=r"n-tile 1"):
        kc.assert_within(bad, ref, kc.gemm_bound(ref, absab), kc.gemm_layout(128))


def test_layernorm_row_with_rstd_off_by_one_percent():
    g = torch.Generator().manual_seed(5)
    M, H = 257, 776
    y = _bf16(M, H, gen=g)
    gam = (1 + 0.1 * torch.randn(H, generator=g, dtype=torch.float64)).to(torch.bfloat16)
    bet = (0.1 * torch.randn(H, generator=g, dtype=torch.float64)).to(torch.bfloat16)
    fw = kc.layernorm_ref(y, gam, bet)
    lay = kc.row_layout()
    kc.assert_within(fw["rstd"].float(), fw["rstd"], fw["b_rstd"], lay, "rstd")
    kc.assert_within(kc.bf16_round(fw["x"]), fw["x"], fw["b_x"], lay, "x")
    rs_bad = fw["rstd"].float().clone()
    rs_bad[100] *= 1.01
    with pytest.raises(AssertionError, match=r"index 100"):
        kc.assert_within(rs_bad, fw["rstd"], fw["b_rstd"], lay, "rstd")
    # the same error carried into the row's output: x of row 100 computed with that rstd
    y64 = y.double()
    x_bad = kc.bf16_round(fw["x"])
    x_bad[100] = kc.bf16_round((y64[100] - fw["mean"][100]) * fw["rstd"][100] * 1.01 * gam.double() + bet.double())
    assert rel(x_bad, fw["x"]) < 1e-2
    with pytest.raises(AssertionError, match=r"row 100"):
        kc.assert_within(x_bad, fw["x"], fw["b_x"], lay, "x")


def test_non_finite_output_always_fails():
    ref = torch.ones(4, 8, dtype=torch.float64)
    out = ref.clone()
    out[2, 3] = float("nan")
    with pytest.raises(AssertionError, match=r"row 2"):
        kc.assert_within(out, ref, torch.ones_like(ref), kc.row_layout())
