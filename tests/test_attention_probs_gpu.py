"""The attention-probabilities kernel (mmfb_attention_probs) on the H100, and the encoders that return its output.

Kernel, element by element against fp64 (tests/kernel_check.py): P[b,h,q,k] = 2^(z - lse2) (* keep * dscale), computed
from the z the kernel stages (fp32 q.k accumulation, fmaf with the clamped mask) and the lse2 the forward saved.  Its
per-element bound (probs_ref below) is the backward's recomputed-p bound of kernel_check.attention_ref:
    |P - P64| <= Kp P ln2 (E + e_lse)  +  u_out Kp P  +  2^-126 Kp
E: exponent error of the staged score (fmaf and mask product 2^-23 (|z| + |m|), fp32 accumulation 2^-20 scale2 |q||k|,
ex2.approx 2^-22); e_lse: error of the forward's lse2 (kernel_check's b_lse2); u_out: output rounding, 2^-24 (fp32) or
2^-8 (bf16); 2^-126: the flush of p below fp32's normal range.  Sweeps sequence edges, far-from-square cross shapes, odd
head counts, mask kinds and keep bits, with output buffers prefilled with NaN between guard regions.  Then consistency
with the forward (row sums, P V against ctx + ctx_lo of the same call) and the encoders at full size against the fp32
oracle."""
import math

import pytest
import torch

import kernel_check as kc
from oracle import fusion_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def probs_layout(B, heads, Sq, Skv):
    """[B, heads, Sq, Skv]: (batch, head, query row and its 64-row tile, key and its 64-key block)"""
    def f(idx):
        b, h, q, k = idx
        return "batch %d, head %d, query row %d (query tile %d), key %d (key block %d)" % (b, h, q, q // 64, k, k // 64)
    return f


def probs_ref(q, k, B, heads, Sq, Skv, mask=None, keep=None, p_drop=0.0, out_dtype=torch.float32, clamp=True):
    """fp64 probabilities and their per-element bound (formula in the module docstring); clamp: the mask as the kernel
    stages it (clamped at -10000), else the original mask"""
    d = q.shape[1] // heads
    Q, K = kc._heads(q, B, Sq, heads, d), kc._heads(k, B, Skv, heads, d)
    scale2 = kc.LOG2E / math.sqrt(d)
    m2 = torch.zeros(B, 1, 1, Skv, dtype=torch.float64, device=Q.device)
    if mask is not None:
        m64 = mask.to(torch.float64)
        m2 = (m64.clamp_min(-10000.0) if clamp else m64).reshape(B, 1, 1, Skv) * kc.LOG2E
    Z = (Q @ K.transpose(-1, -2)) * scale2 + m2
    zmax = Z.amax(-1, keepdim=True)
    lse2 = zmax + torch.log2(torch.exp2(Z - zmax).sum(-1, keepdim=True))
    P = torch.exp2(Z - lse2)
    Kp = torch.ones_like(P) if keep is None else keep.to(torch.float64) / (1.0 - p_drop)
    E = 2.0 ** -23 * (Z.abs() + m2.abs()) + kc.U_ACC * scale2 * (Q.abs() @ K.abs().transpose(-1, -2)) + 2.0 ** -22
    E_max = torch.gather(E, -1, Z.argmax(-1, keepdim=True))
    e_lse = (P * E).sum(-1, keepdim=True) + E_max + 1.5 * (Skv / 4 + 2) * kc.U_F32 + 2.0 ** -20 + 2.0 ** -23 * lse2.abs()
    u_out = kc.U_F32 if out_dtype == torch.float32 else kc.U_BF16
    Pd = P * Kp
    # + kc.U_FTZ: ex2.approx.ftz stores a p below 2^-126 as 0
    bound = Pd * kc.LN2 * (E + e_lse) + u_out * Pd + kc.U_FTZ * Kp
    return Pd, bound, P, kc.LN2 * (E + e_lse) + u_out


def _inputs(B, heads, Sq, Skv, d, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    W = heads * d
    # head slices of fused [rows, 3W] projection buffers, as the engine passes them (row stride 3W)
    qb = (torch.randn(B * Sq, 3 * W, generator=g, device=DEV) * 1.5).to(torch.bfloat16)
    kb = (torch.randn(B * Skv, 3 * W, generator=g, device=DEV) * 1.5).to(torch.bfloat16)
    return qb[:, :W], kb[:, W:2 * W], kb[:, 2 * W:]


def _guarded(shape, dtype, guard):
    """a contiguous output view with NaN in it and `guard` NaN elements on each side"""
    n = math.prod(shape)
    buf = torch.full((n + 2 * guard,), float("nan"), dtype=dtype, device=DEV)
    return buf, buf[guard:guard + n].view(shape)


def _check(B, heads, Sq, Skv, d, mask=None, p_drop=0.0, out_dtype=torch.float32, guard=64, seed=0, ref_mask=None):
    from mmf_b200 import functional as F
    q, k, v = _inputs(B, heads, Sq, Skv, d, seed)
    bits, keep, scale = None, None, 1.0
    if p_drop > 0:
        g = torch.Generator(device=DEV).manual_seed(seed + 1)
        keep = torch.rand(B, heads, Sq, Skv, generator=g, device=DEV) >= p_drop
        bits, scale = F.pack_keep_bits(keep), 1.0 / (1.0 - p_drop)
    ctx, lse2, lo = F.attention_fwd(q, k, v, B, heads, Sq, Skv, mask, bits, scale, save_lo=True)
    buf, out = _guarded((B, heads, Sq, Skv), out_dtype, guard)
    got = F.attention_probs(q, k, lse2, B, heads, Sq, Skv, mask, bits, scale, dtype=out_dtype, out=out)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    n = out.numel()
    assert buf[:guard].isnan().all() and buf[guard + n:].isnan().all(), "the kernel wrote outside [B, heads, Sq, Skv]"
    assert torch.isfinite(out).all(), "an in-range element was not written (or is not finite)"
    Pd, bound, P, r = probs_ref(q, k, B, heads, Sq, Skv, ref_mask if ref_mask is not None else mask, keep, p_drop, out_dtype)
    worst = kc.assert_within(out, Pd, bound, probs_layout(B, heads, Sq, Skv), "probs")
    if keep is not None:
        assert (out[~keep] == 0).all(), "a dropped entry is not exactly 0"
    return worst, (q, k, v, ctx, lse2, lo, out, Pd, P, r, keep, scale)


EDGE = [1, 63, 64, 65, 127, 129]


@pytest.mark.parametrize("d", [64, 128])
def test_probs_kernel_sequence_edges(d):
    limit = 384 if d == 64 else 256
    worst = 0.0
    for Sq in EDGE + [limit]:
        for Skv in EDGE + [limit]:
            if (Sq, Skv) not in ((1, 1), (63, 65), (65, 63), (64, 64), (127, 129), (129, 127), (1, limit), (limit, 1),
                                 (limit, limit), (65, limit), (limit, 129), (63, 127)):
                continue
            w, _ = _check(2, 3, Sq, Skv, d, seed=Sq * 1000 + Skv)
            worst = max(worst, w)
    print("d=%d edges: worst |err|/bound %.3f" % (d, worst))


@pytest.mark.parametrize("d,heads", [(64, 5), (128, 3)])
def test_probs_kernel_cross_shapes_and_odd_heads(d, heads):
    worst = 0.0
    for Sq, Skv in ((2048, 64), (64, 256), (500, 37), (37, 129), (228, 228)):
        w, _ = _check(2, heads, Sq, Skv, d, seed=Sq + Skv)
        worst = max(worst, w)
    print("d=%d heads=%d cross: worst %.3f" % (d, heads, worst))


def _masks(B, Skv):
    lens = torch.tensor([Skv, max(1, Skv // 2), max(1, Skv - 3)][:B], device=DEV)
    pos = torch.arange(Skv, device=DEV)[None]
    suffix = torch.where(pos < lens[:, None], 0.0, -10000.0)
    left = torch.where(pos >= Skv - lens[:, None], 0.0, -10000.0)
    g = torch.Generator(device=DEV).manual_seed(3)
    soft = torch.randn(B, Skv, generator=g, device=DEV) * 2.0
    full = suffix.clone()
    full[-1] = -10000.0                                       # a fully masked sample
    return {"none": None, "suffix": suffix, "left": left, "soft": soft, "fully_masked_sample": full}


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kind", ["none", "suffix", "left", "soft", "fully_masked_sample"])
def test_probs_kernel_masks(d, kind):
    for Sq, Skv in ((65, 129), (1, 63), (130, 64)):
        m = _masks(3, Skv)[kind]
        m = m.contiguous() if m is not None else None
        _check(3, 2, Sq, Skv, d, mask=m, seed=11)


@pytest.mark.parametrize("low", [-1e9, float(torch.finfo(torch.bfloat16).min), float(torch.finfo(torch.float32).min),
                                 float("-inf")])
def test_probs_kernel_dtype_min_masks(low):
    """masks below -10000 act as -10000 (the staged clamp); a sample with an unmasked key matches fp64 computed with the
    ORIGINAL mask, and the fully masked sample gives the softmax of its raw scores"""
    B, Skv = 3, 100
    m = _masks(B, Skv)["left"]
    m = torch.where(m < 0, torch.full_like(m, low), m)
    m[2] = low                                                # fully masked
    w, st = _check(B, 2, 70, Skv, 64, mask=m.contiguous(), seed=5)
    out = st[6]
    # samples with an unmasked key: the original mask (exp of -inf / -1e38 is 0 in fp64 as well)
    m64 = m.double()
    orig = torch.where(torch.isinf(m64), torch.full_like(m64, -1e300), m64)[:2]
    q, k = st[0], st[1]
    Pd, bound, _, _ = probs_ref(q[:2 * 70], k[:2 * Skv], 2, 2, 70, Skv, orig, None, clamp=False)
    kc.assert_within(out[:2], Pd, bound, probs_layout(2, 2, 70, Skv), "probs vs original mask")
    assert torch.isfinite(out).all()


def test_probs_kernel_keep_bits_and_dtypes():
    worst = {}
    for out_dtype in (torch.float32, torch.bfloat16):
        for Skv in range(31, 66):
            w, _ = _check(2, 3, 67, Skv, 64, mask=_masks(2, Skv)["suffix"].contiguous(), p_drop=0.3, out_dtype=out_dtype,
                          seed=Skv)
            worst[out_dtype] = max(worst.get(out_dtype, 0.0), w)
        for d in (64, 128):
            for guard in (64, 3):                                 # 3: unaligned output, the scalar store path
                w, _ = _check(2, 3, 129, 127, d, p_drop=0.1, out_dtype=out_dtype, guard=guard, seed=d + guard)
                worst[out_dtype] = max(worst[out_dtype], w)
    print("keep bits: worst |err|/bound fp32 %.3f bf16 %.3f" % (worst[torch.float32], worst[torch.bfloat16]))


def test_rejects_bad_arguments_on_device():
    from mmf_b200 import functional as F
    q, k, v = _inputs(1, 2, 8, 8, 64, 0)
    _, lse2 = F.attention_fwd(q, k, v, 1, 2, 8, 8)
    with pytest.raises(ValueError, match="dtype"):
        F.attention_probs(q, k, lse2, 1, 2, 8, 8, dtype=torch.float16)
    q2, k2, _ = _inputs(1, 2, 8, 400, 64, 0)
    lse = torch.zeros(1, 2, 8, device=DEV)
    with pytest.raises(ValueError, match="limit"):
        F.attention_probs(q2, k2, lse, 1, 2, 8, 400)


# ---------------------------------------------------------------------------------------------------------------------
# consistency with the forward of the same call
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
def test_rows_sum_to_one_and_pv_matches_the_forward(d):
    worst_sum = worst_pv = 0.0
    for Sq, Skv, kind in ((129, 127, "suffix"), (64, 228 if d == 64 else 200, "left"), (300, 65, "soft")):
        m = _masks(2, Skv)[kind].contiguous()
        _, st = _check(2, 3, Sq, Skv, d, mask=m, seed=Sq)
        q, k, v, ctx, lse2, lo, out, Pd, P, r, keep, scale = st
        P64 = out.double()
        # rows sum to 1 within the sum of the per-element bounds (+ fp64 rounding)
        sb = (P * r).sum(-1) + 1e-12
        err = (P64.sum(-1) - 1.0).abs()
        worst_sum = max(worst_sum, (err / sb).max().item())
        assert (err <= kc.SAFETY * sb).all()
        # P V in fp64 against the forward's ctx + ctx_lo: the forward's own bound (b_lo) plus this P's error times |V|
        fw = kc.attention_ref(q, k, v, 2, 3, Sq, Skv, m.clamp_min(-10000.0))
        V = kc._heads(v, 2, Skv, 3, d)
        pv = kc._merge(P64 @ V)
        b = fw["b_lo"] + kc._merge((P * r) @ V.abs())
        worst_pv = max(worst_pv, kc.assert_within(pv, ctx.double() + lo.double(), b, kc.attn_layout(2, 3, Sq, d), "P V"))
    print("d=%d: row sums worst %.3f, P V vs ctx + ctx_lo worst %.3f of the bound" % (d, worst_sum, worst_pv))


# ---------------------------------------------------------------------------------------------------------------------
# encoders at full size
# ---------------------------------------------------------------------------------------------------------------------
def _bert_cfg(hidden, heads, inter, layers, p=0.0):
    import types
    return types.SimpleNamespace(hidden_size=hidden, num_attention_heads=heads, intermediate_size=inter,
                                 num_hidden_layers=layers, hidden_dropout_prob=p, attention_probs_dropout_prob=p,
                                 layer_norm_eps=1e-12, hidden_act="gelu", initializer_range=0.02)


def _perturb_1d(module):
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.02)


def _oracle_bert_probs(sd, x, add, L, heads, dtype):
    sdc = {k: v.detach().to(dtype) for k, v in sd.items()}
    h, probs = x.detach().to(dtype), []
    with torch.no_grad():
        for i in range(L):
            h, p = O.bert_layer(h, add.to(dtype), sdc, "layer.%d" % i, heads)
            probs.append(p.float())
    return h.float(), probs


def _launches():
    from mmf_b200 import lib
    torch.cuda.synchronize()
    return lib.launch_count()


def test_bert_encoder_12_layers_probs_vs_oracle_and_no_side_effects():
    from mmf_b200.modules import B200BertEncoder
    B, S, H, heads, L = 8, 228, 768, 12, 12
    torch.manual_seed(21)
    enc = B200BertEncoder(_bert_cfg(H, heads, 3072, L)).cuda().eval()
    _perturb_1d(enc)
    g = torch.Generator(device=DEV).manual_seed(22)
    x = torch.randn(B, S, H, generator=g, device=DEV)
    lens = torch.randint(S // 2, S + 1, (B,), generator=g, device=DEV)
    add = O.extended_attention_mask((torch.arange(S, device=DEV)[None] < lens[:, None]).long())
    w = torch.randn(B, S, H, generator=g, device=DEV)
    # eval + no_grad, the main use: one extra launch per layer, none without the flag
    with torch.no_grad():
        n0 = _launches()
        plain = enc(x, add)
        n1 = _launches()
        out = enc(x, add, output_attentions=True, output_hidden_states=True)
        n2 = _launches()
    assert (n2 - n1) - (n1 - n0) == L
    assert torch.equal(plain[0], out[0]) and len(out) == 3 and len(out[2]) == L
    sd = {k: v.to(torch.bfloat16).float() for k, v in enc.state_dict().items()}
    xr = x.to(torch.bfloat16).float()
    _, ref32 = _oracle_bert_probs(sd, xr, add, L, heads, torch.float32)
    _, ref16 = _oracle_bert_probs(sd, xr, add, L, heads, torch.bfloat16)
    errs, errs16 = [rel(a, r) for a, r in zip(out[2], ref32)], [rel(a, r) for a, r in zip(ref16, ref32)]
    print("12L/768 B=8 S=228 probs vs fp32 oracle per layer: %s | bf16 reference: %s" % (
        " ".join("%.1e" % e for e in errs), " ".join("%.1e" % e for e in errs16)))
    assert errs[0] < 1e-2                                       # layer 0: the per-kernel bf16 bar (BASELINE.md 5)
    for e, e16 in zip(errs, errs16):
        assert e <= max(1.5 * e16, 1e-2) and e < 2.5e-2
    for a in out[2]:
        assert a.shape == (B, heads, S, S) and a.dtype == torch.float32 and torch.isfinite(a).all()
    # training: outputs and the input gradient bit-identical with the flag on and off.  The weight gradients accumulate
    # split-K partial sums with fp32 atomics, whose order varies from run to run with or without the flag: they must agree
    # to that rounding (two flag-off runs are compared the same way and printed)
    enc.train()
    for p in (enc.layer[0].attention.self.dropout, enc.layer[0].attention.output.dropout):
        p.p = 0.1
    res = []
    for flag in (False, False, True):
        import mmf_b200.modules as MM
        MM._SEED_COUNTER[0] = 0
        xi = x.clone().requires_grad_(True)
        enc.zero_grad(set_to_none=True)
        o = enc(xi, add, output_attentions=flag)
        (o[0] * w).sum().backward()
        res.append((o, xi.grad.clone(), {k: p.grad.clone() for k, p in enc.named_parameters() if p.grad is not None}))
    (o0, d0, g0), (oo, do, go), (o1, d1, g1) = res
    assert torch.equal(o0[0], o1[0]) and torch.equal(d0, d1) and torch.equal(o0[0], oo[0]) and torch.equal(d0, do)
    assert g0.keys() == g1.keys() == go.keys()
    noise = max(rel(go[k], g0[k]) for k in g0)
    flag = max(rel(g1[k], g0[k]) for k in g0)
    print("weight gradients, max rel difference: flag off vs off %.1e, flag on vs off %.1e" % (noise, flag))
    assert flag < 1e-5
    a0 = o1[1][0]                                              # layer 0 with attention dropout: exact zeros, finite
    assert torch.isfinite(a0).all() and (a0 == 0).float().mean().item() > 0.05


def test_skip_padding_fallback_equals_dense_and_bf16_output():
    from mmf_b200.modules import B200BertEncoder
    B, S, H = 4, 100, 256
    torch.manual_seed(23)
    enc = B200BertEncoder(_bert_cfg(H, 4, 512, 2)).cuda().eval()
    x = torch.randn(B, S, H, device=DEV)
    add = O.extended_attention_mask((torch.arange(S, device=DEV)[None] < torch.tensor([S, 60, 33, 90], device=DEV)[:, None]).long())
    with torch.no_grad():
        dense = enc(x, add, output_attentions=True)
        enc._runner.skip_padding = True
        packed = enc(x, add, output_attentions=True)
        b16 = enc(x.to(torch.bfloat16), add, output_attentions=True)
    assert torch.equal(dense[0], packed[0]) and all(torch.equal(a, b) for a, b in zip(dense[1], packed[1]))
    assert all(a.dtype == torch.bfloat16 for a in b16[1])
    assert all(rel(a, b) < 1e-2 for a, b in zip(b16[1], dense[1]))


def test_vit_encoder_returns_attentions():
    import types
    from mmf_b200.vit import B200ViTEncoder
    cfg = types.SimpleNamespace(hidden_size=768, num_hidden_layers=4, num_attention_heads=12, intermediate_size=3072,
                                hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                                hidden_act="gelu", initializer_range=0.02)
    torch.manual_seed(24)
    enc = B200ViTEncoder(cfg).cuda().eval()
    x = torch.randn(4, 197, 768, device=DEV)
    with torch.no_grad():
        out = enc(x, output_attentions=True, output_hidden_states=True)
    assert len(out.attentions) == 4 and all(a.shape == (4, 12, 197, 197) for a in out.attentions)
    sd = {k: v.to(torch.bfloat16).float() for k, v in enc.state_dict().items()}
    # the layer-0 probabilities against the oracle's pre-LN attention on the same input
    a = O.layer_norm(x.to(torch.bfloat16).float(), sd, "layer.0.layernorm_before")
    _, p0 = O.bert_self_attention(a, None, sd, "layer.0.attention.attention", 12)
    assert rel(out.attentions[0], p0) < 1e-2
    assert torch.allclose(out.attentions[-1].double().sum(-1), torch.ones(4, 12, 197, dtype=torch.float64, device=DEV),
                          atol=1e-4)


def _vilbert_cfg(visualization):
    import types
    return types.SimpleNamespace(
        hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12,
        v_hidden_size=1024, v_num_attention_heads=8, v_intermediate_size=1024, v_num_hidden_layers=6,
        bi_hidden_size=1024, bi_num_attention_heads=8, v_biattention_id=[0, 1, 2, 3, 4, 5],
        t_biattention_id=[6, 7, 8, 9, 10, 11], hidden_dropout_prob=0.0, v_hidden_dropout_prob=0.0,
        attention_probs_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0, initializer_range=0.02,
        visualization=visualization)


def _oracle_vilbert_probs(sd, txt, img, tmask, imask, cfg, dtype):
    """the oracle's ViLBERT schedule with every attention's probabilities (text, image, co-attention pairs)"""
    sdc = {k: v.detach().to(dtype) for k, v in sd.items()}
    t, i = txt.to(dtype), img.to(dtype)
    tm, im = tmask.to(dtype), imask.to(dtype)
    at, av, ac = [], [], []
    with torch.no_grad():
        for kind, j in O.vilbert_schedule(cfg.v_biattention_id, cfg.t_biattention_id, cfg.num_hidden_layers,
                                          cfg.v_num_hidden_layers):
            if kind == "t":
                t, p = O.bert_layer(t, tm, sdc, "layer.%d" % j, cfg.num_attention_heads)
                at.append(p.float())
            elif kind == "v":
                i, p = O.bert_layer(i, im, sdc, "v_layer.%d" % j, cfg.v_num_attention_heads)
                av.append(p.float())
            else:
                pre = "c_layer.%d.biattention" % j
                q2, k1, v1 = (O.linear(t if n[-1] == "2" else i, sdc, pre + "." + n) for n in ("query2", "key1", "value1"))
                q1, k2, v2 = (O.linear(i if n[-1] == "1" else t, sdc, pre + "." + n) for n in ("query1", "key2", "value2"))
                _, p1 = O.attention_core(q2, k1, v1, im, cfg.bi_num_attention_heads)
                _, p2 = O.attention_core(q1, k2, v2, tm, cfg.bi_num_attention_heads)
                ac.append((p1.float(), p2.float()))
                i, t = O.connection_layer(i, im, t, tm, sdc, "c_layer.%d" % j, cfg.bi_num_attention_heads)
    return at, av, ac


def test_vilbert_12_6_6_visualization_vs_oracle():
    from mmf_b200.modules import B200ViLBertEncoder
    cfg = _vilbert_cfg(True)
    torch.manual_seed(25)
    enc = B200ViLBertEncoder(cfg).cuda().eval()
    _perturb_1d(enc)
    B, T, R = 4, 36, 101
    g = torch.Generator(device=DEV).manual_seed(26)
    txt = torch.randn(B, T, 768, generator=g, device=DEV)
    img = torch.randn(B, R, 1024, generator=g, device=DEV)
    tm = O.extended_attention_mask((torch.arange(T, device=DEV)[None] < torch.tensor([T, 20, 9, 30], device=DEV)[:, None]).long())
    im = O.extended_attention_mask((torch.arange(R, device=DEV)[None] < torch.tensor([R, 50, 77, 11], device=DEV)[:, None]).long())
    with torch.no_grad():
        n0 = _launches()
        plain = enc(txt, img, tm, tm, im, None, output_all_encoded_layers=False, output_all_attention_masks=False)
        n1 = _launches()
        out = enc(txt, img, tm, tm, im, None, output_all_encoded_layers=False, output_all_attention_masks=True)
        n2 = _launches()
        enc.config.visualization = False
        empty = enc(txt, img, tm, tm, im, None, output_all_encoded_layers=False, output_all_attention_masks=True)
        n3 = _launches()
        enc.config.visualization = True
    assert (n2 - n1) - (n1 - n0) == 12 + 6 + 2 * 6 and (n3 - n2) == (n1 - n0)
    assert empty[2] == ([], [], []) and torch.equal(empty[0][0], plain[0][0])
    assert torch.equal(plain[0][0], out[0][0]) and torch.equal(plain[1][0], out[1][0])
    gt, gv, gc = out[2]
    assert len(gt) == 12 and len(gv) == 6 and len(gc) == 6
    sd = {k: v.to(torch.bfloat16).float() for k, v in enc.state_dict().items()}
    t32, v32, c32 = _oracle_vilbert_probs(sd, txt.to(torch.bfloat16).float(), img.to(torch.bfloat16).float(), tm, im, cfg,
                                          torch.float32)
    t16, v16, c16 = _oracle_vilbert_probs(sd, txt.to(torch.bfloat16).float(), img.to(torch.bfloat16).float(), tm, im, cfg,
                                          torch.bfloat16)
    pairs = list(zip(gt, t32, t16)) + list(zip(gv, v32, v16))
    for (a1, a2), (r1, r2), (s1, s2) in zip(gc, c32, c16):
        assert a1.shape == (B, 8, T, R) and a2.shape == (B, 8, R, T)
        pairs += [(a1, r1, s1), (a2, r2, s2)]
    errs = [(rel(a, r), rel(s, r)) for a, r, s in pairs]
    print("ViLBERT 12+6+6 probs vs fp32 oracle (ours / bf16 reference): %s" % " ".join("%.1e/%.1e" % e for e in errs))
    for e, e16 in errs:
        assert e <= max(1.5 * e16, 1e-2) and e < 2.5e-2
