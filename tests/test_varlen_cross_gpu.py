"""Packed (variable-length) cross-attention and the two-stream skip-padding mode on the H100.

* kernels: every sample's ctx, lse2, ctx + ctx_lo, dq, dk and dv against fp64 on that sample's unpadded query and key
  slices (tests/kernel_check.py bounds), (q_len, kv_len) pairs at tile edges and the limit, one-sided empty samples, odd
  head counts, with and without keep bits, NaN-prefilled outputs;
* against the dense kernels (suffix padding, 0 / -10000 key mask, no dropout, zero dctx on padded query rows) and against
  packed self-attention (cu_kv = cu_q): bit-identical;
* encoders: ViLBERT at the bench widths and an LXMERT stack, skip vs dense against the fp32 oracle;
* model: the registered vilbert classification model with set_skip_padding(model, two_stream=True); stream capture."""
import os

import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens, dtype=torch.int64).cumsum(0).tolist(), dtype=torch.int32, device="cuda")


def _cross_case(lq, lk, heads, d, p_drop, seed):
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(seed)
    W, tq, tk = heads * d, sum(lq), sum(lk)
    max_q, max_kv = max(lq), max(lk)
    q = (torch.randn(tq, W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    kv = (torch.randn(tk, 2 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    k, v = kv[:, :W], kv[:, W:]
    keep = dm = None
    if p_drop > 0:
        keep = torch.rand(heads, tq, max_kv, generator=g, device="cuda") >= p_drop
        dm = F.pack_keep_bits(keep)
    dsc = 1.0 / (1.0 - p_drop)
    nan = lambda n: torch.full((n, W), float("nan"), device="cuda").to(torch.bfloat16)
    cq, ck = _cu(lq), _cu(lk)
    ctx, lse2, lo = F.attention_varlen_cross_fwd(q, k, v, cq, ck, max_q, max_kv, heads, dm, dsc, out=nan(tq), save_lo=True)
    dctx = torch.randn(tq, W, generator=g, device="cuda").to(torch.bfloat16)
    dq, dk, dv = F.attention_varlen_cross_bwd(dctx, q, k, v, ctx, lse2, cq, ck, max_q, max_kv, heads, dm, dsc, dq=nan(tq),
                                              dk=nan(tk), dv=nan(tk), ctx_lo=lo)
    torch.cuda.synchronize()
    return dict(ctx=ctx, lse2=lse2, ctx_lo=lo, dq=dq, dk=dk, dv=dv), dict(q=q, k=k, v=v, keep=keep, dctx=dctx, p=p_drop)


def _pairs(limit):
    return [(0, 0), (1, 0), (0, 1), (65, 0), (0, 129), (1, 1), (63, 64), (64, 65), (65, 63), (127, 129), (129, 127),
            (limit, limit), (1, limit), (limit, 1), (500, 65), (64, 0), (0, limit)]


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("d,heads", [(64, 3), (128, 3), (64, 12)])
def test_cross_kernels_vs_fp64(d, heads, p_drop):
    pairs = _pairs(384 if d == 64 else 256)
    lq, lk = [a for a, _ in pairs], [b for _, b in pairs]
    out, inp = _cross_case(lq, lk, heads, d, p_drop, seed=d + heads)
    for name in ("ctx", "ctx_lo", "dq", "dk", "dv"):
        assert torch.isfinite(out[name].float()).all(), "%s: a row was not written or is not finite" % name
    qs = ks = 0
    worst = {}
    for b, (nq, nk) in enumerate(pairs):
        qe, ke = qs + nq, ks + nk
        tag = "cross d%d h%d sample %d (q %d, kv %d)" % (d, heads, b, nq, nk)
        if nk == 0:       # queries without keys: zero rows, lse2 = -inf
            for name in ("ctx", "ctx_lo", "dq"):
                assert not out[name][qs:qe].any(), tag + " " + name
            assert (out["lse2"][:, qs:qe] == float("-inf")).all(), tag + " lse2"
        else:
            assert torch.isfinite(out["lse2"][:, qs:qe]).all(), tag + " lse2"
        if nq == 0:       # keys without queries: zero gradients
            assert not out["dk"][ks:ke].any() and not out["dv"][ks:ke].any(), tag + " dk/dv"
        if nq and nk:
            keep = inp["keep"][:, qs:qe, :nk].unsqueeze(0) if inp["keep"] is not None else None
            ref = kc.attention_ref(inp["q"][qs:qe], inp["k"][ks:ke], inp["v"][ks:ke], 1, heads, nq, nk, keep=keep,
                                   p_drop=inp["p"], dctx=inp["dctx"][qs:qe], lo_used=True)
            lq_, lk_ = kc.attn_layout(1, heads, nq, d, "query"), kc.attn_layout(1, heads, nk, d, "key")
            w = {"ctx": kc.assert_within(out["ctx"][qs:qe], ref["ctx"], ref["b_ctx"], lq_, tag + " ctx"),
                 "lse2": kc.assert_within(out["lse2"][:, qs:qe].unsqueeze(0), ref["lse2"], ref["b_lse2"], lq_, tag + " lse2"),
                 "ctx+lo": kc.assert_within(out["ctx"][qs:qe].double() + out["ctx_lo"][qs:qe].double(), ref["ctx"],
                                            ref["b_lo"], lq_, tag + " ctx+ctx_lo"),
                 "dq": kc.assert_within(out["dq"][qs:qe], ref["dq"], ref["b_dq"], lq_, tag + " dq"),
                 "dk": kc.assert_within(out["dk"][ks:ke], ref["dk"], ref["b_dk"], lk_, tag + " dk"),
                 "dv": kc.assert_within(out["dv"][ks:ke], ref["dv"], ref["b_dv"], lk_, tag + " dv")}
            worst = {k_: max(worst.get(k_, 0.0), v_) for k_, v_ in w.items()}
        qs, ks = qe, ke
    print("cross d%d h%d p%.1f: %s" % (d, heads, p_drop, " ".join("%s=%.3f" % kv for kv in worst.items())))


@pytest.mark.parametrize("d", [64, 128])
def test_cross_whole_side_empty(d):
    """no query row at all: the backward still writes dk = dv = 0; no key row at all: ctx = ctx_lo = dq = 0"""
    out, _ = _cross_case([0, 0, 0], [5, 70, 0], 3, d, 0.0, seed=1)
    assert out["ctx"].shape[0] == 0 and not out["dk"].any() and not out["dv"].any()
    out, _ = _cross_case([5, 0, 130], [0, 0, 0], 3, d, 0.0, seed=2)
    assert not out["ctx"].any() and not out["ctx_lo"].any() and not out["dq"].any()
    assert (out["lse2"] == float("-inf")).all() and out["dk"].shape[0] == 0


def test_cross_rejects_a_mask_and_bad_shapes():
    from mmf_b200 import functional as F, lib
    import ctypes
    q = torch.zeros(10, 64, device="cuda", dtype=torch.bfloat16)
    kv = torch.zeros(7, 128, device="cuda", dtype=torch.bfloat16)
    cq, ck = _cu([4, 6]), _cu([3, 4])
    with pytest.raises(ValueError):
        F.attention_varlen_cross_fwd(q, kv[:, :64], kv[:, 64:], cq.long(), ck, 6, 4, 1)
    with pytest.raises(ValueError):
        F.attention_varlen_cross_fwd(q, kv[:, :64], kv[:, 64:], cq, _cu([3, 2, 2]), 6, 4, 1)
    with pytest.raises(ValueError):
        F.attention_varlen_cross_fwd(q, kv[:6, :64], kv[:, 64:], cq, ck, 6, 4, 1)
    with pytest.raises(ValueError):
        F.attention_varlen_cross_fwd(q, kv[:, :64], kv[:, 64:], cq, ck, 6, 4, 1,
                                     drop_mask=torch.zeros(1, 7, 1, dtype=torch.int32, device="cuda"))
    a, tq, tk, _ = F._varlen_cross_args(q, kv[:, :64], kv[:, 64:], cq, ck, 6, 4, 1, None, 1.0)
    m = torch.zeros(2, 4, device="cuda")
    a.mask = m.data_ptr()
    assert lib.LIB.mmfb_attention_varlen_cross_fwd(ctypes.byref(a), cq.data_ptr(), tq, ck.data_ptr(), tk, None) == \
        lib.MMFB_ERR_ARG


@pytest.mark.parametrize("d,heads,lq,lk", [(64, 12, [36, 0, 20, 130, 65], [36, 18, 1, 384, 64]),
                                           (128, 3, [100, 64, 1, 300], [256, 129, 7, 63])])
def test_cross_bit_identical_to_dense(d, heads, lq, lk):
    """suffix padding on both sides, a 0 / -10000 key mask, no dropout, dctx zero on padded query rows: padded keys and
    queries contribute exact zeros in both paths and the 64-row blocks of the valid rows are the same"""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(11)
    B, Sq, Skv, W = len(lq), max(lq), max(lk), heads * d
    vq = torch.arange(Sq, device="cuda")[None, :] < torch.tensor(lq, device="cuda")[:, None]
    vk = torch.arange(Skv, device="cuda")[None, :] < torch.tensor(lk, device="cuda")[:, None]
    mask = torch.where(vk, 0.0, -10000.0).float().contiguous()
    q = (torch.randn(B * Sq, W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    kv = (torch.randn(B * Skv, 2 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    dctx = (torch.randn(B * Sq, W, generator=g, device="cuda") * vq.reshape(-1, 1)).to(torch.bfloat16)
    ctx, lse2, lo = F.attention_fwd(q, kv[:, :W], kv[:, W:], B, heads, Sq, Skv, mask, save_lo=True)
    dq, dk, dv = F.attention_bwd(dctx, q, kv[:, :W], kv[:, W:], ctx, lse2, B, heads, Sq, Skv, mask, ctx_lo=lo)
    rq, rk = vq.reshape(-1).nonzero().squeeze(1), vk.reshape(-1).nonzero().squeeze(1)
    pq, pkv = q.index_select(0, rq), kv.index_select(0, rk)
    cq, ck = _cu(lq), _cu(lk)
    pctx, plse2, plo = F.attention_varlen_cross_fwd(pq, pkv[:, :W], pkv[:, W:], cq, ck, Sq, Skv, heads, save_lo=True)
    pdq, pdk, pdv = F.attention_varlen_cross_bwd(dctx.index_select(0, rq), pq, pkv[:, :W], pkv[:, W:], pctx, plse2, cq, ck, Sq,
                                                 Skv, heads, ctx_lo=plo)
    torch.cuda.synchronize()
    assert torch.equal(pctx, ctx.index_select(0, rq))
    assert torch.equal(plo, lo.index_select(0, rq))
    assert torch.equal(plse2, lse2.permute(1, 0, 2).reshape(heads, B * Sq).index_select(1, rq))
    assert torch.equal(pdq, dq.index_select(0, rq))
    assert torch.equal(pdk, dk.index_select(0, rk)) and torch.equal(pdv, dv.index_select(0, rk))


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("d,heads,lens", [(64, 12, [0, 1, 63, 64, 65, 127, 129, 384, 0, 200]), (128, 3, [65, 0, 1, 256, 129])])
def test_cross_with_one_packing_is_packed_self_attention(d, heads, lens, p_drop):
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(5)
    total, W, S = sum(lens), heads * d, max(lens)
    cu = _cu(lens)
    qkv = (torch.randn(total, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    sl = (qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:])
    dm = F.pack_keep_bits(torch.rand(heads, total, S, generator=g, device="cuda") >= p_drop) if p_drop else None
    dsc = 1.0 / (1.0 - p_drop)
    dctx = torch.randn(total, W, generator=g, device="cuda").to(torch.bfloat16)
    a = F.attention_varlen_fwd(*sl, cu, S, heads, dm, dsc, save_lo=True)
    b = F.attention_varlen_cross_fwd(*sl, cu, cu, S, S, heads, dm, dsc, save_lo=True)
    ga = F.attention_varlen_bwd(dctx, *sl, a[0], a[1], cu, S, heads, dm, dsc, ctx_lo=a[2])
    gb = F.attention_varlen_cross_bwd(dctx, *sl, b[0], b[1], cu, cu, S, S, heads, dm, dsc, ctx_lo=b[2])
    torch.cuda.synchronize()
    for name, x, y in zip(("ctx", "lse2", "ctx_lo", "dq", "dk", "dv"), a + ga, b + gb):
        assert torch.equal(x, y), name


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _perturb(enc):
    with torch.no_grad():
        for p in enc.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return enc


def _valid(B, S, lo, g):
    """at least one token per sample (the first): a random length of at least `lo`, with holes (non-suffix padding)"""
    n = torch.randint(lo, S + 1, (B,), generator=g)
    v = (torch.arange(S)[None] < n[:, None]) & (torch.rand(B, S, generator=g) < 0.85)
    v[:, 0] = True
    return v.cuda()


def _add4(valid):
    return torch.where(valid, 0.0, -10000.0).float()[:, None, None, :]


def _assert_as_accurate(name, skip, dense):
    fmt = lambda e: " ".join("%s %.2e" % kv for kv in e.items())
    print("%s: dense vs fp32 oracle %s | skip vs fp32 oracle %s" % (name, fmt(dense), fmt(skip)))
    for k in dense:
        assert skip[k] <= 1.5 * dense[k] + 1e-3, "%s %s: skip-padding %.2e vs the dense path's %.2e" % (name, k, skip[k],
                                                                                                      dense[k])


def _vilbert_enc():
    import types
    from mmf_b200.modules import B200ViLBertEncoder
    c = dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12, v_hidden_size=1024,
             v_num_attention_heads=8, v_intermediate_size=1024, v_num_hidden_layers=6, bi_hidden_size=1024,
             bi_num_attention_heads=8, v_biattention_id=[0, 1, 2, 3, 4, 5], t_biattention_id=[6, 7, 8, 9, 10, 11])
    cfg = types.SimpleNamespace(hidden_dropout_prob=0.1, v_hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                                v_attention_probs_dropout_prob=0.1, **c)
    torch.manual_seed(0)
    return _perturb(B200ViLBertEncoder(cfg).cuda().eval()), c


@pytest.mark.parametrize("B,T,R", [(64, 36, 36), (8, 128, 100)])
def test_vilbert_encoder_skip_vs_dense_vs_oracle(B, T, R):
    from oracle import fusion_oracle as O
    enc, c = _vilbert_enc()
    g = torch.Generator().manual_seed(B + T)
    vt, vi = _valid(B, T, T // 2, g), _valid(B, R, R // 4, g)
    txt, img = torch.randn(B, T, 768, generator=g).cuda(), torch.randn(B, R, 1024, generator=g).cuda()
    wt, wi = torch.randn(B, T, 768, generator=g).cuda() * vt[..., None], torch.randn(B, R, 1024, generator=g).cuda() * vi[..., None]

    def run(pack):
        enc._runner.pack_streams = pack
        enc.zero_grad(set_to_none=True)
        t, i = txt.clone().requires_grad_(True), img.clone().requires_grad_(True)
        ot, oi, _ = enc(t, i, _add4(vt), None, _add4(vi), output_all_encoded_layers=False)
        ((ot[0] * wt).sum() + (oi[0] * wi).sum()).backward()
        torch.cuda.synchronize()
        return ot[0].detach(), oi[0].detach(), t.grad, i.grad, {k: p.grad.clone() for k, p in enc.named_parameters()
                                                                if p.grad is not None}
    dense, skip = run(False), run(True)
    assert not skip[0][~vt].any() and not skip[2][~vt].any() and not skip[1][~vi].any() and not skip[3][~vi].any()
    sd = {k: v.detach().to(torch.bfloat16).float().clone().requires_grad_(True) for k, v in enc.state_dict().items()}
    tf, vf = txt.to(torch.bfloat16).float().requires_grad_(True), img.to(torch.bfloat16).float().requires_grad_(True)
    to, vo = O.vilbert_encoder(tf, vf, _add4(vt), _add4(vi), sd, "", c)
    ((to * wt).sum() + (vo * wi).sum()).backward()

    def errs(r):
        ot, oi, dt, di, gr = r
        worst = max(rel(gr[k], sd[k].grad) for k in gr if gr[k].dim() == 2 and sd[k].grad is not None)
        return {"t_out": rel(ot[vt], to.detach()[vt]), "v_out": rel(oi[vi], vo.detach()[vi]), "dtxt": rel(dt, tf.grad),
                "dimg": rel(di, vf.grad), "grad": worst}
    _assert_as_accurate("vilbert 12t/6v/6c B%d T%d R%d" % (B, T, R), errs(skip), errs(dense))


def test_lxmert_encoder_skip_vs_dense_vs_oracle():
    import types
    from mmf_b200.lxmert import B200LXMERTEncoder
    from oracle import fusion_oracle as O
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, hidden_dropout_prob=0.1,
                                attention_probs_dropout_prob=0.1, visual_feat_dim=2048, visual_pos_dim=4, l_layers=3,
                                x_layers=3, r_layers=2)
    torch.manual_seed(1)
    enc = _perturb(B200LXMERTEncoder(cfg).cuda().eval())
    B, T, R = 16, 20, 100
    g = torch.Generator().manual_seed(7)
    vl, vv = _valid(B, T, 5, g), _valid(B, R, 10, g)
    lang = torch.randn(B, T, 768, generator=g).cuda()
    feats, boxes = torch.randn(B, R, 2048, generator=g).abs().cuda(), torch.rand(B, R, 4, generator=g).cuda()
    wl, wv = torch.randn(B, T, 768, generator=g).cuda() * vl[..., None], torch.randn(B, R, 768, generator=g).cuda() * vv[..., None]

    def run(pack):
        enc._runner.pack_streams = pack
        enc.zero_grad(set_to_none=True)
        l, f = lang.clone().requires_grad_(True), feats.clone().requires_grad_(True)
        lo, vo = enc(l, _add4(vl), (f, boxes), _add4(vv))
        ((lo * wl).sum() + (vo * wv).sum()).backward()
        torch.cuda.synchronize()
        return lo.detach(), vo.detach(), l.grad, f.grad, {k: p.grad.clone() for k, p in enc.named_parameters()
                                                          if p.grad is not None}
    dense, skip = run(False), run(True)
    assert not skip[0][~vl].any() and not skip[2][~vl].any() and not skip[1][~vv].any()
    sd = {k: v.detach().to(torch.bfloat16).float().clone().requires_grad_(True) for k, v in enc.state_dict().items()}
    lf, ff = lang.to(torch.bfloat16).float().requires_grad_(True), feats.to(torch.bfloat16).float().requires_grad_(True)
    lo, vo = O.lxmert_encoder(lf, _add4(vl), ff, boxes, _add4(vv), sd, "", 3, 3, 2, 12)
    ((lo * wl).sum() + (vo * wv).sum()).backward()

    def errs(r):
        ol, ov, dl, df, gr = r
        worst = max(rel(gr[k], sd[k].grad) for k in gr if gr[k].dim() == 2 and sd[k].grad is not None)
        return {"l_out": rel(ol[vl], lo.detach()[vl]), "v_out": rel(ov[vv], vo.detach()[vv]), "dlang": rel(dl, lf.grad),
                "dfeats": rel(df, ff.grad), "grad": worst}
    _assert_as_accurate("lxmert 3l/2r/3x B%d T%d R%d" % (B, T, R), errs(skip), errs(dense))


def test_vilbert_registered_model_two_stream_skip_padding():
    from mmf_b200 import functional as F, models as MD
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.sample import SampleList
    dev = torch.device("cuda", 0)
    g = torch.load(os.path.join(GOLD, "models.pt"), weights_only=False)
    c = g["vilbert_classification"]
    cfg = MD.load_model_config("vilbert", overrides=dict(c["config"]))
    cfg.losses = [{"type": "cross_entropy"}]
    model = MD.build_model(cfg)
    model.load_state_dict({k: v for k, v in c["state_dict"].items() if k in model.state_dict()})
    model = model.to(dev).eval()
    i, v = g["visual_bert_inputs"], g["vilbert_inputs"]
    calls = [0]
    cross = F.attention_varlen_cross_fwd

    def counted(*a, **k):
        calls[0] += 1
        return cross(*a, **k)

    def run():
        sl = SampleList(input_ids=i["ids"].to(dev), input_mask=i["mask"].to(dev), segment_ids=i["seg"].to(dev),
                        image_feature_0=i["feats"].to(dev), targets=i["targets"].to(dev), dataset_name="golden",
                        dataset_type="train", image_labels=v["image_labels"].to(dev),
                        image_info_0={"max_features": i["max_features"].to(dev), "bbox": v["bbox"].to(dev),
                                      "cls_prob": v["cls_prob"].numpy().copy()})
        model.zero_grad(set_to_none=True)
        out = model(sl)
        out["losses"]["train/golden/cross_entropy"].sum().backward()
        return out["scores"].detach(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    try:
        F.attention_varlen_cross_fwd = counted
        sd, gd = run()
        assert calls[0] == 0
        assert set_skip_padding(model, two_stream=True) >= 1
        sp, gp = run()
        assert calls[0] > 0                                 # the fixture pads both streams: the packed path ran
        worst = max(rel(gp[k], gd[k]) for k in gd if gd[k].norm() > 1e-6 and gd[k].dim() == 2)
        print("vilbert classification two-stream skip-padding vs dense: scores %.2e, worst 2-D param grad %.2e"
              % (rel(sp, sd), worst))
        assert rel(sp, sd) < 1e-2 and worst < 2e-2
        for m in model.modules():                           # a training step with dropout
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.1
        model.train()
        st, gt = run()
        assert torch.isfinite(st).all() and all(torch.isfinite(x).all() for x in gt.values())
    finally:
        F.attention_varlen_cross_fwd = cross
        set_skip_padding(model, False, two_stream=True)


def test_packed_two_stream_call_under_capture_raises():
    import types
    from mmf_b200.modules import B200ViLBertEncoder
    cfg = types.SimpleNamespace(hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=1,
                                v_hidden_size=64, v_num_attention_heads=1, v_intermediate_size=128, v_num_hidden_layers=1,
                                bi_hidden_size=64, bi_num_attention_heads=1, v_biattention_id=[0], t_biattention_id=[0],
                                hidden_dropout_prob=0.0, v_hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                v_attention_probs_dropout_prob=0.0, skip_padding=True)
    enc = B200ViLBertEncoder(cfg).cuda().eval()
    txt, img = torch.randn(2, 8, 64, device="cuda"), torch.randn(2, 5, 64, device="cuda")
    tm = torch.tensor([[0.0] * 8, [0.0] * 5 + [-10000.0] * 3], device="cuda")
    im = torch.zeros(2, 5, device="cuda")
    with torch.no_grad():
        enc(txt, img, tm, None, im, output_all_encoded_layers=False)        # lazy state outside the capture
    torch.cuda.synchronize()
    graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.no_grad(), pytest.raises(RuntimeError, match="pack_streams"):
        with torch.cuda.graph(graph, stream=s):
            enc(txt, img, tm, None, im, output_all_encoded_layers=False)
    torch.cuda.synchronize()
