"""Packed (variable-length) self-attention and the skip-padding encoder mode on the H100.

* kernels: every sample's ctx, lse2, ctx + ctx_lo, dq, dk and dv against fp64 on that sample's unpadded slice
  (tests/kernel_check.py bounds), lengths 0 / 1 / tile edges / the limit, odd head counts, with and without keep bits;
* against the dense kernels: suffix padding, no dropout, zero dctx on padded rows -> bit-identical at valid rows;
* encoder: 12 L / 768 skip-padding vs dense for a loss restricted to valid rows, exact zeros at padded positions;
* model: the registered visual_bert pretraining model with set_skip_padding on and off."""
import os

import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _packed_case(lens, heads, d, p_drop, seed):
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
    ctx, lse2, lo = F.attention_varlen_fwd(q, k, v, cu, max_len, heads, dm, dsc, out=nan(), save_lo=True)
    dctx = torch.randn(total, W, generator=g, device="cuda").to(torch.bfloat16)
    dq, dk, dv = F.attention_varlen_bwd(dctx, q, k, v, ctx, lse2, cu, max_len, heads, dm, dsc, dq=nan(), dk=nan(), dv=nan(),
                                        ctx_lo=lo)
    torch.cuda.synchronize()
    return dict(ctx=ctx, lse2=lse2, ctx_lo=lo, dq=dq, dk=dk, dv=dv), dict(q=q, k=k, v=v, keep=keep, dctx=dctx, p=p_drop)


LENS = {64: [0, 1, 63, 64, 65, 127, 129, 384, 0, 200], 128: [65, 0, 1, 63, 64, 256, 127, 129]}


@pytest.mark.parametrize("p_drop", [0.0, 0.1])
@pytest.mark.parametrize("d,heads", [(64, 3), (128, 3), (64, 12)])
def test_varlen_kernels_vs_fp64(d, heads, p_drop):
    lens = LENS[d]
    out, inp = _packed_case(lens, heads, d, p_drop, seed=d + heads)
    for name in ("ctx", "lse2", "ctx_lo", "dq", "dk", "dv"):
        assert torch.isfinite(out[name].float()).all(), "%s: a row of [0, total) was not written or is not finite" % name
    s = 0
    worst = {}
    for b, n in enumerate(lens):
        e = s + n
        if n == 0:
            continue
        keep = inp["keep"][:, s:e, :n].unsqueeze(0) if inp["keep"] is not None else None
        ref = kc.attention_ref(inp["q"][s:e], inp["k"][s:e], inp["v"][s:e], 1, heads, n, n, keep=keep, p_drop=inp["p"],
                               dctx=inp["dctx"][s:e], lo_used=True)
        lq, lk = kc.attn_layout(1, heads, n, d, "query"), kc.attn_layout(1, heads, n, d, "key")
        tag = "varlen d%d h%d sample %d (len %d)" % (d, heads, b, n)
        w = {"ctx": kc.assert_within(out["ctx"][s:e], ref["ctx"], ref["b_ctx"], lq, tag + " ctx"),
             "lse2": kc.assert_within(out["lse2"][:, s:e].unsqueeze(0), ref["lse2"], ref["b_lse2"], lq, tag + " lse2"),
             "ctx+lo": kc.assert_within(out["ctx"][s:e].double() + out["ctx_lo"][s:e].double(), ref["ctx"], ref["b_lo"], lq,
                                        tag + " ctx+ctx_lo"),
             "dq": kc.assert_within(out["dq"][s:e], ref["dq"], ref["b_dq"], lq, tag + " dq"),
             "dk": kc.assert_within(out["dk"][s:e], ref["dk"], ref["b_dk"], lk, tag + " dk"),
             "dv": kc.assert_within(out["dv"][s:e], ref["dv"], ref["b_dv"], lk, tag + " dv")}
        worst = {k_: max(worst.get(k_, 0.0), v_) for k_, v_ in w.items()}
        s = e
    print("varlen d%d h%d p%.1f: %s" % (d, heads, p_drop, " ".join("%s=%.3f" % kv for kv in worst.items())))


def test_varlen_rejects_a_mask_and_bad_shapes():
    from mmf_b200 import functional as F, lib
    import ctypes
    qkv = torch.zeros(10, 3 * 64, device="cuda", dtype=torch.bfloat16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        F.attention_varlen_fwd(qkv[:, :64], qkv[:, 64:128], qkv[:, 128:], cu.long(), 6, 1)
    with pytest.raises(ValueError):
        F.attention_varlen_fwd(qkv[:, :64], qkv[:9, 64:128], qkv[:, 128:], cu, 6, 1)
    with pytest.raises(ValueError):
        F.attention_varlen_fwd(qkv[:, :64], qkv[:, 64:128], qkv[:, 128:], cu, 6, 1,
                               drop_mask=torch.zeros(1, 10, 2, dtype=torch.int32, device="cuda"))
    a, total, _ = F._varlen_args(qkv[:, :64], qkv[:, 64:128], qkv[:, 128:], cu, 6, 1, None, 1.0)
    m = torch.zeros(2, 6, device="cuda")
    a.mask = m.data_ptr()
    assert lib.LIB.mmfb_attention_varlen_fwd(ctypes.byref(a), cu.data_ptr(), total, None) == lib.MMFB_ERR_ARG


@pytest.mark.parametrize("d,heads,lens", [(64, 12, [228, 1, 100, 150, 65]), (128, 3, [256, 64, 129, 7])])
def test_varlen_bit_identical_to_dense(d, heads, lens):
    """suffix padding with a 0 / -10000 mask, no dropout, dctx zero on padded rows: padded keys contribute exact zeros in
    both paths and the 64-key blocks of the valid keys are the same, so valid rows match bit for bit"""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(7)
    B, S, W = len(lens), max(lens), heads * d
    valid = torch.arange(S, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
    mask = torch.where(valid, 0.0, -10000.0).float().contiguous()
    qkv = (torch.randn(B * S, 3 * W, generator=g, device="cuda") * 0.8).to(torch.bfloat16)
    dctx = (torch.randn(B * S, W, generator=g, device="cuda") * valid.reshape(-1, 1)).to(torch.bfloat16)
    sl = lambda t: (t[:, :W], t[:, W:2 * W], t[:, 2 * W:])
    ctx, lse2, lo = F.attention_fwd(*sl(qkv), B, heads, S, S, mask, save_lo=True)
    dq, dk, dv = F.attention_bwd(dctx, *sl(qkv), ctx, lse2, B, heads, S, S, mask, ctx_lo=lo)
    rows = valid.reshape(-1).nonzero().squeeze(1)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    pq = qkv.index_select(0, rows)
    pctx, plse2, plo = F.attention_varlen_fwd(*sl(pq), cu, S, heads, save_lo=True)
    pdq, pdk, pdv = F.attention_varlen_bwd(dctx.index_select(0, rows), *sl(pq), pctx, plse2, cu, S, heads, ctx_lo=plo)
    torch.cuda.synchronize()
    dense_lse2 = lse2.permute(1, 0, 2).reshape(heads, B * S).index_select(1, rows)
    assert torch.equal(pctx, ctx.index_select(0, rows))
    assert torch.equal(plo, lo.index_select(0, rows))
    assert torch.equal(plse2, dense_lse2)
    for name, a, b in (("dq", pdq, dq), ("dk", pdk, dk), ("dv", pdv, dv)):
        assert torch.equal(a, b.index_select(0, rows)), name


def _encoder(seed=0):
    import types
    from mmf_b200.modules import B200BertEncoder
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12,
                                hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, layer_norm_eps=1e-12)
    torch.manual_seed(seed)
    enc = B200BertEncoder(cfg).cuda()
    with torch.no_grad():
        for p in enc.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return enc


def _grads(enc, x, add, w, skip):
    enc._runner.skip_padding = skip
    enc.zero_grad(set_to_none=True)
    xi = x.clone().requires_grad_(True)
    out = enc(xi, add)[0]
    (out * w).sum().backward()
    torch.cuda.synchronize()
    return out.detach(), xi.grad, {k: p.grad.clone() for k, p in enc.named_parameters()}


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _oracle(enc, x, add, w):
    """fp32 oracle on the bf16-rounded weights and input the kernels consume, same restricted loss"""
    from oracle import fusion_oracle as O
    sd = {k: v.detach().to(torch.bfloat16).float().clone().requires_grad_(True) for k, v in enc.state_dict().items()}
    xf = x.to(torch.bfloat16).float().clone().requires_grad_(True)
    out = O.bert_encoder(xf, add, sd, "", 12, 12)
    (out * w).sum().backward()
    named = dict(enc.named_parameters())
    return out.detach(), xf.grad, {k: v.grad for k, v in sd.items() if k in named}


def _errs(out, dx, grads, ref, valid):
    o, d, g = ref
    worst = max(rel(grads[k], g[k]) for k in g if grads[k].dim() == 2)      # 2-D weights (key biases are analytically 0)
    return rel(out[valid], o[valid]), rel(dx, d), worst


def test_encoder_skip_padding_vs_dense():
    """12 L / 768, B = 16, S = 228 with [text | pad | regions | pad] padding and a loss restricted to valid rows.  Packing
    changes which keys share a 64-key block, so the two paths round differently; through 12 layers that difference is of
    the order of each path's own error against the fp32 oracle.  The check is therefore that skip-padding is as accurate
    as the dense path against the oracle (outputs at valid rows, dx, every 2-D parameter gradient), with exact zeros at
    padded positions; with suffix padding the forward at valid rows is bit-identical."""
    enc = _encoder().eval()
    g = torch.Generator().manual_seed(1)
    B, T, R, H = 16, 128, 100, 768
    lt = torch.randint(8, T + 1, (B,), generator=g)
    nr = torch.randint(10, R + 1, (B,), generator=g)
    valid = torch.cat([torch.arange(T)[None] < lt[:, None], torch.arange(R)[None] < nr[:, None]], 1).cuda()   # [t|pad|r|pad]
    add = torch.where(valid, 0.0, -10000.0).float()[:, None, None, :]
    x = torch.randn(B, T + R, H, generator=g).cuda()
    w = torch.randn(B, T + R, H, generator=g).cuda() * valid[..., None]
    od, dxd, gd = _grads(enc, x, add, w, False)
    op, dxp, gp = _grads(enc, x, add, w, True)
    assert not op[~valid].any() and not dxp[~valid].any()
    between = (rel(op[valid], od[valid]), rel(dxp, dxd), max(rel(gp[k], gd[k]) for k in gd if ".key.bias" not in k))
    ref = _oracle(enc, x, add, w)
    e_dense, e_skip = _errs(od, dxd, gd, ref, valid), _errs(op, dxp, gp, ref, valid)
    fmt = lambda e: "out %.2e dx %.2e grad %.2e" % e
    print("encoder 12L: skip vs dense %s | dense vs fp32 oracle %s | skip vs fp32 oracle %s"
          % (fmt(between), fmt(e_dense), fmt(e_skip)))
    for name, es, ed in zip(("out", "dx", "grad"), e_skip, e_dense):
        assert es <= 1.5 * ed + 1e-3, "%s: skip-padding %.2e vs the dense path's %.2e against the fp32 oracle" % (name, es, ed)
    # suffix padding: the valid rows of the forward output are bit-identical to the dense path
    lens = torch.randint(1, T + R + 1, (B,), generator=g).cuda()
    valid = torch.arange(T + R, device="cuda")[None] < lens[:, None]
    add = torch.where(valid, 0.0, -10000.0).float()[:, None, None, :]
    with torch.no_grad():
        enc._runner.skip_padding = False
        od = enc(x, add)[0]
        enc._runner.skip_padding = True
        op = enc(x, add)[0]
    assert torch.equal(op[valid], od[valid]) and not op[~valid].any()


def test_encoder_skip_padding_train_step_and_capture_guard():
    enc = _encoder(3).train()
    B, S = 8, 160
    lens = torch.randint(0, S + 1, (B,))
    lens[0] = 0                                                  # a sample that is padding throughout
    valid = (torch.arange(S)[None] < lens[:, None]).cuda()
    add = torch.where(valid, 0.0, float(torch.finfo(torch.float32).min))[:, None, None, :]
    x = torch.randn(B, S, 768, device="cuda", requires_grad=True)
    enc._runner.skip_padding = True
    out = enc(x, add)[0]
    (out * valid[..., None]).square().sum().backward()
    assert torch.isfinite(out).all() and torch.isfinite(x.grad).all() and not x.grad[~valid].any()
    assert all(torch.isfinite(p.grad).all() for p in enc.parameters() if p.grad is not None)
    from mmf_b200.graphs import GraphedStep
    with pytest.raises(RuntimeError, match="skip_padding"):
        GraphedStep(enc, lambda b: enc(b["x"], b["m"])[0].sum(), {"x": x.detach(), "m": add})


def test_visual_bert_pretraining_model_skip_padding():
    from mmf_b200 import models as MD
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.sample import SampleList
    dev = torch.device("cuda", 0)
    g = torch.load(os.path.join(GOLD, "models.pt"), weights_only=False)
    c = g["visual_bert_pretraining_default"]
    cfg = MD.load_model_config("visual_bert", overrides=dict(c["config"]))
    cfg.losses = [{"type": "cross_entropy"}]
    model = MD.build_model(cfg)
    model.load_state_dict({k: v for k, v in c["state_dict"].items() if k in model.state_dict()})
    model = model.to(dev).eval()
    i = g["visual_bert_inputs"]

    def run():
        sl = SampleList(input_ids=i["ids"].to(dev), input_mask=i["mask"].to(dev), segment_ids=i["seg"].to(dev),
                        image_feature_0=i["feats"].to(dev), image_info_0={"max_features": i["max_features"].to(dev)},
                        lm_label_ids=i["lm_label_ids"].to(dev), targets=i["targets"].to(dev), dataset_name="golden",
                        dataset_type="train")
        model.zero_grad(set_to_none=True)
        loss = model(sl)["losses"]["golden/train/masked_lm_loss"]
        loss.backward()
        return float(loss.detach()), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}, sl
    ld, gd, sl = run()
    assert (sl["attention_mask"] == 0).any()                     # the batch is padded
    assert set_skip_padding(model) >= 1
    lp, gp, sl = run()
    assert (sl["masked_lm_labels"][sl["attention_mask"] == 0] == -1).all()
    worst = max(rel(gp[k], gd[k]) for k in gd if gd[k].norm() > 1e-6 and ".key.bias" not in k)
    print("visual_bert pretraining skip-padding vs dense: loss %.6f vs %.6f, worst param grad %.2e" % (lp, ld, worst))
    assert abs(lp - ld) < 1e-2 * max(1.0, abs(ld)) and worst < 2e-2
    model.train()
    lt, gt, _ = run()
    assert torch.isfinite(torch.tensor(lt)) and all(torch.isfinite(v).all() for v in gt.values())
    set_skip_padding(model, False)
