"""Skip-padding in the two-stream encoders (ViLBERT co-attention, LXMERT cross-modality layers) on the CPU: the encoder
orchestration over the kernel test double (tests/fake_kernels.py), with a torch restatement of the packed self- and
cross-attention entry points injected next to it.  Checks agreement with the dense path for a loss restricted to valid rows
with non-suffix padding in both streams, exact zeros at padded positions, ViLBERT's per-block states, the trivial packing of
an unpadded stream (and LXMERT's visn_attention_mask=None), the dense path when nothing is padded or a sample has tokens in
one stream only, the all-padding batch, the soft-mask error, the switches and the C ABI of the new entry points."""
import ctypes
import types

import pytest
import torch

from mmf_b200 import engine as E

import fake_kernels as FK

CALLS = {"cross_fwd": 0, "cross_bwd": 0, "self_fwd": 0, "self_bwd": 0}


def _spans(cu_q, cu_kv):
    cq, ck = cu_q.tolist(), cu_kv.tolist()
    assert len(cq) == len(ck) >= 2 and cq[0] == 0 and ck[0] == 0
    return list(zip(cq, cq[1:], ck, ck[1:]))


def _fwd(q, k, v, cu_q, cu_kv, max_q, max_kv, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False):
    """contract of functional.attention_varlen_cross_fwd: sample b's query rows attend to its own key rows of the other
    packing; lse2 [heads, total_q]; a sample without keys gets ctx = ctx_lo = 0 and lse2 = -inf"""
    total_q, W = q.shape
    assert cu_q[-1] == total_q and cu_kv[-1] == k.shape[0] == v.shape[0]
    ctx = torch.zeros(total_q, W, dtype=torch.bfloat16)
    lo = torch.zeros(total_q, W, dtype=torch.bfloat16)
    lse2 = torch.full((heads, total_q), float("-inf"))
    if drop_mask is not None:
        assert tuple(drop_mask.shape) == (heads, total_q, (max_kv + 31) // 32)
    for qs, qe, ks, ke in _spans(cu_q, cu_kv):
        nq, nk = qe - qs, ke - ks
        assert nq <= max_q and nk <= max_kv
        if nq == 0 or nk == 0:
            continue
        dm = drop_mask[:, qs:qe].unsqueeze(0) if drop_mask is not None else None
        c, l2, cl = FK.attention_fwd(q[qs:qe], k[ks:ke], v[ks:ke], 1, heads, nq, nk, None, dm, drop_scale, save_lo=True)
        ctx[qs:qe], lse2[:, qs:qe], lo[qs:qe] = c, l2[0], cl
    if out is not None:
        out.copy_(ctx)
        ctx = out
    return (ctx, lse2, lo) if save_lo else (ctx, lse2)


def _bwd(dctx, q, k, v, ctx, lse2, cu_q, cu_kv, max_q, max_kv, heads, drop_mask=None, drop_scale=1.0, dq=None, dk=None,
         dv=None, ctx_lo=None):
    W = q.shape[1]
    res = [torch.zeros(q.shape[0], W, dtype=torch.bfloat16)] + [torch.zeros(k.shape[0], W, dtype=torch.bfloat16)
                                                                 for _ in range(2)]
    for qs, qe, ks, ke in _spans(cu_q, cu_kv):
        nq, nk = qe - qs, ke - ks
        if nq == 0 or nk == 0:
            continue                       # empty side: dq rows (no keys) / dk, dv rows (no queries) stay 0
        dm = drop_mask[:, qs:qe].unsqueeze(0) if drop_mask is not None else None
        r = FK.attention_bwd(dctx[qs:qe], q[qs:qe], k[ks:ke], v[ks:ke], ctx[qs:qe], lse2[:, qs:qe].unsqueeze(0), 1, heads,
                             nq, nk, None, dm, drop_scale, ctx_lo=ctx_lo[qs:qe] if ctx_lo is not None else None)
        res[0][qs:qe], res[1][ks:ke], res[2][ks:ke] = r
    for dst, src in zip((dq, dk, dv), res):
        if dst is not None:
            dst.copy_(src)
    return tuple(d if d is not None else r for d, r in zip((dq, dk, dv), res))


def _cross_fwd(*a, **k):
    CALLS["cross_fwd"] += 1
    return _fwd(*a, **k)


def _cross_bwd(*a, **k):
    CALLS["cross_bwd"] += 1
    return _bwd(*a, **k)


def _self_fwd(q, k, v, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False):
    """packed self-attention is cross-attention with one packing on both sides"""
    CALLS["self_fwd"] += 1
    return _fwd(q, k, v, cu_seqlens, cu_seqlens, max_len, max_len, heads, drop_mask, drop_scale, out, save_lo)


def _self_bwd(dctx, q, k, v, ctx, lse2, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, dq=None, dk=None,
              dv=None, ctx_lo=None):
    CALLS["self_bwd"] += 1
    return _bwd(dctx, q, k, v, ctx, lse2, cu_seqlens, cu_seqlens, max_len, max_len, heads, drop_mask, drop_scale, dq, dk, dv,
                ctx_lo)


@pytest.fixture()
def fake(monkeypatch):
    import mmf_b200.lxmert as LX
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    monkeypatch.setattr(FK, "attention_varlen_cross_fwd", _cross_fwd, raising=False)
    monkeypatch.setattr(FK, "attention_varlen_cross_bwd", _cross_bwd, raising=False)
    monkeypatch.setattr(FK, "attention_varlen_fwd", _self_fwd, raising=False)
    monkeypatch.setattr(FK, "attention_varlen_bwd", _self_bwd, raising=False)
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPS, "F", FK)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(LX, "_require_cuda", lambda t, what: None)
    for k in CALLS:
        CALLS[k] = 0
    yield types.SimpleNamespace(M=M, LX=LX)


def _vilbert_cfg(p=0.0, skip=False):
    return types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=2,
                                 v_hidden_size=128, v_num_attention_heads=2, v_intermediate_size=128, v_num_hidden_layers=2,
                                 bi_hidden_size=128, bi_num_attention_heads=2, v_biattention_id=[0, 1],
                                 t_biattention_id=[1, 2], hidden_dropout_prob=p, v_hidden_dropout_prob=p,
                                 attention_probs_dropout_prob=p, v_attention_probs_dropout_prob=p, skip_padding=skip)


def _lxmert_cfg(p=0.0, skip=False):
    return types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, hidden_dropout_prob=p,
                                 attention_probs_dropout_prob=p, visual_feat_dim=32, visual_pos_dim=4, l_layers=1,
                                 x_layers=2, r_layers=1, skip_padding=skip)


def _valid(B, S, holes):
    v = torch.ones(B, S, dtype=torch.bool)
    for b, sl in holes:
        v[b, sl] = False
    return v


def _two_stream_valid():
    """B = 4: non-suffix padding in both streams, a sample empty in both, a full sample"""
    vt = _valid(4, 10, [(0, slice(3, 5)), (0, slice(8, None)), (1, slice(6, None)), (2, slice(None))])
    vi = _valid(4, 7, [(0, slice(0, 1)), (0, slice(5, None)), (1, slice(2, 4)), (2, slice(None))])
    return vt, vi


def _add(valid):
    return (~valid).float() * -10000.0


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()


def _vilbert_run(enc, txt, img, vt, vi, wt, wi, blocks=False):
    txt, img = txt.clone().requires_grad_(True), img.clone().requires_grad_(True)
    enc.zero_grad(set_to_none=True)
    ot, oi, _ = enc(txt, img, _add(vt)[:, None, None, :], None, _add(vi)[:, None, None, :], output_all_encoded_layers=blocks)
    if blocks:
        return [t.detach() for t in ot], [i.detach() for i in oi]
    ((ot[0] * wt).sum() + (oi[0] * wi).sum()).backward()
    return ot[0].detach(), oi[0].detach(), txt.grad, img.grad, {k: p.grad.clone() for k, p in enc.named_parameters()
                                                                if p.grad is not None}


def _compare(dense, packed, vt, vi, p):
    odt, odi, dxdt, dxdi, gd = dense
    opt, opi, dxpt, dxpi, gp = packed
    for o, dx, valid in ((opt, dxpt, vt), (opi, dxpi, vi)):
        assert not o[~valid].any() and not dx[~valid].any()
        assert torch.isfinite(o).all() and torch.isfinite(dx).all()
    if p > 0:
        return
    assert rel(opt[vt], odt[vt]) < 1e-2 and rel(opi[vi], odi[vi]) < 1e-2
    assert rel(dxpt, dxdt) < 2e-2 and rel(dxpi, dxdi) < 2e-2
    assert set(gp) == set(gd)
    for k in gd:
        if "key" in k and k.endswith("bias"):
            continue                       # analytically zero
        assert rel(gp[k], gd[k]) < 2e-2, k


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_vilbert_packed_matches_dense_on_valid_rows(fake, p):
    torch.manual_seed(0)
    enc = fake.M.B200ViLBertEncoder(_vilbert_cfg(p)).train(p > 0)
    vt, vi = _two_stream_valid()
    txt = torch.randn(4, 10, 64).to(torch.bfloat16).float()
    img = torch.randn(4, 7, 128).to(torch.bfloat16).float()
    wt, wi = torch.randn(4, 10, 64) * vt[..., None], torch.randn(4, 7, 128) * vi[..., None]
    dense = _vilbert_run(enc, txt, img, vt, vi, wt, wi)
    assert CALLS["cross_fwd"] == CALLS["self_fwd"] == 0
    enc._runner.pack_streams = True
    packed = _vilbert_run(enc, txt, img, vt, vi, wt, wi)
    # 2 co-attention blocks x 2 directions; 2 + 2 self-attention layers
    assert CALLS["cross_fwd"] == CALLS["cross_bwd"] == 4 and CALLS["self_fwd"] == CALLS["self_bwd"] == 4
    _compare(dense, packed, vt, vi, p)


def test_vilbert_block_states_unpacked(fake):
    torch.manual_seed(1)
    enc = fake.M.B200ViLBertEncoder(_vilbert_cfg(skip=True)).eval()
    vt, vi = _two_stream_valid()
    txt, img = torch.randn(4, 10, 64), torch.randn(4, 7, 128)
    bt, bi = _vilbert_run(enc, txt, img, vt, vi, None, None, blocks=True)
    assert CALLS["cross_fwd"] == 4
    enc._runner.pack_streams = False
    dt, di = _vilbert_run(enc, txt, img, vt, vi, None, None, blocks=True)
    assert len(bt) == len(bi) == 2
    for p_, d_, valid, shape in ((bt, dt, vt, (4, 10, 64)), (bi, di, vi, (4, 7, 128))):
        for a, b in zip(p_, d_):
            assert a.shape == shape and not a[~valid].any()
            assert rel(a[valid], b[valid]) < 1e-2


def _lxmert_run(enc, lang, feats, boxes, vl, vv, wl, wv):
    lang, feats = lang.clone().requires_grad_(True), feats.clone().requires_grad_(True)
    enc.zero_grad(set_to_none=True)
    vmask = _add(vv)[:, None, None, :] if vv is not None else None
    lo, vo = enc(lang, _add(vl)[:, None, None, :], (feats, boxes), vmask)
    ((lo * wl).sum() + (vo * wv).sum()).backward()
    return lo.detach(), vo.detach(), lang.grad, feats.grad, {k: p.grad.clone() for k, p in enc.named_parameters()
                                                             if p.grad is not None}


def _lxmert_inputs(vt, vi):
    B, T = vt.shape
    R = vi.shape[1]
    lang = torch.randn(B, T, 64).to(torch.bfloat16).float()
    feats = torch.randn(B, R, 32).to(torch.bfloat16).float()
    boxes = torch.rand(B, R, 4)
    return lang, feats, boxes, torch.randn(B, T, 64) * vt[..., None], torch.randn(B, R, 64) * vi[..., None]


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_lxmert_packed_matches_dense_on_valid_rows(fake, p):
    """feats.grad of padded regions is not zero: the visual feature encoder runs on every region (only the encoder layers
    are packed), so its padded outputs are zero but its input gradient is not checked there"""
    torch.manual_seed(2)
    enc = fake.LX.B200LXMERTEncoder(_lxmert_cfg(p)).train(p > 0)
    vt, vi = _two_stream_valid()
    lang, feats, boxes, wl, wv = _lxmert_inputs(vt, vi)
    dense = _lxmert_run(enc, lang, feats, boxes, vt, vi, wl, wv)
    assert CALLS["cross_fwd"] == CALLS["self_fwd"] == 0
    enc._runner.pack_streams = True
    packed = _lxmert_run(enc, lang, feats, boxes, vt, vi, wl, wv)
    # 2 x-layers x 2 directions; 1 l + 1 r layer + 2 x-layers x 2 streams of self-attention
    assert CALLS["cross_fwd"] == CALLS["cross_bwd"] == 4 and CALLS["self_fwd"] == CALLS["self_bwd"] == 6
    odl, odv, dld, dfd, gd = dense
    opl, opv, dlp, dfp, gp = packed
    assert not opl[~vt].any() and not dlp[~vt].any() and not opv[~vi].any()
    assert all(torch.isfinite(t).all() for t in (opl, opv, dlp, dfp))
    if p > 0:
        return
    assert rel(opl[vt], odl[vt]) < 1e-2 and rel(opv[vi], odv[vi]) < 1e-2
    assert rel(dlp, dld) < 2e-2 and rel(dfp, dfd) < 2e-2
    for k in gd:
        if "key" in k and k.endswith("bias"):
            continue
        assert rel(gp[k], gd[k]) < 2e-2, k


def test_one_padded_stream_gets_the_trivial_packing(fake):
    vt, _ = _two_stream_valid()
    vt[2, 0] = True                                   # every sample has text; regions are not padded
    plan = fake.M.plan_two_stream(_add(vt), torch.zeros(4, 7), 4, 10, 7, torch.device("cpu"))
    pt, pi = plan
    assert pt.rows is not None and pt.varlen.total == int(vt.sum())
    assert pi.rows is None and pi.varlen.cu_seqlens.tolist() == [0, 7, 14, 21, 28]
    assert pi.varlen.cu_seqlens.dtype == torch.int32 and pi.varlen.total == 28 and pi.varlen.max_len == 7
    x = torch.randn(28, 3)
    assert pi.pack(x) is x and pi.unpack(x, 28) is x
    # LXMERT without a visual mask: the regions use the trivial packing, the language stream is packed
    torch.manual_seed(3)
    enc = fake.LX.B200LXMERTEncoder(_lxmert_cfg()).eval()
    vi = torch.ones(4, 7, dtype=torch.bool)
    lang, feats, boxes, wl, wv = _lxmert_inputs(vt, vi)
    dense = _lxmert_run(enc, lang, feats, boxes, vt, None, wl, wv)
    enc._runner.pack_streams = True
    packed = _lxmert_run(enc, lang, feats, boxes, vt, None, wl, wv)
    assert CALLS["cross_fwd"] == 4
    assert not packed[0][~vt].any() and not packed[2][~vt].any()
    assert rel(packed[0][vt], dense[0][vt]) < 1e-2 and rel(packed[1], dense[1]) < 1e-2
    assert rel(packed[2], dense[2]) < 2e-2 and rel(packed[3], dense[3]) < 2e-2


def test_nothing_padded_runs_dense(fake):
    torch.manual_seed(4)
    enc = fake.M.B200ViLBertEncoder(_vilbert_cfg()).eval()
    txt, img = torch.randn(2, 5, 64), torch.randn(2, 3, 128)
    ref = enc(txt, img, torch.zeros(2, 5), None, torch.zeros(2, 3), output_all_encoded_layers=False)
    enc._runner.pack_streams = True
    out = enc(txt, img, torch.zeros(2, 5), None, torch.zeros(2, 3), output_all_encoded_layers=False)
    assert torch.equal(out[0][0], ref[0][0]) and torch.equal(out[1][0], ref[1][0])
    enc(txt, img, None, None, None, output_all_encoded_layers=False)
    assert CALLS["cross_fwd"] == CALLS["self_fwd"] == 0


def test_one_sided_empty_sample_runs_dense(fake):
    """sample 1 has regions but no text: the dense path's image outputs for it attend over padded text rows, so packing
    would change them; the call runs the dense path and its outputs equal the dense run's"""
    torch.manual_seed(5)
    enc = fake.M.B200ViLBertEncoder(_vilbert_cfg()).eval()
    vt, vi = _valid(2, 6, [(1, slice(None))]), _valid(2, 4, [(0, slice(3, None))])
    txt, img = torch.randn(2, 6, 64), torch.randn(2, 4, 128)
    args = lambda: (txt, img, _add(vt), None, _add(vi))
    ref = enc(*args(), output_all_encoded_layers=False)
    enc._runner.pack_streams = True
    out = enc(*args(), output_all_encoded_layers=False)
    assert CALLS["cross_fwd"] == CALLS["self_fwd"] == 0
    assert torch.equal(out[0][0], ref[0][0]) and torch.equal(out[1][0], ref[1][0])
    assert fake.M.plan_two_stream(_add(vt), _add(vi), 2, 6, 4, torch.device("cpu")) is None


def test_all_padding_gives_zeros(fake):
    enc = fake.M.B200ViLBertEncoder(_vilbert_cfg(skip=True)).eval()
    txt = torch.randn(2, 5, 64, requires_grad=True)
    img = torch.randn(2, 3, 128, requires_grad=True)
    ot, oi, _ = enc(txt, img, torch.full((2, 5), -10000.0), None, torch.full((2, 3), float("-inf")),
                    output_all_encoded_layers=False)
    assert not ot[0].any() and not oi[0].any()
    (ot[0].sum() + oi[0].sum()).backward()
    assert not txt.grad.any() and not img.grad.any()
    bt, bi, _ = enc(txt, img, torch.full((2, 5), -10000.0), None, torch.full((2, 3), -10000.0))
    assert len(bt) == len(bi) == 2 and not any(t.any() for t in bt + bi)
    lx = fake.LX.B200LXMERTEncoder(_lxmert_cfg(skip=True)).eval()
    lang = torch.randn(2, 5, 64, requires_grad=True)
    lo, vo = lx(lang, torch.full((2, 5), -10000.0), (torch.randn(2, 3, 32), torch.rand(2, 3, 4)), torch.full((2, 3), -1e4))
    assert not lo.any() and not vo.any()
    lo.sum().backward()
    assert not lang.grad.any() and CALLS["cross_fwd"] == CALLS["self_fwd"] == 0


def test_soft_mask_raises(fake):
    enc = fake.M.B200ViLBertEncoder(_vilbert_cfg(skip=True)).eval()
    vt, vi = _two_stream_valid()
    soft = _add(vi)
    soft[3, 1] = -2.0
    with pytest.raises(ValueError, match="soft bias"):
        enc(torch.randn(4, 10, 64), torch.randn(4, 7, 128), _add(vt), None, soft)
    lx = fake.LX.B200LXMERTEncoder(_lxmert_cfg(skip=True)).eval()
    soft = _add(vt)
    soft[0, 0] = -1.0
    with pytest.raises(ValueError, match="soft bias"):
        lx(torch.randn(4, 10, 64), soft, (torch.randn(4, 7, 32), torch.rand(4, 7, 4)), _add(vi))


def test_set_skip_padding_two_stream_switch(fake):
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.patch import set_skip_padding
    root = torch.nn.Module()
    root.v = fake.M.B200ViLBertEncoder(_vilbert_cfg())
    root.l = fake.LX.B200LXMERTEncoder(_lxmert_cfg())
    root.b = fake.M.B200BertEncoder(types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128,
                                                          num_hidden_layers=1, hidden_dropout_prob=0.0,
                                                          attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12))
    assert set_skip_padding(root) == 1
    assert not root.v._runner.pack_streams and not root.l._runner.pack_streams
    assert set_skip_padding(root, False) == 1
    assert set_skip_padding(root, two_stream=True) == 3
    assert root.v._runner.pack_streams and root.l._runner.pack_streams and root.b._runner.skip_padding
    set_skip_padding(root, False)
    assert root.v._runner.pack_streams and not root.b._runner.skip_padding     # the default call leaves them alone
    with pytest.raises(RuntimeError, match="pack_streams"):                   # before any warm-up or capture
        GraphedStep(root, lambda b: None, {"x": torch.zeros(1)})
    assert set_skip_padding(root, False, two_stream=True) == 3 and not root.v._runner.pack_streams
    assert fake.M.B200ViLBertEncoder(_vilbert_cfg(skip=True))._runner.pack_streams
    assert fake.LX.B200LXMERTEncoder(_lxmert_cfg(skip=True))._runner.pack_streams


def test_cross_symbols_exported_and_need_a_device():
    from mmf_b200 import lib
    syms = lib.header_symbols()
    assert "mmfb_attention_varlen_cross_fwd" in syms and "mmfb_attention_varlen_cross_bwd" in syms
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = lib.AttnArgs()
    for fn in (lib.LIB.mmfb_attention_varlen_cross_fwd, lib.LIB.mmfb_attention_varlen_cross_bwd):
        assert fn(ctypes.byref(a), None, 0, None, 0, None) == lib.MMFB_ERR_DEVICE
        assert "no CPU fallback" in lib.last_error()
