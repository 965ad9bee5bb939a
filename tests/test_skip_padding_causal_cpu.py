"""Skip-padding of encoder calls with a causal tail (M4C's multimodal transformer) on the CPU: the encoder orchestration over
the kernel test double (tests/fake_kernels.py), extended below with the causal tail of the dense attention calls and a
torch restatement of the packed entry points with and without a tail.  Checks the packing plan (the tail rows stay even
where the mask pads them), the arguments that reach attention_varlen_fwd / _bwd, the dense path without pack_tail and for
an unpadded prefix, agreement with the dense path on valid rows, set_skip_padding(..., causal=True), the refusal of
GraphedStep, the registered m4c model's loss and gradients against its dense path, and the C ABI of the new entry points
without a GPU.  The kernels are covered on the GPU (tests/test_attention_varlen_causal_gpu.py,
tests/test_m4c_skip_padding_gpu.py)."""
import contextlib
import ctypes
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402

# ---- the test double, extended ----------------------------------------------------------------------------------------
_TAIL = [0]
_PROBS = FK._probs
CALLS = []


def _probs(q, k, B, heads, Sq, Skv, mask):
    """FK._probs with the last T keys a causal tail: 0 for queries at or past the key, -10000 before it"""
    T = _TAIL[0]
    if not T:
        return _PROBS(q, k, B, heads, Sq, Skv, mask)
    s = _PROBS(q, k, B, heads, Sq, Skv, None)
    P = Skv - T
    m = torch.zeros(B, Sq, Skv)
    if mask is not None:
        m[:, :, :P] = mask.float()[:, None, :P]
    qi, ki = torch.arange(Sq)[:, None], torch.arange(Skv)[None, :]
    m[:, :, P:] = torch.where(ki[:, P:] <= qi, 0.0, -10000.0)
    return s + m[:, None]


@contextlib.contextmanager
def _tail(T):
    _TAIL[0] = int(T)
    try:
        yield
    finally:
        _TAIL[0] = 0


def _attention_fwd(*a, causal_len=0, **k):
    CALLS.append(("dense_fwd", causal_len))
    with _tail(causal_len):
        return FK.attention_fwd(*a, **k)


def _attention_bwd(*a, causal_len=0, **k):
    CALLS.append(("dense_bwd", causal_len))
    with _tail(causal_len):
        return FK.attention_bwd(*a, **k)


def _varlen_fwd(q, k, v, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False,
                causal_len=0):
    """contract of functional.attention_varlen_fwd: each sample alone, its last causal_len rows a causal tail"""
    total, W = q.shape
    cu = cu_seqlens.tolist()
    CALLS.append(("varlen_fwd", causal_len, cu, total, int(max_len)))
    assert cu[0] == 0 and cu[-1] == total and max(b - a for a, b in zip(cu, cu[1:])) <= max_len
    ctx, lo = torch.zeros(total, W, dtype=torch.bfloat16), torch.zeros(total, W, dtype=torch.bfloat16)
    lse2 = torch.zeros(heads, total)
    for s, e in zip(cu, cu[1:]):
        n = e - s
        if n == 0:
            continue
        dm = drop_mask[:, s:e].unsqueeze(0) if drop_mask is not None else None
        with _tail(min(causal_len, n)):
            c, l2, cl = FK.attention_fwd(q[s:e], k[s:e], v[s:e], 1, heads, n, n, None, dm, drop_scale, save_lo=True)
        ctx[s:e], lse2[:, s:e], lo[s:e] = c, l2[0], cl
    if out is not None:
        out.copy_(ctx)
        ctx = out
    return (ctx, lse2, lo) if save_lo else (ctx, lse2)


def _varlen_bwd(dctx, q, k, v, ctx, lse2, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, dq=None, dk=None,
                dv=None, ctx_lo=None, causal_len=0):
    total, W = q.shape
    cu = cu_seqlens.tolist()
    CALLS.append(("varlen_bwd", causal_len, cu, total, int(max_len)))
    res = [torch.zeros(total, W, dtype=torch.bfloat16) for _ in range(3)]
    for s, e in zip(cu, cu[1:]):
        n = e - s
        if n == 0:
            continue
        dm = drop_mask[:, s:e].unsqueeze(0) if drop_mask is not None else None
        with _tail(min(causal_len, n)):
            r = FK.attention_bwd(dctx[s:e], q[s:e], k[s:e], v[s:e], ctx[s:e], lse2[:, s:e].unsqueeze(0), 1, heads, n, n,
                                 None, dm, drop_scale, ctx_lo=ctx_lo[s:e] if ctx_lo is not None else None)
        for dst, src in zip(res, r):
            dst[s:e] = src
    for dst, src in zip((dq, dk, dv), res):
        if dst is not None:
            dst.copy_(src)
    return tuple(d if d is not None else r for d, r in zip((dq, dk, dv), res))


def _fake():
    mod = types.ModuleType("fake_kernels_varlen_causal")
    mod.__dict__.update({k: v for k, v in FK.__dict__.items() if not k.startswith("__")})
    mod.attention_fwd, mod.attention_bwd = _attention_fwd, _attention_bwd
    mod.attention_varlen_fwd, mod.attention_varlen_bwd = _varlen_fwd, _varlen_bwd
    return mod


@pytest.fixture()
def fake(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.encoders as EN
    import mmf_b200.engine as E
    import mmf_b200.m4c_model as MM
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.vilbert as VB
    f = _fake()
    monkeypatch.setattr(FK, "_probs", _probs)
    for mod in (E, OPS, EM):
        monkeypatch.setattr(mod, "F", f)
    for mod in (M, EM, VB, EN, MM):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    CALLS.clear()
    yield M


def _encoder(M, p=0.0, layers=2, pack_tail=True):
    cfg = types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=layers,
                                hidden_dropout_prob=p, attention_probs_dropout_prob=p, layer_norm_eps=1e-12,
                                skip_padding=True)
    enc = M.B200BertEncoder(cfg)
    enc._runner.pack_tail = pack_tail
    return enc


B, S, T = 3, 14, 4


def _mask():
    """[text | pad | regions | pad | tail]: the tail positions hold -10000 in sample 0 and 0 elsewhere - the dense path
    does not read them, and packing keeps them all"""
    valid = torch.ones(B, S, dtype=torch.bool)
    valid[0, 3:5] = False
    valid[0, 8:] = False                          # the mask pads sample 0's tail too
    valid[1, 6:] = False
    valid[2, :S - T] = False                      # only its tail
    add = (~valid).float() * -10000.0
    add[1:, S - T:] = 0.0
    kept = valid.clone()
    kept[:, S - T:] = True
    return add, kept


def test_packing_plan_keeps_the_tail_rows(fake):
    add, kept = _mask()
    enc = _encoder(fake).eval()
    with torch.no_grad():
        out = fake.run_bert_encoder(enc._runner, torch.randn(B, S, 64), add, False, causal_len=T)[0]
    lens = kept.sum(1)
    cu = [0] + torch.cumsum(lens, 0).tolist()
    assert [c[0] for c in CALLS] == ["varlen_fwd"] * 2
    for c in CALLS:
        assert c[1:] == (T, cu, int(lens.sum()), int(lens.max()))
    assert lens.tolist() == [3 + 3 + T, 6 + T, T]
    assert not out[~kept].any() and out[kept].abs().sum(-1).gt(0).all()
    # the plan itself: the rows of every sample in order, its last T rows the tail
    plan = fake._plan_packing(fake._tail_kept(add, T), B, S)
    assert plan.rows.tolist() == [b * S + s for b in range(B) for s in range(S) if kept[b, s]]
    for b in range(B):
        assert plan.rows[cu[b + 1] - T:cu[b + 1]].tolist() == [b * S + s for s in range(S - T, S)]
    assert not add[0, S - T:].eq(0).any()         # the mask did pad sample 0's tail


def test_arguments_reach_the_packed_entry_points(fake):
    add, kept = _mask()
    enc = _encoder(fake, p=0.1).train()
    x = torch.randn(B, S, 64, requires_grad=True)
    out = fake.run_bert_encoder(enc._runner, x, add, True, causal_len=T)[0]
    (out * torch.randn_like(out)).sum().backward()
    lens = kept.sum(1)
    cu, total = [0] + torch.cumsum(lens, 0).tolist(), int(lens.sum())
    assert [c[0] for c in CALLS] == ["varlen_fwd"] * 2 + ["varlen_bwd"] * 2
    assert all(c[1:] == (T, cu, total, int(lens.max())) for c in CALLS)
    assert not x.grad[~kept].any() and torch.isfinite(x.grad).all()


def test_without_pack_tail_the_call_is_dense(fake):
    add, _ = _mask()
    enc = _encoder(fake, pack_tail=False).eval()
    with torch.no_grad():
        fake.run_bert_encoder(enc._runner, torch.randn(B, S, 64), add, False, causal_len=T)
    assert CALLS == [("dense_fwd", T)] * 2


def test_unpadded_prefix_takes_the_dense_path(fake):
    """nothing before the tail is padded (the tail may be): no plan, the dense causal call, and the same numbers"""
    add = torch.zeros(B, S)
    add[0, S - T:] = -10000.0
    enc = _encoder(fake).eval()
    x = torch.randn(B, S, 64)
    with torch.no_grad():
        got = fake.run_bert_encoder(enc._runner, x, add, False, causal_len=T)[0]
        enc._runner.skip_padding = False
        ref = fake.run_bert_encoder(enc._runner, x, add, False, causal_len=T)[0]
    assert CALLS == [("dense_fwd", T)] * 4 and torch.equal(got, ref)


def test_packed_matches_dense_on_kept_rows(fake):
    """a loss over the kept rows: outputs, dx and every parameter gradient agree with the dense path, and the padded rows
    before the tail are exactly zero in the output and dx"""
    torch.manual_seed(0)
    add, kept = _mask()
    enc = _encoder(fake)
    x0 = torch.randn(B, S, 64).to(torch.bfloat16).float()
    w = torch.randn(B, S, 64) * kept[..., None]

    def run():
        x = x0.clone().requires_grad_(True)
        enc.zero_grad(set_to_none=True)
        out = fake.run_bert_encoder(enc._runner, x, add, True, causal_len=T)[0]
        (out * w).sum().backward()
        return out.detach(), x.grad, {k: p.grad.clone() for k, p in enc.named_parameters()}

    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()
    op, dxp, gp = run()
    enc._runner.skip_padding = False
    od, dxd, gd = run()
    assert not op[~kept].any() and not dxp[~kept].any()
    assert rel(op[kept], od[kept]) < 1e-2 and rel(dxp[kept], dxd[kept]) < 2e-2
    for k in gd:
        if ".key.bias" not in k:                  # analytically zero
            assert rel(gp[k], gd[k]) < 2e-2, k


def test_output_attentions_with_a_tail_still_raises(fake):
    add, _ = _mask()
    enc = _encoder(fake).eval()
    with pytest.raises(ValueError, match="causal tail"):
        fake.run_bert_encoder(enc._runner, torch.randn(B, S, 64), add, False, output_attentions=True, causal_len=T)


def _m4c(golden, MD):
    import test_m4c_model_cpu as M4
    return M4.build(MD, golden), M4


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "m4c_model.pt"),
                      weights_only=False)


def test_set_skip_padding_causal_count_and_graphed_step_refusal(fake, golden):
    import mmf_b200.models as MD
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.patch import set_skip_padding
    model, _ = _m4c(golden, MD)
    runners = [model.text_bert.encoder._runner, model.mmt.encoder._runner]
    assert set_skip_padding(model) == 2 and not any(r.pack_tail for r in runners)
    assert set_skip_padding(model, causal=True) == 2
    assert all(r.skip_padding and r.pack_tail for r in runners)
    with pytest.raises(RuntimeError, match="skip_padding"):          # before any warm-up or capture
        GraphedStep(model, lambda b: None, {"x": torch.zeros(1)})
    assert set_skip_padding(model, False, causal=True) == 2
    assert not any(r.skip_padding or r.pack_tail for r in runners)


def test_m4c_loss_and_gradients_equal_the_dense_path(fake, golden):
    """the registered m4c model, teacher-forced: the loss and every parameter gradient of the packed MMT equal the dense
    path's to rounding, and the scores agree at valid answer and OCR slots (m4c_model's docstring says why)"""
    import mmf_b200.models as MD
    from mmf_b200.patch import set_skip_padding
    model, M4 = _m4c(golden, MD)
    model.train()
    for m in model.modules():                      # the same function on both paths: no dropout masks to differ
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    sl = M4.sample_list(golden)
    assert (sl["context_info_0"]["max_features"] < golden["inputs"]["context_feature_0"].shape[1]).any()

    def step():
        model.zero_grad(set_to_none=True)
        CALLS.clear()
        out = model(sl)
        loss = M4.loss_of(out)
        loss.backward()
        return float(loss.detach()), out["scores"].detach(), {n: p.grad.clone() for n, p in model.named_parameters()
                                                      if p.grad is not None}, list(CALLS)

    ld, sd, gd, calls_d = step()
    set_skip_padding(model, causal=True)
    lp, sp, gp, calls_p = step()
    assert ("dense_fwd", golden["inputs"]["train_prev_inds"].shape[1]) in calls_d
    assert any(c[0] == "varlen_fwd" and c[1] > 0 for c in calls_p)
    assert not any(c[0] == "dense_fwd" and c[1] > 0 for c in calls_p)
    assert abs(lp - ld) <= 1e-3 * abs(ld)
    assert gp.keys() == gd.keys()
    for n in gd:
        scale = gd[n].double().norm().clamp_min(1e-6)
        assert ((gp[n].double() - gd[n].double()).norm() / scale).item() < 2e-2, n
    O = golden["inputs"]["context_feature_0"].shape[1]
    ocr_valid = torch.arange(O)[None, :] < sl["context_info_0"]["max_features"][:, None]
    valid = torch.cat([torch.ones(sd.shape[0], sd.shape[-1] - O, dtype=torch.bool), ocr_valid], 1)[:, None, :].expand_as(sd)
    assert ((sp[valid] - sd[valid]).norm() / sd[valid].norm()).item() < 1e-2
    assert (sp[~valid] < -9000).all() and (sd[~valid] < -9000).all()


def test_varlen_causal_symbols_exported_and_need_a_device():
    from mmf_b200 import lib
    syms = lib.header_symbols()
    assert "mmfb_attention_varlen_causal_fwd" in syms and "mmfb_attention_varlen_causal_bwd" in syms
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = lib.AttnArgs()
    for fn in (lib.LIB.mmfb_attention_varlen_causal_fwd, lib.LIB.mmfb_attention_varlen_causal_bwd):
        assert fn(ctypes.byref(a), None, 0, None) == lib.MMFB_ERR_DEVICE
        assert "no CPU fallback" in lib.last_error()
