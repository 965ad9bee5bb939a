"""Skip-padding (packed rows + variable-length attention) on the CPU: the encoder orchestration over the kernel test double
(tests/fake_kernels.py), with a torch restatement of the two varlen attention entry points injected next to it.  Checks the
packing plan (cu_seqlens / total / max_len, row order with non-suffix padding and an all-padding sample), exact zeros at
padded positions, the soft-mask error, the dense fallback when nothing is padded, agreement with the dense path for a
loss restricted to valid rows, and the C ABI of the new entry points without a GPU."""
import ctypes
import types

import pytest
import torch

from mmf_b200 import engine as E

import fake_kernels as FK

CALLS = {"fwd": 0, "bwd": 0}


def _varlen_fwd(q, k, v, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False):
    """contract of functional.attention_varlen_fwd: every sample attends to its own rows; lse2 [heads, total]"""
    CALLS["fwd"] += 1
    total, W = q.shape
    cu = cu_seqlens.tolist()
    assert len(cu) >= 2 and cu[0] == 0 and cu[-1] == total and max(b - a for a, b in zip(cu, cu[1:])) <= max_len
    ctx = torch.zeros(total, W, dtype=torch.bfloat16)
    lo = torch.zeros(total, W, dtype=torch.bfloat16)
    lse2 = torch.zeros(heads, total)
    if drop_mask is not None:
        assert tuple(drop_mask.shape) == (heads, total, (max_len + 31) // 32)
    for s, e in zip(cu, cu[1:]):
        n = e - s
        if n == 0:
            continue
        dm = drop_mask[:, s:e].unsqueeze(0) if drop_mask is not None else None
        c, l2, cl = FK.attention_fwd(q[s:e], k[s:e], v[s:e], 1, heads, n, n, None, dm, drop_scale, save_lo=True)
        ctx[s:e], lse2[:, s:e], lo[s:e] = c, l2[0], cl
    if out is not None:
        out.copy_(ctx)
        ctx = out
    return (ctx, lse2, lo) if save_lo else (ctx, lse2)


def _varlen_bwd(dctx, q, k, v, ctx, lse2, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, dq=None, dk=None,
                dv=None, ctx_lo=None):
    CALLS["bwd"] += 1
    total, W = q.shape
    res = [torch.zeros(total, W, dtype=torch.bfloat16) for _ in range(3)]
    cu = cu_seqlens.tolist()
    for s, e in zip(cu, cu[1:]):
        n = e - s
        if n == 0:
            continue
        dm = drop_mask[:, s:e].unsqueeze(0) if drop_mask is not None else None
        r = FK.attention_bwd(dctx[s:e], q[s:e], k[s:e], v[s:e], ctx[s:e], lse2[:, s:e].unsqueeze(0), 1, heads, n, n, None,
                             dm, drop_scale, ctx_lo=ctx_lo[s:e] if ctx_lo is not None else None)
        for dst, src in zip(res, r):
            dst[s:e] = src
    for dst, src in zip((dq, dk, dv), res):
        if dst is not None:
            dst.copy_(src)
    return tuple(d if d is not None else r for d, r in zip((dq, dk, dv), res))


@pytest.fixture()
def fake(monkeypatch):
    monkeypatch.setattr(FK, "attention_varlen_fwd", _varlen_fwd, raising=False)
    monkeypatch.setattr(FK, "attention_varlen_bwd", _varlen_bwd, raising=False)
    monkeypatch.setattr(E, "F", FK)
    import mmf_b200.modules as M
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    CALLS["fwd"] = CALLS["bwd"] = 0
    yield M


def _cfg(p=0.0, layers=2, skip=False):
    return types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=layers,
                                 hidden_dropout_prob=p, attention_probs_dropout_prob=p, layer_norm_eps=1e-12,
                                 skip_padding=skip)


def _masks():
    """[text | pad | regions | pad] (VisualBERT), suffix padding, an all-padding sample, a full sample"""
    B, S = 4, 12
    valid = torch.ones(B, S, dtype=torch.bool)
    valid[0, 4:6] = False
    valid[0, 10:] = False
    valid[1, 7:] = False
    valid[2, :] = False
    return valid, ((~valid).float() * -10000.0)


def test_packing_plan_non_suffix_padding_and_empty_sample(fake):
    valid, add = _masks()
    plan = fake._plan_packing(add, 4, 12)
    lens = valid.sum(1)
    assert plan.varlen.cu_seqlens.dtype == torch.int32
    assert plan.varlen.cu_seqlens.tolist() == [0] + torch.cumsum(lens, 0).tolist()
    assert plan.varlen.total == int(lens.sum()) == 8 + 7 + 0 + 12 and plan.varlen.max_len == 12 and plan.varlen.B == 4
    expect = [b * 12 + s for b in range(4) for s in range(12) if valid[b, s]]
    assert plan.rows.tolist() == expect                            # original order within each sample
    x = torch.randn(48, 5)
    back = plan.unpack(plan.pack(x), 48)
    assert torch.equal(back[valid.reshape(-1)], x[valid.reshape(-1)]) and not back[~valid.reshape(-1)].any()
    # -inf / finfo.min padding is padding too; no padding at all: no plan
    assert fake._plan_packing(torch.where(valid, 0.0, float("-inf")), 4, 12).varlen.total == 27
    assert fake._plan_packing(torch.zeros(4, 12), 4, 12) is None


def test_soft_mask_raises(fake):
    enc = fake.B200BertEncoder(_cfg(skip=True)).eval()
    _, add = _masks()
    add[3, 2] = -5.0
    with pytest.raises(ValueError, match="soft bias"):
        enc(torch.randn(4, 12, 64), add)


def _run(enc, x, add, w):
    x = x.clone().requires_grad_(True)
    enc.zero_grad(set_to_none=True)
    out = enc(x, add)[0]
    (out * w).sum().backward()
    return out.detach(), x.grad, {k: p.grad.clone() for k, p in enc.named_parameters()}


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_packed_matches_dense_on_valid_rows(fake, p):
    """loss restricted to valid rows: outputs at valid rows, dx and every parameter gradient agree with the dense path;
    padded output and dx rows are exactly zero.  With dropout both runs draw different masks, so only zeros / finiteness
    are checked there."""
    torch.manual_seed(0)
    enc = fake.B200BertEncoder(_cfg(p)).train(p > 0)
    valid, add = _masks()
    x = torch.randn(4, 12, 64).to(torch.bfloat16).float()
    w = torch.randn(4, 12, 64) * valid[..., None]
    enc._runner.skip_padding = False
    od, dxd, gd = _run(enc, x, add, w)
    enc._runner.skip_padding = True
    op, dxp, gp = _run(enc, x, add, w)
    assert CALLS["fwd"] == 2 and CALLS["bwd"] == 2
    pad = ~valid
    assert not op[pad].any() and not dxp[pad].any()
    assert torch.isfinite(op).all() and torch.isfinite(dxp).all()
    if p > 0:
        return
    assert rel(op[valid], od[valid]) < 1e-2
    assert rel(dxp, dxd) < 2e-2
    for k in gd:
        if ".key.bias" in k:
            continue                       # analytically zero
        assert rel(gp[k], gd[k]) < 2e-2, k


def test_output_hidden_states_unpacked(fake):
    enc = fake.B200BertEncoder(_cfg(skip=True)).eval()
    valid, add = _masks()
    out = enc(torch.randn(4, 12, 64), add, output_hidden_states=True)
    assert len(out[1]) == 3
    for h in out[1]:
        assert h.shape == (4, 12, 64) and not h[~valid].any()


def test_nothing_padded_runs_dense(fake):
    torch.manual_seed(1)
    enc = fake.B200BertEncoder(_cfg()).eval()
    x = torch.randn(2, 6, 64)
    ref = enc(x, torch.zeros(2, 6))[0]
    enc._runner.skip_padding = True
    assert torch.equal(enc(x, torch.zeros(2, 6))[0], ref) and torch.equal(enc(x, None)[0], enc(x, None)[0])
    assert CALLS["fwd"] == 0


def test_all_padding_batch_gives_zeros(fake):
    enc = fake.B200BertEncoder(_cfg(skip=True)).eval()
    x = torch.randn(2, 5, 64, requires_grad=True)
    out = enc(x, torch.full((2, 5), -10000.0))[0]
    assert not out.any()
    out.sum().backward()
    assert not x.grad.any() and CALLS["fwd"] == 0


def test_set_skip_padding_covers_single_stream_encoders(fake):
    from transformers import BertConfig
    from transformers.models.bert.modeling_bert import BertEncoder
    from mmf_b200.patch import attach_encoder, set_skip_padding
    from mmf_b200.modules import B200ViLBertEncoder
    root = torch.nn.Module()
    root.a = fake.B200BertEncoder(_cfg(layers=1))
    root.b = attach_encoder(BertEncoder(BertConfig(hidden_size=64, num_attention_heads=1, intermediate_size=128,
                                                   num_hidden_layers=1, vocab_size=50)))
    c = dict(hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=1, v_hidden_size=64,
             v_num_attention_heads=1, v_intermediate_size=128, v_num_hidden_layers=1, bi_hidden_size=64,
             bi_num_attention_heads=1, v_biattention_id=[0], t_biattention_id=[0])
    root.c = B200ViLBertEncoder(types.SimpleNamespace(hidden_dropout_prob=0.0, v_hidden_dropout_prob=0.0,
                                                      attention_probs_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0,
                                                      **c))
    assert set_skip_padding(root) == 2
    assert root.a._runner.skip_padding and root.b._runner.skip_padding
    assert not hasattr(root.c._runner, "skip_padding")
    from mmf_b200.graphs import GraphedStep
    with pytest.raises(RuntimeError, match="skip_padding"):          # before any warm-up or capture
        GraphedStep(root, lambda b: None, {"x": torch.zeros(1)})
    assert set_skip_padding(root, False) == 2 and not root.a._runner.skip_padding


def test_varlen_symbols_exported_and_need_a_device():
    from mmf_b200 import lib
    syms = lib.header_symbols()
    assert "mmfb_attention_varlen_fwd" in syms and "mmfb_attention_varlen_bwd" in syms
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = lib.AttnArgs()
    for fn in (lib.LIB.mmfb_attention_varlen_fwd, lib.LIB.mmfb_attention_varlen_bwd):
        assert fn(ctypes.byref(a), None, 0, None) == lib.MMFB_ERR_DEVICE
        assert "no CPU fallback" in lib.last_error()
