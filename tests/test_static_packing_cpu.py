"""Skip-padding under static_rows() on the CPU: the device-side packing plan against today's host-planned one, the two
row maps inverting each other, the device count reaching every kernel of the layer (over the kernel test double, with the
new bounded entry points restated here), and GraphedStep's acceptances and refusals.  The kernels themselves run on the
H100 (tests/test_static_packing_gpu.py)."""
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402

from mmf_b200 import engine as E  # noqa: E402
from mmf_b200 import modules as M  # noqa: E402
from mmf_b200.graphs import GraphedStep, static_rows  # noqa: E402


def _masks():
    g = torch.Generator().manual_seed(4)
    out = []
    for B, S in ((4, 12), (1, 9), (3, 64), (1, 1)):
        for kind in ("random", "all_valid", "one_sample_padding", "all_padding"):
            valid = torch.rand(B, S, generator=g) < 0.6
            if kind == "all_valid":
                valid[:] = True
            elif kind == "one_sample_padding":
                valid[0] = False
            elif kind == "all_padding":
                valid[:] = False
            out.append((kind, valid, (~valid).float() * -10000.0))
    return out


@pytest.mark.parametrize("kind,valid,mask", _masks())
def test_device_plan_matches_the_host_plan(kind, valid, mask):
    B, S = valid.shape
    st = M._plan_packing_static(mask, B, S)
    n = int(valid.sum())
    vl = st.varlen
    assert (vl.B, vl.total, vl.max_len, vl.causal_len) == (B, B * S, S, 0)
    assert vl.count.dtype == torch.int32 and vl.count.shape == (1,) and int(vl.count) == n
    assert vl.count.data_ptr() == vl.cu_seqlens.data_ptr() + 4 * B           # a view of cu[B]: no copy
    assert st.pack_map.dtype == torch.int32 and st.pack_map.shape == (B * S,)
    assert st.unpack_map.dtype == torch.int32 and st.unpack_map.shape == (B * S,)
    host = M._plan_packing(mask, B, S)
    if host is None:                                  # nothing padded: today runs dense, every row in place
        rows, cu = torch.arange(B * S), torch.arange(B + 1, dtype=torch.int32) * S
    else:
        rows, cu = host.rows, host.varlen.cu_seqlens
    assert torch.equal(vl.cu_seqlens, cu)
    assert torch.equal(st.pack_map[:n].long(), rows) and bool((st.pack_map[n:] == -1).all())


@pytest.mark.parametrize("kind,valid,mask", _masks())
def test_the_maps_invert_each_other(kind, valid, mask):
    B, S = valid.shape
    st = M._plan_packing_static(mask, B, S)
    n = int(valid.sum())
    flat = valid.reshape(-1)
    um, pm = st.unpack_map.long(), st.pack_map.long()
    assert bool((um[~flat] == -1).all())
    assert torch.equal(um[flat], torch.arange(n))                      # valid positions -> packed rows 0 .. n-1 in order
    assert torch.equal(um[pm[:n]], torch.arange(n))                    # unpack(pack(row)) = row
    assert torch.equal(pm[um[flat]], torch.nonzero(flat).reshape(-1))  # pack(unpack(position)) = position


def test_soft_values_count_as_padding_without_a_check():
    mask = torch.tensor([[0.0, -1.0, -10000.0]])
    assert int(M._plan_packing_static(mask, 1, 3).varlen.count) == 1
    with pytest.raises(ValueError, match="soft bias"):
        M._plan_packing(mask, 1, 3)


# ---------------------------------------------------------------------------------------------------------------------
# the device count reaches every kernel of the layer
# ---------------------------------------------------------------------------------------------------------------------
class Double(types.SimpleNamespace):
    """fake_kernels plus the bounded entry points: a bounded call computes the rows below the bound (the GEMMs every row
    of the tiles below it) and records the bound it was given"""

    def __init__(self):
        super().__init__()
        self.calls = []
        for name in dir(FK):
            if not name.startswith("_"):
                setattr(self, name, getattr(FK, name))
        self.gemm, self.layernorm_fwd, self.layernorm_bwd = self._gemm, self._ln_fwd, self._ln_bwd

    def _gemm(self, a, b, *, m_bound=None, k_bound=None, **kw):
        self.calls.append(("gemm", kw.get("epi"), m_bound, k_bound))
        return FK.gemm(a, b, **kw)

    def _ln_fwd(self, *a, m_bound=None, **kw):
        self.calls.append(("ln_fwd", None, m_bound, None))
        return FK.layernorm_fwd(*a, **kw)

    def _ln_bwd(self, *a, m_bound=None, **kw):
        self.calls.append(("ln_bwd", None, m_bound, None))
        return FK.layernorm_bwd(*a, **kw)

    def colsum_bounded(self, x, out, m_bound):
        self.calls.append(("colsum", None, m_bound, None))
        n = int(m_bound.reshape(-1)[0])
        out += x[:n].float().sum(0)
        return out

    def gather_rows(self, x, idx, out=None):
        r = torch.where(idx[:, None] >= 0, x[idx.long().clamp_min(0)], torch.zeros((), dtype=x.dtype))
        return r.to(torch.bfloat16)

    def attention_varlen_fwd(self, q, k, v, cu, max_len, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False):
        ctx = out if out is not None else torch.zeros_like(q)
        lse2 = torch.zeros(heads, q.shape[0])
        cu = cu.tolist()
        for b in range(len(cu) - 1):
            s, e = cu[b], cu[b + 1]
            if e > s:
                ctx[s:e] = FK.attention_fwd(q[s:e], k[s:e], v[s:e], 1, heads, e - s, e - s)[0]
        return (ctx, lse2, ctx.clone()) if save_lo else (ctx, lse2)

    def attention_varlen_bwd(self, dctx, q, k, v, ctx, lse2, cu, max_len, heads, drop_mask=None, drop_scale=1.0, dq=None,
                             dk=None, dv=None, ctx_lo=None):
        cu = cu.tolist()
        for b in range(len(cu) - 1):
            s, e = cu[b], cu[b + 1]
            if e > s:
                c, l2 = FK.attention_fwd(q[s:e], k[s:e], v[s:e], 1, heads, e - s, e - s)
                FK.attention_bwd(dctx[s:e], q[s:e], k[s:e], v[s:e], c, l2, 1, heads, e - s, e - s, dq=dq[s:e], dk=dk[s:e],
                                 dv=dv[s:e])
        return dq, dk, dv


def _encoder(layers=2):
    cfg = types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=layers,
                                hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                                skip_padding=True)
    torch.manual_seed(0)
    return M.B200BertEncoder(cfg)


@pytest.fixture
def double(monkeypatch):
    d = Double()
    monkeypatch.setattr(E, "F", d)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    return d


def test_static_call_bounds_every_kernel_of_the_layer(double):
    enc = _encoder().train()
    B, S = 3, 10
    valid = torch.ones(B, S, dtype=torch.bool)
    valid[0, 6:] = False
    valid[2] = False
    mask = (~valid).float() * -10000.0
    x = torch.randn(B, S, 64, requires_grad=True)
    w = torch.randn(B, S, 64) * valid[..., None]
    with static_rows():
        out = M.run_bert_encoder(enc._runner, x, mask, True)[0]
    (out.float() * w).sum().backward()
    assert not out[~valid].any() and not x.grad[~valid].any()
    bounds = [c for c in double.calls]
    count = {id(c[2]) for c in bounds if c[2] is not None} | {id(c[3]) for c in bounds if c[3] is not None}
    assert len(count) == 1                                    # one device count, cu[B], for the whole call
    n = next(c[2] if c[2] is not None else c[3] for c in bounds)
    assert int(n) == int(valid.sum())
    # per layer: forward 4 GEMMs + 2 LayerNorms; backward 2 LayerNorms, 4 dgrads, 4 wgrads, 2 column sums
    kinds = [(c[0], c[1], c[2] is not None, c[3] is not None) for c in bounds]
    from mmf_b200 import lib
    assert kinds.count(("gemm", lib.EPI_ATOMIC_F32, False, True)) == 2 * 4
    assert all(c[2] is not None for c in bounds if c[0] in ("ln_fwd", "ln_bwd", "colsum"))
    assert sum(1 for c in bounds if c[0] == "gemm" and c[1] != lib.EPI_ATOMIC_F32 and c[2] is not None) == 2 * 8
    assert sum(1 for c in bounds if c[0] in ("ln_fwd", "ln_bwd")) == 2 * 4
    assert sum(1 for c in bounds if c[0] == "colsum") == 2 * 2
    assert all(c[2] is not None or c[3] is not None for c in bounds)


def test_eager_call_outside_the_context_passes_no_bound(double):
    enc = _encoder(1).train()
    mask = torch.zeros(2, 5)
    mask[0, 3:] = -10000.0
    x = torch.randn(2, 5, 64, requires_grad=True)
    M.run_bert_encoder(enc._runner, x, mask, True)[0].sum().backward()
    assert double.calls and all(c[2] is None and c[3] is None for c in double.calls)


# ---------------------------------------------------------------------------------------------------------------------
# GraphedStep
# ---------------------------------------------------------------------------------------------------------------------
def _root(skip=True, causal=False, two_stream=False):
    from mmf_b200.modules import B200ViLBertEncoder
    from mmf_b200.patch import set_skip_padding
    root = torch.nn.Module()
    root.a = _encoder(1)
    c = dict(hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=1, v_hidden_size=64,
             v_num_attention_heads=1, v_intermediate_size=128, v_num_hidden_layers=1, bi_hidden_size=64,
             bi_num_attention_heads=1, v_biattention_id=[0], t_biattention_id=[0])
    root.c = B200ViLBertEncoder(types.SimpleNamespace(hidden_dropout_prob=0.0, v_hidden_dropout_prob=0.0,
                                                      attention_probs_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0,
                                                      **c))
    set_skip_padding(root, False, two_stream=True)
    if skip:
        set_skip_padding(root, True, causal=causal, two_stream=two_stream)
    return root


@pytest.fixture
def no_capture(monkeypatch):
    seen = []
    monkeypatch.setattr(GraphedStep, "_capture", lambda self, *a: seen.append(a))
    return seen


def test_graphed_step_refusals_and_acceptances(no_capture):
    batch = {"x": torch.zeros(1)}
    msg = ("GraphedStep: the model has skip_padding encoders, which read the token count on the host and cannot be captured; "
           "turn them off with mmf_b200.patch.set_skip_padding(model, False)")
    with pytest.raises(RuntimeError) as e:
        GraphedStep(_root(), lambda b: None, batch)
    assert str(e.value) == msg                                          # today's message, unchanged
    GraphedStep(_root(), lambda b: None, batch, static_rows=True)      # accepted
    assert len(no_capture) == 1
    with pytest.raises(RuntimeError, match="pack_tail set, which read the token count on the host for calls with a causal "
                                           "tail even under static_rows"):
        GraphedStep(_root(causal=True), lambda b: None, batch, static_rows=True)
    with pytest.raises(RuntimeError) as e:
        GraphedStep(_root(causal=True), lambda b: None, batch)
    assert str(e.value) == msg
    streams = ("GraphedStep: the model has two-stream encoders with pack_streams set, which read the token counts on the "
               "host%s and cannot be captured; turn them off with "
               "mmf_b200.patch.set_skip_padding(model, False, two_stream=True)")
    root = _root(skip=False)
    root.c._runner.pack_streams = True
    with pytest.raises(RuntimeError) as e:
        GraphedStep(root, lambda b: None, batch)
    assert str(e.value) == streams % ""
    with pytest.raises(RuntimeError) as e:
        GraphedStep(_root(two_stream=True), lambda b: None, batch, static_rows=True)
    assert str(e.value) == streams % " even under static_rows"
    assert len(no_capture) == 1
    GraphedStep(_root(skip=False), lambda b: None, batch)
    assert len(no_capture) == 2


def test_header_declares_the_bounded_layernorm():
    from mmf_b200 import lib
    syms = lib.header_symbols()
    assert "mmfb_layernorm_fwd_bounded" in syms and "mmfb_layernorm_bwd_bounded" in syms
