"""Device-planned packing of causal-tail and two-stream encoder calls, on the CPU: the refusals of GraphedStep and
GraphedForward with and without `device_plan`, set_skip_padding's counts, the plan rules (tests/plan_ref.py) against the
host plans of today's eager packing, and the per-stream device counts reaching every GEMM, LayerNorm and column sum of a
bounded co-attention / cross-modality layer (over tests/fake_kernels.py).  The kernel runs on the H100
(tests/test_device_plan_gpu.py)."""
import contextlib
import os
import sys
import types

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fake_kernels as FK  # noqa: E402
import plan_ref as PR  # noqa: E402

from mmf_b200 import engine as E  # noqa: E402
from mmf_b200 import graphs  # noqa: E402
from mmf_b200 import modules as M  # noqa: E402
from mmf_b200.graphs import GraphedStep  # noqa: E402
from mmf_b200.patch import set_skip_padding  # noqa: E402


# ---------------------------------------------------------------------------------------------------------------------
# GraphedStep / GraphedForward
# ---------------------------------------------------------------------------------------------------------------------
def _bert_cfg(layers=1):
    return types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=layers,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12)


def _vilbert_cfg():
    return types.SimpleNamespace(
        hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=1, v_hidden_size=64,
        v_num_attention_heads=1, v_intermediate_size=128, v_num_hidden_layers=1, bi_hidden_size=64, bi_num_attention_heads=1,
        v_biattention_id=[0], t_biattention_id=[0], hidden_dropout_prob=0.0, v_hidden_dropout_prob=0.0,
        attention_probs_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0)


def _root():
    root = torch.nn.Module()
    root.a = M.B200BertEncoder(_bert_cfg())
    root.c = M.B200ViLBertEncoder(_vilbert_cfg())
    return root


@pytest.fixture
def no_capture(monkeypatch):
    seen = []
    monkeypatch.setattr(GraphedStep, "_capture", lambda self, *a: seen.append(graphs.static_rows_active()))
    return seen


SKIP = ("GraphedStep: the model has skip_padding encoders, which read the token count on the host and cannot be captured; "
        "turn them off with mmf_b200.patch.set_skip_padding(model, False)")
TAIL = ("GraphedStep: the model has skip_padding encoders with pack_tail set, which read the token count on the host for "
        "calls with a causal tail even under static_rows, so they cannot be captured; turn them off with "
        "mmf_b200.patch.set_skip_padding(model, False)")
STREAMS = ("GraphedStep: the model has two-stream encoders with pack_streams set, which read the token counts on the "
           "host%s and cannot be captured; turn them off with "
           "mmf_b200.patch.set_skip_padding(model, False, two_stream=True)")


@pytest.mark.parametrize("device_plan", [False, True])
def test_graphed_step_with_and_without_device_plan(no_capture, device_plan):
    batch = {"x": torch.zeros(1)}
    tail = _root()
    set_skip_padding(tail, True, causal=True, device_plan=device_plan)
    streams = _root()
    set_skip_padding(streams, True, two_stream=True, device_plan=device_plan)
    only_streams = _root()
    set_skip_padding(only_streams, True, two_stream=True, device_plan=device_plan)
    set_skip_padding(only_streams, False)                 # single-stream runners off, the two-stream one still packed
    only_streams.c._runner.pack_streams = True
    # without static_rows every refusal is today's, device_plan or not
    for root, msg in ((tail, SKIP), (streams, SKIP), (only_streams, STREAMS % "")):
        with pytest.raises(RuntimeError) as e:
            GraphedStep(root, lambda b: None, batch)
        assert str(e.value) == msg
    if not device_plan:
        for root, msg in ((tail, TAIL), (streams, STREAMS % " even under static_rows")):
            with pytest.raises(RuntimeError) as e:
                GraphedStep(root, lambda b: None, batch, static_rows=True)
            assert str(e.value) == msg
        assert no_capture == []
        return
    for root in (tail, streams, only_streams):
        GraphedStep(root, lambda b: None, batch, static_rows=True)
    assert no_capture == [True, True, True]
    # the refusals GraphedForward shares with GraphedStep accept them as well, and GraphedTaskSteps never does
    for root in (tail, streams):
        graphs._check_capturable("GraphedForward", root, True)
        with pytest.raises(RuntimeError):
            graphs._check_capturable("GraphedForward", root, False)
        with pytest.raises(RuntimeError):
            graphs._check_runners("GraphedTaskSteps", root, False)


def test_set_skip_padding_counts_runners_as_before():
    for kw in ({}, {"causal": True}, {"two_stream": True}, {"two_stream": True, "causal": True}):
        a, b = _root(), _root()
        assert set_skip_padding(a, True, **kw) == set_skip_padding(b, True, device_plan=True, **kw)
        assert not a.a._runner.device_plan and b.a._runner.device_plan
        assert b.c._runner.device_plan == bool(kw.get("two_stream"))
        assert set_skip_padding(b, False, **kw) == set_skip_padding(a, False, **kw)
        assert not b.a._runner.device_plan


# ---------------------------------------------------------------------------------------------------------------------
# the plan rules against today's host plans
# ---------------------------------------------------------------------------------------------------------------------
def _check_against(got, rows, cu, B, S):
    """a reference plan against a host packing given by its source rows and cu"""
    cu_r, pack_map, unpack_map = got
    n = rows.numel()
    assert torch.equal(cu_r, cu.to(torch.int32)) and int(cu_r[B]) == n
    assert torch.equal(pack_map[:n].long(), rows) and bool((pack_map[n:] == -1).all())
    want = torch.full((B * S,), -1, dtype=torch.int32)
    want[rows] = torch.arange(n, dtype=torch.int32)
    assert torch.equal(unpack_map, want)


def _host_rows(packing, B, S):
    if packing is None or packing.rows is None:
        return torch.arange(B * S), torch.arange(B + 1, dtype=torch.int32) * S
    return packing.rows, packing.varlen.cu_seqlens


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("B,S", [(1, 7), (5, 33), (9, 64), (3, 130)])
def test_single_stream_plan_is_the_static_plan(seed, B, S):
    g = torch.Generator().manual_seed(seed)
    valid = PR.random_valid(B, S, g, kinds=[("empty", 0)] if seed % 2 else [("full", B - 1)])
    for mask in (PR.masks_of(valid), PR.masks_of(valid, soft=-1.0)):
        cu, pm, um = PR.plan([mask], B, [S])[0]
        st = M._plan_packing_static(mask, B, S)
        assert torch.equal(cu, st.varlen.cu_seqlens) and torch.equal(pm, st.pack_map) and torch.equal(um, st.unpack_map)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("B,S,T", [(1, 9, 1), (4, 40, 12), (7, 70, 70), (3, 129, 64)])
def test_causal_tail_plan_is_the_eager_tail_plan(seed, B, S, T):
    g = torch.Generator().manual_seed(seed)
    valid = PR.random_valid(B, S, g, kinds=[("empty", 0)])
    mask = PR.masks_of(valid)
    mask[:, S - T:] = torch.where(torch.rand(B, T, generator=g) < 0.5, -10000.0, 0.0)   # never read in the tail
    got = PR.plan([mask], B, [S], causal_len=T)[0]
    rows, cu = _host_rows(M._plan_packing(M._tail_kept(mask, T), B, S), B, S)
    _check_against(got, rows, cu, B, S)
    assert bool((got[0][1:] - got[0][:-1] >= T).all())                        # every sample keeps its tail


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("B,Sa,Sb,none", [(1, 5, 9, None), (6, 20, 37, None), (8, 64, 36, None), (5, 20, 30, 0),
                                          (5, 20, 30, 1)])
def test_two_stream_plan_is_the_eager_plan_without_one_sided_samples(seed, B, Sa, Sb, none):
    g = torch.Generator().manual_seed(seed)
    va, vb = PR.random_valid(B, Sa, g), PR.random_valid(B, Sb, g)
    both = va.any(1) & vb.any(1)
    if none is None:
        va[~both], vb[~both] = False, False          # every sample has tokens in both streams or in neither
    else:
        (va, vb)[none][:] = True
        (vb, va)[none][~(vb, va)[none].any(1)] = True
    masks = [PR.masks_of(va), PR.masks_of(vb)]
    if none is not None:
        masks[none] = None
    got = PR.plan(masks, B, [Sa, Sb])
    host = M.plan_two_stream(masks[0], masks[1], B, Sa, Sb, "cpu")
    if host == "empty":
        assert all(int(p[0][B]) == 0 for p in got)
        return
    for k, S in enumerate((Sa, Sb)):
        if masks[k] is None:
            assert got[k] is None
            continue
        rows, cu = _host_rows(None if host is None else host[k], B, S)
        _check_against(got[k], rows, cu, B, S)


def test_two_stream_one_sided_and_empty_samples():
    B, Sa, Sb = 4, 6, 5
    va, vb = torch.zeros(B, Sa, dtype=torch.bool), torch.zeros(B, Sb, dtype=torch.bool)
    va[0, :2] = True                                    # sample 0: tokens in a only -> b keeps all 5
    vb[1, 1:4] = True                                   # sample 1: tokens in b only -> a keeps all 6
    va[2, 3] = True                                     # sample 2: both
    vb[2, 0] = True
    # sample 3: neither -> keeps nothing
    a, b = PR.plan([PR.masks_of(va), PR.masks_of(vb)], B, [Sa, Sb])
    assert a[0].tolist() == [0, 2, 8, 9, 9] and b[0].tolist() == [0, 5, 8, 9, 9]
    assert M.plan_two_stream(PR.masks_of(va), PR.masks_of(vb), B, Sa, Sb, "cpu") is None     # today: dense
    # against an unpadded stream every sample of the masked one is one-sided or full: it keeps every row
    a_only = PR.plan([PR.masks_of(va), None], B, [Sa, Sb])
    assert a_only[1] is None and a_only[0][0].tolist() == [0, 2, 8, 9, 15]


# ---------------------------------------------------------------------------------------------------------------------
# per-stream counts in the bounded two-stream layers
# ---------------------------------------------------------------------------------------------------------------------
class Double(types.SimpleNamespace):
    """fake_kernels plus the bounded and packed entry points the two-stream layers call; every call records (kind, epi,
    rows, m_bound, k_bound)"""

    def __init__(self):
        super().__init__()
        self.calls = []
        for name in dir(FK):
            if not name.startswith("_"):
                setattr(self, name, getattr(FK, name))
        self.gemm, self.layernorm_fwd, self.layernorm_bwd, self.colsum = self._gemm, self._ln_fwd, self._ln_bwd, self._colsum

    def _gemm(self, a, b, *, m_bound=None, k_bound=None, **kw):
        self.calls.append(("gemm", kw.get("epi"), a.shape[0], m_bound, k_bound))
        return FK.gemm(a, b, **kw)

    def _ln_fwd(self, y, *a, m_bound=None, **kw):
        self.calls.append(("ln_fwd", None, y.shape[0], m_bound, None))
        return FK.layernorm_fwd(y, *a, **kw)

    def _ln_bwd(self, dx, *a, m_bound=None, **kw):
        self.calls.append(("ln_bwd", None, dx.shape[0], m_bound, None))
        return FK.layernorm_bwd(dx, *a, **kw)

    def _colsum(self, x, out):
        self.calls.append(("colsum", None, x.shape[0], None, None))
        return FK.colsum(x, out)

    def colsum_bounded(self, x, out, m_bound):
        self.calls.append(("colsum", None, x.shape[0], m_bound, None))
        out += x[:int(m_bound.reshape(-1)[0])].float().sum(0)
        return out

    def _segments(self, cu):
        cu = cu.tolist()
        return [(cu[b], cu[b + 1]) for b in range(len(cu) - 1)]

    def attention_varlen_fwd(self, q, k, v, cu, max_len, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False,
                             causal_len=0):
        return self.attention_varlen_cross_fwd(q, k, v, cu, cu, max_len, max_len, heads, out=out, save_lo=save_lo)

    def attention_varlen_bwd(self, dctx, q, k, v, ctx, lse2, cu, max_len, heads, drop_mask=None, drop_scale=1.0, dq=None,
                             dk=None, dv=None, ctx_lo=None, causal_len=0):
        return self.attention_varlen_cross_bwd(dctx, q, k, v, ctx, lse2, cu, cu, max_len, max_len, heads, dq=dq, dk=dk, dv=dv)

    def attention_varlen_cross_fwd(self, q, k, v, cu_q, cu_kv, max_q, max_kv, heads, drop_mask=None, drop_scale=1.0,
                                   out=None, save_lo=False):
        self.calls.append(("attn", None, q.shape[0], None, None))
        ctx = out if out is not None else torch.full_like(q, float("nan"))
        for (qs, qe), (ks, ke) in zip(self._segments(cu_q), self._segments(cu_kv)):
            if qe > qs:
                ctx[qs:qe] = FK.attention_fwd(q[qs:qe], k[ks:ke], v[ks:ke], 1, heads, qe - qs, ke - ks)[0]
        lse2 = torch.zeros(heads, q.shape[0])
        return (ctx, lse2, torch.zeros_like(ctx)) if save_lo else (ctx, lse2)

    def attention_varlen_cross_bwd(self, dctx, q, k, v, ctx, lse2, cu_q, cu_kv, max_q, max_kv, heads, drop_mask=None,
                                   drop_scale=1.0, dq=None, dk=None, dv=None, ctx_lo=None):
        for (qs, qe), (ks, ke) in zip(self._segments(cu_q), self._segments(cu_kv)):
            if qe > qs and ke > ks:
                c, l2 = FK.attention_fwd(q[qs:qe], k[ks:ke], v[ks:ke], 1, heads, qe - qs, ke - ks)
                FK.attention_bwd(dctx[qs:qe], q[qs:qe], k[ks:ke], v[ks:ke], c, l2, 1, heads, qe - qs, ke - ks,
                                 dq=dq[qs:qe], dk=dk[ks:ke], dv=dv[ks:ke])
        return dq, dk, dv

    def gather_rows(self, x, idx, out=None):
        r = torch.where(idx[:, None] >= 0, x[idx.long().clamp_min(0)], torch.zeros((), dtype=x.dtype))
        return r.to(torch.bfloat16)

    def plan_packing(self, masks, B, lens, causal_len=0):
        self.calls.append(("plan", None, B, None, None))
        return PR.plan(masks, B, lens, causal_len)


@pytest.fixture
def double(monkeypatch):
    d = Double()
    monkeypatch.setattr(E, "F", d)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    return d


def _lxmert_encoder():
    from mmf_b200.lxmert import B200LXMERTEncoder
    cfg = types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, l_layers=1, x_layers=1,
                                r_layers=1, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, visual_feat_dim=16,
                                visual_pos_dim=4, skip_padding=True)
    return B200LXMERTEncoder(cfg)


def _two_stream_call(model, x0, x1, m0, m1):
    if isinstance(model, M.B200ViLBertEncoder):
        t, v, _ = model(x0, x1, m0, None, m1, output_all_encoded_layers=False)
        return t[-1], v[-1]
    return tuple(M.run_two_stream_encoder(model._runner, x0, x1, m0, m1, True)[:2])


@pytest.mark.parametrize("kind", ["vilbert", "lxmert"])
def test_bounded_two_stream_layers_take_their_own_streams_count(double, kind):
    torch.manual_seed(0)
    if kind == "vilbert":
        model = M.B200ViLBertEncoder(_vilbert_cfg())
    else:
        model = _lxmert_encoder()
    set_skip_padding(model, True, two_stream=True, device_plan=True)
    model.train()
    B, T, R = 3, 10, 7
    vt = torch.ones(B, T, dtype=torch.bool)
    vt[0, 6:], vt[1, 2:] = False, False
    vr = torch.ones(B, R, dtype=torch.bool)
    vr[2, 4:] = False
    mt, mr = PR.masks_of(vt), PR.masks_of(vr)
    x0 = torch.randn(B, T, 64, requires_grad=True)
    x1 = torch.randn(B, R, 64, requires_grad=True)

    def run(static):
        double.calls.clear()
        x0.grad = x1.grad = None
        with graphs.static_rows() if static else contextlib.nullcontext():
            o0, o1 = _two_stream_call(model, x0, x1, mt, mr)
        ((o0.float() * vt[..., None]).sum() + (o1.float() * vr[..., None]).sum()).backward()
        return o0.detach(), o1.detach(), x0.grad.clone(), x1.grad.clone(), list(double.calls)

    eager = run(False)
    assert all(c[3] is None and c[4] is None for c in eager[4])      # the eager packed path passes no bound
    assert not any(c[0] == "plan" for c in eager[4])
    static = run(True)
    calls = static[4]
    assert sum(c[0] == "plan" for c in calls) == 1                    # one planning launch per encoder call
    counts = {}
    for c in calls:
        if c[0] in ("plan", "attn"):
            continue
        bound = c[3] if c[3] is not None else c[4]
        assert bound is not None, c                                   # every GEMM, LayerNorm and column sum is bounded
        counts.setdefault(c[2], set()).add(id(bound))
        assert int(bound.reshape(-1)[0]) == int((vt if c[2] == B * T else vr).sum()), c
    assert set(counts) == {B * T, B * R} and all(len(v) == 1 for v in counts.values())
    assert counts[B * T] != counts[B * R]                             # each stream its own count
    # the same function on the valid rows
    for e, s, v in ((eager[0], static[0], vt), (eager[1], static[1], vr), (eager[2], static[2], vt), (eager[3], static[3], vr)):
        assert torch.allclose(e.float()[v], s.float()[v], atol=2e-2, rtol=2e-2)


def test_header_declares_the_planner():
    with open(os.path.join(os.path.dirname(HERE), "include", "mmfb200_plan.h")) as fh:
        txt = fh.read()
    assert "int mmfb_plan_packing(" in txt and "B <= 4096" in txt
    with open(os.path.join(os.path.dirname(HERE), "include", "mmfb200.h")) as fh:
        assert '#include "mmfb200_plan.h"' in fh.read()
