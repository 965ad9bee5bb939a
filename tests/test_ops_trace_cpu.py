"""Launch trace of the front-end and head autograd functions of mmf_b200.ops on the CPU: every call they (and the heads
around them) make into mmf_b200.functional, in order, forward and backward, compared with tests/golden/ops_trace.json.

The recorder is the engine trace's (tests/test_engine_trace_cpu.py): per call the entry point, every non-tensor argument
and each tensor operand's provenance, with the arguments bound to the signature of the real mmf_b200.functional entry
point.  The kernels are the test double: tests/fake_kernels.py, the bounded entry points of tests/test_static_rows_cpu.py,
and torch restatements here of the bounded GELU GEMM, the bounded LayerNorm and the KL / MSE region-loss row kernels.

Regenerate the fixture (only when the launches are meant to change) with
    MMFB_WRITE_TRACE=1 python -m pytest tests/test_ops_trace_cpu.py
"""
import functools
import inspect
import json
import os
import types

import pytest
import torch

import fake_kernels as FK
import test_engine_trace_cpu as ET
import test_static_rows_cpu as SR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ops_trace.json")


def _kl_rows_bounded(logits, V, target, tgt_idx, m_bound, scale, row_loss):
    b, r = SR._rows(m_bound, logits.shape[0])
    z = logits[:b, :V].float()
    t = target[tgt_idx[:b].long()].float()
    logp = torch.log_softmax(z, dim=-1)
    row_loss[:b] = torch.where(t > 0, t * (torch.log(t.clamp_min(1e-30)) - logp), torch.zeros_like(t)).sum(-1)
    d = torch.zeros(r, logits.shape[1])
    d[:b, :V] = (logp.exp() * t.sum(-1, keepdim=True) - t) * float(scale[0])
    logits[:r] = d.to(torch.bfloat16)
    return logits


def _mse_rows_bounded(pred, target, tgt_idx, m_bound, scale, row_loss):
    b, r = SR._rows(m_bound, pred.shape[0])
    e = pred[:b].float() - target[tgt_idx[:b].long()].float()
    row_loss[:b] = (e * e).sum(-1)
    d = torch.zeros(r, pred.shape[1])
    d[:b] = 2.0 * e * float(scale[0])
    pred[:r] = d.to(torch.bfloat16)
    return pred


def _layernorm_fwd(y, gamma, beta, eps=FK.LN_EPS, drop_mask=None, drop_scale=1.0, out=None, m_bound=None):
    if m_bound is None:
        return FK.layernorm_fwd(y, gamma, beta, eps, drop_mask, drop_scale, out)
    b, _ = SR._rows(m_bound, y.shape[0])
    x, mean, rstd = torch.zeros_like(y), torch.zeros(y.shape[0]), torch.zeros(y.shape[0])
    if b:
        x[:b], mean[:b], rstd[:b] = FK.layernorm_fwd(y[:b], gamma, beta, eps)
    return x, mean, rstd


def _layernorm_bwd(dx, y, mean, rstd, gamma, dgamma, dbeta, dbias=None, dx2=None, drop_mask=None, drop_scale=1.0,
                   need_dz=True, m_bound=None):
    if m_bound is None:
        return FK.layernorm_bwd(dx, y, mean, rstd, gamma, dgamma, dbeta, dbias, dx2, drop_mask, drop_scale, need_dz)
    b, _ = SR._rows(m_bound, y.shape[0])
    dy = torch.zeros_like(y)
    if b:
        dy[:b], _ = FK.layernorm_bwd(dx[:b], y[:b], mean[:b], rstd[:b], gamma, dgamma, dbeta)
    return dy, dy


def _double():
    """test_static_rows_cpu's Double, with the bounded GELU GEMM, the bounded LayerNorm and the region-loss rows added"""
    d = SR.Double()
    bounded_gemm = d.gemm

    def gemm(a, b, *, m_bound=None, epi=FK.lib.EPI_BIAS, **kw):
        if m_bound is None or epi != FK.lib.EPI_BIAS_GELU:
            return bounded_gemm(a, b, m_bound=m_bound, epi=epi, **kw)
        _, r = SR._rows(m_bound, a.shape[0])
        u, h = (torch.zeros(a.shape[0], b.shape[0], dtype=torch.bfloat16) for _ in range(2))
        if r:
            u[:r], h[:r] = FK.gemm(a[:r], b, epi=epi, **kw)
        return u, h
    d.gemm = gemm
    d.layernorm_fwd, d.layernorm_bwd = _layernorm_fwd, _layernorm_bwd
    d.kl_rows_bounded, d.mse_rows_bounded = _kl_rows_bounded, _mse_rows_bounded
    return d


def _base():
    """the double's entry points, each carrying the signature of the real mmf_b200.functional entry point it stands for"""
    import mmf_b200.functional as REAL
    d = _double()
    ns = types.SimpleNamespace()
    for name in dir(d):
        impl = getattr(d, name)
        if name.startswith("_") or not callable(impl) or not inspect.isfunction(getattr(REAL, name, None)):
            continue
        setattr(ns, name, functools.wraps(getattr(REAL, name))(lambda *a, _impl=impl, **k: _impl(*a, **k)))
    return ns


# ---- scenarios: each runs forward and backward and returns its outputs -------------------------------------------------
def _p(*shape, grad=True):
    return (torch.randn(*shape) * 0.2).requires_grad_(grad)


def _run(y, *inputs):
    if y.dim():
        y = (y.float() * torch.randn(y.shape)).sum()
    y.backward()
    return [y] + [t.grad for t in inputs if t.requires_grad]


# A weight gradient of a 16 x 2560 output over 512 rows gets 8 splits and one of 2560 x 16 gets 6 (best_splits), so the
# wide shapes below also pin the order of best_splits' arguments.
def linear_variants(OPS, HD, MMFT):
    x, w, b = _p(512, 2560), _p(16, 2560), _p(16)
    out = _run(OPS.linear(x, w, b), x, w, b)
    x, w = _p(512, 2560), _p(16, 2560)
    out += _run(OPS.linear(x, w), x, w)
    x, w, b = _p(512, 2560), _p(16, 2560, grad=False), _p(16)
    out += _run(OPS.linear(x, w, b), x, b)
    for fn in (OPS.linear_relu, OPS.linear_gelu):
        x, w, b = _p(512, 2560), _p(16, 2560), _p(16)
        out += _run(fn(x, w, b), x, w, b)
        x, w, b = _p(512, 2560), _p(16, 2560, grad=False), _p(16)
        out += _run(fn(x, w, b), x, b)
    return out


def linear_t_variants(OPS, HD, MMFT):
    x, w, b = _p(512, 2560), _p(2560, 16), _p(16)
    out = _run(OPS.linear_t(x, w, b), x, w, b)
    x, w, b = _p(512, 2560), _p(2560, 16, grad=False), _p(16)
    return out + _run(OPS.linear_t(x, w, b), x, b)


def linear_any_padded(OPS, HD, MMFT):
    x, w, b = _p(24, 5), _p(3, 5), _p(3)
    out = _run(OPS.linear_any(x, w, b), x, w, b)
    x, w = _p(24, 5), _p(3, 5)
    return out + _run(OPS.linear_any(x, w), x, w)


def layer_norm(OPS, HD, MMFT):
    x, g, b = _p(24, 32), _p(32), _p(32)
    return _run(OPS.layer_norm(x, g, b, 1e-5), x, g, b)


def linear_cross_entropy_chunks(OPS, HD, MMFT):
    h, w = _p(1100, 2560), _p(45, 2560)
    labels = torch.randint(0, 45, (1100,))
    labels[::3] = -1
    out = _run(OPS.linear_cross_entropy(h, w, None, labels, -1, chunk_rows=512), h, w)
    h, w, b = _p(1100, 2560), _p(45, 2560), _p(45)
    return out + _run(OPS.linear_cross_entropy(h, w, b, labels, -1, chunk_rows=512), h, w, b)


def _static_mlm(HD, count, deterministic):
    from mmf_b200.models import ConfigNode
    pred = HD.B200BertLMPredictionHead(ConfigNode(dict(hidden_size=32, vocab_size=45, layer_norm_eps=1e-12)))
    seq = _p(3, 700, 32)
    labels = torch.full((3 * 700,), -1, dtype=torch.long)
    labels[torch.randperm(3 * 700)[:count]] = torch.randint(0, 45, (count,))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        return _run(HD.static_masked_lm_loss(pred, seq, labels.view(3, 700)), seq, *pred.parameters())
    finally:
        torch.use_deterministic_algorithms(prev)


def static_mlm_none(OPS, HD, MMFT):
    return _static_mlm(HD, 0, False)


def static_mlm_part(OPS, HD, MMFT):
    return _static_mlm(HD, 2090, False)


def static_mlm_all(OPS, HD, MMFT):
    return _static_mlm(HD, 2100, False)


def static_mlm_part_deterministic(OPS, HD, MMFT):
    return _static_mlm(HD, 1000, True)


def static_mlm_all_deterministic(OPS, HD, MMFT):
    return _static_mlm(HD, 2100, True)


def _region_inputs(D, B=4, T=5, R=128):
    seq = _p(B, T + R, 32)
    masks = torch.zeros(B, T + R, dtype=torch.bool)
    masks[0, T + 1], masks[1, T:T + 30], masks[3, -1] = True, True, True
    return seq, masks, torch.softmax(torch.randn(B, R, D), -1)


def _static_head(head, seq, masks, targets, keys):
    from mmf_b200 import graphs
    with graphs.static_rows():
        loss = head(seq, processed_sample_list=dict(zip(keys, (targets, masks))))["losses"]
    return _run(next(iter(loss.values())), seq, *head.parameters())


def static_mrc_kl(OPS, HD, MMFT):
    seq, masks, targets = _region_inputs(2557)
    head = MMFT.MRCHead(hidden_size=32, label_dim=2557)
    return _static_head(head, seq, masks, targets, ("region_class", "image_region_mask"))


def static_mrc_cross_entropy(OPS, HD, MMFT):
    seq, masks, targets = _region_inputs(2557)
    head = MMFT.MRCHead(hidden_size=32, label_dim=2557, use_kl=False)
    return _static_head(head, seq, masks, targets, ("region_class", "image_region_mask"))


def static_mrfr(OPS, HD, MMFT):
    seq, masks, targets = _region_inputs(2560)
    head = MMFT.MRFRHead(torch.nn.Parameter(torch.randn(32, 2560) * 0.2), hidden_size=32, img_dim=2560)
    return _static_head(head, seq, masks, targets, ("mrfr_region_target", "mrfr_region_mask"))


SCENARIOS = [linear_variants, linear_t_variants, linear_any_padded, layer_norm, linear_cross_entropy_chunks,
             static_mlm_none, static_mlm_part, static_mlm_all, static_mlm_part_deterministic,
             static_mlm_all_deterministic, static_mrc_kl, static_mrc_cross_entropy, static_mrfr]


def _trace(scenario, monkeypatch):
    import mmf_b200.heads as HD
    import mmf_b200.mmft as MMFT
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    rec = ET._Recorder(_base())
    for mod in (OPS, HD, MMFT):
        monkeypatch.setattr(mod, "F", rec)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(HD, "_require_cuda", lambda t, what: None)
    torch.manual_seed(0)
    outs = scenario(OPS, HD, MMFT)
    return {"outputs": rec.describe(outs, known_only=True), "calls": rec.calls}


def _dump(traces):
    """one call per line, so that a difference reads as a line diff"""
    parts = []
    for name, t in traces.items():
        calls = ",\n".join(json.dumps(c, separators=(",", ":"), sort_keys=True) for c in t["calls"])
        parts.append("%s: {\"outputs\": %s,\n\"calls\": [\n%s]}" % (json.dumps(name), json.dumps(t["outputs"]), calls))
    return "{\n" + ",\n".join(parts) + "\n}\n"


def test_ops_launch_trace_matches_golden(monkeypatch):
    traces = {}
    for sc in SCENARIOS:
        with monkeypatch.context() as mp:
            traces[sc.__name__] = json.loads(json.dumps(_trace(sc, mp)))      # the JSON form: tuples become lists
    if os.environ.get("MMFB_WRITE_TRACE"):
        with open(GOLDEN, "w") as f:
            f.write(_dump(traces))
        pytest.skip("wrote %s" % GOLDEN)
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert sorted(golden) == sorted(traces)
    for name, t in traces.items():
        g = golden[name]
        for i, (got, want) in enumerate(zip(t["calls"], g["calls"])):
            assert got == want, "%s: call %d differs\n got  %s\n want %s" % (name, i, got, want)
        assert len(t["calls"]) == len(g["calls"]), name
        assert t["outputs"] == g["outputs"], name
