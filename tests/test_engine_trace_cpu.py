"""Launch trace of the encoders on the CPU: every call the engine makes into mmf_b200.functional, in order, for the BERT,
ViT, ViLBERT and LXMERT encoders in dense and packed mode, forward and backward, compared with tests/golden/engine_trace.json.

The kernels are the test double (tests/fake_kernels.py, with the torch restatements of the packed and probabilities entry
points from the two-stream and probabilities tests) behind a recording wrapper installed as `engine.F`.  Per call it
stores the entry point, every non-tensor argument (dropout draws: the Philox seed relative to the scenario's first seed,
and the offset), and for every tensor operand its provenance rather than its values: which earlier call produced it, or
which host-side tensor (input, parameter buffer, allocation) in order of first use, with the view offset, shape, stride
and dtype.  So a refactor of the host code that launches the same kernels with the same operands in the same order and
draws the same dropout bits passes, and one that swaps two operands, reorders two launches or changes a draw fails,
independently of floating-point rounding.  The data-parallel bucket boundaries (`step_offsets`) of each runner are
recorded too.

Regenerate the fixture (only when the launches are meant to change) with
    MMFB_WRITE_TRACE=1 python -m pytest tests/test_engine_trace_cpu.py
"""
import inspect
import json
import os
import types

import pytest
import torch

import fake_kernels as FK
import test_attention_probs_cpu as TAP
import test_skip_padding_two_stream_cpu as TS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "engine_trace.json")
_DT = {torch.bfloat16: "bf16", torch.float32: "f32", torch.int32: "i32", torch.int64: "i64", torch.bool: "b8"}


class _Recorder:
    """Stands in for mmf_b200.functional: forwards to `base` and appends one entry per call to `calls`."""

    def __init__(self, base):
        self._base = base
        self.calls = []
        self._labels = {}          # storage address -> label
        self._keep = []            # every labelled tensor stays alive, so no address is reused within a scenario
        self._n_host = 0
        self._seed0 = None

    def label(self, t):
        """provenance of a tensor: the call output or the host tensor (by order of first use) that owns its storage"""
        if t.numel() == 0:
            return "empty"
        key = t.untyped_storage().data_ptr()
        if key not in self._labels:
            self._labels[key] = "h%d" % self._n_host
            self._n_host += 1
            self._keep.append(t)
        return self._labels[key]

    def describe(self, v, known_only=False):
        if torch.is_tensor(v):
            if known_only and v.numel() and v.untyped_storage().data_ptr() not in self._labels:
                lab = "?"
            else:
                lab = self.label(v)
            return "%s@%d %s %s %s" % (lab, v.storage_offset(), "x".join(map(str, v.shape)),
                                       ",".join(map(str, v.stride())), _DT.get(v.dtype, str(v.dtype)))
        if isinstance(v, (list, tuple)):
            return [self.describe(x, known_only) for x in v]
        if isinstance(v, (torch.dtype, torch.device)):
            return str(v)
        return v

    def _register(self, out, prefix):
        if torch.is_tensor(out):
            if out.numel() and out.untyped_storage().data_ptr() not in self._labels:
                self._labels[out.untyped_storage().data_ptr()] = prefix
                self._keep.append(out)
        elif isinstance(out, (list, tuple)):
            for i, o in enumerate(out):
                self._register(o, "%s.%d" % (prefix, i))

    def __getattr__(self, name):
        fn = getattr(self._base, name)
        if not inspect.isfunction(fn):
            return fn
        sig = inspect.signature(fn)

        def call(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            rec = {}
            for k, v in bound.arguments.items():
                if v is not None:
                    rec[k] = self.describe(v)
            if name == "dropout_bits":
                if self._seed0 is None:
                    self._seed0 = int(rec["seed"])
                rec["seed"] = int(rec["seed"]) - self._seed0
            out = fn(*args, **kwargs)
            self._register(out, "c%d" % len(self.calls))
            self.calls.append([name, rec])
            return out
        return call


def _base():
    ns = types.SimpleNamespace(**{k: getattr(FK, k) for k in dir(FK) if not k.startswith("__")})
    ns.attention_varlen_cross_fwd, ns.attention_varlen_cross_bwd = TS._fwd, TS._bwd
    ns.attention_varlen_fwd, ns.attention_varlen_bwd = TS._self_fwd, TS._self_bwd
    ns.attention_probs = TAP._attention_probs
    return ns


# ---- scenarios: each builds an encoder, runs it forward (and backward) and returns (module, outputs) --------------------
def _bert_cfg(**kw):
    return types.SimpleNamespace(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=2,
                                 hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, layer_norm_eps=1e-12, **kw)


def _mask(B, S, holes):
    valid = torch.ones(B, S, dtype=torch.bool)
    for b, sl in holes:
        valid[b, sl] = False
    return (~valid).float() * -10000.0


def _backward(outs, *inputs):
    loss = sum((o.float() * torch.randn(o.shape)).sum() for o in outs)
    loss.backward()
    return list(outs) + [i.grad for i in inputs]


def _bert(M, skip=False, attn=False, hidden=False, twice=False):
    enc = M.B200BertEncoder(_bert_cfg(skip_padding=skip)).train()
    x = torch.randn(3, 10, 64, requires_grad=True)
    add = _mask(3, 10, [(0, slice(7, None)), (1, slice(0, 2))])[:, None, None, :]
    outs = enc(x, add, output_attentions=attn, output_hidden_states=hidden)
    if twice:
        outs = enc(outs[0], add)
    res = _backward(outs[:1], x)
    return enc, res + [t for o in outs[1:] for t in o]


def bert_dense(M, LX):
    return _bert(M)


def bert_packed(M, LX):
    return _bert(M, skip=True)


def bert_attentions_hidden(M, LX):
    return _bert(M, attn=True, hidden=True)


def bert_twice(M, LX):
    return _bert(M, twice=True)


def vit_train(M, LX):
    from mmf_b200.vit import B200ViTEncoder
    enc = B200ViTEncoder(types.SimpleNamespace(hidden_size=64, num_hidden_layers=2, num_attention_heads=2,
                                               intermediate_size=128, hidden_dropout_prob=0.1,
                                               attention_probs_dropout_prob=0.1, layer_norm_eps=1e-12)).train()
    x = torch.randn(2, 9, 64, requires_grad=True)
    return enc, _backward([enc(x).last_hidden_state], x)


def _vilbert(M, skip=False):
    cfg = TS._vilbert_cfg(0.1, skip)
    cfg.visualization = True
    enc = M.B200ViLBertEncoder(cfg).train()
    vt, vi = TS._two_stream_valid()
    txt = torch.randn(4, 10, 64, requires_grad=True)
    img = torch.randn(4, 7, 128, requires_grad=True)
    return enc, txt, img, TS._add(vt)[:, None, None, :], TS._add(vi)[:, None, None, :]


def vilbert_dense(M, LX):
    enc, txt, img, tm, im = _vilbert(M)
    ot, oi, _ = enc(txt, img, tm, None, im, output_all_encoded_layers=False)
    return enc, _backward([ot[0], oi[0]], txt, img)


def vilbert_packed(M, LX):
    enc, txt, img, tm, im = _vilbert(M, skip=True)
    ot, oi, _ = enc(txt, img, tm, None, im, output_all_encoded_layers=False)
    return enc, _backward([ot[0], oi[0]], txt, img)


def vilbert_visualization(M, LX):
    enc, txt, img, tm, im = _vilbert(M)
    bt, bi, (at, av, ac) = enc(txt, img, tm, None, im, output_all_encoded_layers=True, output_all_attention_masks=True)
    ot, oi, (at2, av2, ac2) = enc(txt, img, tm, None, im, output_all_encoded_layers=False,
                                  output_all_attention_masks=True)
    return enc, _backward([ot[0], oi[0]], txt, img) + [bt, bi, at, av, ac, at2, av2, ac2]


def _lxmert(LX, skip, visn_mask=True):
    enc = LX.B200LXMERTEncoder(TS._lxmert_cfg(0.1, skip)).train()
    vt, vi = TS._two_stream_valid()
    if not visn_mask:
        vt[2, 0] = True           # every sample has text: otherwise the unmasked regions of sample 2 force the dense path
    lang = torch.randn(4, 10, 64, requires_grad=True)
    feats = torch.randn(4, 7, 32, requires_grad=True)
    vmask = TS._add(vi)[:, None, None, :] if visn_mask else None
    lo, vo = enc(lang, TS._add(vt)[:, None, None, :], (feats, torch.rand(4, 7, 4)), vmask)
    return enc, _backward([lo, vo], lang, feats)


def lxmert_dense(M, LX):
    return _lxmert(LX, False)


def lxmert_packed(M, LX):
    return _lxmert(LX, True)


def lxmert_packed_no_visn_mask(M, LX):
    return _lxmert(LX, True, visn_mask=False)


SCENARIOS = [bert_dense, bert_packed, bert_attentions_hidden, bert_twice, vit_train, vilbert_dense, vilbert_packed,
             vilbert_visualization, lxmert_dense, lxmert_packed, lxmert_packed_no_visn_mask]


def _trace(scenario, monkeypatch):
    import mmf_b200.ddp as D
    import mmf_b200.engine as E
    import mmf_b200.lxmert as LX
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    rec = _Recorder(_base())
    monkeypatch.setattr(E, "F", rec)
    monkeypatch.setattr(OPS, "F", rec)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(LX, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(M, "_SEED_COUNTER", [0])
    torch.manual_seed(0)
    module, outs = scenario(M, LX)
    offsets = {}
    for name, m in module.named_modules():
        r = m.__dict__.get("_runner")
        if r is not None:
            n = len(r.steps) if hasattr(r, "steps") else len(r.layers)
            offsets[name or "."] = [D.B200DataParallel._step_offset(r, j) for j in range(n)]
    return {"step_offsets": offsets, "outputs": rec.describe(outs, known_only=True), "calls": rec.calls}


def _dump(traces):
    """one call per line, so that a difference reads as a line diff"""
    parts = []
    for name, t in traces.items():
        head = json.dumps({k: t[k] for k in ("step_offsets", "outputs")}, separators=(",", ":"))
        calls = ",\n".join(json.dumps(c, separators=(",", ":"), sort_keys=True) for c in t["calls"])
        parts.append("%s: {\"head\": %s,\n\"calls\": [\n%s]}" % (json.dumps(name), head, calls))
    return "{\n" + ",\n".join(parts) + "\n}\n"


def test_launch_trace_matches_golden(monkeypatch):
    traces = {}
    for sc in SCENARIOS:
        with monkeypatch.context() as mp:
            t = json.loads(json.dumps(_trace(sc, mp)))          # the JSON form: tuples become lists
        traces[sc.__name__] = {"step_offsets": t["step_offsets"], "outputs": t["outputs"], "calls": t["calls"]}
    if os.environ.get("MMFB_WRITE_TRACE"):
        with open(GOLDEN, "w") as f:
            f.write(_dump(traces))
        pytest.skip("wrote %s" % GOLDEN)
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert sorted(golden) == sorted(traces)
    for name, t in traces.items():
        g = golden[name]
        assert t["step_offsets"] == g["head"]["step_offsets"], name
        for i, (got, want) in enumerate(zip(t["calls"], g["calls"])):
            assert got == want, "%s: call %d differs\n got  %s\n want %s" % (name, i, got, want)
        assert len(t["calls"]) == len(g["calls"]), name
        assert t["outputs"] == g["head"]["outputs"], name
