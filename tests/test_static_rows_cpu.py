"""Static-rows masked-LM loss on the CPU, over the kernel test double: the chunk loop of ops.linear_cross_entropy with a
device count hands every vocabulary-sized call its chunk's device bound, the head's loss and gradients
equal today's gathered path, GraphedStep refuses exactly what it refused without `static_rows` and accepts VinVL and
ViLT with it, and the C header declares the new entry points.  The kernels themselves run on the H100
(tests/test_static_rows_gpu.py).  Doubles for the new entry points live here, not in tests/fake_kernels.py."""
import math
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TILE = 128


def _rows(bound, M):
    b = min(max(int(bound.reshape(-1)[0]), 0), M)
    return b, min(M, -(-b // TILE) * TILE)


class Double(types.SimpleNamespace):
    """fake_kernels plus the new entry points; records every call that takes a device bound"""

    def __init__(self):
        super().__init__()
        self.calls = []
        for name in dir(FK):
            if not name.startswith("_"):
                setattr(self, name, getattr(FK, name))
        self.gemm = self._gemm

    def _gemm(self, a, b, *, m_bound=None, k_bound=None, out=None, **kw):
        if m_bound is None and k_bound is None:
            return FK.gemm(a, b, out=out, **kw)
        self.calls.append(("gemm", kw.get("epi"), m_bound, k_bound))
        if k_bound is not None:                    # weight gradient: K is the row count
            kb = min(-(-min(max(int(k_bound[0]), 0), a.shape[0]) // 64) * 64, a.shape[0])
            if kb:
                FK.gemm(a[:kb], b[:kb], out=out, **kw)
            return out
        M = a.shape[1] if kw.get("a_mn") else a.shape[0]
        _, r = _rows(m_bound, M)
        if out is None:
            out = torch.full((M, b.shape[1] if kw.get("b_mn") else b.shape[0]), float("nan"), dtype=torch.bfloat16)
        if r:
            out[:r] = FK.gemm(a[:r], b, **kw)
        return out

    def ce_rows_bounded(self, logits, labels, ignore_index, scale, m_bound, loss_sum=None, row_loss=None):
        self.calls.append(("ce_rows", None, m_bound, None))
        _, r = _rows(m_bound, logits.shape[0])
        if r:
            FK.ce_rows(logits[:r], labels[:r], ignore_index, float(scale[0]), loss_sum if loss_sum is not None else
                       torch.zeros(()), row_loss[:r] if row_loss is not None else None)
        return logits

    def colsum_bounded(self, x, out, m_bound):
        self.calls.append(("colsum", None, m_bound, None))
        b, _ = _rows(m_bound, x.shape[0])
        out += x[:b].float().sum(0)
        return out

    def select_rows(self, labels, ignore_index):
        from mmf_b200.functional import SelectedRows
        M = labels.numel()
        idx = torch.nonzero(labels != ignore_index).reshape(-1)
        n = idx.numel()
        state = torch.full((2 + 2 * M,), -1, dtype=torch.int32)
        state[0] = n
        state[1:2] = torch.tensor([1.0 / max(n, 1)], dtype=torch.float32).view(torch.int32)
        state[2:2 + n] = idx.to(torch.int32)
        state[2 + M + idx] = torch.arange(n, dtype=torch.int32)
        out = torch.full((M,), ignore_index, dtype=torch.int64)
        out[:n] = labels[idx]
        return SelectedRows(state, out)

    def gather_rows(self, x, idx, out=None):
        i = idx.long()
        res = torch.zeros(i.numel(), x.shape[1], dtype=torch.bfloat16)
        res[i >= 0] = x[i[i >= 0]]
        return res


@pytest.fixture()
def double(monkeypatch):
    import mmf_b200.heads as HD
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    d = Double()
    monkeypatch.setattr(OPS, "F", d)
    monkeypatch.setattr(HD, "F", d)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(HD, "_require_cuda", lambda t, what: None)
    return d


@pytest.mark.parametrize("capacity,count", [(5000, 2100), (5000, 0), (300, 300), (4096, 2048), (4097, 4097),
                                            (4097, 2048), (2049, 1), (129, 128)])
def test_chunk_loop_hands_every_vocabulary_call_its_device_bound(double, capacity, count):
    from mmf_b200 import lib, ops
    g = torch.Generator().manual_seed(capacity + count)
    V, H, chunk = 72, 64, 2048
    labels = torch.full((capacity,), -1, dtype=torch.int64)
    labels[:count] = torch.randint(0, V, (count,), generator=g)
    h = torch.zeros(capacity, H)
    h[:count] = torch.randn(count, H, generator=g)
    h.requires_grad_(True)
    w = (torch.randn(V, H, generator=g) * 0.1).requires_grad_(True)
    b = (torch.randn(V, generator=g) * 0.1).requires_grad_(True)
    cnt = torch.tensor([count], dtype=torch.int32)
    scale = torch.tensor([1.0 / max(count, 1)], dtype=torch.float32)
    loss = ops.linear_cross_entropy(h, w, b, labels, -1, chunk, count=cnt, scale=scale)
    chunks = math.ceil(capacity / chunk)
    kinds = [(c[0], c[1]) for c in double.calls]
    per_chunk = [("gemm", lib.EPI_BIAS), ("ce_rows", None), ("gemm", lib.EPI_BIAS), ("gemm", lib.EPI_ATOMIC_F32),
                 ("colsum", None)]
    assert kinds == per_chunk * chunks
    for i in range(chunks):
        want = min(max(count - i * chunk, 0), chunk)
        for c in double.calls[5 * i:5 * i + 5]:
            bound = c[2] if c[2] is not None else c[3]
            assert bound.dtype == torch.int32 and bound.numel() == 1 and int(bound[0]) == want, (i, c)
    loss.backward()
    # today's path on the labelled rows alone
    h2, w2, b2 = h.detach()[:max(count, 1)].clone().requires_grad_(True), w.detach().clone().requires_grad_(True), \
        b.detach().clone().requires_grad_(True)
    if count:
        ref = ops.linear_cross_entropy(h2, w2, b2, labels[:count], -1, chunk)
        ref.backward()
        assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
        assert torch.equal(h.grad[:count], h2.grad[:count])
        assert torch.allclose(w.grad, w2.grad, atol=1e-6) and torch.allclose(b.grad, b2.grad, atol=1e-6)
    else:
        assert float(loss) == 0.0 and not w.grad.any() and not b.grad.any()
    assert not h.grad[count:].any()


def test_static_rows_context_routes_both_gathering_positions(double):
    from mmf_b200 import graphs
    from mmf_b200.heads import B200BertPreTrainingHeads, masked_lm_loss
    from mmf_b200.models import ConfigNode
    torch.manual_seed(0)
    cfg = ConfigNode(dict(hidden_size=64, vocab_size=40, layer_norm_eps=1e-12, initializer_range=0.02))
    cls = B200BertPreTrainingHeads(cfg)
    seq = torch.randn(3, 7, 64)
    labels = torch.full((3, 7), -1, dtype=torch.long)
    labels[0, 2], labels[1, 5], labels[2, 0] = 4, 39, 0
    ref, _ = masked_lm_loss(cls, seq, labels, positions="fused")
    assert not graphs.static_rows_active()
    for positions in ("fused", "masked"):
        with graphs.static_rows():
            assert graphs.static_rows_active()
            loss, logits = masked_lm_loss(cls, seq, labels, positions=positions)
        assert logits is None and abs(float(loss) - float(ref)) <= 1e-5 * float(ref)
    assert not graphs.static_rows_active()
    with graphs.static_rows():
        none, _ = masked_lm_loss(cls, seq.requires_grad_(True), torch.full((3, 7), -1, dtype=torch.long),
                                 positions="fused")
    none.backward()
    assert float(none) == 0.0 and not seq.grad.any()


def _model(name, case):
    mod = __import__("test_%s_model_cpu" % name)
    gold = torch.load(os.path.join(GOLD, "%s_model.pt" % name), weights_only=False)
    import mmf_b200.models as MD
    return mod._build(MD, gold, case)


@pytest.fixture()
def models(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.engine as E
    import mmf_b200.heads as HD
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.vilbert as VB
    import mmf_b200.vinvl as VV
    for mod in (E, OPS, EM):
        monkeypatch.setattr(mod, "F", FK)
    for mod in (M, EM, VB, HD, VV):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    import mmf_b200.mmft  # noqa: F401
    return {"vinvl": _model("vinvl", "pretraining"), "vilt": _model("vilt", "pretraining"), "uniter": _model("uniter", "pretraining")}


def test_graphed_step_refuses_without_static_rows_and_accepts_vinvl_and_vilt_with_it(models, monkeypatch):
    from mmf_b200 import graphs
    seen = []
    monkeypatch.setattr(graphs.GraphedStep, "_capture", lambda self, *a: seen.append(graphs.static_rows_active()))
    for name in ("vinvl", "vilt", "uniter"):
        with pytest.raises(RuntimeError, match="cannot be captured"):
            graphs.GraphedStep(models[name], lambda b: None, {})
    assert seen == []
    for name in ("vinvl", "vilt"):
        graphs.GraphedStep(models[name], lambda b: None, {}, static_rows=True)
    assert seen == [True, True] and not graphs.static_rows_active()
    with pytest.raises(RuntimeError, match="UNITER draws its task and region masks on the host"):
        graphs.GraphedStep(models["uniter"], lambda b: None, {}, static_rows=True)


def test_header_lists_the_new_entry_points():
    from mmf_b200 import lib
    syms = lib.header_symbols()
    for name in ("mmfb_gemm_bounded", "mmfb_select_rows", "mmfb_gather_rows", "mmfb_ce_rows_bounded",
                 "mmfb_colsum_bounded"):
        assert name in syms
        assert hasattr(lib.LIB, name)
