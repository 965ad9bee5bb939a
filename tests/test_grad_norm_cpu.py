"""B200AdamW.clip_grad_norm's host logic over a kernel test double defined here: which gradient buffers become segments
of the device table, when the table is rebuilt, the norm_type check, and the clip coefficient reaching exactly one
step().  Also: with arithmetic="torch" and weight_decay=0 the step is torch.optim.Adam's."""
import types

import pytest
import torch

import fake_kernels as FK


class _NormKernels:
    """contract of functional.grad_norm_table / grad_norm (fp64 sum of squares, torch's clip coefficient) and of
    functional.adamw's grad_scale_dev, recording what the optimizer hands them"""

    def __init__(self):
        self.tables, self.adamw_dev = [], []

    def grad_norm_table(self, grads):
        t = types.SimpleNamespace(grads=list(grads), ptrs=[g.data_ptr() for g in grads])
        self.tables.append(t)
        return t

    def grad_norm(self, table, max_norm, norm_type=2.0):
        assert norm_type == 2.0
        assert [g.data_ptr() for g in table.grads] == table.ptrs
        n = torch.stack([g.double().pow(2).sum() for g in table.grads]).sum().sqrt().float()
        return torch.stack([n, torch.clamp(max_norm / (n + 1e-6), max=1.0)])

    def adamw(self, *args, grad_scale=1.0, grad_scale_dev=None, **kw):
        self.adamw_dev.append(grad_scale_dev)
        if grad_scale_dev is not None:
            grad_scale = grad_scale_dev * grad_scale
        FK.adamw(*args, grad_scale=grad_scale, **kw)


@pytest.fixture()
def cpu_engine(monkeypatch):
    import mmf_b200.engine as E
    import mmf_b200.modules as M
    import mmf_b200.optim as OPT
    K = _NormKernels()
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPT, "F", K)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    yield types.SimpleNamespace(E=E, M=M, OPT=OPT, K=K)


class _Model(torch.nn.Module):
    """an engine encoder (parameters in a pack) plus a head outside it"""

    def __init__(self, M):
        super().__init__()
        cfg = types.SimpleNamespace(hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=2,
                                    hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12)
        self.encoder = M.B200BertEncoder(cfg)
        self.head = torch.nn.Linear(64, 3)

    def forward(self, x):
        return self.head(self.encoder(x, None)[0])


def _backward(model, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 5, 64, generator=g)
    (model(x) * torch.randn(2, 5, 3, generator=g) * scale).sum().backward()


def test_a_fully_owned_pack_is_one_segment_and_loose_gradients_follow(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, arithmetic="torch")
    _backward(model, 1)
    opt.clip_grad_norm(1.0)
    pack = model.encoder._runner.pack
    (t,) = cpu_engine.K.tables
    assert t.grads[0].data_ptr() == pack.grad.data_ptr() and t.grads[0].numel() == pack.total
    assert [g.data_ptr() for g in t.grads[1:]] == [model.head.weight.grad.data_ptr(), model.head.bias.grad.data_ptr()]


def test_a_partly_owned_pack_gives_one_segment_per_owned_gradient(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    trained = [p for n, p in model.named_parameters() if not n.startswith("encoder.layer.0.")]
    opt = cpu_engine.OPT.B200AdamW(trained, lr=1e-3, arithmetic="torch")
    _backward(model, 1)
    norm = opt.clip_grad_norm(1.0)
    (t,) = cpu_engine.K.tables
    assert [g.data_ptr() for g in t.grads] == [p.grad.data_ptr() for p in trained]
    expect = torch.stack([p.grad.double().pow(2).sum() for p in trained]).sum().sqrt().float()
    assert torch.equal(norm, expect)


def test_parameters_without_gradients_are_left_out(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, arithmetic="torch")
    for p in model.encoder.parameters():
        p.requires_grad_(False)
    _backward(model, 1)
    opt.clip_grad_norm(1.0)
    (t,) = cpu_engine.K.tables
    assert [g.data_ptr() for g in t.grads] == [model.head.weight.grad.data_ptr(), model.head.bias.grad.data_ptr()]


def test_the_table_is_rebuilt_only_when_a_gradient_moves(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, arithmetic="torch")
    K = cpu_engine.K
    _backward(model, 1)
    opt.clip_grad_norm(1.0)
    opt.step()
    model.zero_grad(set_to_none=False)          # gradients stay where they are
    _backward(model, 2)
    opt.clip_grad_norm(1.0)
    opt.step()
    assert len(K.tables) == 1
    model.zero_grad(set_to_none=True)           # the head's .grad is reallocated by the next backward
    _backward(model, 3)
    opt.clip_grad_norm(1.0)
    assert len(K.tables) == 2
    assert K.tables[1].grads[-1].data_ptr() == model.head.bias.grad.data_ptr()
    model.head.weight.grad = model.head.weight.grad.clone()
    opt.clip_grad_norm(1.0)
    assert len(K.tables) == 3


def test_norm_type_other_than_2_raises(cpu_engine):
    model = _Model(cpu_engine.M).eval()
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3)
    _backward(model, 1)
    for nt in (1.0, 3, float("inf")):
        with pytest.raises(ValueError, match="norm_type"):
            opt.clip_grad_norm(1.0, norm_type=nt)
    assert not cpu_engine.K.tables


def test_the_coefficient_is_consumed_by_exactly_one_step(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    ref = _Model(cpu_engine.M).eval()
    ref.load_state_dict(model.state_dict())
    hp = dict(lr=1e-2, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01, arithmetic="torch")
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), **hp)
    opt_ref = cpu_engine.OPT.B200AdamW(ref.parameters(), **hp)
    K = cpu_engine.K
    for step in range(3):
        for m in (model, ref):
            m.zero_grad(set_to_none=False)
            _backward(m, 10 + step, scale=100.0)
        if step == 0:
            norm = opt.clip_grad_norm(0.5)
            coef = torch.clamp(0.5 / (norm + 1e-6), max=1.0)
            assert coef < 1
            # torch's clip on the reference, then a plain step
            torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.5)
        opt.step()
        opt_ref.step()
        for (n, p), q in zip(model.named_parameters(), ref.parameters()):
            err = (p.detach() - q.detach()).abs().max() / q.detach().abs().max().clamp_min(1e-6)
            assert err < 2e-6, (step, n, float(err))
    # step 0 got the coefficient (pack launch and loose path), steps 1 and 2 did not
    assert K.adamw_dev[0] is not None and K.adamw_dev[1] is None and K.adamw_dev[2] is None
    assert opt._clip_coef is None


def test_torch_arithmetic_without_weight_decay_is_torch_adam(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    ref = _Model(cpu_engine.M).eval()
    ref.load_state_dict(model.state_dict())
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, eps=1e-8, weight_decay=0.0, arithmetic="torch")
    opt_ref = torch.optim.Adam(ref.parameters(), lr=1e-3, eps=1e-8, weight_decay=0.0, foreach=False)
    for step in range(3):
        for m in (model, ref):
            m.zero_grad(set_to_none=False)
            _backward(m, 20 + step)
        opt.step()
        opt_ref.step()
    for (n, p), q in zip(model.named_parameters(), ref.parameters()):
        err = (p.detach() - q.detach()).abs().max() / q.detach().abs().max().clamp_min(1e-6)
        assert err < 2e-6, (n, float(err))
