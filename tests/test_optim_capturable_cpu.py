"""B200AdamW(capturable=True) and GraphedStep(optimizer=...) on the host, over a kernel test double for the new entry points
defined here (mmfb_adamw_hparams, mmfb_adamw_segments and mmfb_adamw's device hyper-parameter table): the segment table's
rows, which parameters go to pack launches and which to the segment launch, the staged and computed hyper-parameters,
the refusals, state_dict round trips with plain B200AdamW and torch.optim.AdamW, GraphedStep's refusals without the new
arguments, and the C header.  The kernels themselves run on the H100 (tests/test_optim_capturable_gpu.py)."""
import ctypes
import io
import math
import types

import pytest
import torch

import fake_kernels as FK
from mmf_b200 import functional as REAL_F
from mmf_b200 import lib


def _elementwise(p, g, m, v, lr, wd, ss, bc2s, b1, b2, eps, mode):
    """the per-element arithmetic of mmfb_adamw on one tensor, in the torch ops of B200AdamW._torch_update"""
    if mode == 0:
        m.mul_(b1).add_(g, alpha=1.0 - b1)
        v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        p.addcdiv_(m, v.sqrt().add_(eps), value=-ss)
        if wd > 0.0:
            p.add_(p, alpha=-lr * wd)
    else:
        p.mul_(1.0 - lr * wd)
        m.lerp_(g, 1.0 - b1)
        v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        p.addcdiv_(m, (v.sqrt() / bc2s).add_(eps), value=-ss)


class _Kernels:
    """contract of the functional wrappers the optimizer calls, recording what it hands them"""

    def __init__(self):
        self.tables, self.calls = [], []
        self.values = {}        # slot -> the hyper-parameters as Python floats (the fp32 table holds their roundings)

    # clipping (as tests/test_grad_norm_cpu.py)
    def grad_norm_table(self, grads):
        return types.SimpleNamespace(grads=list(grads))

    def grad_norm(self, table, max_norm, norm_type=2.0):
        n = torch.stack([g.double().pow(2).sum() for g in table.grads]).sum().sqrt().float()
        return torch.stack([n, torch.clamp(max_norm / (n + 1e-6), max=1.0)])

    # the new entry points
    def adamw_slot_table(self, slots, device):
        return torch.tensor(slots, dtype=torch.int32).reshape(-1, 2)

    def adamw_hparams(self, groups, slots, step, hp, mode):
        self.calls.append("hparams")
        for s, (gi, flags) in enumerate(slots.tolist()):
            lr, wd, b1, b2, eps = groups[gi].tolist()
            if flags & lib.MMFB_ADAMW_SLOT_FROZEN:
                vals = [0.0, 0.0, 0.0, 1.0]
            else:
                step[s] += 1
                t = int(step[s])
                bc1, bc2s = 1.0 - b1 ** t, math.sqrt(1.0 - b2 ** t)
                if mode == 0:
                    vals = [lr, wd, lr * bc2s / bc1 if flags & lib.MMFB_ADAMW_SLOT_CORRECT_BIAS else lr, 1.0]
                else:
                    vals = [lr, wd, lr / bc1, bc2s]
            hp[s] = torch.tensor(vals + [b1, b2, eps, 0.0], dtype=torch.float64).float()
            self.values[s] = vals + [b1, b2, eps]

    def adamw(self, param, grad, m, v, groups, *, beta1, beta2, eps, mode, grad_scale=1.0, group_of_block=None,
              param_bf16=None, grad_scale_dev=None, hp_dev=None):
        self.calls.append("adamw" if hp_dev is None else "adamw_hp")
        if hp_dev is not None:                       # the table's values, betas and eps as the launch passes them
            groups = [dict(lr=h[0], weight_decay=h[1], step_size=h[2], bc2_sqrt=h[3]) for h in hp_dev.tolist()]
        if grad_scale_dev is not None:
            grad_scale = grad_scale_dev * grad_scale
        FK.adamw(param, grad, m, v, groups, beta1=beta1, beta2=beta2, eps=eps, mode=mode, grad_scale=grad_scale,
                 group_of_block=group_of_block)

    def adamw_segment_table(self, segments):
        rows, n_blocks = REAL_F.adamw_segment_rows(segments)
        t = types.SimpleNamespace(rows=rows, n_blocks=n_blocks, segments=list(segments))
        self.tables.append(t)
        return t

    def adamw_segments(self, table, hp, *, mode, grad_scale=1.0, grad_scale_dev=None):
        self.calls.append("segments")
        assert [r[:4] for r in table.rows] == [tuple(t.data_ptr() for t in s[:4]) for s in table.segments if s[0].numel()]
        scale = grad_scale_dev * grad_scale if grad_scale_dev is not None else grad_scale
        for p, g, m, v, slot in table.segments:
            assert hp[slot].tolist()[:7] == torch.tensor(self.values[slot]).float().tolist()
            _elementwise(p, g.float() * scale if grad_scale_dev is not None else g, m, v, *self.values[slot], mode)


@pytest.fixture()
def cpu_engine(monkeypatch):
    import mmf_b200.engine as E
    import mmf_b200.modules as M
    import mmf_b200.optim as OPT
    K = _Kernels()
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPT, "F", K)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    yield types.SimpleNamespace(E=E, M=M, OPT=OPT, K=K)


class _Model(torch.nn.Module):
    """an engine encoder (parameters in a pack) plus a head outside it with an odd number of outputs"""

    def __init__(self, M, n_out=5):
        super().__init__()
        cfg = types.SimpleNamespace(hidden_size=64, num_attention_heads=1, intermediate_size=128, num_hidden_layers=2,
                                    hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12)
        self.encoder = M.B200BertEncoder(cfg)
        self.head = torch.nn.Linear(64, n_out)

    def forward(self, x):
        return self.head(self.encoder(x, None)[0])


def _backward(model, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 5, 64, generator=g)
    y = model(x)
    (y * torch.randn(y.shape, generator=g) * scale).sum().backward()


def _scaled_groups(model, lr=1e-3):
    """m4c-style lr_scale groups: the first encoder layer at lr / 10, the rest of the encoder, the head without decay"""
    first = [p for n, p in model.named_parameters() if n.startswith("encoder.layer.0.")]
    rest = [p for n, p in model.named_parameters() if n.startswith("encoder.") and not n.startswith("encoder.layer.0.")]
    return [{"params": first, "lr": lr * 0.1}, {"params": rest}, {"params": list(model.head.parameters()), "weight_decay": 0.0}]


# ---------------------------------------------------------------------------------------------------------------------
def _aligned(n):
    base = torch.zeros(n + 64)
    off = (-(base.data_ptr() >> 2)) % 4
    return base[off:off + n]


@pytest.mark.parametrize("n", [1, 7, 8, 9, 2047, 2048, 2049, 5000])
def test_segment_rows_of_aligned_tensors(n):
    ts = [_aligned(n) for _ in range(4)]
    rows, n_blocks = REAL_F.adamw_segment_rows([tuple(ts) + (3,)])
    (r,) = rows
    assert r == tuple(t.data_ptr() for t in ts) + (n, 3, 0, 0)
    assert n_blocks == (n + 2047) // 2048


@pytest.mark.parametrize("shift", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 3129])
def test_segment_rows_of_misaligned_views(shift, n):
    views = [_aligned(n + 8)[shift:shift + n] for _ in range(4)]
    rows, n_blocks = REAL_F.adamw_segment_rows([tuple(views) + (0,)])
    head = 4 - shift                                 # elements before the next 16-byte boundary
    assert rows[0][4:] == (n, 0, 0, head)
    assert n_blocks == (n + 8 - head + 2047) // 2048
    # one stream out of step with the others: no common alignment, every element singly
    mixed = [views[0], _aligned(n), views[2], views[3]]
    rows, n_blocks = REAL_F.adamw_segment_rows([tuple(mixed) + (0,)])
    assert rows[0][7] == -1 and n_blocks == (n + 2047) // 2048


def test_segment_rows_first_blocks_slots_and_empty_tensors():
    sizes = [5, 0, 3129, 768 * 768, 3]
    segs = [tuple(_aligned(n) for _ in range(4)) + (10 + i,) for i, n in enumerate(sizes)]
    rows, n_blocks = REAL_F.adamw_segment_rows(segs)
    assert [r[4] for r in rows] == [5, 3129, 768 * 768, 3]
    assert [r[5] for r in rows] == [10, 12, 13, 14]
    assert [r[6] for r in rows] == [0, 1, 3, 3 + 288]
    assert n_blocks == 3 + 288 + 1


def test_segment_rows_refuse_what_the_kernel_cannot_read():
    a = torch.zeros(8, 8)
    with pytest.raises(ValueError, match="contiguous fp32"):
        REAL_F.adamw_segment_rows([(a.t(), a, a, a, 0)])
    with pytest.raises(ValueError, match="contiguous fp32"):
        REAL_F.adamw_segment_rows([(a.bfloat16(), a, a, a, 0)])
    with pytest.raises(ValueError, match="elements"):
        REAL_F.adamw_segment_rows([(a, a[:4], a, a, 0)])


# ---------------------------------------------------------------------------------------------------------------------
def test_packs_and_segments_across_lr_scale_groups(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    # a tied parameter listed twice in its group is stepped once
    groups = _scaled_groups(model)
    groups[2]["params"].append(model.head.bias)
    with pytest.warns(UserWarning):
        opt = cpu_engine.OPT.B200AdamW(groups, lr=1e-3, weight_decay=0.01, arithmetic="torch", capturable=True)
    _backward(model, 1)
    opt.step()
    plan = opt._cap
    pack = model.encoder._runner.pack
    assert [e[0] for e in plan.packs] == [pack]
    _, ent, s0, n, betas, eps = plan.packs[0]
    assert (s0, n) == (0, 3)
    assert plan.slots[:3] == [(0, 1), (1, 1), (0, lib.MMFB_ADAMW_SLOT_FROZEN)]     # the head's group has no pack parameter
    assert [(p is model.head.weight or p is model.head.bias, s) for p, s in plan.loose] == [(True, 3), (True, 4)]
    assert plan.slots[3:] == [(2, 1), (2, 1)]
    (t,) = cpu_engine.K.tables
    assert [r[4] for r in t.rows] == [64 * 5, 5]
    assert cpu_engine.K.calls == ["hparams", "adamw_hp", "segments"]
    # step counts are shared device values, one per slot
    assert all(opt.state[p]["step"].data_ptr() == plan.step[0].data_ptr() for p in groups[0]["params"])
    assert int(opt.state[model.head.bias]["step"]) == 1


def test_mixed_step_counts_inside_a_pack_send_it_to_the_segments(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    plain = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, arithmetic="torch")
    _backward(model, 1)
    plain.step()
    sd = plain.state_dict()
    sd["state"][0]["step"] = 7
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, arithmetic="torch", capturable=True)
    opt.load_state_dict(sd)
    opt.step()
    assert not opt._cap.packs and len(opt._cap.loose) == len(list(model.parameters()))
    assert int(opt.state[next(model.parameters())]["step"]) == 8


def test_the_segment_table_is_rebuilt_only_when_a_gradient_moves_and_never_in_capture(cpu_engine, monkeypatch):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, capturable=True)
    _backward(model, 1)
    opt.step()
    plan = opt._cap
    model.zero_grad(set_to_none=False)
    _backward(model, 2)
    opt.step()
    assert opt._cap is plan and len(cpu_engine.K.tables) == 1
    model.zero_grad(set_to_none=True)            # the head's gradients are reallocated: new table, same slots
    _backward(model, 3)
    opt.step()
    assert opt._cap is plan and len(cpu_engine.K.tables) == 2
    model.head.weight.grad = model.head.weight.grad.clone()
    monkeypatch.setattr(cpu_engine.OPT, "_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="moved during CUDA-graph capture"):
        opt.step()
    model.head.bias.grad = None
    with pytest.raises(RuntimeError, match="parameters with gradients changed during CUDA-graph capture"):
        opt.step()


@pytest.mark.parametrize("arithmetic,correct_bias", [("torch", True), ("transformers", True), ("transformers", False)])
def test_staged_and_computed_hyper_parameters_follow_group_hp(cpu_engine, arithmetic, correct_bias):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    opt = cpu_engine.OPT.B200AdamW(_scaled_groups(model), lr=1e-3, betas=(0.9, 0.98), weight_decay=0.01,
                                   correct_bias=correct_bias, arithmetic=arithmetic, capturable=True)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: min(1.0, (s + 1) / 4))
    for step in range(1, 6):
        _backward(model, step)
        opt.step()
        sched.step()
        plan = opt._cap
        staged = plan.groups.tolist()
        for (gi, flags), h in zip(plan.slots, plan.hp.tolist()):
            if flags & lib.MMFB_ADAMW_SLOT_FROZEN:
                assert h[:4] == [0.0, 0.0, 0.0, 1.0]
                continue
            hp = opt._group_hp(dict(opt.param_groups[gi], lr=staged[gi][0]), step)
            assert h[:4] == [float(torch.tensor(hp[k], dtype=torch.float32)) for k in
                             ("lr", "weight_decay", "step_size", "bc2_sqrt")]
            assert h[4:7] == [float(torch.tensor(x, dtype=torch.float32)) for x in (0.9, 0.98, 1e-6)]
        assert staged[0][0] == pytest.approx(1e-4 * min(1.0, step / 4), rel=1e-12)
    opt.stage_hparams()
    assert opt._cap.groups[:, 0].tolist() == [g["lr"] for g in opt.param_groups]


def test_refusals(cpu_engine):
    torch.manual_seed(0)
    model = _Model(cpu_engine.M).eval()
    model.head.to(torch.bfloat16)
    opt = cpu_engine.OPT.B200AdamW(model.head.parameters(), lr=1e-3, capturable=True)
    model.head.weight.grad = torch.zeros_like(model.head.weight)
    with pytest.raises(ValueError, match="fp32"):
        opt.step()
    lin = torch.nn.Linear(4, 6)
    opt = cpu_engine.OPT.B200AdamW(lin.parameters(), lr=1e-3, capturable=True)
    lin.weight.grad = torch.zeros(4, 6).t()
    lin.bias.grad = torch.zeros(6)
    with pytest.raises(ValueError, match="contiguous fp32"):
        opt.step()
    from mmf_b200.graphs import GraphedStep
    plain = cpu_engine.OPT.B200AdamW(lin.parameters(), lr=1e-3)
    with pytest.raises(ValueError, match="capturable=True"):
        GraphedStep(lin, lambda b: lin(b).sum(), torch.zeros(2, 4), optimizer=plain)
    with pytest.raises(ValueError, match="pass optimizer="):
        GraphedStep(lin, lambda b: lin(b).sum(), torch.zeros(2, 4), max_grad_norm=1.0)


class _HostWork(torch.nn.Module):
    graph_capturable = False
    graph_refusal = "reads its input on the host"


def test_graphed_step_without_the_new_arguments_refuses_as_before(cpu_engine):
    from mmf_b200.graphs import GraphedStep
    model = torch.nn.Sequential(torch.nn.Linear(4, 4), _HostWork())
    with pytest.raises(RuntimeError, match="_HostWork reads its input on the host, so its step cannot be captured"):
        GraphedStep(model, lambda b: model(b).sum(), torch.zeros(2, 4))
    opt = cpu_engine.OPT.B200AdamW(model.parameters(), lr=1e-3, capturable=True)
    with pytest.raises(RuntimeError, match="_HostWork reads its input on the host"):
        GraphedStep(model, lambda b: model(b).sum(), torch.zeros(2, 4), optimizer=opt, max_grad_norm=1.0)


# ---------------------------------------------------------------------------------------------------------------------
def _run(opt, model, seeds, clip=None):
    for s in seeds:
        model.zero_grad()
        _backward(model, s, scale=100.0)
        if clip is not None:
            opt.clip_grad_norm(clip)
        opt.step()


def _ckpt(sd):
    """through a checkpoint file, so that the loading optimizer shares no tensor with the saving one"""
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf)


def _close(a, b, bar=2e-6):
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        err = (p.detach() - q.detach()).abs().max() / q.detach().abs().max().clamp_min(1e-6)
        assert err < bar, (n, float(err))


def test_capturable_steps_match_plain_steps_and_state_dicts_round_trip(cpu_engine):
    torch.manual_seed(0)
    OPT = cpu_engine.OPT
    models = [_Model(cpu_engine.M).eval() for _ in range(3)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    hp = dict(lr=1e-2, betas=(0.9, 0.98), eps=1e-8, weight_decay=0.0, arithmetic="torch")
    cap = OPT.B200AdamW(models[0].parameters(), capturable=True, **hp)
    plain = OPT.B200AdamW(models[1].parameters(), **hp)
    _run(cap, models[0], [1, 2], clip=0.5)
    _run(plain, models[1], [1, 2], clip=0.5)
    _close(models[0], models[1])
    sd = _ckpt(cap.state_dict())
    assert all(type(st["step"]) is int and st["step"] == 2 for st in sd["state"].values())
    assert all(torch.is_tensor(st["step"]) for st in cap.state.values())      # the live state is unchanged
    # capturable -> plain, plain -> capturable, capturable -> torch.optim.Adam, torch -> capturable
    plain2 = OPT.B200AdamW(models[2].parameters(), **hp)
    models[2].load_state_dict(models[0].state_dict())
    plain2.load_state_dict(sd)
    _run(plain2, models[2], [3], clip=0.5)
    _run(cap, models[0], [3], clip=0.5)
    _close(models[0], models[2])
    cap2 = OPT.B200AdamW(models[1].parameters(), capturable=True, **hp)
    models[1].load_state_dict(models[2].state_dict())
    cap2.load_state_dict(_ckpt(plain2.state_dict()))
    ref = torch.optim.Adam(models[2].parameters(), lr=1e-2, betas=(0.9, 0.98), eps=1e-8, foreach=False)
    ref.load_state_dict(_ckpt(cap2.state_dict()))
    _run(cap2, models[1], [4, 5])
    _run(ref, models[2], [4, 5])
    _close(models[1], models[2])
    assert all(int(st["step"]) == 5 for st in ref.state.values())
    cap3 = OPT.B200AdamW(models[0].parameters(), capturable=True, **hp)
    models[0].load_state_dict(models[2].state_dict())
    cap3.load_state_dict(_ckpt(ref.state_dict()))
    _run(cap3, models[0], [6])
    _run(ref, models[2], [6])
    _close(models[0], models[2])
    assert all(int(st["step"]) == 6 for st in cap3.state.values())


def test_header_declares_the_new_entry_points():
    syms = lib.header_symbols()
    for s in ("mmfb_adamw_hparams", "mmfb_adamw_segments"):
        assert s in syms and hasattr(lib.LIB, s)
    assert ctypes.sizeof(lib.AdamWSegment) == 56 and ctypes.sizeof(lib.AdamWSlot) == 8
    assert lib.AdamWArgs.hp_dev.offset == lib.AdamWArgs.grad_scale_dev.offset + 8 == ctypes.sizeof(lib.AdamWArgs) - 8
    with open(lib.os.path.join(lib.os.path.dirname(lib._HERE), "include", "mmfb200.h")) as fh:
        hdr = fh.read()
    assert "#define MMFB_ADAMW_SEGMENT_BLOCK %d" % lib.MMFB_ADAMW_SEGMENT_BLOCK in hdr
    assert "#define MMFB_ADAMW_SLOT_FROZEN %d" % lib.MMFB_ADAMW_SLOT_FROZEN in hdr
    if not torch.cuda.is_available():
        for fn, args in ((lib.LIB.mmfb_adamw_hparams, lib.AdamWHparamsArgs()),
                         (lib.LIB.mmfb_adamw_segments, lib.AdamWSegmentsArgs())):
            a = args
            a.n_slots = 1 if hasattr(a, "n_slots") else 0
            assert fn(ctypes.byref(a), None) in (lib.MMFB_ERR_ARG, lib.MMFB_ERR_DEVICE)
