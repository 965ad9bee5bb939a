"""MMF's fp16 update on a capturable B200AdamW, on the host over a kernel test double: which optimizers advertise torch's
fused-optimizer protocol, that GradScaler's scale and found_inf reach every launch of the step (hyper-parameters, packs,
segments) and clip_grad_norm's scale the norm launch, that the update GradScaler.step drives through them equals its
unscale_ path (skipped steps included), the refusals, and the C header and ctypes mirrors of the new fields.  The kernels
run on the H100 (tests/test_amp_step_gpu.py)."""
import ctypes
import os
import re
import types

import pytest
import torch

import test_optim_capturable_cpu as OC
from mmf_b200 import functional as REAL_F
from mmf_b200 import lib


class _AmpKernels(OC._Kernels):
    """the double of tests/test_optim_capturable_cpu.py with the loss-scaling arguments: found_inf != 0 makes a launch
    write nothing, the scale multiplies every gradient by fp32(1 / fp64(S)) before the launch's own factor"""

    def __init__(self):
        super().__init__()
        self.amp = []           # (entry point, loss_scale_dev, found_inf) of every launch

    @staticmethod
    def _skip(found_inf):
        return found_inf is not None and float(found_inf) != 0.0

    def grad_norm(self, table, max_norm, norm_type=2.0, max_norm_scale_dev=None):
        self.amp.append(("grad_norm", max_norm_scale_dev, None))
        if max_norm_scale_dev is not None:
            max_norm = float(torch.tensor(max_norm, dtype=torch.float32) * max_norm_scale_dev.float())
        return super().grad_norm(table, max_norm, norm_type)

    def adamw_hparams(self, groups, slots, step, hp, mode, found_inf=None):
        self.amp.append(("hparams", None, found_inf))
        if not self._skip(found_inf):
            super().adamw_hparams(groups, slots, step, hp, mode)

    def adamw(self, param, grad, m, v, groups, *, loss_scale_dev=None, found_inf=None, **kw):
        self.amp.append(("adamw", loss_scale_dev, found_inf))
        if self._skip(found_inf):
            return
        if loss_scale_dev is not None:
            grad = grad * loss_scale_dev.double().reciprocal().float()
        super().adamw(param, grad, m, v, groups, **kw)

    def adamw_segments(self, table, hp, *, loss_scale_dev=None, found_inf=None, **kw):
        self.amp.append(("segments", loss_scale_dev, found_inf))
        if self._skip(found_inf):
            return
        if loss_scale_dev is not None:
            inv = loss_scale_dev.double().reciprocal().float()
            table = types.SimpleNamespace(rows=table.rows, n_blocks=table.n_blocks,
                                          segments=[(p, g * inv, m, v, s) for p, g, m, v, s in table.segments])
            table.rows = [tuple(t.data_ptr() for t in s[:4]) + r[4:] for s, r in zip(table.segments, table.rows)]
        super().adamw_segments(table, hp, **kw)


@pytest.fixture()
def amp_engine(monkeypatch):
    import mmf_b200.engine as E
    import mmf_b200.modules as M
    import mmf_b200.optim as OPT
    import fake_kernels as FK
    K = _AmpKernels()
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPT, "F", K)
    monkeypatch.setattr(M, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    yield types.SimpleNamespace(E=E, M=M, OPT=OPT, K=K)


def test_only_capturable_optimizers_advertise_amp_scaling(amp_engine):
    model = OC._Model(amp_engine.M)
    plain = amp_engine.OPT.B200AdamW(model.parameters())
    cap = amp_engine.OPT.B200AdamW(model.parameters(), capturable=True)
    assert not getattr(plain, "_step_supports_amp_scaling", False)
    assert cap._step_supports_amp_scaling is True
    assert not getattr(type(cap), "_step_supports_amp_scaling", False)     # an instance attribute, not a class one


def test_the_scale_and_found_inf_reach_every_launch(amp_engine):
    torch.manual_seed(0)
    model = OC._Model(amp_engine.M)
    opt = amp_engine.OPT.B200AdamW(OC._scaled_groups(model), capturable=True, arithmetic="torch")
    OC._backward(model, 1)
    opt.step()                                  # no scaler: no loss-scaling argument anywhere
    assert all(s is None and f is None for _, s, f in amp_engine.K.amp)
    assert {e for e, _, _ in amp_engine.K.amp} == {"hparams", "adamw", "segments"}
    amp_engine.K.amp.clear()
    scale, found = torch.tensor(1024.0), torch.tensor(0.0)
    opt.grad_scale, opt.found_inf = scale, found          # what GradScaler.step sets for the call
    norm_scale = torch.tensor(8.0)
    opt.clip_grad_norm(0.25, scale=norm_scale)
    opt.step()
    calls = amp_engine.K.amp
    assert calls[0] == ("grad_norm", norm_scale, None)
    assert [c[0] for c in calls[1:]] == ["hparams"] + ["adamw"] * len(opt._cap.packs) + ["segments"]
    assert calls[1][2] is found and all(s is scale and f is found for _, s, f in calls[2:])
    # after unscale_ GradScaler passes grad_scale None: found_inf alone
    amp_engine.K.amp.clear()
    opt.grad_scale = None
    opt.step()
    assert all(s is None and f is found for e, s, f in amp_engine.K.amp if e != "hparams")


def _amp_run(engine, fused, seeds, infs):
    torch.manual_seed(0)
    model = OC._Model(engine.M)
    opt = engine.OPT.B200AdamW(OC._scaled_groups(model), capturable=True, arithmetic="torch")
    if not fused:
        opt._step_supports_amp_scaling = False
    scaler = torch.amp.GradScaler("cpu", init_scale=256.0, growth_interval=2)
    for seed, inf in zip(seeds, infs):
        model.zero_grad()
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(2, 5, 64, generator=g)
        y = model(x)
        loss = (y * torch.randn(y.shape, generator=g)).sum() * (float("inf") if inf else 1.0)
        scaler.scale(loss).backward()
        if fused:
            opt.clip_grad_norm(0.25, scale=scaler._get_scale_async())
        else:
            opt.clip_grad_norm(0.25 * scaler.get_scale())
        scaler.step(opt)
        scaler.update()
    return model, opt, scaler


def test_fused_update_equals_gradscalers_unscale_path(amp_engine):
    seeds, infs = [3, 4, 5, 6, 7], [False, False, True, False, False]
    m1, o1, s1 = _amp_run(amp_engine, True, seeds, infs)
    m2, o2, s2 = _amp_run(amp_engine, False, seeds, infs)
    assert s1.get_scale() == s2.get_scale() and int(s1._growth_tracker) == int(s2._growth_tracker)
    for (n, p), q in zip(m1.named_parameters(), m2.parameters()):
        assert torch.equal(p.detach(), q.detach()), n
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(o1.state[p][k], o2.state[q][k]), (n, k)
        assert int(o1.state[p]["step"]) == int(o2.state[q]["step"]) == 4, n     # the skipped step does not count
    assert all(p.grad is not None for p in m1.parameters())


def test_refusals(amp_engine):
    from mmf_b200.graphs import GraphedStep
    model = OC._Model(amp_engine.M)
    scaler = torch.amp.GradScaler("cpu")
    with pytest.raises(ValueError, match="scaler= .*optimizer="):
        GraphedStep(model, lambda b: model(b).sum(), torch.zeros(2, 5, 64), scaler=scaler)
    plain = amp_engine.OPT.B200AdamW(model.parameters())
    with pytest.raises(ValueError, match="capturable=True"):
        GraphedStep(model, lambda b: model(b).sum(), torch.zeros(2, 5, 64), optimizer=plain, scaler=scaler)
    for bad in (2.0, torch.tensor([1.0, 2.0]), torch.tensor(1.0, dtype=torch.float64), torch.tensor(1.0)):
        with pytest.raises(ValueError, match="one-element fp32 CUDA tensor"):
            REAL_F._req_scalar(bad, "grad_norm", "max_norm_scale_dev")
    assert REAL_F._req_scalar(None, "adamw", "found_inf") is None


HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "mmfb200.h")


@pytest.mark.parametrize("struct, mirror, fields", [
    ("mmfb_adamw_args", lib.AdamWArgs, ["mode", "loss_scale_dev", "found_inf", "grad_scale_dev", "hp_dev"]),
    ("mmfb_adamw_segments_args", lib.AdamWSegmentsArgs, ["grad_scale_dev", "loss_scale_dev", "found_inf"]),
    ("mmfb_adamw_hparams_args", lib.AdamWHparamsArgs, ["mode", "found_inf"]),
    ("mmfb_grad_norm_args", lib.GradNormArgs, ["norm_type", "max_norm_scale_dev"]),
])
def test_header_and_ctypes_mirrors_end_with_the_new_fields(struct, mirror, fields):
    txt = open(HDR).read()
    body = re.search(r"typedef struct \{([^}]*)\} %s;" % struct, txt).group(1)
    names = re.findall(r"(\w+)(?:\[[^\]]*\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names[-len(fields):] == fields
    assert [f[0] for f in mirror._fields_][-len(fields):] == fields
    assert all(mirror._fields_[-i][1] is ctypes.c_void_p for i in range(1, len(fields)))
