"""GraphedTaskSteps(..., scaler=, update_frequency=) on the CPU, with the graphs, the optimizer and the scaler replaced by
recorders: the new refusals (raised before any warm-up or capture, the existing ones unchanged), what a micro-batch
graph and the update graph record, the call schedule (the update on the K-th call and on finish_update()), `.grad`
bound to the union of what the group's tasks reached and None elsewhere, and construction leaving the torch / numpy /
`random` generators, the scaler and the scheduler counter as it found them.  The captures run on the H100
(tests/test_uniter_graphs_update_gpu.py)."""
import random
import types

import numpy as np
import pytest
import torch

from mmf_b200 import graphs
from mmf_b200.graphs import GraphedTaskSteps

TASKS = ["mlm", "itm", "mrc"]


class _Model(torch.nn.Module):
    """draws its task on the host as UNITER does: one head per task, a shared trunk"""
    draws_key = "draws"
    tasks = TASKS

    def __init__(self):
        super().__init__()
        self.trunk = torch.nn.Linear(2, 2)
        self.heads = torch.nn.ModuleDict({t: torch.nn.Linear(2, 1) for t in TASKS})
        self.seq = []

    def draw(self, sl, task=None):
        task = task if task is not None else self.seq.pop(0)
        sl[self.draws_key] = {"x": torch.full((1,), float(TASKS.index(task)))}
        return task


class _Opt:
    capturable = True

    def __init__(self, log, fused=False):
        self.log, self.fused_inf_check = log, fused

    def clip_grad_norm(self, c, scale=None, scaler=None):
        self.log.append(("clip", c, "scale" if scale is not None else None, "scaler" if scaler is not None else None))

    def check_finite(self, scaler):
        self.log.append("check_finite")

    def step(self):
        self.log.append("opt.step")

    def stage_hparams(self, plan):
        self.log.append(("stage", plan))


class _Scaler:
    def __init__(self, log):
        self.log = log
        self._scale, self._growth_tracker = torch.tensor([1024.0]), torch.tensor([3], dtype=torch.int32)

    def scale(self, loss):
        self.log.append("scale")
        return loss * 2.0

    def _get_scale_async(self):
        return self._scale

    def step(self, opt):
        self.log.append("scaler.step")
        opt.step()

    def update(self):
        self.log.append("scaler.update")


class _Sched:
    def __init__(self, opt, log):
        self.optimizer, self.log, self.counter = opt, log, torch.tensor([5])

    def step(self):
        self.log.append("sched.step")

    def refresh(self):
        self.log.append("sched.refresh")


@pytest.fixture
def no_capture(monkeypatch):
    seen = []
    monkeypatch.setattr(GraphedTaskSteps, "_capture", lambda self, *a: seen.append(self.update_frequency))
    return seen


def _make(log, k=4, scaled=True, fused=False, sched=True, max_grad_norm=1.0):
    model = _Model()
    opt = _Opt(log, fused)
    sc = _Scaler(log) if scaled else None
    steps = GraphedTaskSteps(model, lambda b: None, {"x": torch.zeros(1)}, optimizer=opt, max_grad_norm=max_grad_norm,
                             scaler=sc, update_frequency=k, lr_scheduler=_Sched(opt, log) if sched else None)
    return model, steps


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [0, -2, 2.0, "2", True, None])
def test_update_frequency_must_be_a_positive_int(no_capture, k):
    with pytest.raises(ValueError, match=r"GraphedTaskSteps: update_frequency must be a positive int \(MMF's "
                                         r"training.update_frequency\), got %s" % ("'2'" if k == "2" else k)):
        GraphedTaskSteps(_Model(), lambda b: None, {}, optimizer=_Opt([]), update_frequency=k)
    assert no_capture == []


def test_new_refusals_need_the_optimizer(no_capture):
    with pytest.raises(ValueError, match=r"GraphedTaskSteps: scaler= unscales and skips inside the captured optimizer "
                                         r"step; pass optimizer=B200AdamW\(\.\.\., capturable=True\) as well"):
        GraphedTaskSteps(_Model(), lambda b: None, {}, scaler=_Scaler([]))
    with pytest.raises(ValueError, match=r"GraphedTaskSteps: update_frequency=4 accumulates gradients over 4 calls and "
                                         r"updates inside the captured optimizer step; pass optimizer=B200AdamW"):
        GraphedTaskSteps(_Model(), lambda b: None, {}, update_frequency=4)
    # the existing refusals keep their messages and come first
    with pytest.raises(ValueError, match="max_grad_norm clips inside the captured optimizer step"):
        GraphedTaskSteps(_Model(), lambda b: None, {}, max_grad_norm=1.0, scaler=_Scaler([]))
    with pytest.raises(ValueError, match="construct it as mmf_b200.optim.B200AdamW"):
        GraphedTaskSteps(_Model(), lambda b: None, {}, optimizer=torch.optim.SGD(_Model().parameters(), lr=0.1),
                         update_frequency=2)
    with pytest.raises(TypeError, match="must define draw"):
        GraphedTaskSteps(torch.nn.Linear(2, 2), lambda b: None, {}, update_frequency=0)
    assert no_capture == []
    steps = GraphedTaskSteps(_Model(), lambda b: None, {}, optimizer=_Opt([]), update_frequency=np.int64(3))
    assert steps.update_frequency == 3 and type(steps.update_frequency) is int and steps.pending == 0
    assert no_capture == [3]


def test_construction_leaves_generators_scaler_and_scheduler_counter(monkeypatch):
    def capture(self, batch, warmup):
        for t in self.tasks:                       # warm-up and capture draw, update the scale and step the schedule
            self.model.draw(dict(batch), task=t)
        np.random.rand(3)
        random.random()
        torch.rand(2)
        self.scaler._scale.mul_(0.5)
        self.scaler._growth_tracker.add_(1)
        self.lr_scheduler.counter.add_(4)
    monkeypatch.setattr(GraphedTaskSteps, "_capture", capture)
    log = []
    model, opt = _Model(), _Opt(log)
    sc, sched = _Scaler(log), _Sched(opt, log)
    torch.manual_seed(3)
    np.random.seed(3)
    random.seed(3)
    before = (torch.get_rng_state(), np.random.get_state()[1].copy(), random.getstate())
    steps = GraphedTaskSteps(model, lambda b: None, {"x": torch.zeros(1)}, optimizer=opt, max_grad_norm=1.0, scaler=sc,
                             update_frequency=4, lr_scheduler=sched)
    assert torch.equal(before[0], torch.get_rng_state()) and np.array_equal(before[1], np.random.get_state()[1])
    assert before[2] == random.getstate()
    assert steps.scaler._scale.item() == 1024.0 and steps.scaler._growth_tracker.item() == 3
    assert steps.lr_scheduler.counter.item() == 5 and log == ["sched.refresh"]


# ---------------------------------------------------------------------------------------------------------------------
def _wired(model, steps, log):
    """the state _capture_accumulating leaves, with recorders for the graphs: task t reaches the trunk and its head"""
    steps.used = {t: list(model.trunk.parameters()) + list(model.heads[t].parameters()) for t in TASKS}
    steps.grads = {p: torch.zeros_like(p) for p in model.parameters()}
    steps.graphs = {t: types.SimpleNamespace(replay=lambda t=t: log.append(("micro", t))) for t in TASKS}
    steps.update_graph = types.SimpleNamespace(replay=lambda: log.append("update"))
    steps.losses = {t: torch.tensor(float(i)) for i, t in enumerate(TASKS)}
    steps.static = {"x": torch.zeros(1)}
    steps.draws = {t: {"x": torch.zeros(1)} for t in TASKS}
    steps._plan = types.SimpleNamespace(active=torch.zeros(5, dtype=torch.uint8))
    steps._marks = {t: torch.tensor([0, 1 + i]) for i, t in enumerate(TASKS)}
    steps._reached = set()
    steps.epoch = torch.zeros(1, dtype=torch.int64)
    steps._bind_grads(())
    del log[:]                                         # construction's scheduler refresh


def test_micro_and_update_graphs_record_mmfs_update(no_capture):
    log = []
    model, steps = _make(log, fused=False)
    _wired(model, steps, log)
    steps.loss_fn = lambda b: log.append(("loss_fn", b["draws"]["x"].item())) or \
        (model.heads["itm"].weight.sum() * 0 + 3.0)
    # a micro-batch: the dropout epoch, the forward, the scaled backward, its task's slots marked
    steps._micro("itm")
    assert steps.epoch.item() == 1 and log == [("loss_fn", 0.0), "scale"]
    assert steps._plan.active.tolist() == [1, 0, 1, 0, 0]
    # the update: clip at max_grad_norm times the device scale, scaler.step, scaler.update, the schedule, then the
    # gradients and the gate zeroed
    del log[:]
    for g in steps.grads.values():
        g.fill_(1.0)
    steps._update()
    assert log == [("clip", 1.0, "scale", None), "scaler.step", "opt.step", "scaler.update", "sched.step"]
    assert not steps._plan.active.any() and not any(g.any() for g in steps.grads.values())
    # the fused check: with and without clipping
    log2 = []
    model2, steps2 = _make(log2, fused=True)
    _wired(model2, steps2, log2)
    steps2._update()
    assert log2[0] == ("clip", 1.0, None, "scaler")
    log3 = []
    model3, steps3 = _make(log3, fused=True, max_grad_norm=None, sched=False)
    _wired(model3, steps3, log3)
    steps3._update()
    assert log3 == ["check_finite", "scaler.step", "opt.step", "scaler.update"]
    # without a scaler: clip, step
    log4 = []
    model4, steps4 = _make(log4, scaled=False, sched=False)
    _wired(model4, steps4, log4)
    steps4._update()
    assert log4 == [("clip", 1.0, None, None), "opt.step"]


def test_updates_fire_on_calls_k_and_finish_update_and_grads_are_the_groups_union(no_capture):
    log = []
    model, steps = _make(log, k=3)
    _wired(model, steps, log)
    heads = {t: list(model.heads[t].parameters()) for t in TASKS}
    trunk = list(model.trunk.parameters())

    def bound(t):
        return all(p.grad is steps.grads[p] for p in heads[t])
    model.seq = ["mlm", "mlm", "itm", "itm", "mrc", "itm", "mlm"]
    pending, tasks = [], []
    for i in range(7):
        assert steps({"x": torch.full((1,), float(i))}) is steps.losses[steps.task]
        assert steps.static["x"].item() == float(i)
        pending.append(steps.pending)
        tasks.append(steps.task)
        if i == 0:                                     # mid-group: what the group reached so far
            assert bound("mlm") and not bound("itm") and model.heads["itm"].weight.grad is None
        if i == 2:                                     # after the first update: mlm and itm reached, mrc not
            assert bound("mlm") and bound("itm") and all(p.grad is None for p in heads["mrc"])
            assert all(p.grad is steps.grads[p] for p in trunk)
    assert tasks == ["mlm", "mlm", "itm", "itm", "mrc", "itm", "mlm"] and pending == [1, 2, 0, 1, 2, 0, 1]
    micro = lambda ts: [("micro", t) for t in ts]
    assert log == micro(tasks[:3]) + [("stage", steps._plan), "update"] + micro(tasks[3:6]) + \
        [("stage", steps._plan), "update"] + micro(tasks[6:])
    # the third group has reached mlm so far
    assert bound("mlm") and not bound("mrc") and not bound("itm")
    del log[:]
    steps.finish_update()                              # the partial group: one update, then nothing left
    assert log == [("stage", steps._plan), "update"] and steps.pending == 0
    assert bound("mlm") and all(p.grad is None for p in heads["itm"] + heads["mrc"])
    steps.finish_update()
    assert log == [("stage", steps._plan), "update"]
