"""GraphedStep(..., update_frequency=K) on the CPU: the refusals, raised before any warm-up or capture, and the call
schedule with the graphs replaced by recorders - the gradients zeroed before the first micro-batch of a group, the
update on calls K and 2K, finish_update() on a partial group and as a no-op on an empty one, and the hyper-parameters
staged before updates only.  The captures themselves run on the H100 (tests/test_graphed_accumulate_gpu.py)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_static_packing_cpu import _root  # noqa: E402

from mmf_b200.graphs import GraphedStep  # noqa: E402
from mmf_b200.optim import B200AdamW  # noqa: E402


@pytest.fixture
def no_capture(monkeypatch):
    seen = []
    monkeypatch.setattr(GraphedStep, "_capture", lambda self, *a: seen.append(self.update_frequency))
    return seen


@pytest.fixture
def lin():
    return torch.nn.Linear(4, 4)


def _opt(model):
    return B200AdamW(model.parameters(), capturable=True)


@pytest.mark.parametrize("k", [0, -2, 2.0, "2", True, None])
def test_update_frequency_must_be_a_positive_int(no_capture, lin, k):
    with pytest.raises(ValueError, match=r"GraphedStep: update_frequency must be a positive int \(MMF's "
                                         r"training.update_frequency\), got %s" % ("'2'" if k == "2" else k)):
        GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, optimizer=_opt(lin), update_frequency=k)
    assert no_capture == []


def test_accumulation_needs_the_optimizer(no_capture, lin):
    with pytest.raises(ValueError, match=r"update_frequency=4 accumulates gradients over 4 calls and updates inside "
                                         r"the captured optimizer step; pass optimizer=B200AdamW\(\.\.\., "
                                         r"capturable=True\) as well"):
        GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, update_frequency=4)
    assert no_capture == []


def test_refusals_come_before_the_model_checks(no_capture, lin):
    # a skip-padding model would be refused with a RuntimeError by the model scan: the argument is checked first
    with pytest.raises(ValueError, match="positive int"):
        GraphedStep(_root(), lambda b: None, {"x": torch.zeros(1)}, update_frequency=0)
    with pytest.raises(ValueError, match="pass optimizer="):
        GraphedStep(_root(), lambda b: None, {"x": torch.zeros(1)}, update_frequency=2)
    # the existing refusals keep their messages and their order
    with pytest.raises(ValueError, match="max_grad_norm clips inside the captured optimizer step"):
        GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, max_grad_norm=1.0, update_frequency=2)
    with pytest.raises(ValueError, match="construct it as mmf_b200.optim.B200AdamW"):
        GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, optimizer=B200AdamW(lin.parameters()),
                    update_frequency=2)
    with pytest.raises(RuntimeError, match="skip_padding encoders"):
        GraphedStep(_root(), lambda b: None, {"x": torch.zeros(1)}, optimizer=_opt(_root()), update_frequency=2)
    assert no_capture == []


def test_integral_values_are_accepted(no_capture, lin):
    for k, want in ((1, 1), (np.int64(8), 8), (3, 3)):
        step = GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, optimizer=_opt(lin), update_frequency=k)
        assert step.update_frequency == want and type(step.update_frequency) is int and step.pending == 0
    assert no_capture == [1, 8, 3]


def _recorded(step, log):
    """the graphs, the optimizer's staging and the static inputs replaced by recorders"""
    for name in ("graph", "zero_graph", "update_graph"):
        setattr(step, name, types.SimpleNamespace(replay=lambda name=name: log.append(name)))
    step.optimizer.stage_hparams = lambda plan: log.append(("stage", plan))
    step._plan, step.loss, step.static = "plan", torch.tensor(7.0), {"x": torch.zeros(2)}


def test_the_update_fires_on_calls_k_and_2k(no_capture, lin):
    step = GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, optimizer=_opt(lin), max_grad_norm=1.0,
                       update_frequency=3)
    log = []
    _recorded(step, log)
    pending = []
    for i in range(7):
        assert step({"x": torch.full((2,), float(i))}) is step.loss
        assert torch.equal(step.static["x"], torch.full((2,), float(i)))
        pending.append(step.pending)
    assert pending == [1, 2, 0, 1, 2, 0, 1]
    group = ["zero_graph", "graph", "graph", "graph", ("stage", "plan"), "update_graph"]
    assert log == group + group + ["zero_graph", "graph"]
    # the last, partial group: finish_update() stages and updates once, then has nothing left to do
    del log[:]
    step.finish_update()
    assert log == [("stage", "plan"), "update_graph"] and step.pending == 0
    step.finish_update()
    assert log == [("stage", "plan"), "update_graph"]
    # a new group starts from zeroed gradients
    step()
    assert log[2:] == ["zero_graph", "graph"] and step.pending == 1


def test_finish_update_on_an_empty_group_does_nothing(no_capture, lin):
    step = GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, optimizer=_opt(lin), update_frequency=4)
    log = []
    _recorded(step, log)
    step.finish_update()
    assert log == []
    for _ in range(4):
        step()
    step.finish_update()
    assert log.count("update_graph") == 1 and log.count(("stage", "plan")) == 1 and log[-1] == "update_graph"


def test_update_frequency_1_keeps_the_one_graph_schedule(no_capture, lin):
    """one replay per call, each after staging the hyper-parameters; finish_update() has nothing to do"""
    step = GraphedStep(lin, lambda b: None, {"x": torch.zeros(1)}, optimizer=_opt(lin), update_frequency=1)
    log = []
    _recorded(step, log)
    for _ in range(3):
        step()
        step.finish_update()
    assert log == [("stage", "plan"), "graph"] * 3 and step.pending == 0
