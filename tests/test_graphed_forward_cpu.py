"""GraphedForward's refusals on the CPU: each is raised before any warm-up or capture - a model in training mode
(ValueError), the skip-padding / pack_tail / pack_streams encoders and UNITER with GraphedStep's messages, a model that
returns attention probabilities or hidden states, and a model or batch off the GPU.  The captures themselves run on the
H100 (tests/test_graphed_forward_gpu.py)."""
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_static_packing_cpu import _root  # noqa: E402
from test_uniter_model_cpu import _build, cpu_models, golden  # noqa: E402,F401

from mmf_b200 import graphs  # noqa: E402
from mmf_b200.graphs import GraphedForward, GraphedStep  # noqa: E402
from mmf_b200.sample import SampleList  # noqa: E402


@pytest.fixture
def no_capture(monkeypatch):
    seen = []
    monkeypatch.setattr(GraphedForward, "_capture", lambda self, *a: seen.append(graphs.static_rows_active()))
    return seen


def _messages(model, static_rows):
    """GraphedStep's refusal of `model`, and GraphedForward's"""
    with pytest.raises(RuntimeError) as step:
        GraphedStep(model, lambda b: None, {"x": torch.zeros(1)}, static_rows=static_rows)
    with pytest.raises(RuntimeError) as fwd:
        GraphedForward(model.eval(), {"x": torch.zeros(1)}, static_rows=static_rows)
    return str(step.value), str(fwd.value)


def test_training_mode_is_refused(no_capture):
    lin = torch.nn.Linear(4, 4)
    with pytest.raises(ValueError, match="training mode.*model.eval()"):
        GraphedForward(lin, {"x": torch.zeros(2, 4)})
    with pytest.raises(ValueError, match="training mode"):
        GraphedForward(_root(), {"x": torch.zeros(1)})      # before the skip-padding refusal
    assert lin.training and no_capture == []


@pytest.mark.parametrize("kind,static_rows", [("skip_padding", False), ("pack_tail", True), ("pack_tail", False),
                                              ("pack_streams", False), ("pack_streams", True)])
def test_encoder_refusals_are_graphed_steps(no_capture, kind, static_rows):
    root = {"skip_padding": lambda: _root(), "pack_tail": lambda: _root(causal=True),
            "pack_streams": lambda: _root(skip=False, two_stream=False)}[kind]()
    if kind == "pack_streams":
        root.c._runner.pack_streams = True
    step, fwd = _messages(root, static_rows)
    if kind == "pack_streams":
        expected = "pack_streams set"
    else:          # without static_rows a pack_tail encoder is refused as a skip-padding one
        expected = "pack_tail set" if static_rows else "skip_padding encoders"
    assert step.startswith("GraphedStep: the model has ") and expected in step
    assert fwd == step.replace("GraphedStep", "GraphedForward", 1)
    assert no_capture == []


def test_uniter_is_refused_as_by_graphed_step(no_capture, cpu_models, golden):
    for task in ("mlm", "vqa2"):
        model = _build(cpu_models, golden, task)
        for static_rows in (False, True):
            step, fwd = _messages(model, static_rows)
            assert "UNITER draws its task and region masks on the host" in step
            assert fwd == step.replace("GraphedStep", "GraphedForward", 1)
    assert no_capture == []


def test_attention_and_hidden_state_outputs_are_refused(no_capture):
    for attr in ("output_attentions", "output_hidden_states"):
        lin = torch.nn.Linear(4, 4).eval()
        setattr(lin, attr, True)
        with pytest.raises(RuntimeError, match="attention probabilities or hidden states"):
            GraphedForward(lin, {"x": torch.zeros(2, 4)})
    lin = torch.nn.Linear(4, 4).eval()
    lin.config = types.SimpleNamespace(visualization=True)
    with pytest.raises(RuntimeError, match="visualization"):
        GraphedForward(lin, {"x": torch.zeros(2, 4)})
    assert no_capture == []


def test_a_model_or_batch_off_the_gpu_is_refused(no_capture):
    lin = torch.nn.Linear(4, 4).eval()
    with pytest.raises(RuntimeError, match="must be on a CUDA device \\(found cpu\\)"):
        GraphedForward(lin, SampleList(x=torch.zeros(2, 4)))
    with pytest.raises(RuntimeError, match="no tensor in the batch"):
        GraphedForward(torch.nn.Module().eval(), {"name": "x"})
    # a skip-padding model under static_rows passes the encoder checks and stops at the device check
    with pytest.raises(RuntimeError, match="CUDA device"):
        GraphedForward(_root().eval(), {"x": torch.zeros(1)}, static_rows=True)
    assert no_capture == []


def test_static_inputs_keep_their_container_types():
    sl = SampleList(a=torch.ones(2), info={"n": torch.zeros(2)}, name="coco", pair=(torch.ones(1), 3))
    out = graphs._map_keep(lambda t: t.clone(), sl)
    assert type(out) is SampleList and out.name == "coco" and out.pair[1] == 3
    assert out.a is not sl.a and torch.equal(out.a, sl.a) and type(out["info"]) is dict
    shell = graphs._map_keep(lambda t: t, out)
    shell["a"] = torch.zeros(2)                               # a forward replacing a key leaves the static inputs alone
    assert shell is not out and torch.equal(out.a, torch.ones(2)) and shell.info["n"] is out.info["n"]
