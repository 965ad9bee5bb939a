"""UNITER's host draws split from its forward (UNITER.draw) and GraphedTaskSteps' host logic, on the CPU over the kernel
test double: draw + forward makes the choices a forward alone makes from the same seeds, constructing GraphedTaskSteps
leaves the torch / numpy / random generators as they were, GraphedStep still refuses the model, and the region-loss entry
points refuse bad arguments before any launch."""
import ctypes
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_uniter_model_cpu import TASKS, _build, _sample_list, _seed_all, cpu_models, golden  # noqa: E402,F401


def _states():
    return torch.get_rng_state(), np.random.get_state(), random.getstate()


def _same_states(a, b):
    return torch.equal(a[0], b[0]) and a[1][0] == b[1][0] and np.array_equal(a[1][1], b[1][1]) and \
        a[1][2:] == b[1][2:] and a[2] == b[2]


def test_draw_then_forward_makes_todays_choices(cpu_models, golden):
    from mmf_b200.uniter_model import DRAWS_KEY
    model = _build(cpu_models, golden, "mlm")
    seen = set()
    for seed in range(12):
        _seed_all(seed)
        today = _sample_list(golden, "mlm")
        out_today = model(today)
        after_today = _states()
        _seed_all(seed)
        drawn = _sample_list(golden, "mlm")
        task = model.draw(drawn)
        out = model(drawn)
        assert _same_states(after_today, _states()), seed
        assert task == drawn["task"] == today["task"]
        seen.add(task)
        if task in ("mrc", "mrfr"):
            assert drawn[DRAWS_KEY]["image_mask"].dtype == torch.bool
            assert torch.equal(drawn["image_mask"], today["image_mask"])
            assert torch.equal(drawn[DRAWS_KEY]["image_mask"], today["image_mask"])
        else:
            assert "image_mask" not in drawn[DRAWS_KEY]
        for k, v in out_today["losses"].items():
            assert torch.equal(out["losses"][k], v), (seed, task, k)
    assert seen == set(TASKS)


def test_draw_with_a_fixed_task_draws_only_the_masks(cpu_models, golden):
    model = _build(cpu_models, golden, "mlm")
    _seed_all(3)
    before = _states()
    sl = _sample_list(golden, "mlm")
    assert model.draw(sl, task="itm") == "itm"
    assert _same_states(before, _states())
    assert model.draw(sl, task="mrc") == "mrc"
    assert torch.equal(_states()[0], before[0]) and not _same_states(before, _states())
    with pytest.raises(ValueError, match="not one of"):
        model.draw(sl, task="vqa2")


def test_classification_draws_its_one_task(cpu_models, golden):
    model = _build(cpu_models, golden, "vqa2")
    _seed_all(5)
    sl = _sample_list(golden, "vqa2")
    assert model.draw(sl) == "vqa2"
    out = model(sl)
    _seed_all(5)
    ref = model(_sample_list(golden, "vqa2"))
    assert torch.equal(out["scores"], ref["scores"])


def test_graphed_task_steps_restores_the_host_generators(cpu_models, golden, monkeypatch):
    from mmf_b200 import graphs
    model = _build(cpu_models, golden, "mlm")
    seen = []

    def capture(self, batch, warmup):
        seen.append(graphs.static_rows_active())
        for t in self.tasks:                   # warm-up and capture draw on all three generators
            model.draw(dict(batch), task=t)
            model.draw(dict(batch))
        np.random.rand(3)
        random.random()
    monkeypatch.setattr(graphs.GraphedTaskSteps, "_capture", capture)
    _seed_all(11)
    before = _states()
    steps = graphs.GraphedTaskSteps(model, lambda b: None, _sample_list(golden, "mlm"))
    assert seen == [True] and not graphs.static_rows_active()
    assert _same_states(before, _states())
    assert steps.tasks == TASKS


def test_graphed_task_steps_refusals(cpu_models, golden):
    from mmf_b200 import graphs, patch
    model = _build(cpu_models, golden, "mlm")
    with pytest.raises(RuntimeError, match="UNITER draws its task and region masks on the host.*GraphedTaskSteps"):
        graphs.GraphedStep(model, lambda b: None, {}, static_rows=True)
    with pytest.raises(TypeError, match="must define draw"):
        graphs.GraphedTaskSteps(model.uniter, lambda b: None, {})
    with pytest.raises(ValueError, match="capturable=True"):
        graphs.GraphedTaskSteps(model, lambda b: None, {}, optimizer=torch.optim.SGD(model.parameters(), lr=0.1))
    with pytest.raises(ValueError, match="max_grad_norm"):
        graphs.GraphedTaskSteps(model, lambda b: None, {}, max_grad_norm=1.0)
    assert patch.set_skip_padding(model, True) > 0
    with pytest.raises(RuntimeError, match="skip_padding"):
        graphs.GraphedTaskSteps(model, lambda b: None, {})


def test_region_loss_entry_points_refuse_bad_arguments_before_a_launch():
    from mmf_b200 import functional as F
    from mmf_b200 import lib, ops
    syms = lib.header_symbols()
    for name in ("mmfb_kl_rows_bounded", "mmfb_mse_rows_bounded"):
        assert name in syms and hasattr(lib.LIB, name)
        fn = getattr(lib.LIB, name)
        assert fn(None, 8, 4, 8, None, 8, None, None, None, None, None) == lib.MMFB_ERR_ARG
        assert "null pointer" in lib.last_error()
    z, t = torch.zeros(4, 8, dtype=torch.bfloat16), torch.zeros(4, 8)
    idx, c, s, rl = torch.zeros(4, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), torch.ones(1), torch.zeros(4)
    n0 = lib.launch_count()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        F.kl_rows_bounded(z, 8, t, idx, c, s, rl)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        F.mse_rows_bounded(z, t, idx, c, s, rl)
    with pytest.raises(ValueError, match="kind"):
        ops.region_loss_static(z, torch.zeros(8, 8), torch.zeros(8), t, idx, c, s, "ce")
    assert lib.launch_count() == n0
    if not torch.cuda.is_available():
        buf = (ctypes.c_float * 64)()
        p = ctypes.cast(buf, ctypes.c_void_p)
        assert lib.LIB.mmfb_kl_rows_bounded(p, 8, 4, 8, p, 8, p, p, p, p, None) == lib.MMFB_ERR_DEVICE
