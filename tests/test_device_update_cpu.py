"""Host side of the device update, without a GPU: the new C-ABI symbols and their refusals, the schedule descriptor
(the host's powers of lr_ratio, MMF's `is True` warm-up test, the refusals), the scheduler registrations, the
refusals of DeviceLRScheduler, B200AdamW(fused_inf_check=) and GraphedStep(lr_scheduler=), and the schedules the GPU
tests restate against the reference's own functions where the reference tree is present."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

from mmf_b200 import lib  # noqa: E402
from mmf_b200.optim import B200AdamW, DeviceLRScheduler, schedule_desc  # noqa: E402
from mmf_b200.registry import registry  # noqa: E402

NEW = ("mmfb_lr_schedule", "mmfb_grad_norm_check", "mmfb_grad_check")
INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")


def test_new_symbols_are_declared_and_exported():
    import re
    txt = open(os.path.join(INCLUDE, "mmfb200_update.h")).read()
    assert sorted(re.findall(r"^int (mmfb_[a-z0-9_]+)\(", txt, flags=re.M)) == sorted(NEW)
    assert '#include "mmfb200_update.h"' in open(os.path.join(INCLUDE, "mmfb200.h")).read()
    for s in NEW:
        assert hasattr(lib.LIB, s), s


@pytest.mark.skipif(torch.cuda.is_available(), reason="GPU present")
def test_new_entry_points_refuse_bad_arguments_and_need_a_device():
    a = lib.LrScheduleArgs()
    assert lib.LIB.mmfb_lr_schedule(None, None) == lib.MMFB_ERR_ARG
    assert lib.LIB.mmfb_lr_schedule(ctypes.byref(a), None) == lib.MMFB_ERR_ARG           # null pointers
    a.counter, a.base_lr, a.lr, a.n_groups, a.lr_stride = 8, 8, 8, 1, 1
    a.desc.kind = 7
    assert lib.LIB.mmfb_lr_schedule(ctypes.byref(a), None) == lib.MMFB_ERR_ARG           # unknown kind
    a.desc.kind = lib.MMFB_LR_PYTHIA
    assert lib.LIB.mmfb_lr_schedule(ctypes.byref(a), None) == lib.MMFB_ERR_DEVICE
    n = lib.GradNormArgs(8, 1, 1, 8, 8, 1.0, 2.0)
    assert lib.LIB.mmfb_grad_norm_check(ctypes.byref(n), None, None) == lib.MMFB_ERR_ARG
    assert lib.LIB.mmfb_grad_norm_check(ctypes.byref(n), 6, None) == lib.MMFB_ERR_ARG      # misaligned found_inf
    assert lib.LIB.mmfb_grad_norm_check(ctypes.byref(n), 8, None) == lib.MMFB_ERR_DEVICE
    assert lib.LIB.mmfb_grad_check(8, 1, 1, 8, None, None) == lib.MMFB_ERR_ARG
    assert lib.LIB.mmfb_grad_check(8, 0, 1, 8, 8, None) == lib.MMFB_ERR_ARG
    assert lib.LIB.mmfb_grad_check(8, 1, 1, 8, 8, None) == lib.MMFB_ERR_DEVICE
    assert "no CPU fallback" in lib.last_error()


def test_header_and_ctypes_mirror_of_the_schedule_structs_agree():
    hdr = open(os.path.join(INCLUDE, "mmfb200_update.h")).read()
    import re
    for struct, mirror in (("mmfb_lr_schedule_desc", lib.LrScheduleDesc), ("mmfb_lr_schedule_args", lib.LrScheduleArgs)):
        body = re.search(r"typedef struct \{([^}]*)\} %s;" % struct, hdr).group(1)
        names = re.findall(r"(\w+)(?:\[[^\]]*\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
        assert names == [f[0] for f in mirror._fields_], struct
    assert ctypes.sizeof(lib.LrScheduleDesc) == 48 + 8 * 32 + 8 * 33
    assert lib.LrScheduleArgs.desc.offset == 40


def test_descriptor_holds_the_hosts_powers_and_mmfs_warmup_test():
    d = schedule_desc("multi_step", use_warmup=True, lr_steps=[10, 20.0, 35], lr_ratio=0.1, warmup_iterations=4,
                      warmup_factor=0.25)
    assert d.kind == lib.MMFB_LR_MULTI_STEP and d.use_warmup == 1 and d.warmup_iterations == 4
    assert list(d.lr_steps[:3]) == [10, 20, 35] and d.n_lr_steps == 3
    assert [d.ratio_pow[i] for i in range(4)] == [0.1 ** i for i in range(4)]
    assert schedule_desc("pythia", use_warmup=1, lr_steps=[3], lr_ratio=0.5, warmup_iterations=2).use_warmup == 0
    d = schedule_desc("warmup_cosine", num_warmup_steps=3, num_training_steps=9, num_cycles=2)
    assert (d.kind, d.warmup_iterations, d.total_steps, d.num_cycles) == (lib.MMFB_LR_WARMUP_COSINE, 3, 9, 2.0)
    with pytest.raises(ValueError):
        schedule_desc("multi_step", use_warmup=True, lr_steps=[5], warmup_iterations=0)
    with pytest.raises(ValueError):
        schedule_desc("pythia", lr_steps=[2.5])
    with pytest.raises(ValueError):
        schedule_desc("pythia", lr_steps=list(range(1, 40)))
    with pytest.raises(TypeError):
        schedule_desc("warmup_linear", num_warmup_steps=3)
    with pytest.raises(ValueError):
        schedule_desc("step_lr")


def test_registered_under_mmfs_scheduler_names():
    for name in ("warmup_linear", "warmup_cosine", "multi_step", "pythia"):
        cls = registry.get_scheduler_class(name)
        assert cls is not None and issubclass(cls, DeviceLRScheduler), name


def test_refusals():
    p = torch.nn.Parameter(torch.zeros(8))
    with pytest.raises(TypeError, match="capturable=True"):
        DeviceLRScheduler(B200AdamW([p]), "warmup_linear", num_warmup_steps=1, num_training_steps=4)
    with pytest.raises(TypeError, match="capturable=True"):
        DeviceLRScheduler(torch.optim.SGD([p], lr=0.1), "warmup_linear", num_warmup_steps=1, num_training_steps=4)
    with pytest.raises(ValueError, match="fused_inf_check=True needs capturable=True"):
        B200AdamW([p], fused_inf_check=True)
    with pytest.raises(RuntimeError, match="CUDA device"):        # CPU parameters: no device to schedule on
        DeviceLRScheduler(B200AdamW([p], capturable=True), "warmup_linear", num_warmup_steps=1, num_training_steps=4)
    opt = B200AdamW([p], capturable=True)
    with pytest.raises(ValueError, match="needs B200AdamW"):
        opt.clip_grad_norm(1.0, scaler=torch.amp.GradScaler("cpu"))
    with pytest.raises(ValueError, match="warmup_iterations must be below"):
        DeviceLRScheduler(opt, "multi_step", use_warmup=True, lr_steps=[3], lr_ratio=0.1, warmup_iterations=3,
                          warmup_factor=0.1)


def test_graphed_step_refuses_a_scheduler_without_its_optimizer():
    from mmf_b200.graphs import GraphedStep, _check_scheduler
    model = torch.nn.Linear(2, 2)
    with pytest.raises(ValueError, match="lr_scheduler= steps inside the captured update"):
        GraphedStep(model, lambda b: b, {}, lr_scheduler=object())
    opt = B200AdamW(model.parameters(), capturable=True)
    with pytest.raises(ValueError, match="DeviceLRScheduler built on this optimizer"):
        _check_scheduler("GraphedStep", opt, torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 1.0))


def _reference_schedulers():
    """the reference's schedulers.py and lr_lambda_update, loaded by path with the oracle's stubs; None without its tree"""
    try:
        from oracle import ref_loader
    except Exception:
        return None
    root = ref_loader.REF_ROOT
    sched_py = os.path.join(root, "mmf", "modules", "schedulers.py")
    general_py = os.path.join(root, "mmf", "utils", "general.py")
    if not (os.path.exists(sched_py) and os.path.exists(general_py)):
        return None
    import bisect
    src = open(general_py).read()
    start = src.index("def lr_lambda_update")
    ns = {"bisect": bisect.bisect}
    exec(compile(src[start:src.index("\ndef ", start + 1)], general_py, "exec"), ns)
    return ns["lr_lambda_update"]


def test_the_restated_schedules_are_the_references():
    """the restatements the GPU tests compare against: transformers' schedules (the installed release) and MMF's
    lr_lambda_update taken from the reference's own source"""
    import types
    import test_device_update_gpu as T
    try:
        from transformers.optimization import get_cosine_schedule_with_warmup, get_linear_schedule_with_warmup
    except Exception:
        pytest.skip("transformers not importable")
    o = lambda: torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1.0)
    for make, mine in ((lambda x: get_linear_schedule_with_warmup(x, 7, 50), T.ref_linear(7, 50)),
                       (lambda x: get_cosine_schedule_with_warmup(x, 7, 50, 0.5), T.ref_cosine(7, 50, 0.5))):
        s = make(o())
        for t in range(61):
            assert s.lr_lambdas[0](t) == mine(t), t
    lam = _reference_schedulers()
    if lam is None:
        pytest.skip("the reference tree is not present")
    cfg = types.SimpleNamespace(training=types.SimpleNamespace(**T.TRAINING))
    mine = T.ref_pythia(T.TRAINING)
    for t in range(61):
        assert lam(t, cfg) == mine(t), t
    assert math.isfinite(mine(60))
