"""The registered `uniter` model on the GPU against tests/golden/uniter_model.pt (the REFERENCE's own registered UNITER,
tools/make_golden_uniter_model.py): classification and each of the five pretraining tasks.  Bars as for the LXMERT model
(bf16 kernels against an fp32 reference): losses within 1e-2, scores within 1.5e-2, 2-D gradients within 3e-2 relative
L2 - 5e-2 for the attention query / key weights, whose gradient is what is left after the softmax's shift invariance
cancels most of each row's terms, so the bf16 rounding of the probabilities weighs more in it; integer paths bit for bit."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_uniter_model_cpu as C  # noqa: E402  (builders, sample lists and the plumbing check shared with the CPU test)
from oracle.golden_format import kept  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(C.GOLD, "uniter_model.pt"), weights_only=False)


@pytest.mark.parametrize("case", ["vqa2"] + C.TASKS)
def test_registered_model_vs_reference_golden_on_gpu(golden, case):
    import mmf_b200.mmft  # noqa: F401
    import mmf_b200.models as MD
    from mmf_b200 import lib
    model = C._build(MD, golden, case).cuda()
    g = golden[case]
    sl = C._sample_list(golden, case, device="cuda")
    C._seed_all(g.get("seed", 7))
    n0 = lib.launch_count()
    out = model(sl)
    if case != "vqa2":
        assert sl["task"] == case
    C.check_plumbing(sl, g["plumbing"])
    assert list(out["losses"].keys()) == list(g["losses"].keys())
    worst = {}
    for k, v in g["losses"].items():
        got = float(out["losses"][k].detach().sum())
        worst["loss"] = abs(got - float(v)) / max(abs(float(v)), 1e-3)
        assert worst["loss"] < 1e-2, (k, got, float(v))
    if case == "vqa2":
        worst["scores"] = C.rel(out["scores"].cpu(), g["scores"])
        assert worst["scores"] < 1.5e-2
    sum(v.sum() for v in out["losses"].values()).backward()
    torch.cuda.synchronize()
    assert lib.launch_count() > n0                       # the library's own kernels ran
    named = dict(model.named_parameters())
    checked, worst["grad"] = 0, 0.0
    for k, gr in g["grads"].items():
        if k.endswith("mrfr.linear_proj_weight"):
            continue
        assert named[k].grad is not None, k
        if kept(gr, gr)[1].norm() > 1e-6:
            e = C.rel(named[k].grad.cpu(), gr)
            worst["grad"] = max(worst["grad"], e)
            assert e < (5e-2 if ".self.query." in k or ".self.key." in k else 3e-2), (k, e)
            checked += 1
    assert checked >= 0.75 * (len(g["grads"]) - 1)
    print("\nuniter %s: " % case + "  ".join("%s %.2e" % kv for kv in worst.items()) + "  (%d gradients)" % checked)


def test_wra_step_runs_one_kernel_per_direction(golden):
    """the optimal-transport part of a WRA step is two library launches, whatever the iteration count"""
    from mmf_b200 import lib, ops
    seq = golden["ot"]["sequence_output"].to(torch.bfloat16).cuda().requires_grad_(True)
    T, R = golden["ot"]["T_len"], golden["ot"]["R_len"]
    n0 = lib.launch_count()
    d = ops.optimal_transport_dist(seq, T, R, [8, 6, 1, 4], [6, 2, 5, 1])
    assert lib.launch_count() == n0 + 1
    d.sum().backward()
    assert lib.launch_count() == n0 + 2
    assert C.rel(d.cpu(), golden["ot"]["distance"]) < 1e-4


def test_training_step_with_dropout_is_finite(golden):
    import mmf_b200.mmft  # noqa: F401
    import mmf_b200.models as MD
    cfg = dict(golden["pretraining_config"], hidden_dropout_prob=0.1)
    cfg["encoder"] = dict(cfg["encoder"], hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    model = MD.build_model(MD.load_model_config("uniter", overrides=cfg)).cuda().train()
    seen = set()
    for s in range(12):
        C._seed_all(s)
        sl = C._sample_list(golden, "mlm", device="cuda")
        out = model(sl)
        seen.add(sl["task"])
        loss = sum(v.sum() for v in out["losses"].values())
        model.zero_grad(set_to_none=True)
        loss.backward()
        assert torch.isfinite(loss), (sl["task"], loss)
        assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None), sl["task"]
    assert len(seen) >= 3
