"""UNITER in CUDA graphs on the H100: the region-loss row kernels against fp64, the static-rows region heads against
today's, and GraphedTaskSteps' replays against the eager static-rows step, bit for bit under
torch.use_deterministic_algorithms - per task, over a mixed-task training run with a capturable B200AdamW and clipping,
and for classification."""
import contextlib
import copy
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kernel_check as KC  # noqa: E402
import test_uniter_model_cpu as C  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
TILE = 128


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _bound(c):
    return torch.tensor([c], dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("kind", ["kl", "mse"])
def test_region_row_kernels_against_fp64(kind):
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    g = torch.Generator().manual_seed(7 if kind == "kl" else 8)
    cap, V = 300, (1601 if kind == "kl" else 2048)
    Vp = -(-V // 8) * 8
    n_tgt = cap + 37
    if kind == "kl":
        tgt = torch.softmax(torch.randn(n_tgt, V, generator=g) * 3, dim=-1)
        tgt[torch.rand(n_tgt, V, generator=g) < 0.2] = 0.0           # exact zeros: xlogy(0, 0) = 0
    else:
        tgt = torch.randn(n_tgt, V, generator=g)
    tgt = tgt.to(DEV)
    for c in (0, 1, TILE, cap):
        r = min(cap, -(-c // TILE) * TILE)
        z0 = (torch.randn(cap, Vp, generator=g) * 2).to(torch.bfloat16).to(DEV)
        idx = torch.full((cap,), -1, dtype=torch.int32)
        idx[:c] = torch.randperm(n_tgt, generator=g)[:c].to(torch.int32)
        idx = idx.to(DEV)
        scale = torch.tensor([1.0 / max(c, 1) / (1 if kind == "kl" else V)], dtype=torch.float32, device=DEV)
        z, rl = z0.clone(), torch.full((cap,), -5.0, device=DEV)
        n0 = lib.launch_count()
        if kind == "kl":
            F.kl_rows_bounded(z, V, tgt, idx, _bound(c), scale, rl)
        else:
            F.mse_rows_bounded(z, tgt, idx, _bound(c), scale, rl)
        assert lib.launch_count() == n0 + 1
        assert not z[c:r].any() and bool((rl[c:r] == 0).all())
        assert torch.equal(z[r:], z0[r:]) and bool((rl[r:] == -5.0).all())
        if not c:
            continue
        zz, q, s = z0[:c, :V].double(), tgt.index_select(0, idx[:c].long()).double(), scale.double().item()
        if kind == "kl":
            logp = torch.log_softmax(zz, dim=-1)
            Q = q.sum(-1, keepdim=True)
            terms = torch.xlogy(q, q) - q * logp
            loss_ref, loss_abs = terms.sum(-1), (torch.xlogy(q, q).abs() + (q * logp).abs()).sum(-1)
            grad_ref = (logp.exp() * Q - q) * s
            grad_abs = (logp.exp() * Q + q) * s
            assert not z[:c, V:].any()
        else:
            d = zz - q
            loss_ref, loss_abs = (d * d).sum(-1), (d * d).sum(-1)
            grad_ref, grad_abs = 2 * d * s, 2 * (zz.abs() + q.abs()) * s
        # the gradient: fp32 arithmetic of a few terms (exp2 / log, a block sum over the row), rounded once to bf16
        KC.assert_within(z[:c, :V], grad_ref, 2.0 ** -9 * grad_ref.abs() + 64 * KC.U_F32 * grad_abs, KC.row_layout(),
                         "%s gradient (count %d)" % (kind, c))
        # the row loss: fp32 sums of V terms in a fixed tree order
        KC.assert_within(rl[:c], loss_ref, 2 * V * KC.U_F32 * loss_abs + 1e-30, KC.row_layout(), "%s row loss" % kind)


def test_region_row_kernels_refuse_bad_shapes_before_a_launch():
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    z = torch.zeros(16, 1608, dtype=torch.bfloat16, device=DEV)
    tgt = torch.zeros(16, 1601, device=DEV)
    idx, rl, s = torch.zeros(16, dtype=torch.int32, device=DEV), torch.zeros(16, device=DEV), torch.ones(1, device=DEV)
    n0 = lib.launch_count()
    with pytest.raises(ValueError):
        F.kl_rows_bounded(z[:, :1600], 1601, tgt, idx, _bound(1), s, rl)          # no room for the padding columns
    with pytest.raises(ValueError):
        F.kl_rows_bounded(z, 1601, tgt[:, :1600], idx, _bound(1), s, rl)
    with pytest.raises(ValueError):
        F.kl_rows_bounded(z, 1601, tgt, idx[:8], _bound(1), s, rl)
    with pytest.raises(ValueError):
        F.mse_rows_bounded(z, tgt, idx, _bound(1), s, rl)
    with pytest.raises(ValueError):
        F.mse_rows_bounded(z[:, :1600], tgt[:, :1600], idx, _bound(1), s, rl[:8])
    with pytest.raises(ValueError):
        F.mse_rows_bounded(z[:, :1600], tgt[:, :1600].to(torch.float64), idx, _bound(1), s, rl)
    assert lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# the registered model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(C.GOLD, "uniter_model.pt"), weights_only=False)


def _case(golden, case):
    import mmf_b200.mmft  # noqa: F401
    import mmf_b200.models as MD
    model = C._build(MD, golden, case).cuda()
    sl = C._sample_list(golden, case, device=DEV)
    sl["image_info_0"] = {k: torch.as_tensor(v).to(DEV) for k, v in sl["image_info_0"].items()}
    batch = {k: v for k, v in sl.items() if torch.is_tensor(v) or isinstance(v, dict)}
    meta = {k: v for k, v in sl.items() if k not in batch}
    return model, batch, meta


def _loss_fn(model, meta):
    from mmf_b200.sample import SampleList

    def run(b):
        out = model(SampleList(dict(b, **meta)))
        return sum(v.sum() for v in out["losses"].values())
    return run


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("task", C.TASKS)
def test_static_heads_match_todays_heads(golden, task):
    from mmf_b200.graphs import static_rows
    model, batch, meta = _case(golden, "mlm")
    twin = copy.deepcopy(model)
    C._seed_all(3)
    today_sl = dict(batch)
    model.draw(today_sl, task=task)
    static_sl = dict(today_sl)
    model.zero_grad(set_to_none=True)
    ref = _loss_fn(model, meta)(today_sl)
    ref.backward()
    with static_rows():
        got = _loss_fn(twin, meta)(static_sl)
    got.backward()
    assert abs(got.item() - ref.item()) <= 1e-2 * abs(ref.item()) + 1e-6, (task, got.item(), ref.item())
    g_today, g_static = _grads(model), _grads(twin)
    assert set(g_today) == set(g_static)
    for n, gr in g_today.items():
        err = ((g_static[n].double() - gr.double()).norm() / gr.double().norm().clamp_min(1e-12)).item()
        assert err <= 3e-2 or gr.abs().max() < 1e-8, (task, n, err)


def test_static_heads_with_no_masked_region_give_zero(golden):
    """a region mask with no region set: loss exactly 0 and zero gradients from the region heads, never NaN"""
    from mmf_b200.graphs import static_rows
    from mmf_b200.mmft import MRCHead, MRFRHead
    model, batch, meta = _case(golden, "mlm")
    heads = model.uniter.heads
    for task, head in (("mrc", heads["mrc"]), ("mrfr", heads["mrfr"])):
        assert isinstance(head, (MRCHead, MRFRHead))
        sl = dict(batch)
        model.draw(sl, task=task)
        sl[model.draws_key]["image_mask"].zero_()
        model.zero_grad(set_to_none=True)
        with static_rows():
            loss = _loss_fn(model, meta)(sl)
        loss.backward()
        assert loss.item() == 0.0
        for n, p in head.named_parameters():
            if n != "linear_proj_weight":
                assert p.grad is not None and not p.grad.any(), (task, n)


def _states():
    return torch.get_rng_state(), np.random.get_state(), random.getstate()


def _same_states(a, b):
    return torch.equal(a[0], b[0]) and np.array_equal(a[1][1], b[1][1]) and a[1][2:] == b[1][2:] and a[2] == b[2]


@pytest.mark.parametrize("case", ["mlm", "vqa2"])
def test_each_tasks_replay_is_the_eager_static_step_bit_for_bit(golden, case):
    from mmf_b200.graphs import GraphedTaskSteps, static_rows
    model, batch, meta = _case(golden, case)
    with _deterministic():
        twin = copy.deepcopy(model)
        C._seed_all(21)
        before = _states()
        steps = GraphedTaskSteps(model, _loss_fn(model, meta), batch)
        assert _same_states(before, _states())
        counts = {}
        for i in range(16):
            state = _states()
            b = dict(batch, is_correct=(batch["is_correct"] + i) % 2)
            loss = steps(b)
            task = steps.task
            counts[task] = counts.get(task, 0) + 1
            after = _states()
            torch.set_rng_state(state[0]); np.random.set_state(state[1]); random.setstate(state[2])
            sl = dict(b)
            assert twin.draw(sl) == task
            assert _same_states(after, _states())
            twin.zero_grad(set_to_none=True)
            with static_rows():
                ref = _loss_fn(twin, meta)(sl)
            ref.backward()
            torch.cuda.synchronize()
            assert torch.equal(loss.detach(), ref.detach()), (task, loss.item(), ref.item())
            got, want = _grads(model), _grads(twin)
            assert set(got) == set(want), task
            for n, gr in want.items():
                assert torch.equal(got[n], gr), (task, n)
    assert set(counts) == set(model.tasks)


def test_mixed_training_run_matches_eager_static_steps_bit_for_bit(golden):
    from mmf_b200.graphs import GraphedTaskSteps, static_rows
    from mmf_b200.optim import B200AdamW
    model, batch, meta = _case(golden, "mlm")
    twin = copy.deepcopy(model)

    def opt_of(m):
        decay = [p for n, p in m.named_parameters() if not n.endswith("bias") and "LayerNorm" not in n]
        rest = [p for n, p in m.named_parameters() if n.endswith("bias") or "LayerNorm" in n]
        return B200AdamW([{"params": decay, "weight_decay": 0.01}, {"params": rest, "weight_decay": 0.0}], lr=1e-3,
                         capturable=True)
    opt, opt_twin = opt_of(model), opt_of(twin)
    mrc = dict(model.uniter.heads["mrc"].named_parameters())
    checked_unused = False
    with _deterministic():
        C._seed_all(5)
        steps = GraphedTaskSteps(model, _loss_fn(model, meta), batch, optimizer=opt, max_grad_norm=1.0)
        C._seed_all(5)
        tasks = []
        for i in range(20):
            b = dict(batch, is_correct=(batch["is_correct"] + i) % 2)
            state = _states()
            snap = {n: (p.detach().clone(), {k: v.clone() for k, v in opt.state[p].items() if torch.is_tensor(v)})
                    for n, p in mrc.items() if p in opt.state}
            loss = steps(b)
            tasks.append(steps.task)
            torch.set_rng_state(state[0]); np.random.set_state(state[1]); random.setstate(state[2])
            sl = dict(b)
            assert twin.draw(sl) == steps.task
            twin.zero_grad(set_to_none=True)
            with static_rows():
                ref = _loss_fn(twin, meta)(sl)
            ref.backward()
            opt_twin.clip_grad_norm(1.0)
            opt_twin.step()
            torch.cuda.synchronize()
            assert torch.equal(loss.detach(), ref.detach()), (i, steps.task)
            if steps.task != "mrc" and snap:
                # a head the step's task does not reach keeps its values, moments and step count
                for n, p in mrc.items():
                    assert p.grad is None
                    assert torch.equal(p.detach(), snap[n][0]), n
                    for k, v in snap[n][1].items():
                        assert torch.equal(opt.state[p][k], v), (n, k)
                checked_unused = True
        assert checked_unused and set(tasks) == set(model.tasks), tasks
        for (n, p), q in zip(model.named_parameters(), twin.parameters()):
            assert torch.equal(p.detach(), q.detach()), n
            if q in opt_twin.state:
                for k in ("exp_avg", "exp_avg_sq"):
                    assert torch.equal(opt.state[p][k], opt_twin.state[q][k]), (n, k)
        sd, sd_twin = opt.state_dict()["state"], opt_twin.state_dict()["state"]
        assert sd_twin and all(sd[k]["step"] == v["step"] for k, v in sd_twin.items())
