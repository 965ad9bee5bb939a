"""GraphedStep(..., update_frequency=K) on the H100, against MMF's eager accumulation loop (zero_grad, K backwards of
losses not divided by K, clip, step) on a twin of the model from the same state, under deterministic mode: two updates
of K = 3 distinct batches bit for bit (each micro-batch's loss, then parameters, moments, step counts and .grad after
each update) for MMBT, the VisualBERT trunk and LXMERT pretraining under static rows; a GradScaler group with a
non-finite micro-batch skipped and the scale backed off once; finish_update() after a partial group; update_frequency=1
against the one-graph step; and dropout drawing fresh masks per micro-batch, whose accumulated gradient is the sum of
the per-micro-batch ones."""
import contextlib
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

import test_amp_step_gpu as AS  # noqa: E402
import test_optim_capturable_gpu as OC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
K = 3
MAX_NORM = 0.25
INF = float("inf")


def _bits(t):
    return t.detach().float().reshape(-1).contiguous().view(torch.int32)


def _mmbt(n, p_drop=0.0):
    import bench
    torch.manual_seed(0)
    wl = bench.WORKLOADS["mmbt"]()
    model = wl.build(p_drop).to(DEV).train()
    batches = [bench.to_device(wl.host_batch(2, s), DEV) for s in range(n)]
    aux = wl.aux(2, DEV)
    return model, batches, (lambda m: (lambda b: wl.loss(m, b, aux))), (lambda m: list(m.parameters())), \
        dict(lr=1e-4, weight_decay=0.01, arithmetic="torch"), False


def _visual_bert(n):
    model, batches, loss_of, groups, hp = OC._trunk_case()
    assert len(batches) >= n
    return model, batches[:n], loss_of, groups, hp, False


def _lxmert(n):
    model, batches, loss_of, groups, hp, static = OC._lxmert()
    extra = [dict(b, image_feature_0=b["image_feature_0"] * s) for b, s in zip(batches, (0.5, 1.5))]
    batches = batches + extra
    assert len(batches) >= n
    return model, batches[:n], loss_of, groups, hp, static


CASES = {"mmbt": _mmbt, "visual_bert": _visual_bert, "lxmert": _lxmert}


def _torch_dropout_off(model):
    for n, m in model.named_modules():            # torch's own dropout draws differ between replay and eager step
        if isinstance(m, torch.nn.Dropout) and "layer" not in n:
            m.p = 0.0


def _ctx(static):
    from mmf_b200.graphs import static_rows
    return static_rows() if static else contextlib.nullcontext()


def _capture(model, loss_of, example, groups, hp, static, **kw):
    """GraphedStep(..., update_frequency=...) over `model` and an eager twin from the same state (its lazy engine state
    built, no gradients), with capturable optimizers over both; also the dropout seed counter of the captured forward"""
    from mmf_b200 import modules
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW
    twin = copy.deepcopy(model)
    with _ctx(static):
        loss_of(twin)(example).backward()
    twin.zero_grad(set_to_none=True)
    opt, opt_t = B200AdamW(groups(model), capturable=True, **hp), B200AdamW(groups(twin), capturable=True, **hp)
    before = OC._state(model, opt)
    c0 = modules._SEED_COUNTER[0]
    step = GraphedStep(model, loss_of(model), example, warmup=3, static_rows=static, optimizer=opt, **kw)
    c1 = modules._SEED_COUNTER[0]
    seed = c1 - (c1 - c0) // 4                    # three warm-up forwards, then the captured one
    torch.cuda.synchronize()
    after = OC._state(model, opt)
    for n, (p, m, v, s) in before.items():        # capturing does not step
        q, m2, v2, s2 = after[n]
        assert torch.equal(_bits(p), _bits(q)) and s == s2 == 0, n
        assert all(x is None or not x.any() for x in (m2, v2)), n
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert grads and not any(bool(g.any()) for g in grads)        # and leaves the gradients zeroed
    assert step.pending == 0
    return step, twin, opt, opt_t, seed


def _eager_micro(run, b, seed, static, scaler=None):
    """one micro-batch of MMF's loop on the twin, with the dropout seed of the captured forward"""
    from mmf_b200 import modules
    modules._SEED_COUNTER[0] = seed
    with _ctx(static):
        loss = run(b)
    (loss if scaler is None else scaler.scale(loss)).backward()
    return loss


def _eager_update(opt, scaler=None):
    """MMF's _finish_update on the fused optimizer"""
    if scaler is None:
        opt.clip_grad_norm(MAX_NORM)
        opt.step()
        return
    opt.clip_grad_norm(MAX_NORM, scale=scaler._get_scale_async())
    scaler.step(opt)
    scaler.update()


def _same_values(x, y):
    """equal values, NaN where the other is NaN (the sign of a zero gradient may differ: the graph adds the first
    micro-batch to zeros, the eager loop adopts it)"""
    return x.shape == y.shape and bool(((x == y) | (x.isnan() & y.isnan())).all())


def _same(model, opt, twin, opt_t, what, steps=None):
    got, want = OC._state(model, opt), OC._state(twin, opt_t)
    for (n, p), q in zip(model.named_parameters(), twin.parameters()):
        for x, y in zip(got[n][:3], want[n][:3]):
            assert (x is None) == (y is None) and (x is None or torch.equal(_bits(x), _bits(y))), what + (n,)
        assert got[n][3] == want[n][3], what + (n, got[n][3], want[n][3])
        assert steps is None or p.grad is None or got[n][3] == steps, what + (n, got[n][3])
        assert (p.grad is None) == (q.grad is None), what + (n,)
        assert p.grad is None or _same_values(p.grad, q.grad), what + (n,)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_accumulated_updates_equal_the_eager_loop_bit_for_bit(case):
    model, batches, loss_of, groups, hp, static = CASES[case](2 * K)
    _torch_dropout_off(model)
    with OC._deterministic():
        step, twin, opt, opt_t, seed = _capture(model, loss_of, batches[0], groups, hp, static, max_grad_norm=MAX_NORM,
                                                update_frequency=K)
        run = loss_of(twin)
        for u in range(2):
            twin.zero_grad(set_to_none=True)      # MMF's _start_update
            for j in range(K):
                b = batches[u * K + j]
                loss = step(b)
                assert step.pending == (j + 1) % K
                ref = _eager_micro(run, b, seed, static)
                torch.cuda.synchronize()
                assert torch.equal(_bits(loss), _bits(ref)), (case, u, j, loss.item(), ref.item())
            _eager_update(opt_t)
            torch.cuda.synchronize()
            _same(model, opt, twin, opt_t, (case, u), steps=u + 1)


def test_a_non_finite_micro_batch_skips_its_update_once():
    """three groups of fp16-autocast micro-batches under a GradScaler; micro-batch 2 of group 2 overflows"""
    model, batches, loss_of, groups, hp, _ = _mmbt(3 * K)
    _torch_dropout_off(model)
    data = [{"data": b, "mult": torch.tensor(INF if i == K + 1 else 1.0, device=DEV)} for i, b in enumerate(batches)]

    def loss_fn_of(m):
        run = loss_of(m)

        def fn(b):
            with torch.autocast("cuda", dtype=torch.float16, cache_enabled=False):
                return run(b["data"]) * b["mult"]
        return fn
    sc, sc_t = torch.amp.GradScaler("cuda"), torch.amp.GradScaler("cuda")
    with OC._deterministic():
        step, twin, opt, opt_t, seed = _capture(model, loss_fn_of, data[0], groups, hp, False, scaler=sc,
                                                max_grad_norm=MAX_NORM, update_frequency=K)
        assert sc.get_scale() == 65536.0 and int(sc._growth_tracker) == 0
        run = loss_fn_of(twin)
        states = []
        for u in range(3):
            twin.zero_grad(set_to_none=True)
            for j in range(K):
                loss = step(data[u * K + j])
                ref = _eager_micro(run, data[u * K + j], seed, False, sc_t)
                torch.cuda.synchronize()
                assert torch.equal(_bits(loss), _bits(ref)), (u, j)
            _eager_update(opt_t, sc_t)
            torch.cuda.synchronize()
            state = AS._full_state(model, opt, sc)
            AS._assert_same(state, AS._full_state(twin, opt_t, sc_t), ("group", u))
            for (n, p), q in zip(model.named_parameters(), twin.parameters()):
                assert (p.grad is None) == (q.grad is None) and (p.grad is None or _same_values(p.grad, q.grad)), (u, n)
            states.append(state)
        assert [float(s["<scale>"][0]) for s in states] == [65536.0, 32768.0, 32768.0]   # backed off once
        assert sc.get_scale() == sc_t.get_scale() == 32768.0
        # the overflowing group changed no parameter, moment or step count; the next one updated
        AS._assert_same({k: v for k, v in states[1].items() if k != "<scale>"},
                        {k: v for k, v in states[0].items() if k != "<scale>"}, ("skipped",))
        stepped = [n for n, p in model.named_parameters() if p.grad is not None]
        assert stepped and all(states[0][n][3] == states[1][n][3] == 1 and states[2][n][3] == 2 for n in stepped)
        assert any(not torch.equal(states[2][n][0], states[1][n][0]) for n in stepped)


def test_finish_update_after_a_partial_group_is_the_eager_partial_update():
    model, batches, loss_of, groups, hp, _ = _mmbt(2 + K)
    _torch_dropout_off(model)
    with OC._deterministic():
        step, twin, opt, opt_t, seed = _capture(model, loss_of, batches[0], groups, hp, False, max_grad_norm=MAX_NORM,
                                                update_frequency=K)
        run = loss_of(twin)
        start = OC._state(model, opt)
        step.finish_update()                      # nothing pending: nothing happens
        torch.cuda.synchronize()
        for n, x in OC._state(model, opt).items():
            assert torch.equal(_bits(x[0]), _bits(start[n][0])) and x[3] == 0, n
        twin.zero_grad(set_to_none=True)
        for b in batches[:2]:
            step(b)
            _eager_micro(run, b, seed, False)
        assert step.pending == 2
        step.finish_update()
        assert step.pending == 0
        _eager_update(opt_t)
        torch.cuda.synchronize()
        _same(model, opt, twin, opt_t, ("partial",), steps=1)
        step.finish_update()                      # again nothing pending
        torch.cuda.synchronize()
        _same(model, opt, twin, opt_t, ("no-op",), steps=1)
        # the next group is a full one, from zeroed gradients
        twin.zero_grad(set_to_none=True)
        for b in batches[2:]:
            step(b)
            _eager_micro(run, b, seed, False)
        assert step.pending == 0
        _eager_update(opt_t)
        torch.cuda.synchronize()
        _same(model, opt, twin, opt_t, ("full",), steps=2)


def test_update_frequency_1_is_the_one_graph_step():
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp, _ = _mmbt(4)
    _torch_dropout_off(model)
    other = copy.deepcopy(model)
    with OC._deterministic():
        opt, opt_o = B200AdamW(groups(model), capturable=True, **hp), B200AdamW(groups(other), capturable=True, **hp)
        a = GraphedStep(model, loss_of(model), batches[0], optimizer=opt, max_grad_norm=MAX_NORM)
        b = GraphedStep(other, loss_of(other), batches[0], optimizer=opt_o, max_grad_norm=MAX_NORM, update_frequency=1)
        assert not hasattr(b, "update_graph") and not hasattr(b, "zero_graph")
        for i, x in enumerate(batches):
            la, lb = a(x), b(x)
            b.finish_update()                     # nothing to do at K = 1
            torch.cuda.synchronize()
            assert b.pending == 0 and torch.equal(_bits(la), _bits(lb)), i
            _same(model, opt, other, opt_o, ("k=1", i), steps=i + 1)


def test_each_micro_batch_draws_its_own_dropout_masks():
    """K replays of one batch with dropout 0.1 in the fused layers: K different losses, and the accumulated gradient is
    the eager accumulation with each replay's keep bits (bit for bit) and the sum of the per-micro-batch gradients"""
    model, batches, loss_of, groups, hp, _ = _mmbt(1, p_drop=0.1)
    _torch_dropout_off(model)
    b = batches[0]
    with OC._deterministic():
        step, twin, opt, opt_t, seed = _capture(model, loss_of, b, groups, hp, False, update_frequency=K)
        e0 = int(step.epoch)
        losses = []
        for _ in range(K):
            losses.append(step(b).detach().clone())
        torch.cuda.synchronize()
        assert len({float(x) for x in losses}) == K, losses
        acc = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
        run = loss_of(twin)
        per = []
        for j in range(K):                        # each micro-batch alone, with the keep bits of its replay
            twin.zero_grad(set_to_none=True)
            step.epoch.fill_(e0 + j + 1)
            ref = _eager_micro(run, b, seed, False)
            torch.cuda.synchronize()
            assert torch.equal(_bits(ref), _bits(losses[j])), j
            per.append({n: p.grad.clone() for n, p in twin.named_parameters() if p.grad is not None})
        twin.zero_grad(set_to_none=True)
        for j in range(K):                        # MMF's accumulation over the same draws
            step.epoch.fill_(e0 + j + 1)
            _eager_micro(run, b, seed, False)
        torch.cuda.synchronize()
        got = {n: p.grad for n, p in twin.named_parameters() if p.grad is not None}
        assert set(got) == set(acc) == set(per[0])
        for n, g in acc.items():
            assert _same_values(g, got[n]), n
            total = per[0][n] + per[1][n] + per[2][n]
            # the kernels add each micro-batch's partial sums onto the buffer, so the order of the fp32 additions
            # differs from adding finished gradients
            assert float((g - total).abs().max()) <= 1e-5 * float(total.abs().max()) + 1e-30, n
        assert any(not torch.equal(per[0][n], per[1][n]) for n in acc)
