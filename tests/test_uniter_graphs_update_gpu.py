"""MMF's fp16 update and update_frequency on UNITER's per-task graphs, on the H100.

Kernel level: the gated AdamW launches (mmfb_adamw_hparams_active, mmfb_adamw_active, mmfb_adamw_segments_active) with a
random per-slot mask over a pack and loose segments, in the fp32 and the loss-scaling instantiations: active slots equal
the ungated launches bit for bit; inactive slots keep their weights, moments, step counts (their NaN-poisoned gradients
are not read) and get a frozen row; nothing outside the buffers is written; a set found_inf leaves everything alone.

Model level, under torch.use_deterministic_algorithms: GraphedTaskSteps with a GradScaler (K = 1 and 4, with the fused
check too) and with update_frequency=4 against MMF's eager loop on a twin, bit for bit on losses, parameters, moments,
step counts, scaler state and which parameters have a .grad, over updates whose tasks leave a head out and reach it in
the next, with an overflowing micro-batch and a DeviceLRScheduler stepped per update."""
import copy
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import guarded as G  # noqa: E402
import test_uniter_graphs_gpu as UG  # noqa: E402
import test_uniter_model_cpu as C  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
INF = float("inf")


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
PACK_GROUPS = 3
SEG_SIZES = (1, 9, 3129, 20000)


def _inputs(seed, scale_g):
    """a flat pack of PACK_GROUPS groups (slots 0..2) and four loose segments (slots 3..6), each buffer placed between
    sentinel guards; returns the (view, base) pairs"""
    g = torch.Generator().manual_seed(seed)
    blocks = [3, 5, 2]                                      # 2048-element chunks per group, interleaved below
    gid = torch.cat([torch.full((b * 256,), i, dtype=torch.uint8) for i, b in enumerate(blocks)])
    gid = gid[torch.randperm(gid.numel(), generator=g)]
    n = gid.numel() * 8
    rnd = lambda k, s: torch.randn(k, generator=g) * s
    pack = [G.place(t.to(DEV), rows_before=8, rows_after=24)
            for t in (rnd(n, 1.0), rnd(n, scale_g), rnd(n, 1e-3), rnd(n, 1.0).abs() * 1e-5)]
    segs = [[G.place(t.to(DEV), rows_before=5, rows_after=7)
             for t in (rnd(k, 1.0), rnd(k, scale_g), rnd(k, 1e-3), rnd(k, 1.0).abs() * 1e-5)] for k in SEG_SIZES]
    return gid.to(DEV), pack, segs


def _launch(gid, pack, segs, hp_state, mode, amp, active):
    """hparams, then the pack and the segments launches, gated when `active` is given"""
    from mmf_b200 import functional as F
    groups, slots, steps, hp = hp_state
    kw = dict(amp)
    F.adamw_hparams(groups, slots, steps, hp, mode, **({"found_inf": kw["found_inf"]} if "found_inf" in kw else {}),
                    **({} if active is None else {"active": active}))
    p, gr, m, v = (vw for vw, _ in pack)
    F.adamw(p, gr, m, v, None, beta1=0.9, beta2=0.999, eps=1e-6, mode=mode, group_of_block=gid,
            hp_dev=hp[:PACK_GROUPS], grad_scale_dev=kw.pop("coef"), **kw,
            **({} if active is None else {"active": active[:PACK_GROUPS]}))
    table = F.adamw_segment_table([tuple(vw for vw, _ in s) + (PACK_GROUPS + i,) for i, s in enumerate(segs)])
    F.adamw_segments(table, hp, mode=mode, **kw, **({} if active is None else {"active": active}))


def _hp_state(step0):
    from mmf_b200 import functional as F, lib
    n_slots = PACK_GROUPS + len(SEG_SIZES)
    groups = torch.tensor([[1e-3, 0.01, 0.9, 0.999, 1e-6], [2e-3, 0.0, 0.9, 0.999, 1e-6]], dtype=torch.float64,
                          device=DEV)
    slots = F.adamw_slot_table([(s % 2, lib.MMFB_ADAMW_SLOT_CORRECT_BIAS) for s in range(n_slots)], DEV)
    steps, sbase = G.place(step0.to(DEV), rows_before=2, rows_after=2)
    hp, hbase = G.embed((n_slots, 8), torch.float32, rows_before=1, rows_after=1)
    hp.fill_(0.25)
    return (groups, slots, steps, hp), (sbase, hbase)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("amp", [False, True])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gated_launches_equal_ungated_on_active_slots_and_leave_the_rest(mode, amp, seed):
    n_slots = PACK_GROUPS + len(SEG_SIZES)
    g = torch.Generator().manual_seed(100 + seed)
    mask = torch.randint(0, 2, (n_slots,), generator=g, dtype=torch.uint8)
    mask[seed % PACK_GROUPS], mask[(seed + 1) % PACK_GROUPS] = 1, 0   # a pack group on each side
    mask[PACK_GROUPS + seed], mask[PACK_GROUPS + 3] = 0, 1
    mask = mask * torch.randint(1, 256, (n_slots,), generator=g, dtype=torch.uint8).clamp_min(1)  # any non-zero byte
    step0 = torch.randint(0, 9, (n_slots,), generator=g, dtype=torch.int64)
    scale_g = 3000.0 * 1e-2 if amp else 1e-2
    amp_kw = lambda f: dict(coef=torch.tensor([0.37], device=DEV),
                            **({"loss_scale_dev": torch.tensor(3000.0, device=DEV), "found_inf": f} if amp else {}))
    # the ungated reference
    gid, pack_r, segs_r = _inputs(seed, scale_g)
    hp_r, _ = _hp_state(step0)
    _launch(gid, pack_r, segs_r, hp_r, mode, amp_kw(torch.zeros((), device=DEV)), None)
    # the gated launch on the same inputs, with the inactive slots' gradients poisoned
    _, pack, segs = _inputs(seed, scale_g)
    hp_g, (sbase, hbase) = _hp_state(step0)
    off = mask == 0
    blk_off = off[:PACK_GROUPS].to(DEV)[gid.long()].repeat_interleave(8)
    pack[1][0][blk_off] = float("nan")
    before = [vw.clone() for vw, _ in pack]
    seg_before = []
    for i, s in enumerate(segs):
        if off[PACK_GROUPS + i]:
            s[1][0].fill_(float("nan"))
        seg_before.append([vw.clone() for vw, _ in s])
    active, abase = G.place(mask.to(DEV), rows_before=16, rows_after=16)
    _launch(gid, pack, segs, hp_g, mode, amp_kw(torch.zeros((), device=DEV)), active)
    torch.cuda.synchronize()
    for k in (0, 2, 3):
        got, want, old = pack[k][0], pack_r[k][0], before[k]
        assert torch.equal(_bits(got[~blk_off]), _bits(want[~blk_off])), (mode, amp, k)
        assert torch.equal(_bits(got[blk_off]), _bits(old[blk_off])), (mode, amp, k)
    for i, (s, r, b) in enumerate(zip(segs, segs_r, seg_before)):
        for k in (0, 2, 3):
            want = b[k] if off[PACK_GROUPS + i] else r[k][0]
            assert torch.equal(_bits(s[k][0]), _bits(want)), (mode, amp, i, k)
    for vw, base in pack + [x for s in segs for x in s]:
        G.untouched(base, vw, what="adamw guard")
    steps, hp = hp_g[2], hp_g[3]
    assert steps.tolist() == [s0 + (0 if o else 1) for s0, o in zip(step0.tolist(), off.tolist())]
    frozen = torch.tensor([0.0, 0.0, 0.0, 1.0], device=DEV)
    for s in range(n_slots):
        if off[s]:
            assert torch.equal(hp[s, :4], frozen) and torch.equal(_bits(hp[s, 4:7]), _bits(hp_r[3][s, 4:7])), s
        else:
            assert torch.equal(_bits(hp[s]), _bits(hp_r[3][s])), s
    G.untouched(sbase, steps, what="step guard")
    G.untouched(hbase, hp, what="hp guard")
    G.untouched(abase, active, what="active guard")
    assert torch.equal(active.cpu(), mask)                   # read, never written
    if not amp:
        return
    # a set found_inf: the gated launches write nothing, whatever the mask says
    snap = [vw.clone() for vw, _ in pack] + [vw.clone() for s in segs for vw, _ in s] + [steps.clone(), hp.clone()]
    _launch(gid, pack, segs, hp_g, mode, amp_kw(torch.ones((), device=DEV)), active)
    after = [vw for vw, _ in pack] + [vw for s in segs for vw, _ in s] + [steps, hp]
    for a, b in zip(after, snap):
        assert torch.equal(a.view(torch.uint8) if a.dtype == torch.int64 else _bits(a),
                           b.view(torch.uint8) if b.dtype == torch.int64 else _bits(b))


def test_gated_entry_points_refuse_bad_arguments_before_a_launch():
    import ctypes
    from mmf_b200 import functional as F, lib
    n0 = lib.launch_count()
    hp = torch.zeros(2, 8, device=DEV)
    x = torch.zeros(16, device=DEV)
    with pytest.raises(ValueError, match="active must be a contiguous uint8"):
        F.adamw(x, x, x, x, None, beta1=0.9, beta2=0.999, eps=1e-6, mode=0, hp_dev=hp,
                active=torch.ones(3, dtype=torch.uint8, device=DEV))
    with pytest.raises(ValueError, match="pass hp_dev"):
        F.adamw(x, x, x, x, [dict(lr=0.0, weight_decay=0.0, step_size=0.0, bc2_sqrt=1.0)], beta1=0.9, beta2=0.999,
                eps=1e-6, mode=0, active=torch.ones(1, dtype=torch.uint8, device=DEV))
    a = lib.AdamWArgs()
    a.param = a.grad = a.exp_avg = a.exp_avg_sq = x.data_ptr()
    a.n, a.n_groups = 16, 1
    act = torch.ones(1, dtype=torch.uint8, device=DEV)
    assert lib.LIB.mmfb_adamw_active(ctypes.byref(a), act.data_ptr(), None) == lib.MMFB_ERR_ARG   # no hp_dev
    a.hp_dev = hp.data_ptr()
    assert lib.LIB.mmfb_adamw_active(ctypes.byref(a), None, None) == lib.MMFB_ERR_ARG
    assert lib.LIB.mmfb_adamw_hparams_active(ctypes.byref(lib.AdamWHparamsArgs()), None, None) == lib.MMFB_ERR_ARG
    assert lib.LIB.mmfb_adamw_segments_active(ctypes.byref(lib.AdamWSegmentsArgs()), None, None) == lib.MMFB_ERR_ARG
    s = lib.AdamWSegmentsArgs()
    s.found_inf = x.data_ptr() + 2
    assert lib.LIB.mmfb_adamw_segments_active(ctypes.byref(s), act.data_ptr(), None) == lib.MMFB_ERR_ARG
    assert "4-byte aligned" in lib.last_error()
    assert lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# the registered model
# ---------------------------------------------------------------------------------------------------------------------
# mrc is not reached in the first group and is in the second; the third holds the overflowing micro-batch
SEQUENCE = ["mlm", "itm", "mlm", "wra", "mrc", "mlm", "mrfr", "mrc", "itm", "mrfr", "wra", "mlm", "mrc", "wra", "itm",
            "itm", "mrfr", "mlm"]
OVERFLOW = 9
MAX_NORM = 1.0


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(C.GOLD, "uniter_model.pt"), weights_only=False)


def _forced(model, seq):
    """model.draw with the task taken from seq when the caller draws one (the masks are still drawn)"""
    orig = model.draw

    def draw(sl, task=None):
        return orig(sl, task=seq.pop(0) if task is None else task)
    model.draw = draw


def _loss_fn(model, meta):
    run = UG._loss_fn(model, meta)

    def fn(b):
        b = dict(b)
        mult = b.pop("mult")
        return run(b) * mult
    return fn


def _opt(m, fused):
    from mmf_b200.optim import B200AdamW
    decay = [p for n, p in m.named_parameters() if not n.endswith("bias") and "LayerNorm" not in n]
    rest = [p for n, p in m.named_parameters() if n.endswith("bias") or "LayerNorm" in n]
    return B200AdamW([{"params": decay, "weight_decay": 0.01}, {"params": rest, "weight_decay": 0.0}], lr=1e-3,
                     capturable=True, fused_inf_check=fused)


def _states():
    return torch.get_rng_state(), np.random.get_state(), random.getstate()


def _set(state):
    torch.set_rng_state(state[0]); np.random.set_state(state[1]); random.setstate(state[2])


@pytest.mark.parametrize("k,scaled,fused", [(1, True, False), (4, True, False), (4, True, True), (4, False, False)])
def test_replays_equal_mmfs_eager_loop_bit_for_bit(golden, k, scaled, fused):
    from mmf_b200.graphs import GraphedTaskSteps, static_rows
    from mmf_b200.optim import DeviceLRScheduler
    model, batch, meta = UG._case(golden, "mlm")
    twin = copy.deepcopy(model)
    seq, seq_t = list(SEQUENCE), list(SEQUENCE)
    _forced(model, seq)
    _forced(twin, seq_t)
    opt, opt_t = _opt(model, fused), _opt(twin, fused)
    sched = DeviceLRScheduler(opt, "warmup_linear", num_warmup_steps=2, num_training_steps=12)
    sched_t = DeviceLRScheduler(opt_t, "warmup_linear", num_warmup_steps=2, num_training_steps=12)
    sc = torch.amp.GradScaler("cuda", growth_interval=2) if scaled else None
    sc_t = torch.amp.GradScaler("cuda", growth_interval=2) if scaled else None
    one = torch.ones((), device=DEV)
    with UG._deterministic():
        C._seed_all(7)
        before = _states()
        steps = GraphedTaskSteps(model, _loss_fn(model, meta), dict(batch, mult=one), optimizer=opt,
                                 max_grad_norm=MAX_NORM, lr_scheduler=sched, scaler=sc, update_frequency=k)
        assert UG._same_states(before, _states()) and sched.last_epoch == 0
        assert not scaled or (sc._scale is None or sc.get_scale() == 65536.0 and int(sc._growth_tracker) == 0)
        assert all(int(st.get("step", 0)) == 0 for st in opt.state.values())
        loss_t = _loss_fn(twin, meta)
        mrc = list(model.uniter.heads["mrc"].parameters())
        seen = {"skipped_mrc": False, "reached_after": False, "updates": 0}

        def update(group, where):
            if sc_t is None:
                opt_t.clip_grad_norm(MAX_NORM)
                opt_t.step()
            else:
                if fused:
                    opt_t.clip_grad_norm(MAX_NORM, scaler=sc_t)
                else:
                    opt_t.clip_grad_norm(MAX_NORM, scale=sc_t._get_scale_async())
                sc_t.step(opt_t)
                sc_t.update()
            sched_t.step()
            seen["updates"] += 1
            torch.cuda.synchronize()
            assert steps.pending == 0
            if "mrc" not in group:
                seen["skipped_mrc"] = True
                assert all(p.grad is None for p in mrc)
            elif seen["skipped_mrc"]:
                seen["reached_after"] = True
            _assert_same(model, twin, opt, opt_t, where)
            if sc is not None:
                assert sc.get_scale() == sc_t.get_scale(), where
                assert int(sc._growth_tracker) == int(sc_t._growth_tracker), where
            assert sched.last_epoch == sched_t.last_epoch == seen["updates"]

        group = []
        for i in range(len(SEQUENCE)):
            b = dict(batch, is_correct=(batch["is_correct"] + i) % 2,
                     mult=torch.tensor(INF if i == OVERFLOW and scaled else 1.0, device=DEV))
            if not group:
                twin.zero_grad(set_to_none=True)
            state = _states()
            got = steps(b).detach().clone()
            task = steps.task
            group.append(task)
            after = _states()
            _set(state)
            sl = dict(b)
            assert twin.draw(sl) == task
            assert UG._same_states(after, _states())
            with static_rows():
                ref = loss_t(sl)
            (ref if sc_t is None else sc_t.scale(ref)).backward()
            assert torch.equal(_bits(got.float().reshape(1)), _bits(ref.detach().float().reshape(1))), (i, task)
            if len(group) < k:
                assert steps.pending == len(group)
                continue
            update(group, (i, group))
            group = []
        if group:                                           # MMF's last, partial update of a run
            steps.finish_update()
            update(group, ("finish_update", group))
            steps.finish_update()                           # nothing pending: no update
            torch.cuda.synchronize()
            _assert_same(model, twin, opt, opt_t, "second finish_update")
        assert not seq and (k == 1 or (seen["skipped_mrc"] and seen["reached_after"]))
        if scaled:
            assert sc.get_scale() != 65536.0

def _assert_same(model, twin, opt, opt_t, where):
    for (n, p), q in zip(model.named_parameters(), twin.parameters()):
        assert torch.equal(_bits(p.detach()), _bits(q.detach())), (where, n)
        assert (p.grad is None) == (q.grad is None), (where, n)
        if q in opt_t.state:
            for key in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(_bits(opt.state[p][key]), _bits(opt_t.state[q][key])), (where, n, key)
    sd, sd_t = opt.state_dict()["state"], opt_t.state_dict()["state"]
    for key, v in sd_t.items():
        assert int(sd[key]["step"]) == int(v["step"]), (where, key)
    for key, v in sd.items():
        if key not in sd_t:
            assert int(v.get("step", 0)) == 0, (where, key)       # never reached: never stepped
