"""MMF's update finished on the device, on the H100: the learning-rate schedules of mmfb_lr_schedule against the
reference's schedulers on a torch optimizer over 60 updates; the non-finite check of mmfb_grad_norm_check /
mmfb_grad_check against GradScaler's own foreach check, one inf / NaN / finite 1e20 at a time; whole fp32 and fp16
updates of MMBT configs[0] and M4C through GraphedStep(optimizer=, lr_scheduler=) against MMF's eager loop with a host
LambdaLR, bit for bit under deterministic mode; a checkpoint resumed mid-run; and the profiler's view of a fused-check
step (no foreach check kernel)."""
import bisect
import copy
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

import test_graphed_accumulate_gpu as GA  # noqa: E402
import test_optim_capturable_gpu as OC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
INF, NAN = float("inf"), float("nan")
N_UPDATES = 60


# ---------------------------------------------------------------------------------------------------------------------
# the reference's schedules, restated (mmf/modules/schedulers.py, mmf/utils/general.py:lr_lambda_update, and the
# transformers <= 4.10 schedules the reference pins); tests/test_device_update_cpu.py checks them against the
# reference's own functions where its tree is present
def ref_linear(num_warmup_steps, num_training_steps):
    def lr_lambda(current_step):
        if current_step < num_warmup_steps:
            return float(current_step) / float(max(1, num_warmup_steps))
        return max(0.0, float(num_training_steps - current_step) / float(max(1, num_training_steps - num_warmup_steps)))
    return lr_lambda


def ref_cosine(num_warmup_steps, num_training_steps, num_cycles=0.5):
    def lr_lambda(current_step):
        if current_step < num_warmup_steps:
            return float(current_step) / float(max(1, num_warmup_steps))
        progress = float(current_step - num_warmup_steps) / float(max(1, num_training_steps - num_warmup_steps))
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(num_cycles) * 2.0 * progress)))
    return lr_lambda


def ref_pythia(training):
    def lr_lambda(i_iter):
        if training["use_warmup"] is True and i_iter <= training["warmup_iterations"]:
            alpha = float(i_iter) / float(training["warmup_iterations"])
            return training["warmup_factor"] * (1.0 - alpha) + alpha
        idx = bisect.bisect(training["lr_steps"], i_iter)
        return pow(training["lr_ratio"], idx)
    return lr_lambda


class RefMultiStep(torch.optim.lr_scheduler.LambdaLR):
    """MultiStepScheduler (its get_lr; the lambda LambdaLR holds is never called)"""

    def __init__(self, optimizer, **kwargs):
        self.use_warmup = kwargs["use_warmup"]
        self.lr_steps = kwargs["lr_steps"]
        self.lr_ratio = kwargs["lr_ratio"]
        self.warmup_iterations = kwargs["warmup_iterations"] if self.use_warmup else 0
        self.warmup_factor = kwargs["warmup_factor"]
        assert self.warmup_iterations < self.lr_steps[0]
        super().__init__(optimizer, lambda s: 1.0)

    def get_lr(self):
        if self.last_epoch <= self.warmup_iterations and self.use_warmup is True:
            alpha = float(self.last_epoch) / float(self.warmup_iterations)
            lr_ratio = self.warmup_factor * (1.0 - alpha) + alpha
            return [base_lr * lr_ratio for base_lr in self.base_lrs]
        return [base_lr * self.lr_ratio ** bisect.bisect_right(self.lr_steps, self.last_epoch)
                for base_lr in self.base_lrs]


# warm-up end at 7, milestones at 15 / 30 / 44, end of training at 50, updates 51..60 after it
TRAINING = dict(use_warmup=True, warmup_iterations=7, warmup_factor=0.2, lr_steps=[15, 30, 44], lr_ratio=0.3)
SCHEDULES = {
    "warmup_linear": (dict(num_warmup_steps=7, num_training_steps=50), lambda o: torch.optim.lr_scheduler.LambdaLR(
        o, ref_linear(7, 50))),
    "warmup_cosine": (dict(num_warmup_steps=7, num_training_steps=50, num_cycles=0.5),
                      lambda o: torch.optim.lr_scheduler.LambdaLR(o, ref_cosine(7, 50, 0.5))),
    "multi_step": (dict(TRAINING), lambda o: RefMultiStep(o, **TRAINING)),
    "pythia": (None, lambda o: torch.optim.lr_scheduler.LambdaLR(o, ref_pythia(TRAINING))),
}


def device_scheduler(opt, kind):
    from mmf_b200.optim import DeviceLRScheduler
    from mmf_b200.registry import registry
    if kind != "pythia":
        return DeviceLRScheduler(opt, kind, **SCHEDULES[kind][0])
    prev = registry.get("config")
    registry.register("config", {"training": dict(TRAINING)})       # pythia reads training.* from the config
    try:
        return DeviceLRScheduler(opt, "pythia")
    finally:
        registry.register("config", prev)


def host_scheduler(opt, kind):
    return SCHEDULES[kind][1](opt)


def _ulps(a, b):
    return abs(a - b) / math.ulp(b) if b != 0.0 else (0.0 if a == 0.0 else INF)


def _bits(t):
    return t.detach().float().reshape(-1).contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(SCHEDULES))
def test_schedules_equal_the_reference_schedulers(kind):
    """60 updates of the device schedule against the reference's scheduler on a torch optimizer, two groups with
    different base lrs: bit for bit; warmup_cosine within 2 ulp of the host's cosine term, carried through 1 + cos
    (near the end of a half cycle 1 + cos cancels, and one ulp of cos is several ulp of the lr); the lr before the
    first step is the step-0 value"""
    from mmf_b200.optim import B200AdamW
    a, b = torch.nn.Parameter(torch.zeros(8, device=DEV)), torch.nn.Parameter(torch.zeros(8, device=DEV))
    opt = B200AdamW([{"params": [a]}, {"params": [b], "lr": 3.7e-5}], lr=1.3e-4, capturable=True)
    sched = device_scheduler(opt, kind)
    host_opt = torch.optim.SGD([{"params": [torch.nn.Parameter(torch.zeros(1))]},
                                {"params": [torch.nn.Parameter(torch.zeros(1))], "lr": 3.7e-5}], lr=1.3e-4)
    ref = host_scheduler(host_opt, kind)
    worst = 0.0
    bases = [1.3e-4, 3.7e-5]
    for t in range(N_UPDATES + 1):
        if t:
            sched.step()
            ref.step()
        got, want = sched.get_last_lr(), [g["lr"] for g in host_opt.param_groups]
        assert sched.last_epoch == ref.last_epoch == t
        for x, y, base in zip(got, want, bases):
            if kind == "warmup_cosine":
                worst = max(worst, _ulps(x, y))
                # lr = base * 0.5 * (1 + cos): 2 ulp of cos (2 * 2**-53 near |cos| = 1) is base * 2**-53 of lr
                assert abs(x - y) <= base * 2.0 ** -53 + 2 * math.ulp(y), (kind, t, x, y)
            else:
                assert x == y, (kind, t, x, y)
    print("%s: largest difference %.1f ulp" % (kind, worst))
    assert [g["lr"] for g in opt.param_groups] == [1.3e-4, 3.7e-5]      # the host groups keep their base lr


def test_the_schedule_is_what_the_next_adamw_step_reads():
    """the group table after sched.step() holds the lr an eager step with a host LambdaLR stages"""
    from mmf_b200.optim import B200AdamW
    torch.manual_seed(3)
    p = torch.nn.Parameter(torch.randn(40, device=DEV))
    q = torch.nn.Parameter(p.detach().clone())
    opt = B200AdamW([p], lr=2e-3, capturable=True, arithmetic="torch")
    opt_h = B200AdamW([q], lr=2e-3, capturable=True, arithmetic="torch")
    sched = device_scheduler(opt, "warmup_linear")
    ref = torch.optim.lr_scheduler.LambdaLR(opt_h, ref_linear(7, 50))
    for t in range(12):
        g = torch.randn(40, device=DEV)
        p.grad, q.grad = g.clone(), g.clone()
        opt.step()
        opt_h.step()
        sched.step()
        ref.step()
        assert torch.equal(_bits(p), _bits(q)), t


# ---------------------------------------------------------------------------------------------------------------------
def _grad_set(g):
    """a pack-sized fp32 buffer, a loose fp32 gradient, a bf16 one with a scalar tail, and an fp32 view off 16-byte
    alignment (read element by element)"""
    base = torch.randn(3 * 16384 + 1000, generator=g).to(DEV)
    return [torch.randn(40000, generator=g).to(DEV) * 1e-2, torch.randn(1000, generator=g).to(DEV),
            torch.randn(333, generator=g).to(DEV).to(torch.bfloat16), base[1:1 + 2 * 16384 + 77]]


PLACES = {"pack": (0, 12345), "loose": (1, 0), "segment_end": (3, -1), "bf16_tail": (2, -1)}


@pytest.mark.parametrize("value", [INF, -INF, NAN, 1e20, None])
@pytest.mark.parametrize("place", list(PLACES))
def test_found_inf_equals_gradscalers_check(place, value):
    """mmfb_grad_norm_check and mmfb_grad_check against torch's _amp_foreach_non_finite_check_and_unscale_ on the same
    gradients: the same flag; a finite 1e20 (its square overflows fp32) is not a skip; the norm keeps grad_norm's bits"""
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(5)
    grads = _grad_set(g)
    if value is not None:
        i, j = PLACES[place]
        grads[i][j] = value
    table = F.grad_norm_table(grads)
    want = torch.zeros((), device=DEV)
    # GradScaler's kernel has no bf16 variant; widening to fp32 keeps every value and so its finiteness
    torch._amp_foreach_non_finite_check_and_unscale_([x.float() for x in grads], want, torch.ones((), device=DEV))
    with OC._deterministic():
        for _ in range(2):
            found = torch.full((1,), 7.0, device=DEV)
            out = F.grad_norm_check(table, 1.0, found)
            ref = F.grad_norm(table, 1.0)
            assert found.item() == want.item(), (place, value)
            assert torch.equal(out.view(torch.int32), ref.view(torch.int32))
            found2 = torch.full((1,), 7.0, device=DEV)
            F.grad_check(table, found2)
            assert found2.item() == want.item(), (place, value)
    assert (want.item() == 0.0) == (value is None or value == 1e20)


# ---------------------------------------------------------------------------------------------------------------------
def _mmbt_case():
    model, batches, loss_of, groups, hp, _ = GA._mmbt(6)
    return model, batches, loss_of, groups, hp


CASES = {"mmbt": _mmbt_case, "m4c": OC._m4c_case}


def _loose(model):
    from mmf_b200 import engine as E
    packed = {id(p) for pk in (E.ParamPack._live or ()) for p in pk.params}
    return [p for p in model.parameters() if id(p) not in packed and p.grad is not None]


def _packed(model):
    from mmf_b200 import engine as E
    packed = {id(p) for pk in (E.ParamPack._live or ()) for p in pk.params}
    return [p for p in model.parameters() if id(p) in packed and p.grad is not None]


@pytest.mark.parametrize("clip", [True, False])
def test_fused_check_updates_equal_gradscalers_path(clip):
    """eager fp16-style updates of MMBT: the fused check (clip_grad_norm(c, scaler=) or check_finite) against the same
    capturable optimizer under GradScaler's own check, one inf / NaN / 1e20 per update in a pack, a loose parameter
    and the last element of a loose segment: found_inf, skips, back-off and growth, parameters and moments"""
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp = _mmbt_case()
    twin = copy.deepcopy(model)
    opt = B200AdamW(groups(model), capturable=True, fused_inf_check=True, **hp)
    opt_t = B200AdamW(groups(twin), capturable=True, **hp)
    mk = lambda: torch.amp.GradScaler("cuda", init_scale=2.0 ** 10, growth_interval=2)
    sc, sc_t = mk(), mk()
    inject = [None, ("pack", INF), ("loose", NAN), ("segment_end", 1e20), ("pack", -INF), None, None,
              ("loose", 1e20), None]
    with OC._deterministic():
        for u, inj in enumerate(inject):
            b = batches[u % len(batches)]
            for m, s in ((model, sc), (twin, sc_t)):
                m.zero_grad(set_to_none=True)
                s.scale(loss_of(m)(b)).backward()
                if inj is not None:
                    where, v = inj
                    ps = _packed(m) if where == "pack" else _loose(m)
                    t = ps[len(ps) // 2].grad if where == "pack" else ps[0].grad
                    t.view(-1)[-1 if where == "segment_end" else 0] = v
            if clip:
                opt.clip_grad_norm(0.25, scaler=sc)
                opt_t.clip_grad_norm(0.25, scale=sc_t._get_scale_async())
            else:
                opt.check_finite(sc)
            found = sum(v.item() for v in sc._per_optimizer_states[id(opt)]["found_inf_per_device"].values())
            sc.step(opt)
            sc_t.step(opt_t)
            found_t = sum(v.item() for v in sc_t._per_optimizer_states[id(opt_t)]["found_inf_per_device"].values())
            assert found == found_t == (1.0 if inj is not None and inj[1] != 1e20 else 0.0), (u, inj)
            sc.update()
            sc_t.update()
            assert sc.get_scale() == sc_t.get_scale() and torch.equal(sc._growth_tracker, sc_t._growth_tracker), u
            got, want = OC._state(model, opt), OC._state(twin, opt_t)
            for n in got:
                for x, y in zip(got[n][:3], want[n][:3]):
                    assert (x is None and y is None) or torch.equal(_bits(x), _bits(y)), (u, n)
                assert got[n][3] == want[n][3], (u, n)


# ---------------------------------------------------------------------------------------------------------------------
def _eager_update(opt, scaler, sched):
    if scaler is None:
        opt.clip_grad_norm(GA.MAX_NORM)
        opt.step()
    else:
        opt.clip_grad_norm(GA.MAX_NORM, scale=scaler._get_scale_async())
        scaler.step(opt)
        scaler.update()
    sched.step()


@pytest.mark.parametrize("variant", ["plain", "accumulate", "scaler"])
@pytest.mark.parametrize("case", list(CASES))
def test_graphed_schedule_equals_the_eager_loop_with_a_host_lambdalr(case, variant):
    """20 updates of GraphedStep(optimizer=, lr_scheduler=DeviceLRScheduler) against MMF's eager loop on a twin with a
    host LambdaLR, under deterministic mode: parameters, moments and step counts bit for bit after every update.
    accumulate: update_frequency=4.  scaler: a GradScaler starting at 2**120, so the first updates overflow and are
    skipped while the schedule still advances; the graphed side checks with the fused launch"""
    from mmf_b200 import modules
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW, DeviceLRScheduler
    model, batches, loss_of, groups, hp = CASES[case]()
    GA._torch_dropout_off(model)
    K = 4 if variant == "accumulate" else 1
    mk = (lambda: torch.amp.GradScaler("cuda", init_scale=2.0 ** 120, growth_interval=3)) if variant == "scaler" \
        else (lambda: None)
    sc, sc_t = mk(), mk()
    with OC._deterministic():
        twin = copy.deepcopy(model)
        loss_of(twin)(batches[0]).backward()
        twin.zero_grad(set_to_none=True)
        opt = B200AdamW(groups(model), capturable=True, fused_inf_check=sc is not None, **hp)
        opt_t = B200AdamW(groups(twin), capturable=True, **hp)
        sched = DeviceLRScheduler(opt, "warmup_linear", num_warmup_steps=5, num_training_steps=15)
        sched_t = torch.optim.lr_scheduler.LambdaLR(opt_t, ref_linear(5, 15))
        c0 = modules._SEED_COUNTER[0]
        step = GraphedStep(model, loss_of(model), batches[0], warmup=3, optimizer=opt, max_grad_norm=GA.MAX_NORM,
                           scaler=sc, update_frequency=K, lr_scheduler=sched)
        c1 = modules._SEED_COUNTER[0]
        seed = c1 - (c1 - c0) // 4
        assert sched.last_epoch == 0 and sched.get_last_lr() == [g["lr"] for g in opt_t.param_groups]
        run = loss_of(twin)
        for u in range(20):
            twin.zero_grad(set_to_none=True)
            for j in range(K):
                b = batches[(u * K + j) % len(batches)]
                step(b)
                GA._eager_micro(run, b, seed, False, sc_t)
            _eager_update(opt_t, sc_t, sched_t)
            torch.cuda.synchronize()
            assert sched.last_epoch == sched_t.last_epoch == u + 1
            assert sched.get_last_lr() == [g["lr"] for g in opt_t.param_groups], (case, variant, u)
            got, want = OC._state(model, opt), OC._state(twin, opt_t)
            for n in got:
                for x, y in zip(got[n][:3], want[n][:3]):
                    assert (x is None and y is None) or torch.equal(_bits(x), _bits(y)), (case, variant, u, n)
                assert got[n][3] == want[n][3], (case, variant, u, n)
            if sc is not None:
                assert sc.get_scale() == sc_t.get_scale(), (case, u)
        if sc is not None and case == "mmbt":      # MMBT's gradients overflow at 2**120, M4C's do not
            assert sc.get_scale() < 2.0 ** 120      # updates were skipped (backed off), and the schedule still moved


def test_a_checkpoint_resumes_at_the_same_counter():
    """MMBT, 14 updates with a device multi_step schedule: 7 graphed updates, the model / optimizer / scheduler
    state_dicts into fresh objects, 7 more graphed updates; against 14 uninterrupted eager updates, bit for bit"""
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp = _mmbt_case()
    GA._torch_dropout_off(model)
    with OC._deterministic():
        ref_model = copy.deepcopy(model)
        fresh = copy.deepcopy(model)
        ref_opt = B200AdamW(groups(ref_model), capturable=True, **hp)
        ref_sched = device_scheduler(ref_opt, "multi_step")
        for u in range(14):
            ref_model.zero_grad(set_to_none=True)
            loss_of(ref_model)(batches[u % len(batches)]).backward()
            ref_opt.clip_grad_norm(GA.MAX_NORM)
            ref_opt.step()
            ref_sched.step()
        opt = B200AdamW(groups(model), capturable=True, **hp)
        sched = device_scheduler(opt, "multi_step")
        step = GraphedStep(model, loss_of(model), batches[0], optimizer=opt, max_grad_norm=GA.MAX_NORM,
                           lr_scheduler=sched)
        for u in range(7):
            step(batches[u % len(batches)])
        ck = (copy.deepcopy(model.state_dict()), copy.deepcopy(opt.state_dict()), copy.deepcopy(sched.state_dict()))
        assert ck[2]["last_epoch"] == 7
        fresh.load_state_dict(ck[0])
        opt2 = B200AdamW(groups(fresh), capturable=True, **hp)
        opt2.load_state_dict(ck[1])
        sched2 = device_scheduler(opt2, "multi_step")
        sched2.load_state_dict(ck[2])
        assert sched2.last_epoch == 7 and sched2.get_last_lr() == sched.get_last_lr()
        step2 = GraphedStep(fresh, loss_of(fresh), batches[0], optimizer=opt2, max_grad_norm=GA.MAX_NORM,
                            lr_scheduler=sched2)
        assert sched2.last_epoch == 7
        for u in range(7, 14):
            step2(batches[u % len(batches)])
        torch.cuda.synchronize()
        assert sched2.last_epoch == ref_sched.last_epoch == 14
        got, want = OC._state(fresh, opt2), OC._state(ref_model, ref_opt)
        for n in got:
            for x, y in zip(got[n][:3], want[n][:3]):
                assert (x is None and y is None) or torch.equal(_bits(x), _bits(y)), n
            assert got[n][3] == want[n][3], n


# ---------------------------------------------------------------------------------------------------------------------
def _cuda_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA], \
        [e.name for e in prof.events()]


def test_the_foreach_check_is_gone():
    """a replayed fused-check update and an eager one contain no kernel of GradScaler's foreach check; GradScaler's
    own path, profiled the same way, does"""
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp = _mmbt_case()
    twin = copy.deepcopy(model)
    opt = B200AdamW(groups(model), capturable=True, fused_inf_check=True, **hp)
    sc = torch.amp.GradScaler("cuda")
    step = GraphedStep(model, loss_of(model), batches[0], optimizer=opt, max_grad_norm=GA.MAX_NORM, scaler=sc)
    step(batches[1])
    kernels, _ = _cuda_kernels(lambda: step(batches[2]))
    assert kernels and not any("non_finite" in k or "foreach" in k for k in kernels), kernels

    opt_t = B200AdamW(groups(twin), capturable=True, fused_inf_check=True, **hp)
    sc_t = torch.amp.GradScaler("cuda")

    def eager(fused):
        twin.zero_grad(set_to_none=True)
        sc_t.scale(loss_of(twin)(batches[3])).backward()
        torch.cuda.synchronize()

        def update():
            if fused:
                opt_t.clip_grad_norm(GA.MAX_NORM, scaler=sc_t)
            else:
                opt_t.clip_grad_norm(GA.MAX_NORM, scale=sc_t._get_scale_async())
            sc_t.step(opt_t)
            sc_t.update()
        return _cuda_kernels(update)
    eager(True)                                   # builds the tables
    kernels, ops = eager(True)
    assert not any("non_finite" in k or "foreach" in k for k in kernels + ops), kernels + ops
    kernels, ops = eager(False)
    assert any("non_finite_check_and_unscale" in k for k in kernels + ops)


# ---------------------------------------------------------------------------------------------------------------------
def test_new_entry_points_read_and_write_only_their_buffers():
    """NaN around everything the three launches read (a NaN read would show in found_inf or an lr) and sentinels around
    everything they write: only the lr column, the counter, found_inf and the workspace inside its bounds change"""
    from mmf_b200 import functional as F, lib
    g = torch.Generator().manual_seed(9)
    store = torch.full((3 * 16384 + 64,), NAN, device=DEV)          # gradients inside NaN
    grads = [store[8:8 + 40000], store[40016:40016 + 333]]
    for t in grads:
        t.copy_(torch.randn(t.numel(), generator=g).to(DEV))
    table = F.grad_norm_table(grads)
    fi = torch.full((5,), -3.0, device=DEV)
    for launch in (lambda f: F.grad_norm_check(table, 1.0, f), lambda f: F.grad_check(table, f)):
        launch(fi[2:3])
        assert fi[2].item() == 0.0 and fi[[0, 1, 3, 4]].eq(-3.0).all()
    # the workspace: exactly 2 * n_blocks doubles (check) or n_blocks (check only) inside sentinels
    ws = torch.full((2 * table.n_blocks + 4,), -7.0, dtype=torch.float64, device=DEV)
    a = lib.GradNormArgs(table.segments.data_ptr(), table.n_segments, table.n_blocks, ws[2:].data_ptr(),
                         torch.empty(2, device=DEV).data_ptr(), 1.0, 2.0)
    import ctypes
    lib.check(lib.LIB.mmfb_grad_norm_check(ctypes.byref(a), fi[2:3].data_ptr(), lib._stream_ptr()))
    torch.cuda.synchronize()
    assert ws[:2].eq(-7.0).all() and ws[-2:].eq(-7.0).all() and not ws[2:-2].eq(-7.0).any()
    # the schedule: base lrs inside NaN, the table's other columns NaN, the counter between sentinels
    base = torch.full((6,), NAN, dtype=torch.float64, device=DEV)
    base[2:4] = torch.tensor([1e-3, 2e-4], dtype=torch.float64)
    tab = torch.full((2 * 5 + 6,), NAN, dtype=torch.float64, device=DEV)
    cnt = torch.tensor([-5, 4, -5], dtype=torch.int64, device=DEV)
    from mmf_b200.optim import schedule_desc
    d = schedule_desc("multi_step", use_warmup=True, lr_steps=[6], lr_ratio=0.5, warmup_iterations=3,
                      warmup_factor=0.1)
    F.lr_schedule(cnt[1:2], base[2:4], tab[3:3 + 6], d, True, lr_stride=5)
    torch.cuda.synchronize()
    assert cnt.tolist() == [-5, 5, -5]
    lr = tab[3:3 + 6]
    assert lr[0].item() == 1e-3 * 0.5 ** 0 and lr[5].item() == 2e-4 * 0.5 ** 0
    keep = torch.ones(tab.numel(), dtype=torch.bool, device=DEV)
    keep[3], keep[8] = False, False
    assert tab[keep].isnan().all()
