"""MMF's fp16 update on the fused optimizer, on the H100: the loss-scaling fields of mmfb_adamw, mmfb_adamw_segments,
mmfb_adamw_hparams and mmfb_grad_norm against the same launches on gradients GradScaler.unscale_ already rewrote, bit
for bit; a skipped step (found_inf = 1) writing nothing inside sentinel guards; four models through six fp16-autocast
steps in MMF's order (clip, scaler.step, scaler.update, one step with non-finite gradients) against the same optimizer
with `_step_supports_amp_scaling` forced off; the fused update without a host synchronisation; and
GraphedStep(scaler=...) replays against the eager fused sequence bit for bit."""
import contextlib
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

import guarded as G  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
INF, NAN = float("inf"), float("nan")


def _bits(t):
    return t.contiguous().view(torch.int32)


def _inv(scale):
    """GradScaler.unscale_'s factor: _scale.double().reciprocal().float()"""
    return scale.double().reciprocal().float()


def _hp(mode, step=4):
    import test_optim_capturable_gpu as OC
    return OC._hp_table(mode, step)


def _bufs(n, g, scale_g=1e-2):
    p = torch.randn(n, generator=g).to(DEV)
    gr = (torch.randn(n, generator=g) * scale_g).to(DEV)
    m = (torch.randn(n, generator=g) * 1e-3).to(DEV)
    v = (torch.randn(n, generator=g).abs() * 1e-5).to(DEV)
    return p, gr, m, v


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [2.0 ** 16, 3000.0])
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("hp_dev", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
def test_adamw_loss_scale_is_unscale_then_step_bit_for_bit(S, clip, hp_dev, mode):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(11 + mode)
    n = 3 * 2048 + 40
    p, gr, m, v = _bufs(n, g, scale_g=S * 1e-2)
    gr[5], gr[77] = 1e30, -3e-38                    # overflow and underflow of g * inv stay as unscale_ gives them
    scale = torch.tensor(S, device=DEV)
    found = torch.zeros((), device=DEV)
    coef = torch.tensor([0.37], device=DEV) if clip else None
    hp = _hp(mode) if hp_dev else None
    groups = None if hp_dev else [dict(lr=1e-3, weight_decay=0.01, step_size=2.7e-3, bc2_sqrt=0.06)]
    pb, pb_ref = (torch.empty(n, dtype=torch.bfloat16, device=DEV) for _ in range(2))
    ref = [t.clone() for t in (p, gr, m, v)]
    ref[1].mul_(_inv(scale))                        # what unscale_ leaves in .grad
    kw = dict(beta1=0.9, beta2=0.999, eps=1e-6, mode=mode, grad_scale=0.5, grad_scale_dev=coef, hp_dev=hp)
    F.adamw(*ref, groups, param_bf16=pb_ref, **kw)
    g0 = gr.clone()
    F.adamw(p, gr, m, v, groups, param_bf16=pb, loss_scale_dev=scale, found_inf=found, **kw)
    for got, want in ((p, ref[0]), (m, ref[2]), (v, ref[3])):
        assert torch.equal(_bits(got), _bits(want)), (S, clip, hp_dev, mode)
    assert torch.equal(pb.view(torch.int16), pb_ref.view(torch.int16))
    assert torch.equal(_bits(gr), _bits(g0))        # the scaled gradient is read, not rewritten
    # the scale alone, without a found_inf pointer
    p2, gr2, m2, v2 = (t.clone() for t in (ref[0], g0, ref[2], ref[3]))
    r2 = [p2.clone(), g0 * _inv(scale), m2.clone(), v2.clone()]
    F.adamw(*r2, groups, **kw)
    F.adamw(p2, gr2, m2, v2, groups, loss_scale_dev=scale, **kw)
    assert torch.equal(_bits(p2), _bits(r2[0])) and torch.equal(_bits(m2), _bits(r2[2]))


@pytest.mark.parametrize("S", [2.0 ** 16, 3000.0])
@pytest.mark.parametrize("clip", [False, True])
def test_segments_loss_scale_is_unscale_then_step_bit_for_bit(S, clip):
    import test_optim_capturable_gpu as OC
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(29)
    hp = _hp(1, 6)
    scale = torch.tensor(S, device=DEV)
    found = torch.zeros((), device=DEV)
    coef = torch.tensor([0.61], device=DEV) if clip else None
    segs, refs = [], []
    for n in (1, 9, 3129, 20000):
        for shifts in ((0, 0, 0, 0), (1, 1, 1, 1), (1, 0, 2, 3)):
            p, gr = OC._view(n, shifts[0], g), OC._view(n, shifts[1], g, S * 1e-2)
            m, v = OC._view(n, shifts[2], g, 1e-3), OC._view(n, shifts[3], g).abs_().mul_(1e-5)
            segs.append((p, gr, m, v, 0))
            refs.append((p.clone(), gr * _inv(scale), m.clone(), v.clone(), 0))
    F.adamw_segments(F.adamw_segment_table(refs), hp, mode=1, grad_scale_dev=coef)
    F.adamw_segments(F.adamw_segment_table(segs), hp, mode=1, grad_scale_dev=coef, loss_scale_dev=scale,
                     found_inf=found)
    for s, r in zip(segs, refs):
        for i in (0, 2, 3):
            assert torch.equal(_bits(s[i]), _bits(r[i])), (S, clip, s[0].numel())


def test_found_inf_writes_nothing():
    """found_inf = 1: params, the bf16 copy, moments, the device step counts and the hyper-parameter table keep their
    bits, and nothing around them is written"""
    from mmf_b200 import functional as F, lib
    g = torch.Generator().manual_seed(41)
    n = 2048 + 16
    found = torch.ones((), device=DEV)
    scale = torch.tensor(65536.0, device=DEV)
    coef = torch.tensor([0.5], device=DEV)
    for mode in (0, 1):
        hp = _hp(mode)
        views = []
        for t in _bufs(n, g):
            views.append(G.place(t, rows_before=8, rows_after=24))
        pb, pb_base = G.embed((n,), torch.bfloat16, rows_before=8, rows_after=24)
        pb.fill_(1.5)
        before = [vw.clone() for vw, _ in views] + [pb.clone()]
        (p, _), (gr, _), (m, _), (v, _) = views
        F.adamw(p, gr, m, v, None, beta1=0.9, beta2=0.999, eps=1e-6, mode=mode, param_bf16=pb, grad_scale_dev=coef,
                hp_dev=hp, loss_scale_dev=scale, found_inf=found)
        F.adamw(p, gr, m, v, [dict(lr=1e-3, weight_decay=0.0, step_size=1e-3, bc2_sqrt=1.0)], beta1=0.9, beta2=0.999,
                eps=1e-6, mode=mode, found_inf=found)
        F.adamw_segments(F.adamw_segment_table([(p, gr, m, v, 0)]), hp, mode=mode, loss_scale_dev=scale, found_inf=found)
        for (vw, base), b in zip(views, before):
            assert torch.equal(_bits(vw), _bits(b)), mode
            G.untouched(base, vw, what="adamw guard")
        assert torch.equal(pb.view(torch.int16), before[4].view(torch.int16))
        G.untouched(pb_base, pb, what="bf16 copy guard")
        # the step counts and the table
        groups = torch.tensor([[1e-3, 0.01, 0.9, 0.999, 1e-6]], dtype=torch.float64, device=DEV)
        slots = F.adamw_slot_table([(0, lib.MMFB_ADAMW_SLOT_CORRECT_BIAS)] * 3, DEV)
        steps, sbase = G.place(torch.tensor([4, 0, 9], dtype=torch.int64, device=DEV), rows_before=2, rows_after=2)
        table, tbase = G.embed((3, 8), torch.float32, rows_before=1, rows_after=1)
        table.fill_(0.25)
        F.adamw_hparams(groups, slots, steps, table, mode, found_inf=found)
        assert steps.tolist() == [4, 0, 9] and bool((table == 0.25).all())
        G.untouched(tbase, table, what="hp guard")
        G.untouched(sbase, steps, what="step guard")
        F.adamw_hparams(groups, slots, steps, table, mode, found_inf=torch.zeros((), device=DEV))
        assert steps.tolist() == [5, 1, 10]


@pytest.mark.parametrize("S", [2.0 ** 16, 3000.0, 0.5])
@pytest.mark.parametrize("max_norm", [0.25, 1.0, 0.1])
def test_grad_norm_device_scale_equals_the_host_product(S, max_norm):
    import numpy as np
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(7)
    grads = [(torch.randn(n, generator=g) * S * 1e-3).to(DEV) for n in (5, 16384 + 3, 700)]
    table = F.grad_norm_table(grads)
    host = float(np.float32(max_norm) * np.float32(S))       # fp32(max_norm) * S, rounded once
    want = F.grad_norm(table, host)
    got = F.grad_norm(table, max_norm, max_norm_scale_dev=torch.tensor(S, device=DEV))
    assert torch.equal(_bits(got), _bits(want)), (S, max_norm, got.tolist(), want.tolist())


# ---------------------------------------------------------------------------------------------------------------------
def _mmbt_case(p_drop=0.1):
    import bench
    torch.manual_seed(0)
    wl = bench.WORKLOADS["mmbt"]()
    model = wl.build(p_drop).to(DEV).train()
    batches = [bench.to_device(wl.host_batch(2, s), DEV) for s in range(6)]
    aux = wl.aux(2, DEV)
    return model, batches, (lambda m: (lambda b: wl.loss(m, b, aux))), (lambda m: list(m.parameters())), \
        dict(lr=1e-4, weight_decay=0.01, arithmetic="torch"), False


def _visual_bert_case():
    import test_optim_capturable_gpu as OC
    model, batches, loss_of, groups, hp = OC._trunk_case()
    return model, batches, loss_of, groups, hp, False


def _lxmert_case():
    import test_optim_capturable_gpu as OC
    model, batches, loss_of, groups, hp, static = OC._lxmert()
    while len(batches) < 6:
        batches = batches + batches
    return model, batches[:6], loss_of, groups, hp, static


def _m4c_case():
    import test_optim_capturable_gpu as OC
    model, batches, loss_of, groups, hp = OC._m4c_case()
    return model, batches, loss_of, groups, hp, False


CASES = {"mmbt": _mmbt_case, "visual_bert": _visual_bert_case, "lxmert": _lxmert_case, "m4c": _m4c_case}
MAX_NORM = 0.25          # an fp32 value: max_norm * S on the host and in fp32 on the device agree for every S
OVERFLOW_STEP = 3


def _autocast():
    return torch.autocast("cuda", dtype=torch.float16)


def _full_state(model, opt, scaler):
    out = {}
    for n, p in model.named_parameters():
        st = opt.state.get(p, {})
        out[n] = (p.detach().clone(), *(st[k].clone() if k in st else None for k in ("exp_avg", "exp_avg_sq")),
                  int(st["step"]) if "step" in st else 0)
    out["<scale>"] = (scaler._scale.clone(), scaler._growth_tracker.clone())
    return out


def _assert_same(got, want, what):
    """bitwise; a moment one side has not created yet equals zeros (a capturable step creates the state of the
    parameters it steps even when found_inf skips the update, as torch's fused Adam does)"""
    for k, w in want.items():
        for x, y in zip(got[k], w):
            if (x is None) != (y is None):
                assert not (x if y is None else y).any(), what + (k,)
            elif torch.is_tensor(y):
                assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                                   y.view(torch.int32) if y.dtype == torch.float32 else y), what + (k,)
            else:
                assert x == y, what + (k, x, y)


@pytest.mark.parametrize("case", list(CASES))
def test_fused_amp_steps_equal_unscale_then_step_bit_for_bit(case):
    """six fp16-autocast steps in MMF's order, one with non-finite gradients: the fused update (scale and found_inf read
    by the kernels) against GradScaler's unscale_ + host read + step on the same optimizer class"""
    from mmf_b200.graphs import static_rows
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp, static = CASES[case]()
    ctx = static_rows if static else contextlib.nullcontext
    ref = copy.deepcopy(model)
    opt, opt_r = B200AdamW(groups(model), capturable=True, **hp), B200AdamW(groups(ref), capturable=True, **hp)
    assert opt._step_supports_amp_scaling and opt_r._step_supports_amp_scaling
    opt_r._step_supports_amp_scaling = False
    sc, sc_r = torch.amp.GradScaler("cuda", growth_interval=2), torch.amp.GradScaler("cuda", growth_interval=2)
    skipped = 0
    for step in range(6):
        mult = INF if step == OVERFLOW_STEP else 1.0
        for m, s in ((model, sc), (ref, sc_r)):
            m.zero_grad()
            with ctx(), _autocast():
                loss = loss_of(m)(batches[step]) * mult
            s.scale(loss).backward()
        for p, q in zip(model.parameters(), ref.parameters()):
            assert (p.grad is None) == (q.grad is None)
            if p.grad is not None:
                q.grad.copy_(p.grad)                 # in place: packed gradients stay in their flat buffers
        torch.cuda.synchronize()
        if step >= 1:
            torch.cuda.set_sync_debug_mode("error")
        try:
            opt.clip_grad_norm(MAX_NORM, scale=sc._get_scale_async())
            sc.step(opt)
            sc.update()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        s_before = sc_r.get_scale()
        opt_r.clip_grad_norm(MAX_NORM * s_before)    # MMF: clip_gradients(..., scale=scaler.get_scale())
        sc_r.step(opt_r)
        sc_r.update()
        skipped += sc_r.get_scale() < s_before
        _assert_same(_full_state(model, opt, sc), _full_state(ref, opt_r, sc_r), (case, step))
    assert skipped >= 1, case                        # the overflow step was skipped (and backed the scale off)
    assert opt._cap is not None and (opt._cap.packs or opt._cap.loose)


def test_non_capturable_optimizer_keeps_the_unscale_path():
    from mmf_b200.optim import B200AdamW
    opt = B200AdamW([torch.nn.Parameter(torch.zeros(8, device=DEV))])
    assert not getattr(opt, "_step_supports_amp_scaling", False)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["mmbt", "visual_bert"])
def test_graphed_amp_step_is_the_eager_fused_step_bit_for_bit(case):
    import test_optim_capturable_gpu as OC
    model, batches, loss_of, groups, hp, _ = _mmbt_case(0.0) if case == "mmbt" else CASES[case]()
    for n, m in model.named_modules():           # torch's own dropout draws differ between replay and eager step
        if isinstance(m, torch.nn.Dropout) and "layer" not in n:
            m.p = 0.0
    with OC._deterministic():
        _graph_vs_eager(case, model, batches, loss_of, groups, hp)


def _graph_vs_eager(case, model, batches, loss_of, groups, hp):
    from mmf_b200 import modules
    from mmf_b200.graphs import GraphedStep
    from mmf_b200.optim import B200AdamW
    mults = [torch.tensor(INF if i == OVERFLOW_STEP else 1.0, device=DEV) for i in range(len(batches))]

    def loss_fn_of(m):
        run = loss_of(m)

        def fn(b):
            with torch.autocast("cuda", dtype=torch.float16, cache_enabled=False):
                return run(b["data"]) * b["mult"]
        return fn
    twin = copy.deepcopy(model)
    with _autocast():
        loss_of(twin)(batches[0]).backward()     # the twin's lazy engine state
    twin.zero_grad(set_to_none=True)
    opt, opt_t = B200AdamW(groups(model), capturable=True, **hp), B200AdamW(groups(twin), capturable=True, **hp)
    sc, sc_t = torch.amp.GradScaler("cuda", growth_interval=2), torch.amp.GradScaler("cuda", growth_interval=2)
    params0 = {n: p.detach().clone() for n, p in model.named_parameters()}
    c0 = modules._SEED_COUNTER[0]
    step = GraphedStep(model, loss_fn_of(model), {"data": batches[0], "mult": mults[0]}, warmup=3, optimizer=opt,
                       max_grad_norm=MAX_NORM, scaler=sc)
    c1 = modules._SEED_COUNTER[0]
    per_step = (c1 - c0) // 4
    torch.cuda.synchronize()
    # capturing changes neither the model, nor the optimizer, nor the scaler
    for n, p in model.named_parameters():
        assert torch.equal(_bits(p.detach()), _bits(params0[n])), n
        st = opt.state.get(p, {})
        assert int(st.get("step", 0)) == 0 and all(not st[k].any() for k in ("exp_avg", "exp_avg_sq") if k in st), n
    assert sc.get_scale() == 65536.0 and int(sc._growth_tracker) == 0
    with pytest.raises(ValueError, match="scaler"):
        GraphedStep(model, loss_fn_of(model), {"data": batches[0], "mult": mults[0]}, scaler=sc)
    for i, b in enumerate(batches):
        loss = step({"data": b, "mult": mults[i]})
        twin.zero_grad(set_to_none=True)
        modules._SEED_COUNTER[0] = c1 - per_step
        ref = loss_fn_of(twin)({"data": b, "mult": mults[i]})
        sc_t.scale(ref).backward()
        opt_t.clip_grad_norm(MAX_NORM, scale=sc_t._get_scale_async())
        sc_t.step(opt_t)
        sc_t.update()
        torch.cuda.synchronize()
        assert torch.equal(_bits(loss.detach().float().reshape(1)), _bits(ref.detach().float().reshape(1))), (case, i)
        _assert_same(_full_state(model, opt, sc), _full_state(twin, opt_t, sc_t), (case, i))
        for (n, p), q in zip(model.named_parameters(), twin.parameters()):
            assert (p.grad is None) == (q.grad is None), (case, i, n)
            if p.grad is not None:                # both hold the scaled gradients (non-finite ones at a skipped step)
                assert torch.equal(_bits(p.grad), _bits(q.grad)), (case, i, n)
    assert sc.get_scale() == sc_t.get_scale() != 65536.0
