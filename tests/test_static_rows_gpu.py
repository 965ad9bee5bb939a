"""Static-rows masked-LM loss on the H100: the row selection and its gather, the device-bounded GEMM (forward, dgrad,
wgrad in the atomic and the ordered mode), the bounded ce_rows and column sums, the static linear + cross-entropy against
today's, and the registered LXMERT, VinVL and ViLT pretraining steps captured by GraphedStep(static_rows=True) against the
eager static-rows step, bit for bit under torch.use_deterministic_algorithms."""
import contextlib
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kernel_check as KC  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
TILE = 128


def _counts(cap):
    return sorted({0, 1, 63, 64, 65, 127, 128, 129, cap - 1, cap})


def _rounded(c, cap):
    return min(cap, -(-c // TILE) * TILE)


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


@pytest.mark.parametrize("cap", [300, 5000])
def test_selection_and_its_backward_equal_index_select(cap):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(cap)
    H = 768
    x = torch.randn(cap, H, generator=g).to(torch.bfloat16).to(DEV)
    for c in _counts(cap):
        labels = torch.full((cap,), -1, dtype=torch.int64)
        where = torch.randperm(cap, generator=g)[:c]
        labels[where] = torch.randint(0, 30522, (c,), generator=g)
        if c > 2:
            labels[where[0]], labels[where[1]] = 40000, -7      # outside [0, V): still selected
        labels = labels.to(DEV)
        sel = F.select_rows(labels, -1)
        idx = torch.nonzero(labels != -1).reshape(-1)
        assert int(sel.count) == c == idx.numel()
        assert sel.scale.item() == torch.tensor(1.0 / max(c, 1), dtype=torch.float32).item()
        assert torch.equal(sel.pos[:c].long(), idx) and bool((sel.pos[c:] == -1).all())
        inv = torch.full((cap,), -1, dtype=torch.int64, device=DEV)
        inv[idx] = torch.arange(c, device=DEV)
        assert torch.equal(sel.inv.long(), inv)
        assert torch.equal(sel.labels[:c], labels[idx]) and bool((sel.labels[c:] == -1).all())
        rows = F.gather_rows(x, sel.pos)
        assert torch.equal(rows[:c], x.index_select(0, idx)) and not rows[c:].any()
        dg = torch.randn(cap, H, generator=g).to(torch.bfloat16).to(DEV)
        dx = F.gather_rows(dg, sel.inv)
        ref = torch.zeros_like(x).index_copy_(0, idx, dg[:c])
        assert torch.equal(dx, ref)


@pytest.mark.parametrize("cap", [1000, 4160])
def test_bounded_gemm_forward_and_dgrad(cap):
    from mmf_b200 import functional as F, lib
    g = torch.Generator().manual_seed(cap)
    V, H = 1024, 768
    w = (torch.randn(V, H, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    bias = (torch.randn(V, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    h = torch.randn(cap, H, generator=g).to(torch.bfloat16).to(DEV)
    z = (torch.randn(cap, V, generator=g) * 0.01).to(torch.bfloat16).to(DEV)
    sentinel = -77.0
    for c in _counts(cap):
        r = _rounded(c, cap)
        out = torch.full((cap, V), sentinel, dtype=torch.bfloat16, device=DEV)
        F.gemm(h, w, epi=lib.EPI_BIAS, bias=bias, out=out, m_bound=_bound(c))
        if c:
            assert torch.equal(out[:c], F.gemm(h[:c], w, epi=lib.EPI_BIAS, bias=bias))
        assert bool((out[r:] == sentinel).all())
        dh = torch.full((cap, H), sentinel, dtype=torch.bfloat16, device=DEV)
        F.gemm(z, w, b_mn=True, epi=lib.EPI_BIAS, out=dh, m_bound=_bound(c))
        if c:
            assert torch.equal(dh[:c], F.gemm(z[:c], w, b_mn=True, epi=lib.EPI_BIAS))
        assert bool((dh[r:] == sentinel).all())


@pytest.mark.parametrize("cap", [1000, 4160])
def test_bounded_wgrad_atomic_and_ordered(cap):
    from mmf_b200 import functional as F, lib
    from mmf_b200.engine import best_splits
    g = torch.Generator().manual_seed(cap + 1)
    V, H = 1024, 768
    splits = best_splits(V, H, cap)
    for c in _counts(cap):
        kb = min(cap, -(-c // 64) * 64)
        z = (torch.randn(cap, V, generator=g) * 0.01).to(torch.bfloat16)
        h = torch.randn(cap, H, generator=g).to(torch.bfloat16)
        z[c:kb], h[c:kb] = 0, 0                      # the invariant: rows between the count and its k-block edge are zero
        z[kb:], h[kb:] = float("nan"), float("nan")  # never read
        z, h = z.to(DEV), h.to(DEV)
        init = (torch.randn(V, H, generator=g) * 0.5).to(DEV)
        ref = init.double() + z[:c].double().t() @ h[:c].double()
        absab = z[:c].double().abs().t() @ h[:c].double().abs()
        out = init.clone()
        F.gemm(z, h, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=out, splits=splits, k_bound=_bound(c))
        assert bool(((out.double() - ref).abs() <= KC.gemm_bound(ref, absab, extra=init.double().abs(),
                                                                  bf16_out=False)).all()), c
        if c == 0:
            assert torch.equal(out, init)
        with _deterministic():
            o1, o2 = init.clone(), init.clone()
            F.gemm(z, h, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=o1, splits=splits, k_bound=_bound(c))
            F.gemm(z, h, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=o2, splits=splits, k_bound=_bound(c))
            assert torch.equal(o1, o2)
            if c:
                o3 = init.clone()
                F.gemm(z[:c], h[:c], a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=o3, splits=splits)
                assert torch.equal(o1, o3), c
        assert bool(((o1.double() - ref).abs() <= KC.gemm_bound(ref, absab, extra=init.double().abs(),
                                                                 bf16_out=False)).all()), c


@pytest.mark.parametrize("M", [1000, 4160])
def test_m_bounded_split_k_leaves_rows_past_the_bound_alone(M):
    """an M bound on the split-K weight-gradient GEMM, atomic and ordered: rows below the rounded bound are the unbounded
    call's (bit for bit in the ordered mode), and C past it keeps its sentinel - the ordered reduce neither reads nor
    writes those rows, whatever the workspace holds"""
    from mmf_b200 import functional as F, lib
    g = torch.Generator().manual_seed(M + 3)
    K, N, splits = 2048, 768, 4
    a = (torch.randn(K, M, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    b = torch.randn(K, N, generator=g).to(torch.bfloat16).to(DEV)
    init = (torch.randn(M, N, generator=g) * 0.5).to(DEV)
    ref = init.double() + a.double().t() @ b.double()
    absab = a.double().abs().t() @ b.double().abs()
    sentinel = -7.0
    for c in _counts(M):
        r = _rounded(c, M)
        base = init.clone()
        base[r:] = sentinel
        out = base.clone()
        F.gemm(a, b, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=out, splits=splits, m_bound=_bound(c))
        assert bool((out[r:] == sentinel).all()), c
        assert bool(((out[:r].double() - ref[:r]).abs() <= KC.gemm_bound(ref[:r], absab[:r], extra=init[:r].double().abs(),
                                                                           bf16_out=False)).all()), c
        with _deterministic():
            full = init.clone()
            F.gemm(a, b, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=full, splits=splits)
            out = base.clone()
            # leave NaN in the allocator's free block of the workspace's size, where that workspace comes from
            junk = torch.full((splits * M * N,), float("nan"), device=DEV)
            del junk
            F.gemm(a, b, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=out, splits=splits, m_bound=_bound(c))
        assert bool((out[r:] == sentinel).all()), c
        assert torch.equal(out[:r], full[:r]), c


@pytest.mark.parametrize("cap", [300, 2500])
def test_bounded_ce_rows_and_colsum(cap):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(cap + 2)
    V = 30528
    for c in _counts(cap):
        r = _rounded(c, cap)
        z0 = (torch.randn(cap, V, generator=g) * 2).to(torch.bfloat16).to(DEV)
        labels = torch.full((cap,), -1, dtype=torch.int64)
        labels[:c] = torch.randint(0, 30522, (c,), generator=g)
        labels = labels.to(DEV)
        scale = torch.tensor([1.0 / max(c, 1)], dtype=torch.float32, device=DEV)
        z, rl = z0.clone(), torch.full((cap,), -5.0, device=DEV)
        F.ce_rows_bounded(z, labels, -1, scale, _bound(c), loss_sum=torch.zeros((), device=DEV), row_loss=rl)
        if c:
            zr, rlr = z0[:c].clone(), torch.zeros(c, device=DEV)
            F.ce_rows(zr, labels[:c], -1, 1.0 / max(c, 1), torch.zeros((), device=DEV), row_loss=rlr)
            assert torch.equal(z[:c], zr) and torch.equal(rl[:c], rlr)
        assert not z[c:r].any() and bool((rl[c:r] == 0).all())
        assert torch.equal(z[r:], z0[r:]) and bool((rl[r:] == -5.0).all())
        x = KC.exact_ints(cap, 768, gen=g).to(DEV)
        out0 = KC.exact_ints(768, gen=g).float().to(DEV)
        exact = out0.double() + x[:c].double().sum(0)
        for det in (False, True):
            with _deterministic() if det else contextlib.nullcontext():
                out = out0.clone()
                F.colsum_bounded(x, out, _bound(c))
                assert torch.equal(out.double(), exact), (c, det)
                if det and c:
                    ref = out0.clone()
                    F.colsum(x[:c], ref)
                    assert torch.equal(out, ref)


@pytest.mark.parametrize("cap,c", [(5000, 2100), (5000, 4999), (700, 1), (700, 0), (4097, 4097), (4096, 2048),
                                   (2049, 2049), (300, 129)])
def test_static_linear_cross_entropy_matches_todays(cap, c):
    from mmf_b200 import ops
    g = torch.Generator().manual_seed(cap + c)
    V, H = 30522, 768
    w = (torch.randn(V, H, generator=g) * 0.05).to(DEV).requires_grad_(True)
    b = (torch.randn(V, generator=g) * 0.1).to(DEV).requires_grad_(True)
    hf = torch.zeros(cap, H)
    hf[:c] = torch.randn(c, H, generator=g)
    labels = torch.full((cap,), -1, dtype=torch.int64)
    labels[:c] = torch.randint(0, V, (c,), generator=g)
    h, labels = hf.to(DEV).to(torch.bfloat16).requires_grad_(True), labels.to(DEV)
    with _deterministic():
        loss = ops.linear_cross_entropy(h, w, b, labels, count=_bound(c),
                                        scale=torch.tensor([1.0 / max(c, 1)], dtype=torch.float32, device=DEV))
        loss.backward()
        if not c:
            assert loss.item() == 0.0 and not h.grad.any() and not w.grad.any() and not b.grad.any()
            return
        h2 = h.detach()[:c].clone().requires_grad_(True)
        w2 = w.detach().clone().requires_grad_(True)
        ref = ops.linear_cross_entropy(h2, w2, b.detach(), labels[:c])
        ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    assert torch.equal(h.grad[:c], h2.grad) and not h.grad[c:].any()
    # dW and db element by element against fp64 of the kernels' own operands: the bf16 h, and the bf16 d(logits) that the
    # vocabulary GEMM over the bf16-rounded, padded weight and bias followed by ce_rows write for the labelled rows
    from mmf_b200 import lib
    from mmf_b200 import functional as F
    wb = torch.nn.functional.pad(w.detach().to(torch.bfloat16), (0, 0, 0, 6))
    bb = torch.cat([b.detach().to(torch.bfloat16), torch.full((6,), -30000.0, dtype=torch.bfloat16, device=DEV)])
    dz = F.gemm(h[:c].detach(), wb, epi=lib.EPI_BIAS, bias=bb)
    F.ce_rows(dz, labels[:c], -1, 1.0 / c, torch.zeros((), device=DEV))
    dz64, h64 = dz[:, :V].double(), h[:c].detach().double()
    dw64, dw_abs = dz64.t() @ h64, dz64.abs().t() @ h64.abs()
    # A row of dW is dominated by one term (-h_r / c of the row labelled with that token) followed by many tiny softmax
    # terms, which is not the sign-random regime of KC.U_ACC: the accumulator's error then grows with the number of k16
    # steps (kernel_check's docstring).  Worst case: one fp32 ulp (2^-23, truncation included) of sum |a||b| per k16 step,
    # plus the split and chunk additions.  Today's path (w2's gradient) is held to the same bound.
    steps = -(-c // 16) + 16
    ratio = lambda got: ((got.double() - dw64).abs() / (dw_abs * 2 * KC.U_F32).clamp_min(1e-300)).max().item()
    r_static, r_today = ratio(w.grad), ratio(w2.grad)
    print("dW error / (2^-23 sum|a||b|): static %.1f, today %.1f, worst case %d" % (r_static, r_today, steps))
    assert r_static <= steps and r_today <= steps, (r_static, r_today, steps)
    # db: fp32 sums of c bf16 terms, each partial sum rounded once per add
    db64, db_abs = dz64.sum(0), dz64.abs().sum(0)
    assert bool(((b.grad.double() - db64).abs() <= KC.SAFETY * c * KC.U_F32 * db_abs).all())


# ---------------------------------------------------------------------------------------------------------------------
# registered models
# ---------------------------------------------------------------------------------------------------------------------
def _case(name):
    import importlib
    import mmf_b200.mmft  # noqa: F401
    import mmf_b200.models as MD
    C = importlib.import_module("test_%s_model_cpu" % name)
    golden = torch.load(os.path.join(C.GOLD, "%s_model.pt" % name), weights_only=False)
    case = {"lxmert": "pretraining_masked_vqa2", "vinvl": "pretraining", "vilt": "pretraining"}[name]
    model = C._build(MD, golden, case).cuda().train()
    sl = C._sample_list(golden, case, device=DEV)
    if name == "lxmert":
        sl["image_info_0"]["cls_prob"] = torch.as_tensor(sl["image_info_0"]["cls_prob"]).to(DEV)
    batch = {k: v for k, v in sl.items() if torch.is_tensor(v) or isinstance(v, dict)}
    meta = {k: v for k, v in sl.items() if k not in batch}
    return model, batch, meta


def _label_sets(batch):
    lm = batch["lm_label_ids"]
    every = batch["input_ids"].clone()
    return [lm.clone(), torch.full_like(lm, -1), every.reshape(lm.shape) if every.shape == lm.shape else lm.clone()]


@pytest.mark.parametrize("name", ["lxmert", "vinvl", "vilt"])
def test_graphed_static_rows_step_is_the_eager_step_bit_for_bit(name):
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.sample import SampleList
    model, batch, meta = _case(name)

    def loss_fn_of(m):
        def run(b):
            out = m(SampleList(dict(b, **meta)))
            return sum(v.sum() for v in out["losses"].values())
        return run

    def grads(m):
        return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}

    sets = _label_sets(batch)
    assert int((sets[1] != -1).sum()) == 0 and int((sets[2] != -1).sum()) == sets[2].numel()
    with _deterministic():
        twin, today = copy.deepcopy(model), copy.deepcopy(model)
        # today's eager step against the eager static-rows step, at the golden parity bars
        today.zero_grad(set_to_none=True)
        ref_today = loss_fn_of(today)(batch)
        ref_today.backward()
        g_today = grads(today)
        twin.zero_grad(set_to_none=True)
        with static_rows():
            s = loss_fn_of(twin)(batch)
        s.backward()
        g_static = grads(twin)
        assert abs(s.item() - ref_today.item()) <= 1e-2 * abs(ref_today.item()) + 1e-6
        for n, gr in g_today.items():
            err = ((g_static[n].double() - gr.double()).norm() / gr.double().norm().clamp_min(1e-12)).item()
            assert err <= 3e-2 or gr.abs().max() < 1e-8, (n, err)
        step = GraphedStep(model, loss_fn_of(model), batch, static_rows=True)
        for labels in sets:
            b = dict(batch, lm_label_ids=labels)
            twin.zero_grad(set_to_none=True)
            torch.cuda.set_sync_debug_mode("error")
            try:
                with static_rows():
                    ref = loss_fn_of(twin)(b)
                ref.backward()
                loss = step(b)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            assert torch.equal(loss.detach(), ref.detach()), (name, loss.item(), ref.item())
            got, want = grads(model), grads(twin)
            assert len(want) > 20
            for n, gr in want.items():
                assert torch.equal(got[n], gr), (name, n)
