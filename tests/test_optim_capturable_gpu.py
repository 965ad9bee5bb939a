"""The capturable optimizer step on the H100: mmfb_adamw_segments against mmfb_adamw bit for bit, the device step size and
bias corrections against the host's, B200AdamW(capturable=True) against today's step, and GraphedStep(optimizer=...)
replays against eager capturable steps bit for bit (dense VisualBERT, LXMERT pretraining and skip-padding VisualBERT under
static_rows, m4c)."""
import contextlib
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAN, INF = float("nan"), float("inf")


@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _hp_table(mode, step, lr=1e-3, wd=0.01, betas=(0.9, 0.98), eps=1e-6, correct_bias=True):
    """one slot at step `step` (after the launch) through the real mmfb_adamw_hparams"""
    from mmf_b200 import functional as F, lib
    groups = torch.tensor([[lr, wd, betas[0], betas[1], eps]], dtype=torch.float64, device=DEV)
    slots = F.adamw_slot_table([(0, lib.MMFB_ADAMW_SLOT_CORRECT_BIAS if correct_bias else 0)], DEV)
    steps = torch.tensor([step - 1], dtype=torch.int64, device=DEV)
    hp = torch.empty(1, 8, dtype=torch.float32, device=DEV)
    F.adamw_hparams(groups, slots, steps, hp, mode)
    assert int(steps) == step
    return hp


def _view(n, shift, g, scale=1.0):
    base = torch.empty(n + 16, device=DEV)
    off = (-(base.data_ptr() >> 2)) % 4 + shift
    v = base[off:off + n]
    v.copy_(torch.randn(n, generator=g).to(DEV) * scale)
    return v


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("clip", [False, True])
def test_segments_equal_the_flat_kernel_bit_for_bit(mode, clip):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(3 + mode)
    hp = _hp_table(mode, 7)
    coef = torch.tensor([0.37], device=DEV) if clip else None
    segs, cases = [], []
    for n in (1, 7, 8, 9, 3129, 20000):
        for shifts in ((0, 0, 0, 0), (1, 1, 1, 1), (2, 2, 2, 2), (3, 3, 3, 3), (1, 0, 2, 3)):
            p, gr = _view(n, shifts[0], g), _view(n, shifts[1], g, 1e-2)
            m, v = _view(n, shifts[2], g, 1e-3), _view(n, shifts[3], g).abs_().mul_(1e-5)
            if n >= 9:
                gr[3], gr[n - 1] = INF, NAN
            cases.append((p.clone(), gr.clone(), m.clone(), v.clone()))
            segs.append((p, gr, m, v, 0))
    table = F.adamw_segment_table(segs)
    assert {r[7] for r in table.rows} == {-1, 0, 1, 2, 3}
    F.adamw_segments(table, hp, mode=mode, grad_scale=0.5, grad_scale_dev=coef)
    for (p, gr, m, v, _), ref in zip(segs, cases):
        n = p.numel()
        n8 = (n + 7) // 8 * 8
        flat = [torch.zeros(n8, device=DEV) for _ in range(4)]
        for f, r in zip(flat, ref):
            f[:n] = r
        F.adamw(*flat, None, beta1=0.0, beta2=0.0, eps=0.0, mode=mode, grad_scale=0.5, grad_scale_dev=coef, hp_dev=hp)
        for got, want in ((p, flat[0]), (m, flat[2]), (v, flat[3])):
            assert torch.equal(_bits(got), _bits(want[:n])), (n, mode, clip)
        assert torch.equal(_bits(gr), _bits(ref[1]))


def test_the_device_table_equals_the_launch_fields_bit_for_bit():
    from mmf_b200 import functional as F
    from mmf_b200.optim import B200AdamW
    g = torch.Generator().manual_seed(5)
    for mode, arith in ((0, "transformers"), (1, "torch")):
        hp = _hp_table(mode, 3)
        opt = B200AdamW([torch.nn.Parameter(torch.zeros(1))], lr=1e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01,
                        arithmetic=arith)
        host = opt._group_hp(opt.param_groups[0], 3)
        bufs = [torch.randn(4096, generator=g).to(DEV) for _ in range(4)]
        bufs[3].abs_()
        a = [b.clone() for b in bufs]
        F.adamw(*a, [host], beta1=0.9, beta2=0.98, eps=1e-6, mode=mode)
        F.adamw(*bufs, None, beta1=0.0, beta2=0.0, eps=0.0, mode=mode, hp_dev=hp)
        for x, y in zip(a, bufs):
            assert torch.equal(_bits(x), _bits(y)), mode


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.9, 0.98)])
def test_device_step_size_and_bias_correction_against_the_host(betas):
    """t = 1 ... 100 000 in one launch: the fp32 values the device computes against _group_hp rounded to fp32"""
    from mmf_b200 import functional as F, lib
    from mmf_b200.optim import B200AdamW
    T = 100_000
    report = []
    for mode, arith in ((0, "transformers"), (1, "torch")):
        opt = B200AdamW([torch.nn.Parameter(torch.zeros(1))], lr=1e-4, betas=betas, arithmetic=arith)
        grp = opt.param_groups[0]
        groups = torch.tensor([[1e-4, 0.0, betas[0], betas[1], 1e-6]], dtype=torch.float64, device=DEV)
        slots = F.adamw_slot_table([(0, lib.MMFB_ADAMW_SLOT_CORRECT_BIAS)] * T, DEV)
        steps = torch.arange(T, dtype=torch.int64, device=DEV)
        hp = torch.empty(T, 8, dtype=torch.float32, device=DEV)
        F.adamw_hparams(groups, slots, steps, hp, mode)
        assert torch.equal(steps.cpu(), torch.arange(1, T + 1))
        host = [opt._group_hp(grp, t) for t in range(1, T + 1)]
        for col, key in ((2, "step_size"), (3, "bc2_sqrt")):
            want = torch.tensor([h[key] for h in host], dtype=torch.float64).float()
            got = hp[:, col].cpu()
            ulp = (_bits(got).long() - _bits(want).long()).abs()
            report.append((arith, key, int((ulp != 0).sum()), int(ulp.max())))
            assert int(ulp.max()) <= 1, report[-1]
    print("device vs host hyper-parameters (mode, value, differing t, max ulp) at betas %s: %s" % (betas, report))


# ---------------------------------------------------------------------------------------------------------------------
class _Trunk(torch.nn.Module):
    """VisualBERT trunk (its fusion layers live in a parameter pack) plus a head outside any pack"""

    def __init__(self):
        super().__init__()
        import bench
        from mmf_b200.visual_bert import B200VisualBERT
        self.trunk = B200VisualBERT(bench.bert_config(768, 12, 3072, 2, 0.0, visual_embedding_dim=2048))
        self.head = torch.nn.Linear(768, 5)

    def forward(self, batch):
        return self.head(self.trunk(batch)["sequence_output"])


def _trunk_case():
    import bench
    torch.manual_seed(0)
    model = _Trunk().to(DEV).train()
    wl = bench.WORKLOADS["visual_bert"]()
    batches = [bench.to_device(wl.host_batch(4, s), DEV) for s in range(6)]

    def loss_of(m):
        def run(b):
            out = m(b)
            return (out * torch.linspace(-1, 1, out.numel(), device=DEV).view(out.shape)).sum() * 10.0
        return run
    groups = lambda m: [{"params": list(m.trunk.parameters())}, {"params": list(m.head.parameters()), "lr": 3e-3}]
    return model, batches, loss_of, groups, dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01,
                                                arithmetic="torch")


def _m4c_batch(seed, B=8):
    from mmf_b200.sample import SampleList
    T, R, O, D = 20, 100, 50, 12
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)
    sl = dict(text=torch.randint(1, 30522, (B, T), generator=g), text_len=torch.randint(1, T + 1, (B,), generator=g),
              image_feature_0=torch.randn(B, R, 2048, generator=g).relu(), obj_bbox_coordinates=r(B, R, 4),
              image_info_0={"max_features": torch.randint(10, R + 1, (B,), generator=g)},
              context_feature_0=torch.randn(B, O, 300, generator=g), context_feature_1=r(B, O, 604),
              image_feature_1=torch.randn(B, O, 2048, generator=g).relu(), order_vectors=torch.zeros(B, O, 50),
              ocr_bbox_coordinates=r(B, O, 4), context_info_0={"max_features": torch.randint(0, O + 1, (B,), generator=g)},
              train_prev_inds=torch.randint(0, 5050, (B, D), generator=g), targets=(r(B, D, 5050) < 0.01).float(),
              train_loss_mask=(r(B, D) < 0.7).float())
    to = lambda x: {k: to(v) for k, v in x.items()} if isinstance(x, dict) else x.to(DEV)
    return to(sl)


def _m4c_case():
    import mmf_b200.models as MD
    from mmf_b200.models import ConfigNode
    from mmf_b200.registry import registry
    from mmf_b200.sample import SampleList
    import test_m4c_model_cpu as C
    golden = torch.load(os.path.join(C.GOLD, "m4c_model.pt"), weights_only=False)
    C.register(golden)
    registry.register(golden["dataset"] + "_num_final_outputs", 5050)
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).to(DEV).train()
    batches = [_m4c_batch(s) for s in range(6)]
    cfg = ConfigNode({"optimizer": {"type": "Adam", "params": {"lr": 1e-4, "eps": 1e-8, "weight_decay": 0}}})

    def loss_of(m):
        def run(b):
            return C.loss_of(m(SampleList(dict(b, dataset_name="textvqa", dataset_type="train")))).sum()
        return run
    return model, batches, loss_of, (lambda m: m.get_optimizer_parameters(cfg)), dict(lr=1e-4, eps=1e-8,
                                                                                        weight_decay=0.0,
                                                                                        arithmetic="torch")


def _loose_close(p, q, what):
    """a loose parameter stepped by the kernel against one stepped by torch ops: tests/test_grad_norm_gpu.py's bars, 2e-6
    of the largest value, or rtol 1e-6 / atol 1e-7 for parameters that start at zero (LayerNorm biases), whose values are
    then of the size of the update: there the kernel's fp32 `1 - beta2` (0.999f gives 0.00099998713) against torch's
    fp64 one rounded (0.001f) shows as about 6e-6 of the update"""
    p, q = p.detach(), q.detach()
    err = float((p - q).abs().max() / q.abs().max().clamp_min(1e-6))
    assert err < 2e-6 or torch.allclose(p, q, rtol=1e-6, atol=1e-7), what + (err,)


def _warmup_linear(opt):
    return torch.optim.lr_scheduler.LambdaLR(opt, lambda s: min(1.0, (s + 1) / 3))


def _packed_ids(model):
    from mmf_b200 import engine as E
    mine = {id(p) for p in model.parameters()}
    return {id(p) for pack in list(E.ParamPack._live or ()) for p in pack.params if id(p) in mine}


@pytest.mark.parametrize("case", ["visual_bert", "m4c"])
def test_capturable_eager_steps_match_todays_steps(case):
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp = {"visual_bert": _trunk_case, "m4c": _m4c_case}[case]()
    with _deterministic():
        ref = copy.deepcopy(model)
        opt, opt_r = B200AdamW(groups(model), capturable=True, **hp), B200AdamW(groups(ref), **hp)
        sch, sch_r = _warmup_linear(opt), _warmup_linear(opt_r)
        for step in range(5):
            for m in (model, ref):
                m.zero_grad()
                loss_of(m)(batches[step]).backward()
            # one set of gradients for both optimizers (copied in place, so the packed ones stay in the flat buffers): the
            # loose parameters differ in their last bits, and so would every later gradient computed from them
            for p, q in zip(model.parameters(), ref.parameters()):
                if p.grad is not None:
                    q.grad.copy_(p.grad)
            packed = _packed_ids(model)                # the engine builds its packs in the first forward
            assert packed and len(packed) < len(list(model.parameters()))
            torch.cuda.synchronize()
            if step >= 1:
                torch.cuda.set_sync_debug_mode("error")
            try:
                opt.clip_grad_norm(0.25)
                opt.step()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            opt_r.clip_grad_norm(0.25)
            opt_r.step()
            sch.step()
            sch_r.step()
            assert opt._cap.loose and (case == "m4c" or opt._cap.packs)
            for (n, p), q in zip(model.named_parameters(), ref.parameters()):
                if id(p) in packed:
                    assert torch.equal(_bits(p.detach()), _bits(q.detach())), (case, step, n)
                else:
                    _loose_close(p, q, (case, step, n))
        sd = opt.state_dict()
        assert {st["step"] for st in sd["state"].values()} == {5}


# ---------------------------------------------------------------------------------------------------------------------
def _visual_bert_dense():
    model, batches, loss_of, groups, hp = _trunk_case()
    return model, batches[:4], loss_of, groups, hp, False


def _visual_bert_skip_padding():
    import test_static_packing_gpu as SP
    model, batches, loss_of = SP._visual_bert()
    batches = batches + [batches[0]]
    return model, batches, loss_of, (lambda m: list(m.parameters())), dict(lr=1e-4, weight_decay=0.01,
                                                                           arithmetic="torch"), True


def _lxmert():
    import test_static_rows_gpu as SR
    from mmf_b200.sample import SampleList
    model, batch, meta = SR._case("lxmert")
    sets = SR._label_sets(batch)
    batches = [dict(batch, lm_label_ids=s) for s in sets] + [batch]

    def loss_of(m):
        def run(b):
            out = m(SampleList(dict(b, **meta)))
            return sum(v.sum() for v in out["losses"].values())
        return run
    return model, batches, loss_of, (lambda m: list(m.parameters())), dict(lr=1e-4, weight_decay=0.01,
                                                                           arithmetic="transformers"), True


def _m4c_graph():
    model, batches, loss_of, groups, hp = _m4c_case()
    return model, batches[:4], loss_of, groups, hp, False


def _state(model, opt):
    out = {}
    for n, p in model.named_parameters():
        st = opt.state.get(p, {})
        out[n] = (p.detach().clone(), *(st[k].clone() if k in st else None for k in ("exp_avg", "exp_avg_sq")),
                  int(st["step"]) if "step" in st else 0)
    return out


@pytest.mark.parametrize("name", ["visual_bert", "lxmert", "visual_bert_skip_padding", "m4c"])
def test_graphed_whole_step_is_the_eager_capturable_step_bit_for_bit(name):
    from mmf_b200 import functional as F, modules
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.optim import B200AdamW
    model, batches, loss_of, groups, hp, static = {"visual_bert": _visual_bert_dense, "lxmert": _lxmert,
                                                   "visual_bert_skip_padding": _visual_bert_skip_padding,
                                                   "m4c": _m4c_graph}[name]()
    assert len(batches) >= 4
    for n, m in model.named_modules():            # torch's own dropout draws differ between replay and eager step
        if isinstance(m, torch.nn.Dropout) and "layer" not in n:
            m.p = 0.0
    ctx = static_rows if static else contextlib.nullcontext
    with _deterministic():
        twin = copy.deepcopy(model)
        with ctx():
            loss_of(twin)(batches[0]).backward()     # the twin's lazy engine state
        twin.zero_grad(set_to_none=True)
        opt, opt_t = B200AdamW(groups(model), capturable=True, **hp), B200AdamW(groups(twin), capturable=True, **hp)
        sch, sch_t = _warmup_linear(opt), _warmup_linear(opt_t)
        before = _state(model, opt)
        c0 = modules._SEED_COUNTER[0]
        step = GraphedStep(model, loss_of(model), batches[0], warmup=3, static_rows=static, optimizer=opt,
                           max_grad_norm=1.0)
        c1 = modules._SEED_COUNTER[0]
        per_step = (c1 - c0) // 4
        torch.cuda.synchronize()
        after = _state(model, opt)
        for n, (p, m, v, s) in before.items():     # capturing does not step
            q, m2, v2, s2 = after[n]
            assert torch.equal(_bits(p), _bits(q)) and s == s2 == 0, (name, n)
            for x in (m2, v2):
                assert x is None or not x.any(), (name, n)
        for i, b in enumerate(batches):
            loss = step(b)
            twin.zero_grad(set_to_none=True)
            modules._SEED_COUNTER[0] = c1 - per_step
            with ctx():
                ref = loss_of(twin)(b)
            ref.backward()
            opt_t.clip_grad_norm(1.0)
            opt_t.step()
            sch.step()
            sch_t.step()
            torch.cuda.synchronize()
            assert torch.equal(loss.detach(), ref.detach()), (name, i, loss.item(), ref.item())
            got, want = _state(model, opt), _state(twin, opt_t)
            for (n, p), q in zip(model.named_parameters(), twin.parameters()):
                for x, y in zip(got[n][:3], want[n][:3]):
                    assert (x is None and y is None) or torch.equal(x, y), (name, i, n)
                assert got[n][3] == want[n][3] == i + 1 or p.grad is None, (name, i, n)
                assert (p.grad is None) == (q.grad is None) and (p.grad is None or torch.equal(p.grad, q.grad)), (name, n)
        assert opt.param_groups[0]["lr"] == hp["lr"]
        # a checkpoint taken after the replays continues in a plain B200AdamW like the graph
        plain = B200AdamW(groups(twin), **hp)
        plain.load_state_dict(copy.deepcopy(opt.state_dict()))
        twin.load_state_dict(model.state_dict())
        b = batches[1]
        step(b)
        twin.zero_grad(set_to_none=True)
        modules._SEED_COUNTER[0] = c1 - per_step
        with ctx():
            loss_of(twin)(b).backward()
        plain.clip_grad_norm(1.0)
        plain.step()
        torch.cuda.synchronize()
        packed = _packed_ids(model)
        for (n, p), q in zip(model.named_parameters(), twin.parameters()):
            if id(p) in packed:
                assert torch.equal(p.detach(), q.detach()), (name, n)
            else:
                _loose_close(p, q, (name, n))
