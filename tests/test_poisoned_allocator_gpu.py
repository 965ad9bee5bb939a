"""Whole training steps after torch's caching allocator has been filled with 0, NaN and -3e38 (tests/guarded.py
poison_cache), and static-rows replays in a non-monotone order of label counts.

A buffer that host code allocates with torch.empty and reads before a kernel has written every element of it (rows
past a device count, a sample with keys but no queries, a slack column) holds zeros in a fresh process and passes every
other test.  Here each step runs once unpoisoned, to size the fill from its peak, and then once after each fill: loss,
outputs and every parameter gradient must be finite and the same bits after all three.  torch's own NaN fill of
uninitialised memory under use_deterministic_algorithms is switched off for these runs, so that torch.empty returns
what the allocator holds.

The replays go all -> N -> 0 -> N' -> all labelled rows (N' != N, not a multiple of 128): going from a larger count to a
smaller non-zero one leaves stale rows of the larger replay between the count and the 128-row tile edge, which the
bounded kernels must not let through."""
import contextlib
import copy
import os
import sys

import pytest
import torch

import guarded as G

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

pytestmark = pytest.mark.gpu

DEV = "cuda"
FILLS = (0.0, float("nan"), -3e38)


@contextlib.contextmanager
def _deterministic_without_fill():
    import torch.utils.deterministic as D
    prev, prev_fill = torch.are_deterministic_algorithms_enabled(), D.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    D.fill_uninitialized_memory = False
    try:
        yield
    finally:
        D.fill_uninitialized_memory = prev_fill
        torch.use_deterministic_algorithms(prev)


@pytest.fixture(autouse=True)
def _keep_global_draw_state():
    """the steps here reset the library's seed counter and advance the dropout epoch; the tests after this file draw
    their dropout masks from both, so they get them back as they were"""
    from mmf_b200 import functional as F, modules
    counter = modules._SEED_COUNTER[0]
    epoch = F.dropout_epoch(DEV)
    epoch_value = None if epoch is None else epoch.clone()
    rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    yield
    modules._SEED_COUNTER[0] = counter
    if epoch_value is not None:
        F.dropout_epoch(DEV).copy_(epoch_value)
    torch.set_rng_state(rng[0])
    torch.cuda.set_rng_state(rng[1])


def _bits(t):
    t = t.detach()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


# ---------------------------------------------------------------------------------------------------------------------
# models: (model, loss_fn(model) -> {name: tensor}) with the golden inputs where the suite has them
# ---------------------------------------------------------------------------------------------------------------------
def _golden_visual_bert(skip):
    import test_models_gpu as TM
    from mmf_b200 import models as MD
    from mmf_b200.patch import set_skip_padding
    g = torch.load(os.path.join(TM.GOLD, "models.pt"), weights_only=False)
    c = g["visual_bert_pretraining_default"]
    model = MD.build_model(MD.load_model_config("visual_bert", overrides=dict(c["config"])))
    model.load_state_dict({k: v for k, v in c["state_dict"].items() if k in model.state_dict()})
    model = model.to(DEV).train()
    if skip:
        assert set_skip_padding(model) >= 1
    sl = TM._sample_list(g, DEV)
    return model, lambda m: m(type(sl)(sl))["losses"]


@contextlib.contextmanager
def _count_calls(module, name):
    """counts the calls of module.name while the context is open"""
    orig, n = getattr(module, name), [0]

    def spy(*a, **k):
        n[0] += 1
        return orig(*a, **k)
    setattr(module, name, spy)
    try:
        yield n
    finally:
        setattr(module, name, orig)


def _golden_vilbert(mode):
    """mode "dense"; "packed": skip-padding with every sample holding tokens in both streams and some text padding, so
    the step runs the packed cross-attention (asserted); "one_sample_without_text": one sample's text is all padding while
    its regions stay, which plan_two_stream does not pack (a sample with keys but no queries on one side): the step falls
    back to the dense kernels (asserted), and the packed kernels' keys-without-queries rows are covered by
    test_poison_guard_gpu.py::test_varlen_cross_attention_poisoned instead"""
    import test_models_gpu as TM
    from mmf_b200 import models as MD
    from mmf_b200.patch import set_skip_padding
    g = torch.load(os.path.join(TM.GOLD, "models.pt"), weights_only=False)
    c = g["vilbert_pretraining"]
    model = MD.build_model(MD.load_model_config("vilbert", overrides=dict(c["config"])))
    model.load_state_dict({k: v for k, v in c["state_dict"].items() if k in model.state_dict()})
    from mmf_b200 import functional as F
    model = model.to(DEV).train()
    if mode != "dense":
        assert set_skip_padding(model, True, two_stream=True) >= 1
    v = g["vilbert_inputs"]
    sl = TM._sample_list(g, DEV)
    sl["image_labels"] = v["image_labels"].to(DEV)
    info = {"max_features": g["visual_bert_inputs"]["max_features"].to(DEV), "bbox": v["bbox"].to(DEV),
            "cls_prob": v["cls_prob"].numpy().copy()}
    if mode == "packed":
        sl["input_mask"][0, -2:] = 0              # text padding in sample 0; every sample keeps tokens in both streams
        assert bool((sl["input_mask"].sum(1) > 0).all()) and bool((info["max_features"] > 0).all())
    elif mode == "one_sample_without_text":
        sl["input_mask"][-1] = 0

    def run(m):
        s = type(sl)(sl)
        s["image_info_0"] = dict(info)
        with _count_calls(F, "attention_varlen_cross_fwd") as n:
            out = m(s)["losses"]
        if mode == "packed":
            assert n[0] > 0, "the packed two-stream plan was not taken"
        elif mode == "one_sample_without_text":
            assert n[0] == 0, "a one-sided sample is expected to fall back to the dense kernels"
        return out
    return model, run


def _golden_registered(name, static):
    import test_static_rows_gpu as SR
    from mmf_b200.graphs import static_rows
    from mmf_b200.sample import SampleList
    model, batch, meta = SR._case(name)

    def run(m):
        with static_rows() if static else contextlib.nullcontext():
            return m(SampleList(dict(batch, **meta)))["losses"]
    return model, run


def _mmbt():
    import test_graphed_forward_gpu as GF
    from mmf_b200 import models as MD
    model, sl = GF._mmbt(MD)
    model = model.to(DEV).train()
    return model, lambda m: m(type(sl)(sl))["losses"]


def _m4c_captioner():
    import test_m4c_model_cpu as C
    from mmf_b200 import models as MD
    golden = torch.load(os.path.join(C.GOLD, "m4c_model.pt"), weights_only=False)
    model = C.build(MD, golden, captioner=True, device=DEV).train()
    sl = C.sample_list(golden, device=DEV)
    return model, lambda m: m(type(sl)(sl))["losses"]


def _albef_vit():
    """the ALBEF ViT encoder in training mode with MLP dropout and stochastic depth (the configuration of
    test_albef_vit_gpu.py's training-step check)"""
    import test_albef_vit_gpu as AV
    torch.manual_seed(21)
    enc = AV._encoder(AV.TRAIN_CFG).train()
    g = torch.Generator().manual_seed(22)
    images = torch.randn(4, 3, 224, 224, generator=g).to(DEV)
    w = torch.randn(4, 197, AV.TRAIN_CFG["embed_dim"], generator=g).to(DEV)

    def run(m):
        x = images.clone().requires_grad_(True)
        out = m(x)
        return {"loss": (out.float() * w.reshape(out.shape)).sum(), "out": out}
    return enc, run


def _uniter(task):
    import test_deterministic_gpu  # noqa: F401  (puts tools/ on sys.path)
    import mmf_b200.mmft  # noqa: F401
    from bench_uniter import sample_list
    from mmf_b200 import models as MD
    torch.manual_seed(0)
    cfg = MD.load_model_config("uniter", overrides=dict(do_pretraining=True, tasks=task, mask_probability=0.15,
                                                        heads={task: {"type": task}}))
    model = MD.build_model(cfg).to(DEV).train()
    base = sample_list(8, DEV, torch.Generator().manual_seed(4))
    return model, lambda m: m(type(base)(base))["losses"]


def _m4c():
    import test_deterministic_gpu  # noqa: F401
    from bench_m4c import sample_list, ANS, OCR_MAX
    from mmf_b200 import models as MD
    from mmf_b200.registry import registry
    registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
    registry.register("textvqa_num_final_outputs", ANS + OCR_MAX)
    registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1}))
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).to(DEV).train()
    sl = sample_list(8, DEV, torch.Generator().manual_seed(182))
    return model, lambda m: m(sl)["losses"]


def _static(build):
    """the eager static-rows step of a model: packing planned on the device, layers bounded by the device count"""
    def make():
        from mmf_b200.graphs import static_rows
        model, run = build()

        def static_run(m):
            with static_rows():
                return run(m)
        return model, static_run
    return make


def _mmf_transformer(skip):
    import test_static_packing_gpu as SP
    model, batches, loss_of = SP._mmf_transformer()
    if not skip:
        from mmf_b200.patch import set_skip_padding
        set_skip_padding(model, False)
    return model, lambda m: {"loss": loss_of(m)(batches[2])}


MODELS = {
    "visual_bert": lambda: _golden_visual_bert(False),
    "visual_bert_skip_padding": lambda: _golden_visual_bert(True),
    "vilbert": lambda: _golden_vilbert("dense"),
    "vilbert_packed": lambda: _golden_vilbert("packed"),
    "vilbert_one_sample_without_text": lambda: _golden_vilbert("one_sample_without_text"),
    "lxmert": lambda: _golden_registered("lxmert", False),
    "lxmert_static_rows": lambda: _golden_registered("lxmert", True),
    "vinvl": lambda: _golden_registered("vinvl", False),
    "vinvl_static_rows": lambda: _golden_registered("vinvl", True),
    "vilt": lambda: _golden_registered("vilt", False),
    "vilt_static_rows": lambda: _golden_registered("vilt", True),
    "uniter_mlm": lambda: _uniter("mlm"),
    "uniter_wra": lambda: _uniter("wra"),
    "m4c": _m4c,
    "m4c_captioner": _m4c_captioner,
    "mmbt": _mmbt,
    "albef_vit": _albef_vit,
    "mmf_transformer": lambda: _mmf_transformer(False),
    "mmf_transformer_skip_padding": lambda: _mmf_transformer(True),
    "visual_bert_skip_padding_static_rows": _static(lambda: _golden_visual_bert(True)),
    "mmf_transformer_skip_padding_static_rows": _static(lambda: _mmf_transformer(True)),
}


def _step(model, loss_fn, state):
    from mmf_b200 import modules
    with torch.no_grad():
        for k, p in model.named_parameters():
            p.copy_(state[k])
    model.zero_grad(set_to_none=True)
    torch.manual_seed(0)
    modules._SEED_COUNTER[0] = 0
    losses = loss_fn(model)
    sum(v.float().sum() for v in losses.values()).backward()
    torch.cuda.synchronize()
    out = {"loss/" + k: v.detach().float().clone() for k, v in losses.items()}
    out.update({"grad/" + k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None})
    return out


@pytest.mark.parametrize("name", list(MODELS))
def test_step_does_not_depend_on_what_the_allocator_held(name):
    model, loss_fn = MODELS[name]()
    state = {k: p.detach().clone() for k, p in model.named_parameters()}
    with _deterministic_without_fill():
        _step(model, loss_fn, state)                           # lazy state (engines, tables) outside the comparison
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        _step(model, loss_fn, state)
        peak = torch.cuda.max_memory_reserved()
        runs = []
        for value in FILLS:
            G.poison_cache(value, peak)
            runs.append(_step(model, loss_fn, state))
    first = runs[0]
    assert len([k for k in first if k.startswith("grad/")]) > 5, name
    for k, v in first.items():
        G.assert_finite(v, "%s %s" % (name, k))
    for value, r in zip(FILLS[1:], runs[1:]):
        assert r.keys() == first.keys(), (name, value)
        for k, v in first.items():
            assert torch.equal(_bits(r[k]), _bits(v)), (name, k, "differs after poison_cache(%r)" % value)


# ---------------------------------------------------------------------------------------------------------------------
# static-rows replays: all -> N -> 0 -> N' -> all
# ---------------------------------------------------------------------------------------------------------------------
def _label_order(batch):
    """labels with every row, the golden N, none, N' (a different count, not a multiple of 128) and every row again"""
    lm = batch["lm_label_ids"]
    every = batch["input_ids"].reshape(lm.shape).clone()
    n = int((lm != -1).sum())
    flat_every = every.reshape(-1)
    n2 = n // 2 + 1 if n > 2 else min(flat_every.numel() - 1, n + 3)
    assert n2 != n and n2 % 128 and 0 < n2 < flat_every.numel()
    other = torch.full_like(flat_every, -1)
    other[:n2] = flat_every[:n2]
    return [every, lm.clone(), torch.full_like(lm, -1), other.reshape(lm.shape), every.clone()]


@pytest.mark.parametrize("name", ["lxmert", "vinvl", "vilt"])
def test_graphed_static_rows_step_in_non_monotone_label_order(name):
    import test_static_rows_gpu as SR
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.sample import SampleList
    model, batch, meta = SR._case(name)

    def loss_fn_of(m):
        def run(b):
            out = m(SampleList(dict(b, **meta)))
            return sum(v.sum() for v in out["losses"].values())
        return run

    def grads(m):
        return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}

    with SR._deterministic():
        twin = copy.deepcopy(model)
        step = GraphedStep(model, loss_fn_of(model), batch, static_rows=True)
        for i, labels in enumerate(_label_order(batch)):
            b = dict(batch, lm_label_ids=labels)
            twin.zero_grad(set_to_none=True)
            with static_rows():
                ref = loss_fn_of(twin)(b)
            ref.backward()
            loss = step(b)
            torch.cuda.synchronize()
            assert torch.equal(loss.detach(), ref.detach()), (name, i, loss.item(), ref.item())
            got, want = grads(model), grads(twin)
            assert len(want) > 20
            for n, gr in want.items():
                assert torch.equal(got[n], gr), (name, i, n)


@pytest.mark.parametrize("name", ["lxmert", "vinvl", "vilt"])
def test_graphed_static_rows_forward_in_non_monotone_label_order(name):
    import test_graphed_forward_gpu as GF
    import test_static_rows_gpu as SR
    from mmf_b200.graphs import GraphedForward, static_rows
    from mmf_b200.sample import SampleList
    model, batch, meta = SR._case(name)
    model = model.eval()
    full = dict(batch, **meta)
    with SR._deterministic():
        fwd = GraphedForward(model, SampleList(full), static_rows=True)
        for i, labels in enumerate(_label_order(batch)):
            b = SampleList(dict(full, lm_label_ids=labels))
            got = GF._snapshot(fwd(b))
            with torch.no_grad(), static_rows():
                want = model(GF._fresh(b))
            torch.cuda.synchronize()
            GF._assert_same(got, want, "%s/%d" % (name, i))
