"""GraphedForward on the H100: the eval forward of every registered model below, captured once and replayed on three
other seeded batches, equals the eager model.eval() + no_grad forward on the same batch bit for bit (scores, losses and
every other output, torch.equal); the eager forwards run under torch.cuda.set_sync_debug_mode("error"), so none of them
reads a value on the host.  M4C at TextVQA shapes: the whole 12-step greedy decode is one graph whose scores and argmax
equal the eager decode.  static_rows=True: LXMERT and VinVL pretraining evals and a skip-padding VisualBERT trunk equal
the eager forward inside static_rows() bit for bit.

The forward kernels use no atomics (the split-K weight-gradient GEMMs are backward only), so exact equality is the bar
without torch.use_deterministic_algorithms - except for the masked-LM loss under static_rows(), whose cross-entropy adds
its row losses into the loss with atomics: the LXMERT and VinVL pretraining cases are captured and run eagerly under
torch.use_deterministic_algorithms(True), which sums them in a fixed order."""
import contextlib
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODELS = ["visual_bert", "vilbert", "mmbt", "lxmert", "mmf_transformer", "vinvl", "vilt", "m4c", "m4c_captioner"]


def _load(name):
    return torch.load(os.path.join(GOLD, name), weights_only=False)


def _on_device(info):
    """image_info_0 with its numpy cls_prob as a device tensor: a host array would be copied in every forward"""
    return {k: (torch.as_tensor(v).to(DEV) if k == "cls_prob" else v) for k, v in info.items()}


def _models_pt_case(MD, model_name, case, cls_prob=False):
    import test_models_gpu as G
    g = _load("models.pt")
    c = g[case]
    cfg = MD.load_model_config(model_name, overrides=dict(c["config"]))
    cfg.losses = [{"type": "cross_entropy"}]
    model = MD.build_model(cfg)
    model.load_state_dict({k: v for k, v in c["state_dict"].items() if k in model.state_dict()})
    sl = G._sample_list(g, DEV)
    if cls_prob:
        v = g["vilbert_inputs"]
        sl["image_labels"] = v["image_labels"].to(DEV)
        sl["image_info_0"] = _on_device({"max_features": g["visual_bert_inputs"]["max_features"].to(DEV),
                                         "bbox": v["bbox"].to(DEV), "cls_prob": v["cls_prob"]})
    return model, sl


def _mmbt(MD):
    from mmf_b200.sample import SampleList
    cfg = MD.load_model_config("mmbt", overrides={
        "training_head_type": "classification", "num_labels": 2, "direct_features_input": True, "modal_hidden_size": 40,
        "modal_encoder": {"type": "identity", "params": {"in_dim": 40}},
        "text_encoder": {"type": "transformer", "params": {
            "num_segments": 2, "bert_model_name": None, "hidden_size": 64, "num_hidden_layers": 1, "num_attention_heads": 1,
            "intermediate_size": 128, "vocab_size": 50, "max_position_embeddings": 64, "hidden_dropout_prob": 0.0,
            "attention_probs_dropout_prob": 0.0}},
        "losses": [{"type": "cross_entropy"}]})
    torch.manual_seed(5)
    model = MD.build_model(cfg)
    g = _load("mmbt.pt")
    sl = SampleList(input_ids=g["ids"].to(DEV), input_mask=g["mask"].to(DEV), segment_ids=g["seg"].to(DEV),
                    image_feature_0=g["feats"].to(DEV), targets=torch.tensor([1, 0], device=DEV), dataset_name="hm",
                    dataset_type="val")
    return model, sl


def _mmf_transformer(MD):
    import mmf_b200.mmft  # noqa: F401
    from mmf_b200.sample import SampleList
    from test_mmft_cpu import SMALL
    mods = [dict(type="text", key="text", embedding_dim=64, position_dim=128, segment_id=0),
            dict(type="image", key="image", embedding_dim=48, position_dim=8, segment_id=1, encoder=dict(type="identity"))]
    cfg = MD.load_model_config("mmf_transformer", overrides={
        "modalities": mods, "num_labels": 3, "transformer_config": SMALL,
        "heads": [{"type": "mlp", "hidden_size": 64, "num_labels": 3}], "losses": [{"type": "cross_entropy"}]})
    torch.manual_seed(3)
    model = MD.build_model(cfg)
    g = torch.Generator().manual_seed(10)
    B, T = 4, 10
    mask = (torch.arange(T)[None] < torch.tensor([10, 7, 3, 9])[:, None]).long()
    sl = SampleList(input_ids=torch.randint(1, 512, (B, T), generator=g), input_mask=mask,
                    image=torch.rand(B, 6, 48, generator=g), targets=torch.randint(0, 3, (B,), generator=g),
                    is_correct=torch.ones((), dtype=torch.long), dataset_name="golden", dataset_type="val")
    return model, sl.to(DEV)


def _golden_case(module, fixture, case):
    import importlib
    import mmf_b200.models as MD
    C = importlib.import_module(module)
    golden = _load(fixture)
    model = C._build(MD, golden, case)
    sl = C._sample_list(golden, case, device=DEV)
    if "image_info_0" in sl and "cls_prob" in sl["image_info_0"]:
        sl["image_info_0"] = _on_device(sl["image_info_0"])
    return model, sl


def _case(name):
    """(model on the GPU in eval mode, its golden-sized SampleList on the GPU)"""
    import mmf_b200.models as MD
    if name in ("m4c", "m4c_captioner"):
        import test_m4c_model_cpu as C
        golden = _load("m4c_model.pt")
        model, sl = C.build(MD, golden, captioner=name == "m4c_captioner"), C.sample_list(golden, DEV)
    elif name == "visual_bert":
        model, sl = _models_pt_case(MD, "visual_bert", "visual_bert_classification_vqa")
    elif name == "vilbert":
        model, sl = _models_pt_case(MD, "vilbert", "vilbert_classification", cls_prob=True)
    elif name == "mmbt":
        model, sl = _mmbt(MD)
    elif name == "mmf_transformer":
        model, sl = _mmf_transformer(MD)
    elif name == "lxmert":
        model, sl = _golden_case("test_lxmert_model_cpu", "lxmert_model.pt", "classification")
    elif name == "vinvl":
        model, sl = _golden_case("test_vinvl_model_cpu", "vinvl_model.pt", "classification")
    else:
        model, sl = _golden_case("test_vilt_model_cpu", "vilt_model.pt", "classification")
    return model.to(DEV).eval(), sl


def _variant(batch, seed):
    """another batch of the same shapes: the samples permuted (every tensor with the batch dimension alike) and the float
    features of rank >= 3 scaled element-wise by factors in [1, 1.25)"""
    from mmf_b200.graphs import _flatten, _map_keep
    B = next(t for t in _flatten(batch) if t.dim() >= 2).size(0)
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(B, generator=g).to(DEV)

    def one(t):
        if t.dim() >= 1 and t.size(0) == B:
            t = t.index_select(0, perm)
        if t.is_floating_point() and t.dim() >= 3:
            t = t * (1 + 0.25 * torch.rand(t.shape, generator=g)).to(t.device, t.dtype)
        return t
    return _map_keep(one, batch)


def _fresh(batch):
    from mmf_b200.graphs import _map_keep
    return _map_keep(lambda t: t, batch)


def _snapshot(out):
    from mmf_b200.graphs import _map_keep
    return _map_keep(lambda t: t.detach().clone(), out)


def _assert_same(got, want, where):
    if isinstance(want, dict):
        assert set(got) == set(want), (where, sorted(got), sorted(want))
        for k in want:
            _assert_same(got[k], want[k], "%s.%s" % (where, k))
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), where
        for i, (a, b) in enumerate(zip(got, want)):
            _assert_same(a, b, "%s[%d]" % (where, i))
    elif torch.is_tensor(want):
        assert got.dtype == want.dtype and got.shape == want.shape, where
        assert torch.equal(got, want), (where, (got.double() - want.double()).abs().max().item())
    else:
        assert got == want, where


@contextlib.contextmanager
def _no_host_reads():
    torch.cuda.set_sync_debug_mode("error")
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(0)


def _epoch():
    from mmf_b200 import functional as F
    ep = F.dropout_epoch(DEV)
    return None if ep is None else int(ep.item())


@pytest.mark.parametrize("name", MODELS)
def test_replay_is_the_eager_eval_forward_bit_for_bit(name):
    from mmf_b200.graphs import GraphedForward, static_rows
    model, batch = _case(name)
    # VinVL declares graph_capturable = False for its pretraining gather, whatever its heads: static_rows covers it, and
    # changes nothing in a classification forward
    rows = static_rows if name == "vinvl" else contextlib.nullcontext
    with torch.no_grad(), rows():
        first = _snapshot(model(_fresh(batch)))      # the lazy engine state, outside the sync check
    assert "scores" in first, sorted(first)
    epoch = _epoch()
    fwd = GraphedForward(model, batch, static_rows=name == "vinvl")
    for seed in (1, 2, 3):
        b = _variant(batch, seed)
        got = _snapshot(fwd(b))
        torch.cuda.synchronize()
        with torch.no_grad(), rows(), _no_host_reads():
            want = model(_fresh(b))
        torch.cuda.synchronize()
        assert not torch.equal(want["scores"], first["scores"]), (name, seed)    # a batch the capture did not see
        _assert_same(got, want, "%s/%d" % (name, seed))
    assert _epoch() == epoch


def test_m4c_textvqa_shape_decode_is_one_graph():
    """the default m4c configuration at TextVQA shapes (test_m4c_model_gpu.test_textvqa_shape_training_step's batch):
    20 question tokens, 100 objects, 50 OCR tokens, 12 decoding steps, 5000 answers + 50 OCR copies"""
    import test_m4c_model_cpu as C
    import mmf_b200.models as MD
    from mmf_b200.graphs import GraphedForward
    from mmf_b200.registry import registry
    from mmf_b200.sample import SampleList
    golden = _load("m4c_model.pt")
    C.register(golden)
    registry.register(golden["dataset"] + "_num_final_outputs", 5050)
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).cuda().eval()
    B, T, R, O, D = 32, 20, 100, 50, 12

    def batch(seed):
        torch.manual_seed(seed)
        dev = DEV
        return SampleList(
            text=torch.randint(1, 30522, (B, T), device=dev), text_len=torch.randint(1, T + 1, (B,), device=dev),
            image_feature_0=torch.randn(B, R, 2048, device=dev).relu(), obj_bbox_coordinates=torch.rand(B, R, 4, device=dev),
            image_info_0={"max_features": torch.randint(10, R + 1, (B,), device=dev)},
            context_feature_0=torch.randn(B, O, 300, device=dev), context_feature_1=torch.rand(B, O, 604, device=dev),
            image_feature_1=torch.randn(B, O, 2048, device=dev).relu(), order_vectors=torch.zeros(B, O, 50, device=dev),
            ocr_bbox_coordinates=torch.rand(B, O, 4, device=dev),
            context_info_0={"max_features": torch.randint(0, O + 1, (B,), device=dev)},
            train_prev_inds=torch.randint(0, 5050, (B, D), device=dev),
            targets=(torch.rand(B, D, 5050, device=dev) < 0.001).float(),
            train_loss_mask=(torch.rand(B, D, device=dev) < 0.7).float(), dataset_name="textvqa", dataset_type="val")

    batches = [batch(s) for s in (0, 1, 2)]
    with torch.no_grad():
        model(_fresh(batches[0]))                    # the lazy engine state, outside the sync check
    fwd = GraphedForward(model, batches[0])
    for b in batches:
        got = _snapshot(fwd(b))
        with torch.no_grad(), _no_host_reads():
            want = model(_fresh(b))
        torch.cuda.synchronize()
        assert want["scores"].shape == (B, D, 5050)
        assert torch.equal(got["scores"], want["scores"])
        assert torch.equal(got["scores"].argmax(-1), want["scores"].argmax(-1))
        _assert_same(got, want, "m4c_textvqa")


# ---------------------------------------------------------------------------------------------------------------------
# static_rows=True
# ---------------------------------------------------------------------------------------------------------------------
def _pretraining(name):
    if name == "lxmert":
        return _golden_case("test_lxmert_model_cpu", "lxmert_model.pt", "pretraining_masked_vqa2")
    return _golden_case("test_vinvl_model_cpu", "vinvl_model.pt", "pretraining")


def _visual_bert_skip_padding():
    import bench
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.visual_bert import B200VisualBERT
    wl = bench.VisualBertWL()
    torch.manual_seed(0)
    model = B200VisualBERT(wl.config(0.1))
    assert set_skip_padding(model) >= 1
    return model, bench.to_device(wl.host_batch(32, 17), DEV)


@pytest.mark.parametrize("name", ["lxmert", "vinvl", "visual_bert_skip_padding"])
def test_static_rows_replay_is_the_eager_static_rows_forward(name):
    with _deterministic() if name in ("lxmert", "vinvl") else contextlib.nullcontext():
        _static_rows_case(name)


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _static_rows_case(name):
    from mmf_b200.graphs import GraphedForward, static_rows
    model, batch = _visual_bert_skip_padding() if name == "visual_bert_skip_padding" else _pretraining(name)
    model = model.to(DEV).eval()
    with torch.no_grad(), static_rows():
        first = _snapshot(model(_fresh(batch)))
    fwd = GraphedForward(model, batch, static_rows=True)
    for seed in (1, 2, 3):
        b = _variant(batch, seed)
        if "lm_label_ids" in b and seed == 2:
            b["lm_label_ids"] = torch.full_like(b["lm_label_ids"], -1)      # no labelled row: a loss of exactly 0
        got = _snapshot(fwd(b))
        with torch.no_grad(), static_rows(), _no_host_reads():
            want = model(_fresh(b))
        torch.cuda.synchronize()
        key = "sequence_output" if name == "visual_bert_skip_padding" else "losses"
        assert not _equal_tree(want[key], first[key]), (name, seed)
        _assert_same(got, want, "%s/%d" % (name, seed))


def _equal_tree(a, b):
    try:
        _assert_same(a, b, "")
        return True
    except AssertionError:
        return False


def test_replays_leave_the_model_untouched():
    """capture and replay change no parameter and no buffer"""
    from mmf_b200.graphs import GraphedForward
    model, batch = _case("m4c")
    before = {k: v.detach().clone() for k, v in model.state_dict().items()}
    fwd = GraphedForward(model, batch, warmup=2)
    fwd(_variant(batch, 4))
    torch.cuda.synchronize()
    after = model.state_dict()
    assert after.keys() == before.keys() and all(torch.equal(after[k], v) for k, v in before.items())
    assert not model.training
