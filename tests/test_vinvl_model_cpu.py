"""The registered `vinvl` model (mmf_b200.vinvl_model.VinVL) on the CPU: config handling, the attention masks of the
SampleList plumbing, classification and masked-LM + three-way contrastive pretraining run over the kernel test double
(tests/fake_kernels.py) and are held to tests/golden/vinvl_model.pt - outputs of the REFERENCE's own registered VinVL
(tools/make_golden_vinvl_model.py).  The kernels themselves are covered on the GPU (tests/test_vinvl_model_gpu.py)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["classification", "pretraining", "pretraining_no_mlm"]
FORMS = {"classification": "1d", "pretraining": "2d", "pretraining_no_mlm": "absent"}


def rel(a, b):
    a, b = kept(a, b)
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "vinvl_model.pt"), weights_only=False)


@pytest.fixture()
def cpu_models(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.engine as E
    import mmf_b200.heads as HD
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.vilbert as VB
    import mmf_b200.vinvl as VV
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPS, "F", FK)
    monkeypatch.setattr(EM, "F", FK)
    for mod in (M, EM, VB, HD, VV):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    import mmf_b200.mmft  # noqa: F401  (the head table)
    import mmf_b200.models as MD
    return MD


def _ref_keys(keys):
    # transformers 5 lists the MLM decoder's bias under `decoder.bias` as well as `predictions.bias`
    return {k for k in keys if not k.endswith("predictions.decoder.bias")}


def _state_dict(golden, case):
    sd = dict(golden["pretraining_state_dict"])
    if case == "classification":
        sd = {k: v for k, v in sd.items() if k.startswith("vinvl.bert.")}
        sd.update(golden["classification"]["head_state_dict"])
    return {k: v for k, v in sd.items() if k in _ref_keys(sd)}


def _build(MD, golden, case, **over):
    cfg = MD.load_model_config("vinvl", overrides=dict(golden[case]["config"], **over))
    model = MD.build_model(cfg).eval()
    model.load_state_dict(_state_dict(golden, case), strict=False)
    return model


def _image_info(i, form, device):
    if form == "absent":
        return {}
    return {"max_features": (i["max_features"] if form == "1d" else i["max_features_2d"]).to(device)}


def _sample_list(golden, case, device="cpu"):
    from mmf_b200.sample import SampleList
    i = golden["inputs"]
    lm = torch.full_like(i["lm_label_ids"], -1) if case == "pretraining_no_mlm" else i["lm_label_ids"]
    return SampleList(input_ids=i["ids"].to(device), input_ids_masked=i["ids_masked"].to(device),
                      input_ids_corrupt=i["ids_corrupt"].to(device), lm_label_ids=lm.to(device),
                      input_mask=i["mask"].to(device), input_mask_corrupt=i["mask_corrupt"].to(device),
                      segment_ids=i["segment"].to(device), segment_ids_corrupt=i["segment_corrupt"].to(device),
                      image_feature_0=i["feats"].to(device), image_info_0=_image_info(i, FORMS[case], device),
                      contrastive_labels=i["contrastive_labels"].to(device), labels=i["labels"].to(device),
                      dataset_name="test", dataset_type="train")


def _trunk_masks(model):
    """the attention masks the registered forward hands to the trunk, in call order"""
    seen = []
    hook = model.vinvl.bert.register_forward_pre_hook(lambda mod, a, kw: seen.append(kw["attention_mask"].clone()),
                                                      with_kwargs=True)
    return seen, hook


def check_case(model, golden, case, device, loss_tol, score_tol, grad_tol):
    """losses, scores, the trunk's attention masks (bit for bit) and sampled 2-D gradients against the golden; returns
    the worst errors"""
    g = golden[case]
    masks, hook = _trunk_masks(model)
    out = model(_sample_list(golden, case, device))
    hook.remove()
    assert len(masks) == len(g["attention_masks"])
    for got, ref in zip(masks, g["attention_masks"]):
        assert got.dtype == ref.dtype and torch.equal(got.cpu(), ref)
    assert list(out["losses"].keys()) == list(g["losses"].keys())
    worst = {"loss": 0.0}
    for k, v in g["losses"].items():
        got = float(out["losses"][k].detach())
        err = abs(got - float(v)) / max(abs(float(v)), 1e-3)
        worst["loss"] = max(worst["loss"], err)
        assert err < loss_tol, (k, got, float(v))
        if float(v) == 0.0:
            assert got == 0.0, k
    if case == "classification":
        worst["scores"] = rel(out["scores"].cpu(), g["scores"])
        assert worst["scores"] < score_tol
    sum(v for v in out["losses"].values()).backward()
    named = dict(model.named_parameters())
    checked, worst["grad"] = 0, 0.0
    for k, gr in g["grads"].items():
        if kept(gr, gr)[1].norm() == 0:
            # the reference runs the MLM head on zero rows and gets zero gradients; here it is not run
            assert named[k].grad is None or named[k].grad.abs().max() == 0, k
            continue
        assert named[k].grad is not None, k
        if kept(gr, gr)[1].norm() > 1e-6:
            e = rel(named[k].grad.cpu(), gr)
            worst["grad"] = max(worst["grad"], e)
            assert e < grad_tol(k), (k, e)
            checked += 1
    assert checked >= 0.75 * len(g["grads"]), (checked, len(g["grads"]))
    return out, worst


def test_restated_defaults_equal_the_reference_yaml(cpu_models, golden):
    MD = cpu_models
    from mmf_b200 import vinvl_model as VM
    assert dict(MD.ConfigNode(MD.MODEL_DEFAULTS["vinvl"])) == dict(MD.ConfigNode(golden["defaults"]))
    assert VM.CONFIG_DEFAULTS == golden["config_defaults"]
    assert MD.registry.get_model_class("vinvl") is VM.VinVL
    assert VM.VinVL.config_path() == "configs/models/vinvl/defaults.yaml"
    import mmf_b200
    assert mmf_b200.VinVL is VM.VinVL


def test_default_yaml_classifies_with_a_two_label_mlp(cpu_models):
    """the default YAML's `heads.test` is not read: without a head under the key `mlp` the classifier is MLPHead
    ({"num_layers": 0}) - pooler + Linear(768, 2) - on a bert-base trunk with 2054-wide region features"""
    MD = cpu_models
    m = MD.build_model(MD.load_model_config("vinvl"))
    assert type(m.vinvl).__name__ == "B200VinVLForClassification" and not hasattr(m, "losses")
    assert m.config.do_pretraining is False and m.config.img_feature_dim == 2054 and m.config.loss_type == "sfmx"
    c = m.vinvl.classifier
    assert c.num_labels == 2 and len(c.classifier) == 1 and tuple(c.classifier[0].weight.shape) == (2, 768)
    assert len(m.vinvl.bert.encoder.layer) == 12 and m.vinvl.bert.img_embedding[0].in_features == 2054
    assert m.vinvl.bert.use_img_layernorm and m.vinvl.ce_loss.ignore_index == -100
    m = MD.build_model(MD.load_model_config("vinvl", overrides={"heads": {"mlp": {"num_labels": 3129}},
                                                                "ce_loss": {"ignore_index": -1}}))
    assert m.vinvl.classifier.num_labels == 3129 and len(m.vinvl.classifier.classifier) == 3     # num_layers 1
    assert m.vinvl.ce_loss.ignore_index == -1


def test_default_pretraining_heads(cpu_models):
    MD = cpu_models
    m = MD.build_model(MD.load_model_config("vinvl", overrides={"do_pretraining": True,
                                                                "heads": {"mlm": {"hidden_size": 768}}}))
    p = m.vinvl
    assert type(p).__name__ == "B200VinVLForPretraining"
    assert p.mlm_head.vocab_size == 30522 and p.mlm_head.config.ignore_index == -1
    c = p.contrast_head
    assert c.config.loss_name == "three_way_contrastive_loss" and c.config.num_labels == 3 and c.config.num_layers == 0
    assert c.config.constrastive_label_key == "contrastive_labels" and c.config.ignore_index == -1
    assert len(c.contrast_head.classifier) == 1 and tuple(c.contrast_head.classifier[0].weight.shape) == (3, 768)


@pytest.mark.parametrize("case", ["classification", "pretraining"])
def test_state_dict_keys_are_the_references(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, case)
    assert _ref_keys(model.state_dict().keys()) == _ref_keys(golden[case]["state_dict_keys"])
    res = model.load_state_dict(_state_dict(golden, case), strict=False)
    assert not res.unexpected_keys and _ref_keys(res.missing_keys) == set()


@pytest.mark.parametrize("form", ["absent", "1d", "2d"])
def test_attention_masks_bit_for_bit(cpu_models, golden, form):
    """_get_attention_mask for image_info_0 without max_features, with [B] ints and with the [B, R] floats the
    reference's own test passes"""
    MD = cpu_models
    model = _build(MD, golden, "pretraining")
    i = golden["inputs"]
    got = model._get_attention_mask(i["feats"], _image_info(i, form, "cpu"), i["mask"])
    ref = golden["masks"][form]
    assert got.dtype == ref.dtype and torch.equal(got, ref)


@pytest.mark.parametrize("case", CASES)
def test_registered_model_vs_reference_golden(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, case)
    check_case(model, golden, case, "cpu", 2e-2, 2e-2, lambda k: 8e-2)


def test_pretraining_gradients_are_the_sum_of_both_trunk_passes(cpu_models, golden):
    """the two trunk passes of a pretraining forward (masked captions for the MLM loss, corrupt captions for the
    contrastive loss) reach one ParamPack: one backward of the sum gives each loss's own gradients added"""
    MD = cpu_models
    g = golden["pretraining"]
    model = _build(MD, golden, "pretraining")
    named = dict(model.named_parameters())
    own = {}
    for loss_name in g["losses"]:
        model.zero_grad(set_to_none=True)
        model(_sample_list(golden, "pretraining"))["losses"][loss_name].backward()
        own[loss_name] = {k: named[k].grad.clone() for k in g["by_loss"][loss_name]["grads"]}
        for k, ref in g["by_loss"][loss_name]["grads"].items():
            assert rel(own[loss_name][k], ref) < 8e-2, (loss_name, k)
    model.zero_grad(set_to_none=True)
    sum(model(_sample_list(golden, "pretraining"))["losses"].values()).backward()
    for k in own["masked_lm_loss"]:
        total = named[k].grad
        parts = own["masked_lm_loss"][k] + own["three_way_contrastive_loss"][k]
        assert rel(total, parts) < 1e-5, k
        assert own["masked_lm_loss"][k].abs().max() > 0 and own["three_way_contrastive_loss"][k].abs().max() > 0, k
        assert rel(total, g["grads"][k]) < 8e-2, k


def test_no_kept_mlm_label_gives_zero_loss_and_the_contrastive_loss_trains(cpu_models, golden):
    MD = cpu_models
    model = _build(MD, golden, "pretraining_no_mlm")
    with pytest.warns(UserWarning, match="NaN detected in masked_lm_loss"):
        out = model(_sample_list(golden, "pretraining_no_mlm"))
    assert float(out["losses"]["masked_lm_loss"]) == 0.0
    sum(out["losses"].values()).backward()
    head = model.vinvl.mlm_head.cls.predictions
    assert head.decoder.weight.grad is None or head.decoder.weight.grad.abs().max() == 0
    assert model.vinvl.contrast_head.contrast_head.classifier[0].weight.grad.abs().max() > 0


def test_classification_without_labels_returns_scores_only(cpu_models, golden):
    MD = cpu_models
    model = _build(MD, golden, "classification")
    sl = _sample_list(golden, "classification")
    del sl["labels"]
    out = model(sl)
    assert out["losses"] == {} and rel(out["scores"], golden["classification"]["scores"]) < 2e-2


def test_contrastive_label_fallback_key(cpu_models, golden):
    from mmf_b200.mmft import ThreeWayContrastiveHead
    head = ThreeWayContrastiveHead({"hidden_size": 16, "constrastive_label_key": "nsp"})
    seq = torch.randn(4, 5, 16)
    labels = torch.tensor([0, 2, 1, -1])
    a = head(seq, {"three_way_constrastive_labels": {"nsp": labels}})["losses"]["three_way_contrastive_loss"]
    b = head(seq, {"nsp": labels})["losses"]["three_way_contrastive_loss"]
    scores = head.contrast_head(seq)["scores"]
    assert torch.equal(a, b) and torch.allclose(a, torch.nn.functional.cross_entropy(scores, labels, ignore_index=-1))
    with pytest.raises(AssertionError, match="requires three_way_constrastive_labels to be in sample list"):
        head(seq, {"three_way_constrastive_labels": None})


def test_contrastive_head_in_an_mmft_config(cpu_models):
    """the head is in the shared table: an MMFT config can name it, its parameters are `contrast_head.*` under the
    head's index, and MMFT's three-argument head call reaches it"""
    MD = cpu_models
    small = {"hidden_size": 64, "num_hidden_layers": 1, "num_attention_heads": 1, "intermediate_size": 128,
             "vocab_size": 512, "max_position_embeddings": 128, "hidden_dropout_prob": 0.0,
             "attention_probs_dropout_prob": 0.0}
    cfg = MD.load_model_config("mmf_transformer", overrides={
        "transformer_config": small, "modalities": [dict(type="text", key="text", embedding_dim=64, position_dim=128,
                                                         segment_id=0, encoder=dict(type="identity"))],
        "heads": [{"type": "contrastive_three_way", "hidden_size": 64}]})
    m = MD.build_model(cfg)
    keys = {k for k in m.state_dict() if k.startswith("heads.")}
    assert keys == {"heads.0.contrast_head.pooler.dense.weight", "heads.0.contrast_head.pooler.dense.bias",
                    "heads.0.contrast_head.classifier.0.weight", "heads.0.contrast_head.classifier.0.bias"}
    seq = torch.randn(2, 3, 64)
    labels = torch.tensor([1, 0])
    out = m.postprocess_output(seq, [], {"three_way_constrastive_labels": {"contrastive_labels": labels}})
    scores = m.heads[0].contrast_head(seq)["scores"]
    assert torch.allclose(out["losses"]["three_way_contrastive_loss"], torch.nn.functional.cross_entropy(scores, labels))


def test_three_d_masks_stay_unsupported(cpu_models, golden):
    MD = cpu_models
    model = _build(MD, golden, "classification")
    i = golden["inputs"]
    with pytest.raises(NotImplementedError, match="per-query"):
        model.vinvl(i["ids"], i["segment"], torch.ones(4, 14, 14, dtype=torch.long), i["feats"])


def test_graphed_step_refuses_the_model(cpu_models, golden):
    from mmf_b200.graphs import GraphedStep
    model = _build(cpu_models, golden, "pretraining")
    with pytest.raises(RuntimeError, match="VinVL gathers a data-dependent number of rows.*cannot be captured"):
        GraphedStep(model, lambda b: None, {})
