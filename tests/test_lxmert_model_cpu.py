"""The registered `lxmert` model (mmf_b200.models.LXMERT) on the CPU: config handling, the SampleList plumbing with its
integer tensors, the pretraining heads and losses and the classifier run over the kernel test double
(tests/fake_kernels.py) and are held to tests/golden/lxmert_model.pt - outputs of the REFERENCE's own registered LXMERT
(tools/make_golden_lxmert_model.py).  The kernels themselves are covered on the GPU (tests/test_lxmert_model_gpu.py)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF_ROOT = os.environ.get("MMF_REFERENCE_ROOT", "/root/reference")


def rel(a, b):
    a, b = kept(a, b)        # a sampled golden gradient: compare the elements it stores
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "lxmert_model.pt"), weights_only=False)


@pytest.fixture()
def cpu_models(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.engine as E
    import mmf_b200.heads as HD
    import mmf_b200.lxmert as LX
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.vilbert as VB
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPS, "F", FK)
    monkeypatch.setattr(EM, "F", FK)
    for mod in (M, EM, VB, HD, LX):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    import mmf_b200.models as MD
    return MD


def _ref_keys(keys):
    # HF registers `position_ids` / `token_type_ids` buffers in BertEmbeddings; aside from those the key sets are LXMERT's
    return {k for k in keys if not k.endswith("position_ids") and not k.endswith("token_type_ids")}


def _build(MD, golden, case):
    cfg_dict = golden["pretraining_config"] if case.startswith("pretraining") else golden[case]["config"]
    cfg = MD.load_model_config("lxmert", overrides=dict(cfg_dict))
    if case == "classification":
        cfg.losses = [{"type": "logit_bce"}]
    elif case == "nlvr2":
        cfg.losses = [{"type": "cross_entropy"}]
    model = MD.build_model(cfg).eval()
    sd = {k: v for k, v in golden["pretraining_state_dict"].items()}
    if not case.startswith("pretraining"):
        sd = {k: v for k, v in sd.items() if k.startswith("model.bert.")}
        sd.update(golden[case]["head_state_dict"])
    model.load_state_dict({k: v for k, v in sd.items() if k in _ref_keys(sd)})
    return model


def _sample_list(golden, case, device="cpu"):
    from mmf_b200.sample import SampleList
    i = golden["inputs"]
    name, targets = {"pretraining_masked_vqa2": ("masked_vqa2", i["vqa_targets"]),
                     "pretraining_masked_gqa": ("masked_gqa", i["gqa_targets"]),
                     "classification": ("vqa2", i["vqa_targets"]), "nlvr2": ("nlvr2", i["nlvr2_targets"])}[case]
    return SampleList(input_ids=i["ids"].to(device), input_mask=i["mask"].to(device), segment_ids=i["seg"].to(device),
                      lm_label_ids=i["lm_label_ids"].to(device), image_feature_0=i["feats"].to(device),
                      image_info_0={"max_features": i["max_features"].to(device), "bbox": i["bbox"].to(device),
                                    "cls_prob": i["cls_prob"].numpy().copy()},
                      image_labels=i["image_labels"].to(device), targets=targets.to(device),
                      is_correct=i["is_correct"].to(device), dataset_name=name, dataset_type="train")


def _record(model):
    """the keyword arguments the registered model hands its head model"""
    seen = {}
    inner = model.model.forward

    def fwd(**kw):
        seen.update({k: v for k, v in kw.items() if torch.is_tensor(v)})
        return inner(**kw)
    model.model.forward = fwd
    return seen


def _check_plumbing(seen, ref):
    for k in ("token_type_ids", "attention_mask", "visual_pos", "visual_attention_mask", "masked_image_labels",
              "obj_labels"):
        if k in ref:
            assert torch.equal(seen[k].cpu(), ref[k]), k
    if "obj_index" in ref:
        top = seen["obj_labels"].max(-1)
        assert torch.equal(top.indices.cpu(), ref["obj_index"]) and torch.equal(top.values.cpu(), ref["obj_conf"])
        assert torch.equal((seen["masked_image_labels"] == 1).float().cpu(), ref["feat_mask"])


def test_restated_defaults_equal_the_reference_yaml(cpu_models, golden):
    """MODEL_DEFAULTS["lxmert"] restates model_config.lxmert of configs/models/lxmert/defaults.yaml (read by the product's
    own YAML loader when the fixture was made)"""
    MD = cpu_models
    assert dict(MD.ConfigNode(MD.MODEL_DEFAULTS["lxmert"])) == dict(MD.ConfigNode(golden["defaults"]))
    assert MD.registry.get_model_class("lxmert") is MD.LXMERT
    assert MD.LXMERT.config_path() == "configs/models/lxmert/pretrain.yaml"


def test_default_config_builds_both_heads(cpu_models):
    MD = cpu_models
    assert type(MD.build_model(MD.load_model_config("lxmert")).model).__name__ == "B200LXMERTForPretraining"
    m = MD.build_model(MD.load_model_config("lxmert", overrides={"training_head_type": "classification"}))
    assert type(m.model).__name__ == "B200LXMERTForClassification"
    assert m.model.classifier.logit_fc[3].out_features == 3129 and m.model.classifier.logit_gqa[3].out_features == 1534


@pytest.mark.parametrize("case", ["pretraining", "classification", "nlvr2"])
def test_state_dict_keys_are_the_references(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, "pretraining_masked_vqa2" if case == "pretraining" else case)
    ref = golden["pretraining_state_dict"].keys() if case == "pretraining" else golden[case]["state_dict_keys"]
    assert set(model.state_dict().keys()) == _ref_keys(ref)
    if case == "pretraining":       # the tie: one parameter, one gradient
        assert model.model.cls.predictions.decoder.weight is model.model.bert.embeddings.word_embeddings.weight


@pytest.mark.parametrize("case", ["pretraining_masked_vqa2", "pretraining_masked_gqa", "classification", "nlvr2"])
def test_registered_model_vs_reference_golden(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, case)
    seen = _record(model)
    out = model(_sample_list(golden, case))
    g = golden[case]
    _check_plumbing(seen, g["plumbing"])
    if case.startswith("pretraining"):
        assert list(out["losses"].keys()) == list(g["losses"].keys())
        for k, v in g["losses"].items():
            got = float(out["losses"][k].detach())
            assert abs(got - float(v)) < 2e-2 * abs(float(v)), (k, got, float(v))
        loss = sum(out["losses"].values())
    else:
        assert rel(out["scores"], g["scores"]) < 2e-2, rel(out["scores"], g["scores"])
        key = "train/%s/%s" % ("vqa2" if case == "classification" else "nlvr2",
                               "logit_bce" if case == "classification" else "cross_entropy")
        assert list(out["losses"].keys()) == [key]
        loss = out["losses"][key].sum()
        assert abs(float(loss.detach()) - float(g["loss"])) < 2e-2 * abs(float(g["loss"]))
    loss.backward()
    named = dict(model.named_parameters())
    checked = 0
    for k, gr in g["grads"].items():
        assert named[k].grad is not None, k
        # the relational layer's query / key gradients of this one-head fixture are ~1e-8: no signal to compare
        if kept(gr, gr)[1].norm() > 1e-6:
            assert rel(named[k].grad, gr) < 8e-2, (k, rel(named[k].grad, gr))
            checked += 1
    assert checked >= 0.75 * len(g["grads"])


def test_masked_lm_loss_without_labelled_positions_is_zero(cpu_models, golden):
    MD = cpu_models
    model = _build(MD, golden, "pretraining_masked_vqa2")
    sl = _sample_list(golden, "pretraining_masked_vqa2")
    sl["lm_label_ids"] = torch.full_like(sl["lm_label_ids"], -1)
    out = model(sl)
    assert float(out["losses"]["masked_vqa2/train/masked_lm_loss"]) == 0.0
    assert all(torch.isfinite(v).all() for v in out["losses"].values())


def test_freeze_base_leaves_the_trunk_without_gradients(cpu_models, golden):
    MD = cpu_models
    cfg = MD.load_model_config("lxmert", overrides=dict(golden["pretraining_config"], freeze_base=True))
    model = MD.build_model(cfg).eval()
    out = model(_sample_list(golden, "pretraining_masked_vqa2"))
    sum(out["losses"].values()).backward()
    assert all(p.grad is None for p in model.model.bert.parameters())
    assert model.model.answer_head.logit_fc[0].weight.grad is not None
    assert model.model.obj_predict_head.decoder_dict["obj"].weight.grad is not None


@pytest.mark.parametrize("key", ["dynamic_attention", "in_batch_pairs", "fast_mode", "output_attentions",
                                 "output_hidden_states", "visualization"])
def test_unsupported_options_raise(cpu_models, key):
    MD = cpu_models
    with pytest.raises(NotImplementedError, match=key):
        MD.build_model(MD.load_model_config("lxmert", overrides={key: True}))


def test_packed_streams_are_refused_by_the_registered_model(cpu_models, golden):
    """segment_ids are the text attention mask (the reference's swap): packing would drop [CLS] and the MLM rows"""
    from mmf_b200.patch import set_skip_padding
    MD = cpu_models
    model = _build(MD, golden, "pretraining_masked_vqa2")
    assert set_skip_padding(model, two_stream=True) == 1
    with pytest.raises(ValueError, match="swap"):
        model(_sample_list(golden, "pretraining_masked_vqa2"))
    set_skip_padding(model, False, two_stream=True)
    assert "losses" in model(_sample_list(golden, "pretraining_masked_vqa2"))


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF_ROOT, "projects", "lxmert")), reason="needs the MMF tree")
def test_project_yamls_load(cpu_models):
    MD = cpu_models
    root = os.path.join(REF_ROOT, "mmf")
    proj = os.path.join(REF_ROOT, "projects", "lxmert", "configs")
    c = MD.load_model_config("lxmert", yaml_path=os.path.join(proj, "vqa2", "defaults.yaml"), mmf_root=root)
    assert c.training_head_type == "classification" and c.num_labels == 3129 and c.losses[0]["type"] == "logit_bce"
    assert type(MD.build_model(c).model).__name__ == "B200LXMERTForClassification"
    c = MD.load_model_config("lxmert", yaml_path=os.path.join(proj, "gqa", "pretrain.yaml"), mmf_root=root)
    assert c.num_labels == 1534 and c.visual_loss_config.obj[0] == 1600 and c.model == "lxmert"
    for sub in ("coco", "vqa2"):
        c = MD.load_model_config("lxmert", yaml_path=os.path.join(proj, sub, "pretrain.yaml"), mmf_root=root)
        assert c.training_head_type == "pretraining" and c.l_layers == 9
