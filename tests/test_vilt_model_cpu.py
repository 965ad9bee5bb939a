"""The registered `vilt` model (mmf_b200.vilt_model.ViLT) on the CPU: config handling, the attention masks of the sample
list plumbing, VQA classification and masked-LM + ITM pretraining run over the kernel test double (tests/fake_kernels.py)
and held to tests/golden/vilt_model.pt - outputs of the REFERENCE's own registered ViLT (tools/make_golden_vilt_model.py).
The kernels themselves are covered on the GPU (tests/test_vilt_model_gpu.py)."""
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["classification", "classification_nomask", "pretraining", "pretraining_no_mlm"]


def rel(a, b):
    a, b = kept(a, b)
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "vilt_model.pt"), weights_only=False)


@pytest.fixture()
def cpu_models(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.engine as E
    import mmf_b200.heads as HD
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.vilbert as VB
    import mmf_b200.vit as VT
    monkeypatch.setattr(E, "F", FK)
    monkeypatch.setattr(OPS, "F", FK)
    monkeypatch.setattr(EM, "F", FK)
    for mod in (M, EM, VB, HD, VT):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    import mmf_b200.mmft  # noqa: F401  (the head table)
    import mmf_b200.models as MD
    return MD


def _ref_keys(keys):
    # transformers 5 lists the MLM decoder's bias under `decoder.bias` as well as `predictions.bias`
    return {k for k in keys if not k.endswith("predictions.decoder.bias")}


def _state_dict(golden, case):
    sd = dict(golden["pretraining_state_dict"])
    if case.startswith("classification"):
        sd = {k: v for k, v in sd.items() if not k.startswith("heads_dict.")}
        sd.update(golden["classification_head_state_dict"])
    return {k: v for k, v in sd.items() if k in _ref_keys(sd)}


def _build(MD, golden, case, **over):
    cfg = MD.load_model_config("vilt", overrides=dict(golden[case]["config"], **over))
    model = MD.build_model(cfg).eval()
    model.load_state_dict(_state_dict(golden, case), strict=False)
    return model


def _sample_list(golden, case, device="cpu", plain=False):
    from mmf_b200.sample import SampleList
    i = golden["inputs"]
    sl = dict(input_ids=i["ids"], segment_ids=i["segment"], image=i["image"], dataset_name=None, dataset_type="train")
    sl["dataset_name"] = "vqa2" if case.startswith("classification") else "masked_coco"
    if case != "classification_nomask":
        sl["input_mask"] = i["mask"]
    if case.startswith("classification"):
        sl["targets"] = i["targets"]
    else:
        sl.update(input_ids_masked=i["ids_masked"], is_correct=i["is_correct"],
                  lm_label_ids=torch.full_like(i["lm_label_ids"], -1) if case == "pretraining_no_mlm"
                  else i["lm_label_ids"])
    sl = {k: (v.clone().to(device) if torch.is_tensor(v) else v) for k, v in sl.items()}
    return sl if plain else SampleList(sl)


def _encoder_masks(model):
    """the masks the registered forward hands to the encoder, in call order"""
    seen = []

    def grab(mod, a, kw):
        am = kw.get("attention_mask")
        seen.append(None if am is None else am.clone())
    return seen, model.encoder.register_forward_pre_hook(grab, with_kwargs=True)


def check_case(model, golden, case, device, loss_tol, score_tol, grad_tol):
    """losses, scores, the encoder's masks (bit for bit) and sampled gradients against the golden; returns the worst
    errors"""
    g = golden[case]
    masks, hook = _encoder_masks(model)
    out = model(_sample_list(golden, case, device))
    hook.remove()
    assert len(masks) == len(g["attention_masks"])
    for got, ref in zip(masks, g["attention_masks"]):
        assert (got is None) == (ref is None)
        if ref is not None:
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
    if "scores" in g:
        worst["scores"] = rel(out["scores"].cpu(), g["scores"])
        assert worst["scores"] < score_tol
    else:
        assert isinstance(out["scores"], int) and out["scores"] == 0          # no head returned scores
    sum(v.sum() for v in out["losses"].values()).backward()
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
    from mmf_b200 import vilt_model as VM
    assert dict(MD.ConfigNode(MD.MODEL_DEFAULTS["vilt"])) == dict(MD.ConfigNode(golden["defaults"]))
    assert MD.registry.get_model_class("vilt") is VM.ViLT
    assert VM.ViLT.config_path() == "configs/models/vilt/defaults.yaml"
    import mmf_b200
    assert mmf_b200.ViLT is VM.ViLT
    from mmf_b200.encoders import B200ViTImageEncoder
    assert MD.registry.get_encoder_class("vit") is B200ViTImageEncoder


@pytest.mark.parametrize("case", ["classification", "pretraining"])
def test_state_dict_keys_are_the_references(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, case)
    keys = _ref_keys(model.state_dict().keys())
    assert keys == _ref_keys(golden[case]["state_dict_keys"])
    assert any(k.startswith("encoder.module.embeddings.") for k in keys)          # built, never called
    assert any(k.startswith("encoder.embeddings.") for k in keys)                 # and its alias
    res = model.load_state_dict(_state_dict(golden, case), strict=False)
    assert not res.unexpected_keys and _ref_keys(res.missing_keys) == set()


@pytest.mark.parametrize("case", ["classification", "pretraining"])
def test_optimizer_groups_are_the_references(cpu_models, golden, case):
    model = _build(cpu_models, golden, case)
    names = {id(p): n for n, p in model.named_parameters()}
    got = [{"names": [names[id(p)] for p in g["params"]], "weight_decay": g.get("weight_decay")}
           for g in model.get_optimizer_parameters(None)]
    ref = [dict(g, names=[n for n in g["names"] if n in _ref_keys([n])]) for g in golden[case]["groups"]]
    assert got == ref


@pytest.mark.parametrize("form", ["sample_list", "dict", "image_mask_only", "absent"])
def test_attention_mask_bit_for_bit(cpu_models, golden, form):
    """getattr() on the sample list: a SampleList yields its masks, a plain dict none; a missing half is ones in the
    embedding's dtype"""
    from mmf_b200.sample import SampleList
    model = _build(cpu_models, golden, "pretraining")
    i = golden["inputs"]
    sl = _sample_list(golden, "pretraining", plain=form == "dict")
    if form == "image_mask_only":
        del sl["input_mask"]
        sl["image_mask"] = i["image_mask"]
    elif form == "absent":
        sl = SampleList(input_ids=i["ids"])
    with torch.no_grad():
        te = model.text_embeddings(i["ids"], i["segment"])
        ie = model.image_embeddings(i["image"])
    got = model.get_attention_mask(sl, te, ie)
    ref = golden["masks"][form]
    if ref is None:
        assert got is None
    else:
        assert got.dtype == ref.dtype and torch.equal(got, ref)


@pytest.mark.parametrize("case", CASES)
def test_registered_model_vs_reference_golden(cpu_models, golden, case):
    model = _build(cpu_models, golden, case)
    check_case(model, golden, case, "cpu", 2e-2, 2e-2, lambda k: 8e-2)


def test_mlm_pass_is_image_first_with_the_text_first_mask_and_labels(cpu_models, golden):
    """the masked-LM pass runs on [image, text] with cat(text_mask, image_mask) and cat(text_labels, -1): its loss is
    the cross-entropy of the head on the first T rows of that sequence"""
    model = _build(cpu_models, golden, "pretraining")
    i = golden["inputs"]
    masks, hook = _encoder_masks(model)
    seen = []
    h2 = model.encoder.register_forward_pre_hook(lambda mod, a, kw: seen.append(a[0].detach().clone()), with_kwargs=True)
    sl = _sample_list(golden, "pretraining")
    with torch.no_grad():
        out = model(sl)
    hook.remove()
    h2.remove()
    T = i["ids"].shape[1]
    P = model.image_embeddings.num_positions
    assert len(seen) == 2                                           # the masked-LM pass runs first, in preprocess_sample
    text, image = seen[1][:, :T], seen[1][:, T:]
    assert torch.equal(seen[0][:, :P], image)                       # the image embedding, reused
    assert torch.equal(masks[0], masks[1])                          # the text-first mask for both passes
    assert torch.equal(sl["mlm_labels"]["combined_labels"][:, :T], i["lm_label_ids"])
    assert (sl["mlm_labels"]["combined_labels"][:, T:] == -1).all()
    head = model.heads_dict.heads["masked_coco"][0].mlm_head
    hs = sl["hs_masked_for_mlm"]
    sel = i["lm_label_ids"] != -1
    with torch.no_grad():
        logits = head.cls.predictions(hs[:, :T][sel])
    ref = torch.nn.functional.cross_entropy(logits.float(), i["lm_label_ids"][sel])
    assert torch.allclose(out["losses"]["masked_lm_loss"], ref)
    assert not torch.equal(seen[0][:, P:], text)                    # the masked captions, not the plain ones


def test_pretraining_gradients_are_the_sum_of_both_trunk_passes(cpu_models, golden):
    """both trunk passes (the plain captions for ITM, the masked ones for the masked LM) reach the trunk's one
    ParamPack: one backward of the sum gives each loss's own gradients added"""
    g = golden["pretraining"]
    model = _build(cpu_models, golden, "pretraining")
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
        parts = own["masked_lm_loss"][k] + own["itm_loss"][k]
        # the trunk's gradients add in its flat buffer; the patch projection's backward GEMM runs once on the summed
        # (bf16) gradient of the shared image embedding, so its sum holds to rounding only
        assert rel(named[k].grad, parts) < (5e-3 if k.startswith("image_embeddings.") else 1e-5), k
        assert own["masked_lm_loss"][k].abs().max() > 0 and own["itm_loss"][k].abs().max() > 0, k


def test_is_correct_defaults_to_true(cpu_models, golden):
    model = _build(cpu_models, golden, "pretraining")
    sl = _sample_list(golden, "pretraining")
    del sl["is_correct"]
    lab = model._infer_itm_labels(sl)["is_correct"]
    assert lab.dim() == 0 and lab.dtype == torch.long and int(lab) == 1


def test_top_level_head_list(cpu_models, golden):
    """a list of heads serves every task: one ModuleList, keys `heads_dict.heads.<i>.*`"""
    MD = cpu_models
    cfg = dict(golden["classification"]["config"])
    heads = cfg["heads"]["vqa2"]
    model = MD.build_model(_list_config(MD, cfg, heads)).eval()
    model.load_state_dict({k.replace("heads_dict.heads.vqa2.", "heads_dict.heads."): v
                           for k, v in _state_dict(golden, "classification").items()}, strict=False)
    assert isinstance(model.heads_dict.heads, torch.nn.ModuleList) and model.heads_dict.head_names == ["mlp"]
    out = model(_sample_list(golden, "classification"))
    assert rel(out["scores"], golden["classification"]["scores"]) < 2e-2


def _list_config(MD, cfg, heads):
    c = MD.load_model_config("vilt", overrides=cfg)
    c["heads"] = MD.ConfigNode({"h": heads})["h"]
    del c["tasks"]
    return c


@pytest.mark.parametrize("name,positions,patch,text_positions", [
    ("vqa2/vit_b32_384", 145, 32, 512), ("vqa2/vit_b16_224", 197, 16, 512), ("masked_coco/pretrain", 145, 32, 40)])
def test_project_yamls_build(cpu_models, golden, name, positions, patch, text_positions):
    MD = cpu_models
    task = "masked_coco" if name.startswith("masked") else "vqa2"
    block = golden["yamls"][name]
    assert block["tasks"] == "${datasets}"                  # the trainer's dataset list
    m = MD.build_model(MD.load_model_config("vilt", overrides=dict(block, tasks=task)))
    emb = m.image_embeddings.embedding
    assert tuple(emb.position_embeddings.shape) == (1, positions, 768)
    assert tuple(emb.patch_embeddings.projection.weight.shape) == (768, 3, patch, patch)
    assert tuple(m.encoder.module.embeddings.position_embeddings.shape) == (1, positions, 768)
    assert m.text_embeddings.text_embeddings.position_embeddings.weight.shape[0] == text_positions
    assert m.text_embeddings.text_embeddings.word_embeddings.weight.shape[0] == 30522
    hf = m.encoder.hf_config
    assert len(m.encoder.module.encoder.layer) == 12 and hf.hidden_dropout_prob == 0.1
    assert hf.attention_probs_dropout_prob == 0.0 and hf.layer_norm_eps == 1e-12 and m.encoder.module.pooler is None
    assert m.encoder.out_dim == 768 and m.encoder.embeddings is m.encoder.module.embeddings
    heads = m.heads_dict.heads[task]
    if task == "vqa2":
        mlp = heads[0]
        assert m.heads_dict.head_loss_names == {"vqa2": ["vqa2_mlp"]} and "vqa2_mlp" in m.losses
        assert tuple(mlp.classifier[-1].weight.shape) == (3129, 1536) and mlp.in_dim == 768
        assert m.graph_capturable
    else:
        assert m.heads_dict.head_names == {"masked_coco": ["mlm_multi", "itm"]}
        assert heads[0].mlm_head.vocab_size == 30522 and not m.graph_capturable


def test_vit_encoder_plugin_table_and_refusals(cpu_models):
    from mmf_b200.encoders import build_encoder, vit_hf_config
    hf = vit_hf_config({"pretrained_model_name": "google/vit-base-patch32-384", "hidden_dim": 1, "mlp_dim": 1,
                        "regularize_bias": True, "pretrained_model": "x"})
    assert (hf.hidden_size, hf.num_hidden_layers, hf.num_attention_heads, hf.intermediate_size) == (768, 12, 12, 3072)
    assert (hf.image_size, hf.patch_size, hf.layer_norm_eps, hf.attention_probs_dropout_prob) == (384, 32, 1e-12, 0.0)
    assert vit_hf_config({})["image_size"] == 224 and vit_hf_config({})["patch_size"] == 16
    assert vit_hf_config({"patch_size": 8, "image_size": [16, 16]}).patch_size == 8
    with pytest.raises(ValueError, match="pretrained_model_name"):
        vit_hf_config({"pretrained_model_name": "google/vit-large-patch16-224"})
    with pytest.raises(NotImplementedError, match="gradient_checkpointing"):
        vit_hf_config({"gradient_checkpointing": True})
    enc = build_encoder({"type": "vit", "params": {"hidden_size": 64, "num_hidden_layers": 1, "num_attention_heads": 1,
                                                   "intermediate_size": 128, "image_size": 16, "patch_size": 8}})
    assert enc.out_dim == 64 and enc.module.pooler is not None     # add_pooling_layer defaults to True, as in HF


def test_too_many_positions_raise_before_any_launch(cpu_models, golden, monkeypatch):
    """ViT-B/16 at 384 px: 40 tokens + 577 image positions"""
    MD = cpu_models
    m = MD.build_model(MD.load_model_config("vilt", overrides=dict(golden["yamls"]["vqa2/vit_b16_224"], tasks="vqa2",
                                                                   image_encoder={"params": {"image_size": [384, 384]}})))
    assert m.image_embeddings.num_positions == 577

    def boom(*a, **k):
        raise AssertionError("a kernel was called")
    for name in dir(FK):
        if not name.startswith("_") and callable(getattr(FK, name)):
            monkeypatch.setattr(FK, name, boom)
    sl = {"input_ids": torch.zeros(2, 40, dtype=torch.long), "segment_ids": torch.zeros(2, 40, dtype=torch.long),
          "image": torch.zeros(2, 3, 384, 384), "dataset_name": "vqa2"}
    with pytest.raises(ValueError, match="40 text tokens \\+ 577 image positions = 617 exceed the 384"):
        m(sl)


def test_graphed_step_refuses_pretraining_before_warm_up(cpu_models, golden):
    from mmf_b200.graphs import GraphedStep
    model = _build(cpu_models, golden, "pretraining")
    calls = []
    with pytest.raises(RuntimeError, match="ViLT gathers a data-dependent number of rows.*cannot be captured"):
        GraphedStep(model, lambda b: calls.append(b), {})
    assert calls == []
    vqa = _build(cpu_models, golden, "classification")
    assert all(getattr(m, "graph_capturable", True) for m in vqa.modules())


def test_vit_model_turns_a_01_mask_into_the_additive_one(cpu_models):
    """B200ViTModel.forward with a 0/1 [B, S] mask equals the encoder fed (1 - m) * -10000, as ViTModel.forward
    (vit.py:276-284) does"""
    from mmf_b200.vit import B200ViTModel
    cfg = types.SimpleNamespace(hidden_size=128, num_attention_heads=2, intermediate_size=256, num_hidden_layers=2,
                                hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                                hidden_act="gelu", image_size=16, patch_size=8, num_channels=3, initializer_range=0.02,
                                do_patch_embeddings=False, add_pooling_layer=False)
    torch.manual_seed(0)
    m = B200ViTModel(cfg).eval()
    x = torch.randn(3, 11, 128)
    mask = torch.ones(3, 11, dtype=torch.long)
    mask[1, 7:] = 0
    mask[2, 3:5] = 0
    seq, pooled = m(x, attention_mask=mask)
    enc = m.encoder(x, attention_mask=(1.0 - mask[:, None, None, :].float()) * -10000.0, return_dict=False)[0]
    ref = torch.nn.functional.layer_norm(enc.float(), (128,), m.layernorm.weight, m.layernorm.bias, 1e-12)
    assert pooled is None and rel(seq, ref) < 1e-2
    assert torch.equal(m(x)[0], m(x, attention_mask=torch.ones(3, 11))[0])
    assert not torch.allclose(seq, m(x)[0])
    with pytest.raises(NotImplementedError, match="per-query"):
        m(x, attention_mask=torch.ones(3, 11, 11))
