"""The registered `m4c` and `m4c_captioner` models (mmf_b200.m4c_model) on the CPU: config handling, state-dict keys, the
prefix-LM mask, teacher-forced training and greedy decoding run over the kernel test double (tests/fake_kernels.py, with
the causal tail of the attention calls added below) and are held to tests/golden/m4c_model.pt - outputs of the
REFERENCE's own M4C and M4CCaptioner (tools/make_golden_m4c_model.py).  The kernels are covered on the GPU
(tests/test_attention_causal_gpu.py, tests/test_m4c_model_gpu.py)."""
import contextlib
import os
import sys
import types
import zlib

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, b):
    a, b = kept(a, b)
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "m4c_model.pt"), weights_only=False)


# ---- the test double's attention with a causal tail ----------------------------------------------------------------
_TAIL = [0]
_PROBS = FK._probs


def _probs(q, k, B, heads, Sq, Skv, mask):
    """FK._probs with the key mask of the tail keys replaced: 0 for keys <= the query, -10000 after it"""
    T = _TAIL[0]
    if not T:
        return _PROBS(q, k, B, heads, Sq, Skv, mask)
    s = _PROBS(q, k, B, heads, Sq, Skv, None)
    P = Skv - T
    m = torch.zeros(B, Sq, Skv)
    if mask is not None:
        m[:, :, :P] = mask.float()[:, None, :P]
    qi, ki = torch.arange(Sq)[:, None], torch.arange(Skv)[None, :]
    m[:, :, P:] = torch.where(ki[:, P:] <= qi, 0.0, -10000.0)
    return s + m[:, None]


@contextlib.contextmanager
def _tail(T):
    _TAIL[0] = int(T)
    try:
        yield
    finally:
        _TAIL[0] = 0


def _causal_fake():
    """FK with attention_fwd / _bwd that take causal_len"""
    mod = types.ModuleType("fake_kernels_causal")
    mod.__dict__.update({k: v for k, v in FK.__dict__.items() if not k.startswith("__")})

    def attention_fwd(*a, causal_len=0, **k):
        with _tail(causal_len):
            return FK.attention_fwd(*a, **k)

    def attention_bwd(*a, causal_len=0, **k):
        with _tail(causal_len):
            return FK.attention_bwd(*a, **k)
    mod.attention_fwd, mod.attention_bwd = attention_fwd, attention_bwd
    return mod


@pytest.fixture()
def cpu_models(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.encoders as EN
    import mmf_b200.engine as E
    import mmf_b200.m4c_model as MM
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.vilbert as VB
    fake = _causal_fake()
    monkeypatch.setattr(FK, "_probs", _probs)
    monkeypatch.setattr(E, "F", fake)
    monkeypatch.setattr(OPS, "F", fake)
    monkeypatch.setattr(EM, "F", fake)
    for mod in (M, EM, VB, EN, MM):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    import mmf_b200.models as MD
    return MD


# ---- builders shared with the GPU test ------------------------------------------------------------------------------
def _q8(x, base):
    """oracle/make_golden._q8"""
    return torch.round((x - base) * 1024.0).clamp(-127, 127) / 1024.0 + base


def weights(golden):
    """the fixture's weights, drawn from their names as tools/make_golden_m4c_model.weight_value draws them"""
    out = {}
    for n, (shape, base, std) in golden["weight_spec"].items():
        g = torch.Generator().manual_seed(golden["weight_seed"] * 1000003 + zlib.crc32(n.encode()))
        out[n] = _q8(base + torch.randn(shape, generator=g) * std, base)
    return out


def register(golden):
    from mmf_b200.models import ConfigNode
    from mmf_b200.registry import registry
    ds = golden["dataset"]
    registry.register("config", ConfigNode({"datasets": ds}))
    registry.register(ds + "_num_final_outputs", golden["num_final_outputs"])
    registry.register(ds + "_answer_processor", ConfigNode({"BOS_IDX": golden["bos_idx"], "UNK_IDX": golden["unk_idx"]}))


def build(MD, golden, captioner=False, device="cpu"):
    register(golden)
    name = "m4c_captioner" if captioner else "m4c"
    cfg = MD.load_model_config(name, overrides=golden["captioner_config" if captioner else "config"])
    model = MD.build_model(cfg)
    model.load_state_dict(weights(golden), strict=True)
    return model.to(device)


def sample_list(golden, device="cpu", **over):
    from mmf_b200.sample import SampleList
    i = dict(golden["inputs"], **over)
    return SampleList(text=i["text"].to(device), text_len=i["text_len"].to(device),
                      image_feature_0=i["image_feature_0"].to(device), obj_bbox_coordinates=i["obj_bbox_coordinates"].to(device),
                      image_info_0={"max_features": i["obj_max_features"].to(device)},
                      context_feature_0=i["context_feature_0"].to(device), context_feature_1=i["context_feature_1"].to(device),
                      image_feature_1=i["image_feature_1"].to(device), order_vectors=i["order_vectors"].to(device),
                      ocr_bbox_coordinates=i["ocr_bbox_coordinates"].to(device),
                      context_info_0={"max_features": i["ocr_max_features"].to(device)},
                      train_prev_inds=i["train_prev_inds"].to(device), targets=i["targets"].to(device),
                      train_loss_mask=i["train_loss_mask"].to(device), dataset_name=golden["dataset"], dataset_type="train")


def loss_of(out):
    (k, v), = out["losses"].items()
    assert k == "train/%s/m4c_decoding_bce_with_mask" % "textvqa"
    return v


def rel_scores(got, ref):
    """relative L2 error over the scores that are not masked: the -10000 of padded OCR tokens (and the captioner's -1e10)
    would otherwise carry the norm"""
    keep = ref > -1000.0
    return rel(got.cpu()[keep], ref[keep])


def check_train(model, golden, device, loss_tol, score_tol, grad_tol):
    g = golden["train"]
    model.train()
    out = model(sample_list(golden, device))
    worst = {"loss": abs(float(loss_of(out).detach()) - float(g["loss"])) / abs(float(g["loss"])),
             "scores": rel_scores(out["scores"], g["scores"])}
    assert worst["loss"] < loss_tol and worst["scores"] < score_tol, worst
    loss_of(out).sum().backward()
    named = dict(model.named_parameters())
    worst["grad"], checked = 0.0, 0
    for k, gr in g["grads"].items():
        if kept(gr, gr)[1].norm() <= 1e-6:
            continue
        assert named[k].grad is not None, k
        e = rel(named[k].grad.cpu(), gr)
        worst["grad"] = max(worst["grad"], e)
        assert e < grad_tol(k), (k, e)
        checked += 1
    assert checked >= 0.75 * len(g["grads"]), (checked, len(g["grads"]))
    return worst


def check_decoding(model, golden, case, device, score_tol):
    g = golden[case]
    model.eval()
    with torch.no_grad():
        out = model(sample_list(golden, device))
    e = rel_scores(out["scores"], g["scores"])
    assert e < score_tol, e
    prev = out["scores"].argmax(-1)[:, :-1].cpu()
    assert torch.equal(prev, g["prev_inds"][:, 1:])
    return e


# ---- tests ----------------------------------------------------------------------------------------------------------
def test_restated_defaults_equal_the_reference_yaml(cpu_models, golden):
    MD = cpu_models
    from mmf_b200 import m4c_model as MM
    for name in ("m4c", "m4c_captioner"):
        assert dict(MD.ConfigNode(MD.MODEL_DEFAULTS[name])) == dict(MD.ConfigNode(golden["defaults"][name])), name
    assert MD.registry.get_model_class("m4c") is MM.M4C and MD.registry.get_model_class("m4c_captioner") is MM.M4CCaptioner
    assert MM.M4C.config_path() == "configs/models/m4c/defaults.yaml"
    assert MM.M4CCaptioner.config_path() == "configs/models/m4c_captioner/defaults.yaml"
    import mmf_b200
    assert mmf_b200.M4C is MM.M4C and mmf_b200.M4CCaptioner is MM.M4CCaptioner


def test_default_config_builds_the_textvqa_model(cpu_models, golden):
    """the default YAML: bert-base text BERT with 3 layers, 4-layer 768-wide MMT, K = 3002 OCR features, 5000 answers"""
    MD = cpu_models
    from mmf_b200.registry import registry
    register(golden)
    registry.register(golden["dataset"] + "_num_final_outputs", 5050)
    m = MD.build_model(MD.load_model_config("m4c"))
    assert len(m.text_bert.encoder.layer) == 3 and m.text_bert.embeddings.word_embeddings.num_embeddings == 30522
    assert len(m.mmt.encoder.layer) == 4 and isinstance(m.text_bert_out_linear, torch.nn.Identity)
    assert m.linear_ocr_feat_to_mmt_in.in_features == 3002 and m.classifier.module.out_features == 5000
    assert [type(x).__name__ for x in m.finetune_modules] == ["dict"] * 4
    assert [d["lr_scale"] for d in m.finetune_modules] == [0.1, 0.1, 0.1, 1.0]


def test_state_dict_keys_are_the_references(cpu_models, golden):
    model = build(cpu_models, golden)
    assert sorted(model.state_dict().keys()) == golden["train"]["state_dict_keys"]
    # the fc7 encoders keep the legacy `module.` prefix of FinetuneFasterRcnnFpnFc7 checkpoints
    sd = {k.replace("obj_faster_rcnn_fc7.lc.", "obj_faster_rcnn_fc7.module.lc."): v for k, v in weights(golden).items()}
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys


def test_extended_mask_is_the_references(cpu_models, golden):
    """the encoder call's key mask plus causal tail is the reference's [B, 1, S, S] prefix-LM mask, bit for bit"""
    from mmf_b200 import m4c_model as MM
    i = golden["inputs"]
    T, R, O = i["text"].shape[1], i["image_feature_0"].shape[1], i["context_feature_0"].shape[1]
    key_mask = torch.cat([MM._get_mask(i["text_len"], T), MM._get_mask(i["obj_max_features"], R),
                          MM._get_mask(i["ocr_max_features"], O)], dim=1)
    got = MM.extended_attention_mask(key_mask, i["train_prev_inds"].shape[1])
    ref = golden["train"]["extended_mask"]
    assert got.dtype == ref.dtype and torch.equal(got, ref)
    # and the test double's causal attention reads the same mask
    S = ref.shape[-1]
    add = torch.cat([(1.0 - key_mask) * -10000.0, torch.zeros(key_mask.shape[0], S - key_mask.shape[1])], dim=1)
    q = torch.zeros(key_mask.shape[0] * S, 64, dtype=torch.bfloat16)
    with _tail(S - key_mask.shape[1]):
        s = _probs(q, q, key_mask.shape[0], 1, S, S, add)
    assert torch.equal(s[:, 0], ref[:, 0])


def test_training_step_vs_reference_golden(cpu_models, golden):
    model = build(cpu_models, golden)
    check_train(model, golden, "cpu", 2e-2, 2e-2, lambda k: 8e-2)


@pytest.mark.parametrize("case", ["eval", "captioner"])
def test_greedy_decoding_vs_reference_golden(cpu_models, golden, case):
    model = build(cpu_models, golden, captioner=case == "captioner")
    check_decoding(model, golden, case, "cpu", 2e-2)


def test_captioner_removes_unk(cpu_models, golden):
    model = build(cpu_models, golden, captioner=True).eval()
    with torch.no_grad():
        scores = model(sample_list(golden))["scores"]
    assert (scores[..., golden["unk_idx"]] == -1e10).all()


def test_optimizer_groups_are_the_references(cpu_models, golden):
    from mmf_b200.models import ConfigNode
    model = build(cpu_models, golden)
    names = {id(p): n for n, p in model.named_parameters()}
    groups = model.get_optimizer_parameters(ConfigNode({"optimizer": {"params": {"lr": 1e-4}}}))
    got = [{"names": [names[id(p)] for p in g["params"]], "lr": g.get("lr")} for g in groups]
    assert len(got) == len(golden["optimizer"])
    for a, b in zip(got, golden["optimizer"]):
        assert a["names"] == b["names"]
        assert (a["lr"] is None and b["lr"] is None) or abs(a["lr"] - b["lr"]) < 1e-12


def test_loss_formula_and_all_zero_mask(cpu_models, golden):
    from mmf_b200.models import LOSSES
    fn = LOSSES["m4c_decoding_bce_with_mask"]
    g = torch.Generator().manual_seed(5)
    scores, targets = torch.randn(3, 4, 7, generator=g), (torch.rand(3, 4, 7, generator=g) < 0.3).float()
    mask = torch.tensor([[1., 1., 0., 0.], [1., 0., 0., 0.], [1., 1., 1., 1.]])
    ref = (torch.nn.functional.binary_cross_entropy_with_logits(scores, targets, reduction="none")
           * mask[..., None]).sum() / mask.sum()
    got = fn({"targets": targets, "train_loss_mask": mask}, {"scores": scores})
    assert torch.allclose(got, ref, rtol=1e-6)
    zero = fn({"targets": targets, "train_loss_mask": torch.zeros_like(mask)}, {"scores": scores})
    assert float(zero) == 0.0 == float(golden["train"]["loss_zero_mask"])


def test_update_registry_for_pretrained(cpu_models, golden):
    from mmf_b200 import m4c_model as MM
    from mmf_b200.models import ConfigNode
    from mmf_b200.registry import registry
    MM.M4C.update_registry_for_pretrained(ConfigNode({"classifier": {"ocr_max_num": 50}}),
                                          {"classifier.module.weight": torch.zeros(5000, 8)},
                                          {"full_config": ConfigNode({"datasets": "stvqa,textvqa"})})
    assert registry.get("config").datasets == "stvqa,textvqa"
    assert registry.get("stvqa_num_final_outputs") == 5050 and registry.get("stvqa_answer_processor").BOS_IDX == 1


def test_causal_tail_takes_the_dense_path_with_skip_padding(cpu_models, monkeypatch):
    """skip_padding is set, the mask pads keys, and still the call with a tail runs dense attention (packing a tail is not
    supported) - and asking for probabilities with a tail raises"""
    import mmf_b200.engine as E
    import mmf_b200.modules as M
    from mmf_b200.models import ConfigNode, BERT_BASE
    cfg = ConfigNode(dict(BERT_BASE, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=64,
                          hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, skip_padding=True))
    enc = M.B200BertEncoder(cfg)
    calls = []
    fake = E.F
    monkeypatch.setattr(fake, "attention_varlen_fwd", lambda *a, **k: calls.append("varlen"), raising=False)
    orig = fake.attention_fwd

    def dense(*a, **k):
        calls.append(("dense", k.get("causal_len", 0)))
        return orig(*a, **k)
    monkeypatch.setattr(fake, "attention_fwd", dense)
    x = torch.randn(2, 6, 64)
    mask = torch.zeros(2, 6)
    mask[0, 2:4] = -10000.0
    out = M.run_bert_encoder(enc._runner, x, mask, False, causal_len=2)
    assert calls == [("dense", 2)] and out[0].shape == (2, 6, 64)
    with pytest.raises(ValueError, match="causal tail"):
        M.run_bert_encoder(enc._runner, x, mask, False, output_attentions=True, causal_len=2)
    with pytest.raises(ValueError, match="causal_len"):
        M.run_bert_encoder(enc._runner, x, mask, False, causal_len=7)
