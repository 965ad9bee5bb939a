"""The registered `uniter` model (mmf_b200.uniter_model.UNITER) on the CPU: config handling, the SampleList plumbing, the
seeded task and region-mask draws, the five pretraining heads and the classifier run over the kernel test double
(tests/fake_kernels.py plus the double of the two optimal-transport entry points below) and are held to
tests/golden/uniter_model.pt - outputs of the REFERENCE's own registered UNITER (tools/make_golden_uniter_model.py).
The kernels themselves are covered on the GPU (tests/test_ot_gpu.py, tests/test_uniter_model_gpu.py)."""
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fake_kernels as FK  # noqa: E402
from oracle import ot_oracle as FO  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TASKS = ["mlm", "itm", "mrc", "mrfr", "wra"]
BF = torch.bfloat16


# ---- double of mmfb_ot_fwd / mmfb_ot_bwd: a torch restatement of their contract (include/mmfb200.h), strided views included
def _pads(lens, width):
    return torch.arange(width).unsqueeze(0) >= torch.as_tensor(lens).reshape(-1, 1)


def ot_fwd(x, y, x_len, y_len, beta=0.5, iterations=50, k=1, want_cost=False):
    assert x.dtype == BF and y.dtype == BF and x.stride(-1) == 1 and y.stride(-1) == 1
    B, M, H = x.shape
    N = y.shape[1]
    if M > 128 or N > 128 or H % 64 or H > 1024 or min(x_len) < 1 or min(y_len) < 1 or max(x_len) > M or max(y_len) > N:
        raise ValueError("ot_fwd: unsupported shape or length")
    xp, yp = _pads(x_len, M), _pads(y_len, N)
    xf = x.float().masked_fill(xp.unsqueeze(-1), 0.0)          # rows past the lengths are never read
    yf = y.float().masked_fill(yp.unsqueeze(-1), 0.0)
    dist, cost, plan = FO.optimal_transport_dist(xf, yf, xp, yp, beta, iterations, k, return_all=True)
    nx, ny = xf.norm(dim=-1).clamp_min(1e-5), yf.norm(dim=-1).clamp_min(1e-5)
    cos = 1.0 - cost
    saved = torch.cat([nx, ny, (plan * cos.transpose(1, 2)).sum(1), (plan * cos.transpose(1, 2)).sum(2)], dim=1)
    return (dist, plan, saved, cost) if want_cost else (dist, plan, saved)


def ot_bwd(g, plan, saved, x, y, x_len, y_len, dx, dy):
    B, M, H = x.shape
    N = y.shape[1]
    xp, yp = _pads(x_len, M), _pads(y_len, N)
    nx, ny, px, py = saved.split([M, N, M, N], dim=1)
    xh = x.float().masked_fill(xp.unsqueeze(-1), 0.0) / nx.unsqueeze(-1)
    yh = y.float().masked_fill(yp.unsqueeze(-1), 0.0) / ny.unsqueeze(-1)
    px = torch.where(nx > 1e-5, px, torch.zeros_like(px))
    py = torch.where(ny > 1e-5, py, torch.zeros_like(py))
    gg = -g.view(B, 1, 1)
    gx = gg / nx.unsqueeze(-1) * (plan.transpose(1, 2) @ yh - xh * px.unsqueeze(-1))
    gy = gg / ny.unsqueeze(-1) * (plan @ xh - yh * py.unsqueeze(-1))
    dx.copy_(gx.masked_fill(xp.unsqueeze(-1), 0.0).to(BF))       # in place, through the strided views
    dy.copy_(gy.masked_fill(yp.unsqueeze(-1), 0.0).to(BF))
    return dx, dy


class _Kernels(types.ModuleType):
    def __getattr__(self, name):
        return getattr(FK, name)


KERNELS = _Kernels("fake_kernels_with_ot")
KERNELS.ot_fwd, KERNELS.ot_bwd = ot_fwd, ot_bwd


def rel(a, b):
    a, b = kept(a, b)
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "uniter_model.pt"), weights_only=False)


@pytest.fixture()
def cpu_models(monkeypatch):
    import mmf_b200.embeddings as EM
    import mmf_b200.engine as E
    import mmf_b200.heads as HD
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    import mmf_b200.uniter as UN
    import mmf_b200.vilbert as VB
    monkeypatch.setattr(E, "F", KERNELS)
    monkeypatch.setattr(OPS, "F", KERNELS)
    monkeypatch.setattr(EM, "F", KERNELS)
    for mod in (M, EM, VB, HD, UN):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    import mmf_b200.mmft  # noqa: F401  (the head table)
    import mmf_b200.models as MD
    return MD


def _ref_keys(keys):
    # HF registers `position_ids` / `token_type_ids` buffers in BertEmbeddings, and transformers 5 lists the MLM decoder's
    # bias under `decoder.bias` as well as `predictions.bias`; aside from those the key sets are UNITER's
    return {k for k in keys if not k.endswith("position_ids") and not k.endswith("token_type_ids")
            and not k.endswith("predictions.decoder.bias")}


def _build(MD, golden, case):
    cfg = MD.load_model_config("uniter", overrides=dict(golden["vqa2"]["config"] if case == "vqa2"
                                                        else golden["pretraining_config"]))
    model = MD.build_model(cfg).eval()
    sd = dict(golden["pretraining_state_dict"])
    if case == "vqa2":
        sd = {k: v for k, v in sd.items() if k.startswith("uniter.uniter.")}
        sd.update(golden["vqa2"]["head_state_dict"])
    model.load_state_dict({k: v for k, v in sd.items() if k in _ref_keys(sd)}, strict=False)
    return model


def _sample_list(golden, case, device="cpu"):
    from mmf_b200.sample import SampleList
    i = golden["inputs"]
    return SampleList(input_ids=i["ids"].to(device), input_ids_masked=i["ids_masked"].to(device),
                      input_mask=i["mask"].to(device), lm_label_ids=i["lm_label_ids"].to(device),
                      image_feature_0=i["feats"].to(device),
                      image_info_0={"max_features": i["max_features"].to(device), "bbox": i["bbox"].numpy().copy(),
                                    "image_width": i["image_width"].numpy().copy(),
                                    "image_height": i["image_height"].numpy().copy(), "cls_prob": i["cls_prob"].numpy().copy()},
                      targets=i["targets"].to(device), is_correct=i["is_correct"].to(device),
                      dataset_name="vqa2" if case == "vqa2" else "coco", dataset_type="train")


def _seed_all(s):
    torch.manual_seed(s)
    np.random.seed(s)
    random.seed(s)


def check_plumbing(sl, ref):
    """integer paths bit for bit; the 7-d position feature and the gathered targets are fp32 arithmetic on the host"""
    for k in ("image_mask", "attention_mask", "position_ids", "input_ids", "combined_labels", "image_region_mask",
              "mrfr_region_mask"):
        if k in ref:
            got = sl["mlm_labels"][k] if k == "combined_labels" else sl[k]
            assert got.dtype == ref[k].dtype and torch.equal(got.cpu(), ref[k]), k
    for k in ("img_pos_feat", "region_class", "mrfr_region_target"):
        if k in ref:
            assert torch.allclose(sl[k].float().cpu(), ref[k], rtol=1e-6, atol=1e-7), k


def test_oracle_optimal_transport_equals_the_references(golden):
    """oracle/ot_oracle.optimal_transport_dist against the reference's own cost_matrix_cosine / ipot / trace"""
    g = golden["ot"]
    seq = g["sequence_output"]
    T, R = g["T_len"], g["R_len"]
    dist, cost, plan = FO.optimal_transport_dist(seq[:, :T], seq[:, T:T + R], g["txt_pad"], g["img_pad"], return_all=True)
    for name, got in (("cost", cost), ("T", plan), ("distance", dist)):
        assert tuple(got.shape) == tuple(g[name].shape)
        assert torch.allclose(got, g[name], rtol=1e-5, atol=1e-5 * float(g[name].abs().max())), name
    d64 = FO.optimal_transport_dist(seq[:, :T].double(), seq[:, T:T + R].double(), g["txt_pad"], g["img_pad"])
    assert torch.allclose(d64.float(), g["distance"], rtol=1e-4)


def test_kernel_double_follows_the_oracle_through_strided_views(golden):
    g = golden["ot"]
    T, R = g["T_len"], g["R_len"]
    seq = g["sequence_output"].to(BF)
    xl, yl = (~g["txt_pad"]).sum(1).tolist(), (~g["img_pad"]).sum(1).tolist()
    dist, plan, saved, cost = ot_fwd(seq[:, :T], seq[:, T:T + R], xl, yl, want_cost=True)
    assert torch.allclose(plan, g["T"], atol=1e-5 * float(g["T"].abs().max())) and torch.allclose(dist, g["distance"], rtol=1e-5)
    s64 = g["sequence_output"].double().requires_grad_(True)
    w = torch.tensor([1.0, -1.0, 2.0, 0.5])
    (FO.optimal_transport_dist(s64[:, :T], s64[:, T:T + R], g["txt_pad"], g["img_pad"]) * w.double()).sum().backward()
    dseq = torch.zeros_like(seq)
    ot_bwd(w, plan, saved, seq[:, :T], seq[:, T:T + R], xl, yl, dseq[:, :T], dseq[:, T:T + R])
    assert rel(dseq.float(), s64.grad.float()) < 5e-3
    assert (dseq[:, :T][g["txt_pad"]] == 0).all() and (dseq[:, T:T + R][g["img_pad"]] == 0).all()


def test_restated_defaults_equal_the_reference_yaml(cpu_models, golden):
    MD = cpu_models
    assert dict(MD.ConfigNode(MD.MODEL_DEFAULTS["uniter"])) == dict(MD.ConfigNode(golden["defaults"]))
    from mmf_b200.uniter_model import UNITER
    assert MD.registry.get_model_class("uniter") is UNITER
    assert UNITER.config_path() == "configs/models/uniter/defaults.yaml"
    m = MD.build_model(MD.load_model_config("uniter"))          # the reference's YAML as it stands: bert-base, vqa2 head
    assert type(m.uniter).__name__ == "B200UNITERForClassification" and m.tasks == ["vqa2"]
    assert len(m.uniter.uniter.encoder.layer) == 12 and m.uniter.heads["vqa2"].num_labels == 3129
    assert m.config.img_dim == 2048 and m.config.do_pretraining is False and not hasattr(m, "losses")


def test_default_pretraining_heads_and_tasks(cpu_models):
    from mmf_b200 import uniter_model as UM
    m = UM.B200UNITERForPretraining(mask_probability=0.15)
    assert m.tasks == TASKS and sorted(m.heads.keys()) == sorted(TASKS)
    assert m.heads["mrc"].region_classifier[3].out_features == 1601
    assert m.heads["mrfr"].linear_proj_weight is m.uniter.img_embeddings.img_linear.weight


@pytest.mark.parametrize("case", ["pretraining", "vqa2"])
def test_state_dict_keys_are_the_references(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, "mlm" if case == "pretraining" else "vqa2")
    ref = golden["pretraining_state_dict"].keys() if case == "pretraining" else golden["vqa2"]["state_dict_keys"]
    assert _ref_keys(model.state_dict().keys()) == _ref_keys(ref)
    sd = dict(golden["pretraining_state_dict"])
    if case == "vqa2":
        sd = {k: v for k, v in sd.items() if k.startswith("uniter.uniter.")}
        sd.update(golden["vqa2"]["head_state_dict"])
    res = model.load_state_dict({k: v for k, v in sd.items() if k in _ref_keys(sd)}, strict=False)
    assert not res.unexpected_keys and _ref_keys(res.missing_keys) == set()


@pytest.mark.parametrize("case", ["vqa2"] + TASKS)
def test_registered_model_vs_reference_golden(cpu_models, golden, case):
    MD = cpu_models
    model = _build(MD, golden, case)
    g = golden[case]
    sl = _sample_list(golden, case)
    _seed_all(g.get("seed", 7))
    out = model(sl)
    if case != "vqa2":
        assert sl["task"] == case                       # the seeded draw picks the reference's task ...
    check_plumbing(sl, g["plumbing"])                   # ... and, for mrc / mrfr, its region masks
    assert list(out["losses"].keys()) == list(g["losses"].keys())
    for k, v in g["losses"].items():
        got = float(out["losses"][k].detach().sum())
        assert abs(got - float(v)) < 2e-2 * abs(float(v)) + 1e-4, (k, got, float(v))
    if case == "vqa2":
        assert rel(out["scores"], g["scores"]) < 2e-2, rel(out["scores"], g["scores"])
    sum(v.sum() for v in out["losses"].values()).backward()
    named = dict(model.named_parameters())
    checked = 0
    for k, gr in g["grads"].items():
        if k.endswith("mrfr.linear_proj_weight"):       # the tied weight: named_parameters lists it once, under the trunk
            continue
        assert named[k].grad is not None, k
        if kept(gr, gr)[1].norm() > 1e-6:
            assert rel(named[k].grad, gr) < 8e-2, (k, rel(named[k].grad, gr))
            checked += 1
    assert checked >= 0.75 * (len(g["grads"]) - 1), (checked, len(g["grads"]))


def test_tied_mrfr_weight_gets_the_sum_of_both_uses(cpu_models, golden):
    MD = cpu_models
    model = _build(MD, golden, "mrfr")
    w = model.uniter.uniter.img_embeddings.img_linear.weight
    assert model.uniter.heads["mrfr"].linear_proj_weight is w
    sl = _sample_list(golden, "mrfr")
    _seed_all(golden["mrfr"]["seed"])
    loss = sum(model(sl)["losses"].values())
    tied = torch.autograd.grad(loss, w, retain_graph=True)[0]
    # the same step with the head's use cut out of the graph gives the embedding's share; the head's share is the rest
    head = model.uniter.heads["mrfr"]
    head.linear_proj_weight = torch.nn.Parameter(w.detach().clone())
    sl = _sample_list(golden, "mrfr")
    _seed_all(golden["mrfr"]["seed"])
    loss2 = sum(model(sl)["losses"].values())
    emb_share, head_share = torch.autograd.grad(loss2, [w, head.linear_proj_weight])
    assert head_share.abs().max() > 0 and emb_share.abs().max() > 0
    assert rel(tied, emb_share + head_share) < 1e-3
    assert rel(tied, golden["mrfr"]["grads"]["uniter.uniter.img_embeddings.img_linear.weight"]) < 8e-2


def test_remove_mismatched_captions_changes_nothing(cpu_models, golden):
    MD = cpu_models
    model = _build(MD, golden, "mlm")
    sl = _sample_list(golden, "mlm")
    sl["image_feat"], sl["attention_mask"] = sl["image_feature_0"], torch.ones(4, 14, dtype=torch.long)
    sl["cls_prob"] = torch.as_tensor(sl["image_info_0"]["cls_prob"])
    before = {k: v.clone() for k, v in sl.items() if torch.is_tensor(v)}
    model.uniter._remove_mismatched_captions(sl)
    assert set(k for k, v in sl.items() if torch.is_tensor(v)) == set(before)
    for k, v in before.items():
        assert torch.equal(sl[k], v), k


def test_wra_reads_lengths_from_suffix_pads_and_refuses_other_masks(cpu_models, golden):
    from mmf_b200.mmft import WRAHead
    g = golden["ot"]
    seq = g["sequence_output"]
    T, R = g["T_len"], g["R_len"]
    labels = torch.tensor([1, 0, 1, 1])
    sl = {"input_ids": torch.zeros(4, T, dtype=torch.long), "image_feat": torch.zeros(4, R, 3), "is_correct": labels,
          "wra_info": {"txt_pad": g["txt_pad"], "img_pad": g["img_pad"]}}
    loss = WRAHead()(seq, processed_sample_list=sl)["losses"]["wra_loss"]
    d = g["distance"]
    assert abs(float(loss) - float((d[labels == 1].sum() - d[labels == 0].sum()) / 4)) < 1e-3
    holes = g["txt_pad"].clone()
    holes[0, 2] = True
    sl["wra_info"] = {"txt_pad": holes, "img_pad": g["img_pad"]}
    with pytest.raises(ValueError, match="suffix"):
        WRAHead()(seq, processed_sample_list=sl)


@pytest.mark.parametrize("where", ["encoder", "text_embeddings"])
@pytest.mark.parametrize("key", ["output_attentions", "output_hidden_states"])
def test_unsupported_options_raise(cpu_models, golden, where, key):
    MD = cpu_models
    cfg = dict(golden["vqa2"]["config"])
    cfg[where] = dict(cfg[where], **{key: True})
    with pytest.raises(NotImplementedError, match=key):
        MD.build_model(MD.load_model_config("uniter", overrides=cfg))


def test_unknown_head_and_unsupported_task_raise(cpu_models, golden):
    MD = cpu_models
    cfg = dict(golden["vqa2"]["config"])
    cfg["heads"] = {"vqa2": {"type": "refiner"}}
    with pytest.raises(NotImplementedError, match="refiner"):
        MD.build_model(MD.load_model_config("uniter", overrides=cfg))
    model = _build(MD, golden, "mlm")
    sl = _sample_list(golden, "mlm")
    model.tasks = ["caption"]
    with pytest.raises(ValueError, match="not supported for pretraining"):
        model(sl)


def test_graphed_step_refuses_the_model(cpu_models, golden):
    from mmf_b200.graphs import GraphedStep
    model = _build(cpu_models, golden, "mlm")
    with pytest.raises(RuntimeError, match="cannot be captured"):
        GraphedStep(model, lambda b: None, {})
