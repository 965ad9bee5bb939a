"""The registered `lxmert` model on the H100 (through the C ABI):
* against the REFERENCE's own registered LXMERT (tests/golden/lxmert_model.pt): pretraining losses, classification and
  nlvr2 scores, every stored 2-D parameter gradient;
* at the reference's default depth and widths (l/r/x = 9/5/5, 768/12h/3072, 20 tokens + 36 regions x 2048, B = 16): the
  four pretraining losses and trunk-weight gradients no worse than the same arithmetic (oracle/fusion_oracle.py) run in
  bf16, measured against it in fp32 - the rule of tests/test_depth_gpu.py;
* a training step with dropout, and the refusal of two-stream skip-padding by the registered model."""
import os

import pytest
import torch
from oracle import fusion_oracle as O
from oracle.golden_format import kept  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def rel(a, b):
    a, b = kept(a, b)        # a sampled golden gradient: compare the elements it stores
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "lxmert_model.pt"), weights_only=False)


def _ref_keys(keys):
    return {k for k in keys if not k.endswith("position_ids") and not k.endswith("token_type_ids")}


def _build(golden, case, **over):
    from mmf_b200 import models as MD
    cfg_dict = golden["pretraining_config"] if case.startswith("pretraining") else golden[case]["config"]
    cfg = MD.load_model_config("lxmert", overrides=dict(cfg_dict, **over))
    cfg.losses = [{"type": "logit_bce" if case == "classification" else "cross_entropy"}]
    model = MD.build_model(cfg)
    sd = dict(golden["pretraining_state_dict"])
    if not case.startswith("pretraining"):
        sd = {k: v for k, v in sd.items() if k.startswith("model.bert.")}
        sd.update(golden[case]["head_state_dict"])
    model.load_state_dict({k: v for k, v in sd.items() if k in _ref_keys(sd)})
    return model.to(DEV).eval()


def _sample_list(golden, case):
    from mmf_b200.sample import SampleList
    i = golden["inputs"]
    name, targets = {"pretraining_masked_vqa2": ("masked_vqa2", i["vqa_targets"]),
                     "pretraining_masked_gqa": ("masked_gqa", i["gqa_targets"]),
                     "classification": ("vqa2", i["vqa_targets"]), "nlvr2": ("nlvr2", i["nlvr2_targets"])}[case]
    return SampleList(input_ids=i["ids"].to(DEV), input_mask=i["mask"].to(DEV), segment_ids=i["seg"].to(DEV),
                      lm_label_ids=i["lm_label_ids"].to(DEV), image_feature_0=i["feats"].to(DEV),
                      image_info_0={"max_features": i["max_features"].to(DEV), "bbox": i["bbox"].to(DEV),
                                    "cls_prob": i["cls_prob"].numpy().copy()},
                      image_labels=i["image_labels"].to(DEV), targets=targets.to(DEV), is_correct=i["is_correct"].to(DEV),
                      dataset_name=name, dataset_type="train")


@pytest.mark.parametrize("case", ["pretraining_masked_vqa2", "pretraining_masked_gqa", "classification", "nlvr2"])
def test_lxmert_registered_model_vs_reference_golden(golden, case):
    from mmf_b200 import lib
    model = _build(golden, case)
    g = golden[case]
    n0 = lib.launch_count()
    out = model(_sample_list(golden, case))
    assert lib.launch_count() > n0
    if case.startswith("pretraining"):
        assert list(out["losses"].keys()) == list(g["losses"].keys())
        errs = {k: abs(float(out["losses"][k].detach()) - float(v)) / max(1.0, abs(float(v))) for k, v in g["losses"].items()}
        print(case, "loss errors", {k.split("/")[-1]: "%.2e" % e for k, e in errs.items()})
        assert max(errs.values()) < 1e-2, errs
        loss = sum(out["losses"].values())
    else:
        e = rel(out["scores"], g["scores"])
        print(case, "scores rel %.2e" % e)
        assert e < 1.5e-2
        loss = sum(v.sum() for v in out["losses"].values())
    loss.backward()
    named = dict(model.named_parameters())
    num = den = 0.0
    for k, gr in g["grads"].items():
        a, b = kept(named[k].grad.detach().double().cpu(), gr.double())
        num, den = num + float((a - b).pow(2).sum()), den + float(b.pow(2).sum())
    total = (num / den) ** 0.5
    print(case, "all stored 2-D parameter gradients: rel %.2e over %d parameters" % (total, len(g["grads"])))
    assert total < 3e-2


# ---------------------------------------------------------------------------------------------------------------------
# full depth at the reference's default shape
# ---------------------------------------------------------------------------------------------------------------------
L_LAYERS, R_LAYERS, X_LAYERS, H, HEADS, T, R, B, FEAT, NCLS = 9, 5, 5, 768, 12, 20, 36, 16, 2048, 1600


def _depth_inputs():
    g = torch.Generator().manual_seed(905)
    ids = torch.randint(1, 30522, (B, T), generator=g)
    lens = torch.randint(T // 2, T + 1, (B,), generator=g)
    mask = (torch.arange(T)[None] < lens[:, None]).long()
    seg = ((torch.arange(T)[None] >= lens[:, None] // 2) & (mask == 1)).long()      # a second segment: keys the swap keeps
    labels = torch.full((B, T), -1, dtype=torch.long)
    pick = torch.rand(B, T, generator=g) < 0.15
    labels[pick & (mask == 1)] = torch.randint(0, 30522, (B, T), generator=g)[pick & (mask == 1)]
    labels[0, 1] = 5
    feats = torch.randn(B, R, FEAT, generator=g).abs().to(torch.bfloat16).float()     # the kernels read bf16
    bbox = torch.rand(B, R, 4, generator=g)
    maxf = torch.randint(R // 2, R + 1, (B,), generator=g)
    image_labels = (torch.rand(B, R, generator=g) < 0.15).long()
    cls_prob = torch.softmax(torch.randn(B, R, NCLS, generator=g) * 3.0, dim=-1)
    targets = torch.softmax(torch.randn(B, 3129, generator=g) * 3.0, dim=-1)
    is_correct = torch.randint(0, 2, (B,), generator=g)
    return dict(ids=ids, mask=mask, seg=seg, labels=labels, feats=feats, bbox=bbox, maxf=maxf, image_labels=image_labels,
                cls_prob=cls_prob, targets=targets, is_correct=is_correct)


def _oracle_losses(sd, i, cfg, dtype):
    """LXMERTForPretraining's losses (lxmert.py:496-572) over LXMERTBase (:349-414) with the registered model's argument
    swap (input_mask as token types, segment ids as the text mask); logits in `dtype`, losses in fp32"""
    f32 = torch.float32
    emb = O.bert_embeddings(i["ids"], i["mask"], sd, "model.bert.embeddings")
    lmask = O.extended_attention_mask(i["seg"], dtype)
    vmask = O.extended_attention_mask((torch.arange(R, device=DEV)[None] < i["maxf"][:, None]).long(), dtype)
    lang, visn = O.lxmert_encoder(emb, lmask, i["feats"].to(dtype), i["bbox"].to(dtype), vmask, sd, "model.bert.encoder",
                                  L_LAYERS, X_LAYERS, R_LAYERS, HEADS)
    pooled = O.bert_pooler(lang, sd, "model.bert.pooler")
    scores, rel_score = O.bert_pretraining_heads(lang, pooled, sd, "model.cls")
    out = {"masked_lm_loss": O.masked_lm_loss(scores.to(f32), i["labels"]),
           "matched_loss": torch.nn.functional.cross_entropy(rel_score.to(f32), i["is_correct"])}
    p = "model.obj_predict_head"
    h = O.layer_norm(O.gelu_erf(O.linear(visn, sd, p + ".transform.dense")), sd, p + ".transform.LayerNorm")
    top = i["cls_prob"].max(-1)
    obj = torch.nn.functional.cross_entropy(O.linear(h, sd, p + ".decoder_dict.obj").to(f32).reshape(-1, cfg.visual_loss_config.obj[0]),
                                            top.indices.reshape(-1), reduction="none")
    feat = torch.nn.functional.smooth_l1_loss(O.linear(h, sd, p + ".decoder_dict.feat").to(f32).reshape(-1, FEAT),
                                              i["feats"].reshape(-1, FEAT), reduction="none").mean(1)
    out["visn_loss"] = ((obj * top.values.reshape(-1)).mean() * 6.67
                        + (feat * (i["image_labels"] == 1).float().reshape(-1)).mean() * 6.67)
    a = "model.answer_head.logit_fc"
    ans = O.linear(O.layer_norm(O.gelu_erf(O.linear(pooled, sd, a + ".0")), sd, a + ".2"), sd, a + ".3")
    out["answer_loss"] = torch.nn.functional.cross_entropy(ans.to(f32), i["targets"].argmax(-1))
    return out


def test_full_depth_lxmert_pretraining_no_worse_than_bf16_reference():
    from mmf_b200 import models as MD
    from mmf_b200.sample import SampleList
    torch.manual_seed(41)
    cfg = MD.load_model_config("lxmert", overrides={"hidden_dropout_prob": 0.0, "attention_probs_dropout_prob": 0.0})
    model = MD.build_model(cfg).to(DEV).eval()
    with torch.no_grad():                       # non-trivial biases / LayerNorm parameters
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.02)
    i = {k: v.to(DEV) for k, v in _depth_inputs().items()}
    sl = SampleList(input_ids=i["ids"], input_mask=i["mask"], segment_ids=i["seg"], lm_label_ids=i["labels"],
                    image_feature_0=i["feats"], image_info_0={"max_features": i["maxf"], "bbox": i["bbox"],
                                                              "cls_prob": i["cls_prob"]},
                    image_labels=i["image_labels"], targets=i["targets"], is_correct=i["is_correct"],
                    dataset_name="masked_vqa2", dataset_type="train")
    out = model(sl)
    losses = {k.split("/")[-1]: v for k, v in out["losses"].items()}
    sum(losses.values()).backward()
    named = dict(model.named_parameters())
    sd = {k: v.detach().to(torch.bfloat16).float() for k, v in model.state_dict().items()}
    sd["model.cls.predictions.decoder.weight"] = sd["model.bert.embeddings.word_embeddings.weight"]

    def run(dtype):
        sdc = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()
               if k != "model.cls.predictions.decoder.weight"}
        sdc["model.cls.predictions.decoder.weight"] = sdc["model.bert.embeddings.word_embeddings.weight"]
        ls = _oracle_losses(sdc, i, cfg, dtype)
        sum(ls.values()).backward()
        return {k: v.detach().float() for k, v in ls.items()}, {k: v.grad.float() for k, v in sdc.items() if v.grad is not None}
    f_l, f_g = run(torch.float32)
    b_l, b_g = run(torch.bfloat16)
    pre = "model.bert.encoder."
    probes = [pre + n for n in ("layer.0.attention.self.query.weight", "layer.%d.output.dense.weight" % (L_LAYERS - 1),
                                "r_layers.0.intermediate.dense.weight", "x_layers.0.visual_attention.att.key.weight",
                                "x_layers.%d.lang_output.dense.weight" % (X_LAYERS - 1),
                                "x_layers.%d.visn_inter.dense.weight" % (X_LAYERS // 2), "visn_fc.visn_fc.weight")]
    ours, drift = {}, {}
    for k in f_l:
        ours[k] = abs(float(losses[k].detach()) - float(f_l[k])) / abs(float(f_l[k]))
        drift[k] = abs(float(b_l[k]) - float(f_l[k])) / abs(float(f_l[k]))
    for n in probes:
        ours[n], drift[n] = rel(named[n].grad, f_g[n]), rel(b_g[n], f_g[n])
    print("LXMERT 9/5/5 pretraining (B=%d, T=%d, R=%d): product vs fp32 oracle / bf16-reference drift: %s" % (
        B, T, R, " ".join("%s=%.2e/%.2e" % (k.replace(pre, ""), ours[k], drift[k]) for k in ours)))
    for k in f_l:
        assert ours[k] < 2.5e-2, (k, ours[k])
    for k in ours:
        assert ours[k] <= 1.5 * drift[k] + 2e-3, (k, ours[k], drift[k])


def test_train_step_with_dropout_is_finite(golden):
    model = _build(golden, "pretraining_masked_vqa2", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1).train()
    out = model(_sample_list(golden, "pretraining_masked_vqa2"))
    assert len(out["losses"]) == 4 and all(torch.isfinite(v).all() for v in out["losses"].values())
    sum(out["losses"].values()).backward()
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert len(grads) > 100 and all(torch.isfinite(g).all() for g in grads)


def test_skip_padding_refused_by_registered_model_and_kept_by_the_trunk(golden):
    from mmf_b200.patch import set_skip_padding
    model = _build(golden, "pretraining_masked_vqa2")
    assert set_skip_padding(model, two_stream=True) == 1
    with pytest.raises(ValueError, match="swap"):
        model(_sample_list(golden, "pretraining_masked_vqa2"))
    # the trunk with real masks (padding in both streams, every sample with tokens in both) runs the packed path: its
    # outputs are exact zeros at padded rows
    i = golden["inputs"]
    vmask = (torch.arange(i["feats"].shape[1])[None] < i["max_features"][:, None]).long()
    (lang, visn), pooled = model.model.bert(i["ids"].to(DEV), None, i["mask"].to(DEV), i["feats"].to(DEV),
                                            i["bbox"][:, :i["feats"].shape[1], :4].to(DEV), vmask.to(DEV))
    assert bool((lang[i["mask"].to(DEV) == 0] == 0).all()) and bool((visn[vmask.to(DEV) == 0] == 0).all())
    assert bool((lang[i["mask"].to(DEV) == 1].abs().sum(-1) > 0).all()) and torch.isfinite(pooled).all()
    set_skip_padding(model, False, two_stream=True)
    (lang_d, _), _ = model.model.bert(i["ids"].to(DEV), None, i["mask"].to(DEV), i["feats"].to(DEV),
                                      i["bbox"][:, :i["feats"].shape[1], :4].to(DEV), vmask.to(DEV))
    assert bool((lang_d[i["mask"].to(DEV) == 0] != 0).any())
    m = i["mask"].to(DEV) == 1
    assert rel(lang[m], lang_d[m]) < 2e-2
