#!/usr/bin/env python
"""TEST INFRASTRUCTURE - writes tests/golden/lxmert_model.pt by running the REFERENCE's registered LXMERT model.

Needs the reference tree (MMF_REFERENCE_ROOT, see oracle/ref_loader.py):   python tools/make_golden_lxmert_model.py
It writes that one fixture and nothing else.  Storage, weight grid and gradient sampling are oracle/make_golden.py's.

The reference's `LXMERT` (mmf/models/lxmert.py:647-786) runs here with four stand-ins for what needs a network or MMF's
runtime: LXMERTBase.from_pretrained builds `cls(config)`; LXMERTBase.init_weights is a no-op (transformers 5 needs the
post_init() bookkeeping the <= 4.10-era class never did; weights are set explicitly below); `OmegaConf` and
`get_mmf_cache_dir` are shimmed; `registry.get("config").training.device` is "cpu".  The encoder runs under the
reference's replace_with_jit(), as its constructors install it.

Cases (B = 4, H = 64, one head, l/x/r = 2/2/1, 40 feature dims, 17 region classes, eval mode):
  pretraining       - the four losses, dataset "masked_vqa2" (answer head `logit_fc`), then "masked_gqa" (`logit_gqa`)
  classification    - vqa2 scores, loss logit_bce as projects/lxmert/configs/vqa2/defaults.yaml configures it
  nlvr2             - pooled output viewed as [B/2, 2H], num_labels = 2, cross_entropy
"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden as MG  # noqa: E402
from oracle import ref_loader as R  # noqa: E402

B, T, RR, FEAT, NCLS, VOCAB, NUM_LABELS, GQA_LABELS = 4, 8, 6, 40, 17, 50, 7, 5


def model_config(head, num_labels=NUM_LABELS):
    return dict(
        bert_model_name=None, training_head_type=head, random_initialize=True, num_labels=num_labels,
        gqa_labels=GQA_LABELS, num_hidden_layers=3, num_attention_heads=1, intermediate_size=128, hidden_size=64,
        hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, max_position_embeddings=32,
        type_vocab_size=2, initializer_range=0.02, pad_token_id=0, layer_norm_eps=1e-12, mode="lxr", l_layers=2,
        x_layers=2, r_layers=1, visual_feat_dim=FEAT, visual_pos_dim=4, task_matched=True, task_mask_lm=True,
        task_obj_predict=True, task_qa=True, visual_losses=["obj", "feat"],
        visual_loss_config={"obj": [NCLS, "ce", [-1], 6.67], "attr": [11, "ce", [-1], 6.67],
                            "feat": [FEAT, "l2", [-1, FEAT], 6.67]},
        freeze_base=False, vocab_size=VOCAB)


def inputs():
    g = torch.Generator().manual_seed(711)
    ids = torch.randint(1, VOCAB, (B, T), generator=g)
    mask = torch.ones(B, T, dtype=torch.long)
    mask[1, 6:] = 0
    mask[3, 4:] = 0
    seg = torch.zeros(B, T, dtype=torch.long)       # non-zero segment ids: the reference uses them as the attention mask
    seg[0, 3:6] = 1
    seg[2, 1:] = 1
    labels = torch.full((B, T), -1, dtype=torch.long)
    labels[0, 2], labels[1, 4], labels[2, 1], labels[2, 6] = 7, 11, 3, 40
    feats = torch.randn(B, RR, FEAT, generator=g).abs()
    bbox = torch.rand(B, RR + 2, 5, generator=g)    # more rows and columns than the model reads: [:, :R, :4]
    maxf = torch.tensor([6, 2, 5, 4])
    image_labels = torch.tensor([[1, 0, 0, 1, 0, -1, 1, 1], [0, 1, 0, 0, 0, 1, 0, 0], [0, 0, 0, 0, 1, 1, 0, 0],
                                 [1, 1, 0, -1, 0, 0, 1, 0]])
    cls_prob = torch.softmax(torch.randn(B, RR + 1, NCLS, generator=g) * 2.0, dim=-1)
    vqa_targets = torch.softmax(torch.randn(B, NUM_LABELS, generator=g) * 3.0, dim=-1)
    gqa_targets = torch.softmax(torch.randn(B, GQA_LABELS, generator=g) * 3.0, dim=-1)
    is_correct = torch.tensor([1, 0, 1, 1])
    nlvr2_targets = torch.tensor([1, 0])
    return dict(ids=ids, mask=mask, seg=seg, lm_label_ids=labels, feats=feats, bbox=bbox, max_features=maxf,
                image_labels=image_labels, cls_prob=cls_prob, vqa_targets=vqa_targets, gqa_targets=gqa_targets,
                is_correct=is_correct, nlvr2_targets=nlvr2_targets)


def sample_list(i, dataset_name, targets):
    return MG._Cfg(input_ids=i["ids"].clone(), input_mask=i["mask"].clone(), segment_ids=i["seg"].clone(),
                   lm_label_ids=i["lm_label_ids"].clone(), image_feature_0=i["feats"].clone(),
                   image_info_0=MG._Cfg(max_features=i["max_features"].clone(), bbox=i["bbox"].clone(),
                                        cls_prob=i["cls_prob"].numpy().copy()),
                   image_labels=i["image_labels"].clone(), targets=targets.clone(), is_correct=i["is_correct"].clone(),
                   dataset_name=dataset_name, dataset_type="train")


def _ref_lxmert():
    R._install()
    hl = R.hf_layers()
    lx = R.lxmert()
    lx.OmegaConf = MG._OmegaConfShim
    lx.get_mmf_cache_dir = lambda: "/tmp"
    lx.LXMERTBase.init_weights = lambda self: None
    lx.LXMERTBase.from_pretrained = classmethod(lambda cls, name, config=None, cache_dir=None, **kw: cls(config))
    lx.registry = types.SimpleNamespace(get=lambda key: MG._Cfg(training=MG._Cfg(device="cpu")))
    return hl, lx


def _recorder(m):
    """what the reference's model hands its head model: the plumbing's integer tensors, checked with torch.equal"""
    seen = {}
    inner = m.model.forward

    def fwd(**kw):
        for k in ("token_type_ids", "attention_mask", "visual_pos", "visual_attention_mask", "masked_image_labels",
                  "obj_labels"):
            if kw.get(k) is not None:
                seen[k] = kw[k].detach().clone()
        if kw.get("obj_labels") is not None:
            top = kw["obj_labels"].max(-1)
            seen["obj_index"], seen["obj_conf"] = top.indices.clone(), top.values.detach().clone()
        if kw.get("masked_image_labels") is not None:
            seen["feat_mask"] = (kw["masked_image_labels"] == 1).float()
        return inner(**kw)
    m.model.forward = fwd
    return seen


# gradients stored of the classification cases (the pretraining case stores every 2-D one): the classifier and a path
# through the trunk - the fixture stays under 1 MB
CLS_GRADS = ("classifier.", "pooler.", "x_layers.1.", "r_layers.0.attention", "layer.0.intermediate", "visn_fc.visn_fc",
             "word_embeddings")


def _grads_2d(m, parts=None):
    """gradients of the 2-D parameters (all of them, or those whose name contains one of `parts`)"""
    return MG._grads(m, [n for n, p in m.named_parameters() if p.grad is not None and p.dim() == 2 and (
        parts is None or any(s in n for s in parts))])


def _build(lx, cfg, seed):
    m = MG._new_base_model(lx.LXMERT, MG._Cfg(cfg))
    m.build()
    m.eval()
    MG._perturb(m, seed)
    return m


def golden_lxmert_model():
    hl, lx = _ref_lxmert()
    import mmf_b200.models as MD
    mmf_root = os.path.join(R.REF_ROOT, "mmf")
    doc = MD.read_yaml_with_includes(os.path.join(mmf_root, "configs/models/lxmert/defaults.yaml"), mmf_root)
    defaults = MD._resolve_interpolations(doc["model_config"]["lxmert"], doc)
    i = inputs()
    out = {"defaults": _plain(defaults), "inputs": i}
    hl.replace_with_jit()
    try:
        # ---- pretraining: the same weights under a vqa and a gqa dataset name
        cfg = model_config("pretraining")
        m = _build(lx, cfg, 801)
        out["pretraining_config"] = cfg
        out["pretraining_state_dict"] = {k: v.detach().clone() for k, v in m.state_dict().items()}
        for name, targets in (("masked_vqa2", i["vqa_targets"]), ("masked_gqa", i["gqa_targets"])):
            m.zero_grad(set_to_none=True)
            seen = _recorder(m)
            o = m.forward(sample_list(i, name, targets))
            loss = sum(v for v in o["losses"].values())
            loss.backward()
            del m.model.forward
            out["pretraining_" + name] = {
                "losses": {k: v.detach().clone() for k, v in o["losses"].items()}, "plumbing": seen,
                "grads": _grads_2d(m, None if name == "masked_vqa2" else ("logit_gqa",))}
        # ---- classification (vqa2) and nlvr2: the pretraining trunk's weights, heads of their own
        trunk = {k: v for k, v in out["pretraining_state_dict"].items() if k.startswith("model.bert.")}
        for case, head, nl, targets in (("classification", "classification", NUM_LABELS, i["vqa_targets"]),
                                        ("nlvr2", "nlvr2", 2, i["nlvr2_targets"])):
            cfg = model_config(head, nl)
            m = _build(lx, cfg, 802 if case == "classification" else 803)
            m.load_state_dict(trunk, strict=False)
            seen = _recorder(m)
            o = m.forward(sample_list(i, "vqa2" if case == "classification" else "nlvr2", targets))
            scores = o["scores"]
            if case == "classification":        # logit_bce (mmf/modules/losses.py:226-251), the vqa2 YAML's loss
                loss = torch.nn.functional.binary_cross_entropy_with_logits(scores, targets) * targets.size(1)
            else:
                loss = torch.nn.functional.cross_entropy(scores, targets)
            loss.backward()
            sd = m.state_dict()
            out[case] = {"config": cfg, "state_dict_keys": sorted(sd.keys()),
                         "head_state_dict": {k: v.detach().clone() for k, v in sd.items() if k not in trunk},
                         "scores": scores.detach().clone(), "loss": loss.detach().clone(), "plumbing": seen,
                         "grads": _grads_2d(m, CLS_GRADS)}
    finally:
        hl.undo_replace_with_jit()
    MG._save("lxmert_model", out)


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)
    golden_lxmert_model()
