#!/usr/bin/env python
"""TEST INFRASTRUCTURE - writes tests/golden/vinvl_model.pt by running the REFERENCE's registered VinVL model.

Needs the reference tree (MMF_REFERENCE_ROOT, see oracle/ref_loader.py):   python tools/make_golden_vinvl_model.py
It needs a full checkout: the head files are not among those oracle/build_ref.py stages.  It writes that one fixture and
nothing else.  Storage and gradient sampling are oracle/make_golden.py's.

The reference's `VinVL` (mmf/models/vinvl.py:392-505), `VinVLForClassification`, `VinVLForPretraining` and its
transformer heads (mmf/models/transformers/heads/{mlp,mlm,contrastive}.py) run here with stand-ins for what needs a
network or MMF's runtime: BertConfig.from_pretrained returns the small config below; the encoder is the reference's
BertEncoderJit (what replace_with_jit() installs; transformers 5's BertEncoder no longer returns hidden states itself);
`retry_n` calls once; OmegaConf / open_dict are shimmed; BaseTransformerHead is its three-line constructor; SampleList is
a dict.

Cases (B = 4, T = 8 tokens, R = 6 regions x 46 features - 46 = 6 mod 8 like 2054 -, hidden 128 / 2 heads / 2 layers,
vocab 50, eval, dropout 0; padded text and regions):
  classification     - heads.mlp with 7 labels and one transform layer, ce_loss ignore_index -1 with one ignored label;
                       max_features of shape [B]
  pretraining        - masked LM + three-way contrastive; max_features [B, R] float, as the reference's own test passes;
                       the corrupt captions have their own padding.  Also each loss's own gradients for a few trunk
                       parameters: the two trunk passes' shares, whose sum is the total
  pretraining_no_mlm - every MLM label -1 (masked_lm_loss 0, the contrastive loss still trains); no max_features
Each: scores (classification) or losses, the attention masks the reference built, sampled 2-D gradients, the reference's
state-dict keys.  Plus the reference's _get_attention_mask for each max_features form.
"""
import contextlib
import dataclasses
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden as MG  # noqa: E402
from oracle import ref_loader as R  # noqa: E402

B, T, RR, FEAT, VOCAB, NUM_LABELS, HID = 4, 8, 6, 46, 50, 7, 128
HEADS = "mmf/models/transformers/heads/"
SPLIT_PARAMS = ("vinvl.bert.embeddings.word_embeddings.weight", "vinvl.bert.img_embedding.0.weight",
                "vinvl.bert.encoder.layer.0.attention.self.query.weight", "vinvl.bert.encoder.layer.1.output.dense.weight")


class Cfg(dict):
    """attribute-access dict: what the reference's classes get instead of a DictConfig"""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v

    def __deepcopy__(self, memo):
        import copy
        return Cfg({k: copy.deepcopy(v, memo) for k, v in self.items()})


class _OmegaConf:
    @staticmethod
    def create(d):
        return Cfg(d)


def bert_overrides():
    return dict(hidden_size=HID, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256, vocab_size=VOCAB,
                max_position_embeddings=32, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


def model_config(case):
    cfg = dict(random_init=True, bert_model_name="bert-base-uncased", img_feature_dim=FEAT, use_img_layernorm=True,
               img_layer_norm_eps=1e-12, bert_overrides=bert_overrides(), do_pretraining=case != "classification")
    if case == "classification":
        cfg.update(heads=dict(mlp=dict(type="mlp", num_labels=NUM_LABELS, hidden_size=HID, hidden_dropout_prob=0.0)),
                   ce_loss=dict(ignore_index=-1))
    else:
        cfg.update(heads=dict(mlm=dict(type="mlm", vocab_size=VOCAB, hidden_size=HID, hidden_dropout_prob=0.0),
                              contrast=dict(hidden_size=HID, hidden_dropout_prob=0.0)))
    return cfg


def inputs():
    g = torch.Generator().manual_seed(1711)
    ids = torch.randint(1, VOCAB, (B, T), generator=g)
    ids_masked, ids_corrupt = ids.clone(), torch.randint(1, VOCAB, (B, T), generator=g)
    labels = torch.full((B, T), -1, dtype=torch.long)
    for b, t in ((0, 2), (1, 4), (2, 1), (2, 5), (3, 3)):
        labels[b, t] = ids[b, t]
        ids_masked[b, t] = 3
    mask = torch.ones(B, T, dtype=torch.long)
    mask[1, 6:] = 0
    mask[3, 5:] = 0
    mask_corrupt = torch.ones(B, T, dtype=torch.long)
    mask_corrupt[0, 4:] = 0
    mask_corrupt[2, 7:] = 0
    segment = torch.zeros(B, T, dtype=torch.long)
    segment[:, 5:] = 1
    feats = torch.randn(B, RR, FEAT, generator=g)
    maxf = torch.tensor([6, 2, 5, 4])
    return dict(ids=ids, ids_masked=ids_masked, ids_corrupt=ids_corrupt, lm_label_ids=labels, mask=mask,
                mask_corrupt=mask_corrupt, segment=segment, segment_corrupt=torch.zeros(B, T, dtype=torch.long),
                feats=feats, max_features=maxf, max_features_2d=maxf.float().unsqueeze(1).expand(B, RR).clone(),
                contrastive_labels=torch.tensor([[0], [1], [2], [1]]), labels=torch.tensor([[3], [-1], [0], [6]]))


def image_info(i, form):
    if form == "absent":
        return {}
    return {"max_features": (i["max_features"] if form == "1d" else i["max_features_2d"]).clone()}


def sample_list(i, form, no_mlm=False):
    return Cfg(input_ids=i["ids"].clone(), input_ids_masked=i["ids_masked"].clone(), input_ids_corrupt=i["ids_corrupt"].clone(),
               lm_label_ids=torch.full_like(i["lm_label_ids"], -1) if no_mlm else i["lm_label_ids"].clone(),
               input_mask=i["mask"].clone(), input_mask_corrupt=i["mask_corrupt"].clone(), segment_ids=i["segment"].clone(),
               segment_ids_corrupt=i["segment_corrupt"].clone(), image_feature_0=i["feats"].clone(),
               image_info_0=image_info(i, form), contrastive_labels=i["contrastive_labels"].clone(),
               labels=i["labels"].clone(), dataset_name="test", dataset_type="train")


def _ref_vinvl():
    from transformers import BertConfig
    R._install()
    base = types.ModuleType("mmf.models.transformers.base")

    class BaseTransformerHead(torch.nn.Module):          # mmf/models/transformers/base.py:380-399
        @dataclasses.dataclass
        class Config:
            type: str = "base"
            freeze: bool = False
            lr_multiplier: float = 1.0

        def __init__(self, config, *args, **kwargs):
            super().__init__()
            self.config = Cfg({**dataclasses.asdict(self.Config()), **config})

    base.BaseTransformerHead = BaseTransformerHead
    sys.modules[base.__name__] = base
    R._REAL[base.__name__] = base
    mods = {n: R.load(HEADS + n + ".py", "mmf.models.transformers.heads." + n) for n in ("mlp", "mlm", "contrastive")}
    mods["mlp"].OmegaConf = _OmegaConf
    mods["mlp"].open_dict = lambda cfg: contextlib.nullcontext()
    hl = R.hf_layers()
    vv = R.vinvl()
    vv.OmegaConf = _OmegaConf
    vv.SampleList = Cfg
    vv.retry_n = lambda n, fn, *a, **k: fn(*a, **k)
    vv.BertConfig = type("BertConfig", (BertConfig,), {
        "from_pretrained": classmethod(lambda cls, name, **kw: BertConfig(**dict(bert_overrides(), **kw)))})
    return vv, hl


def _build(vv, case, seed):
    cfg = model_config(case)
    m = MG._new_base_model(vv.VinVL, Cfg({**dataclasses.asdict(vv.VinVL.Config()), **cfg}))   # VinVL.__init__ (:421-424)
    m.do_pretraining = m.config.do_pretraining
    m.build()
    m.eval()
    g = torch.Generator().manual_seed(seed)
    ln = {id(mod.weight) for mod in m.modules() if isinstance(mod, torch.nn.LayerNorm)}
    with torch.no_grad():                               # normal(0, 0.02), LayerNorm weights around 1, on the int8 grid
        for _, p in m.named_parameters():
            base = 1.0 if id(p) in ln else 0.0
            p.copy_(MG._q8(base + torch.randn(p.shape, generator=g) * 0.02, base))
    return m


def _grads_2d(m):
    return MG._grads(m, [n for n, p in m.named_parameters() if p.grad is not None and p.dim() == 2])


def _run(m, sl):
    """the registered forward, with the attention masks it built captured on the way into the trunk"""
    masks = []
    hook = m.vinvl.bert.register_forward_pre_hook(lambda mod, a, kw: masks.append(kw["attention_mask"].clone()),
                                                  with_kwargs=True)
    try:
        return m.forward(sl), masks
    finally:
        hook.remove()


def golden_vinvl_model():
    vv, hl = _ref_vinvl()
    import mmf_b200.models as MD
    mmf_root = os.path.join(R.REF_ROOT, "mmf")
    doc = MD.read_yaml_with_includes(os.path.join(mmf_root, "configs/models/vinvl/defaults.yaml"), mmf_root)
    i = inputs()
    out = {"defaults": _plain(MD._resolve_interpolations(doc["model_config"]["vinvl"], doc)), "inputs": i,
           "config_defaults": {k: v for k, v in dataclasses.asdict(vv.VinVL.Config()).items() if k != "heads"}}   # MISSING
    hl.replace_with_jit()
    try:
        m = _build(vv, "pretraining", 1721)
        out["masks"] = {form: m._get_attention_mask(i["feats"], image_info(i, form), i["mask"])
                        for form in ("absent", "1d", "2d")}
        out["pretraining_state_dict"] = {k: v.detach().clone() for k, v in m.state_dict().items()}
        for case, form, no_mlm in (("pretraining", "2d", False), ("pretraining_no_mlm", "absent", True)):
            m.zero_grad(set_to_none=True)
            o, masks = _run(m, sample_list(i, form, no_mlm))
            sum(o["losses"].values()).backward()
            out[case] = {"config": model_config("pretraining"), "state_dict_keys": sorted(m.state_dict().keys()),
                         "losses": {k: v.detach().clone() for k, v in o["losses"].items()},
                         "attention_masks": masks, "grads": _grads_2d(m)}
            if case == "pretraining":
                named, out[case]["by_loss"] = dict(m.named_parameters()), {}
                for k in o["losses"]:
                    m.zero_grad(set_to_none=True)
                    o1, _ = _run(m, sample_list(i, form, no_mlm))
                    o1["losses"][k].backward()
                    out[case]["by_loss"][k] = {"grads": {n: named[n].grad.detach().clone() for n in SPLIT_PARAMS}}

        trunk = {k: v for k, v in out["pretraining_state_dict"].items() if k.startswith("vinvl.bert.")}
        m = _build(vv, "classification", 1722)
        m.load_state_dict(trunk, strict=False)
        o, masks = _run(m, sample_list(i, "1d"))
        sum(o["losses"].values()).backward()
        sd = m.state_dict()
        out["classification"] = {"config": model_config("classification"), "state_dict_keys": sorted(sd.keys()),
                                 "head_state_dict": {k: v.detach().clone() for k, v in sd.items() if k not in trunk},
                                 "scores": o["scores"].detach().clone(),
                                 "losses": {k: v.detach().clone() for k, v in o["losses"].items()},
                                 "attention_masks": masks, "grads": _grads_2d(m)}
    finally:
        hl.undo_replace_with_jit()
    MG._save("vinvl_model", out)


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)
    golden_vinvl_model()
