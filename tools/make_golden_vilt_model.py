#!/usr/bin/env python
"""TEST INFRASTRUCTURE - writes tests/golden/vilt_model.pt by running the REFERENCE's registered ViLT model.

Needs the reference tree (MMF_REFERENCE_ROOT, see oracle/ref_loader.py):   python tools/make_golden_vilt_model.py
It needs a full checkout: the model and head files are not among those oracle/build_ref.py stages.  It writes that one
fixture and nothing else.  Storage and gradient sampling are oracle/make_golden.py's.

The reference's `ViLT` (mmf/models/vilt.py:118-283), its text and image embeddings, `ViTEncoder` (mmf/modules/encoders.py:
830-857) around `ViTModel` (mmf/modules/vit.py:178-335), build_heads_dict / HeadsDict (heads/utils.py) and the `mlp`,
`mlm_multi` and `itm` heads run here with stand-ins for what needs a network or MMF's runtime:
  * AutoConfig / ViTConfig.from_pretrained return the small configs below ("the hub"), overridden by the keys passed,
    as from_pretrained(name, **kw) does;
  * ViTModel.init_weights is skipped (every weight is set below) and get_head_mask returns no head mask;
  * ViTModel.get_extended_attention_mask is the pinned transformers' (<= 4.10.1) arithmetic, (1 - m) * -10000;
  * `retry_n` calls once; OmegaConf / open_dict are shimmed; BaseTransformerHead is its constructor; the registry's
    head, encoder and loss look-ups are tables of the reference's own classes; the sample list is an attribute-access
    dict (as MMF's SampleList), so the reference's getattr() mask look-up sees the masks.

Shapes: B = 4, T = 8 tokens (padded), 16 x 16 images with patch 8 (4 patches + [CLS] = 5 image positions), hidden 128 /
2 heads / 2 layers / intermediate 256, vocab 50, eval, dropout 0.  Cases:
  classification       - heads.vqa2 = [mlp] with 7 labels, logit_bce; input_mask present
  classification_nomask - the same with neither input_mask nor image_mask (the encoder gets mask None)
  pretraining          - masked_coco = [mlm_multi, itm]; input_ids_masked, lm_label_ids, is_correct given; also each
                         loss's own gradients for a few parameters (the two trunk passes' shares)
  pretraining_no_mlm   - every lm_label_ids -1 (masked_lm_loss 0)
Each: scores or losses, the masks the reference's encoder received, sampled gradients, state-dict keys and optimizer
groups (by parameter name).  Plus get_attention_mask for an attribute-access sample list, a plain dict, an image mask
alone, and no mask; and the restated defaults (the reference YAML, interpolations resolved).
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

B, T, IMG, PATCH, VOCAB, NUM_LABELS, HID = 4, 8, 16, 8, 50, 7, 128
HEADS = "mmf/models/transformers/heads/"
SPLIT_PARAMS = ("text_embeddings.text_embeddings.word_embeddings.weight",
                "image_embeddings.embedding.patch_embeddings.projection.weight",
                "encoder.module.encoder.layer.0.attention.attention.query.weight",
                "encoder.module.encoder.layer.1.output.dense.weight")

# the stand-in hub: what from_pretrained returns before the passed keys override it
SMALL_BERT = dict(hidden_size=HID, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256, vocab_size=VOCAB,
                  max_position_embeddings=32, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
SMALL_VIT = dict(hidden_size=HID, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256, image_size=IMG,
                 patch_size=PATCH, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12,
                 # PretrainedConfig fields of the pinned transformers that BertSelfAttention reads
                 is_decoder=False, chunk_size_feed_forward=0, position_embedding_type="absolute",
                 max_position_embeddings=64)


class Cfg(dict):
    """attribute-access dict: what the reference's classes get instead of a DictConfig / SampleList"""

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


def _cfg(x):
    if isinstance(x, dict):
        return Cfg({k: _cfg(v) for k, v in x.items()})
    if isinstance(x, list):
        return [_cfg(v) for v in x]
    return x


class _OmegaConf:
    @staticmethod
    def create(d):
        return Cfg(d)

    @staticmethod
    def to_container(cfg, resolve=True):
        return dict(cfg)


def model_config(case):
    """the user-level config of each case; both sides merge it over the default YAML"""
    image = dict(random_init=True, image_size=[IMG, IMG], patch_size=PATCH, hidden_size=HID, num_hidden_layers=2,
                 num_attention_heads=2, intermediate_size=256, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    text = dict(random_init=True, hidden_size=HID, max_position_embeddings=16,
                bert_overrides=dict(vocab_size=VOCAB, num_attention_heads=2, hidden_dropout_prob=0.0))
    cfg = dict(image_encoder=dict(params=image), text_embeddings=text)
    if case.startswith("classification"):
        cfg.update(tasks="vqa2", heads=dict(vqa2=[dict(type="mlp", num_layers=1, loss="vqa2_mlp", in_dim=HID,
                                                       hidden_size=2 * HID, num_labels=NUM_LABELS,
                                                       hidden_dropout_prob=0.0, pooler_name="bert_pooler")]),
                   losses=dict(vqa2_mlp="logit_bce"))
    else:
        cfg.update(tasks="masked_coco", heads=dict(masked_coco=[
            dict(type="mlm_multi", hidden_size=HID, vocab_size=VOCAB, hidden_dropout_prob=0.0),
            dict(type="itm", hidden_size=HID, label_key="is_correct")]))
    return cfg


def inputs():
    g = torch.Generator().manual_seed(1811)
    ids = torch.randint(1, VOCAB, (B, T), generator=g)
    ids_masked = ids.clone()
    labels = torch.full((B, T), -1, dtype=torch.long)
    for b, t in ((0, 2), (1, 4), (2, 1), (2, 5), (3, 3)):
        labels[b, t] = ids[b, t]
        ids_masked[b, t] = 3
    mask = torch.ones(B, T, dtype=torch.long)
    mask[1, 6:] = 0
    mask[3, 5:] = 0
    segment = torch.zeros(B, T, dtype=torch.long)
    segment[:, 5:] = 1
    targets = (torch.rand(B, NUM_LABELS, generator=g) < 0.3).float()
    return dict(ids=ids, ids_masked=ids_masked, lm_label_ids=labels, mask=mask, segment=segment,
                image=torch.randn(B, 3, IMG, IMG, generator=g), image_mask=(torch.arange(5)[None] < torch.tensor(
                    [[5], [3], [5], [4]])).long(), is_correct=torch.tensor([1, 0, 1, 1]), targets=targets)


def sample_list(i, case):
    dataset = "vqa2" if case.startswith("classification") else "masked_coco"
    sl = Cfg(input_ids=i["ids"].clone(), segment_ids=i["segment"].clone(), image=i["image"].clone(),
             dataset_name=dataset, dataset_type="train")
    if case != "classification_nomask":
        sl["input_mask"] = i["mask"].clone()
    if case.startswith("classification"):
        sl["targets"] = i["targets"].clone()
    else:
        sl.update(input_ids_masked=i["ids_masked"].clone(), is_correct=i["is_correct"].clone(),
                  lm_label_ids=torch.full_like(i["lm_label_ids"], -1) if case == "pretraining_no_mlm"
                  else i["lm_label_ids"].clone())
    return sl


def _ref_vilt():
    from transformers import BertConfig, ViTConfig
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
    heads = {n: R.load(HEADS + n + ".py", "mmf.models.transformers.heads." + n) for n in ("mlp", "mlm", "itm")}
    heads["mlp"].OmegaConf = _OmegaConf
    heads["mlp"].open_dict = lambda cfg: contextlib.nullcontext()
    head_table = {"mlp": heads["mlp"].MLP, "mlm": heads["mlm"].MLM, "mlm_multi": heads["mlm"].MLMForMultiHeads,
                  "itm": heads["itm"].ITM}
    utils = R.load(HEADS + "utils.py", "mmf.models.transformers.heads.utils")
    utils.registry = types.SimpleNamespace(get_transformer_head_class=head_table.get)

    vit = R.vit()
    vit.OmegaConf = _OmegaConf
    vit.retry_n = lambda n, fn, *a, **k: fn(*a, **k)
    vit.ViTModel.init_weights = lambda self: None
    vit.ViTModel.get_head_mask = lambda self, head_mask, n: [None] * n

    def extended_mask(self, attention_mask, input_shape, device=None):     # transformers 4.10.1, 2-D masks
        ext = attention_mask[:, None, None, :].to(dtype=self.dtype)
        return (1.0 - ext) * -10000.0
    vit.ViTModel.get_extended_attention_mask = extended_mask
    vit.vit = types.SimpleNamespace(**{k: getattr(vit.vit, k) for k in dir(vit.vit) if not k.startswith("__")})
    vit.vit.ViTConfig = type("ViTConfig", (ViTConfig,), {
        "from_pretrained": classmethod(lambda cls, _pretrained, **kw: ViTConfig(**dict(SMALL_VIT, **kw)))})

    enc = R.encoders()
    enc.OmegaConf = _OmegaConf
    enc.AutoConfig = types.SimpleNamespace(from_pretrained=lambda _pretrained, **kw: BertConfig(**dict(SMALL_BERT, **kw)))

    losses = R.load("mmf/modules/losses.py", "mmf.modules.losses")
    losses.registry = types.SimpleNamespace(get_loss_class={"logit_bce": losses.LogitBinaryCrossEntropy}.get)
    R.load("mmf/utils/modeling.py", "mmf.utils.modeling")

    vl = R.load("mmf/models/vilt.py", "mmf.models.vilt")
    vl.OmegaConf = _OmegaConf
    vl.build_encoder = lambda config: enc.ViTEncoder(config["params"])       # mmf/utils/build.py:517-546, type `vit`
    return vl


def _build(vl, defaults, case, seed):
    import mmf_b200.models as MD
    cfg = _cfg(dict(MD._merge(defaults, model_config(case))))
    m = MG._new_base_model(vl.ViLT, cfg)
    m.build()
    m.init_losses()
    m.eval()
    g = torch.Generator().manual_seed(seed)
    ln = {id(mod.weight) for mod in m.modules() if isinstance(mod, torch.nn.LayerNorm)}
    with torch.no_grad():                               # normal(0, 0.02), LayerNorm weights around 1, on the int8 grid
        for _, p in m.named_parameters():
            base = 1.0 if id(p) in ln else 0.0
            p.copy_(MG._q8(base + torch.randn(p.shape, generator=g) * 0.02, base))
    return m


def _run(m, sl):
    """the registered forward, with the attention masks the encoder received captured on the way in"""
    masks = []

    def grab(mod, a, kw):
        am = kw.get("attention_mask")
        masks.append(None if am is None else am.clone())
    hook = m.encoder.register_forward_pre_hook(grab, with_kwargs=True)
    try:
        return m.forward(sl), masks
    finally:
        hook.remove()


def _groups(m):
    names = {id(p): n for n, p in m.named_parameters()}
    return [{"names": [names[id(p)] for p in g["params"]], "weight_decay": g.get("weight_decay")}
            for g in m.get_optimizer_parameters(None)]


def _grads(m):
    return MG._grads(m, [n for n, p in m.named_parameters() if p.grad is not None and p.dim() >= 2])


def _record(m, i, case):
    m.zero_grad(set_to_none=True)
    o, masks = _run(m, sample_list(i, case))
    sum(o["losses"].values()).backward()
    rec = {"config": model_config(case), "state_dict_keys": sorted(m.state_dict().keys()), "groups": _groups(m),
           "losses": {k: v.detach().clone() for k, v in o["losses"].items()}, "attention_masks": masks,
           "grads": _grads(m)}
    if torch.is_tensor(o["scores"]):
        rec["scores"] = o["scores"].detach().clone()
    return rec


def golden_vilt_model():
    vl = _ref_vilt()
    import mmf_b200.models as MD
    mmf_root = os.path.join(R.REF_ROOT, "mmf")
    doc = MD.read_yaml_with_includes(os.path.join(mmf_root, "configs/models/vilt/defaults.yaml"), mmf_root)
    defaults = _plain(MD._resolve_interpolations(doc["model_config"]["vilt"], doc))
    i = inputs()
    out = {"defaults": defaults, "inputs": i}
    m = _build(vl, defaults, "pretraining", 1821)
    out["pretraining_state_dict"] = {k: v.detach().clone() for k, v in m.state_dict().items()}
    with torch.no_grad():
        sl = sample_list(i, "pretraining")
        te = m.text_embeddings(sl["input_ids"], sl["segment_ids"])
        ie = m.image_embeddings(sl["image"])
        plain = dict(sl)
        only_image = Cfg({k: v for k, v in sl.items() if k != "input_mask"}, image_mask=i["image_mask"].clone())
        out["masks"] = {"sample_list": m.get_attention_mask(sl, te, ie), "dict": m.get_attention_mask(plain, te, ie),
                        "image_mask_only": m.get_attention_mask(only_image, te, ie),
                        "absent": m.get_attention_mask(Cfg(input_ids=sl["input_ids"]), te, ie)}
    for case in ("pretraining", "pretraining_no_mlm"):
        out[case] = _record(m, i, case)
        if case == "pretraining":
            named, out[case]["by_loss"] = dict(m.named_parameters()), {}
            for k in out[case]["losses"]:
                m.zero_grad(set_to_none=True)
                o1, _ = _run(m, sample_list(i, case))
                o1["losses"][k].backward()
                out[case]["by_loss"][k] = {"grads": {n: named[n].grad.detach().clone() for n in SPLIT_PARAMS}}

    trunk = {k: v for k, v in out["pretraining_state_dict"].items() if not k.startswith("heads_dict.")}
    m = _build(vl, defaults, "classification", 1822)
    m.load_state_dict(trunk, strict=False)
    out["classification_head_state_dict"] = {k: v.detach().clone() for k, v in m.state_dict().items()
                                             if k not in trunk}
    for case in ("classification", "classification_nomask"):
        out[case] = _record(m, i, case)
    out["yamls"] = {name: _project_model_config(os.path.join(R.REF_ROOT, "projects/vilt/configs", name + ".yaml"))
                    for name in PROJECT_YAMLS}
    MG._save("vilt_model", out)


PROJECT_YAMLS = ("vqa2/vit_b32_384", "vqa2/vit_b16_224", "masked_coco/pretrain")


def _project_model_config(path):
    """model_config.vilt of a project YAML with its `./` includes merged first and the other_configs interpolations
    resolved; the dataset includes (`../projects/unit/...`) carry no model config and are skipped"""
    import yaml
    import mmf_b200.models as MD

    def read(p):
        with open(p) as fh:
            doc = MD._yaml_numbers(yaml.safe_load(fh) or {})
        out = MD.ConfigNode()
        for inc in doc.pop("includes", None) or []:
            if inc.startswith("./"):
                out = MD._merge(out, read(os.path.join(os.path.dirname(p), inc)))
        return MD._merge(out, doc)
    doc = read(path)
    return _plain(MD._resolve_interpolations(doc["model_config"]["vilt"], doc))


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)
    golden_vilt_model()
