#!/usr/bin/env python
"""TEST INFRASTRUCTURE - writes tests/golden/uniter_model.pt by running the REFERENCE's registered UNITER model.

Needs the reference tree (MMF_REFERENCE_ROOT, see oracle/ref_loader.py):   python tools/make_golden_uniter_model.py
It needs a full checkout: the head files and ot.py are not among those oracle/build_ref.py stages.  It writes that one
fixture and nothing else.  Storage and gradient sampling are oracle/make_golden.py's.

The reference's `UNITER` (mmf/models/uniter.py:615-774), `UNITERForClassification`, `UNITERForPretraining` and its
transformer heads (mmf/models/transformers/heads/{mlp,mlm,itm,mrc,mrfr,wra}.py, mmf/modules/ot.py) run here with stand-ins
for what needs a network or MMF's runtime: BertConfig.from_pretrained builds the config from its keyword overrides;
BertModel is the reference's BertEncoderJit (what replace_with_jit() installs) plus HF's BertPooler; `retry_n` calls
once; OmegaConf / open_dict are shimmed; BaseTransformerHead is its three-line constructor; MMFLoss is logit_bce under
the reference's key; `registry.get_transformer_head_class` looks the loaded head classes up.

Entries (B = 4, T = 8 tokens, R = 6 regions, hidden 128 / 2 heads / 2 layers, 40 feature dims, 17 region classes, eval):
  vqa2                       - classification scores and logit_bce loss
  mlm, itm, mrc, mrfr, wra   - one pretraining forward each: the seed under which the reference's task draw picks the
                               task, the region masks it drew, the loss, the integer plumbing, sampled gradients
  ot                         - optimal_transport_dist of the reference on the WRA entry's sequence output rounded to
                               bf16, with ragged pads: its cost, plan T and distance
"""
import contextlib
import dataclasses
import os
import random
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden as MG  # noqa: E402
from oracle import ref_loader as R  # noqa: E402

B, T, RR, FEAT, NCLS, VOCAB, NUM_LABELS, HID = 4, 8, 6, 40, 17, 50, 7, 128
TASKS = ["mlm", "itm", "mrc", "mrfr", "wra"]
HEADS = "mmf/models/transformers/heads/"


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

    @staticmethod
    def to_container(cfg, resolve=True):
        return dict(cfg)


def bert_overrides():
    return dict(hidden_size=HID, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256, vocab_size=VOCAB,
                max_position_embeddings=32, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


def model_config(pretraining):
    cfg = dict(random_init=True, bert_model_name="bert-base-uncased", img_dim=FEAT, hidden_size=HID, hidden_dropout_prob=0,
               text_embeddings=bert_overrides(), encoder=bert_overrides(), do_pretraining=pretraining)
    if pretraining:
        cfg.update(tasks=",".join(TASKS), mask_probability=0.3, losses={}, heads=dict(
            mlm=dict(type="mlm", vocab_size=VOCAB, hidden_size=HID), itm=dict(type="itm", hidden_size=HID),
            mrc=dict(type="mrc", hidden_size=HID, label_dim=NCLS), mrfr=dict(type="mrfr", hidden_size=HID, img_dim=FEAT),
            wra=dict(type="wra")))
    else:
        cfg.update(tasks=["vqa2"], losses=dict(vqa2="logit_bce"), heads=dict(vqa2=dict(
            type="mlp", freeze=False, lr_multiplier=1.0, in_dim=HID, hidden_size=2 * HID, num_labels=NUM_LABELS,
            hidden_dropout_prob=0.0, pooler_name="bert_pooler")))
    return cfg


def inputs():
    g = torch.Generator().manual_seed(911)
    ids = torch.randint(1, VOCAB, (B, T), generator=g)
    ids_masked = ids.clone()
    labels = torch.full((B, T), -1, dtype=torch.long)
    for b, t in ((0, 2), (1, 4), (2, 1), (2, 6)):
        labels[b, t] = ids[b, t]
        ids_masked[b, t] = 3
    mask = torch.ones(B, T, dtype=torch.long)
    mask[1, 6:] = 0
    mask[3, 4:] = 0
    feats = torch.randn(B, RR, FEAT, generator=g).abs()
    # pixel boxes whose first coordinate is 0: the reference then divides by the image size (uniter.py:686-700)
    wh = torch.tensor([[640.0, 480.0], [500.0, 375.0], [800.0, 600.0], [320.0, 240.0]])
    lo = torch.rand(B, RR, 2, generator=g) * 0.5
    hi = lo + 0.1 + torch.rand(B, RR, 2, generator=g) * 0.4
    bbox = torch.cat([lo * wh[:, None], hi * wh[:, None], torch.rand(B, RR, 1, generator=g)], dim=-1)
    bbox[0, 0, 0] = 0.0
    maxf = torch.tensor([6, 2, 5, 4])
    cls_prob = torch.softmax(torch.randn(B, RR, NCLS, generator=g) * 2.0, dim=-1)
    targets = torch.softmax(torch.randn(B, NUM_LABELS, generator=g) * 3.0, dim=-1)
    return dict(ids=ids, ids_masked=ids_masked, lm_label_ids=labels, mask=mask, feats=feats, bbox=bbox, image_width=wh[:, 0],
                image_height=wh[:, 1], max_features=maxf, cls_prob=cls_prob, targets=targets,
                is_correct=torch.tensor([1, 0, 1, 1]))


def sample_list(i, dataset_name):
    return Cfg(input_ids=i["ids"].clone(), input_ids_masked=i["ids_masked"].clone(), input_mask=i["mask"].clone(),
               lm_label_ids=i["lm_label_ids"].clone(), image_feature_0=i["feats"].clone(),
               image_info_0=Cfg(max_features=i["max_features"].clone(), bbox=i["bbox"].numpy().copy(),
                                image_width=i["image_width"].numpy().copy(), image_height=i["image_height"].numpy().copy(),
                                cls_prob=i["cls_prob"].numpy().copy()),
               targets=i["targets"].clone(), is_correct=i["is_correct"].clone(), dataset_name=dataset_name,
               dataset_type="train")


def _ref_uniter():
    from transformers import BertConfig
    from transformers.models.bert.modeling_bert import BertPooler
    R._install()
    hl = R.hf_layers()
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
    R.load("mmf/modules/ot.py", "mmf.modules.ot")
    R.load(HEADS + "utils.py", "mmf.models.transformers.heads.utils")
    mods = {n: R.load(HEADS + n + ".py", "mmf.models.transformers.heads." + n) for n in ("mlp", "mlm", "itm", "mrc", "mrfr", "wra")}
    mods["mlp"].OmegaConf = _OmegaConf
    mods["mlp"].open_dict = lambda cfg: contextlib.nullcontext()
    table = {"mlp": mods["mlp"].MLP, "mlm": mods["mlm"].MLM, "itm": mods["itm"].ITM, "mrc": mods["mrc"].MRC,
             "mrfr": mods["mrfr"].MRFR, "wra": mods["wra"].WRA}
    un = R.uniter()
    un.OmegaConf = _OmegaConf
    un.retry_n = lambda n, fn, *a, **k: fn(*a, **k)
    un.registry = types.SimpleNamespace(get_transformer_head_class=lambda t: table[t])
    un.BertConfig = type("BertConfig", (BertConfig,), {
        "from_pretrained": classmethod(lambda cls, name, **kw: BertConfig(**kw))})

    class BertModel(torch.nn.Module):
        def __init__(self, config):
            super().__init__()
            self.encoder, self.pooler = hl.BertEncoderJit(config), BertPooler(config)
    un.BertModel = BertModel

    class MMFLoss(torch.nn.Module):                       # logit_bce, mmf/modules/losses.py:132-251
        def __init__(self, name):
            super().__init__()
            assert name == "logit_bce"

        def forward(self, sl, out):
            loss = torch.nn.functional.binary_cross_entropy_with_logits(out["scores"], sl["targets"]) * sl["targets"].size(1)
            return {"%s/%s/logit_bce" % (sl["dataset_type"], sl["dataset_name"]): loss}
    un.MMFLoss = MMFLoss
    return un, R.load("mmf/modules/ot.py", "mmf.modules.ot")


def _perturb(module, seed):
    """normal(0, 0.02) weights and biases, LayerNorm weights around 1, every value on the int8 grid of MG._q8"""
    g = torch.Generator().manual_seed(seed)
    ln = {id(m.weight) for m in module.modules() if isinstance(m, torch.nn.LayerNorm)}
    with torch.no_grad():
        for _, p in module.named_parameters():
            base = 1.0 if id(p) in ln else 0.0
            p.copy_(MG._q8(base + torch.randn(p.shape, generator=g) * 0.02, base))


def _build(un, cfg, seed):
    m = MG._new_base_model(un.UNITER, Cfg({k: (Cfg(v) if isinstance(v, dict) else v) for k, v in cfg.items()}))
    for task, hc in m.config["heads"].items():
        m.config["heads"][task] = Cfg(hc)
    m.do_pretraining = cfg["do_pretraining"]
    m.build()
    m.eval()
    _perturb(m, seed)
    return m


def _seed_all(s):
    torch.manual_seed(s)
    np.random.seed(s)
    random.seed(s)


def _seed_for(task):
    for s in range(1000, 1200):
        torch.manual_seed(s)
        if TASKS[torch.randint(len(TASKS), (1,)).item()] == task:
            return s
    raise RuntimeError(task)


def _grads_2d(m):
    return MG._grads(m, [n for n, p in m.named_parameters() if p.grad is not None and p.dim() == 2])


def _plumbing(sl):
    out = {k: sl[k].detach().clone() for k in ("image_mask", "attention_mask", "position_ids", "img_pos_feat", "input_ids")}
    if "mlm_labels" in sl:
        out["combined_labels"] = sl["mlm_labels"]["combined_labels"].clone()
    for k in ("image_region_mask", "mrfr_region_mask", "region_class", "mrfr_region_target"):
        if k in sl:
            out[k] = sl[k].detach().clone()
    return out


def golden_uniter_model():
    un, ot = _ref_uniter()
    import mmf_b200.models as MD
    mmf_root = os.path.join(R.REF_ROOT, "mmf")
    doc = MD.read_yaml_with_includes(os.path.join(mmf_root, "configs/models/uniter/defaults.yaml"), mmf_root)
    i = inputs()
    out = {"defaults": _plain(MD._resolve_interpolations(doc["model_config"]["uniter"], doc)), "inputs": i, "tasks": TASKS}

    cfg = model_config(True)
    m = _build(un, cfg, 901)
    out["pretraining_config"] = cfg
    out["pretraining_state_dict"] = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for task in TASKS:
        seed = _seed_for(task)
        _seed_all(seed)
        m.zero_grad(set_to_none=True)
        sl = sample_list(i, "coco")
        seen = {}
        hook = m.uniter.uniter.register_forward_hook(lambda mod, a, o: seen.update(seq=o.final_layer.detach().clone()))
        o = m.forward(sl)
        hook.remove()
        assert sl["task"] == task
        sum(o["losses"].values()).backward()
        out[task] = {"seed": seed, "losses": {k: v.detach().clone() for k, v in o["losses"].items()},
                     "plumbing": _plumbing(sl), "grads": _grads_2d(m)}
        if task == "wra":
            # the reference's own cost / ipot / distance on bf16-exact inputs with ragged pads
            seq = seen["seq"].to(torch.bfloat16).float()
            txt_pad = torch.arange(T).unsqueeze(0) >= torch.tensor([8, 6, 1, 4]).unsqueeze(1)
            img_pad = torch.arange(RR).unsqueeze(0) >= torch.tensor([6, 2, 5, 1]).unsqueeze(1)
            txt, img = seq[:, :T], seq[:, T:T + RR]
            cost = ot.cost_matrix_cosine(txt, img)
            joint = txt_pad.unsqueeze(-1) | img_pad.unsqueeze(-2)
            cost.masked_fill_(joint, 0)
            plan = ot.ipot(cost, (T - txt_pad.sum(1)).float(), txt_pad, (RR - img_pad.sum(1)).float(), img_pad, joint,
                           0.5, 50, 1)
            distance = ot.optimal_transport_dist(txt, img, txt_pad, img_pad)
            assert torch.equal(distance, ot.trace(cost.matmul(plan)))
            out["ot"] = {"sequence_output": seq, "T_len": T, "R_len": RR, "txt_pad": txt_pad, "img_pad": img_pad,
                         "cost": cost, "T": plan, "distance": distance}

    trunk = {k: v for k, v in out["pretraining_state_dict"].items() if k.startswith("uniter.uniter.")}
    cfg = model_config(False)
    m = _build(un, cfg, 902)
    m.load_state_dict(trunk, strict=False)
    _seed_all(7)
    sl = sample_list(i, "vqa2")
    o = m.forward(sl)
    loss = sum(o["losses"].values())
    loss.backward()
    sd = m.state_dict()
    out["vqa2"] = {"config": cfg, "state_dict_keys": sorted(sd.keys()),
                   "head_state_dict": {k: v.detach().clone() for k, v in sd.items() if k not in trunk},
                   "scores": o["scores"].detach().clone(), "losses": {k: v.detach().clone() for k, v in o["losses"].items()},
                   "plumbing": _plumbing(sl), "grads": _grads_2d(m)}
    MG._save("uniter_model", out)


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)
    golden_uniter_model()
