#!/usr/bin/env python
"""TEST INFRASTRUCTURE - writes tests/golden/m4c_model.pt by running the REFERENCE's registered M4C and M4CCaptioner.

Needs the reference tree (MMF_REFERENCE_ROOT, see oracle/ref_loader.py):   python tools/make_golden_m4c_model.py
It writes that one fixture and nothing else.  Storage and gradient sampling are oracle/make_golden.py's.

The reference's `M4C` (mmf/models/m4c.py:34-347) with its own TextBert, MMT, PrevPredEmbeddings, OcrPtrNet and
`M4CCaptioner` (mmf/models/m4c_captioner.py) run here with stand-ins for what needs a network or MMF's runtime: the
registry (config, `<dataset>_num_final_outputs`, `<dataset>_answer_processor`), ClassifierLayer("linear") as its
nn.Linear `module`, the fc7 encoder as relu(Linear(2048, 2048)) named `lc` (FinetuneFasterRcnnFpnFc7 without its pickles),
TextBert.from_pretrained as the constructor, and OmegaConf.create as a dict.  BertEncoder runs the reference's
BertEncoderJit forward (hf_layers.replace_with_jit, as MMF installs it).  The loss is the reference's own
M4CDecodingBCEWithMaskLoss (mmf/modules/losses.py).

The weights are not stored: every parameter is drawn from its name (weight_value below, restated by the tests) on the
int8 grid of oracle/make_golden._q8, so the fixture stays small although the text BERT is 768 wide (m4c.py:70) and the
two fc7 layers are 2048 x 2048.

Cases (B = 4; MMT hidden 128 / 2 heads (d = 64) / 2 layers; text BERT 768 / 12 heads / 1 layer; 8 text tokens, 6
objects, 5 OCR tokens (300 + 604 + 2048 + 50 features), 4 decoding steps; 20 fixed answers + 5 OCR copies; dropout 0;
padding in every stream, sample 1 without OCR tokens):
  train     - m4c in training (teacher forcing from train_prev_inds): scores, the loss, sampled 2-D gradients, the 4-D
              extended mask the reference's MMT built, the state-dict keys
  eval      - m4c greedy decoding: final prev_inds and scores.  The weight seed is the first one for which every step's
              top-2 margin at the position that decides the next token is >= 0.08 (in this case and the next), so bf16
              rounding cannot flip a decoded token, and the decoded tokens are at least 4 distinct ones with an OCR copy
  captioner - m4c_captioner greedy decoding with remove_unk_in_pred
  optimizer - get_optimizer_parameters: the groups' parameter names and learning rates
"""
import os
import sys
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden as MG  # noqa: E402
from oracle import ref_loader as R  # noqa: E402

B, T, RR, O, D, HID, ANS = 4, 8, 6, 5, 4, 128, 20
DATASET = "textvqa"
BOS_IDX, UNK_IDX = 1, 3


class Cfg(dict):
    """attribute-access dict: what the reference's classes get instead of a DictConfig / SampleList"""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v


class _OmegaConf:
    @staticmethod
    def create(d):
        return Cfg(d)


class _Registry:
    def __init__(self):
        self.state = {}

    def register(self, name, obj):
        self.state[name] = obj

    def get(self, name, default=None):
        return self.state.get(name, default)


class _Classifier(torch.nn.Module):
    """ClassifierLayer("linear") (mmf/modules/layers.py): `module` = nn.Linear"""

    def __init__(self, classifier_type, in_dim, out_dim, **kwargs):
        super().__init__()
        assert classifier_type == "linear"
        self.module = torch.nn.Linear(in_dim, out_dim)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)


class _Fc7(torch.nn.Module):
    """FinetuneFasterRcnnFpnFc7's forward (mmf/modules/encoders.py:176-179) with its `lc` not read from pickles"""

    def __init__(self, in_dim=2048):
        super().__init__()
        self.lc = torch.nn.Linear(in_dim, in_dim)

    def forward(self, image):
        return torch.nn.functional.relu(self.lc(image))


def model_config(captioner=False):
    cfg = dict(lr_scale_frcn=0.1, lr_scale_text_bert=0.1, lr_scale_mmt=1.0, text_bert_init_from_bert_base=True,
               text_bert=dict(num_hidden_layers=1, vocab_size=50, max_position_embeddings=16, intermediate_size=128,
                              hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0),
               obj=dict(mmt_in_dim=2048, dropout_prob=0.0), ocr=dict(mmt_in_dim=3002, dropout_prob=0.0),
               mmt=dict(hidden_size=HID, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0),
               classifier=dict(type="linear", ocr_max_num=O, ocr_ptr_net=dict(hidden_size=HID, query_key_size=HID),
                               params={}),
               model_data_dir="unused", losses=[dict(type="m4c_decoding_bce_with_mask")])
    if captioner:
        cfg["remove_unk_in_pred"] = True
    return cfg


def weight_value(name, shape, base, std, seed):
    """the value of parameter `name`: base + N(0, std) drawn from a generator seeded by the name, on the _q8 grid"""
    g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
    return MG._q8(base + torch.randn(shape, generator=g) * std, base)


def weight_spec(m):
    """name -> (shape, base, std): LayerNorm weights around 1; the classifier and pointer network wider, so that greedy
    decoding has clear margins.  The answer embeddings' LayerNorm weight is around 0: the classifier row of the previous
    token is tied to its input embedding, and at full scale it outscores every other answer, so that decoding would only
    ever repeat the first token"""
    ln = {id(mod.weight) for mod in m.modules() if isinstance(mod, torch.nn.LayerNorm)}
    ln.discard(id(m.mmt.prev_pred_embeddings.ans_layer_norm.weight))
    return {n: (tuple(p.shape), 1.0 if id(p) in ln else 0.0, 0.1 if n.startswith(("classifier.", "ocr_ptr_net.")) else 0.02)
            for n, p in m.named_parameters()}


def _q(x):
    return MG._q8(x, 0.0)


def inputs():
    g = torch.Generator().manual_seed(2203)
    text = torch.randint(1, 50, (B, T), generator=g)
    prev = torch.randint(0, ANS + O, (B, D), generator=g)
    prev[:, 0] = BOS_IDX
    targets = (torch.rand(B, D, ANS + O, generator=g) < 0.1).float()
    ocr_max = torch.tensor([5, 0, 3, 2])
    targets[:, :, ANS:] *= (torch.arange(O) < ocr_max[:, None]).float()[:, None, :]   # no target on a padded OCR token
    loss_mask = torch.ones(B, D)
    loss_mask[1, 2:] = 0
    loss_mask[3, 3:] = 0
    return dict(text=text, text_len=torch.tensor([8, 5, 3, 6]),
                image_feature_0=_q(torch.randn(B, RR, 2048, generator=g) * 0.04),
                obj_bbox_coordinates=_q(torch.rand(B, RR, 4, generator=g) * 0.12),
                obj_max_features=torch.tensor([6, 4, 2, 5]),
                context_feature_0=_q(torch.randn(B, O, 300, generator=g) * 0.04),
                context_feature_1=_q(torch.randn(B, O, 604, generator=g) * 0.04),
                image_feature_1=_q(torch.randn(B, O + 2, 2048, generator=g) * 0.04),
                order_vectors=_q(torch.rand(B, O, 50, generator=g) * 0.12),
                ocr_bbox_coordinates=_q(torch.rand(B, O, 4, generator=g) * 0.12),
                ocr_max_features=ocr_max,
                train_prev_inds=prev, targets=targets, train_loss_mask=loss_mask)


def sample_list(i):
    return Cfg(text=i["text"].clone(), text_len=i["text_len"].clone(), image_feature_0=i["image_feature_0"].clone(),
               obj_bbox_coordinates=i["obj_bbox_coordinates"].clone(),
               image_info_0=Cfg(max_features=i["obj_max_features"].clone()),
               context_feature_0=i["context_feature_0"].clone(), context_feature_1=i["context_feature_1"].clone(),
               image_feature_1=i["image_feature_1"].clone(), order_vectors=i["order_vectors"].clone(),
               ocr_bbox_coordinates=i["ocr_bbox_coordinates"].clone(),
               context_info_0=Cfg(max_features=i["ocr_max_features"].clone()),
               train_prev_inds=i["train_prev_inds"].clone(), targets=i["targets"].clone(),
               train_loss_mask=i["train_loss_mask"].clone(), dataset_name=DATASET, dataset_type="train")


def _ref_m4c():
    from transformers import BertConfig
    hl = R.hf_layers()
    m4c = R.load("mmf/models/m4c.py", "mmf.models.m4c")
    cap = R.load("mmf/models/m4c_captioner.py", "mmf.models.m4c_captioner")
    losses = R.load("mmf/modules/losses.py", "mmf.modules.losses")
    reg = _Registry()
    reg.register("config", Cfg(datasets=DATASET))
    reg.register(DATASET + "_num_final_outputs", ANS + O)
    reg.register(DATASET + "_answer_processor", Cfg(BOS_IDX=BOS_IDX, UNK_IDX=UNK_IDX))
    for mod in (m4c, cap):
        mod.registry = reg
    m4c.OmegaConf = _OmegaConf
    m4c.ClassifierLayer = _Classifier
    m4c.build_image_encoder = lambda config, direct_features=False: _Fc7(config["params"]["in_dim"])
    m4c.TextBert.from_pretrained = classmethod(lambda cls, name, config: cls(config))
    # BertPreTrainedModel.init_weights of transformers 5 wants post_init() bookkeeping the <= 4.10-era classes never did;
    # every weight is set explicitly below
    m4c.TextBert.init_weights = lambda self: None
    m4c.MMT.init_weights = lambda self: None
    return m4c, cap, losses, hl, BertConfig


def _build(m4c, cap, BertConfig, captioner, seed):
    cls = cap.M4CCaptioner if captioner else m4c.M4C
    cfg = Cfg(model_config(captioner))
    for k in ("text_bert", "obj", "ocr", "mmt", "classifier"):
        cfg[k] = Cfg(cfg[k])
    cfg.classifier.ocr_ptr_net = Cfg(cfg.classifier.ocr_ptr_net)
    m = MG._new_base_model(cls, cfg)                     # M4C.__init__ (m4c.py:36-39) without BaseModel
    m.mmt_config = BertConfig(**cfg.mmt)
    m._datasets = m4c.registry.get("config").datasets.split(",")
    if captioner:
        m.remove_unk_in_pred = cfg.remove_unk_in_pred
    m.build()
    spec = weight_spec(m)
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.copy_(weight_value(n, *spec[n], seed))
    return m, spec


def _record_steps(m):
    """the scores of every _forward_output call (one per decoding step)"""
    steps, orig = [], m._forward_output

    def rec(sl, fr):
        orig(sl, fr)
        steps.append(fr["scores"].detach().clone())
    m._forward_output = rec
    return steps


def _decision_margin(steps):
    """the smallest top-2 margin over the scores that decide a token: position s at step s (its prefix is final there)"""
    worst = float("inf")
    for s, sc in enumerate(steps[:-1]):
        top = sc[:, s, :].topk(2, dim=-1).values
        worst = min(worst, float((top[:, 0] - top[:, 1]).min()))
    return worst


def _decoded(steps):
    """the distinct tokens decoded at the positions that decide one"""
    return {int(x) for s, sc in enumerate(steps[:-1]) for x in sc[:, s, :].argmax(dim=-1)}


def _eval(m, i):
    m.eval()
    steps = _record_steps(m)
    with torch.no_grad():
        out = m.forward(sample_list(i))
    return out, steps


def golden_m4c_model():
    m4c, cap, losses, hl, BertConfig = _ref_m4c()
    import mmf_b200.models as MD
    mmf_root = os.path.join(R.REF_ROOT, "mmf")
    defaults = {}
    for name in ("m4c", "m4c_captioner"):
        doc = MD.read_yaml_with_includes(os.path.join(mmf_root, "configs/models/%s/defaults.yaml" % name), mmf_root)
        defaults[name] = _plain(MD._resolve_interpolations(doc["model_config"][name], doc))
    i = inputs()
    hl.replace_with_jit()
    try:
        seed = 0
        while True:     # the first weight seed whose decoded tokens vary and have clear margins in both eval cases
            seed += 1
            m, spec = _build(m4c, cap, BertConfig, False, seed)
            c, _ = _build(m4c, cap, BertConfig, True, seed)
            sm, sc = _eval(m, i)[1], _eval(c, i)[1]
            if (min(_decision_margin(sm), _decision_margin(sc)) >= 0.08 and len(_decoded(sm)) >= 4
                    and any(t >= ANS for t in _decoded(sm))):
                break
        print("weight seed", seed)
        out = {"defaults": defaults, "inputs": i, "config": model_config(), "captioner_config": model_config(True),
               "weight_seed": seed, "weight_spec": spec, "bos_idx": BOS_IDX, "unk_idx": UNK_IDX, "dataset": DATASET,
               "num_final_outputs": ANS + O}

        m, _ = _build(m4c, cap, BertConfig, False, seed)
        m.train()
        masks = []
        hook = m.mmt.encoder.register_forward_pre_hook(lambda mod, args: masks.append(args[1].detach().clone()))
        o = m.forward(sample_list(i))
        hook.remove()
        loss = losses.M4CDecodingBCEWithMaskLoss()(sample_list(i), o)
        loss.backward()
        out["train"] = {"state_dict_keys": sorted(m.state_dict().keys()), "scores": o["scores"].detach().clone(),
                        "loss": loss.detach().clone(), "extended_mask": masks[0],
                        "grads": MG._grads(m, [n for n, p in m.named_parameters() if p.grad is not None and p.dim() == 2])}
        sl = sample_list(i)
        sl.train_loss_mask = torch.zeros_like(sl.train_loss_mask)
        out["train"]["loss_zero_mask"] = losses.M4CDecodingBCEWithMaskLoss()(sl, o).detach().clone()

        for case, captioner in (("eval", False), ("captioner", True)):
            mm, _ = _build(m4c, cap, BertConfig, captioner, seed)
            o, steps = _eval(mm, i)
            out[case] = {"scores": o["scores"].clone(), "prev_inds": None, "margin": _decision_margin(steps)}
            # the final prev_inds: the argmax shifted by one, as the last loop iteration leaves them (m4c.py:303-304)
            prev = torch.zeros_like(i["train_prev_inds"])
            prev[:, 0] = BOS_IDX
            prev[:, 1:] = o["scores"].argmax(dim=-1)[:, :-1]
            out[case]["prev_inds"] = prev

        names = {id(p): n for n, p in m.named_parameters()}
        groups = m.get_optimizer_parameters(Cfg(optimizer=Cfg(params=Cfg(lr=1e-4))))
        out["optimizer"] = [{"names": [names[id(p)] for p in g["params"]], "lr": g.get("lr")} for g in groups]
    finally:
        hl.undo_replace_with_jit()
    MG._save("m4c_model", out)


def _plain(x):
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_plain(v) for v in x]
    return x


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)
    golden_m4c_model()
