"""Model plugins: the 4th form of the reference's drop-in boundary (SURVEY.md 8b "Model plugin + data contract").

  registry.register_model("visual_bert")  VisualBERT   <->  mmf/models/visual_bert.py:407-601
  registry.register_model("vilbert")      ViLBERT      <->  mmf/models/vilbert.py:1336-1472
  registry.register_model("mmbt")         MMBT         <->  mmf/models/mmbt.py:565-643
  registry.register_model("lxmert")       LXMERT       <->  mmf/models/lxmert.py:647-790
  registry.register_model("uniter")       UNITER       <->  mmf/models/uniter.py:615-774   (mmf_b200/uniter_model.py)
  registry.register_model("vinvl")        VinVL        <->  mmf/models/vinvl.py:392-505    (mmf_b200/vinvl_model.py)
  registry.register_model("m4c")          M4C          <->  mmf/models/m4c.py:34-347       (mmf_b200/m4c_model.py)
  registry.register_model("m4c_captioner") M4CCaptioner <->  mmf/models/m4c_captioner.py:6-24
  registry.register_model("vilt")         ViLT         <->  mmf/models/vilt.py:118-283     (mmf_b200/vilt_model.py)

Each is a `BaseModel` (mmf/models/base_model.py:67-337 contract: ctor(config) -> build() -> forward(SampleList) -> dict
with "scores" and/or "losses"; `config_path()` names the model's default YAML; `__call__` fills "losses" from the
configured loss list when the forward did not), built from the SAME configuration keys as the reference's YAML
(mmf/configs/models/{visual_bert,vilbert,mmbt,lxmert}/*.yaml).  `load_model_config()` reads such a YAML with PyYAML
(`includes:` honoured) when an MMF checkout is at hand; the defaults themselves are restated in `MODEL_DEFAULTS` so that
nothing is read from the reference tree at run time (tests/test_models_cpu.py pins the restatement to the YAML files).

The trunk (embeddings -> encoder) is the B200 engine; the heads are the reference's heads on the same kernels
(`BertPredictionHeadTransform` = GEMM + GELU epilogue -> row LayerNorm, classifier / decoder GEMMs, poolers = GEMM +
activation).  There is no pretrained-weight download here (no network): `bert_model_name` only selects the BERT-base
hyper-parameters; weights arrive through load_state_dict with the reference's key names.
"""
import collections
import copy
import os
import warnings

import torch
from torch import nn

from . import ops
from .heads import B200BertLMPredictionHead, B200BertPredictionHeadTransform, B200BertPreTrainingHeads, masked_lm_loss
from .modules import _init_bert_weights
from .registry import registry


# ------------------------------------------------------------------------------------------------------
# configuration
# ------------------------------------------------------------------------------------------------------
class ConfigNode(dict):
    """attribute-access dict standing in for OmegaConf's DictConfig on this path (`cfg.key`, `cfg.get(key, default)`,
    `key in cfg`); nested dicts become nodes."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        for key, v in list(self.items()):
            self[key] = _nodeify(v)

    def __getattr__(self, key):
        try:
            return self[key]
        except KeyError:
            raise AttributeError(key)

    def __setattr__(self, key, value):
        self[key] = _nodeify(value)

    def __deepcopy__(self, memo):
        return ConfigNode({k: copy.deepcopy(v, memo) for k, v in self.items()})


def _nodeify(v):
    if isinstance(v, ConfigNode):
        return v
    if isinstance(v, dict):
        return ConfigNode(v)
    if isinstance(v, (list, tuple)):
        return [_nodeify(x) for x in v]
    return v


def _merge(base, over):
    out = ConfigNode(copy.deepcopy(dict(base)))
    for k, v in over.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict):
            out[k] = _merge(out[k], v)
        else:
            out[k] = _nodeify(copy.deepcopy(v))
    return out


# HF BertConfig defaults = bert-base-uncased (what `BertConfig.from_dict(model_config)` fills in for keys the model
# YAML does not carry: mmf/models/visual_bert.py:171-173, vilbert.py:1061-1063, mmf/modules/encoders.py:543-549)
BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                 hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, max_position_embeddings=512,
                 type_vocab_size=2, initializer_range=0.02, layer_norm_eps=1e-12, pad_token_id=0)

# restatement of the `model_config.<name>` blocks of the reference's default YAMLs (file cited per entry)
MODEL_DEFAULTS = {
    # mmf/configs/models/visual_bert/defaults.yaml:1-17
    "visual_bert": dict(
        bert_model_name="bert-base-uncased", training_head_type="pretraining", visual_embedding_dim=2048,
        special_visual_initialize=True, embedding_strategy="plain", bypass_transformer=False, output_attentions=False,
        output_hidden_states=False, random_initialize=False, freeze_base=False, finetune_lr_multiplier=1,
        pooler_strategy="default", zerobias=False),
    # mmf/configs/models/vilbert/defaults.yaml:1-59
    "vilbert": dict(
        bert_model_name="bert-base-uncased", training_head_type="pretraining", visual_embedding_dim=2048,
        special_visual_initialize=True, hard_cap_seq_len=None, cut_first="text", embedding_strategy="plain",
        bypass_transformer=False, output_attentions=False, output_hidden_states=False, text_only=False,
        random_initialize=False, freeze_base=False, finetune_lr_multiplier=1, attention_probs_dropout_prob=0.1,
        layer_norm_eps=1e-12, hidden_act="gelu", hidden_dropout_prob=0.1, hidden_size=768, initializer_range=0.02,
        intermediate_size=3072, max_position_embeddings=512, num_attention_heads=12, num_hidden_layers=12,
        type_vocab_size=2, vocab_size=30522, v_feature_size=2048, v_target_size=1601, v_hidden_size=1024,
        v_num_hidden_layers=6, v_num_attention_heads=8, v_intermediate_size=1024, bi_hidden_size=1024,
        bi_num_attention_heads=8, bi_intermediate_size=1024, bi_attention_type=1, v_attention_probs_dropout_prob=0.1,
        v_hidden_act="gelu", v_hidden_dropout_prob=0.1, v_initializer_range=0.02, v_biattention_id=[0, 1, 2, 3, 4, 5],
        t_biattention_id=[6, 7, 8, 9, 10, 11], pooling_method="mul", fusion_method="mul", fast_mode=False,
        with_coattention=True, dynamic_attention=False, in_batch_pairs=False, task_specific_tokens=False, fixed_v_layer=0,
        fixed_t_layer=0, visualization=False, visual_target=0, objective=0, num_negative=128, model="bert"),
    # mmf/configs/models/mmbt/defaults.yaml:1-49 (the text encoder's bert_model_name interpolation resolved)
    "mmbt": dict(
        training_head_type="pretraining", bert_model_name="bert-base-uncased", direct_features_input=False,
        freeze_text=False, freeze_modal=False, freeze_complete_base=False, finetune_lr_multiplier=1,
        fused_feature_only=False, modal_hidden_size=2048, text_hidden_size=768, num_labels=2,
        modal_encoder=dict(type="resnet152", params=dict(pretrained=True, pool_type="avg", num_output_features=1)),
        use_modal_start_token=True, use_modal_end_token=True,
        text_encoder=dict(type="transformer", params=dict(
            num_segments=2, bert_model_name="bert-base-uncased", hidden_size=768, num_hidden_layers=12,
            num_attention_heads=12, output_attentions=False, output_hidden_states=False))),
    # mmf/configs/models/lxmert/defaults.yaml:1-74
    "lxmert": dict(
        bert_model_name="bert-base-uncased", training_head_type="pretraining", random_initialize=False, num_labels=3129,
        gqa_labels=1534, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, hidden_size=768,
        hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, max_position_embeddings=512,
        type_vocab_size=2, initializer_range=0.02, pad_token_id=0, layer_norm_eps=1e-12, mode="lxr", l_layers=9,
        x_layers=5, r_layers=5, visual_feat_dim=2048, visual_pos_dim=4, task_matched=True, task_mask_lm=True,
        task_obj_predict=True, task_qa=True, visual_losses=["obj", "feat"],
        visual_loss_config=dict(obj=[3129, "ce", [-1], 6.67], attr=[400, "ce", [-1], 6.67],
                                feat=[2048, "l2", [-1, 2048], 6.67]),
        special_visual_initialize=True, hard_cap_seq_len=36, cut_first="text", embedding_strategy="plain",
        bypass_transformer=False, output_attentions=False, output_hidden_states=False, text_only=False,
        freeze_base=False, finetune_lr_multiplier=1, vocab_size=30522, fast_mode=False, dynamic_attention=False,
        in_batch_pairs=False, visualization=False, model="bert"),
}


def _resolve_interpolations(node, root):
    """${a.b.c} references of the reference YAMLs (OmegaConf interpolation), resolved against the loaded tree; unknown
    roots (${env.data_dir}) are left as they are"""
    import re
    pat = re.compile(r"^\$\{([A-Za-z0-9_.]+)\}$")

    def look(path):
        cur = root
        for part in path.split("."):
            if not isinstance(cur, dict) or part not in cur:
                return None
            cur = cur[part]
        return cur

    def walk(v):
        if isinstance(v, dict):
            for k in list(v.keys()):
                v[k] = walk(v[k])
            return v
        if isinstance(v, list):
            return [walk(x) for x in v]
        if isinstance(v, str):
            m = pat.match(v)
            if m:
                r = look(m.group(1))
                if r is not None and not isinstance(r, dict):
                    return r
        return v
    return walk(node)


def _yaml_numbers(v):
    """PyYAML (YAML 1.1) reads `1e-12` as a string; OmegaConf, which the reference loads its YAML with, as a float"""
    import re
    if isinstance(v, dict):
        return {k: _yaml_numbers(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_yaml_numbers(x) for x in v]
    if isinstance(v, str) and re.match(r"^[-+]?\d+(\.\d*)?[eE][-+]?\d+$", v):
        return float(v)
    return v


def read_yaml_with_includes(path, mmf_root=None):
    """One reference YAML, its `includes:` merged first (mmf/utils/configuration.py:84-116: paths relative to the mmf
    package root, or `./x.yaml` relative to the including file)."""
    import yaml
    with open(path) as fh:
        doc = _yaml_numbers(yaml.safe_load(fh) or {})
    out = ConfigNode()
    for inc in doc.pop("includes", None) or []:
        if inc.startswith("."):
            inc_path = os.path.join(os.path.dirname(path), inc)
        else:
            if mmf_root is None:
                raise ValueError("%s includes %s: pass mmf_root (the directory that holds `configs/`)" % (path, inc))
            inc_path = os.path.join(mmf_root, inc)
        out = _merge(out, read_yaml_with_includes(inc_path, mmf_root))
    return _merge(out, doc)


def load_model_config(model, yaml_path=None, overrides=None, mmf_root=None):
    """`model_config.<model>` as the reference's build_config would hand it to the model: the model's defaults (restated
    here, or read from `yaml_path` - e.g. <mmf>/configs/models/visual_bert/classification.yaml - when given), then
    `overrides` (a dict, the user-config level).  `mmf_root` defaults to $MMF_ROOT."""
    if model not in MODEL_DEFAULTS:
        raise ValueError("unknown model %r (have: %s)" % (model, sorted(MODEL_DEFAULTS)))
    cfg = ConfigNode(copy.deepcopy(MODEL_DEFAULTS[model]))
    if yaml_path is not None:
        root = mmf_root or os.environ.get("MMF_ROOT")
        if not os.path.isabs(yaml_path) and root is not None:
            yaml_path = os.path.join(root, yaml_path)
        doc = read_yaml_with_includes(yaml_path, root)
        block = (doc.get("model_config") or {}).get(model)
        if block is None:
            raise ValueError("%s has no model_config.%s block" % (yaml_path, model))
        cfg = _merge(cfg, _resolve_interpolations(block, doc))
    if overrides:
        cfg = _merge(cfg, overrides)
    # the trainer stamps the registry name over whatever the block carries (vilbert's YAML has `model: bert`):
    # mmf/trainers/mmf_trainer.py:84-95 `attributes.model = self.config.model`
    cfg["model"] = model
    return cfg


def bert_config_of(config):
    """BertConfig.from_dict(model_config): BERT-base defaults overridden by every key the model config carries"""
    merged = dict(BERT_BASE)
    merged.update({k: v for k, v in dict(config).items() if not isinstance(v, dict)})
    return ConfigNode(merged)


# ------------------------------------------------------------------------------------------------------
# losses + BaseModel
# ------------------------------------------------------------------------------------------------------
def _loss_cross_entropy(sample_list, model_output, **params):
    return nn.functional.cross_entropy(model_output["scores"].float(), sample_list["targets"], **params)   # losses.py:595-602


def _loss_logit_bce(sample_list, model_output):
    scores, targets = model_output["scores"].float(), sample_list["targets"]
    return nn.functional.binary_cross_entropy_with_logits(scores, targets, reduction="mean") * targets.size(1)   # losses.py:226-251


def _loss_bce(sample_list, model_output):
    scores, targets = model_output["scores"].float(), sample_list["targets"]
    return nn.functional.binary_cross_entropy(scores, targets, reduction="mean") * targets.size(1)


LOSSES = {"cross_entropy": _loss_cross_entropy, "logit_bce": _loss_logit_bce, "bce": _loss_bce}


class Losses(nn.Module):
    """mmf/modules/losses.py:52-129 (`Losses`) + :132-223 (`MMFLoss`) for the loss types the fusion configs use; keys are
    "{dataset_type}/{dataset_name}/{loss}" like the reference's."""

    def __init__(self, loss_list):
        super().__init__()
        self.items = []
        for item in loss_list:
            name = item if isinstance(item, str) else item["type"]
            params = {} if isinstance(item, str) else dict(item.get("params", {}) or {})
            if name not in LOSSES:
                raise ValueError("No loss named %s is registered to registry" % name)
            self.items.append((name, params))

    def forward(self, sample_list, model_output):
        out = {}
        if "targets" not in sample_list:
            warnings.warn("Sample list has not field 'targets', are you sure that your ImDB has labels?")
            return out
        for name, params in self.items:
            v = LOSSES[name](sample_list, model_output, **params)
            key = "%s/%s/%s" % (sample_list["dataset_type"], sample_list["dataset_name"], name)
            out[key] = v.view(1) if v.dim() == 0 else v
        return out


class BaseModel(nn.Module):
    """mmf/models/base_model.py:67-337 for this path: config -> build() -> forward(sample_list) -> dict; `__call__` adds
    "losses" (from `config.losses`) unless the forward produced them; `load_state_dict` runs `format_state_key`."""

    def __init__(self, config):
        super().__init__()
        self.config = config if isinstance(config, ConfigNode) else ConfigNode(dict(config))
        self._logged_warning = {"losses_present": False}
        self.is_pretrained = False

    @classmethod
    def config_path(cls):
        return None

    @classmethod
    def format_state_key(cls, key):
        return key

    def build(self):
        raise NotImplementedError("Build method not implemented in the child model class.")

    def init_losses(self):
        """base_model.py:223-249: instantiate `self.losses` from config.losses"""
        losses = self.config.get("losses", [])
        if len(losses) == 0 and not self.is_pretrained:
            warnings.warn("No losses are defined in model configuration. You are expected to return loss in your return "
                          "dict from forward.")
        self.losses = Losses(losses)

    def load_state_dict(self, state_dict, *args, **kwargs):
        return super().load_state_dict({self.format_state_key(k): v for k, v in state_dict.items()}, *args, **kwargs)

    def __call__(self, sample_list, *args, **kwargs):
        model_output = super().__call__(sample_list, *args, **kwargs)
        if self.is_pretrained:
            return model_output
        assert isinstance(model_output, collections.abc.Mapping), "A dict must be returned from the forward of the model."
        if "losses" in model_output:
            if not self._logged_warning["losses_present"]:
                warnings.warn("'losses' already present in model output. No calculation will be done in base model.")
                self._logged_warning["losses_present"] = True
            assert isinstance(model_output["losses"], collections.abc.Mapping), "'losses' must be a dict."
        elif hasattr(self, "losses"):
            model_output["losses"] = self.losses(sample_list, model_output)
        else:
            model_output["losses"] = {}
        return model_output


def build_model(config):
    """mmf/utils/build.py:95-140 for registered models: class by `config.model`, build(), init_losses()"""
    name = config["model"]
    cls = registry.get_model_class(name)
    if cls is None:
        raise RuntimeError("No model registered for name: %s" % name)
    model = cls(config)
    model.build()
    model.init_losses()
    return model


# ------------------------------------------------------------------------------------------------------
# heads shared by the three models
# ------------------------------------------------------------------------------------------------------
class B200Linear(nn.Linear):
    """nn.Linear parameters (`weight`, `bias`), forward on the wgmma GEMM (any feature counts, ops.linear_any)"""

    def forward(self, x):
        shape = x.shape
        y = ops.linear_any(x.reshape(-1, shape[-1]), self.weight, self.bias)
        return y.reshape(*shape[:-1], self.out_features)


def classifier_head(config, hidden_size, num_labels):
    """nn.Sequential(BertPredictionHeadTransform(config), nn.Linear(hidden, num_labels)) - visual_bert.py:327-330,
    vilbert.py:1263-1266, mmbt.py:535-538; state_dict keys `0.dense.*`, `0.LayerNorm.*`, `1.*` as in the reference."""
    c = ConfigNode(dict(config))
    c.hidden_size = hidden_size
    return nn.Sequential(B200BertPredictionHeadTransform(c), B200Linear(hidden_size, num_labels))


def _sl_get(obj, key, default=None):
    """getattr(sample_list, key, default) for SampleList / dict / namespace"""
    if obj is None:
        return default
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


def image_mask_from_dim(features, image_dim):
    """`arange(R).expand(...) < image_dim` -> int64 (visual_bert.py:538-556, vilbert.py:1432-1440): integer path, bit-exact"""
    mask = torch.arange(features.size(-2), device=features.device).expand(features.size()[:-1])
    if image_dim.dim() < mask.dim():
        image_dim = image_dim.unsqueeze(-1)
        assert image_dim.dim() == mask.dim()
    return (mask < image_dim).long()


# ------------------------------------------------------------------------------------------------------
# VisualBERT
# ------------------------------------------------------------------------------------------------------
class B200VisualBERTForClassification(nn.Module):
    """VisualBERTForClassification (visual_bert.py:284-404): trunk -> (pooler | vqa gather) -> dropout -> classifier"""

    def __init__(self, config):
        super().__init__()
        from .visual_bert import B200VisualBERTBase
        self.config = config
        # The reference's trunk calls its encoder without output_attentions (visual_bert.py:144-157), so the
        # attention_weights it reports are always the empty tuple; so are they here.
        self.output_attentions = bool(config.get("output_attentions", False))
        self.output_hidden_states = bool(config.get("output_hidden_states", False))
        self.pooler_strategy = config.get("pooler_strategy", "default")
        self.bert_config = bert_config_of(config)
        self.bert = B200VisualBERTBase(self.bert_config)
        self.training_head_type = config.training_head_type
        self.num_labels = config.num_labels
        self.dropout = nn.Dropout(self.bert_config.hidden_dropout_prob)
        hidden = self.bert_config.hidden_size * (2 if self.training_head_type == "nlvr2" else 1)
        self.classifier = classifier_head(self.bert_config, hidden, self.num_labels)
        _init_bert_weights(self.classifier, float(self.bert_config.initializer_range))
        if "losses" in config and config.get("zerobias", False):       # visual_bert.py:343-347
            for loss in config.losses:
                if "bce" in (loss if isinstance(loss, str) else loss["type"]):
                    self.classifier[1].bias.data.fill_(config.biasfill)

    def forward(self, input_ids, input_mask, attention_mask=None, token_type_ids=None, visual_embeddings=None,
                visual_embeddings_type=None, image_text_alignment=None, masked_lm_labels=None):
        sequence_output, pooled_output, _ = self.bert(input_ids, attention_mask, token_type_ids, visual_embeddings,
                                                      visual_embeddings_type, image_text_alignment)
        if self.training_head_type == "nlvr2":                         # 2B x H -> B x 2H
            b = pooled_output.size(0)
            pooled_output = torch.cat([pooled_output[: b // 2], pooled_output[b // 2:]], dim=1)
        out = {}
        if self.output_attentions:
            out["attention_weights"] = ()
        if self.output_hidden_states:
            out["sequence_output"], out["pooled_output"] = sequence_output, pooled_output
        if self.pooler_strategy == "vqa":                              # second-last attended token (integer gather)
            idx = input_mask.sum(1) - 2
            pooled_output = torch.gather(sequence_output, 1,
                                         idx.view(-1, 1, 1).expand(idx.size(0), 1, sequence_output.size(-1)))
        pooled_output = self.dropout(pooled_output)
        logits = self.classifier(pooled_output)
        out["scores"] = logits.contiguous().view(-1, self.num_labels).to(sequence_output.dtype)
        return out


@registry.register_model("visual_bert")
class VisualBERT(BaseModel):
    def __init__(self, config):
        super().__init__(config)
        self.training_head_type = self.config.training_head_type

    @classmethod
    def config_path(cls):
        return "configs/models/visual_bert/pretrain.yaml"

    @classmethod
    def format_state_key(cls, key):                                    # visual_bert.py:560-566
        return key.replace("bert.bert", "model.bert").replace("bert.cls", "model.cls").replace(
            "bert.classifier", "model.classifier")

    def build(self):
        from .visual_bert import B200VisualBERTForPretraining
        if self.training_head_type == "pretraining":
            self.model = B200VisualBERTForPretraining(bert_config_of(self.config),
                                                      mlm_positions=self.config.get("mlm_positions", "all"))
        else:
            self.model = B200VisualBERTForClassification(self.config)
        # special_visual_initialize copies the text type/position tables into the visual ones (embeddings.py:330-345)
        if self.config.get("special_visual_initialize", False):
            emb = self.model.bert.embeddings
            if hasattr(emb, "initialize_visual_from_pretrained"):
                emb.initialize_visual_from_pretrained()
        if self.config.get("freeze_base", False):
            for p in self.model.bert.parameters():
                p.requires_grad = False

    # ---- SampleList plumbing (visual_bert.py:427-556), integer paths exact ----
    def update_sample_list_based_on_head(self, sl):
        ids, mask, seg = sl["input_ids"], sl["input_mask"], sl["segment_ids"]
        if self.training_head_type == "nlvr2":
            ids, mask, seg = torch.cat([ids, ids]), torch.cat([mask, mask]), torch.cat([seg, seg])
            img0, img1 = _sl_get(sl, "img0", {}), _sl_get(sl, "img1", {})
            feats = torch.cat([_sl_get(img0, "image_feature_0"), _sl_get(img1, "image_feature_0")])
            dim = torch.cat([_sl_get(_sl_get(img0, "image_info_0", {}), "max_features"),
                             _sl_get(_sl_get(img1, "image_info_0", {}), "max_features")])
        else:
            dim = _sl_get(_sl_get(sl, "image_info_0", {}), "max_features", None)
            feats = _sl_get(sl, "image_feature_0", None)
        if dim is None:
            dim = feats.new_full(size=(feats.size(0), 1), fill_value=feats.size(1))
        sl["visual_embeddings"], sl["image_dim"] = feats, dim
        sl["input_ids"], sl["input_mask"], sl["token_type_ids"] = ids, mask, seg
        return sl

    def add_custom_params(self, sl):
        if self.training_head_type == "pretraining":
            sl["masked_lm_labels"] = sl["lm_label_ids"]
        sl["image_mask"] = image_mask_from_dim(sl["visual_embeddings"], sl["image_dim"].to(sl["visual_embeddings"].device))
        return sl

    def flatten_for_bert(self, sl):
        keys = ["input_ids", "token_type_ids", "input_mask", "image_mask"]
        if self.training_head_type == "pretraining":
            keys.append("masked_lm_labels")
        for k in keys:                                                 # transform_to_batch_sequence (modeling.py)
            t = sl[k]
            if t is not None and t.dim() > 2:
                sl[k] = t.contiguous().view(-1, t.size(-1))
        v = sl["visual_embeddings"]
        if v is not None and v.dim() > 3:                              # transform_to_batch_sequence_dim
            sl["visual_embeddings"] = v.contiguous().view(-1, v.size(-2), v.size(-1))
        return sl

    def add_post_flatten_params(self, sl):
        sl["visual_embeddings_type"] = torch.zeros_like(sl["image_mask"])
        attention_mask = torch.cat((sl["input_mask"], sl["image_mask"]), dim=-1)
        sl["attention_mask"] = attention_mask
        if self.training_head_type == "pretraining":
            lab = sl["masked_lm_labels"]
            assert lab.size(-1) == sl["input_mask"].size(-1) and lab.dim() == 2
            new = torch.ones_like(attention_mask) * -1
            new[: lab.size(0), : lab.size(1)] = lab
            sl["masked_lm_labels"] = new
        return sl

    def forward(self, sample_list):
        sl = self.update_sample_list_based_on_head(sample_list)
        sl = self.add_custom_params(sl)
        sl = self.flatten_for_bert(sl)
        sl = self.add_post_flatten_params(sl)
        out = self.model(sl["input_ids"], sl["input_mask"], sl["attention_mask"], sl["token_type_ids"],
                         sl["visual_embeddings"], sl["visual_embeddings_type"], _sl_get(sl, "image_text_alignment", None),
                         _sl_get(sl, "masked_lm_labels", None))
        if self.training_head_type == "pretraining":
            key = "%s/%s" % (sl["dataset_name"], sl["dataset_type"])
            out["losses"] = {key + "/masked_lm_loss": out.pop("masked_lm_loss")}
        return out


# ------------------------------------------------------------------------------------------------------
# ViLBERT
# ------------------------------------------------------------------------------------------------------
class B200ViLBERTImagePredictionHead(nn.Module):
    """BertImagePredictionHead (vilbert.py:830-860): GELU transform over v_hidden -> LayerNorm -> decoder to v_target_size"""

    def __init__(self, config):
        super().__init__()
        c = ConfigNode(dict(config))
        c.hidden_size = config.v_hidden_size
        c.layer_norm_eps = 1e-12
        self.transform = B200BertPredictionHeadTransform(c)
        self.decoder = B200Linear(config.v_hidden_size, config.v_target_size)

    def forward(self, hidden_states):
        return self.decoder(self.transform(hidden_states))


class B200ViLBERTPreTrainingHeads(nn.Module):
    """vilbert.BertPreTrainingHeads (vilbert.py:863-892)"""

    def __init__(self, config):
        super().__init__()
        self.predictions = B200BertLMPredictionHead(config)
        self.bi_seq_relationship = nn.Linear(config.bi_hidden_size, 2)
        self.imagePredictions = B200ViLBERTImagePredictionHead(config)
        self.fusion_method = config.fusion_method
        self.dropout = nn.Dropout(0.1)

    def forward(self, sequence_output_t, sequence_output_v, pooled_output_t, pooled_output_v):
        if self.fusion_method == "sum":
            pooled = self.dropout(pooled_output_t + pooled_output_v)
        elif self.fusion_method == "mul":
            pooled = self.dropout(pooled_output_t * pooled_output_v)
        else:
            raise AssertionError
        return (self.predictions(sequence_output_t), self.imagePredictions(sequence_output_v),
                self.bi_seq_relationship(pooled.to(self.bi_seq_relationship.weight.dtype)))


class B200ViLBERTForPretraining(nn.Module):
    """ViLBERTForPretraining (vilbert.py:1054-1243) with visual_target 0 (KL on region class distributions, the config
    default) and 1 (MSE); 2 (negative sampling) raises."""

    def __init__(self, config):
        super().__init__()
        from .vilbert import B200ViLBERTBase
        self.config = config
        self.bert = B200ViLBERTBase(bert_config_of(config))
        self.cls = B200ViLBERTPreTrainingHeads(bert_config_of(config))
        _init_bert_weights(self.cls, float(config.get("initializer_range", 0.02)))
        # like the reference's constructor, the decoder is NOT tied here: ViLBERTForPretraining.__init__ (vilbert.py:1054-1078)
        # never calls init_weights(); tie_weights() below is what :1095-1102 would do
        self.vocab_size = config.vocab_size
        self.visual_target = config.visual_target
        if self.visual_target not in (0, 1):
            raise NotImplementedError("ViLBERT visual_target=%r (negative sampling) is not on the B200 path" % self.visual_target)

    def tie_weights(self):
        self.cls.predictions.decoder.weight = self.bert.embeddings.word_embeddings.weight

    def forward(self, input_ids, image_feature, image_location, token_type_ids, attention_mask, image_attention_mask,
                masked_lm_labels=None, image_label=None, image_target=None, output_all_attention_masks=False):
        seq_t, seq_v, pooled_t, pooled_v, _, _, _ = self.bert(
            input_ids, image_feature, image_location, token_type_ids, attention_mask, image_attention_mask,
            output_all_encoded_layers=False, output_all_attention_masks=output_all_attention_masks, reference_outputs=True)
        scores_t, scores_v, _ = self.cls(seq_t, seq_v, pooled_t, pooled_v)
        out = {}
        if image_label is not None and image_target is not None:
            sel = torch.eq(image_label, 1)
            if self.visual_target == 1:
                img_loss = nn.functional.mse_loss(scores_v.float(), image_target, reduction="none")
                denom = max(torch.sum(sel.unsqueeze(2).expand_as(img_loss)), 1)
            else:
                img_loss = nn.functional.kl_div(nn.functional.log_softmax(scores_v.float(), dim=2), image_target,
                                                reduction="none")
                denom = max(torch.sum(sel), 0)
            out["masked_img_loss"] = (torch.sum(img_loss * sel.unsqueeze(2).float()) / denom).unsqueeze(0)
        if masked_lm_labels is not None:
            out["masked_lm_loss"] = nn.functional.cross_entropy(
                scores_t.reshape(-1, self.vocab_size).float(), masked_lm_labels.reshape(-1), ignore_index=-1).unsqueeze(0)
        return out


class B200ViLBERTForClassification(nn.Module):
    """ViLBERTForClassification (vilbert.py:1246-1333)"""

    def __init__(self, config):
        super().__init__()
        from .vilbert import B200ViLBERTBase
        self.config = config
        bc = bert_config_of(config)
        self.bert = B200ViLBERTBase(bc)
        self.training_head_type = config.training_head_type
        self.num_labels = config.num_labels
        self.fusion_method = config.fusion_method
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        hidden = config.bi_hidden_size * (2 if self.training_head_type == "nlvr2" else 1)
        self.classifier = classifier_head(bc, hidden, self.num_labels)
        _init_bert_weights(self.classifier, float(config.get("initializer_range", 0.02)))

    def forward(self, input_ids, image_feature, image_location, token_type_ids=None, attention_mask=None,
                image_attention_mask=None, masked_lm_labels=None, image_label=None, image_target=None,
                next_sentence_label=None, output_all_attention_masks=False):
        seq_t, seq_v, pooled_t, pooled_v, _, _, _ = self.bert(
            input_ids, image_feature, image_location, token_type_ids, attention_mask, image_attention_mask,
            output_all_encoded_layers=False, output_all_attention_masks=output_all_attention_masks, reference_outputs=True)
        if self.fusion_method == "sum":
            pooled = self.dropout(pooled_t + pooled_v)
        elif self.fusion_method == "mul":
            pooled = self.dropout(pooled_t * pooled_v)
        else:
            raise AssertionError
        if self.training_head_type == "nlvr2":
            pooled = pooled.view(-1, pooled.size(1) * 2)
        logits = self.classifier(pooled)
        return {"scores": logits.contiguous().view(-1, self.num_labels).to(seq_t.dtype)}


@registry.register_model("vilbert")
class ViLBERT(BaseModel):
    @classmethod
    def config_path(cls):
        return "configs/models/vilbert/pretrain.yaml"

    @classmethod
    def format_state_key(cls, key):                                    # vilbert.py:1346-1352
        return key.replace("bert.bert", "model.bert").replace("bert.cls", "model.cls").replace(
            "bert.classifier", "model.classifier")

    def build(self):
        if self.config.training_head_type == "pretraining":
            self.model = B200ViLBERTForPretraining(self.config)
        else:
            self.model = B200ViLBERTForClassification(self.config)
        if self.config.get("freeze_base", False):
            for p in self.model.bert.parameters():
                p.requires_grad = False

    def get_image_and_text_features(self, sl):                         # vilbert.py:1364-1418
        ids, mask, seg = sl["input_ids"], sl["input_mask"], sl["segment_ids"]
        if _sl_get(sl, "dataset_name", None) == "nlvr2":
            ids, mask, seg = torch.cat([ids, ids]), torch.cat([mask, mask]), torch.cat([seg, seg])
            parts = []
            for name in ("img0", "img1"):
                img = _sl_get(sl, name, {})
                info = _sl_get(img, "image_info_0", {})
                parts.append((_sl_get(info, "max_features"), _sl_get(img, "image_feature_0"), _sl_get(info, "bbox")))
            dim = torch.cat([p[0] for p in parts])
            feat = torch.cat([p[1] for p in parts])
            loc = torch.cat([p[2] for p in parts])
            label = target = None
        else:
            info = _sl_get(sl, "image_info_0", {})
            dim, feat = _sl_get(info, "max_features", None), _sl_get(sl, "image_feature_0", None)
            label, loc = _sl_get(sl, "image_labels", None), _sl_get(info, "bbox", None)
            cls_prob = _sl_get(info, "cls_prob", None)
            target = None
            if cls_prob is not None:
                target = torch.as_tensor(cls_prob, dtype=torch.float, device=ids.device)
        return {"input_ids": ids, "attention_mask": mask, "token_type_ids": seg, "image_dim": dim, "image_feature": feat,
                "image_location": loc, "image_target": target, "image_label": label}

    def forward(self, sample_list):
        p = self.get_image_and_text_features(sample_list)
        p["masked_lm_labels"] = _sl_get(sample_list, "lm_label_ids", None)
        if p["image_feature"] is not None and p["image_dim"] is not None:
            p["image_attention_mask"] = image_mask_from_dim(p["image_feature"], p["image_dim"].to(p["image_feature"].device))
        else:
            p["image_attention_mask"] = None
        p.pop("image_dim")
        out = self.model(p["input_ids"], p["image_feature"], p["image_location"], p["token_type_ids"], p["attention_mask"],
                         p["image_attention_mask"], p["masked_lm_labels"], p["image_label"], p["image_target"])
        if self.config.training_head_type == "pretraining":
            key = "%s/%s" % (sample_list["dataset_name"], sample_list["dataset_type"])
            out["losses"] = {key + "/masked_lm_loss": out.pop("masked_lm_loss"),
                             key + "/masked_img_loss": out.pop("masked_img_loss")}
        return out


# ------------------------------------------------------------------------------------------------------
# MMBT
# ------------------------------------------------------------------------------------------------------
def _mmbt_base(config):
    from .mmbt import B200MMBTBase
    if not config.get("direct_features_input", False):
        raise NotImplementedError("MMBT with an image backbone (resnet152 modal encoder) is outside the fusion path; use "
                                  "`direct_features_input: true` (configs/models/mmbt/with_features.yaml)")
    return B200MMBTBase.from_config(config)


class B200MMBTForClassification(nn.Module):
    """MMBTForClassification (mmbt.py:521-562)"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.bert = _mmbt_base(config)
        self.encoder_config = self.bert.mmbt.config
        self.num_labels = config.num_labels
        self.fused_feature_only = config.get("fused_feature_only", False)
        self.dropout = nn.Dropout(float(self.encoder_config.hidden_dropout_prob))
        self.classifier = classifier_head(ConfigNode(vars(self.encoder_config)), self.encoder_config.hidden_size,
                                          self.num_labels)
        _init_bert_weights(self.classifier, float(getattr(self.encoder_config, "initializer_range", 0.02)))

    def forward(self, sample_list):
        pooled = self.dropout(self.bert(sample_list)[1])
        if self.fused_feature_only:
            return {"fused_feature": self.classifier[0](pooled)}
        logits = self.classifier(pooled)
        return {"scores": logits.contiguous().view(-1, self.num_labels).to(pooled.dtype)}


class B200MMBTForPreTraining(nn.Module):
    """MMBTForPreTraining (mmbt.py:447-518): MLM over the TEXT positions (the last T scores), decoder tied to the
    transformer's word embeddings"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.bert = _mmbt_base(config)
        self.encoder_config = self.bert.mmbt.config
        ec = ConfigNode(vars(self.encoder_config))
        self.cls = B200BertPreTrainingHeads(ec, self.bert.mmbt.transformer.embeddings.word_embeddings.weight)

    def forward(self, sample_list):
        out_seq, pooled = self.bert(sample_list)[:2]
        output = {}
        key = "%s/%s" % (sample_list["dataset_name"], sample_list["dataset_type"])
        labels = _sl_get(sample_list, "lm_label_ids", None)
        if labels is not None:
            T = labels.size(1)
            loss, logits = masked_lm_loss(self.cls, out_seq[:, -T:], labels, positions=self.config.get("mlm_positions", "all"))
            output["logits"] = logits
            output["losses"] = {key + "/masked_lm_loss": loss}
        return output


@registry.register_model("mmbt")
class MMBT(BaseModel):
    @classmethod
    def config_path(cls):
        return "configs/models/mmbt/pretrain.yaml"

    @classmethod
    def format_state_key(cls, key):                                    # mmbt.py:613-619
        return key.replace("base.bert", "model.bert").replace("base.cls", "model.cls").replace(
            "base.classifier", "model.classifier")

    def build(self):
        if self.config.training_head_type == "pretraining":
            self.model = B200MMBTForPreTraining(self.config)
        else:
            self.model = B200MMBTForClassification(self.config)
        if self.config.get("freeze_complete_base", False) or self.config.get("freeze_text", False):
            for p in self.model.bert.mmbt.transformer.parameters():
                p.requires_grad = False
        if self.config.get("freeze_complete_base", False) or self.config.get("freeze_modal", False):
            for p in self.model.bert.mmbt.modal_encoder.parameters():
                p.requires_grad = False

    def forward(self, sample_list):
        return self.model(sample_list)


# ------------------------------------------------------------------------------------------------------
# LXMERT
# ------------------------------------------------------------------------------------------------------
class B200LogitHead(nn.Sequential):
    """nn.Sequential(Linear(in, 2H), GeLU(), LayerNorm(2H, eps=1e-12), Linear(2H, out)) of BertVisualAnswerHead
    (lxmert.py:143-156), keys `0.*`, `2.*`, `3.*`: the first GEMM with the bias + GELU epilogue, the row LayerNorm, the
    output GEMM."""

    def __init__(self, in_dim, hid_dim, out_dim):
        super().__init__(nn.Linear(in_dim, hid_dim), nn.GELU(), nn.LayerNorm(hid_dim, eps=1e-12),
                         B200Linear(hid_dim, out_dim))

    def forward(self, x):
        shape = x.shape
        h = ops.linear_gelu(x.reshape(-1, shape[-1]), self[0].weight, self[0].bias)
        h = ops.layer_norm(h, self[2].weight, self[2].bias, self[2].eps)
        y = self[3](h)
        return y.view(*shape[:-1], y.shape[-1])


class B200BertVisualAnswerHead(nn.Module):
    """BertVisualAnswerHead (lxmert.py:129-162): `logit_fc`, plus `logit_gqa` when num_labels is the [num_labels,
    gqa_labels] pair; forward(h, name) takes `logit_gqa` when the dataset name contains "gqa"."""

    def __init__(self, config, num_labels):
        super().__init__()
        hid = config.hidden_size
        if config.training_head_type == "nlvr2":
            in_dim, out_dim = hid * 2, 2
        else:
            in_dim, out_dim = hid, config.num_labels
        if isinstance(num_labels, (list, tuple)):
            self.logit_gqa = B200LogitHead(in_dim, hid * 2, num_labels[1])
            out_dim = num_labels[0]
        self.logit_fc = B200LogitHead(in_dim, hid * 2, out_dim)

    def forward(self, hidden_states, name=None):
        if name is None or "gqa" not in name:
            return self.logit_fc(hidden_states)
        return self.logit_gqa(hidden_states)


class B200BertVisualObjHead(nn.Module):
    """BertVisualObjHead (lxmert.py:165-186): one transform, then `decoder_dict.<key>` per entry of visual_losses"""

    def __init__(self, config, visual_losses, visual_loss_config):
        super().__init__()
        self.transform = B200BertPredictionHeadTransform(config)
        self.visual_losses = list(visual_losses)
        self.decoder_dict = nn.ModuleDict({key: B200Linear(config.hidden_size, visual_loss_config[key][0])
                                           for key in self.visual_losses})

    def forward(self, hidden_states):
        h = self.transform(hidden_states)
        return {key: self.decoder_dict[key](h) for key in self.visual_losses}


_LXMERT_LOSSES = {
    "l2": lambda x, y: nn.functional.smooth_l1_loss(x, y, reduction="none"),
    "ce": lambda x, y: nn.functional.cross_entropy(x, y, ignore_index=-1, reduction="none"),
}


class B200LXMERTForPretraining(nn.Module):
    """LXMERTForPretraining (lxmert.py:417-572): trunk, `cls` (BertPreTrainingHeads with the decoder tied to the word
    embeddings), `obj_predict_head`, `answer_head`.  The losses are the reference's, in fp32 from the bf16 head outputs.
    The masked-LM loss runs on the fused vocabulary GEMM + cross-entropy (heads.masked_lm_loss(positions="fused")): the
    same loss without the [B, T, V] logits; a batch without a labelled position gives the zero loss documented there."""

    def __init__(self, config):
        super().__init__()
        from .lxmert import B200LXMERTBase
        self.config = config
        bc = bert_config_of(config)
        self.bert = B200LXMERTBase(bc)
        self.num_labels, self.gqa_labels = config.num_labels, config.gqa_labels
        self.task_mask_lm, self.task_obj_predict = config.task_mask_lm, config.task_obj_predict
        self.task_matched, self.task_qa = config.task_matched, config.task_qa
        self.visual_losses, self.visual_loss_config = list(config.visual_losses), config.visual_loss_config
        self.cls = B200BertPreTrainingHeads(bc, self.bert.embeddings.word_embeddings.weight)
        # the reference's own LM head has a bias-free decoder and one `predictions.bias` (lxmert.py:108-126): no
        # `decoder.bias` alias, so the state_dict keys are LXMERT's
        self.cls.predictions.decoder.register_parameter("bias", None)
        if self.task_obj_predict:
            self.obj_predict_head = B200BertVisualObjHead(bc, self.visual_losses, self.visual_loss_config)
        if self.task_qa:
            self.answer_head = B200BertVisualAnswerHead(bc, [self.num_labels, self.gqa_labels])
        for m in (getattr(self, "obj_predict_head", None), getattr(self, "answer_head", None)):
            if m is not None:
                _init_bert_weights(m, float(bc.initializer_range))

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, visual_feats=None, visual_pos=None,
                visual_attention_mask=None, masked_lm_labels=None, masked_image_labels=None, obj_labels=None,
                matched_label=None, ans=None, num_features=None, name=None, output_all_attention_masks=False,
                output_all_encoded_layers=False):
        (lang_output, visn_output), pooled_output = self.bert(
            input_ids, token_type_ids, attention_mask, visual_feats, visual_pos, visual_attention_mask,
            output_all_attention_masks, output_all_encoded_layers)
        output = {}
        if ans is not None and self.task_qa:
            answer_score = self.answer_head(pooled_output, name)
            n = self.config.num_labels if name is None or "gqa" not in name else self.config.gqa_labels
            output["answer_loss"] = nn.functional.cross_entropy(answer_score.reshape(-1, n).float(), ans.argmax(-1),
                                                                ignore_index=-1)
        if masked_lm_labels is not None and self.task_mask_lm:
            output["masked_lm_loss"] = masked_lm_loss(self.cls, lang_output, masked_lm_labels, positions="fused")[0]
        if matched_label is not None and self.task_matched:
            score = self.cls.seq_relationship(pooled_output)
            output["matched_loss"] = nn.functional.cross_entropy(score.reshape(-1, 2).float(), matched_label.long(),
                                                                 ignore_index=-1)
        if obj_labels is not None and self.task_obj_predict:
            total = 0.0
            scores = self.obj_predict_head(visn_output)
            for key in self.visual_losses:
                output_dim, loss_name, _, weight = self.visual_loss_config[key]
                if key == "attr":                                       # the reference skips it (lxmert.py:549-550)
                    continue
                if key == "obj":
                    top = obj_labels.max(-1)
                    mask_conf = top.values
                    loss = _LXMERT_LOSSES[loss_name](scores[key].reshape(-1, output_dim).float(), top.indices.reshape(-1))
                elif key == "feat":
                    mask_conf = (masked_image_labels == 1).float()
                    loss = _LXMERT_LOSSES[loss_name](scores[key].reshape(-1, output_dim).float(),
                                                     visual_feats.reshape(-1, output_dim).float())
                else:
                    raise NotImplementedError("LXMERT visual loss %r: the reference defines obj, attr and feat" % key)
                if loss.dim() > 1:                                      # regression losses
                    loss = loss.mean(1)
                total = total + (loss * mask_conf.reshape(-1)).mean() * weight
            output["visn_loss"] = total
        return output


class B200LXMERTForClassification(nn.Module):
    """LXMERTForClassification (lxmert.py:575-644): trunk + `classifier` (BertVisualAnswerHead over the pooled output;
    nlvr2 views it as [-1, 2H])"""

    def __init__(self, config):
        super().__init__()
        from .lxmert import B200LXMERTBase
        self.config = config
        self.num_labels, self.gqa_labels = config.num_labels, config.gqa_labels
        self.mode = config.mode
        bc = bert_config_of(config)
        self.bert = B200LXMERTBase(bc)
        self.classifier = B200BertVisualAnswerHead(bc, [self.num_labels, self.gqa_labels])
        _init_bert_weights(self.classifier, float(bc.initializer_range))

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, visual_feats=None, visual_pos=None,
                visual_attention_mask=None, masked_lm_labels=None, obj_labels=None, matched_label=None, ans=None,
                max_features=None, output_all_attention_masks=False, output_all_encoded_layers=False):
        (_, _), pooled_output = self.bert(input_ids, token_type_ids, attention_mask, visual_feats, visual_pos,
                                          visual_attention_mask, output_all_encoded_layers, output_all_attention_masks)
        if self.config.training_head_type == "nlvr2":
            pooled_output = pooled_output.view(-1, pooled_output.size(1) * 2)
        logits = self.classifier(pooled_output)
        return {"scores": logits.contiguous().view(-1, self.config.num_labels).to(pooled_output.dtype)}


# options of the reference's YAML that its LXMERT does not implement ("need to implement", defaults.yaml:63-73) or that
# only other models read: a value other than the default raises instead of being ignored
_LXMERT_UNSUPPORTED = ("dynamic_attention", "in_batch_pairs", "fast_mode", "output_attentions", "output_hidden_states",
                       "visualization")


@registry.register_model("lxmert")
class LXMERT(BaseModel):
    """The registered `lxmert` model (lxmert.py:647-786).

    The SampleList plumbing is the reference's, including its argument swap (lxmert.py:705-708): `input_mask` goes in as
    `token_type_ids` and `segment_ids` as `attention_mask`.  That is what MMF computes for this model, so it is what is
    computed here.  The text mask is then (1 - segment_ids) * -10000: with segment ids of 0 every text key gets -10000,
    and such a row is the softmax of the raw scores (DESIGN.md 4.2), as in the fp32 reference.

    Because of the swap the text "padding" is every token with segment id 0, [CLS] and the masked-LM positions included.
    Packing it away would zero those rows and change the losses, so forward() raises ValueError when the encoder's
    two-stream skip-padding (`pack_streams`) is set.  B200LXMERTBase called with real masks keeps the packed path."""

    @classmethod
    def config_path(cls):
        return "configs/models/lxmert/pretrain.yaml"

    def build(self):
        for key in _LXMERT_UNSUPPORTED:
            if self.config.get(key, False):
                raise NotImplementedError("LXMERT `%s: true` is not implemented (the reference's YAML marks it as not "
                                          "implemented or its LXMERT never reads it)" % key)
        if self.config.training_head_type == "pretraining":
            self.model = B200LXMERTForPretraining(self.config)
        else:
            self.model = B200LXMERTForClassification(self.config)
        if self.config.get("freeze_base", False):
            for p in self.model.bert.parameters():
                p.requires_grad = False

    def get_image_and_text_features(self, sl, device):               # lxmert.py:666-719
        feats = _sl_get(sl, "image_feature_0", None)
        R = feats.shape[1]
        info = _sl_get(sl, "image_info_0", {})
        bbox = _sl_get(info, "bbox", None)
        if bbox is not None:
            bbox = bbox[:, :R, :4]
        labels = _sl_get(sl, "image_labels", None)
        if labels is not None:
            labels = labels[:, :R, None].unsqueeze(-1).to(device)
        cls_prob = _sl_get(info, "cls_prob", None)
        if cls_prob is not None:
            cls_prob = torch.as_tensor(cls_prob)[:, :R, None].to(device)
        answers = _sl_get(sl, "targets", None)
        if answers is None:
            answers = _sl_get(sl, "answers", None)
        if answers is not None:
            answers = torch.as_tensor(answers).to(device)
        is_correct = _sl_get(sl, "is_correct", None)
        if is_correct is not None:
            is_correct = torch.as_tensor(is_correct).to(device)
        return {"input_ids": sl["input_ids"], "token_type_ids": sl["input_mask"], "attention_mask": sl["segment_ids"],
                "masked_lm_labels": _sl_get(sl, "lm_label_ids", None), "visual_feats": feats, "pos": bbox,
                "masked_image_labels": labels, "obj_labels": cls_prob, "matched_label": is_correct, "ans": answers,
                "image_dim": _sl_get(info, "max_features", None), "dataset_name": str(sl["dataset_name"])}

    def forward(self, sample_list):
        if self.model.bert.encoder._runner.pack_streams:
            raise ValueError("the registered LXMERT model passes segment_ids as the text attention mask (the reference's "
                             "argument swap, lxmert.py:707-708): its text padding is every segment-0 token, [CLS] and the "
                             "masked-LM positions included, so two-stream skip-padding would change the losses; turn it off "
                             "for this model (patch.set_skip_padding(model, False, two_stream=True))")
        p = self.get_image_and_text_features(sample_list, sample_list["input_ids"].device)
        if p["visual_feats"] is not None and p["image_dim"] is not None:
            p["image_attention_mask"] = image_mask_from_dim(p["visual_feats"], p["image_dim"].to(p["visual_feats"].device))
        else:
            p["image_attention_mask"] = None
        if self.config.training_head_type == "pretraining":
            out = self.model(input_ids=p["input_ids"], token_type_ids=p["token_type_ids"],
                             attention_mask=p["attention_mask"], visual_feats=p["visual_feats"], visual_pos=p["pos"],
                             visual_attention_mask=p["image_attention_mask"], masked_lm_labels=p["masked_lm_labels"],
                             masked_image_labels=p["masked_image_labels"], obj_labels=p["obj_labels"],
                             matched_label=p["matched_label"], ans=p["ans"], name=p["dataset_name"])
            key = "%s/%s" % (sample_list["dataset_name"], sample_list["dataset_type"])
            out["losses"] = {}
            for name in ("masked_lm_loss", "matched_loss", "visn_loss", "answer_loss"):
                if name in out:
                    out["losses"][key + "/" + name] = out.pop(name)
            return out
        return self.model(input_ids=p["input_ids"], token_type_ids=p["token_type_ids"],
                          attention_mask=p["attention_mask"], visual_feats=p["visual_feats"], visual_pos=p["pos"],
                          visual_attention_mask=p["image_attention_mask"])


from . import uniter_model  # noqa: E402,F401  (registers "uniter"; it needs the names defined above)
from . import vinvl_model  # noqa: E402,F401  (registers "vinvl"; it needs the names defined above)
from . import m4c_model  # noqa: E402,F401  (registers "m4c" and "m4c_captioner"; it needs the names defined above)
from . import vilt_model  # noqa: E402,F401  (registers "vilt"; it needs the names defined above)
