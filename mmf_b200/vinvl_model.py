"""The registered `vinvl` model on the fused trunk.

  registry.register_model("vinvl")  VinVL                        <->  mmf/models/vinvl.py:392-505
  B200VinVLForClassification                                     <->  :153-233
  B200VinVLForPretraining                                        <->  :236-389   (masked LM + three-way contrastive)

The trunk is mmf_b200.vinvl.B200VinVLBase; the heads come from the transformer-head table of mmf_b200.mmft (`mlp`, `mlm`,
`contrastive_three_way`).  State-dict keys equal the reference's: `vinvl.bert.*`, `vinvl.classifier.*`,
`vinvl.mlm_head.cls.predictions.*`, `vinvl.contrast_head.contrast_head.*`.  Pretraining runs the trunk twice per
forward (masked captions, then corrupt captions); both passes use the trunk's one ParamPack, and one backward sums their
gradients in its flat buffer.

What the reference does, and so what is done here:
  * `build()` looks the classifier up under `heads["mlp"]`, whatever other heads the config names: the default YAML's
    `heads.test` (and a project's `heads.vqa2`) is read by nobody, and classification gets MLPHead({"num_layers": 0}) -
    2 labels, pooler + one Linear - unless a head is configured under the key `mlp`;
  * the classifier's loss is `nn.CrossEntropyLoss(**ce_loss)` from the config key `ce_loss`; the YAML's
    `loss_type: sfmx` is read by nobody;
  * the masked-LM labels of the regions are -1 whatever the head's ignore_index; when no label of a batch is kept
    `masked_lm_loss` is 0 (the reference replaces the NaN of an empty mean), and the contrastive loss still trains;
  * the image mask is all ones when `image_info_0` has no `max_features`, else `arange(R) < max_features`, for
    `max_features` of shape [B] or [B, R] (any dtype), as int64;
  * a 3-D attention mask stays NotImplementedError in B200VinVLBase; the registered model always builds 2-D masks.
There is no hub here: `random_init` / `bert_model_name` select nothing but the bert-base hyper-parameters, and weights
arrive through load_state_dict.  (With `random_init` the reference constructs `VinVLBase(config)`, which never calls
`init_weights()`: its modules keep PyTorch's default initialisation - Kaiming-uniform Linear weights and uniform biases,
N(0, 1) embeddings.  B200VinVLBase initialises as HF's `_init_weights` does, N(0, 0.02) weights and zero biases.  Parity
is pinned on loaded weights.)  `bert_overrides`, a key the reference does not read, overrides those hyper-parameters
(e.g. a smaller model).  The masked-LM loss gathers a data-dependent number of rows, so GraphedStep refuses this model.
"""
import copy

import torch
from torch import nn

from .models import BERT_BASE, MODEL_DEFAULTS, BaseModel, ConfigNode, _sl_get, image_mask_from_dim
from .registry import registry
from .vinvl import B200VinVLBase

# mmf/configs/models/vinvl/defaults.yaml:1-18
MODEL_DEFAULTS["vinvl"] = dict(
    heads=dict(test=dict(type="mlp", freeze=False, lr_multiplier=1.0, in_dim=768, hidden_size=1536, num_labels=3129,
                         pooler_name="bert_pooler")),
    bert_model_name="bert-base-uncased", loss_type="sfmx", img_feature_dim=2054, img_feature_type="frcnn",
    use_img_layernorm=1, img_layer_norm_eps=1e-12, max_img_seq_len=70)

# VinVL.Config (vinvl.py:408-419); `heads` is MISSING there and comes from the YAML
CONFIG_DEFAULTS = dict(random_init=False, bert_model_name="bert-base-uncased", hidden_size=768, do_pretraining=False,
                       img_feature_dim=2054, img_feature_type="frcnn", use_img_layernorm=True, img_layer_norm_eps=1e-12,
                       max_img_seq_len=70)


def _heads():
    from . import mmft              # mmft imports models, which imports this module: resolved at construction time
    return mmft


def build_vinvl_base(bert_model_name="bert-base-uncased", img_feature_dim=2054, use_img_layernorm=True,
                     img_layer_norm_eps=1e-12, random_init=True, bert_overrides=None):
    """vinvl.py:124-150 without the hub: the bert-base BertConfig (overridden by `bert_overrides`) plus the three image
    keys"""
    cfg = ConfigNode(dict(BERT_BASE, **dict(bert_overrides or {})))
    cfg.img_feature_dim = int(img_feature_dim)
    cfg.use_img_layernorm = use_img_layernorm
    cfg.img_layer_norm_eps = float(img_layer_norm_eps)
    return B200VinVLBase(cfg)


class B200VinVLForClassification(nn.Module):
    def __init__(self, mlp_config=None, loss_config=None, random_init=False, bert_model_name="bert-base-uncased",
                 img_feature_dim=2054, use_img_layernorm=True, img_layer_norm_eps=1e-12, bert_overrides=None,
                 *args, **kwargs):
        super().__init__()
        if mlp_config is None:
            mlp_config = {"num_layers": 0}
        if loss_config is None:
            loss_config = {}
        self.bert = build_vinvl_base(bert_model_name, img_feature_dim, use_img_layernorm, img_layer_norm_eps, random_init,
                                     bert_overrides)
        self.classifier = _heads().MLPHead(mlp_config)
        self.ce_loss = nn.CrossEntropyLoss(**dict(loss_config))

    def forward(self, input_ids, token_type_ids, attention_mask, img_feats, position_ids=None, labels=None):
        sequence_output = self.bert(input_ids, img_feats=img_feats, position_ids=position_ids,
                                    token_type_ids=token_type_ids, attention_mask=attention_mask).last_hidden_state
        logits = self.classifier(sequence_output)["scores"]
        result = {"scores": logits}
        if labels is not None:
            result["losses"] = {"ce": self.ce_loss(logits.view(-1, logits.size(1)).float(), labels.view(-1))}
        return result


class B200VinVLForPretraining(nn.Module):
    """Masked LM on the masked captions and three-way contrastive classification (0 match, 1 corrupt caption, 2 corrupt
    image) on the corrupt ones: two trunk passes per forward."""

    def __init__(self, mlm_config=None, contrast_config=None, random_init=False, bert_model_name="bert-base-uncased",
                 img_feature_dim=2054, use_img_layernorm=True, img_layer_norm_eps=1e-12, bert_overrides=None,
                 *args, **kwargs):
        super().__init__()
        heads = _heads()
        self.bert = build_vinvl_base(bert_model_name, img_feature_dim, use_img_layernorm, img_layer_norm_eps, random_init,
                                     bert_overrides)
        self.mlm_head = heads.MLMHead(mlm_config if mlm_config is not None else {})
        self.ce_loss = nn.CrossEntropyLoss()
        self.contrast_head = heads.ThreeWayContrastiveHead(contrast_config if contrast_config is not None else {})

    def mlm_forward(self, input_ids_masked, lm_label_ids, token_type_ids, attention_mask, img_feats, position_ids=None):
        hidden = self.bert(input_ids_masked, img_feats=img_feats, position_ids=position_ids, token_type_ids=token_type_ids,
                           attention_mask=attention_mask).last_hidden_state
        mlm_labels = {"text": lm_label_ids,
                      "image": torch.full(img_feats.shape[:2], fill_value=-1, dtype=torch.long, device=lm_label_ids.device)}
        mlm_labels["combined_labels"] = torch.cat([mlm_labels["text"], mlm_labels["image"]], dim=-1)
        return self.mlm_head(hidden, processed_sample_list={"mlm_labels": mlm_labels})["losses"]

    def contrastive_forward(self, input_ids, token_type_ids, attention_mask, img_feats, contrastive_labels,
                            position_ids=None):
        last = self.bert(input_ids, img_feats=img_feats, position_ids=position_ids, token_type_ids=token_type_ids,
                         attention_mask=attention_mask).last_hidden_state
        return self.contrast_head(last, {"contrastive_labels": contrastive_labels})["losses"]

    def forward(self, input_ids_masked, input_ids_corrupt, lm_label_ids, contrastive_labels, token_type_ids,
                attention_mask, token_type_ids_corrupt, attention_mask_corrupt, img_feats, position_ids=None):
        mlm = self.mlm_forward(input_ids_masked, lm_label_ids, token_type_ids, attention_mask, img_feats, position_ids)
        contrastive = self.contrastive_forward(input_ids_corrupt, token_type_ids_corrupt, attention_mask_corrupt,
                                               img_feats, contrastive_labels, position_ids)
        return {"losses": {**mlm, **contrastive}}


@registry.register_model("vinvl")
class VinVL(BaseModel):
    """VinVL (vinvl.py:392-505): Oscar-style BERT over caption tokens and detector region features"""

    graph_capturable = False        # see mmf_b200.graphs.GraphedStep
    graph_refusal = "gathers a data-dependent number of rows (the labelled masked-LM positions) in every pretraining forward"
    static_rows_capturable = True   # that gather is the only refusal: GraphedStep(..., static_rows=True) captures the step

    def __init__(self, config):
        super().__init__(config)
        self.config = ConfigNode(dict(copy.deepcopy(CONFIG_DEFAULTS), **self.config))
        self.do_pretraining = self.config.do_pretraining

    @classmethod
    def config_path(cls):
        return "configs/models/vinvl/defaults.yaml"

    def build(self):
        kwargs = {k: v for k, v in self.config.items() if k not in ("mlm_config", "contrast_config", "mlp_config",
                                                                     "loss_config")}
        if self.do_pretraining:
            self.vinvl = B200VinVLForPretraining(mlm_config=self.config.heads.get("mlm"),
                                                 contrast_config=self.config.heads.get("contrast"), **kwargs)
        else:
            self.vinvl = B200VinVLForClassification(mlp_config=self.config.heads.get("mlp"),
                                                    loss_config=self.config.get("ce_loss"), **kwargs)

    def init_losses(self):
        """Defer loss management to submodels, do nothing when called by build_model."""

    def forward(self, sample_list):
        attention_mask = self._get_attention_mask(sample_list["image_feature_0"], sample_list["image_info_0"],
                                                  sample_list["input_mask"])
        if self.do_pretraining:
            corrupt_attention_mask = self._get_attention_mask(sample_list["image_feature_0"], sample_list["image_info_0"],
                                                              sample_list["input_mask_corrupt"])
            return self.vinvl(sample_list["input_ids_masked"], sample_list["input_ids_corrupt"],
                              sample_list["lm_label_ids"], sample_list["contrastive_labels"], sample_list["segment_ids"],
                              attention_mask, sample_list["segment_ids_corrupt"], corrupt_attention_mask,
                              sample_list["image_feature_0"])
        return self.vinvl(sample_list["input_ids"], sample_list["segment_ids"], attention_mask,
                          sample_list["image_feature_0"], labels=sample_list.get("labels"))

    def _get_attention_mask(self, image_feat, image_info, input_mask):
        image_dim = _sl_get(image_info, "max_features")
        if image_dim is None:
            image_mask = torch.ones((image_feat.size(0), image_feat.size(1)), device=image_feat.device).long()
        else:
            image_mask = image_mask_from_dim(image_feat, torch.as_tensor(image_dim, device=image_feat.device))
        return torch.cat((input_mask, image_mask), dim=-1)
