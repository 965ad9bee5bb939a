"""MMFTransformer model plugin on the B200 engine (BASELINE.json configs[3]).

  registry.register_model("mmft") / ("mmf_transformer")  MMFTransformer  <->  mmf/models/mmf_transformer.py:35-442
      preprocess_sample + the `_infer_*` family (:176-392): per-modality input ids / position ids / segment ids / masks /
      MLM labels (with `combined_labels`) / ITM labels - INTEGER paths, bit-exact with the reference's known answers
      (its tests/models/test_mmf_transformer.py:205-402, mirrored in tests/test_mmft_cpu.py)
      forward (:394-419): backend(input_ids, position_ids, segment_ids, masks) -> heads
  heads (registry "transformer_head" table of the reference):
      "mlp"  MLPHead  <-> mmf/models/transformers/heads/mlp.py:19-96    pooler -> [dropout, transform] x n -> Linear
      "mlm"  MLMHead  <-> heads/mlm.py:20-97     labelled positions gathered FIRST, transform -> vocabulary decoder -> CE
      "mlm_multi" MLMForMultiHeads <-> heads/mlm.py:101-113   the "mlm" head on the sample list's `hs_masked_for_mlm`
      "itm"  ITMHead  <-> heads/itm.py:19-74     pooler -> Linear(H, 2) -> CE
      "mrc"  MRCHead  <-> heads/mrc.py:15-90     masked regions -> Linear -> GELU -> LayerNorm -> Linear(1601) -> KL / CE
      "mrfr" MRFRHead <-> heads/mrfr.py:15-93    masked regions -> Linear -> GELU -> LayerNorm -> tied projection -> MSE
      "wra"  WRAHead  <-> heads/wra.py:13-83     optimal-transport distance of text rows x region rows (one kernel)
      "contrastive_three_way"  ThreeWayContrastiveHead  <-> heads/contrastive.py:14-79   MLPHead(num_labels=3) -> CE
  build_heads_dict / HeadsDict  <-> heads/utils.py:11-166   per-task head lists, configured losses, summed losses / scores

The backend is the registered "b200" transformer backend (mmf_b200.mmft_backend); a config that says `backend.type:
huggingface` (the reference default, configs/models/mmf_transformer/defaults.yaml:4-7) is served by it as well - that is
the drop-in.  `transformer_base` cannot be downloaded here: the BERT-base hyper-parameters are used and overridden by
`backend.params` / `transformer_config` keys; weights arrive through load_state_dict.
"""
import collections.abc
import warnings

import torch
from torch import nn

from . import functional as F
from . import ops
from .encoders import build_encoder
from .graphs import static_rows_active
from .heads import B200BertLMPredictionHead, B200BertPredictionHeadTransform, static_masked_lm_loss
from .models import BERT_BASE, MODEL_DEFAULTS, B200Linear, BaseModel, ConfigNode
from .modules import _init_bert_weights
from .registry import registry
from .visual_bert import BertPooler

# mmf/configs/models/mmf_transformer/defaults.yaml:1-41 (the heads' num_labels interpolation resolved)
MODEL_DEFAULTS["mmf_transformer"] = dict(
    transformer_base="bert-base-uncased", backend=dict(type="huggingface", freeze=False, params={}),
    heads=[dict(type="mlp", freeze=False, lr_multiplier=1.0, hidden_size=768, num_labels=2)],
    modalities=[
        dict(type="text", key="text", position_dim=512, segment_id=0, embedding_dim=768, layer_norm_eps=1e-12,
             hidden_dropout_prob=0.1),
        dict(type="image", key="image", embedding_dim=2048, position_dim=1, segment_id=1, layer_norm_eps=1e-12,
             hidden_dropout_prob=0.1,
             encoder=dict(type="resnet152", params=dict(pretrained=True, pool_type="avg", num_output_features=1)))],
    initializer_range=0.02, initializer_mean=0.0, token_noise_std=0.01, token_noise_mean=0.0, layer_norm_weight_fill=1.0,
    random_initialize=False, freeze_image_encoder=False, tie_weight_to_encoder=None, num_labels=2)
MODEL_DEFAULTS["mmft"] = MODEL_DEFAULTS["mmf_transformer"]

HEADS = {}


def register_transformer_head(name):
    def wrap(cls):
        HEADS[name] = cls
        return cls
    return wrap


# ------------------------------------------------------------------------------------------------------
# heads
# ------------------------------------------------------------------------------------------------------
class _TransformWithInDim(B200BertPredictionHeadTransform):
    """PredictionHeadTransformWithInDim (mlp.py:90-93): the transform's dense maps in_dim -> hidden_size"""

    def __init__(self, config):
        super().__init__(config)
        self.dense = nn.Linear(config.in_dim, config.hidden_size)


@register_transformer_head("multilayer_mlp")
@register_transformer_head("mlp")
class MLPHead(nn.Module):
    DEFAULTS = dict(type="mlp", num_labels=2, hidden_size=768, hidden_dropout_prob=0.1, layer_norm_eps=1e-6,
                    hidden_act="gelu", pooler_name="bert_pooler", num_layers=1, in_dim=None)      # mlp.py:22-32

    def __init__(self, config):
        super().__init__()
        self.config = c = ConfigNode(dict(self.DEFAULTS, **dict(config)))
        self.num_labels, self.hidden_size = c.num_labels, c.hidden_size
        self.in_dim = c.in_dim = c.hidden_size if c.in_dim is None else c.in_dim
        if c.pooler_name == "bert_pooler":
            self.pooler = BertPooler(self.in_dim)
        elif c.pooler_name == "identity":
            self.pooler = nn.Identity()
        else:
            raise NotImplementedError("%s is not implemented." % c.pooler_name)
        if c.num_layers < 0:
            raise AssertionError("num_layers must be >= 0")
        layers, hc = [], ConfigNode(dict(c))
        for _ in range(c.num_layers):
            layers.append(nn.Dropout(c.hidden_dropout_prob))
            layers.append(_TransformWithInDim(ConfigNode(dict(hc))))
            hc.in_dim = hc.hidden_size
        self.classifier = nn.Sequential(*layers, B200Linear(self.hidden_size, self.num_labels))

    def forward(self, sequence_output, encoded_layers=None, processed_sample_list=None):
        assert sequence_output.size(-1) == self.in_dim, "Mismatch between MLP head hidden_size and sequence_output last dim."
        pooled = self.pooler(sequence_output)
        return {"scores": self.classifier(pooled).reshape(-1, self.num_labels).to(sequence_output.dtype)}


@register_transformer_head("mlm")
class MLMHead(nn.Module):
    DEFAULTS = dict(type="mlm", vocab_size=30522, hidden_size=768, hidden_dropout_prob=0.1, layer_norm_eps=1e-5,
                    hidden_act="gelu", ignore_index=-1, loss_name="masked_lm_loss", label_key=None)   # mlm.py:23-32

    def __init__(self, config):
        super().__init__()
        self.config = c = ConfigNode(dict(self.DEFAULTS, **dict(config)))
        self.cls = nn.Module()                                     # BertOnlyMLMHead: `cls.predictions.*`
        self.cls.predictions = B200BertLMPredictionHead(c)
        self.vocab_size = c.vocab_size

    def tie_weights(self, module=None):
        self.cls.predictions.decoder.weight = module.weight

    def forward(self, sequence_output, encoded_layers=None, processed_sample_list=None):
        assert processed_sample_list is not None, "MLM head requires 'processed_sample_list' argument"
        c = self.config
        if c.label_key is not None:
            assert c.label_key in processed_sample_list
            labels = processed_sample_list[c.label_key]
        else:
            assert processed_sample_list.get("mlm_labels") is not None
            assert "combined_labels" in processed_sample_list["mlm_labels"]
            labels = processed_sample_list["mlm_labels"]["combined_labels"]
        if static_rows_active():
            # rows selected and counted on the device (mmf_b200.graphs.static_rows): capturable, no logits, no warning
            loss = static_masked_lm_loss(self.cls.predictions, sequence_output, labels, c.ignore_index)
            return {"logits": None, "losses": {c.loss_name: loss}}
        sel = labels.ne(c.ignore_index)                             # gather the labelled rows first (mlm.py:79-82)
        labels = labels[sel]
        if labels.numel() == 0:
            # CrossEntropyLoss over zero targets is NaN, which the reference replaces by 0 (mlm.py:89-93)
            warnings.warn("NaN detected in masked_lm_loss. Replacing it with 0.")
            return {"logits": sequence_output.new_zeros(0, self.vocab_size),
                    "losses": {c.loss_name: sequence_output.sum() * 0.0}}
        rows = sequence_output[sel, :]
        logits = self.cls.predictions(rows)
        loss = nn.functional.cross_entropy(logits.reshape(-1, self.vocab_size).float(), labels.reshape(-1),
                                           ignore_index=c.ignore_index)
        return {"logits": logits, "losses": {c.loss_name: loss}}


@register_transformer_head("mlm_multi")
class MLMForMultiHeads(nn.Module):
    """heads/mlm.py:101-113: the `mlm` head (as `mlm_head`) run on the sample list's `hs_masked_for_mlm` - the trunk
    output of a second pass over the masked captions (ViLT's _encode_mlm) - instead of the sequence it is handed"""

    def __init__(self, config):
        super().__init__()
        self.config = ConfigNode(dict(config))
        self.mlm_head = MLMHead(config)

    def forward(self, _, processed_sample_list):
        return self.mlm_head(processed_sample_list["hs_masked_for_mlm"], processed_sample_list=processed_sample_list)


@register_transformer_head("itm")
class ITMHead(nn.Module):
    DEFAULTS = dict(type="itm", hidden_size=768, loss_name="itm_loss", ignore_index=-1, itm_label_key="is_correct")   # itm.py:22-27

    def __init__(self, config):
        super().__init__()
        self.config = c = ConfigNode(dict(self.DEFAULTS, **dict(config)))
        self.pooler = BertPooler(c.hidden_size)
        self.cls = nn.Module()                                     # BertOnlyNSPHead: `cls.seq_relationship`
        self.cls.seq_relationship = B200Linear(c.hidden_size, 2)

    def forward(self, sequence_output, encoded_layers=None, processed_sample_list=None):
        assert processed_sample_list is not None, "ITM head requires 'processed_sample_list' argument"
        c = self.config
        if c.itm_label_key in processed_sample_list:
            labels = processed_sample_list[c.itm_label_key]
        else:
            assert processed_sample_list.get("itm_labels") is not None
            labels = processed_sample_list["itm_labels"][c.itm_label_key]
        score = self.cls.seq_relationship(self.pooler(sequence_output))
        loss = nn.functional.cross_entropy(score.reshape(-1, 2).float(), labels.reshape(-1), ignore_index=c.ignore_index)
        return {"losses": {c.loss_name: loss}}


CONTRASTIVE_LABEL_KEY = "three_way_constrastive_labels"          # the reference's spelling (contrastive.py:11)


@register_transformer_head("contrastive_three_way")
class ThreeWayContrastiveHead(nn.Module):
    """VinVL's three-way contrastive head (heads/contrastive.py:14-79): an MLPHead built from the head's own merged config
    (pooler -> Linear(H, 3) with the defaults), cross-entropy over 0 = match, 1 = corrupt caption, 2 = corrupt image.
    Parameters `contrast_head.pooler.dense.*`, `contrast_head.classifier.0.*`.

    The reference's forward takes (sequence_output, processed_sample_list), which MMFT's three-argument head call
    (sequence_output, encoded_layers, processed_sample_list) does not fit; here the sample list is the last positional
    argument (or the keyword), so both call forms work."""
    DEFAULTS = dict(type="three_way_contrastive", freeze=False, lr_multiplier=1.0, hidden_size=768,
                    loss_name="three_way_contrastive_loss", ignore_index=-1, constrastive_label_key="contrastive_labels",
                    num_layers=0, num_labels=3, hidden_dropout_prob=0.1, layer_norm_eps=1e-6, hidden_act="gelu",
                    pooler_name="bert_pooler", in_dim=None)          # contrastive.py:26-39

    def __init__(self, config):
        super().__init__()
        self.config = c = ConfigNode(dict(self.DEFAULTS, **dict(config)))
        self.contrast_head = MLPHead(c)

    def forward(self, sequence_output, *args, processed_sample_list=None):
        if processed_sample_list is None and args:
            processed_sample_list = args[-1]
        c = self.config
        if c.constrastive_label_key in processed_sample_list:
            labels = processed_sample_list[c.constrastive_label_key]
        else:
            assert (CONTRASTIVE_LABEL_KEY in processed_sample_list
                    and processed_sample_list[CONTRASTIVE_LABEL_KEY] is not None), (
                "Constrastive three way pretraining requires %s to be in sample list with value not None."
                % CONTRASTIVE_LABEL_KEY)
            labels = processed_sample_list[CONTRASTIVE_LABEL_KEY][c.constrastive_label_key]
        scores = self.contrast_head(sequence_output)["scores"]
        loss = nn.functional.cross_entropy(scores.reshape(-1, 3).float(), labels.reshape(-1), ignore_index=c.ignore_index)
        return {"losses": {c.loss_name: loss}}


def _head_from_config(config):
    head_type = config.get("type", "mlp")
    if head_type not in HEADS:
        raise NotImplementedError("transformer head %r is not on the B200 path (have: %s)" % (head_type, sorted(HEADS)))
    return HEADS[head_type](config)


def build_heads_dict(head_configs, tasks, losses):
    """heads/utils.py:11-66: a list of head configs gives one nn.ModuleList for every task; a task-keyed mapping gives an
    nn.ModuleDict of one ModuleList per task of `tasks` (a task without a head raises ValueError).  Each head's `loss`
    names the entry of `losses` applied to a head that returns no losses itself."""
    if isinstance(head_configs, collections.abc.Sequence):
        heads = nn.ModuleList([_head_from_config(c) for c in head_configs])
        head_loss_names = [c.get("loss") for c in head_configs]
        head_names = [c.get("type", "mlp") for c in head_configs]
    if isinstance(head_configs, collections.abc.Mapping):
        heads, head_names, head_loss_names = nn.ModuleDict(), {}, {}
        for task in tasks:
            head_config = head_configs.get(task)
            if head_config is None:
                raise ValueError("No head defined for %s. Dataset task %s requires a head to return dict with 'losses'"
                                 % (task, task))
            config_list = head_config if isinstance(head_config, collections.abc.Sequence) else [head_config]
            heads[task] = nn.ModuleList([_head_from_config(c) for c in config_list])
            head_loss_names[task] = [c.get("loss") for c in config_list]
            head_names[task] = [c.get("type", "mlp") for c in config_list]
    return HeadsDict(heads, head_names, losses, head_loss_names)


class HeadsDict(nn.Module):
    """heads/utils.py:69-166: runs every head of a task on the sequence; a head that returns no `losses` gets its
    configured loss applied to its scores (flattened to [-1, n]); losses that share a key are summed, and so are the
    scores (a head without scores counts as 0)."""

    def __init__(self, heads, head_names, losses, head_loss_names):
        super().__init__()
        self.heads = heads
        self.head_names = head_names
        self.losses = losses
        self.head_loss_names = head_loss_names

    def forward(self, task, sequence, sample_list):
        if isinstance(self.heads, nn.ModuleList):
            modules, loss_names, names = self.heads, self.head_loss_names, self.head_names
        else:
            modules, loss_names, names = self.heads[task], self.head_loss_names[task], self.head_names[task]
        outputs_list = [head(sequence, processed_sample_list=sample_list) for head in modules]
        assert len(loss_names) == len(outputs_list)
        processed = [self._process_head_output(o, ln, hn, sample_list)
                     for o, ln, hn in zip(outputs_list, loss_names, names)]
        loss_result = {}
        for output in processed:
            for k, v in output["losses"].items():
                loss_result[k] = loss_result[k] + v if k in loss_result else v
        return {"losses": loss_result, "scores": sum([output.get("scores", 0) for output in processed])}

    def _process_head_output(self, outputs, loss_name, head_name, sample_list):
        if isinstance(outputs, collections.abc.MutableMapping) and "losses" in outputs:
            return outputs
        if isinstance(outputs, collections.abc.MutableMapping) and "scores" in outputs:
            logits = outputs["scores"]
        else:
            logits = outputs
        logits = logits.contiguous().view(-1, logits.size(-1))
        if loss_name is None:
            raise ValueError("Transformer head %s must either define a 'loss' in its config or return a dict that "
                             "contains key 'losses'." % head_name)
        return {"losses": self.losses[loss_name](sample_list, {"scores": logits}), "scores": logits}


def compute_masked_hidden(hidden, mask):
    """heads/utils.py:169-179: the rows of hidden [B, S, H] where the bool mask [B, S] is True, as [n, H]"""
    mask = mask.unsqueeze(-1).expand_as(hidden)
    return hidden[mask].contiguous().view(-1, hidden.size(-1))


def _required(processed_sample_list, key, head):
    assert key in processed_sample_list and processed_sample_list[key] is not None, (
        "%s pretraining requires %s to be in sample list with value not None." % (head, key))
    return processed_sample_list[key]


def _linear_gelu_ln(seq, x, count=None):
    """nn.Sequential(Linear, GELU, LayerNorm) of the region heads: GEMM with the GELU epilogue, then the row LayerNorm;
    with `count` (int32 [1] on the device) both and their backward are bounded by it, and rows past it are zero"""
    h = ops.linear_gelu(x, seq[0].weight, seq[0].bias, count)
    return ops.layer_norm(h, seq[2].weight, seq[2].bias, seq[2].eps, count)


def _static_region_rows(seq, sequence_output, masks, targets):
    """Static-rows form of compute_masked_hidden + the region transform: inside graphs.static_rows() the label / target
    entry holds every region's target [B, R, D] and the regions are the last R rows of the sequence (UNITER's layout:
    text, then regions).  The masked regions are selected on the device into a fixed capacity of B * R rows
    (F.select_rows over the region mask), gathered, and run through Linear -> GELU -> LayerNorm bounded by the device
    count.  Returns (h, selection, fp32 targets [B * R, D])."""
    B, R, D = targets.shape
    H = sequence_output.shape[-1]
    region = masks[:, masks.shape[1] - R:].reshape(-1).to(torch.int64).contiguous()
    sel = F.select_rows(region, 0)
    rows = ops.gather_rows(sequence_output[:, sequence_output.shape[1] - R:].reshape(B * R, H), sel)
    return _linear_gelu_ln(seq, rows, sel.count), sel, targets.reshape(B * R, D).float().contiguous()


def _static_region_loss(seq, sequence_output, masks, targets, kind, projection=None):
    """MRC's KL loss (kind "kl", the classifier's last Linear) or MRFR's mean squared error (kind "mse", the tied
    projection read MN-major) over the masked regions, bounded by their device count: 0 with zero gradients when no
    region is masked"""
    h, sel, tgt = _static_region_rows(seq, sequence_output, masks, targets)
    if kind == "kl":
        last = seq[3]
        return ops.region_loss_static(h, last.weight, last.bias, tgt, sel.pos, sel.count, sel.scale, "kl")
    weight, bias = projection
    return ops.region_loss_static(h, weight, bias, tgt, sel.pos, sel.count, sel.scale * (1.0 / tgt.shape[1]), "mse",
                                  weight_t=True)


def _static_region_ce(seq, sequence_output, masks, targets, ignore_index):
    """MRC without KL: cross-entropy against the arg-max of each target row past the background class, found on the
    device, through the bounded cross-entropy row kernel.  The 1601-wide projection is padded to a multiple of 8 with a
    -30000 bias, so the padding columns vanish from the softmax."""
    h, sel, tgt = _static_region_rows(seq, sequence_output, masks, targets)
    labels = torch.max(tgt[:, 1:], dim=-1)[1] + 1
    labels = torch.where(sel.pos >= 0, labels.index_select(0, sel.pos.clamp_min(0)).to(torch.int64),
                         torch.full_like(labels, ignore_index))
    last = seq[3]
    return ops.linear_cross_entropy(h, last.weight, last.bias, labels, ignore_index, count=sel.count, scale=sel.scale)


@register_transformer_head("mrc")
class MRCHead(nn.Module):
    """Masked region classification (heads/mrc.py:15-90); parameters `region_classifier.{0,2,3}.*`"""

    def __init__(self, hidden_size=768, loss_name="mrc_loss", ignore_index=-1, mrc_label_key="region_class",
                 mrc_mask_key="image_region_mask", label_dim=1601, eps=1e-12, use_kl=True, *args, **kwargs):
        super().__init__()
        self.loss_name, self.ignore_index, self.use_kl = loss_name, ignore_index, use_kl
        self.mrc_label_key, self.mrc_mask_key = mrc_label_key, mrc_mask_key
        self.region_classifier = nn.Sequential(nn.Linear(hidden_size, hidden_size), nn.GELU(),
                                               nn.LayerNorm(hidden_size, eps=eps), nn.Linear(hidden_size, label_dim))

    def forward(self, sequence_output, encoded_layers=None, processed_sample_list=None):
        region_labels = _required(processed_sample_list, self.mrc_label_key, "MRC")
        masks = _required(processed_sample_list, self.mrc_mask_key, "MRC")
        if static_rows_active():
            if self.use_kl:
                loss = _static_region_loss(self.region_classifier, sequence_output, masks, region_labels, "kl")
            else:
                loss = _static_region_ce(self.region_classifier, sequence_output, masks, region_labels,
                                         self.ignore_index)
            return {"losses": {self.loss_name: loss}}
        h = _linear_gelu_ln(self.region_classifier, compute_masked_hidden(sequence_output, masks))
        last = self.region_classifier[3]
        logits = ops.linear_any(h, last.weight, last.bias).float()       # label_dim = 1601 is not a multiple of 8
        if self.use_kl:
            loss = nn.functional.kl_div(nn.functional.log_softmax(logits, dim=-1), region_labels.float(),
                                        reduction="batchmean")
        else:
            targets = torch.max(region_labels[:, 1:], dim=-1)[1] + 1      # background class should not be the target
            loss = nn.functional.cross_entropy(logits, targets, ignore_index=self.ignore_index, reduction="mean")
        return {"losses": {self.loss_name: loss}}


@register_transformer_head("mrfr")
class MRFRHead(nn.Module):
    """Masked region feature regression (heads/mrfr.py:15-93).  `linear_proj_weight` IS the image embedding's projection
    weight [hidden, img_dim] (one Parameter under two names, as in the reference); the projection back to the feature
    space reads it transposed, in place (ops.linear_t), and autograd adds both uses' gradients."""

    def __init__(self, img_embedding_weight, hidden_size=768, loss_name="mrfr_loss", mrfr_target_key="mrfr_region_target",
                 mrfr_mask_key="mrfr_region_mask", img_dim=2048, eps=1e-12, *args, **kwargs):
        super().__init__()
        self.loss_name, self.mrfr_target_key, self.mrfr_mask_key = loss_name, mrfr_target_key, mrfr_mask_key
        assert img_embedding_weight is not None and tuple(img_embedding_weight.shape) == (hidden_size, img_dim), (
            "MRFR head requires 'img_embedding_weight' with shape (%d, %d)." % (hidden_size, img_dim))
        self.linear_proj_weight = img_embedding_weight
        self.linear_proj_bias = nn.Parameter(torch.zeros(img_dim))
        self.feat_regress = nn.Sequential(nn.Linear(hidden_size, hidden_size), nn.GELU(), nn.LayerNorm(hidden_size, eps=eps))

    def forward(self, sequence_output, encoded_layers=None, processed_sample_list=None):
        feat_targets = _required(processed_sample_list, self.mrfr_target_key, "MRFR")
        masks = _required(processed_sample_list, self.mrfr_mask_key, "MRFR")
        if static_rows_active():
            loss = _static_region_loss(self.feat_regress, sequence_output, masks, feat_targets, "mse",
                                       (self.linear_proj_weight, self.linear_proj_bias))
            return {"losses": {self.loss_name: loss}}
        h = _linear_gelu_ln(self.feat_regress, compute_masked_hidden(sequence_output, masks))
        prediction = ops.linear_t(h, self.linear_proj_weight, self.linear_proj_bias)
        loss = nn.functional.mse_loss(prediction.float(), feat_targets.float(), reduction="mean")
        return {"losses": {self.loss_name: loss}}


@register_transformer_head("wra")
class WRAHead(nn.Module):
    """Word-region alignment (heads/wra.py:13-83): the optimal-transport distance between each sample's text rows and
    region rows - cost, IPOT plan and distance in one kernel (ops.optimal_transport_dist) - positives minus negatives.

    The kernel takes lengths, not masks: `txt_pad` / `img_pad` must mark a suffix of each row as padding, which is what
    UNITER's `_preprocess_wra` builds (uniter.py:560-583).  `wra_info` may carry the lengths as host lists (`txt_lens`,
    `img_lens`); otherwise they are read back from the pads, and a pad that is not a suffix raises ValueError."""

    def __init__(self, loss_name="wra_loss", ot_inputs_key="wra_info", wra_label_key="is_correct", *args, **kwargs):
        super().__init__()
        self.loss_name, self.ot_inputs_key, self.wra_label_key = loss_name, ot_inputs_key, wra_label_key

    @staticmethod
    def _lengths(pad, lens, width, what):
        if lens is not None:
            return [int(v) for v in lens]
        pad = pad.bool().cpu()
        n = (~pad).sum(1)
        if pad.size(1) != width or not torch.equal(pad, torch.arange(width).unsqueeze(0) >= n.unsqueeze(1)):
            raise ValueError("WRA: %s must be [B, %d] and mark a suffix of each row as padding" % (what, width))
        return n.tolist()

    def forward(self, sequence_output, encoded_layers=None, processed_sample_list=None):
        ot_inputs = _required(processed_sample_list, self.ot_inputs_key, "WRA")
        assert ot_inputs.get("txt_pad") is not None and ot_inputs.get("img_pad") is not None, (
            "WRA pretraining requires 'txt_pad', and 'img_pad' to be in 'processed_sample_list[%s]' with values not None."
            % self.ot_inputs_key)
        assert processed_sample_list.get(self.wra_label_key) is not None, (
            "WRA pretraining requires %s to be in sample list with value not None." % self.wra_label_key)
        tl = processed_sample_list["input_ids"].size(1)
        il = processed_sample_list["image_feat"].size(1)
        x_len = self._lengths(ot_inputs["txt_pad"], ot_inputs.get("txt_lens"), tl, "txt_pad")
        y_len = self._lengths(ot_inputs["img_pad"], ot_inputs.get("img_lens"), il, "img_pad")
        itm_labels = processed_sample_list[self.wra_label_key]
        ot_dist = ops.optimal_transport_dist(sequence_output, tl, il, x_len, y_len).to(sequence_output.dtype)
        if static_rows_active():
            # the same loss from masked sums and a device count: nothing is read on the host
            pos, neg = itm_labels == 1, itm_labels == 0
            zero = ot_dist.new_zeros(())
            total = torch.where(pos, ot_dist, zero).sum() - torch.where(neg, ot_dist, zero).sum()
            return {"losses": {self.loss_name: total / (pos.sum() + neg.sum()).to(ot_dist.dtype)}}
        ot_pos = ot_dist.masked_select(itm_labels == 1)
        ot_neg = ot_dist.masked_select(itm_labels == 0)
        loss = (ot_pos.sum() - ot_neg.sum()) / (ot_pos.size(0) + ot_neg.size(0))
        return {"losses": {self.loss_name: loss}}


# ------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------
def _text_slice(tensor, text_index):
    """stacked text fields [B, n_text, L] hold one row per text modality, in config order (mmf_transformer.py:233-241)"""
    return (tensor[:, text_index], text_index + 1) if tensor.dim() > 2 else (tensor, text_index)


@registry.register_model("mmft")
@registry.register_model("mmf_transformer")
class MMFTransformer(BaseModel):
    def __init__(self, config, *args, **kwargs):
        super().__init__(config)
        self.modality_keys, self.modality_type, self.modality_segments = [], [], []
        for m in self.config.modalities:
            self.modality_keys.append(m["key"])
            self.modality_type.append(m["type"])
            self.modality_segments.append(m["segment_id"] if "segment_id" in m else -1)

    @classmethod
    def config_path(cls):
        return "configs/models/mmf_transformer/defaults.yaml"

    @classmethod
    def format_state_key(cls, key):                                # mmf_transformer.py:97-104
        if key.startswith("pooler.") or key.startswith("classifier."):
            return key.replace("pooler.", "heads.0.pooler.").replace("classifier.", "heads.0.classifier.")
        return key

    # ---- construction (transformers/base.py:100-111, 170-238) ----
    def build(self):
        self.build_backend()
        self.build_encoders()
        self.build_heads()
        self.init_weights()

    def _transformer_config(self):
        tc = dict(BERT_BASE)
        tc.update(dict(self.config.get("transformer_config", {}) or {}))
        tc.update(dict((self.config.get("backend", {}) or {}).get("params", {}) or {}))
        return ConfigNode(tc)

    def build_backend(self):
        backend_config = self.config.get("backend", {}) or {}
        btype = backend_config.get("type", "huggingface")
        # the reference's default type is served by the B200 backend: that IS the drop-in for this path
        from . import mmft_backend  # noqa: F401  (registers "b200")
        cls = registry.get_transformer_backend_class("b200" if btype == "huggingface" else btype)
        if cls is None:
            raise RuntimeError("no transformer backend registered under %r" % btype)
        bc = ConfigNode(dict(self.config))
        bc.transformer_config = self._transformer_config()
        self.backend = cls(bc)
        if backend_config.get("freeze", False):
            for p in self.backend.parameters():
                p.requires_grad = False

    def build_encoders(self):
        self.encoders = nn.ModuleDict()
        for m in self.config.modalities:
            if "encoder" not in m or m["encoder"] is None:
                if m["type"] == "image" and "image_encoder" in self.config:
                    ec = self.config.image_encoder
                else:
                    ec = {"type": "identity", "params": {"in_dim": 100}}
            else:
                ec = m["encoder"]
            enc = build_encoder(ec)
            self.encoders[m["key"]] = enc
            frozen = (m["type"] == "image" and self.config.get("freeze_image_encoder", False)) or (
                m["type"] == "text" and self.config.get("freeze_text_encoder", False))
            if frozen:
                for p in enc.parameters():
                    p.requires_grad = False

    def build_heads(self):
        self.heads = nn.ModuleList()
        for hc in self.config.get("heads", []):
            htype = hc.get("type", "mlp")
            if htype not in HEADS:
                raise NotImplementedError("transformer head %r is not on the B200 path (have: %s)" % (htype, sorted(HEADS)))
            self.heads.append(HEADS[htype](hc))

    def init_weights(self):
        if self.config.get("random_initialize", False) is False and self.config.get("transformer_base", None) is None:
            _init_bert_weights(self.heads, float(self.config.get("initializer_range", 0.02)))
        self.tie_weights()

    def tie_weights(self):
        """mmf_transformer.py:145-174: heads with a tie_weights() share the text modality's token table"""
        if "text" not in self.modality_type:
            return
        idx = self.modality_type.index("text")
        for head in self.heads:
            if hasattr(head, "tie_weights"):
                head.tie_weights(self.backend.embeddings.token_embeddings[idx])

    # ---- SampleList -> per-modality integer tensors (mmf_transformer.py:176-392) ----
    @staticmethod
    def _first_present(sample_list, keys):
        for k in keys:
            if k in sample_list:
                return sample_list[k]
        expected = keys[0] if len(keys) == 1 else "%s or %s" % (", ".join(keys[:-1]), keys[-1])
        raise TypeError("Missing modality in SampleList. Expected to find %s" % expected)

    def _infer_input_ids(self, sample_list):
        out, ti = {}, 0
        for idx, (key, enc) in enumerate(zip(self.modality_keys, self.encoders.values())):
            kind = self.modality_type[idx]
            if kind == "text":
                out[key], ti = _text_slice(self._first_present(sample_list, ("input_ids", key)), ti)
            elif kind == "image":
                out[key] = self._first_present(sample_list, (key, "image", "input_modal", "image_feature_0"))
            else:
                out[key] = self._first_present(sample_list, (key,))
            if enc is not None:
                out[key] = enc(out[key])
            if kind != "text" and out[key].dim() == 2:             # [B, D] feature = one position
                out[key] = out[key].unsqueeze(1)
        return out

    def _infer_position_ids(self, input_ids):
        out = {}
        for key in self.modality_keys:
            B, n = input_ids[key].size(0), input_ids[key].size(1)
            out[key] = torch.arange(0, n, dtype=torch.long, device=input_ids[key].device).unsqueeze(0).expand((B, n))
        return out

    def _infer_masks(self, sample_list, input_ids):
        out, ti = {}, 0
        for idx, key in enumerate(self.modality_keys):
            if self.modality_type[idx] == "text" and "input_mask" in sample_list:
                out[key], ti = _text_slice(sample_list["input_mask"], ti)
            elif (key + "_mask") in sample_list:
                out[key] = sample_list[key + "_mask"]
            else:
                out[key] = torch.ones(input_ids[key].size()[:2], dtype=torch.long, device=input_ids[key].device)
        return out

    def _infer_segment_ids(self, sample_list, input_ids):
        out, ti = {}, 0
        for idx, key in enumerate(self.modality_keys):
            if self.modality_segments[idx] == -1:
                continue
            if self.modality_type[idx] == "text" and "segment_ids" in sample_list:
                out[key], ti = _text_slice(sample_list["segment_ids"], ti)
            else:
                out[key] = torch.full(input_ids[key].size()[:2], fill_value=self.modality_segments[idx], dtype=torch.long,
                                      device=input_ids[key].device)
        return out

    def _infer_itm_labels(self, sample_list, input_ids):
        if "is_correct" in sample_list:
            return {"is_correct": sample_list["is_correct"]}
        return {"is_correct": torch.tensor(True, dtype=torch.long, device=input_ids[self.modality_keys[0]].device)}

    def _infer_mlm_labels(self, sample_list, input_ids):
        out, ti = {}, 0
        for idx, key in enumerate(self.modality_keys):
            if self.modality_type[idx] == "text" and "lm_label_ids" in sample_list:
                out[key], ti = _text_slice(sample_list["lm_label_ids"], ti)
            else:
                out[key] = torch.full(input_ids[key].size()[:2], fill_value=-1, dtype=torch.long, device=input_ids[key].device)
        if self.modality_keys:
            out["combined_labels"] = torch.cat([out[k] for k in self.modality_keys], dim=-1)
        return out

    def preprocess_sample(self, sample_list):
        input_ids = self._infer_input_ids(sample_list)
        return {"input_ids": input_ids, "position_ids": self._infer_position_ids(input_ids),
                "segment_ids": self._infer_segment_ids(sample_list, input_ids),
                "masks": self._infer_masks(sample_list, input_ids),
                "mlm_labels": self._infer_mlm_labels(sample_list, input_ids),
                "itm_labels": self._infer_itm_labels(sample_list, input_ids)}

    def forward(self, sample_list):
        processed = self.preprocess_sample(sample_list)
        processed["target_key"] = sample_list
        masks = [processed["masks"][k] for k in self.modality_keys]
        sequence_output, encoded_layers = self.backend(processed["input_ids"], processed["position_ids"],
                                                       processed["segment_ids"], masks)
        return self.postprocess_output(sequence_output, encoded_layers, processed)

    def postprocess_output(self, sequence_output, encoded_layers, processed_sample_list):
        out = {}
        for head in self.heads:
            out.update(head(sequence_output, encoded_layers, processed_sample_list))
        return out
