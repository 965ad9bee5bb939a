"""The registered `uniter` model on the fused trunk (BASELINE.json configs[4]).

  registry.register_model("uniter")  UNITER                     <->  mmf/models/uniter.py:615-774
  B200UNITERForClassification                                    <->  :278-348
  B200UNITERForPretraining                                       <->  :351-612   (mlm, itm, mrc, mrfr, wra)
  _infer_with_heads                                              <->  :249-275

The trunk is mmf_b200.uniter.B200UNITERModelBase; the heads come from the transformer-head table of mmf_b200.mmft (the
reference's `registry.get_transformer_head_class`).  State-dict keys equal the reference's: `uniter.uniter.*`,
`uniter.heads.<task>.*`, with MRFR's `linear_proj_weight` the same Parameter as `img_embeddings.img_linear.weight`.

What the reference does, and so what is done here:
  * the task of a forward is drawn with torch.randint and the masked regions with np.random.binomial + random.choice, the
    same calls in the same order, so seeding torch / numpy / random reproduces the reference's choices;
  * `_remove_mismatched_captions` selects the positive pairs into a local and drops the result (uniter.py:601-612), so
    every task trains on all pairs; it is kept as the no-op it is;
  * `encoder` / `text_embeddings` are keyword overrides of the bert-base BertConfig (`type`, `params` and other nested
    entries of the default YAML are carried by that config and read by nobody).
There is no hub here: `random_init` / `bert_model_name` only select the bert-base hyper-parameters and weights arrive
through load_state_dict.

CUDA graphs: `UNITER.draw(sample_list)` makes a forward's host draws (the task, and for mrc / mrfr the region masks) up
front and stores them in the sample list under DRAWS_KEY; a forward that finds them there draws nothing and, inside
graphs.static_rows(), reads nothing on the host (device-side position-feature normalisation, WRA pads built on the device,
region heads bounded by a device count).  mmf_b200.graphs.GraphedTaskSteps captures one graph per task on that basis;
GraphedStep refuses the model, whose every step draws on the host.
"""
import collections.abc
import copy
import random
import warnings

import numpy as np
import torch
from torch import nn

from .models import BERT_BASE, MODEL_DEFAULTS, BaseModel, ConfigNode, Losses, _sl_get
from .graphs import static_rows_active
from .registry import registry
from .uniter import B200UNITERModelBase

# mmf/configs/models/uniter/defaults.yaml:1-28
MODEL_DEFAULTS["uniter"] = dict(
    heads=dict(vqa2=dict(type="mlp", freeze=False, lr_multiplier=1.0, in_dim=768, hidden_size=1536, num_labels=3129,
                         pooler_name="bert_pooler")),
    text_embeddings=dict(type="bert_embeddings"),
    image_embeddings=dict(type="uniter_image_embeddings", params=dict(name="uniter_image_embeddings")),
    encoder=dict(type="transformer", params=dict(bert_model_name="bert-base-uncased", hidden_size=768, num_hidden_layers=12,
                                                 num_attention_heads=12, output_attentions=False,
                                                 output_hidden_states=False)),
    tasks=["vqa2"])

# UNITER.Config (uniter.py:619-631); `heads` and `tasks` are MISSING there and come from the YAML
CONFIG_DEFAULTS = dict(random_init=False, bert_model_name="bert-base-uncased", img_dim=2048, hidden_size=768,
                       hidden_dropout_prob=0, text_embeddings={}, encoder={}, losses={}, do_pretraining=False)

DEFAULT_PRETRAINING_HEAD_CONFIGS = {"mlm": {"type": "mlm"}, "itm": {"type": "itm"}, "mrc": {"type": "mrc"},
                                    "mrfr": {"type": "mrfr"}, "wra": {"type": "wra"}}
DEFAULT_PRETRAINING_TASKS = "mlm,itm,mrc,mrfr,wra"

DRAWS_KEY = "uniter_draws"       # {"task": name, "image_mask": bool [B, R] (mrc / mrfr)}: see UNITER.draw

_UNSUPPORTED = ("output_attentions", "output_hidden_states", "is_decoder", "add_cross_attention")


def _bert_config(overrides, what):
    """BertConfig.from_pretrained("bert-base-uncased", **overrides) (uniter.py:119-139) without the hub"""
    overrides = dict(overrides or {})
    for key in _UNSUPPORTED:
        if overrides.get(key, False):
            raise NotImplementedError("UNITER `%s.%s: true` has no path on the fused encoder" % (what, key))
    return ConfigNode(dict(BERT_BASE, **overrides))


def _trunk(img_dim, hidden_size, hidden_dropout_prob, text_embeddings, encoder):
    enc, txt = _bert_config(encoder, "encoder"), _bert_config(text_embeddings, "text_embeddings")
    if enc.hidden_size != hidden_size or txt.hidden_size != hidden_size:
        raise ValueError("UNITER: hidden_size (%d) must equal the encoder's (%d) and the text embeddings' (%d)"
                         % (hidden_size, enc.hidden_size, txt.hidden_size))
    return B200UNITERModelBase(enc, img_dim=img_dim, hidden_dropout_prob=hidden_dropout_prob, text_config=txt)


def _head_class(head_type):
    from .mmft import HEADS          # mmft imports models, which imports this module: resolved at construction time
    if head_type not in HEADS:
        raise NotImplementedError("transformer head %r is not on the B200 path (have: %s)" % (head_type, sorted(HEADS)))
    return HEADS[head_type]


def _split_tasks(tasks):
    return tasks.split(",") if isinstance(tasks, str) else list(tasks)


def _init_losses(module):
    """uniter.py:333-343, 408-418: one MMFLoss per task that configures one"""
    module.losses = nn.ModuleDict()
    for task in module.tasks:
        if task not in module.loss_configs:
            warnings.warn("No loss defined for %s. Head is expected to return dict with 'losses'" % task)
            continue
        module.losses[task] = Losses([module.loss_configs[task]])


def _infer_with_heads(processed_sample_list, uniter_model, heads, losses):
    sequence_output = uniter_model(
        processed_sample_list["input_ids"], processed_sample_list["position_ids"], processed_sample_list["image_feat"],
        processed_sample_list["img_pos_feat"], processed_sample_list["attention_mask"],
        img_masks=processed_sample_list["image_mask"]).final_layer
    dataset_name = processed_sample_list["dataset_name"]
    task = processed_sample_list.get("task", dataset_name)
    outputs = heads[task](sequence_output, processed_sample_list=processed_sample_list)
    if isinstance(outputs, collections.abc.MutableMapping) and "losses" in outputs:
        return outputs
    logits = outputs
    if isinstance(outputs, collections.abc.MutableMapping) and "scores" in outputs:
        logits = outputs["scores"]
    logits = logits.contiguous().view(-1, logits.size(-1))
    output = losses[dataset_name](processed_sample_list, {"scores": logits})
    return {"losses": output, "scores": logits}


class B200UNITERForClassification(nn.Module):
    """head_configs = {"vqa2": {"type": "mlp", "num_labels": 3129}}, loss_configs = {"vqa2": "logit_bce"}, tasks = "vqa2" """

    def __init__(self, head_configs, loss_configs, tasks, random_init=False, bert_model_name="bert-base-uncased",
                 img_dim=2048, hidden_size=768, hidden_dropout_prob=0, text_embeddings=None, encoder=None):
        super().__init__()
        self.loss_configs = loss_configs
        self.uniter = _trunk(img_dim, hidden_size, hidden_dropout_prob, text_embeddings, encoder)
        self.heads = nn.ModuleDict()
        self.tasks = _split_tasks(tasks)
        for task in self.tasks:
            assert task in head_configs, (
                "Task %s is specified in your model configs but there is no head configured for the task. Head configs can "
                "be added under model_config.heads in your yaml configs. Either remove this task if UNITER is not meant to "
                "run on a dataset named %s or add a head config." % (task, task))
            head_config = head_configs[task]
            self.heads[task] = _head_class(head_config.get("type", "mlp"))(head_config)
        _init_losses(self)

    def forward(self, processed_sample_list):
        return _infer_with_heads(processed_sample_list, self.uniter, self.heads, self.losses)


class B200UNITERForPretraining(nn.Module):
    def __init__(self, head_configs=None, loss_configs=None, tasks=DEFAULT_PRETRAINING_TASKS, mask_probability=0,
                 random_init=False, bert_model_name="bert-base-uncased", img_dim=2048, hidden_size=768,
                 hidden_dropout_prob=0, text_embeddings=None, encoder=None):
        super().__init__()
        if head_configs is None:
            head_configs = copy.deepcopy(DEFAULT_PRETRAINING_HEAD_CONFIGS)
        self.loss_configs = {} if loss_configs is None else loss_configs
        self.mask_probability = mask_probability
        self.uniter = _trunk(img_dim, hidden_size, hidden_dropout_prob, text_embeddings, encoder)
        self.heads = nn.ModuleDict()
        self.tasks = _split_tasks(tasks)
        for task in self.tasks:
            head_config = head_configs[task]
            head_type = head_config.get("type", "mlp")
            head_class = _head_class(head_type)
            if head_type == "mrfr":
                self.heads[task] = head_class(self.uniter.img_embeddings.img_linear.weight, **head_config)
            elif head_type in ("itm", "mlm", "mlp"):
                self.heads[task] = head_class(head_config)
            else:
                self.heads[task] = head_class(**head_config)
        _init_losses(self)

    def forward(self, processed_sample_list):
        assert "is_correct" in processed_sample_list, (
            "UNITER pretraining requires mismatched captions. Please add 'false_caption': true under dataset_config in "
            "your yaml configs.")
        self._process_sample_list_for_pretraining(processed_sample_list)
        task = processed_sample_list["task"]
        if task not in ("mlm", "itm", "mrc", "mrfr", "wra"):
            raise ValueError("Task %s is not supported for pretraining!" % task)
        getattr(self, "_preprocess_" + task)(processed_sample_list)
        return _infer_with_heads(processed_sample_list, self.uniter, self.heads, self.losses)

    def _process_sample_list_for_pretraining(self, sl):
        task = sl["task"]
        if task in ("mrfr", "mrc"):
            self._add_image_feat_masked(sl)
            # cls_prob becomes a key of the sample list (uniter.py:453-458)
            sl["cls_prob"] = torch.as_tensor(_sl_get(sl["image_info_0"], "cls_prob"))
        if task not in ("wra", "itm"):
            self._remove_mismatched_captions(sl)

    def draw_image_masks(self, image_feat):
        """one region mask per sample (uniter.py:476-481), as a bool [B, R] tensor on image_feat's device"""
        img_masks = torch.tensor([self._get_img_mask(self.mask_probability, image_feat.size(1))
                                  for _ in range(image_feat.size(0))]).bool()
        if image_feat.is_cuda:           # from pinned memory: the copy does not wait for the work queued before it
            return img_masks.pin_memory().to(image_feat.device, non_blocking=True)
        return img_masks

    def _add_image_feat_masked(self, sl):
        img_feat_masked = torch.clone(sl["image_feat"])
        drawn = sl.get(DRAWS_KEY)
        if drawn is not None and drawn.get("image_mask") is not None:
            img_masks = drawn["image_mask"]
        else:
            img_masks = self.draw_image_masks(img_feat_masked)
        sl["image_feat_masked"] = img_feat_masked.data.masked_fill(img_masks.unsqueeze(-1).expand_as(img_feat_masked), 0)
        sl["image_mask"] = img_masks

    def _get_img_mask(self, mask_prob, num_bb):
        img_mask = list(map(bool, np.random.binomial(1, mask_prob, num_bb)))
        if not any(img_mask):
            img_mask[random.choice(range(num_bb))] = True        # at least mask 1
        return img_mask

    def _preprocess_mlm(self, sl):
        assert "lm_label_ids" in sl
        assert "input_ids_masked" in sl
        ignore_index = self.heads["mlm"].config.ignore_index
        mlm_labels = {"text": sl["lm_label_ids"]}
        mlm_labels["image"] = torch.full(sl["image_feat"].shape[:2], fill_value=ignore_index, dtype=torch.long,
                                         device=mlm_labels["text"].device)
        mlm_labels["combined_labels"] = torch.cat([mlm_labels["text"], mlm_labels["image"]], dim=-1)
        sl["mlm_labels"] = mlm_labels
        sl["input_ids"] = sl["input_ids_masked"]

    def _preprocess_itm(self, sl):
        assert "is_correct" in sl
        sl["itm_labels"] = {"is_correct": sl["is_correct"]}

    def _get_feature_mask(self, image_mask, sentence_len):
        padding_for_txt = torch.zeros((image_mask.size(0), sentence_len), dtype=image_mask.dtype, device=image_mask.device)
        return torch.cat([padding_for_txt, image_mask], dim=-1)

    def _mask_inputs_in_sample_list(self, sl, mask_key):
        assert "image_feat_masked" in sl
        sl[mask_key] = self._get_feature_mask(sl["image_mask"], sl["input_ids"].size(1))
        sl["image_feat"] = sl["image_feat_masked"]

    def _preprocess_mrc(self, sl):
        assert "cls_prob" in sl
        assert "image_mask" in sl
        assert "image_feat_masked" in sl
        image_mask = sl["image_mask"]
        cls_prob = sl["cls_prob"].to(image_mask.device)
        if static_rows_active():         # every region's target: the head selects the masked ones on the device
            sl[self.heads["mrc"].mrc_label_key] = cls_prob
        else:
            img_masks_ext = image_mask.unsqueeze(-1).expand_as(cls_prob)
            sl[self.heads["mrc"].mrc_label_key] = cls_prob[img_masks_ext].contiguous().view(-1, cls_prob.size(2))
        self._mask_inputs_in_sample_list(sl, self.heads["mrc"].mrc_mask_key)

    def _preprocess_mrfr(self, sl):
        assert "image_mask" in sl
        assert "image_feat_masked" in sl
        image_mask, image_feat = sl["image_mask"], sl["image_feat"]
        if static_rows_active():
            sl[self.heads["mrfr"].mrfr_target_key] = image_feat
        else:
            img_masks_ext = image_mask.unsqueeze(-1).expand_as(image_feat)
            sl[self.heads["mrfr"].mrfr_target_key] = image_feat[img_masks_ext].contiguous().view(-1, image_feat.size(2))
        self._mask_inputs_in_sample_list(sl, self.heads["mrfr"].mrfr_mask_key)

    def _preprocess_wra(self, sl):
        assert "is_correct" in sl
        txt_lens = [i.size(0) for i in sl["input_ids"]]
        num_bbs = [f.size(0) for f in sl["image_feat"]]

        device = sl["input_ids"].device

        def _compute_pad(lens):
            # uniter.py:565-570, built on the device: row i is padding from lens[i] on
            pad = torch.zeros(len(lens), max(lens), dtype=torch.bool, device=device)
            for i, n in enumerate(lens):
                if n < pad.size(1):
                    pad[i, n:] = True
            return pad

        # the lengths are the padded sizes, so they depend only on shapes; they ride along on the host, where the kernel
        # takes them as launch parameters
        sl[self.heads["wra"].ot_inputs_key] = {"txt_pad": _compute_pad(txt_lens), "img_pad": _compute_pad(num_bbs),
                                               "txt_lens": txt_lens, "img_lens": num_bbs}
        sl[self.heads["wra"].wra_label_key] = sl["is_correct"]

    def _remove_mismatched_captions(self, sl):
        """uniter.py:585-612 indexes each tensor by the positive pairs and binds the result to a local (`x = x[...]`), so
        the sample list is left as it was: negative pairs stay in every task's batch.  Only its assertions act."""
        assert "is_correct" in sl
        pos_pairs = sl["is_correct"].ne(0)
        for name in ("input_ids", "input_mask", "image_feat", "img_pos_feat", "attention_mask", "image_mask",
                     "image_feat_masked", "lm_label_ids", "cls_prob"):
            x = sl.get(name)
            if x is not None and x.dim() == 1:
                assert x.size(0) == pos_pairs.size(0), (
                    "tensor %s has shape %s but expected %d at dim 0." % (name, tuple(x.shape), pos_pairs.size(0)))


@registry.register_model("uniter")
class UNITER(BaseModel):
    """Modification for Joint Vision-Language Encoding (uniter.py:615-774)"""

    graph_capturable = False        # host-side task / mask draws: see mmf_b200.graphs.GraphedTaskSteps
    graph_refusal = ("draws its task and region masks on the host in every forward and gathers a data-dependent number of "
                     "rows; capture one graph per task with mmf_b200.graphs.GraphedTaskSteps")

    draws_key = DRAWS_KEY

    def __init__(self, config):
        super().__init__(config)
        self.config = ConfigNode(dict(copy.deepcopy(CONFIG_DEFAULTS), **self.config))
        self.do_pretraining = self.config.do_pretraining

    @classmethod
    def config_path(cls):
        return "configs/models/uniter/defaults.yaml"

    def build(self):
        configs = dict(**self.config)
        configs["head_configs"] = configs.pop("heads")
        configs["loss_configs"] = configs.pop("losses")
        params_keys = ["head_configs", "loss_configs", "tasks", "random_init", "bert_model_name", "img_dim", "hidden_size",
                       "hidden_dropout_prob", "text_embeddings", "encoder"]
        if self.do_pretraining:
            # take value from config when the key exists, otherwise use constructor defaults
            params_keys += ["mask_probability"]
            self.uniter = B200UNITERForPretraining(**{key: configs[key] for key in params_keys if key in configs})
        else:
            self.uniter = B200UNITERForClassification(**{key: configs[key] for key in params_keys if key in configs})
        self.tasks = _split_tasks(self.config.tasks)

    def init_losses(self):
        """Defer loss management to submodels, do nothing when called by build_model."""

    def draw(self, sample_list, task=None):
        """Make the host draws of a forward, in the reference's order, and store them in the sample list under DRAWS_KEY:
        the task with torch.randint over `tasks` (classification too), then for mrc / mrfr one region mask per sample
        with np.random.binomial + random.choice, as a bool [B, R] tensor on the features' device.  A forward that finds
        them draws nothing, so `draw` followed by a forward makes the same choices from the same seeds as a forward
        alone.  `task` fixes the task instead of drawing it (the masks are still drawn).  Returns the task's name."""
        if task is None:
            task = self.tasks[torch.randint(len(self.tasks), (1,)).item()]
        elif task not in self.tasks:
            raise ValueError("UNITER.draw: task %r is not one of %s" % (task, self.tasks))
        draws = {"task": task}
        if self.do_pretraining and task in ("mrc", "mrfr"):
            draws["image_mask"] = self.uniter.draw_image_masks(sample_list["image_feature_0"])
        sample_list[DRAWS_KEY] = draws
        return task

    def add_pos_feat(self, sample_list):
        info = _sl_get(sample_list, "image_info_0", None)
        assert info is not None
        assert _sl_get(info, "bbox", None) is not None
        # (x1, y1, x2, y2), dim = (bs, num_feats, 4)
        bboxs = torch.as_tensor(_sl_get(info, "bbox"))[:, :, :4]
        norm_xy = torch.clone(bboxs)

        def max_image_size():
            img_h = torch.as_tensor(_sl_get(info, "image_height")).unsqueeze(1).unsqueeze(1)
            img_w = torch.as_tensor(_sl_get(info, "image_width")).unsqueeze(1).unsqueeze(1)
            return torch.cat([img_w, img_h, img_w, img_h], dim=-1).to(norm_xy.device)

        if DRAWS_KEY in sample_list and _sl_get(info, "image_height", None) is not None:
            # the same rule selected on the device, so a captured step reads nothing on the host
            norm_xy = torch.where(norm_xy[0, 0, 0] < 1, norm_xy / max_image_size(), norm_xy)
        elif norm_xy[0, 0, 0] < 1:        # the reference's rule, kept as written (uniter.py:686-700)
            norm_xy /= max_image_size()
        bbox_w = (norm_xy[:, :, 2] - norm_xy[:, :, 0]).unsqueeze(-1)
        bbox_h = (norm_xy[:, :, 3] - norm_xy[:, :, 1]).unsqueeze(-1)
        area = bbox_w * bbox_h
        # normalized (x1, y1, x2, y2, w, h, area)
        sample_list["img_pos_feat"] = torch.cat([norm_xy, bbox_w, bbox_h, area], dim=-1).to(sample_list["image_feature_0"])

    def add_custom_params(self, sample_list):
        image_feat = sample_list["image_feat"] = sample_list["image_feature_0"]
        image_dim = _sl_get(_sl_get(sample_list, "image_info_0", {}), "max_features", None)
        sample_list["image_dim"] = image_dim
        image_mask = torch.arange(image_feat.size(-2), device=image_feat.device).expand(image_feat.size()[:-1])
        if len(image_dim.size()) < len(image_mask.size()):
            image_dim = image_dim.unsqueeze(-1)
            assert len(image_dim.size()) == len(image_mask.size())
        sample_list["image_mask"] = (image_mask < image_dim).long()
        sample_list["attention_mask"] = torch.cat((sample_list["input_mask"], sample_list["image_mask"]), dim=-1)
        if DRAWS_KEY in sample_list:
            sample_list["task"] = sample_list[DRAWS_KEY]["task"]
        else:
            task_index = torch.randint(len(self.tasks), (1,)).item()
            sample_list["task"] = self.tasks[task_index]
        sample_list["position_ids"] = torch.arange(0, sample_list["input_ids"].size(1), dtype=torch.long,
                                                   device=image_feat.device).unsqueeze(0)
        self.add_pos_feat(sample_list)
        return sample_list

    def forward(self, sample_list):
        sample_list = self.add_custom_params(sample_list)
        return self.uniter(sample_list)

    def get_attention_mask(self, sample_list, text_embedding, image_embedding):
        image_mask = _sl_get(sample_list, "image_mask", None)
        input_mask = _sl_get(sample_list, "input_mask", None)
        if image_mask is not None and input_mask is not None:
            return torch.cat((input_mask, image_mask), dim=-1)
        if image_mask is not None:
            text_mask = torch.ones(text_embedding.size()[:-1], dtype=text_embedding.dtype, device=text_embedding.device)
            return torch.cat((image_mask, text_mask), dim=-1)
        if input_mask is not None:
            image_mask = torch.ones(image_embedding.size()[:-1], dtype=image_embedding.dtype, device=image_embedding.device)
            return torch.cat((image_mask, input_mask), dim=-1)
        return None
