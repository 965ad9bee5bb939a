"""The registered `vilt` model on the fused pre-LN (ViT) trunk.

  registry.register_model("vilt")  ViLT                      <->  mmf/models/vilt.py:118-283
  B200ViLTImageEmbedding                                     <->  ViLTImageEmbedding  vilt.py:22-79
  B200ViLTTextEmbedding                                      <->  ViLTTextEmbedding   vilt.py:82-115

Text: BERT embeddings (word + position + type -> LayerNorm -> dropout, one composer launch, mmf_b200.vilbert) plus a
second type table added on top ("official vilt repo adds type embeddings twice").  Image: the ViT patch projection as one
GEMM over the unfolded patches, [CLS], the position table and dropout (mmf_b200.vit.B200ViTEmbeddings), plus the image type
row.  Encoder: the registered `vit` encoder (mmf_b200.encoders.B200ViTImageEncoder) - the fused pre-LN layers and the final
LayerNorm; its own patch embeddings are built, as in the reference, and never called.  Heads: the transformer-head table of
mmf_b200.mmft through build_heads_dict / HeadsDict.  State-dict keys equal the reference's, the encoder's
`encoder.module.embeddings.*` and its alias `encoder.embeddings.*` included.

Torch ops on the path, all O(B * S * H) or less: the second type-table add of the text and the image type-row add, the
image embedding's [CLS] concatenation, position add and dropout, the [text, image] concatenation, the 0/1 -> additive
mask arithmetic, and the heads' losses (BCE with logits; the masked-LM and ITM cross-entropies with the masked-LM row
gather).

What the reference does, and so what is done here:
  * the masked-LM pass concatenates [image, text] but keeps the mask cat(text_mask, image_mask) and the labels
    cat(text_labels, image_labels = -1): the masked words are predicted from the outputs at the first T positions of
    [image, text] - [CLS] and the first image patches - and the key mask is misaligned the same way;
  * `input_mask` / `image_mask` are read by attribute: a plain dict sample list yields no mask (the encoder then masks
    nothing), a SampleList yields one; a missing one of the two is all ones (in the embedding's dtype);
  * ITM and MLM preprocessing is chosen by substring tests on the joined head names; `is_correct` defaults to
    tensor(True) when the sample list lacks it;
  * the additive mask is (1 - m) * -10000, the arithmetic of the reference's pinned transformers (<= 4.10.1);
  * a top-level list of heads without `tasks` builds here; the reference evaluates `heads.keys()` and raises.
The masked-LM head gathers a data-dependent number of rows, so a model with an `mlm` head refuses GraphedStep; a model
without one captures.
"""
import collections.abc

import torch
from torch import nn

from .encoders import build_encoder, transformer_hparams, vit_hf_config
from .models import MODEL_DEFAULTS, BaseModel, ConfigNode, Losses
from .modules import _init_bert_weights
from .registry import registry
from .vilbert import B200BertTextEmbeddings
from .vit import B200ViTEmbeddings

# mmf/configs/models/vilt/defaults.yaml:1-45 (the other_configs interpolations resolved)
MODEL_DEFAULTS["vilt"] = dict(
    heads=dict(test=[dict(type="mlp", loss="test_mlp", freeze=False, lr_multiplier=1.0, in_dim=768, hidden_size=1536,
                          num_labels=3129, pooler_name="bert_pooler")]),
    losses=dict(test_mlp="logit_bce"),
    image_encoder=dict(type="vit", params=dict(
        random_init=True, pretrained_model_name="google/vit-base-patch16-224", do_pooling=False, hidden_dropout_prob=0.1,
        add_pooling_layer=False, do_patch_embeddings=False, image_size=[224, 224], hidden_dim=768,
        pretrained_model="vit_base_patch16_224", mlp_dim=3072)),
    text_embeddings=dict(type="vilt_text_embedding", bert_model_name="bert-base-uncased", hidden_dim=768, hidden_size=768))


def max_positions(head_dim):
    """the longest sequence the attention kernels take (include/mmfb200.h): 384 keys at head size 64, 256 at 128"""
    return 384 if head_dim == 64 else 256


def get_bert_configured_parameters(module, lr=None, weight_decay=0.01):
    """mmf/utils/modeling.py:18-46: weight decay `weight_decay` / 0 for biases and LayerNorm parameters"""
    named = list(module.named_parameters()) if isinstance(module, nn.Module) else module
    no_decay = ["bias", "LayerNorm.bias", "LayerNorm.weight"]
    groups = [{"params": [p for n, p in named if not any(nd in n for nd in no_decay)], "weight_decay": weight_decay},
              {"params": [p for n, p in named if any(nd in n for nd in no_decay)], "weight_decay": 0.0}]
    if lr is not None:
        for g in groups:
            g["lr"] = lr
    return groups


class B200ViLTImageEmbedding(nn.Module):
    """ViLTImageEmbedding: the embeddings of a ViT built from the same keys (`embedding.*`: patch projection, [CLS],
    position table) plus `token_type_embeddings` [2, H], whose row 1 is added to every image position.  Keys other than
    the ones below are ignored, as in the reference."""

    def __init__(self, random_init=True, pretrained_model_name="google/vit-base-patch16-224", image_size=None,
                 hidden_dropout_prob=None, hidden_size=None, patch_size=None, num_channels=None, *args, **kwargs):
        super().__init__()
        config = {"random_init": random_init, "pretrained_model_name": pretrained_model_name}
        for key, v in (("image_size", image_size), ("hidden_dropout_prob", hidden_dropout_prob),
                       ("hidden_size", hidden_size), ("patch_size", patch_size), ("num_channels", num_channels)):
            if v is not None:
                config[key] = v
        hf = vit_hf_config(config)
        self.embedding = B200ViTEmbeddings(hf)
        std = float(hf.initializer_range)
        self.embedding.cls_token.data.normal_(0.0, std)
        self.embedding.position_embeddings.data.normal_(0.0, std)
        self.token_type_embeddings = nn.Embedding(2, hf.hidden_size)

    @property
    def num_positions(self):
        return self.embedding.position_embeddings.shape[1]

    def forward(self, image):
        if image.dim() == 5:
            image = image.permute(1, 0, 2, 3, 4).flatten(start_dim=0, end_dim=1)
        img_embeddings = self.embedding(image)
        return img_embeddings + self.token_type_embeddings.weight[1]


class B200ViLTTextEmbedding(nn.Module):
    """ViLTTextEmbedding: BERT embeddings (`text_embeddings.*`) with the hyper-parameters the `transformer` encoder
    resolves from the same keys, plus a second `token_type_embeddings` [2, H] added after them.  `bert_overrides`, a key
    the reference does not read, overrides the bert-base hyper-parameters (e.g. a smaller vocabulary)."""

    def __init__(self, random_init=True, bert_model_name="bert-base-uncased", hidden_size=None,
                 max_position_embeddings=None, bert_overrides=None, *args, **kwargs):
        super().__init__()
        config = dict(bert_overrides or {}, bert_model_name=bert_model_name, random_init=random_init)
        if hidden_size is not None:
            config["hidden_size"] = hidden_size
        if max_position_embeddings is not None:
            config["max_position_embeddings"] = max_position_embeddings
        hp = transformer_hparams(config)
        self.text_embeddings = B200BertTextEmbeddings(hp)
        _init_bert_weights(self.text_embeddings, float(hp.initializer_range))
        self.token_type_embeddings = nn.Embedding(2, hp.hidden_size)

    def forward(self, input_ids, segment_ids):
        text_embedding = self.text_embeddings(input_ids, token_type_ids=segment_ids)
        return text_embedding + self.token_type_embeddings(segment_ids)


@registry.register_model("vilt")
class ViLT(BaseModel):
    """ViLT (vilt.py:118-283): [text tokens | image patches] through one pre-LN transformer; VQA classification through
    an `mlp` head, masked-COCO pretraining through `mlm_multi` + `itm`"""

    graph_refusal = "gathers a data-dependent number of rows (the labelled masked-LM positions) in every pretraining forward"
    static_rows_capturable = True   # that gather is the only refusal: GraphedStep(..., static_rows=True) captures the step

    @classmethod
    def config_path(cls):
        return "configs/models/vilt/defaults.yaml"

    def build(self):
        from .mmft import build_heads_dict                 # mmft imports models: resolved at construction time
        self.text_embeddings = B200ViLTTextEmbedding(**self.config.text_embeddings)
        self.image_embeddings = B200ViLTImageEmbedding(**self.config.image_encoder.params)
        self.encoder = build_encoder(self.config.image_encoder)
        head_configs = self.config.get("heads", {})
        tasks = self.config.get("tasks")
        if tasks is None:
            tasks = list(head_configs.keys()) if isinstance(head_configs, collections.abc.Mapping) else []
        self.tasks = tasks.split(",") if isinstance(tasks, str) else tasks
        self.losses = nn.ModuleDict()
        self.heads_dict = build_heads_dict(head_configs, self.tasks, self.losses)
        self.modality_keys = self.modality_type = ["text", "image"]
        names = self.heads_dict.head_names
        names = [n for v in names.values() for n in v] if isinstance(names, collections.abc.Mapping) else names
        # the masked-LM head gathers a data-dependent number of rows: see mmf_b200.graphs.GraphedStep
        self.graph_capturable = not any("mlm" in n for n in names)

    def init_losses(self):
        for loss_name, loss_config in self.config.get("losses", {}).items():
            self.losses[loss_name] = Losses([loss_config])

    def _check_length(self, input_ids):
        hf = self.encoder.hf_config
        S = input_ids.size(1) + self.image_embeddings.num_positions
        limit = max_positions(hf.hidden_size // hf.num_attention_heads)
        if S > limit:
            raise ValueError("ViLT: %d text tokens + %d image positions = %d exceed the %d positions the attention "
                             "kernels take" % (input_ids.size(1), self.image_embeddings.num_positions, S, limit))

    def forward(self, sample_list):
        self._check_length(sample_list["input_ids"])
        text_embedding = self.text_embeddings(sample_list["input_ids"], sample_list["segment_ids"])
        image_embedding = self.image_embeddings(sample_list["image"])
        self.preprocess_sample(sample_list, image_embedding)
        embeddings = torch.cat([text_embedding, image_embedding], dim=1)
        attention_mask = self.get_attention_mask(sample_list, text_embedding, image_embedding)
        sequence, _ = self.encoder(embeddings, attention_mask=attention_mask)
        if sequence.dim() != 3:
            sequence = sequence.unsqueeze(1)
        return self.heads_dict(sample_list["dataset_name"], sequence, sample_list)

    def preprocess_sample(self, sample_list, image_embedding):
        head_names = self.heads_dict.head_names
        if isinstance(head_names, collections.abc.Mapping):
            head_names = head_names[sample_list["dataset_name"]]
        head_string = " ".join(head_names)
        if "itm" in head_string:
            sample_list["itm_labels"] = self._infer_itm_labels(sample_list)
        if "mlm" in head_string:
            sample_list["mlm_labels"] = self._infer_mlm_labels(sample_list, image_embedding.size()[:-1])
            self._encode_mlm(sample_list, image_embedding)

    def get_optimizer_parameters(self, config):
        """vilt.py:187-195: the encoder, the text embeddings and the heads (decay / no decay), the image embeddings"""
        if hasattr(self.encoder, "get_optimizer_parameters"):
            params = self.encoder.get_optimizer_parameters(config)
        else:
            params = [{"params": list(self.encoder.parameters())}]
        params += get_bert_configured_parameters(self.text_embeddings)
        params += get_bert_configured_parameters(self.heads_dict)
        params += [{"params": list(self.image_embeddings.parameters())}]
        return params

    def get_attention_mask(self, sample_list, text_embedding, image_embedding):
        text_mask = getattr(sample_list, "input_mask", None)
        image_mask = getattr(sample_list, "image_mask", None)
        if text_mask is None and image_mask is None:
            return None
        if text_mask is None:
            text_mask = torch.ones(text_embedding.size()[:-1], dtype=text_embedding.dtype, device=text_embedding.device)
        if image_mask is None:
            image_mask = torch.ones(image_embedding.size()[:-1], dtype=image_embedding.dtype,
                                    device=image_embedding.device)
        return torch.cat((text_mask, image_mask), dim=-1)

    def _infer_itm_labels(self, sample_list):
        if "is_correct" in sample_list:
            return {"is_correct": sample_list["is_correct"]}
        return {"is_correct": torch.tensor(True, dtype=torch.long, device=sample_list["input_ids"].device)}

    def _infer_mlm_labels(self, sample_list, image_embeddings_size):
        input_ids = sample_list["input_ids"]
        mlm_labels = {}
        if "lm_label_ids" in sample_list:
            lm = sample_list["lm_label_ids"]
            mlm_labels["text"] = lm[:, 0] if lm.dim() > 2 else lm
        else:
            mlm_labels["text"] = torch.full(input_ids.size(), fill_value=-1, dtype=torch.long, device=input_ids.device)
        mlm_labels["image"] = torch.full(image_embeddings_size, fill_value=-1, dtype=torch.long, device=input_ids.device)
        mlm_labels["combined_labels"] = torch.cat([mlm_labels["text"], mlm_labels["image"]], dim=-1)
        return mlm_labels

    def _encode_mlm(self, sample_list, image_embedding):
        """the second trunk pass, on the masked captions; the image embedding of the first is reused (no second patch
        GEMM, no second dropout draw) and the sequence is [image, text] - see the module docstring"""
        assert "lm_label_ids" in sample_list
        input_ids = sample_list.get("input_ids_masked", sample_list["input_ids"])
        text_embedding = self.text_embeddings(input_ids, sample_list["segment_ids"])
        embeddings = torch.cat([image_embedding, text_embedding], dim=1)
        attention_mask = self.get_attention_mask(sample_list, text_embedding, image_embedding)
        sequence, _ = self.encoder(embeddings, attention_mask=attention_mask)
        if sequence.dim() != 3:
            sequence = sequence.unsqueeze(1)
        sample_list["hs_masked_for_mlm"] = sequence
