"""Encoder plugins of the fusion path (SURVEY.md 8a row a13), registered under the reference's names.

  B200FinetuneFasterRcnnFpnFc7  <->  FinetuneFasterRcnnFpnFc7   mmf/modules/encoders.py:116-180   relu(Linear(feat))
  B200IdentityEncoder           <->  IdentityEncoder            mmf/modules/encoders.py:183-198
  B200TransformerEncoder        <->  TransformerEncoder         mmf/modules/encoders.py:513-585   BertModelJit wrapper
  B200ViTImageEncoder           <->  ViTEncoder                 mmf/modules/encoders.py:830-857   ViTModel wrapper (`vit`)

The reference builds these through `build_encoder({type, params})` (mmf/utils/build.py:517-546); here the classes are
registered with `registry.register_encoder(name)` in the shim and take the same config keys.
"""
import torch
from torch import nn

from . import ops
from .modules import B200BertEncoder, _init_bert_weights, _require_cuda
from .registry import registry
from .vilbert import B200BertTextEmbeddings
from .visual_bert import BertPooler


def _get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


@registry.register_encoder("finetune_faster_rcnn_fpn_fc7")
class B200FinetuneFasterRcnnFpnFc7(nn.Module):
    """fc7 of the detector re-applied to region features: relu(lc(image)).  The reference loads `lc` from pickled
    detectron weights (download); here it is random-init or filled by load_state_dict (key `lc.*`, legacy `module.lc.*`)."""

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        in_dim = _get(config, "in_dim")
        out_dim = _get(config, "out_dim", in_dim)
        self.lc = nn.Linear(in_dim, out_dim)
        self.out_dim = out_dim

    def _load_from_state_dict(self, state_dict, prefix, *a, **k):
        old_prefix = prefix + "module."
        for key in list(state_dict.keys()):
            if key.startswith(old_prefix):
                state_dict[key.replace(old_prefix, prefix)] = state_dict.pop(key)
        super()._load_from_state_dict(state_dict, prefix, *a, **k)

    def forward(self, image):
        _require_cuda(image, "image")
        shape = image.shape
        y = ops.linear_relu(image.reshape(-1, shape[-1]), self.lc.weight, self.lc.bias)
        return y.view(*shape[:-1], self.out_dim).to(image.dtype)


@registry.register_encoder("identity")
class B200IdentityEncoder(nn.Module):
    def __init__(self, config=None, *args, **kwargs):
        super().__init__()
        self.module = nn.Identity()
        self.in_dim = _get(config, "in_dim", 100) if config is not None else 100
        self.out_dim = self.in_dim

    def forward(self, x):
        return self.module(x)


class _BertModel(nn.Module):
    """BertModelJit's children and forward contract (mmf/modules/hf_layers.py:358-475) on the engine."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embeddings = B200BertTextEmbeddings(config)
        self.encoder = B200BertEncoder(config)
        self.pooler = BertPooler(config.hidden_size)
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, position_ids=None, head_mask=None,
                inputs_embeds=None, encoder_hidden_states=None, encoder_attention_mask=None):
        if inputs_embeds is not None or head_mask is not None or encoder_hidden_states is not None:
            raise NotImplementedError("inputs_embeds / head_mask / encoder_hidden_states are not on the B200 path")
        if input_ids is None:
            raise ValueError("You have to specify either input_ids or inputs_embeds")
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        dt = self.pooler.dense.weight.dtype
        if attention_mask.dim() == 2:
            ext = attention_mask[:, None, None, :]
        else:
            raise ValueError("Wrong shape for input_ids (shape %s) or attention_mask (shape %s)"
                             % (tuple(input_ids.shape), tuple(attention_mask.shape)))
        ext = (1.0 - ext.to(dt)) * -10000.0
        emb = self.embeddings(input_ids, token_type_ids, position_ids)
        seq = self.encoder(emb, ext)[0].to(dt)
        return seq, self.pooler(seq), ()


def transformer_hparams(config):
    """the BERT hyper-parameters TransformerEncoder resolves from its config keys (AutoConfig.from_pretrained(bert_model_name,
    **config), encoders.py:576-579): bert-base, overridden by the keys the config carries"""
    import types
    return types.SimpleNamespace(
        hidden_size=_get(config, "hidden_size", 768), num_hidden_layers=_get(config, "num_hidden_layers", 12),
        num_attention_heads=_get(config, "num_attention_heads", 12),
        intermediate_size=_get(config, "intermediate_size", 4 * _get(config, "hidden_size", 768)),
        vocab_size=_get(config, "vocab_size", 30522), max_position_embeddings=_get(config, "max_position_embeddings", 512),
        type_vocab_size=_get(config, "type_vocab_size", 2), hidden_dropout_prob=_get(config, "hidden_dropout_prob", 0.1),
        attention_probs_dropout_prob=_get(config, "attention_probs_dropout_prob", 0.1),
        layer_norm_eps=_get(config, "layer_norm_eps", 1e-12), hidden_act="gelu",
        initializer_range=_get(config, "initializer_range", 0.02))


@registry.register_encoder("transformer")
class B200TransformerEncoder(nn.Module):
    """config keys as TransformerEncoder.Config: hidden_size, num_hidden_layers, num_attention_heads, num_segments,
    plus any BertConfig key (vocab_size, intermediate_size, ...).  Always random-init here (no hub access); weights
    come from load_state_dict (`module.*` keys as in the reference)."""

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        self.original_config = config
        bert = transformer_hparams(config)
        self.module = _BertModel(bert)
        self.embeddings = self.module.embeddings
        self.config = bert
        self._init_segment_embeddings()

    def _init_segment_embeddings(self):
        """encoders.py:556-569: widen the type table to num_segments (rows 2..n-2 start at the mean of the first two)"""
        num_segments = _get(self.original_config, "num_segments", None)
        if num_segments:
            old = self.embeddings.token_type_embeddings.weight
            new_embeds = nn.Embedding(num_segments, self.config.hidden_size)
            new_embeds.weight.data[:2].copy_(old.data[:2])
            for idx in range(2, num_segments - 1):
                new_embeds.weight.data[idx].copy_(old.data.mean(dim=0))
            self.embeddings.token_type_embeddings = new_embeds

    def forward(self, *args, return_sequence=False, **kwargs):
        output = self.module(*args, **kwargs)
        return output[0] if return_sequence else output[1]


# the hub configs of the two ViT checkpoints the reference's ViLT configurations name (HF ViTConfig fields)
_VIT_BASE = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, initializer_range=0.02, layer_norm_eps=1e-12,
                 num_channels=3, qkv_bias=True)
VIT_PRETRAINED = {
    "google/vit-base-patch16-224": dict(_VIT_BASE, image_size=224, patch_size=16),
    "google/vit-base-patch32-384": dict(_VIT_BASE, image_size=384, patch_size=32),
}

# ViTModel.Config (mmf/modules/vit.py:179-186)
VIT_MODEL_DEFAULTS = dict(name="vit", pretrained_model_name="google/vit-base-patch16-224", random_init=False,
                          gradient_checkpointing=False, do_patch_embeddings=True)


def vit_hf_config(config):
    """ViTModel.from_config's hf_config (vit.py:310-323): the named checkpoint's hyper-parameters, then ViTModel.Config's
    defaults and every key of `config` on top (`ViTConfig.from_pretrained(name, **config)`, then `hf_config.update(config)`).
    Keys nothing reads (`hidden_dim`, `mlp_dim`, `regularize_*`, `pretrained_model`, `do_pooling`) are carried along and
    change nothing, as in the reference."""
    from .models import ConfigNode
    merged = dict(VIT_MODEL_DEFAULTS, **dict(config or {}))
    name = merged["pretrained_model_name"]
    if name not in VIT_PRETRAINED:
        raise ValueError("no ViT hyper-parameters for pretrained_model_name %r (there is no hub here; known: %s)"
                         % (name, sorted(VIT_PRETRAINED)))
    if merged.get("gradient_checkpointing"):
        raise NotImplementedError("gradient_checkpointing is not supported on the B200 ViT path")
    return ConfigNode(dict(VIT_PRETRAINED[name], **merged))


@registry.register_encoder("vit")
class B200ViTImageEncoder(nn.Module):
    """ViTEncoder (mmf/modules/encoders.py:830-857): `.module` a ViTModel on the fused pre-LN trunk (mmf_b200.vit),
    `.embeddings` the alias of its embeddings (state-dict keys under both names, as in the reference), `.hf_config`,
    `.out_dim`.  There is no hub: `pretrained_model_name` selects hyper-parameters from VIT_PRETRAINED, and with
    `random_init: False` the weights arrive through load_state_dict."""

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        from .vit import B200ViTModel
        self.config = config
        self.hf_config = vit_hf_config(config)
        self.module = B200ViTModel(self.hf_config)
        self.embeddings = self.module.embeddings
        self.out_dim = self.hf_config.hidden_size

    def forward(self, *args, output_hidden_states=False, **kwargs):
        out = self.module(*args, output_hidden_states=output_hidden_states, **kwargs)
        return out[0], (out[2] if output_hidden_states else None)


# ------------------------------------------------------------------------------------------------
# factories / builders (mmf/modules/encoders.py:59-113, mmf/utils/build.py:495-546)
# ------------------------------------------------------------------------------------------------
class _Projection(nn.Module):
    """ImageFeatureEncoderFactory type "projection" with module "linear" (ProjectionEmbedding -> nn.Linear,
    mmf/modules/embeddings.py ProjectionEmbedding) on the GEMM of the C ABI."""

    def __init__(self, in_dim, out_dim):
        super().__init__()
        self.layers = nn.Linear(in_dim, out_dim)
        self.out_dim = out_dim

    def forward(self, x):
        _require_cuda(x, "x")
        shape = x.shape
        y = ops.linear(x.reshape(-1, shape[-1]), self.layers.weight, self.layers.bias)
        return y.view(*shape[:-1], self.out_dim).to(x.dtype)


class B200ImageFeatureEncoderFactory(nn.Module):
    """ImageFeatureEncoderFactory (encoders.py:79-113): {type, params} -> .module, .out_dim"""

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        encoder_type = _get(config, "type")
        encoder_type = getattr(encoder_type, "value", encoder_type)
        params = _get(config, "params")
        if params is None or _get(params, "in_dim") is None:
            raise AssertionError("ImageFeatureEncoder require 'in_dim' param in config")
        if encoder_type in ("default", "identity"):
            self.module = nn.Identity()
            self.module.in_dim = _get(params, "in_dim")
            self.module.out_dim = _get(params, "in_dim")
        elif encoder_type == "projection":
            if _get(params, "module", "linear") != "linear":
                raise NotImplementedError("projection module %r is not on the B200 path" % _get(params, "module"))
            self.module = _Projection(_get(params, "in_dim"), _get(params, "out_dim"))
        elif encoder_type == "finetune_faster_rcnn_fpn_fc7":
            self.module = B200FinetuneFasterRcnnFpnFc7(params)
        else:
            raise NotImplementedError("Unknown Image Encoder: %s" % encoder_type)
        self.out_dim = self.module.out_dim

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)


class B200TextEncoderFactory(nn.Module):
    """TextEncoderFactory (encoders.py:454-485): identity / transformer (the `embedding` type wraps MMF's LSTM/attention
    text embeddings, which are not on the fusion path)."""

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        self._type = getattr(_get(config, "type"), "value", _get(config, "type"))
        if self._type == "identity":
            self.module = nn.Identity()
        elif self._type == "transformer":
            self._module = B200TransformerEncoder(_get(config, "params"))
            self.module = self._module.module          # the reference keeps the bare BertModel here (encoders.py:470-472)
        else:
            raise NotImplementedError("Unknown Text Encoder %s" % self._type)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)


def build_text_encoder(config, *args, **kwargs):
    return B200TextEncoderFactory(config, *args, **kwargs).module


def build_image_encoder(config, direct_features=False, **kwargs):
    if not direct_features:
        raise NotImplementedError("raw-image encoders (ResNet / detectron) are upstream of the fusion path: "
                                  "use direct_features_input")
    return B200ImageFeatureEncoderFactory(config).module


def build_encoder(config):
    """build_encoder (mmf/utils/build.py:517-546): `{type, params}` or a structured config with `name`."""
    if _get(config, "type") is not None:
        name = getattr(_get(config, "type"), "value", _get(config, "type"))
        params = _get(config, "params", None)
    else:
        name, params = _get(config, "name"), config
    cls = registry.get_encoder_class(name)
    if cls is None:
        raise KeyError("no encoder registered under %r" % name)
    return cls(params if params is not None else {})


class B200MultiModalEncoderBase(nn.Module):
    """MultiModalEncoderBase (encoders.py:588-646): builds `text_encoder` / `modal_encoder` from the config."""

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        self.config = config
        self._modal_encoder_config = _get(config, "modal_encoder", None)
        self._is_direct_features_input = _get(config, "direct_features_input", False)
        self.build()
        self.modal_hidden_size = _get(config, "modal_hidden_size", None)
        self.text_hidden_size = _get(config, "text_hidden_size", None)

    def build(self):
        self.text_encoder, self.modal_encoder = self._build_encoders(self.config)
        self._encoder_config = self.text_encoder.config if self.text_encoder is not None else None

    @property
    def encoder_config(self):
        return self._encoder_config

    def _build_encoders(self, config):
        text_encoder = modal_encoder = None
        if _get(config, "text_encoder", None):
            text_encoder = build_text_encoder(_get(config, "text_encoder"))
        if _get(config, "modal_encoder", None):
            modal_encoder = self._build_modal_encoder(_get(config, "modal_encoder"))
        return text_encoder, modal_encoder

    def _build_modal_encoder(self, config):
        return build_image_encoder(config, direct_features=self._is_direct_features_input)
