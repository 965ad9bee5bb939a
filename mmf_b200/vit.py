"""ViT (pre-LN) trunk on the B200 engine (SURVEY.md 8f item 3, kernel row K7: "ViLT / ViT pre-LN variant").

  B200ViTLayer / B200ViTEncoder  <->  ViTLayer / ViTEncoder   mmf/modules/vit.py:35-175  (HF ViT blocks with
                                      BertSelfAttention inside so that vision-language inputs can be MASKED, vit.py:37-44)
  B200ViTEmbeddings              <->  HF ViTEmbeddings (patch projection + [CLS] + position table), used at vit.py:190
  B200ViTModel                   <->  ViTModel.forward  vit.py:178-274: embeddings -> encoder -> final LayerNorm -> pooler

Parameter names are HF's / the reference's (`encoder.layer.{i}.attention.attention.query.weight`,
`...attention.output.dense`, `layernorm_before`, `layernorm_after`, `intermediate.dense`, `output.dense`, `layernorm`,
`embeddings.{cls_token,position_embeddings,patch_embeddings.projection}`), so ViT / ViLT checkpoints keep loading.
The layer is engine.vit_layer_fwd / vit_layer_bwd: the post-LN layer's kernels in pre-LN order.
"""
import torch
from torch import nn

from . import engine as E
from . import ops
from .modules import (B200BertIntermediate, B200BertSelfAttention, EncoderRunner, _Holder, _init_bert_weights, _require_cuda,
                      run_bert_encoder, split_encoder_outputs)


class _ViTSelfOutput(_Holder):
    def __init__(self, hidden, p_hidden):
        super().__init__()
        self.dense = nn.Linear(hidden, hidden)
        self.dropout = nn.Dropout(p_hidden)


class _ViTAttention(_Holder):
    def __init__(self, hidden, heads, p_attn, p_hidden):
        super().__init__()
        self.attention = B200BertSelfAttention(hidden, heads, p_attn)     # vit.py:44: BertSelfAttention inside ViTAttention
        self.output = _ViTSelfOutput(hidden, p_hidden)


class _ViTOutput(_Holder):
    def __init__(self, inter, hidden, p_hidden):
        super().__init__()
        self.dense = nn.Linear(inter, hidden)
        self.dropout = nn.Dropout(p_hidden)


class B200ViTLayer(_Holder):
    def __init__(self, hidden, heads, inter, p_attn, p_hidden, eps):
        super().__init__()
        self.attention = _ViTAttention(hidden, heads, p_attn, p_hidden)
        self.intermediate = B200BertIntermediate(hidden, inter)
        self.output = _ViTOutput(inter, hidden, p_hidden)
        self.layernorm_before = nn.LayerNorm(hidden, eps=eps)
        self.layernorm_after = nn.LayerNorm(hidden, eps=eps)


class ViTRunner(EncoderRunner):
    """its own type: mmf_b200.patch.set_skip_padding never packs a ViT stack"""
    W = E.ViTLayerW


class B200ViTEncoder(nn.Module):
    """config: HF ViTConfig-like (hidden_size, num_hidden_layers, num_attention_heads, intermediate_size, dropouts,
    layer_norm_eps, hidden_act = "gelu")."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        act = getattr(config, "hidden_act", "gelu")
        if act != "gelu":
            raise ValueError("B200 fusion block implements the erf GELU of the reference configs, got %r" % (act,))
        eps = float(getattr(config, "layer_norm_eps", 1e-12))
        self.layer = nn.ModuleList([
            B200ViTLayer(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                         float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob), eps)
            for _ in range(config.num_hidden_layers)])
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))
        self._runner = ViTRunner(self.layer)

    def forward(self, hidden_states, attention_mask=None, head_mask=None, output_attentions=False,
                output_hidden_states=False, return_dict=True):
        """ViTEncoder.forward (vit.py:118-175).  return_dict=True gives an object with `last_hidden_state` / `hidden_states`
        / `attentions` attributes (HF BaseModelOutput's fields).  output_attentions: `attentions` is the tuple of the
        layers' probabilities [B, heads, S, S] (one extra kernel per layer; no gradient flows through them)."""
        if head_mask is not None and not (isinstance(head_mask, (list, tuple)) and all(h is None for h in head_mask)):
            raise NotImplementedError("head_mask is not supported on the B200 path")
        outs = run_bert_encoder(self._runner, hidden_states, attention_mask, self.training, output_hidden_states,
                                output_attentions)
        last, hidden, attn = split_encoder_outputs(outs, len(self.layer), output_hidden_states, output_attentions)
        if not return_dict:
            return tuple(v for v in (last, hidden, attn) if v is not None)
        import types
        return types.SimpleNamespace(last_hidden_state=last, hidden_states=hidden, attentions=attn)


class _PatchEmbeddings(nn.Module):
    """HF ViTPatchEmbeddings: Conv2d(C, H, kernel = stride = patch) == one GEMM over the unfolded patches"""

    def __init__(self, config):
        super().__init__()
        size, patch = config.image_size, config.patch_size
        size = size if isinstance(size, (tuple, list)) else (size, size)
        patch = patch if isinstance(patch, (tuple, list)) else (patch, patch)
        self.image_size, self.patch_size, self.num_channels = tuple(size), tuple(patch), getattr(config, "num_channels", 3)
        self.num_patches = (size[0] // patch[0]) * (size[1] // patch[1])
        self.projection = nn.Conv2d(self.num_channels, config.hidden_size, kernel_size=patch, stride=patch)

    def forward(self, pixel_values):
        B, C, Hh, Ww = pixel_values.shape
        if C != self.num_channels:
            raise ValueError("Make sure that the channel dimension of the pixel values match with the one set in the "
                             "configuration. Expected %d but got %d." % (self.num_channels, C))
        ph, pw = self.patch_size
        # unfold into [B * n_patches, C * ph * pw] rows in the conv weight's (C, kh, kw) order
        x = pixel_values.reshape(B, C, Hh // ph, ph, Ww // pw, pw).permute(0, 2, 4, 1, 3, 5).reshape(
            B * (Hh // ph) * (Ww // pw), C * ph * pw)
        w = self.projection.weight.reshape(self.projection.weight.shape[0], -1)
        return ops.linear_any(x, w, self.projection.bias).view(B, -1, w.shape[0])


class B200ViTEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, config.hidden_size))
        self.patch_embeddings = _PatchEmbeddings(config)
        self.position_embeddings = nn.Parameter(torch.zeros(1, self.patch_embeddings.num_patches + 1, config.hidden_size))
        self.dropout = nn.Dropout(float(config.hidden_dropout_prob))

    def forward(self, pixel_values):
        _require_cuda(pixel_values, "pixel_values")
        emb = self.patch_embeddings(pixel_values).to(self.position_embeddings.dtype)
        emb = torch.cat((self.cls_token.expand(emb.shape[0], -1, -1), emb), dim=1) + self.position_embeddings
        return self.dropout(emb)


def extended_attention_mask(attention_mask, dtype):
    """get_extended_attention_mask of the reference's pinned transformers (<= 4.10.1) for a 2-D mask: (1 - m) * -10000
    as [B, 1, 1, S].  None stays None (the reference's all-ones mask adds 0 to every score).  A 3-D per-query mask is
    not supported by the kernels."""
    if attention_mask is None:
        return None
    if attention_mask.dim() == 3:
        raise NotImplementedError("per-query [B, S, S] attention masks are not supported on the B200 ViT path")
    if attention_mask.dim() != 2:
        raise ValueError("Wrong shape for attention_mask (shape %s)" % (tuple(attention_mask.shape),))
    return (1.0 - attention_mask[:, None, None, :].to(dtype)) * -10000.0


class B200ViTModel(nn.Module):
    """ViTModel (vit.py:178-274): `do_patch_embeddings=False` (vit.py:187, ViLT feeds already-embedded tokens) skips the
    patch embedding; output (sequence_output, pooled_output[, hidden_states])."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embeddings = B200ViTEmbeddings(config)
        self.encoder = B200ViTEncoder(config)
        self.layernorm = nn.LayerNorm(config.hidden_size, eps=float(getattr(config, "layer_norm_eps", 1e-12)))
        self.pooler = None
        if getattr(config, "add_pooling_layer", True):
            self.pooler = nn.Module()
            self.pooler.dense = nn.Linear(config.hidden_size, config.hidden_size)
        std = float(getattr(config, "initializer_range", 0.02))
        _init_bert_weights(self, std)
        self.embeddings.cls_token.data.normal_(0.0, std)
        self.embeddings.position_embeddings.data.normal_(0.0, std)

    def forward(self, input_values=None, attention_mask=None, output_hidden_states=False):
        """attention_mask: the 0/1 key mask [B, S] (1 = attend), as ViTModel.forward takes it (vit.py:276-284); it is turned
        into the additive (1 - m) * -10000 of get_extended_attention_mask before the encoder"""
        if input_values is None:
            raise ValueError("You have to specify input_values")
        do_patch = getattr(self.config, "do_patch_embeddings", True)
        emb = self.embeddings(input_values) if do_patch else input_values
        enc = self.encoder(emb, attention_mask=extended_attention_mask(attention_mask, self.layernorm.weight.dtype),
                           output_hidden_states=output_hidden_states, return_dict=True)
        shape = enc.last_hidden_state.shape
        seq = ops.layer_norm(enc.last_hidden_state.reshape(-1, shape[-1]), self.layernorm.weight, self.layernorm.bias,
                             self.layernorm.eps).view(shape).to(self.layernorm.weight.dtype)
        pooled = None
        if self.pooler is not None:                       # HF ViTPooler: tanh(dense(first token))
            pooled = torch.tanh(ops.linear_any(seq[:, 0], self.pooler.dense.weight, self.pooler.dense.bias).to(seq.dtype))
        return (seq, pooled, enc.hidden_states) if output_hidden_states else (seq, pooled)
