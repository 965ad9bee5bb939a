"""LXMERT encoder on the B200 engine (BASELINE.json configs[4] class; SURVEY.md 8f item 3).

  B200VisualFeatEncoder  <->  VisualFeatEncoder   mmf/models/lxmert.py:196-223
  B200LXMERTXLayer       <->  LXMERTXLayer        mmf/models/lxmert.py:226-283   (parameter holder)
  B200LXMERTEncoder      <->  LXMERTEncoder       mmf/models/lxmert.py:286-336
  B200LXMERTBase         <->  LXMERTBase          mmf/models/lxmert.py:339-414   (embeddings + encoder + pooler)

Same sub-module / parameter names (`visn_fc.{visn_fc,visn_layer_norm,box_fc,box_layer_norm}`, `layer.{i}`,
`r_layers.{i}`, `x_layers.{i}.{visual_attention.att,visual_attention.output,lang_self_att,visn_self_att,lang_inter,
lang_output,visn_inter,visn_output}`) and the forward signature `(lang_feats, lang_attention_mask, (feats, boxes),
visn_attention_mask) -> (lang_feats, visn_feats)`.  No new device code: language / relational layers are BERT layers,
the cross-modality layer is engine.xlayer_fwd/bwd (one shared cross-attention block used in both directions), and
modules.TwoStreamRunner runs them as it runs ViLBERT's layers.
The registered model and its heads are in mmf_b200.models (`lxmert`).
"""
import torch
from torch import nn

from . import engine as E
from . import ops
from .modules import (B200BertAttention, B200BertIntermediate, B200BertLayer, B200BertSelfAttention,
                      B200BertSelfOutput, TwoStreamRunner, _Holder, _init_bert_weights, _require_cuda, run_two_stream_encoder)
from .vilbert import B200BertTextEmbeddings
from .visual_bert import BertPooler


class B200VisualFeatEncoder(nn.Module):
    """(LN(fc(feats)) + LN(fc(boxes))) / 2 -> dropout   (no final LayerNorm; without boxes the first term alone)"""

    def __init__(self, config):
        super().__init__()
        self.visn_fc = nn.Linear(config.visual_feat_dim, config.hidden_size)
        self.visn_layer_norm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.box_fc = nn.Linear(config.visual_pos_dim, config.hidden_size)
        self.box_layer_norm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(float(config.hidden_dropout_prob))

    def forward(self, visn_input):
        feats, boxes = visn_input
        _require_cuda(feats, "feats")
        B, R, Fd = feats.shape
        H = self.visn_layer_norm.weight.shape[0]
        x = ops.layer_norm(ops.linear(feats.reshape(B * R, Fd), self.visn_fc.weight, self.visn_fc.bias),
                           self.visn_layer_norm.weight, self.visn_layer_norm.bias, self.visn_layer_norm.eps)
        if boxes is not None:
            pd = boxes.shape[-1]
            pad = (-pd) % 8          # 4 box coordinates: below the 16-byte TMA row pitch
            b_in = nn.functional.pad(boxes.reshape(B * R, pd).to(self.box_fc.weight.dtype), (0, pad))
            y = ops.layer_norm(ops.linear(b_in, nn.functional.pad(self.box_fc.weight, (0, pad)), self.box_fc.bias),
                               self.box_layer_norm.weight, self.box_layer_norm.bias, self.box_layer_norm.eps)
            x = (x + y) / 2
        return self.dropout(x).view(B, R, H)


def _layer_norm_eps(config):
    """the eps of HF's BertAttention / BertOutput / BertSelfOutput, which every LXMERT layer is built from
    (lxmert.py:69-80, 233-248, 305-311): config.layer_norm_eps.  Only the visual feature encoder and the answer head
    fix 1e-12."""
    return float(getattr(config, "layer_norm_eps", 1e-12))


class _CrossAtt(_Holder):
    def __init__(self, hidden, heads, p_attn, p_hidden, eps):
        super().__init__()
        self.att = B200BertSelfAttention(hidden, heads, p_attn)
        self.output = B200BertSelfOutput(hidden, hidden, p_hidden, eps)


class B200LXMERTXLayer(_Holder):
    def __init__(self, config):
        super().__init__()
        h, nh, it = config.hidden_size, config.num_attention_heads, config.intermediate_size
        pa, ph = float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob)
        eps = _layer_norm_eps(config)
        self.visual_attention = _CrossAtt(h, nh, pa, ph, eps)
        self.lang_self_att = B200BertAttention(h, nh, pa, ph, eps)
        self.visn_self_att = B200BertAttention(h, nh, pa, ph, eps)
        self.lang_inter = B200BertIntermediate(h, it)
        self.lang_output = B200BertSelfOutput(it, h, ph, eps)
        self.visn_inter = B200BertIntermediate(h, it)
        self.visn_output = B200BertSelfOutput(it, h, ph, eps)


class B200LXMERTEncoder(nn.Module):
    """config: BertConfig-like + visual_feat_dim, visual_pos_dim, l_layers, x_layers, r_layers
    (mmf/configs/models/lxmert/defaults.yaml)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.visn_fc = B200VisualFeatEncoder(config)
        self.num_l_layers, self.num_x_layers, self.num_r_layers = config.l_layers, config.x_layers, config.r_layers
        mk = lambda: B200BertLayer(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                                   float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob),
                                   _layer_norm_eps(config))
        self.layer = nn.ModuleList([mk() for _ in range(self.num_l_layers)])
        self.x_layers = nn.ModuleList([B200LXMERTXLayer(config) for _ in range(self.num_x_layers)])
        self.r_layers = nn.ModuleList([mk() for _ in range(self.num_r_layers)])
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))
        # execution order: language layers, relational (vision) layers, cross-modality layers (lxmert.py:318-334)
        self._runner = TwoStreamRunner([(m, E.BertLayerW, (0,)) for m in self.layer] +
                                       [(m, E.BertLayerW, (1,)) for m in self.r_layers] +
                                       [(m, E.XLayerW, (0, 1)) for m in self.x_layers])
        self._runner.pack_streams = bool(getattr(config, "skip_padding", False))

    def forward(self, lang_feats, lang_attention_mask, visn_feats, visn_attention_mask=None):
        _require_cuda(lang_feats, "lang_feats")
        visn = self.visn_fc(visn_feats)
        visn = visn.to(lang_feats.dtype)
        outs = run_two_stream_encoder(self._runner, lang_feats, visn, lang_attention_mask, visn_attention_mask, self.training)
        if outs is None:              # every token of both streams is padding: outputs and input gradients are zeros
            return lang_feats * 0, visn * 0
        return outs


class B200LXMERTBase(nn.Module):
    """LXMERTBase (lxmert.py:339-414): HF BertEmbeddings (`embeddings`), the two-stream encoder (`encoder`) and the tanh
    pooler on the first language token (`pooler.dense`), so LXMERT checkpoints load key for key.

    forward(input_ids, token_type_ids, attention_mask, visual_feats, visual_loc, visual_attention_mask,
    output_all_attention_masks, output_all_encoded_layers) -> ((lang_feats, visn_feats), pooled_output).  Both masks
    become (1 - m) * -10000 in the parameter dtype; visual_attention_mask=None stays None (no key of the visual stream is
    masked).  The encoder's skip-padding (`config.skip_padding`, patch.set_skip_padding(two_stream=True)) applies here."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embeddings = B200BertTextEmbeddings(config)
        self.encoder = B200LXMERTEncoder(config)
        self.pooler = BertPooler(config.hidden_size)
        for m in (self.embeddings, self.pooler):
            _init_bert_weights(m, float(getattr(config, "initializer_range", 0.02)))

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, visual_feats=None, visual_loc=None,
                visual_attention_mask=None, output_all_attention_masks=False, output_all_encoded_layers=False):
        if output_all_encoded_layers:
            raise NotImplementedError("LXMERT output_all_encoded_layers: the reference raises too (lxmert.py:360-361)")
        if output_all_attention_masks:
            raise NotImplementedError("LXMERT output_all_attention_masks: the reference raises too (lxmert.py:362-363)")
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        dt = next(self.parameters()).dtype
        ext = (1.0 - attention_mask.unsqueeze(1).unsqueeze(2).to(dt)) * -10000.0
        ext_v = None
        if visual_attention_mask is not None:
            ext_v = (1.0 - visual_attention_mask.unsqueeze(1).unsqueeze(2).to(dt)) * -10000.0
        emb = self.embeddings(input_ids, token_type_ids)
        lang, visn = self.encoder(emb, ext, (visual_feats, visual_loc), ext_v)
        lang, visn = lang.to(dt), visn.to(dt)
        return (lang, visn), self.pooler(lang)
