"""LXMERT encoder on the B200 engine (BASELINE.json configs[4] class; SURVEY.md 8f item 3).

  B200VisualFeatEncoder  <->  VisualFeatEncoder   mmf/models/lxmert.py:196-223
  B200LXMERTXLayer       <->  LXMERTXLayer        mmf/models/lxmert.py:226-283   (parameter holder)
  B200LXMERTEncoder      <->  LXMERTEncoder       mmf/models/lxmert.py:286-336
  B200LXMERTBase         <->  LXMERTBase          mmf/models/lxmert.py:339-414   (embeddings + encoder + pooler)

Same sub-module / parameter names (`visn_fc.{visn_fc,visn_layer_norm,box_fc,box_layer_norm}`, `layer.{i}`,
`r_layers.{i}`, `x_layers.{i}.{visual_attention.att,visual_attention.output,lang_self_att,visn_self_att,lang_inter,
lang_output,visn_inter,visn_output}`) and the forward signature `(lang_feats, lang_attention_mask, (feats, boxes),
visn_attention_mask) -> (lang_feats, visn_feats)`.  No new device code: language / relational layers are BERT layers,
the cross-modality layer is engine.xlayer_fwd/bwd (one shared cross-attention block used in both directions).
The registered model and its heads are in mmf_b200.models (`lxmert`).
"""
import torch
from torch import nn

from . import engine as E
from . import ops
from .modules import (B200BertAttention, B200BertIntermediate, B200BertLayer, B200BertSelfAttention,
                      B200BertSelfOutput, _Holder, _Packing, _fresh_dropout_state, _init_bert_weights, _require_cuda,
                      plan_two_stream)
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


class _CrossAtt(_Holder):
    def __init__(self, hidden, heads, p_attn, p_hidden):
        super().__init__()
        self.att = B200BertSelfAttention(hidden, heads, p_attn)
        self.output = B200BertSelfOutput(hidden, hidden, p_hidden, 1e-12)


class B200LXMERTXLayer(_Holder):
    def __init__(self, config):
        super().__init__()
        h, nh, it = config.hidden_size, config.num_attention_heads, config.intermediate_size
        pa, ph = float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob)
        self.visual_attention = _CrossAtt(h, nh, pa, ph)
        self.lang_self_att = B200BertAttention(h, nh, pa, ph, 1e-12)
        self.visn_self_att = B200BertAttention(h, nh, pa, ph, 1e-12)
        self.lang_inter = B200BertIntermediate(h, it)
        self.lang_output = B200BertSelfOutput(it, h, ph, 1e-12)
        self.visn_inter = B200BertIntermediate(h, it)
        self.visn_output = B200BertSelfOutput(it, h, ph, 1e-12)


class LxmertRunner:
    """execution order: language layers, relational (vision) layers, cross-modality layers (lxmert.py:318-334)"""

    def __init__(self, layer, r_layers, x_layers):
        self.layer, self.r_layers, self.x_layers = list(layer), list(r_layers), list(x_layers)
        self.steps = [("l", i) for i in range(len(self.layer))] + [("r", i) for i in range(len(self.r_layers))] + \
                     [("x", i) for i in range(len(self.x_layers))]
        self.pack = None
        self.w = None
        self.grad_ready_hook = None
        # skip padded tokens in both streams (modules.plan_two_stream): every layer runs on each stream's valid rows only
        self.pack_streams = False

    def _mod(self, kind, i):
        return {"l": self.layer, "r": self.r_layers, "x": self.x_layers}[kind][i]

    def ensure(self, device):
        if self.pack is not None and self.pack.intact() and self.pack.device == device:
            return
        params = []
        for kind, i in self.steps:
            params += (E.XLayerW if kind == "x" else E.BertLayerW).params(self._mod(kind, i))
        for p in params:
            _require_cuda(p, "encoder parameter")
        self.pack = E.ParamPack(params, device)
        self.w = {(k, i): (E.XLayerW if k == "x" else E.BertLayerW)(self.pack, self._mod(k, i)) for k, i in self.steps}
        # offsets where the parameters of each execution step start (data-parallel bucket boundaries)
        self.step_offsets, idx = [], 0
        for kind, i in self.steps:
            self.step_offsets.append(self.pack.offsets[idx])
            idx += len((E.XLayerW if kind == "x" else E.BertLayerW).params(self._mod(kind, i)))

    @staticmethod
    def _p(mod):
        d = getattr(mod, "dropout", None)
        return float(getattr(d, "p", 0.0)) if d is not None else 0.0

    def forward(self, lang, visn, lmask, vmask, B, T, R, training, need_grad):
        ds = _fresh_dropout_state() if training else None
        saved = []
        for kind, i in self.steps:
            m, w = self._mod(kind, i), self.w[(kind, i)]
            if kind == "x":
                pa, ph = (self._p(m.visual_attention.att), self._p(m.visual_attention.output)) if training else (0.0, 0.0)
                lang, visn, s = E.xlayer_fwd(lang, visn, lmask, vmask, w, B, T, R, pa, ph, ds)
            else:
                pa, ph = (self._p(m.attention.self), self._p(m.attention.output)) if training else (0.0, 0.0)
                if kind == "l":
                    lang, s = E.bert_layer_fwd(lang, lmask, w, B, T, pa, ph, ds)
                else:
                    visn, s = E.bert_layer_fwd(visn, vmask, w, B, R, pa, ph, ds)
            saved.append(s if need_grad else None)
        return lang, visn, saved

    def backward(self, dl, dv, saved, lmask, vmask, B, T, R):
        for j in range(len(self.steps) - 1, -1, -1):
            kind, i = self.steps[j]
            w = self.w[(kind, i)]
            if kind == "x":
                dl, dv = E.xlayer_bwd(dl, dv, saved[j], lmask, vmask, w, B, T, R)
            elif kind == "l":
                dl = E.bert_layer_bwd(dl, saved[j], lmask, w, B, T)
            else:
                dv = E.bert_layer_bwd(dv, saved[j], vmask, w, B, R)
            saved[j] = None
            if self.grad_ready_hook is not None:
                E.join_side()
                self.grad_ready_hook(j)
        return dl, dv


class _LxmertEncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, runner, lmask, vmask, training, lang, visn, *params):
        B, T, H = lang.shape
        R = visn.shape[1]
        need_grad = any(ctx.needs_input_grad)
        runner.pack.refresh()
        l = lang.detach().to(torch.bfloat16).contiguous().view(B * T, H)
        v = visn.detach().to(torch.bfloat16).contiguous().view(B * R, H)
        if isinstance(lmask, _Packing):
            l, v, saved = runner.forward(lmask.pack(l), vmask.pack(v), lmask.varlen, vmask.varlen, B, T, R, training, need_grad)
            l, v = lmask.unpack(l, B * T), vmask.unpack(v, B * R)
        else:
            l, v, saved = runner.forward(l, v, lmask, vmask, B, T, R, training, need_grad)
        ctx.runner, ctx.saved, ctx.masks, ctx.dims, ctx.dtypes = runner, saved, (lmask, vmask), (B, T, R, H), (lang.dtype, visn.dtype)
        return l.view(B, T, H).to(lang.dtype), v.view(B, R, H).to(visn.dtype)

    @staticmethod
    def backward(ctx, dlang, dvisn):
        runner = ctx.runner
        B, T, R, H = ctx.dims
        if ctx.saved is None:
            raise RuntimeError("B200 LXMERT encoder: backward called twice")
        aliased = runner.pack.prepare_grads()
        dev = runner.pack.device
        dl = (dlang if dlang is not None else torch.zeros(B, T, H, device=dev)).to(torch.bfloat16).contiguous().view(B * T, H)
        dv = (dvisn if dvisn is not None else torch.zeros(B, R, H, device=dev)).to(torch.bfloat16).contiguous().view(B * R, H)
        lm, vm = ctx.masks
        if isinstance(lm, _Packing):
            dl, dv = runner.backward(lm.pack(dl), vm.pack(dv), ctx.saved, lm.varlen, vm.varlen, B, T, R)
            dl, dv = lm.unpack(dl, B * T), vm.unpack(dv, B * R)
        else:
            dl, dv = runner.backward(dl, dv, ctx.saved, lm, vm, B, T, R)
        ctx.saved = None
        return (None, None, None, None, dl.view(B, T, H).to(ctx.dtypes[0]), dv.view(B, R, H).to(ctx.dtypes[1])) + tuple(
            runner.pack.autograd_grads(aliased))


class B200LXMERTEncoder(nn.Module):
    """config: BertConfig-like + visual_feat_dim, visual_pos_dim, l_layers, x_layers, r_layers
    (mmf/configs/models/lxmert/defaults.yaml)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.visn_fc = B200VisualFeatEncoder(config)
        self.num_l_layers, self.num_x_layers, self.num_r_layers = config.l_layers, config.x_layers, config.r_layers
        mk = lambda: B200BertLayer(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                                   float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob), 1e-12)
        self.layer = nn.ModuleList([mk() for _ in range(self.num_l_layers)])
        self.x_layers = nn.ModuleList([B200LXMERTXLayer(config) for _ in range(self.num_x_layers)])
        self.r_layers = nn.ModuleList([mk() for _ in range(self.num_r_layers)])
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))
        self._runner = LxmertRunner(self.layer, self.r_layers, self.x_layers)
        self._runner.pack_streams = bool(getattr(config, "skip_padding", False))

    def forward(self, lang_feats, lang_attention_mask, visn_feats, visn_attention_mask=None):
        _require_cuda(lang_feats, "lang_feats")
        visn = self.visn_fc(visn_feats)
        B, T, _ = lang_feats.shape
        R = visn.shape[1]
        self._runner.ensure(lang_feats.device)
        lmask = E.additive_mask_2d(lang_attention_mask, B, T)
        vmask = E.additive_mask_2d(visn_attention_mask, B, R)
        visn = visn.to(lang_feats.dtype)
        if self._runner.pack_streams:
            plan = plan_two_stream(lmask, vmask, B, T, R, lang_feats.device)
            if plan == "empty":       # every token of both streams is padding: outputs and input gradients are zeros
                return lang_feats * 0, visn * 0
            if plan is not None:
                lmask, vmask = plan
        return _LxmertEncoderFn.apply(self._runner, lmask, vmask, self.training, lang_feats, visn, *self._runner.pack.params)


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
