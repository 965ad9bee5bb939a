"""UNITER trunk on the B200 engine (BASELINE.json configs[4]: UNITER / LXMERT-large class models; SURVEY.md 8f item 3).

  B200UNITERImageEmbeddings  <->  UNITERImageEmbeddings   mmf/models/uniter.py:43-88
  B200UNITERModelBase        <->  UNITERModelBase         mmf/models/uniter.py:91-243

Same sub-module / parameter names (`text_embeddings`, `img_embeddings.{img_linear,img_layer_norm,pos_linear,
pos_layer_norm,mask_embedding,final_layer_norm}`, `encoder`, `pooler`), forward signature and return structure
(`TransformerOutput(final_layer, hidden_layers)`).  Everything is a composition of the kernels the other front-ends use
(GEMM + bias, row LayerNorm, embedding composer + LayerNorm, the encoder); no new device code.
"""
from collections import namedtuple

import torch
from torch import nn

from . import ops
from .modules import B200BertEncoder, _init_bert_weights, _require_cuda
from .vilbert import B200BertTextEmbeddings
from .visual_bert import BertPooler


class B200UNITERImageEmbeddings(nn.Module):
    def __init__(self, img_dim=2048, hidden_size=768, eps=1e-12, hidden_dropout_prob=0.0, pos_dim=7):
        super().__init__()
        self.img_linear = nn.Linear(img_dim, hidden_size)
        self.img_layer_norm = nn.LayerNorm(hidden_size, eps=eps)
        self.pos_layer_norm = nn.LayerNorm(hidden_size, eps=eps)
        self.pos_linear = nn.Linear(pos_dim, hidden_size)
        self.mask_embedding = nn.Embedding(2, img_dim, padding_idx=0)
        self.final_layer_norm = nn.LayerNorm(hidden_size, eps=eps)
        self.dropout = nn.Dropout(hidden_dropout_prob)

    def forward(self, img_feat, img_pos_feat, type_embeddings, img_masks=None):
        _require_cuda(img_feat, "img_feat")
        B, R, Fd = img_feat.shape
        H = self.final_layer_norm.weight.shape[0]
        if img_masks is not None:                       # masked-region modelling: uniter.py:76-79
            self.mask_embedding.weight.data[0, :].fill_(0)
            img_feat = img_feat + self.mask_embedding(img_masks.long())
        im = ops.layer_norm(ops.linear(img_feat.reshape(B * R, Fd), self.img_linear.weight, self.img_linear.bias),
                            self.img_layer_norm.weight, self.img_layer_norm.bias, self.img_layer_norm.eps)
        # pos_dim = 7 is below the 16-byte TMA row pitch: zero-pad the columns (and the weight) to a multiple of 8
        pd = img_pos_feat.shape[-1]
        pad = (-pd) % 8
        pos_in = nn.functional.pad(img_pos_feat.reshape(B * R, pd).to(self.pos_linear.weight.dtype), (0, pad))
        pos = ops.layer_norm(ops.linear(pos_in, nn.functional.pad(self.pos_linear.weight, (0, pad)), self.pos_linear.bias),
                             self.pos_layer_norm.weight, self.pos_layer_norm.bias, self.pos_layer_norm.eps)
        rows = torch.arange(B * R, device=img_feat.device, dtype=torch.int32)
        # three dense terms: the composer takes two, the type embeddings join the position term first
        pos = pos + type_embeddings.reshape(B * R, H).to(pos.dtype)
        y = ops.compose_ln(B * R, H, [(im, rows), (pos, rows)], [], self.final_layer_norm.weight, self.final_layer_norm.bias,
                           self.final_layer_norm.eps, float(self.dropout.p), self.training)
        return y.view(B, R, H)


class B200UNITERModelBase(nn.Module):
    """config: BertConfig-like (hidden_size, num_hidden_layers, num_attention_heads, intermediate_size, vocab_size,
    max_position_embeddings, type_vocab_size, dropouts ...).  Random-init here (the reference pulls bert-base-uncased
    from the hub); weights arrive through load_state_dict."""

    def __init__(self, config, img_dim=2048, hidden_dropout_prob=0.0, text_config=None):
        super().__init__()
        self.config = config
        # the reference builds the text embeddings from a BertConfig of their own (uniter.py:119-125)
        self.text_embeddings = B200BertTextEmbeddings(config if text_config is None else text_config)
        self.img_embeddings = B200UNITERImageEmbeddings(img_dim=img_dim, hidden_size=config.hidden_size,
                                                        hidden_dropout_prob=hidden_dropout_prob)
        self.encoder = B200BertEncoder(config)
        self.pooler = BertPooler(config.hidden_size)
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))

    def _compute_txt_embeddings(self, input_ids, position_ids, token_type_ids=None):
        return self.text_embeddings(input_ids=input_ids, position_ids=position_ids, token_type_ids=token_type_ids)

    def _compute_img_embeddings(self, img_feat, img_pos_feat, img_masks=None, img_type_ids=None):
        if img_type_ids is None:
            img_type_ids = torch.ones_like(img_feat[:, :, 0].long())
        img_type_embeddings = self.text_embeddings.token_type_embeddings(img_type_ids)
        return self.img_embeddings(img_feat, img_pos_feat, img_type_embeddings, img_masks)

    def _compute_img_txt_embeddings(self, input_ids, position_ids, img_feat, img_pos_feat, img_masks=None,
                                    txt_type_ids=None, img_type_ids=None):
        txt = self._compute_txt_embeddings(input_ids, position_ids, txt_type_ids)
        img = self._compute_img_embeddings(img_feat, img_pos_feat, img_masks, img_type_ids)
        return torch.cat([txt, img.to(txt.dtype)], dim=1)

    def forward(self, input_ids, position_ids, img_feat, img_pos_feat, attention_mask, img_masks=None, txt_type_ids=None,
                img_type_ids=None, input_modality="image-text"):
        ext = attention_mask.unsqueeze(1).unsqueeze(2).to(dtype=next(self.parameters()).dtype)
        ext = (1.0 - ext) * -10000.0
        if input_modality == "image":
            emb = self._compute_img_embeddings(img_feat, img_pos_feat, img_masks, img_type_ids)
        elif input_modality == "text":
            emb = self._compute_txt_embeddings(input_ids, position_ids, txt_type_ids)
        else:
            emb = self._compute_img_txt_embeddings(input_ids, position_ids, img_feat, img_pos_feat, img_masks,
                                                   txt_type_ids, img_type_ids)
        out = self.encoder(emb, ext, output_hidden_states=True)
        layers = namedtuple("TransformerOutput", ["final_layer", "hidden_layers"])
        dt = next(self.parameters()).dtype
        return layers(out[0].to(dt), out[1])
