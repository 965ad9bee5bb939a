"""VisualBERT trunk on the B200 engine - the single-stream configuration of the fusion block
(BASELINE.json config 2: 12L/768, 128 tokens + 100 regions).

Mirrors, for the hot path only (embeddings -> 12x BERT layer -> pooler), the reference's
  VisualBERTBase.forward                      mmf/models/visual_bert.py:74-157
  VisualBERT.add_custom_params / add_post_flatten_params / flatten_for_bert   visual_bert.py:444-481, 538-556
with the same sub-module names (`embeddings`, `encoder`, `pooler`) so `bert.*` checkpoint keys map 1:1.
Task heads (MLM decoder, classifier) are consumers of this trunk and stay in torch (SURVEY.md 8f).
"""
import torch
from torch import nn

from .embeddings import B200VisioLinguisticEmbeddings
from .modules import B200BertEncoder, B200BertLayer, EncoderRunner, _init_bert_weights, run_bert_encoder


class BertPooler(nn.Module):
    """HF BertPooler: tanh(dense(h[:, 0])) (visual_bert.py:146): the [B, H] x [H, H]^T product on the wgmma GEMM, tanh as
    a torch elementwise op on the [B, H] result."""

    def __init__(self, hidden):
        super().__init__()
        self.dense = nn.Linear(hidden, hidden)
        self.activation = nn.Tanh()

    def forward(self, hidden_states):
        from . import ops
        first = hidden_states[:, 0]
        return self.activation(ops.linear_any(first, self.dense.weight, self.dense.bias).to(self.dense.weight.dtype))


def image_mask_from_dims(max_features, num_regions):
    """image_mask = arange(R) < image_dim   (int64 [B,R])  - visual_bert.py:538-556, bit-exact integer path"""
    ar = torch.arange(num_regions, device=max_features.device).expand(max_features.shape[0], num_regions)
    return (ar < max_features.unsqueeze(-1)).long()


class B200VisualBERTBase(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embeddings = B200VisioLinguisticEmbeddings(config)
        self.embeddings.output_dtype = torch.bfloat16   # internal hand-over to the encoder stays bf16 in HBM
        self.encoder = B200BertEncoder(config)
        self.pooler = BertPooler(config.hidden_size)
        _init_bert_weights(self.pooler, float(getattr(config, "initializer_range", 0.02)))
        self.bypass_transformer = bool(getattr(config, "bypass_transformer", False))
        if self.bypass_transformer:
            # visual_bert.py:66-67, 118-143: the encoder sees the text only; ONE extra BERT layer fuses
            # [text output ; visual embeddings].  The layer is a parameter holder driven by its own runner
            # (`_runner` on the module is also how mmf_b200.ddp finds the pack).
            self.additional_layer = B200BertLayer(
                config.hidden_size, config.num_attention_heads, config.intermediate_size,
                float(config.attention_probs_dropout_prob), float(config.hidden_dropout_prob),
                float(getattr(config, "layer_norm_eps", 1e-12)))
            _init_bert_weights(self.additional_layer, float(getattr(config, "initializer_range", 0.02)))
            self.additional_layer._runner = EncoderRunner([self.additional_layer])

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, visual_embeddings=None,
                visual_embeddings_type=None, image_text_alignment=None):
        """-> (sequence_output [B,S,H], pooled_output [B,H], [])   (visual_bert.py:74-157)"""
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        # (1 - mask) * -10000 in the parameters' dtype (visual_bert.py:94-106)
        ext = attention_mask.unsqueeze(1).unsqueeze(2).to(dtype=next(self.parameters()).dtype)
        ext = (1.0 - ext) * -10000.0
        emb = self.embeddings(input_ids, token_type_ids, visual_embeddings=visual_embeddings,
                              visual_embeddings_type=visual_embeddings_type,
                              image_text_alignment=image_text_alignment)
        dt = next(self.pooler.parameters()).dtype
        if self.bypass_transformer and visual_embeddings is not None:
            T = input_ids.size(1)
            text_out = self.encoder(emb[:, :T], ext[:, :, :T, :T])[0]        # [B,1,1,S] sliced -> [B,1,1,T]
            new_input = torch.cat((text_out.to(emb.dtype), emb[:, T:]), dim=1)
            seq = run_bert_encoder(self.additional_layer._runner, new_input, ext, self.training)[0].to(dt)
            return seq, self.pooler(seq), []
        seq = self.encoder(emb, ext)[0].to(dt)
        return seq, self.pooler(seq), []


class B200VisualBERT(nn.Module):
    """SampleList-level trunk: consumes the keys the reference reads (visual_bert.py:483-556) and returns the fused
    sequence / pooled output.  `sample_list` may be a SampleList or a plain dict of tensors."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.bert = B200VisualBERTBase(config)

    def forward(self, sample_list):
        input_ids = sample_list["input_ids"]
        input_mask = sample_list["input_mask"]
        segment_ids = sample_list["segment_ids"]
        feats = sample_list["image_feature_0"]
        info = sample_list.get("image_info_0", None) if hasattr(sample_list, "get") else None
        R = feats.shape[1]
        max_features = None
        if info is not None:
            max_features = info.get("max_features", None) if hasattr(info, "get") else getattr(info, "max_features", None)
        if max_features is None:
            max_features = torch.full((feats.shape[0],), R, dtype=torch.long, device=feats.device)
        image_mask = image_mask_from_dims(max_features.to(feats.device), R)          # add_custom_params
        visual_embeddings_type = torch.zeros_like(image_mask)                        # add_post_flatten_params
        attention_mask = torch.cat((input_mask, image_mask), dim=-1)
        seq, pooled, _ = self.bert(input_ids, attention_mask, segment_ids, feats, visual_embeddings_type)
        return {"sequence_output": seq, "pooled_output": pooled, "attention_mask": attention_mask,
                "image_mask": image_mask}


class B200VisualBERTForPretraining(nn.Module):
    """VisualBERTForPretraining (visual_bert.py:160-279) on the engine: `bert` trunk + `cls` heads with the decoder tied to
    the word embeddings (:219-228) + CrossEntropyLoss(ignore_index=-1).  STAGED with mmf_b200.heads (SURVEY.md 8f item 1).
    forward returns the reference's output dict: `logits`, `masked_lm_loss`, `loss` (when labels are given), plus
    `sequence_output` / `pooled_output` when `output_hidden_states` is set."""

    def __init__(self, config, mlm_positions="all"):
        super().__init__()
        from .heads import B200BertPreTrainingHeads
        self.config = config
        self.output_hidden_states = bool(getattr(config, "output_hidden_states", False))
        # The reference's trunk calls its encoder without output_attentions (visual_bert.py:144-157), so the
        # attention_weights it reports are always the empty tuple; so are they here.
        self.output_attentions = bool(getattr(config, "output_attentions", False))
        self.bert = B200VisualBERTBase(config)
        self.vocab_size = config.vocab_size
        self.cls = B200BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight)
        self.mlm_positions = mlm_positions

    def forward(self, input_ids, input_mask, attention_mask=None, token_type_ids=None, visual_embeddings=None,
                visual_embeddings_type=None, image_text_alignment=None, masked_lm_labels=None):
        from .heads import masked_lm_loss
        sequence_output, pooled_output, _ = self.bert(input_ids, attention_mask, token_type_ids, visual_embeddings,
                                                      visual_embeddings_type, image_text_alignment)
        out = {}
        if self.output_attentions:
            out["attention_weights"] = ()
        if self.output_hidden_states:
            out["sequence_output"], out["pooled_output"] = sequence_output, pooled_output
        if masked_lm_labels is not None:
            loss, logits = masked_lm_loss(self.cls, sequence_output, masked_lm_labels, positions=self.mlm_positions)
            out["logits"] = logits
            out["masked_lm_loss"] = loss
            out["loss"] = loss
        return out
