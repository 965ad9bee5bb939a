"""Masked-LM pre-training head on the B200 kernels (SURVEY.md 8f item 1; STAGED: host code CPU-verified against the
HuggingFace module the reference instantiates, not yet run or measured on the GPU).

  B200BertPredictionHeadTransform / B200BertLMPredictionHead / B200BertPreTrainingHeads
      <->  HF BertPreTrainingHeads, used as `self.cls` at mmf/models/visual_bert.py:205-214, 269-277
           (prediction_scores over ALL positions, CrossEntropyLoss(ignore_index=-1)).

Parameter names follow the reference's pinned transformers (<= 4.10): `predictions.transform.{dense,LayerNorm}`,
`predictions.decoder.weight` (tied to the word embeddings, visual_bert.py:219-228), `predictions.bias` with
`predictions.decoder.bias` as an alias, `seq_relationship`.

The vocabulary GEMM [tokens, H] x [V, H]^T is 10.7 GFLOP per VisualBERT sample forward (SURVEY.md 8a row a15).  V = 30522
is not a multiple of 8 (the 16-byte TMA row pitch), so the bf16 compute copy of the decoder weight / bias - which is
re-made from the fp32 master every step anyway - is zero-padded to the next multiple of 8 and the logits are a
column slice of the padded product; autograd's slice / pad backward routes the gradients.
`positions="masked"` evaluates only the rows whose label is not ignore_index (what MMFT's MLM head does,
mmf/models/transformers/heads/mlm.py:79-82): identical loss, ~7x less work; the default reproduces the reference's
full `logits` output.
Inside mmf_b200.graphs.static_rows() the "fused" and "masked" positions run `static_masked_lm_loss`: the labelled rows
are selected and counted on the device, so the head can be captured in a CUDA graph (no logits are returned).
"""
import torch
from torch import nn

from . import functional as F
from . import graphs
from . import ops
from .modules import _init_bert_weights, _require_cuda


class B200BertPredictionHeadTransform(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=float(getattr(config, "layer_norm_eps", 1e-12)))

    def forward(self, hidden_states):
        shape = hidden_states.shape
        h = ops.linear_gelu(hidden_states.reshape(-1, shape[-1]), self.dense.weight, self.dense.bias)
        h = ops.layer_norm(h, self.LayerNorm.weight, self.LayerNorm.bias, self.LayerNorm.eps)
        return h.view(*shape[:-1], -1)


class B200BertLMPredictionHead(nn.Module):
    def __init__(self, config, bert_model_embedding_weights=None):
        super().__init__()
        self.transform = B200BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        if bert_model_embedding_weights is not None:
            self.decoder.weight = bert_model_embedding_weights           # tie (visual_bert.py:219-228)
        self.bias = nn.Parameter(torch.zeros(config.vocab_size))
        self.decoder.bias = self.bias                                    # the alias transformers <= 4.10 keeps

    def forward(self, hidden_states):
        h = self.transform(hidden_states)
        shape = h.shape
        V = self.decoder.weight.shape[0]
        pad = (-V) % 8
        w = nn.functional.pad(self.decoder.weight, (0, 0, 0, pad)) if pad else self.decoder.weight
        b = nn.functional.pad(self.bias, (0, pad)) if pad else self.bias
        logits = ops.linear(h.reshape(-1, shape[-1]), w, b)
        return logits[:, :V].view(*shape[:-1], V)


class B200BertPreTrainingHeads(nn.Module):
    """forward(sequence_output, pooled_output) -> (prediction_scores [B,S,V], seq_relationship_score [B,2])"""

    def __init__(self, config, bert_model_embedding_weights=None):
        super().__init__()
        self.predictions = B200BertLMPredictionHead(config, bert_model_embedding_weights)
        self.seq_relationship = nn.Linear(config.hidden_size, 2)         # [B, H] x [2, H]^T: a consumer, left to torch
        _init_bert_weights(self.predictions.transform, float(getattr(config, "initializer_range", 0.02)))
        _init_bert_weights(self.seq_relationship, float(getattr(config, "initializer_range", 0.02)))

    def forward(self, sequence_output, pooled_output):
        _require_cuda(sequence_output, "sequence_output")
        scores = self.predictions(sequence_output).to(sequence_output.dtype)
        return scores, self.seq_relationship(pooled_output)


def static_masked_lm_loss(predictions, sequence_output, labels, ignore_index=-1):
    """mean CE of the masked-LM head over the labelled rows, with no host read: the rows are selected on the device
    (F.select_rows) into a fixed capacity of every row of `labels`, zero past the count; the transform runs on the whole
    capacity, the vocabulary GEMM and the loss only on the labelled rows (ops.linear_cross_entropy with a count).  A
    batch with no labelled row gives a loss of exactly 0 and zero gradients.  `predictions` is a
    B200BertLMPredictionHead."""
    H = sequence_output.shape[-1]
    sel = F.select_rows(labels.reshape(-1).to(torch.int64).contiguous(), ignore_index)
    rows = ops.gather_rows(sequence_output.reshape(-1, H), sel)
    h = predictions.transform(rows)
    return ops.linear_cross_entropy(h, predictions.decoder.weight, predictions.bias, sel.labels, ignore_index,
                                    count=sel.count, scale=sel.scale)


def masked_lm_loss(cls, sequence_output, masked_lm_labels, ignore_index=-1, positions="all"):
    """the reference's loss (visual_bert.py:269-277).  Returns (loss, logits): logits are [B,S,V] for positions="all",
    [n_masked, V] for positions="masked" (rows in row-major order of the labelled positions).
    positions="fused": the labelled rows are gathered first (like "masked": identical loss and gradients, the ignored rows
    contribute nothing), then transform -> vocabulary GEMM -> cross-entropy run chunk by chunk with the loss kernel writing
    d(logits) in place (ops.linear_cross_entropy): no logits tensor is returned (None) or ever materialised as a whole.
    Inside graphs.static_rows(), "fused" and "masked" run static_masked_lm_loss and return (loss, None)."""
    labels = masked_lm_labels.reshape(-1)
    H = sequence_output.shape[-1]
    if positions in ("fused", "masked") and graphs.static_rows_active():
        return static_masked_lm_loss(cls.predictions, sequence_output, labels, ignore_index), None
    if positions == "fused":
        idx = torch.nonzero(labels != ignore_index, as_tuple=False).squeeze(1)
        if idx.numel() == 0:
            return sequence_output.sum() * 0.0, None
        pred = cls.predictions
        h = pred.transform(sequence_output.reshape(-1, H).index_select(0, idx))
        loss = ops.linear_cross_entropy(h.reshape(-1, H), pred.decoder.weight, pred.bias, labels.index_select(0, idx),
                                        ignore_index)
        return loss, None
    if positions == "masked":
        idx = torch.nonzero(labels != ignore_index, as_tuple=False).squeeze(1)
        if idx.numel() == 0:
            # no labelled position in the batch: the reference's mean over zero targets is NaN and training goes on; the
            # GEMM rejects an empty problem, so hand back a zero loss that still connects to the graph
            return sequence_output.sum() * 0.0, sequence_output.new_zeros(0, cls.predictions.decoder.weight.shape[0])
        logits = cls.predictions(sequence_output.reshape(-1, H).index_select(0, idx))
        loss = nn.functional.cross_entropy(logits.float(), labels.index_select(0, idx), ignore_index=ignore_index)
        return loss, logits
    logits = cls.predictions(sequence_output)
    loss = nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]).float(), labels, ignore_index=ignore_index)
    return loss, logits
