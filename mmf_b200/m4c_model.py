"""The registered `m4c` and `m4c_captioner` models on the fused trunk.

  registry.register_model("m4c")            M4C           <->  mmf/models/m4c.py:34-347
  registry.register_model("m4c_captioner")  M4CCaptioner  <->  mmf/models/m4c_captioner.py:6-24
  B200TextBert                                            <->  TextBert             m4c.py:350-372
  B200MMT                                                 <->  MMT                  m4c.py:375-456
  B200PrevPredEmbeddings                                  <->  PrevPredEmbeddings   m4c.py:493-539
  B200OcrPtrNet                                           <->  OcrPtrNet            m4c.py:459-490

State-dict keys equal the reference's (`text_bert.encoder.layer.*`, `mmt.prev_pred_embeddings.*`, `mmt.encoder.layer.*`,
`obj_faster_rcnn_fc7.lc.*` - legacy `module.lc.*` accepted -, `ocr_ptr_net.query.*`, `classifier.module.*` ...), so M4C
checkpoints load.

What runs where:
  * the text BERT is the library's BERT text embeddings (composer + LayerNorm) and a B200BertEncoder with its 2-D key
    mask.  It does not read `prev_inds`, so greedy decoding runs it once per forward, not once per step;
  * the object and OCR encodings run their fc7 (GEMM + ReLU epilogue), their projections (the K = 3002 OCR features and
    the K = 4 boxes zero-padded to the GEMM's pitch by ops.linear_any) and their LayerNorms on the library;
  * the multimodal transformer is ONE encoder call over [text | objects | OCR | decoding steps]: the key mask of the first
    three plus a causal tail over the decoding steps (engine.CausalTail, `causal_len` of the attention kernels) - the
    reference's prefix-LM mask (m4c.py:418-437) without a [B, S, S] tensor;
  * PrevPredEmbeddings: the answer and OCR LayerNorms (the answer one reads the tied `classifier.module.weight`; autograd
    sums the gradients of its two uses), and position + type embeddings -> LayerNorm -> dropout in the composer;
  * the answer classifier and the pointer network's query / key projections are library GEMMs.
Torch ops on kernel outputs: F.normalize of the fc7 / FastText / PHOC features, the sums of the two LayerNorm branches,
the dropouts of the object / OCR encodings, the gather of the previous predictions' embeddings (_batch_gather), the
pointer network's [B, dec, ocr] score product (a batched product, about 1.5 MFLOP per sample at TextVQA shapes: the GEMM
ABI has no batch) and its mask, the argmax of greedy decoding and the loss `m4c_decoding_bce_with_mask`.

Skip-padding (`patch.set_skip_padding(model, causal=True)`): the text BERT packs its valid question tokens, and the MMT
call packs the valid text, object and OCR rows plus every decoding step, and runs the packed attention kernels with the
causal tail.  The padded MMT rows then come out as exact zeros instead of the dense values.  This changes neither the loss
nor a parameter gradient beyond rounding and the dropout masks drawn:
  * the only padded MMT rows any consumer reads are the OCR rows, which B200OcrPtrNet scores with -10000 added (its
    key projection of a zero row is its bias, so both paths give a score near -10000 there);
  * m4c_decoding_bce_with_mask gives such a logit x, whose target is 0, the loss log1p(exp(x)) and the gradient
    sigmoid(x), both exactly 0 in fp32, so nothing flows back into those rows;
  * every valid row and every decoding step has at least one unmasked key, so the dense path gives each padded key
    (mask -10000) a softmax weight of exactly 0 in fp32 - the keys packing removes.
So the returned `scores` differ only at padded OCR slots, where both paths are near -10000, and greedy decoding picks the
same tokens unless two valid scores tie within rounding.  (With `causal=False`, skip_padding packs the text BERT only.)

There is no hub: `text_bert_init_from_bert_base: true` selects the bert-base hyper-parameters (BertConfig's defaults
under `text_bert`) and puts the text BERT in its own learning-rate group, as the reference does; its weights, and the
fc7 weights and biases the reference reads from detectron pickles, arrive through load_state_dict.
"""
import copy
import math

import torch
from torch import nn

from . import ops
from .encoders import build_image_encoder
from .models import BERT_BASE, LOSSES, MODEL_DEFAULTS, BaseModel, ConfigNode
from .modules import B200BertEncoder, _init_bert_weights, _require_cuda, run_bert_encoder
from .registry import registry
from .vilbert import B200BertTextEmbeddings

TEXT_BERT_HIDDEN_SIZE = 768   # m4c.py:70, fixed in the reference

# mmf/configs/models/m4c/defaults.yaml:1-29
MODEL_DEFAULTS["m4c"] = dict(
    lr_scale_frcn=0.1, lr_scale_text_bert=0.1, lr_scale_mmt=1.0, text_bert_init_from_bert_base=True,
    text_bert=dict(num_hidden_layers=3), obj=dict(mmt_in_dim=2048, dropout_prob=0.1),
    ocr=dict(mmt_in_dim=3002, dropout_prob=0.1), mmt=dict(hidden_size=768, num_hidden_layers=4),
    classifier=dict(type="linear", ocr_max_num=50, ocr_ptr_net=dict(hidden_size=768, query_key_size=768), params={}),
    model_data_dir="${env.data_dir}", losses=[dict(type="m4c_decoding_bce_with_mask")])
# mmf/configs/models/m4c_captioner/defaults.yaml:1-30
MODEL_DEFAULTS["m4c_captioner"] = dict(copy.deepcopy(MODEL_DEFAULTS["m4c"]), remove_unk_in_pred=True)


def _loss_m4c_decoding_bce_with_mask(sample_list, model_output):
    """mmf/modules/losses.py:576-592: BCE with logits per decoding step and answer, times train_loss_mask, summed, over
    max(sum(train_loss_mask), 1)"""
    scores, targets, loss_mask = model_output["scores"].float(), sample_list["targets"], sample_list["train_loss_mask"]
    assert scores.dim() == 3 and loss_mask.dim() == 2
    losses = nn.functional.binary_cross_entropy_with_logits(scores, targets.float(), reduction="none")
    losses = losses * loss_mask.unsqueeze(-1)
    count = torch.clamp_min(torch.sum(loss_mask).float(), 1.0)
    return torch.sum(losses) / count


LOSSES["m4c_decoding_bce_with_mask"] = _loss_m4c_decoding_bce_with_mask


def bert_config(overrides):
    """BertConfig(**overrides): the bert-base defaults under the given keys"""
    return ConfigNode(dict(BERT_BASE, **dict(overrides or {})))


def _get_mask(nums, max_num):
    """m4c.py:542-548: float [B, max_num], 1 on the first nums[b] positions"""
    arange = torch.arange(0, max_num, device=nums.device).unsqueeze(0).expand(nums.size(0), -1)
    return arange.lt(nums.unsqueeze(-1)).to(torch.float32)


def extended_attention_mask(key_mask, dec_len):
    """The [B, 1, S, S] additive mask the reference's MMT builds (m4c.py:427-437) from the 0/1 key mask of the encoding
    steps [B, S - dec_len]: what the encoder call's 2-D mask plus causal tail compute, as a tensor (for inspection)"""
    B, P = key_mask.shape
    S = P + dec_len
    m = torch.cat([key_mask.float(), key_mask.new_zeros(B, dec_len, dtype=torch.float32)], dim=1)
    m = m[:, None, None, :].repeat(1, 1, S, 1)
    m[:, :, -dec_len:, -dec_len:] = torch.tril(torch.ones(dec_len, dec_len, device=key_mask.device))
    return (1.0 - m) * -10000.0


def _linear(x, lin):
    shape = x.shape
    return ops.linear_any(x.reshape(-1, shape[-1]), lin.weight, lin.bias).view(*shape[:-1], lin.out_features)


def _layer_norm(x, ln):
    shape = x.shape
    return ops.layer_norm(x.reshape(-1, shape[-1]), ln.weight, ln.bias, ln.eps).view(shape)


class B200TextBert(nn.Module):
    """TextBert (m4c.py:350-372): BERT embeddings of the question tokens -> BERT encoder with their key mask"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embeddings = B200BertTextEmbeddings(config)
        self.encoder = B200BertEncoder(config)
        _init_bert_weights(self, float(config.initializer_range))

    def forward(self, txt_inds, txt_mask):
        emb = self.embeddings(txt_inds)
        ext = (1.0 - txt_mask[:, None, None, :]) * -10000.0
        return self.encoder(emb, ext)[0]


class B200PrevPredEmbeddings(nn.Module):
    """PrevPredEmbeddings (m4c.py:493-539): embeddings of the previous step's predictions - the LayerNormed answer
    embedding (the classifier's weight row) or OCR token - plus LayerNorm(position + type embeddings)"""

    MAX_DEC_LENGTH, MAX_TYPE_NUM = 100, 5

    def __init__(self, config):
        super().__init__()
        H, eps = config.hidden_size, float(config.layer_norm_eps)
        self.position_embeddings = nn.Embedding(self.MAX_DEC_LENGTH, H)
        self.token_type_embeddings = nn.Embedding(self.MAX_TYPE_NUM, H)
        self.ans_layer_norm = nn.LayerNorm(H, eps=eps)
        self.ocr_layer_norm = nn.LayerNorm(H, eps=eps)
        self.emb_layer_norm = nn.LayerNorm(H, eps=eps)
        self.emb_dropout = nn.Dropout(float(config.hidden_dropout_prob))

    def forward(self, ans_emb, ocr_emb, prev_inds):
        assert prev_inds.dim() == 2 and prev_inds.dtype == torch.long
        assert ans_emb.dim() == 2
        B, T = prev_inds.shape
        A, O, H = ans_emb.size(0), ocr_emb.size(1), ocr_emb.size(2)
        ans = _layer_norm(ans_emb, self.ans_layer_norm)
        ocr = _layer_norm(ocr_emb, self.ocr_layer_norm).reshape(B * O, H)
        # _batch_gather (m4c.py:561-573) over [answers | this sample's OCR tokens], without the [B, A + O, H] copy
        is_ocr = prev_inds.ge(A)
        ans_rows = torch.where(is_ocr, torch.zeros_like(prev_inds), prev_inds).reshape(-1)
        ocr_rows = (torch.arange(B, device=prev_inds.device).unsqueeze(-1) * O
                    + torch.where(is_ocr, prev_inds - A, torch.zeros_like(prev_inds))).reshape(-1)
        raw = torch.where(is_ocr.reshape(-1, 1), ocr.index_select(0, ocr_rows), ans.index_select(0, ans_rows))
        position_ids = torch.arange(T, device=prev_inds.device).unsqueeze(0).expand(B, T)
        emb = ops.compose_ln(B * T, H, [], [(self.position_embeddings.weight, ops.i32(position_ids)),
                                            (self.token_type_embeddings.weight, ops.i32(is_ocr.long()))],
                             self.emb_layer_norm.weight, self.emb_layer_norm.bias, self.emb_layer_norm.eps,
                             float(self.emb_dropout.p), self.training)
        return (raw.float() + emb.float()).view(B, T, H)


class B200MMT(nn.Module):
    """MMT (m4c.py:375-456): one BERT encoder call over [text | objects | OCR | decoding steps] with the prefix-LM mask -
    every query attends to the valid text, object and OCR keys, decoding step t also to decoding steps 0..t"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.prev_pred_embeddings = B200PrevPredEmbeddings(config)
        self.encoder = B200BertEncoder(config)
        _init_bert_weights(self, float(config.initializer_range))

    def forward(self, txt_emb, txt_mask, obj_emb, obj_mask, ocr_emb, ocr_mask, fixed_ans_emb, prev_inds):
        dec_emb = self.prev_pred_embeddings(fixed_ans_emb, ocr_emb, prev_inds)
        dt = torch.bfloat16
        x = torch.cat([txt_emb.to(dt), obj_emb.to(dt), ocr_emb.to(dt), dec_emb.to(dt)], dim=1)
        T, R, O, D = txt_mask.size(-1), obj_mask.size(-1), ocr_mask.size(-1), dec_emb.size(1)
        # the tail's keys take their mask from causal_len: the zeros here are never read
        key_mask = torch.cat([txt_mask, obj_mask, ocr_mask], dim=1)
        add_mask = torch.cat([(1.0 - key_mask) * -10000.0, key_mask.new_zeros(key_mask.size(0), D)], dim=1)
        seq = run_bert_encoder(self.encoder._runner, x, add_mask, self.training, causal_len=D)[0]
        return {"mmt_seq_output": seq, "mmt_txt_output": seq[:, :T], "mmt_ocr_output": seq[:, T + R:T + R + O],
                "mmt_dec_output": seq[:, -D:]}


class B200OcrPtrNet(nn.Module):
    """OcrPtrNet (m4c.py:459-490): scaled dot-product scores of the decoding steps over the OCR tokens, OCR padding at
    -10000"""

    def __init__(self, hidden_size, query_key_size=None):
        super().__init__()
        if query_key_size is None:
            query_key_size = hidden_size
        self.hidden_size, self.query_key_size = hidden_size, query_key_size
        self.query = nn.Linear(hidden_size, query_key_size)
        self.key = nn.Linear(hidden_size, query_key_size)

    def forward(self, query_inputs, key_inputs, attention_mask):
        extended_attention_mask = ((1.0 - attention_mask) * -10000.0).unsqueeze(1)
        query_layer = _linear(query_inputs, self.query).float()
        squeeze_result = query_layer.dim() == 2
        if squeeze_result:
            query_layer = query_layer.unsqueeze(1)
        key_layer = _linear(key_inputs, self.key).float()
        scores = torch.matmul(query_layer, key_layer.transpose(-1, -2)) / math.sqrt(self.query_key_size)
        scores = scores + extended_attention_mask
        return scores.squeeze(1) if squeeze_result else scores


class B200ClassifierLayer(nn.Module):
    """ClassifierLayer (mmf/modules/layers.py) of type "linear": `module` is the nn.Linear, run on the library GEMM"""

    def __init__(self, classifier_type, in_dim, out_dim, **kwargs):
        super().__init__()
        if classifier_type != "linear":
            raise NotImplementedError("M4C classifier type %r is not on the B200 path (linear only)" % (classifier_type,))
        self.module = nn.Linear(in_dim, out_dim, **kwargs)

    def forward(self, x):
        return _linear(x, self.module)


@registry.register_model("m4c")
class M4C(BaseModel):
    """M4C (m4c.py:34-347): TextVQA / ST-VQA answers decoded step by step from a fixed vocabulary or copied from the OCR
    tokens"""

    def __init__(self, config):
        super().__init__(config)
        self.mmt_config = bert_config(self.config.mmt)
        self._datasets = registry.get("config").datasets.split(",")

    @classmethod
    def config_path(cls):
        return "configs/models/m4c/defaults.yaml"

    def build(self):
        self.finetune_modules = []
        self._build_txt_encoding()
        self._build_obj_encoding()
        self._build_ocr_encoding()
        self._build_mmt()
        self._build_output()

    def _build_encoder_config(self):
        return {"type": "finetune_faster_rcnn_fpn_fc7",
                "params": {"in_dim": 2048, "weights_file": "models/detectron.defaults/fc7_w.pkl",
                           "bias_file": "models/detectron.defaults/fc7_b.pkl",
                           "model_data_dir": self.config.get("model_data_dir")}}

    def _build_txt_encoding(self):
        self.text_bert_config = bert_config(self.config.text_bert)
        self.text_bert = B200TextBert(self.text_bert_config)
        if self.config.text_bert_init_from_bert_base:
            self.finetune_modules.append({"module": self.text_bert, "lr_scale": self.config.lr_scale_text_bert})
        if self.mmt_config.hidden_size != TEXT_BERT_HIDDEN_SIZE:
            self.text_bert_out_linear = nn.Linear(TEXT_BERT_HIDDEN_SIZE, self.mmt_config.hidden_size)
        else:
            self.text_bert_out_linear = nn.Identity()

    def _build_obj_encoding(self):
        H = self.mmt_config.hidden_size
        self.obj_faster_rcnn_fc7 = build_image_encoder(self._build_encoder_config(), direct_features=True)
        self.finetune_modules.append({"module": self.obj_faster_rcnn_fc7, "lr_scale": self.config.lr_scale_frcn})
        self.linear_obj_feat_to_mmt_in = nn.Linear(self.config.obj.mmt_in_dim, H)
        self.linear_obj_bbox_to_mmt_in = nn.Linear(4, H)
        self.obj_feat_layer_norm = nn.LayerNorm(H)
        self.obj_bbox_layer_norm = nn.LayerNorm(H)
        self.obj_drop = nn.Dropout(self.config.obj.dropout_prob)

    def _build_ocr_encoding(self):
        H = self.mmt_config.hidden_size
        ocr = self.config.ocr
        self.remove_ocr_fasttext = ocr.get("remove_ocr_fasttext", False)
        self.remove_ocr_phoc = ocr.get("remove_ocr_phoc", False)
        self.remove_ocr_frcn = ocr.get("remove_ocr_frcn", False)
        self.remove_ocr_semantics = ocr.get("remove_ocr_semantics", False)
        self.remove_ocr_bbox = ocr.get("remove_ocr_bbox", False)
        self.ocr_faster_rcnn_fc7 = build_image_encoder(self._build_encoder_config(), direct_features=True)
        self.finetune_modules.append({"module": self.ocr_faster_rcnn_fc7, "lr_scale": self.config.lr_scale_frcn})
        self.linear_ocr_feat_to_mmt_in = nn.Linear(ocr.mmt_in_dim, H)
        self.linear_ocr_bbox_to_mmt_in = nn.Linear(4, H)
        self.ocr_feat_layer_norm = nn.LayerNorm(H)
        self.ocr_bbox_layer_norm = nn.LayerNorm(H)
        self.ocr_drop = nn.Dropout(ocr.dropout_prob)

    def _build_mmt(self):
        self.mmt = B200MMT(self.mmt_config)
        self.finetune_modules.append({"module": self.mmt, "lr_scale": self.config.lr_scale_mmt})

    def _build_output(self):
        cls = self.config.classifier
        self.ocr_ptr_net = B200OcrPtrNet(**cls.ocr_ptr_net)
        num_choices = registry.get(self._datasets[0] + "_num_final_outputs") - cls.ocr_max_num
        self.classifier = B200ClassifierLayer(cls.type, in_dim=self.mmt_config.hidden_size, out_dim=num_choices,
                                              **cls.get("params", {}))
        self.answer_processor = registry.get(self._datasets[0] + "_answer_processor")

    # ---- forward ----------------------------------------------------------------------------------------------------
    def forward(self, sample_list):
        _require_cuda(sample_list["text"], "text")
        fwd_results = {}
        self._forward_txt_encoding(sample_list, fwd_results)
        self._forward_obj_encoding(sample_list, fwd_results)
        self._forward_ocr_encoding(sample_list, fwd_results)
        self._forward_mmt_and_output(sample_list, fwd_results)
        return {"scores": fwd_results["scores"]}

    def _forward_txt_encoding(self, sample_list, fwd_results):
        fwd_results["txt_inds"] = sample_list["text"]
        fwd_results["txt_mask"] = _get_mask(sample_list["text_len"], sample_list["text"].size(1))

    def _encode(self, feat, bbox, lin_feat, ln_feat, lin_bbox, ln_bbox, drop):
        """LN(Linear(feat)) + LN(Linear(bbox)) -> dropout (m4c.py:201-204, 245-248)"""
        out = _layer_norm(_linear(feat, lin_feat), ln_feat).float() + _layer_norm(_linear(bbox, lin_bbox), ln_bbox).float()
        return drop(out)

    def _forward_obj_encoding(self, sample_list, fwd_results):
        obj_fc7 = nn.functional.normalize(self.obj_faster_rcnn_fc7(sample_list["image_feature_0"]).float(), dim=-1)
        fwd_results["obj_mmt_in"] = self._encode(obj_fc7, sample_list["obj_bbox_coordinates"], self.linear_obj_feat_to_mmt_in,
                                                 self.obj_feat_layer_norm, self.linear_obj_bbox_to_mmt_in,
                                                 self.obj_bbox_layer_norm, self.obj_drop)
        obj_nums = _info(sample_list["image_info_0"], "max_features")
        fwd_results["obj_mask"] = _get_mask(obj_nums, fwd_results["obj_mmt_in"].size(1))

    def _forward_ocr_encoding(self, sample_list, fwd_results):
        ocr_fasttext = nn.functional.normalize(sample_list["context_feature_0"], dim=-1)
        assert ocr_fasttext.size(-1) == 300
        ocr_phoc = nn.functional.normalize(sample_list["context_feature_1"], dim=-1)
        assert ocr_phoc.size(-1) == 604
        ocr_fc6 = sample_list["image_feature_1"][:, :ocr_fasttext.size(1), :]
        ocr_fc7 = nn.functional.normalize(self.ocr_faster_rcnn_fc7(ocr_fc6).float(), dim=-1)
        ocr_order_vectors = torch.zeros_like(sample_list["order_vectors"])
        if self.remove_ocr_fasttext:
            ocr_fasttext = torch.zeros_like(ocr_fasttext)
        if self.remove_ocr_phoc:
            ocr_phoc = torch.zeros_like(ocr_phoc)
        if self.remove_ocr_frcn:
            ocr_fc7 = torch.zeros_like(ocr_fc7)
        ocr_feat = torch.cat([ocr_fasttext, ocr_phoc, ocr_fc7, ocr_order_vectors.to(ocr_fc7.dtype)], dim=-1)
        ocr_bbox = sample_list["ocr_bbox_coordinates"]
        if self.remove_ocr_semantics:
            ocr_feat = torch.zeros_like(ocr_feat)
        if self.remove_ocr_bbox:
            ocr_bbox = torch.zeros_like(ocr_bbox)
        fwd_results["ocr_mmt_in"] = self._encode(ocr_feat, ocr_bbox, self.linear_ocr_feat_to_mmt_in, self.ocr_feat_layer_norm,
                                                 self.linear_ocr_bbox_to_mmt_in, self.ocr_bbox_layer_norm, self.ocr_drop)
        ocr_nums = _info(sample_list["context_info_0"], "max_features")
        fwd_results["ocr_mask"] = _get_mask(ocr_nums, fwd_results["ocr_mmt_in"].size(1))

    def _forward_txt_bert(self, fwd_results):
        text_bert_out = self.text_bert(txt_inds=fwd_results["txt_inds"], txt_mask=fwd_results["txt_mask"])
        lin = self.text_bert_out_linear
        fwd_results["txt_emb"] = text_bert_out if isinstance(lin, nn.Identity) else _linear(text_bert_out, lin)

    def _forward_mmt(self, sample_list, fwd_results):
        fwd_results.update(self.mmt(txt_emb=fwd_results["txt_emb"], txt_mask=fwd_results["txt_mask"],
                                    obj_emb=fwd_results["obj_mmt_in"], obj_mask=fwd_results["obj_mask"],
                                    ocr_emb=fwd_results["ocr_mmt_in"], ocr_mask=fwd_results["ocr_mask"],
                                    fixed_ans_emb=self.classifier.module.weight, prev_inds=fwd_results["prev_inds"]))

    def _forward_output(self, sample_list, fwd_results):
        mmt_dec_output = fwd_results["mmt_dec_output"]
        fixed_scores = self.classifier(mmt_dec_output).float()
        dynamic_ocr_scores = self.ocr_ptr_net(mmt_dec_output, fwd_results["mmt_ocr_output"], fwd_results["ocr_mask"])
        fwd_results["scores"] = torch.cat([fixed_scores, dynamic_ocr_scores], dim=-1)

    def _forward_mmt_and_output(self, sample_list, fwd_results):
        # the text BERT does not read prev_inds: once per forward, also when decoding
        self._forward_txt_bert(fwd_results)
        if self.training:
            fwd_results["prev_inds"] = sample_list["train_prev_inds"].clone()
            self._forward_mmt(sample_list, fwd_results)
            self._forward_output(sample_list, fwd_results)
        else:
            dec_step_num = sample_list["train_prev_inds"].size(1)
            fwd_results["prev_inds"] = torch.zeros_like(sample_list["train_prev_inds"])
            fwd_results["prev_inds"][:, 0] = self.answer_processor.BOS_IDX
            # greedy decoding (m4c.py:295-304)
            for _ in range(dec_step_num):
                self._forward_mmt(sample_list, fwd_results)
                self._forward_output(sample_list, fwd_results)
                argmax_inds = fwd_results["scores"].argmax(dim=-1)
                fwd_results["prev_inds"][:, 1:] = argmax_inds[:, :-1]

    def get_optimizer_parameters(self, config):
        """m4c.py:306-328: the fc7 encoders, the text BERT (when initialised from bert-base) and the MMT at their scaled
        learning rates; every other parameter at the base rate, in the first group"""
        base_lr = config.optimizer.params.lr
        groups, finetune = [], set()
        for m in self.finetune_modules:
            params = list(m["module"].parameters())
            groups.append({"params": params, "lr": base_lr * m["lr_scale"]})
            finetune.update(params)
        groups.insert(0, {"params": [p for p in self.parameters() if p not in finetune]})
        return groups

    @classmethod
    def update_registry_for_pretrained(cls, config, checkpoint, full_output):
        """m4c.py:330-347: the registry entries build() reads, from a checkpoint's config and classifier"""
        datasets = full_output["full_config"].datasets
        dataset = datasets.split(",")[0]
        registry.register("config", ConfigNode({"datasets": datasets}))
        registry.register(dataset + "_num_final_outputs",
                          checkpoint["classifier.module.weight"].size(0) + config.classifier.ocr_max_num)
        registry.register(dataset + "_answer_processor", ConfigNode({"BOS_IDX": 1}))


@registry.register_model("m4c_captioner")
class M4CCaptioner(M4C):
    """M4CCaptioner (m4c_captioner.py:6-24): M4C for TextCaps; `remove_unk_in_pred` keeps <unk> out of the captions"""

    def __init__(self, config):
        super().__init__(config)
        self.remove_unk_in_pred = self.config.remove_unk_in_pred

    @classmethod
    def config_path(cls):
        return "configs/models/m4c_captioner/defaults.yaml"

    def _forward_output(self, sample_list, fwd_results):
        super()._forward_output(sample_list, fwd_results)
        if self.remove_unk_in_pred:
            fwd_results["scores"][..., self.answer_processor.UNK_IDX] = -1e10
        return fwd_results


def _info(info, key):
    return info[key] if isinstance(info, dict) else getattr(info, key)
