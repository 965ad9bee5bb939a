"""TEST INFRASTRUCTURE - CPU restatement of the reference's multimodal-fusion hot path.

This file is the parity ORACLE.  It is not part of the product: only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import it, and only as the checker (or as
the timed CPU baseline).  mmf_b200/ never imports it.

Every function restates, in plain (differentiable) torch ops on whatever device/dtype it is given,
one function of facebookresearch/mmf (paths relative to /root/reference) or of the HuggingFace
`transformers` classes the reference imports (pinned >=3.4.0,<=4.10.1, requirements.txt:12; the
arithmetic of BertSelfOutput / BertIntermediate / BertOutput / BertPooler is unchanged in the
installed 5.5.0, SURVEY.md 8c).  Weights come in as a flat dict with the REFERENCE's state_dict
key names, so the same dict drives the reference module, this oracle and the CUDA path.

Pinning: the reference's tests hold no golden vectors for this path (SURVEY.md 4, 8c).  The oracle
is pinned instead against outputs of the reference's own source files executed in the build
container (oracle/make_golden.py -> tests/golden/*.pt, checked by tests/test_oracle_golden.py).

Dropout: the reference draws masks from torch's RNG, which no other implementation can reproduce;
every function here takes optional explicit keep-masks (bool, same shape as the dropped tensor)
and a probability p, and applies `x * keep / (1-p)` exactly where the reference applies
nn.Dropout.  keep=None means eval mode / p=0.
"""
import math

import torch
import torch.nn.functional as F

LN_EPS = 1e-12  # BertLayerNorm eps, mmf/models/vilbert.py:254,303,483,490; HF config.layer_norm_eps


# ----------------------------------------------------------------------------------------------
# primitives
# ----------------------------------------------------------------------------------------------
def linear(x, sd, prefix):
    return F.linear(x, sd[prefix + ".weight"], sd[prefix + ".bias"])


def layer_norm(x, sd, prefix, eps=LN_EPS):
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], eps)


def gelu_erf(x):
    """ACT2FN["gelu"]: exact erf GELU (mmf/models/vilbert.py:288-291)."""
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def dropout(x, keep, p):
    """keep: None (eval), a bool keep-mask (parity tests), or the string "rng" = draw like nn.Dropout does (used only
    by the timed CPU baseline, where the reference's own fused dropout is the fair comparison)."""
    if keep is None or p == 0.0:
        return x
    if isinstance(keep, str):
        return F.dropout(x, p, True)
    return x * keep.to(x.dtype) / (1.0 - p)


def extended_attention_mask(mask, dtype=torch.float32):
    """(1 - mask[:,None,None,:]) * -10000.0  - mmf/models/visual_bert.py:94-106,
    mmf/modules/hf_layers.py:439-455, mmf/models/mmbt.py:268-285, huggingface.py:216-222."""
    ext = mask[:, None, None, :].to(dtype)
    return (1.0 - ext) * -10000.0


def transpose_for_scores(x, heads):
    """mmf/modules/hf_layers.py:153-159"""
    b, s, h = x.shape
    return x.view(b, s, heads, h // heads).permute(0, 2, 1, 3)


def attention_core(q, k, v, add_mask, heads, keep=None, p=0.0):
    """softmax(QK^T/sqrt(d) + M) -> dropout -> .V -> merge heads.
    mmf/modules/hf_layers.py:182-210; mmf/models/vilbert.py:81-103, 421-437, 441-461."""
    if q.shape[-1] % heads != 0:
        raise ValueError(
            "The hidden size (%d) is not a multiple of the number of attention heads (%d)" % (q.shape[-1], heads))
    ql, kl, vl = (transpose_for_scores(t, heads) for t in (q, k, v))
    scores = torch.matmul(ql, kl.transpose(-1, -2))
    scores = scores / math.sqrt(ql.shape[-1])
    if add_mask is not None:
        scores = scores + add_mask
    probs = F.softmax(scores, dim=-1)
    probs = dropout(probs, keep, p)
    ctx = torch.matmul(probs, vl)
    ctx = ctx.permute(0, 2, 1, 3).contiguous()
    return ctx.view(ctx.shape[0], ctx.shape[1], -1), probs


# ----------------------------------------------------------------------------------------------
# BERT layer / encoder  (single stream: VisualBERT, MMBT, MMFTransformer, UNITER-shaped trunks)
# ----------------------------------------------------------------------------------------------
def bert_self_attention(x, add_mask, sd, prefix, heads, keep=None, p=0.0, kv=None, kv_mask=None):
    """BertSelfAttentionJit.forward, mmf/modules/hf_layers.py:161-213 (kv = encoder_hidden_states)."""
    q = linear(x, sd, prefix + ".query")
    src = x if kv is None else kv
    k = linear(src, sd, prefix + ".key")
    v = linear(src, sd, prefix + ".value")
    return attention_core(q, k, v, add_mask if kv is None else kv_mask, heads, keep, p)


def bert_self_output(ctx, residual, sd, prefix, keep=None, p=0.0):
    """HF BertSelfOutput / BertOutput: LayerNorm(dropout(dense(h)) + input); called at
    mmf/modules/hf_layers.py:248,290; ViLBERT copies mmf/models/vilbert.py:250-261,299-310."""
    h = linear(ctx, sd, prefix + ".dense")
    h = dropout(h, keep, p)
    return layer_norm(h + residual, sd, prefix + ".LayerNorm")


def bert_intermediate(x, sd, prefix):
    """HF BertIntermediate: gelu(dense(x)); mmf/modules/hf_layers.py:289, vilbert.py:284-296."""
    return gelu_erf(linear(x, sd, prefix + ".dense"))


def bert_layer(x, add_mask, sd, prefix, heads, masks=None, p_attn=0.0, p_hidden=0.0):
    """BertLayerJit.forward, mmf/modules/hf_layers.py:273-292 (== vilbert.BertLayer / BertImageLayer
    with dynamic_attention off, mmf/models/vilbert.py:138-146, 320-332).
    masks: optional dict with keep-masks 'attn' [B,h,S,S], 'self_out' [B,S,H], 'out' [B,S,H]."""
    masks = masks or {}
    ctx, probs = bert_self_attention(x, add_mask, sd, prefix + ".attention.self", heads, masks.get("attn"), p_attn)
    att = bert_self_output(ctx, x, sd, prefix + ".attention.output", masks.get("self_out"), p_hidden)
    inter = bert_intermediate(att, sd, prefix + ".intermediate")
    out = bert_self_output(inter, att, sd, prefix + ".output", masks.get("out"), p_hidden)
    return out, probs


def bert_encoder(x, add_mask, sd, prefix, num_layers, heads, masks=None, p_attn=0.0, p_hidden=0.0,
                 output_hidden_states=False):
    """BertEncoderJit.forward, mmf/modules/hf_layers.py:316-355. prefix e.g. 'encoder' -> encoder.layer.i"""
    all_h = []
    for i in range(num_layers):
        if output_hidden_states:
            all_h.append(x)
        lm = masks[i] if masks else None
        x, _ = bert_layer(x, add_mask, sd, "%s.layer.%d" % (prefix, i) if prefix else "layer.%d" % i, heads, lm,
                          p_attn, p_hidden)
    if output_hidden_states:
        all_h.append(x)
        return x, all_h
    return x


def bert_pooler(x, sd, prefix):
    """HF BertPooler: tanh(dense(h[:,0])); mmf/models/visual_bert.py:146, mmbt.py:311."""
    return torch.tanh(linear(x[:, 0], sd, prefix + ".dense"))


# ----------------------------------------------------------------------------------------------
# ViLBERT two-stream encoder
# ----------------------------------------------------------------------------------------------
def bi_attention(img, img_mask, txt, txt_mask, sd, prefix, heads, keep1=None, keep2=None, p_v=0.0, p_t=0.0):
    """BertBiAttention.forward, mmf/models/vilbert.py:388-475.
    Stream 1 = image (query1/key1/value1 on v_hidden), stream 2 = text.  context1 = text queries over
    image keys/values (masked by the IMAGE mask); context2 = image queries over text keys/values.
    The co-attention mask is built by the caller but never applied (vilbert.py:424-425,448-449)."""
    q1, k1, v1 = (linear(img, sd, prefix + "." + n + "1") for n in ("query", "key", "value"))
    q2, k2, v2 = (linear(txt, sd, prefix + "." + n + "2") for n in ("query", "key", "value"))
    ctx1, _ = attention_core(q2, k1, v1, img_mask, heads, keep1, p_v)   # [B,T,bi]
    ctx2, _ = attention_core(q1, k2, v2, txt_mask, heads, keep2, p_t)   # [B,R,bi]
    return ctx1, ctx2


def bi_output(h1, in1, h2, in2, sd, prefix, keep1=None, keep2=None, p_v=0.0, p_t=0.0):
    """BertBiOutput.forward, mmf/models/vilbert.py:496-512 (q_dense1/q_dense2 are never used)."""
    c1 = dropout(linear(h1, sd, prefix + ".dense1"), keep1, p_v)
    c2 = dropout(linear(h2, sd, prefix + ".dense2"), keep2, p_t)
    return layer_norm(c1 + in1, sd, prefix + ".LayerNorm1"), layer_norm(c2 + in2, sd, prefix + ".LayerNorm2")


def connection_layer(img, img_mask, txt, txt_mask, sd, prefix, heads, masks=None, p_v_attn=0.0, p_t_attn=0.0,
                     p_v_hidden=0.0, p_t_hidden=0.0):
    """BertConnectionLayer.forward, mmf/models/vilbert.py:528-556."""
    m = masks or {}
    bi1, bi2 = bi_attention(img, img_mask, txt, txt_mask, sd, prefix + ".biattention", heads, m.get("attn1"),
                            m.get("attn2"), p_v_attn, p_t_attn)
    # biOutput(bi_output2, input_tensor1, bi_output1, input_tensor2): image stream gets ctx2
    a1, a2 = bi_output(bi2, img, bi1, txt, sd, prefix + ".biOutput", m.get("bo1"), m.get("bo2"), p_v_hidden,
                       p_t_hidden)
    i1 = bert_intermediate(a1, sd, prefix + ".v_intermediate")
    o1 = bert_self_output(i1, a1, sd, prefix + ".v_output", m.get("v_out"), p_v_hidden)
    i2 = bert_intermediate(a2, sd, prefix + ".t_intermediate")
    o2 = bert_self_output(i2, a2, sd, prefix + ".t_output", m.get("t_out"), p_t_hidden)
    return o1, o2


def vilbert_schedule(v_biattention_id, t_biattention_id, num_t_layers, num_v_layers):
    """The layer interleaving of ViLBERT's BertEncoder.forward (mmf/models/vilbert.py:619-785) as a
    list of ('t', i) / ('v', i) / ('c', i) steps (fixed_*_layer = 0, with_coattention = True)."""
    steps, v_start, t_start = [], 0, 0
    for count, (v_end, t_end) in enumerate(zip(v_biattention_id, t_biattention_id)):
        steps += [("t", i) for i in range(t_start, t_end)]
        steps += [("v", i) for i in range(v_start, v_end)]
        steps.append(("c", count))
        v_start, t_start = v_end, t_end
    steps += [("v", i) for i in range(v_start, num_v_layers)]
    steps += [("t", i) for i in range(t_start, num_t_layers)]
    return steps


def vilbert_encoder(txt, img, txt_mask, img_mask, sd, prefix, cfg, masks=None, p_t_attn=0.0, p_t_hidden=0.0,
                    p_v_attn=0.0, p_v_hidden=0.0):
    """ViLBERT BertEncoder.forward, mmf/models/vilbert.py:590-796 (dynamic_attention, in_batch_pairs and FAST_MODE off
    as in mmf/configs/models/vilbert/defaults.yaml).
    cfg: dict with num_hidden_layers, v_num_hidden_layers, num_attention_heads, v_num_attention_heads,
    bi_num_attention_heads, v_biattention_id, t_biattention_id.
    masks: optional list of keep-mask dicts, one per step of vilbert_schedule (bert_layer's keys for a text / image layer,
    connection_layer's for a co-attention layer); p_t_* are the text stream's probabilities (attention_probs_dropout_prob,
    hidden_dropout_prob), p_v_* the image stream's (v_*)."""
    pre = prefix + "." if prefix else ""
    steps = vilbert_schedule(cfg["v_biattention_id"], cfg["t_biattention_id"], cfg["num_hidden_layers"],
                             cfg["v_num_hidden_layers"])
    for j, (kind, i) in enumerate(steps):
        m = masks[j] if masks else None
        if kind == "t":
            txt, _ = bert_layer(txt, txt_mask, sd, "%slayer.%d" % (pre, i), cfg["num_attention_heads"], m, p_t_attn,
                                p_t_hidden)
        elif kind == "v":
            img, _ = bert_layer(img, img_mask, sd, "%sv_layer.%d" % (pre, i), cfg["v_num_attention_heads"], m, p_v_attn,
                                p_v_hidden)
        else:
            img, txt = connection_layer(img, img_mask, txt, txt_mask, sd, "%sc_layer.%d" % (pre, i),
                                        cfg["bi_num_attention_heads"], m, p_v_attn, p_t_attn, p_v_hidden, p_t_hidden)
    return txt, img


def image_feature_embeddings(feat, loc, sd, prefix, keep=None, p=0.0):
    """BertImageFeatureEmbeddings.forward, mmf/models/vilbert.py:904-913."""
    e = linear(feat, sd, prefix + ".image_embeddings") + linear(loc, sd, prefix + ".image_location_embeddings")
    return dropout(layer_norm(e, sd, prefix + ".LayerNorm"), keep, p)


# ----------------------------------------------------------------------------------------------
# embeddings (VisualBERT / MMBT / MMFTransformer)
# ----------------------------------------------------------------------------------------------
def visio_linguistic_embeddings(input_ids, token_type_ids, visual_embeddings, visual_embeddings_type, sd, prefix,
                                image_text_alignment=None, keep=None, p=0.0):
    """BertVisioLinguisticEmbeddings.forward, mmf/modules/embeddings.py:423-459
    (encode_text :329-345, encode_image :347-370, get_position_embeddings_visual :372-421)."""
    B, T = input_ids.shape
    pos = torch.arange(T, dtype=torch.long, device=input_ids.device).unsqueeze(0).expand_as(input_ids)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    text = (embedding(sd[prefix + ".word_embeddings.weight"], input_ids, 0) + sd[prefix + ".position_embeddings.weight"][pos]
            + sd[prefix + ".token_type_embeddings.weight"][token_type_ids])
    if visual_embeddings is not None and visual_embeddings_type is not None:
        v = linear(visual_embeddings, sd, prefix + ".projection")
        tt = sd[prefix + ".token_type_embeddings_visual.weight"][visual_embeddings_type]
        zeros = torch.zeros(v.shape[:-1], dtype=torch.long, device=v.device)
        if image_text_alignment is not None:
            am = (image_text_alignment != -1).long()
            ali = am * image_text_alignment
            pv = sd[prefix + ".position_embeddings.weight"][ali] * am.unsqueeze(-1)
            pv = pv.sum(2)
            cnt = am.sum(2)
            cnt = torch.where(cnt == 0, torch.ones_like(cnt), cnt)
            pv = pv / cnt.unsqueeze(-1)
            pv = pv + sd[prefix + ".position_embeddings_visual.weight"][zeros]
        else:
            pv = sd[prefix + ".position_embeddings_visual.weight"][zeros]
        emb = torch.cat((text, v + pv + tt), dim=1)
    else:
        emb = text
    return dropout(layer_norm(emb, sd, prefix + ".LayerNorm"), keep, p)


def visual_bert_masks(input_mask, max_features, num_regions):
    """image_mask = arange(R) < image_dim; attention_mask = cat(input_mask, image_mask)
    mmf/models/visual_bert.py:538-556 (add_custom_params), :444-467 (add_post_flatten_params)."""
    image_mask = torch.arange(num_regions, device=input_mask.device).expand(input_mask.shape[0], num_regions)
    image_mask = (image_mask < max_features.unsqueeze(-1)).long()
    visual_embeddings_type = torch.zeros_like(image_mask)
    attention_mask = torch.cat((input_mask, image_mask), dim=-1)
    return image_mask, visual_embeddings_type, attention_mask


def embedding(table, ids, padding_idx=None):
    """nn.Embedding lookup; with padding_idx the row is read but receives no gradient (HF BertEmbeddings builds
    word_embeddings with padding_idx=config.pad_token_id=0; huggingface.py:70-75 does the same)."""
    out = table[ids]
    if padding_idx is None:
        return out
    return torch.where((ids == padding_idx).unsqueeze(-1), out.detach(), out)


def visual_bert_base(input_ids, attention_mask, token_type_ids, visual_embeddings, visual_embeddings_type, sd, num_layers,
                     heads, bypass_transformer=False, image_text_alignment=None):
    """VisualBERTBase.forward, mmf/models/visual_bert.py:74-157 -> (sequence_output, pooled_output).
    bypass_transformer (:118-143): encoder over the text part only, then `additional_layer` over [text ; visual]."""
    add = extended_attention_mask(attention_mask)
    emb = visio_linguistic_embeddings(input_ids, token_type_ids, visual_embeddings, visual_embeddings_type, sd, "embeddings",
                                      image_text_alignment)
    if bypass_transformer and visual_embeddings is not None:
        T = input_ids.shape[1]
        text = bert_encoder(emb[:, :T], add[:, :, :T, :T], sd, "encoder", num_layers, heads)
        seq, _ = bert_layer(torch.cat((text, emb[:, T:]), dim=1), add, sd, "additional_layer", heads)
    else:
        seq = bert_encoder(emb, add, sd, "encoder", num_layers, heads)
    return seq, bert_pooler(seq, sd, "pooler")


def bert_embeddings(input_ids, token_type_ids, sd, prefix, position_ids=None, keep=None, p=0.0, padding_idx=0):
    """BertEmbeddingsJit.forward, mmf/modules/hf_layers.py:107-135."""
    B, T = input_ids.shape
    if position_ids is None:
        position_ids = torch.arange(T, dtype=torch.long, device=input_ids.device).unsqueeze(0).expand(B, T)
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    e = (embedding(sd[prefix + ".word_embeddings.weight"], input_ids, padding_idx) + sd[prefix + ".position_embeddings.weight"][position_ids]
         + sd[prefix + ".token_type_embeddings.weight"][token_type_ids])
    return dropout(layer_norm(e, sd, prefix + ".LayerNorm"), keep, p)


def fc7_encoder(image, sd, prefix):
    """FinetuneFasterRcnnFpnFc7.forward: relu(lc(image)), mmf/modules/encoders.py:176-179."""
    return torch.relu(linear(image, sd, prefix + ".lc" if prefix else "lc"))


def widen_segment_table(old, num_segments, fresh):
    """TransformerEncoder._init_segment_embeddings, mmf/modules/encoders.py:563-575: rows 0,1 copied, rows
    2..n-2 = mean of the old table, the last row keeps its fresh nn.Embedding init (`fresh` [n,H])."""
    new = fresh.clone()
    new[:2] = old[:2]
    for idx in range(2, num_segments - 1):
        new[idx] = old.mean(dim=0)
    return new


def transformer_encoder(input_ids, attention_mask, token_type_ids, sd, prefix, num_layers, heads, return_sequence=False):
    """TransformerEncoder.forward (mmf/modules/encoders.py:582-585) over BertModelJit.forward
    (mmf/modules/hf_layers.py:358-475): embeddings -> encoder -> pooler; pooled output unless return_sequence."""
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids)
    emb = bert_embeddings(input_ids, token_type_ids, sd, prefix + ".embeddings")
    seq = bert_encoder(emb, extended_attention_mask(attention_mask, emb.dtype), sd, prefix + ".encoder", num_layers, heads)
    return seq if return_sequence else bert_pooler(seq, sd, prefix + ".pooler")


def extract_modal_end_token(input_ids, input_mask):
    """MMBTBase.extract_modal_end_token, mmf/models/mmbt.py:349-374.  Returns (end_token, new_ids, new_mask)."""
    gather_index = input_mask.sum(1, keepdim=True) - 1
    end = torch.gather(input_ids, 1, gather_index).squeeze(1).clone()
    new_ids = torch.cat([input_ids[:, 1:], input_ids[:, -1:]], dim=1)
    new_mask = torch.cat([input_mask[:, 1:], torch.zeros_like(input_mask[:, :1])], dim=1)
    return end, new_ids, new_mask


def mmbt_modal_token_type(segment_ids, num_max_segment=2):
    """token_value rule of MMBTBase.forward, mmf/models/mmbt.py:393-414."""
    token_value = 0
    max_id, min_id = int(segment_ids.max()), int(segment_ids.min())
    if max_id == min_id:
        if max_id == 0:
            token_value = 1
    else:
        max_segment = num_max_segment - 1
        if max_id != max_segment:
            token_value = max_segment
    return token_value


def modal_embeddings(input_modal, start_token, end_token, token_type_ids, sd, emb_prefix, proj_prefix, keep=None,
                     p=0.0):
    """ModalEmbeddings.forward, mmf/models/mmbt.py:84-129 (encoder = identity on region features).
    emb_prefix: the text transformer's `embeddings` (word/position/token_type/LayerNorm are shared);
    proj_prefix: `proj_embeddings`.  token_type_ids [B,1] broadcasts over the modal sequence."""
    tok = linear(input_modal, sd, proj_prefix)
    if start_token is not None:
        tok = torch.cat([embedding(sd[emb_prefix + ".word_embeddings.weight"], start_token, 0).unsqueeze(1), tok], dim=1)
    if end_token is not None:
        tok = torch.cat([tok, embedding(sd[emb_prefix + ".word_embeddings.weight"], end_token, 0).unsqueeze(1)], dim=1)
    B, L = tok.shape[:2]
    pos = torch.arange(L, dtype=torch.long, device=tok.device).unsqueeze(0).expand(B, L)
    if token_type_ids is None:
        token_type_ids = torch.zeros((B, L), dtype=torch.long, device=tok.device)
    e = tok + sd[emb_prefix + ".position_embeddings.weight"][pos] + sd[emb_prefix + ".token_type_embeddings.weight"][
        token_type_ids]
    return dropout(layer_norm(e, sd, emb_prefix + ".LayerNorm"), keep, p)


def mmbt_forward(input_modal, input_ids, input_mask, segment_ids, sd, cfg):
    """MMBTBase.forward + MMBTModel.forward, mmf/models/mmbt.py:376-444, 176-318 (eval dropout).
    sd keys: 'modal_encoder.proj_embeddings.*', 'transformer.embeddings.*', 'transformer.encoder.layer.*',
    'transformer.pooler.*'.  Returns (sequence_output, pooled_output, additive_mask)."""
    start = input_ids[:, 0].clone()
    end, ids, mask = extract_modal_end_token(input_ids, input_mask)
    tv = mmbt_modal_token_type(segment_ids, cfg.get("num_segments", 2))
    modal_tt = torch.full((input_modal.shape[0], 1), tv, dtype=torch.long, device=input_modal.device)
    modal = modal_embeddings(input_modal, start, end, modal_tt, sd, "transformer.embeddings",
                             "modal_encoder.proj_embeddings")
    txt = bert_embeddings(ids, segment_ids, sd, "transformer.embeddings")
    emb = torch.cat([modal, txt], 1)
    full_mask = torch.cat([torch.ones(modal.shape[:2], dtype=torch.long, device=mask.device), mask], dim=1)
    add_mask = extended_attention_mask(full_mask, emb.dtype)
    seq = bert_encoder(emb, add_mask, sd, "transformer.encoder", cfg["num_hidden_layers"],
                       cfg["num_attention_heads"])
    return seq, bert_pooler(seq, sd, "transformer.pooler"), add_mask


def hf_multimodal_embeddings(tokens, position_ids, segment_ids, sd, prefix, modalities):
    """HuggingfaceEmbeddings.forward, mmf/models/transformers/backends/huggingface.py:131-159.
    modalities: list of dicts {key, type ('text'|'image'), idx}; text modality i uses an embedding table
    `token_embeddings.i.weight`, others Sequential(Linear, LayerNorm) `token_embeddings.i.0/.1`."""
    outs = []
    for i, m in enumerate(modalities):
        key = m["key"]
        if m["type"] == "text":
            e = embedding(sd["%s.token_embeddings.%d.weight" % (prefix, i)], tokens[key], m.get("pad_token_id", 0))
        else:
            e = linear(tokens[key], sd, "%s.token_embeddings.%d.0" % (prefix, i))
            e = layer_norm(e, sd, "%s.token_embeddings.%d.1" % (prefix, i), m.get("layer_norm_eps", LN_EPS))
        if key in position_ids:
            e = e + sd["%s.pos_embeddings.%d.weight" % (prefix, i)][position_ids[key]]
        if key in segment_ids:
            e = e + sd[prefix + ".token_type_embeddings.weight"][segment_ids[key]]
        outs.append(layer_norm(e, sd, "%s.layer_norms.%d" % (prefix, i), m.get("layer_norm_eps", LN_EPS)))
    return torch.cat(outs, dim=1)


def hf_attention_mask(masks):
    """HuggingfaceBackend.generate_attention_mask, huggingface.py:216-222."""
    m = torch.cat(masks, dim=-1)
    return (1.0 - m.unsqueeze(1).unsqueeze(2)) * -10000.0


# ----------------------------------------------------------------------------------------------
# synthetic inputs / weights (SURVEY.md 8d): identical generators feed oracle, reference and CUDA path
# ----------------------------------------------------------------------------------------------
def init_bert_layer_weights(sd, prefix, hidden, inter, gen, std=0.02, in_hidden=None):
    """normal(0, 0.02) Linear weights, zero biases, LN (1, 0): mmf/models/transformers/base.py:213-223.
    Biases/LN are perturbed slightly so parity tests exercise them."""
    def lin(name, o, i):
        sd[name + ".weight"] = torch.randn(o, i, generator=gen) * std
        sd[name + ".bias"] = torch.randn(o, generator=gen) * std

    def ln(name, n):
        sd[name + ".weight"] = 1.0 + torch.randn(n, generator=gen) * std
        sd[name + ".bias"] = torch.randn(n, generator=gen) * std

    for n in ("query", "key", "value"):
        lin("%s.attention.self.%s" % (prefix, n), hidden, hidden)
    lin(prefix + ".attention.output.dense", hidden, hidden)
    ln(prefix + ".attention.output.LayerNorm", hidden)
    lin(prefix + ".intermediate.dense", inter, hidden)
    lin(prefix + ".output.dense", hidden, inter)
    ln(prefix + ".output.LayerNorm", hidden)
    return sd


def make_encoder_weights(num_layers, hidden, inter, seed=0, prefix="layer"):
    gen = torch.Generator().manual_seed(seed)
    sd = {}
    for i in range(num_layers):
        init_bert_layer_weights(sd, "%s.%d" % (prefix, i), hidden, inter, gen)
    return sd


# ----------------------------------------------------------------------------------------------
# UNITER (BASELINE.json configs[4] class; SURVEY.md 8f item 3)
# ----------------------------------------------------------------------------------------------
def uniter_image_embeddings(img_feat, img_pos_feat, type_embeddings, sd, prefix, img_masks=None, eps=LN_EPS):
    """UNITERImageEmbeddings.forward, mmf/models/uniter.py:69-88 (dropout p = 0)."""
    if img_masks is not None:
        table = sd[prefix + ".mask_embedding.weight"].clone()
        table[0] = 0.0                                   # padding_idx row is forced to zero on every call (:77)
        img_feat = img_feat + table[img_masks.long()]
    im = layer_norm(linear(img_feat, sd, prefix + ".img_linear"), sd, prefix + ".img_layer_norm", eps)
    pos = layer_norm(linear(img_pos_feat, sd, prefix + ".pos_linear"), sd, prefix + ".pos_layer_norm", eps)
    return layer_norm(im + pos + type_embeddings, sd, prefix + ".final_layer_norm", eps)


def uniter_forward(input_ids, position_ids, img_feat, img_pos_feat, attention_mask, sd, num_layers, heads, img_masks=None,
                   txt_type_ids=None, img_type_ids=None, input_modality="image-text"):
    """UNITERModelBase.forward, mmf/models/uniter.py:197-243 -> (final_layer, hidden_layers)"""
    add = extended_attention_mask(attention_mask)
    parts = []
    if input_modality != "image":
        parts.append(bert_embeddings(input_ids, txt_type_ids, sd, "text_embeddings", position_ids))
    if input_modality != "text":
        if img_type_ids is None:
            img_type_ids = torch.ones_like(img_feat[:, :, 0].long())
        tt = sd["text_embeddings.token_type_embeddings.weight"][img_type_ids]
        parts.append(uniter_image_embeddings(img_feat, img_pos_feat, tt, sd, "img_embeddings", img_masks))
    emb = torch.cat(parts, dim=1)
    out, hiddens = bert_encoder(emb, add, sd, "encoder", num_layers, heads, output_hidden_states=True)
    return out, hiddens


# ----------------------------------------------------------------------------------------------
# LXMERT encoder (BASELINE.json configs[4] class; SURVEY.md 8f item 3)
# ----------------------------------------------------------------------------------------------
def visual_feat_encoder(feats, boxes, sd, prefix):
    """VisualFeatEncoder.forward, mmf/models/lxmert.py:211-223 (dropout p = 0)."""
    x = layer_norm(linear(feats, sd, prefix + ".visn_fc"), sd, prefix + ".visn_layer_norm")
    if boxes is None:
        return x
    y = layer_norm(linear(boxes, sd, prefix + ".box_fc"), sd, prefix + ".box_layer_norm")
    return (x + y) / 2


def lxmert_xlayer(lang, lang_mask, visn, visn_mask, sd, prefix, heads, masks=None, p_attn=0.0, p_hidden=0.0):
    """LXMERTXLayer.forward, mmf/models/lxmert.py:244-283: ONE cross-attention block (BertCrossattLayer :68-82) used in
    both directions from the layer inputs, then per-stream self-attention (BertAttention) and FFN.
    masks: optional dict of keep-masks.  'x_attn_lang' [B,h,T,R] / 'x_attn_visn' [B,h,R,T] on the cross-attention
    probabilities and 'x_out_lang' [B,T,H] / 'x_out_visn' [B,R,H] in BertAttOutput, per direction (language queries first);
    'lang' / 'visn': bert_layer's dict ('attn', 'self_out', 'out') for each stream's self-attention and FFN."""
    m = masks or {}
    ca = prefix + ".visual_attention"

    def cross(x, ctx, ctx_mask, name):
        out, _ = bert_self_attention(x, None, sd, ca + ".att", heads, m.get("x_attn_" + name), p_attn, kv=ctx,
                                     kv_mask=ctx_mask)
        return bert_self_output(out, x, sd, ca + ".output", m.get("x_out_" + name), p_hidden)
    la, va = cross(lang, visn, visn_mask, "lang"), cross(visn, lang, lang_mask, "visn")
    outs = []
    for x, mask, name in ((la, lang_mask, "lang"), (va, visn_mask, "visn")):
        sm = m.get(name) or {}
        ctx, _ = bert_self_attention(x, mask, sd, "%s.%s_self_att.self" % (prefix, name), heads, sm.get("attn"), p_attn)
        att = bert_self_output(ctx, x, sd, "%s.%s_self_att.output" % (prefix, name), sm.get("self_out"), p_hidden)
        inter = bert_intermediate(att, sd, "%s.%s_inter" % (prefix, name))
        outs.append(bert_self_output(inter, att, sd, "%s.%s_output" % (prefix, name), sm.get("out"), p_hidden))
    return outs[0], outs[1]


def lxmert_encoder(lang, lang_mask, feats, boxes, visn_mask, sd, prefix, l_layers, x_layers, r_layers, heads, masks=None,
                   p_attn=0.0, p_hidden=0.0):
    """LXMERTEncoder.forward, mmf/models/lxmert.py:309-336; masks are the additive [B,1,1,S] tensors.
    masks (keep-masks): optional dict with per-layer lists 'l' and 'r' (bert_layer's dicts) and 'x' (lxmert_xlayer's).
    The visual feature encoder's own dropout is not modelled (p = 0 there)."""
    pre = prefix + "." if prefix else ""
    km = masks or {}
    visn = visual_feat_encoder(feats, boxes, sd, pre + "visn_fc")
    for i in range(l_layers):
        lang, _ = bert_layer(lang, lang_mask, sd, "%slayer.%d" % (pre, i), heads, km["l"][i] if km else None, p_attn,
                             p_hidden)
    for i in range(r_layers):
        visn, _ = bert_layer(visn, visn_mask, sd, "%sr_layers.%d" % (pre, i), heads, km["r"][i] if km else None, p_attn,
                             p_hidden)
    for i in range(x_layers):
        lang, visn = lxmert_xlayer(lang, lang_mask, visn, visn_mask, sd, "%sx_layers.%d" % (pre, i), heads,
                                   km["x"][i] if km else None, p_attn, p_hidden)
    return lang, visn


# ----------------------------------------------------------------------------------------------
# masked-LM pre-training head (SURVEY.md 8a row a15 / 8f item 1)
# ----------------------------------------------------------------------------------------------
def vinvl_forward(input_ids, img_feats, attention_mask, sd, num_layers, heads, token_type_ids=None, use_img_layernorm=True):
    """VinVLBase.forward, mmf/models/vinvl.py:68-122 (eval): BertEmbeddings(text) ++ img_embedding(regions) -> BertEncoder"""
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    text = bert_embeddings(input_ids, token_type_ids, sd, "embeddings")
    img = linear(img_feats, sd, "img_embedding.0")
    if use_img_layernorm:
        img = layer_norm(img, sd, "img_embedding.1")
    emb = torch.cat((text, img), 1)
    return bert_encoder(emb, extended_attention_mask(attention_mask, emb.dtype), sd, "encoder", num_layers, heads)


def vit_layer(x, add_mask, sd, prefix, heads, masks=None, p_attn=0.0, p_hidden=0.0):
    """ViTLayer.forward, mmf/modules/vit.py:79-108 (pre-LN block).  ViTAttention = BertSelfAttention on
    layernorm_before(x) -> ViTSelfOutput (dense -> dropout, no residual inside, HF modeling_vit); the two residuals are
    added in the layer: h = attn + x (:96), out = ViTOutput(intermediate(layernorm_after(h)), h) = dropout(dense(.)) + h
    (:99-105).  masks: optional dict with keep-masks 'attn' [B,h,S,S], 'self_out' [B,S,H] (ViTSelfOutput) and 'out'
    [B,S,H] (ViTOutput), as bert_layer's."""
    m = masks or {}
    a = layer_norm(x, sd, prefix + ".layernorm_before")
    ctx, _ = bert_self_attention(a, add_mask, sd, prefix + ".attention.attention", heads, m.get("attn"), p_attn)
    h = dropout(linear(ctx, sd, prefix + ".attention.output.dense"), m.get("self_out"), p_hidden) + x
    b = layer_norm(h, sd, prefix + ".layernorm_after")
    y = linear(gelu_erf(linear(b, sd, prefix + ".intermediate.dense")), sd, prefix + ".output.dense")
    return dropout(y, m.get("out"), p_hidden) + h


def vit_encoder(x, add_mask, sd, prefix, num_layers, heads, masks=None, p_attn=0.0, p_hidden=0.0):
    """ViTEncoder.forward, vit.py:118-175.  masks: optional list of vit_layer's dicts, one per layer."""
    pre = prefix + "." if prefix else ""
    for i in range(num_layers):
        x = vit_layer(x, add_mask, sd, "%slayer.%d" % (pre, i), heads, masks[i] if masks else None, p_attn, p_hidden)
    return x


def bert_pretraining_heads(sequence_output, pooled_output, sd, prefix):
    """HF BertPreTrainingHeads (transformers, pinned <= 4.10), the reference's `self.cls`
    (mmf/models/visual_bert.py:205-214): transform = LayerNorm(gelu(dense(h))), decoder = h W^T + bias (W tied to the
    word embeddings), seq_relationship = Linear(pooled).  -> (prediction_scores, seq_relationship_score)"""
    p = prefix + ".predictions"
    h = layer_norm(gelu_erf(linear(sequence_output, sd, p + ".transform.dense")), sd, p + ".transform.LayerNorm")
    scores = h @ sd[p + ".decoder.weight"].t() + sd[p + ".bias"]
    return scores, linear(pooled_output, sd, prefix + ".seq_relationship")


def masked_lm_loss(prediction_scores, labels, ignore_index=-1):
    """CrossEntropyLoss(ignore_index=-1) over all positions, mmf/models/visual_bert.py:215, 269-277"""
    V = prediction_scores.shape[-1]
    return F.cross_entropy(prediction_scores.reshape(-1, V), labels.reshape(-1), ignore_index=ignore_index)


# ----------------------------------------------------------------------------------------------
# optimizer "adam_w" (SURVEY.md 8f item 2)
# ----------------------------------------------------------------------------------------------
def adamw_step_transformers(p, g, m, v, step, lr, beta1, beta2, eps, weight_decay, correct_bias=True):
    """One step of the transformers AdamW arithmetic as it stands in the reference tree
    (mmf/modules/optimizers.py:60-84); `step` is the 1-based step count.  In place on p, m, v."""
    m.mul_(beta1).add_(g, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    denom = v.sqrt().add_(eps)
    step_size = lr
    if correct_bias:
        step_size = step_size * math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)
    p.addcdiv_(m, denom, value=-step_size)
    if weight_decay > 0.0:
        p.add_(p, alpha=-lr * weight_decay)


def adamw_step_torch(p, g, m, v, step, lr, beta1, beta2, eps, weight_decay):
    """torch.optim.AdamW (single-tensor path), what `adam_w` resolves to when transformers ships no AdamW
    (mmf/modules/optimizers.py:8-14).  In place on p, m, v."""
    p.mul_(1.0 - lr * weight_decay)
    m.lerp_(g, 1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-(lr / bc1))
