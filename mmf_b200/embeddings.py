"""Embedding front-ends of the fusion block on the B200 engine (kernel group K1).

  B200VisioLinguisticEmbeddings  <->  BertVisioLinguisticEmbeddings   mmf/modules/embeddings.py:309-459
  B200ImageFeatureEmbeddings     <->  BertImageFeatureEmbeddings      mmf/models/vilbert.py:891-913

Data flow (all on device): region features -> wgmma projection GEMM (bias epilogue) -> one row-composer
kernel that gathers word / position / type rows (or the projected region row + visual type / position rows),
sums them in fp32 and writes the pre-LN row -> LayerNorm (+dropout) kernel.  All embedding tables of a module
are adjacent in its flat parameter pack and are addressed as ONE table with row offsets, so the composer and
its scatter backward take three (table, index) slots whatever the number of logical tables.
Integer work (index construction) is exact torch integer arithmetic on the device.
"""
import torch
from torch import nn

from . import engine as E
from . import functional as F
from . import lib
from .modules import _fresh_dropout_state, _init_bert_weights, _require_cuda


class _EmbedRunner:
    def __init__(self, tables, others):
        self.tables, self.others = list(tables), list(others)
        self.pack = None
        self.grad_ready_hook = None
        self.step_offsets = [0]   # one step: one gradient bucket
        self.eps = F.LN_EPS       # set by the owning module from its LayerNorm holder

    def ensure(self, device):
        if self.pack is not None and self.pack.intact() and self.pack.device == device:
            return
        params = self.tables + self.others
        for p in params:
            _require_cuda(p, "embedding parameter")
        H = self.tables[0].shape[1]
        if any(t.shape[1] != H for t in self.tables) or H % 8:
            raise ValueError("embedding tables must share a hidden size that is a multiple of 8")
        self.pack = E.ParamPack(params, device)
        self.H = H
        self.row_offset, r = [], 0
        for t in self.tables:
            self.row_offset.append(r)
            r += t.shape[0]
        self.total_rows = r
        # one [total_rows, H] view over all tables (they are adjacent, each a multiple of 8 elements)
        o0 = self.pack.offsets[0]
        self.big_w = self.pack.compute[o0:o0 + r * H].view(r, H)
        self.big_g = self.pack.grad[o0:o0 + r * H].view(r, H)
        self.h = [self.pack.handle(p) for p in self.others]


class _VLEmbedFn(torch.autograd.Function):
    """inputs: int32 index tensors (precomputed), region features [B*R, F] bf16; params via *params"""

    @staticmethod
    def forward(ctx, runner, idx, dims, p_drop, training, out_dtype, feats, *params):
        B, T, R, H = dims
        pk = runner.pack
        pk.refresh()
        proj_w, proj_b, ln_g, ln_b = runner.h
        M = B * (T + R)
        srcs = ()
        fb = None
        if R > 0:
            fb = feats.detach().to(torch.bfloat16).contiguous().view(B * R, -1)
            proj = F.gemm(fb, proj_w.w, epi=lib.EPI_BIAS, bias=proj_b.w)
            srcs = ((proj, idx["src_row"]),)
        tabs = ((runner.big_w, idx["i0"]), (runner.big_w, idx["i1"]), (runner.big_w, idx["i2"]))
        y = F.embed_compose(M, H, srcs=srcs, tabs=tabs, device=pk.device)
        bits, scale = (None, 1.0)
        if training and p_drop > 0.0:
            bits, scale = _fresh_dropout_state().bits((M,), H, p_drop, pk.device), 1.0 / (1.0 - p_drop)
        x, mean, rstd = F.layernorm_fwd(y, ln_g.w, ln_b.w, runner.eps, drop_mask=bits, drop_scale=scale)
        ctx.runner, ctx.idx, ctx.dims = runner, idx, dims
        ctx.saved = (fb, y, mean, rstd, bits, scale)
        ctx.feats_dtype = feats.dtype if feats is not None else None
        ctx.feats_shape = tuple(feats.shape) if feats is not None else None
        return x.view(B, T + R, H).to(out_dtype)

    @staticmethod
    def backward(ctx, dout):
        runner, idx = ctx.runner, ctx.idx
        B, T, R, H = ctx.dims
        pk = runner.pack
        fb, y, mean, rstd, bits, scale = ctx.saved
        proj_w, proj_b, ln_g, ln_b = runner.h
        aliased = pk.prepare_grads()
        M = B * (T + R)
        d = dout.to(torch.bfloat16).contiguous().view(M, H)
        if bits is not None:
            # dropout sits AFTER the LayerNorm here (embeddings.py:457-458): undo it on the incoming gradient
            keep = F.unpack_keep_bits(bits, H)
            d = (d * keep * scale).to(torch.bfloat16)
        dy, _ = F.layernorm_bwd(d, y, mean, rstd, ln_g.w, ln_g.g, ln_b.g)
        dsrcs = ()
        dproj = None
        if R > 0:
            dproj = torch.empty(B * R, H, dtype=torch.bfloat16, device=pk.device)
            dsrcs = ((dproj, idx["src_row"]),)
        if dsrcs:
            F.embed_scatter(dy, dsrcs=dsrcs)
        for k in ("i0", "i1", "i2"):
            if k + "_sorted" not in idx:      # indices are known in the forward; sorted lazily once per batch
                idx[k + "_sorted"] = F.sort_indices(idx.get(k + "_bwd", idx[k]))
            F.embed_scatter_sorted(dy, runner.big_g, *idx[k + "_sorted"])
        dfeats = None
        if R > 0:
            F.colsum(dproj, proj_b.g)
            F.gemm(dproj, fb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=proj_w.g,
                   splits=E.best_splits(proj_w.w.shape[0], proj_w.w.shape[1], B * R))
            if ctx.needs_input_grad[6]:
                dfeats = F.gemm(dproj, proj_w.w, b_mn=True, epi=lib.EPI_BIAS).view(ctx.feats_shape).to(ctx.feats_dtype)
        ctx.saved = None
        if runner.grad_ready_hook is not None:
            runner.grad_ready_hook(0)
        return (None, None, None, None, None, None, dfeats) + tuple(pk.autograd_grads(aliased))


class B200VisioLinguisticEmbeddings(nn.Module):
    """BertVisioLinguisticEmbeddings (embeddings.py:309-459): same parameter names / shapes / forward signature."""

    def __init__(self, config):
        super().__init__()
        H = config.hidden_size
        # HF BertEmbeddings: padding_idx = pad_token_id, i.e. the [PAD] row gets no gradient
        self.word_embeddings = nn.Embedding(config.vocab_size, H, padding_idx=getattr(config, "pad_token_id", 0))
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, H)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, H)
        self.token_type_embeddings_visual = nn.Embedding(config.type_vocab_size, H)
        self.position_embeddings_visual = nn.Embedding(config.max_position_embeddings, H)
        self.LayerNorm = nn.LayerNorm(H, eps=float(getattr(config, "layer_norm_eps", 1e-12)))
        self.dropout = nn.Dropout(float(config.hidden_dropout_prob))
        self.projection = nn.Linear(config.visual_embedding_dim, H)
        _init_bert_weights(self, float(getattr(config, "initializer_range", 0.02)))
        self.output_dtype = None
        self._runner = _EmbedRunner(
            [self.word_embeddings.weight, self.position_embeddings.weight, self.token_type_embeddings.weight,
             self.token_type_embeddings_visual.weight, self.position_embeddings_visual.weight],
            [self.projection.weight, self.projection.bias, self.LayerNorm.weight, self.LayerNorm.bias])
        self._runner.eps = float(self.LayerNorm.eps)

    def initialize_visual_from_pretrained(self):
        """embeddings.py:320-327"""
        with torch.no_grad():
            self.token_type_embeddings_visual.weight.copy_(self.token_type_embeddings.weight)
            self.position_embeddings_visual.weight.copy_(self.position_embeddings.weight)

    def build_indices(self, input_ids, token_type_ids, visual_embeddings_type):
        """int32 row-composer indices; text rows (b, s<T): word[ids] + pos[s] + type[seg];
        image rows: projection row + type_visual[vtype] + pos_visual[0]  (embeddings.py:329-370, 412-420)."""
        r = self._runner
        B, T = input_ids.shape
        R = 0 if visual_embeddings_type is None else visual_embeddings_type.shape[1]
        dev = input_ids.device
        o_word, o_pos, o_type, o_tvis, o_pvis = r.row_offset
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        pos = torch.arange(T, device=dev).unsqueeze(0).expand(B, T)
        neg = torch.full((B, R), -1, dtype=torch.long, device=dev)
        i0 = torch.cat([input_ids + o_word] + ([visual_embeddings_type + o_tvis] if R else []), dim=1)
        i1 = torch.cat([pos + o_pos] + ([torch.full((B, R), o_pvis, dtype=torch.long, device=dev)] if R else []), dim=1)
        i2 = torch.cat([token_type_ids + o_type] + ([neg] if R else []), dim=1)
        src = torch.cat([torch.full((B, T), -1, dtype=torch.long, device=dev)] +
                        ([torch.arange(B * R, device=dev).view(B, R)] if R else []), dim=1)
        to32 = lambda t: t.reshape(-1).to(torch.int32).contiguous()
        out = {"i0": to32(i0), "i1": to32(i1), "i2": to32(i2), "src_row": to32(src)}
        pad = self.word_embeddings.padding_idx
        if pad is not None:   # nn.Embedding(padding_idx=): the row is read but gets no gradient
            ids_b = torch.where(input_ids == pad, torch.full_like(input_ids, -1), input_ids + o_word)
            out["i0_bwd"] = to32(torch.cat([ids_b] + ([visual_embeddings_type + o_tvis] if R else []), dim=1))
        return out

    def forward(self, input_ids, token_type_ids=None, visual_embeddings=None, visual_embeddings_type=None,
                image_text_alignment=None):
        _require_cuda(input_ids, "input_ids")
        if image_text_alignment is not None and visual_embeddings is not None and visual_embeddings_type is not None:
            return self._forward_with_alignment(input_ids, token_type_ids, visual_embeddings, visual_embeddings_type,
                                                image_text_alignment)
        self._runner.ensure(input_ids.device)
        B, T = input_ids.shape
        use_img = visual_embeddings is not None and visual_embeddings_type is not None
        R = visual_embeddings.shape[1] if use_img else 0
        idx = self.build_indices(input_ids, token_type_ids, visual_embeddings_type if use_img else None)
        feats = visual_embeddings if use_img else torch.zeros(0, device=input_ids.device)
        # output dtype: the parameters' dtype like the reference; a trunk that feeds the B200 encoder directly sets
        # `output_dtype = torch.bfloat16` to skip a bf16 -> fp32 -> bf16 round trip through HBM
        out_dtype = self.output_dtype or self.word_embeddings.weight.dtype
        return _VLEmbedFn.apply(self._runner, idx, (B, T, R, self._runner.H), float(self.dropout.p), self.training,
                                out_dtype, feats, *self._runner.pack.params)

    def _forward_with_alignment(self, input_ids, token_type_ids, visual_embeddings, visual_embeddings_type,
                                image_text_alignment):
        """get_position_embeddings_visual with image_text_alignment (embeddings.py:375-410): each region's position
        embedding is the mean of the position embeddings of the words it is aligned to (-1 = padding) plus
        position_embeddings_visual[0].  LayerNorm is per row, so text rows and image rows are composed by two
        composer + LN launches sharing the LayerNorm parameters; the alignment gather/mean itself is integer indexing
        plus a tiny torch reduction whose gradient flows into position_embeddings.weight through autograd."""
        from . import ops
        B, T = input_ids.shape
        R = visual_embeddings.shape[1]
        H = self.LayerNorm.weight.shape[0]
        dev = input_ids.device
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        pos = torch.arange(T, device=dev).unsqueeze(0).expand(B, T)
        p_drop = float(self.dropout.p)
        text = ops.compose_ln(B * T, H, [], [(self.word_embeddings.weight, ops.i32(input_ids), self.word_embeddings.padding_idx),
                                             (self.position_embeddings.weight, ops.i32(pos)),
                                             (self.token_type_embeddings.weight, ops.i32(token_type_ids))],
                              self.LayerNorm.weight, self.LayerNorm.bias, self.LayerNorm.eps, p_drop, self.training)
        am = (image_text_alignment != -1).long()
        ali = am * image_text_alignment
        pv = (self.position_embeddings.weight[ali] * am.unsqueeze(-1)).sum(2)
        cnt = am.sum(2)
        cnt = torch.where(cnt == 0, torch.ones_like(cnt), cnt)
        pv = (pv / cnt.unsqueeze(-1)).reshape(B * R, H)
        proj = ops.linear(visual_embeddings.reshape(B * R, -1), self.projection.weight, self.projection.bias)
        rows = torch.arange(B * R, device=dev, dtype=torch.int32)
        zeros = torch.zeros(B * R, device=dev, dtype=torch.int32)
        img = ops.compose_ln(B * R, H, [(proj, rows), (pv, rows)],
                             [(self.token_type_embeddings_visual.weight, ops.i32(visual_embeddings_type)),
                              (self.position_embeddings_visual.weight, zeros)],
                             self.LayerNorm.weight, self.LayerNorm.bias, self.LayerNorm.eps, p_drop, self.training)
        out = torch.cat([text.view(B, T, H), img.view(B, R, H)], dim=1)
        return out.to(self.output_dtype or self.word_embeddings.weight.dtype)
