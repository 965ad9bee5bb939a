"""Differentiable building blocks over the C-ABI kernels, for the front-ends around the encoder trunk
(MMBT modal embeddings, MMFTransformer per-modality embeddings, ViLBERT image embeddings).

Unlike the encoder/VisualBERT-embedding fast path (flat parameter pack, one autograd node per module), these are
ordinary `torch.autograd.Function`s taking the parameters as inputs: the front-ends are a few percent of the block's
FLOPs, so flexibility wins over launch count.  All arithmetic still runs in libmmfb200 kernels; activations bf16.
"""
import torch

from . import functional as F
from . import lib
from .engine import _bnd, best_splits


def _bf16(t):
    return t.detach().to(torch.bfloat16).contiguous()


_EPI = {None: lib.EPI_BIAS, "relu": lib.EPI_BIAS_RELU, "gelu": lib.EPI_BIAS_GELU}


def _linear_grads(need, dz, xb, wb, weight_t=False, count=None, dx=None, dw=None, db=None):
    """The gradients of z = x W^T + b (W [N, K]), or of z = x W + b with W stored [K, N] (weight_t), from dz = dL/dz (bf16),
    for the inputs (x, W, b) that `need` flags: dx = the dgrad GEMM, written into `dx` (allocated by the GEMM when None);
    dW = the split-K weight-gradient GEMM and db = the column sum of dz, accumulated in fp32 into `dw` / `db` (allocated
    zero when None).  With `count` (int32 [1] on the device) every kernel reads only the rows of dz below it.  Returns
    (dx, dw, db), None where not needed."""
    if need[0]:
        dx = F.gemm(dz, wb, b_mn=not weight_t, epi=lib.EPI_BIAS, out=dx, **_bnd("m_bound", count))
    if need[1]:
        if dw is None:
            dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)
        a, b = (xb, dz) if weight_t else (dz, xb)           # weight_t: [K, N] = x^T dz, otherwise [N, K] = dz^T x
        F.gemm(a, b, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=best_splits(*wb.shape, xb.shape[0]),
               **_bnd("k_bound", count))
    if need[2]:
        if db is None:
            db = torch.zeros(dz.shape[1], dtype=torch.float32, device=dz.device)
        if count is None:
            F.colsum(dz, db)
        else:
            F.colsum_bounded(dz, db, count)
    return dx, dw, db


class _Linear(torch.autograd.Function):
    """y = act(x W^T + b) on the wgmma GEMM with the bias (+ ReLU / GELU) epilogue; the GELU epilogue also writes the
    pre-activation u, saved for the backward.  weight_t: W is stored [K, N] and read MN-major (the layout the dgrad calls
    use), so a weight that is another layer's nn.Linear weight - MRFR's projection back to the feature space, tied to
    UNITER's img_linear (heads/mrfr.py:48-49, 86-88) - is consumed as it lies and autograd sums both uses' gradients into
    the one parameter.  count: int32 [1] on the device, the live rows of a fixed capacity whose later rows are zero; the
    GEMM and the dgrad, weight gradient and bias column sum of the backward are bounded by it, so nothing is read on the
    host.  Backward: dy masked by (y > 0) (relu_bwd) or times GELU'(u) (gelu_bwd), then _linear_grads."""

    @staticmethod
    def forward(ctx, x, weight, bias, act, weight_t, count):
        xb, wb = _bf16(x), _bf16(weight)
        bb = _bf16(bias) if bias is not None else None
        y = F.gemm(xb, wb, b_mn=weight_t, epi=_EPI[act], bias=bb, **_bnd("m_bound", count))
        aux = None
        if act == "gelu":
            aux, y = y
        elif act == "relu":
            aux = y
        ctx.save_for_backward(xb, wb, aux, count)
        ctx.act, ctx.weight_t = act, weight_t
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype if bias is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, wb, aux, count = ctx.saved_tensors
        dz = dy.to(torch.bfloat16).contiguous()
        if ctx.act == "relu":
            dz = F.relu_bwd(dz, aux)
        elif ctx.act == "gelu":
            # with a count: u is finite up to the 128-row tile edge, which is as far as the dgrad reads dz (the weight
            # gradient reads it to the 64-row k-block edge); dy is zero at and past the count
            dz = F.gelu_bwd(dz, aux)
        grads = _linear_grads(ctx.needs_input_grad, dz, xb, wb, ctx.weight_t, count)
        return tuple([g if g is None else g.to(t) for g, t in zip(grads, ctx.dtypes)]) + (None, None, None)


def linear(x2d, weight, bias=None):
    """x2d [M, K] (any float dtype) -> bf16 [M, N].  K and N must be multiples of 8 (TMA row pitch)."""
    return _Linear.apply(x2d, weight, bias, None, False, None)


def linear_relu(x2d, weight, bias):
    return _Linear.apply(x2d, weight, bias, "relu", False, None)


def linear_gelu(x2d, weight, bias, count=None):
    """gelu(x2d W^T + b); with `count` (int32 [1] on the device) only the rows below it are computed, later rows are zero"""
    return _Linear.apply(x2d, weight, bias, "gelu", False, count)


def linear_t(x2d, weight_kn, bias):
    """F.linear(x, weight_kn.t(), bias): x2d [M, K], weight_kn [K, N] -> bf16 [M, N]; K and N multiples of 8."""
    return _Linear.apply(x2d, weight_kn, bias, None, True, None)


class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, count):
        xb, g, b = _bf16(x), _bf16(weight), _bf16(bias)
        y, mean, rstd = F.layernorm_fwd(xb, g, b, eps, **_bnd("m_bound", count))
        ctx.save_for_backward(xb, mean, rstd, g, count)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, mean, rstd, g, count = ctx.saved_tensors
        dg = torch.zeros(g.shape, dtype=torch.float32, device=g.device)
        db = torch.zeros_like(dg)
        dx, _ = F.layernorm_bwd(dy.to(torch.bfloat16).contiguous(), xb, mean, rstd, g, dg, db, **_bnd("m_bound", count))
        return dx.to(ctx.dtypes[0]), dg.to(ctx.dtypes[1]), db.to(ctx.dtypes[2]), None, None


def layer_norm(x2d, weight, bias, eps=1e-12, count=None):
    """row LayerNorm; with `count` (int32 [1] on the device) only the rows below it are read and written, later output rows
    and their gradients are zero"""
    return _LayerNorm.apply(x2d, weight, bias, eps, count)


class _ComposeLN(torch.autograd.Function):
    """out = dropout(LN(sum_k src_k[rows_k] + sum_k table_k[idx_k]))  - the embedding composer + LayerNorm.

    inputs: n_src dense sources then n_tab tables then (ln_w, ln_b); index tensors are int32 [M] (negative = absent).
    """

    @staticmethod
    def forward(ctx, meta, *tensors):
        M, H, n_src, n_tab, rows, idxs, eps, bits, scale = meta
        srcs = [_bf16(t) for t in tensors[:n_src]]
        tabs = [_bf16(t) for t in tensors[n_src:n_src + n_tab]]
        g, b = _bf16(tensors[-2]), _bf16(tensors[-1])
        y = F.embed_compose(M, H, srcs=list(zip(srcs, rows)), tabs=list(zip(tabs, idxs[0])), device=g.device)
        x, mean, rstd = F.layernorm_fwd(y, g, b, eps, drop_mask=bits, drop_scale=scale)
        ctx.meta = meta
        ctx.src_shapes = [tuple(t.shape) for t in srcs]
        ctx.tab_shapes = [tuple(t.shape) for t in tabs]
        ctx.dtypes = [t.dtype for t in tensors]
        ctx.save_for_backward(y, mean, rstd, g)
        return x

    @staticmethod
    def backward(ctx, dout):
        M, H, n_src, n_tab, rows, idxs, eps, bits, scale = ctx.meta
        y, mean, rstd, g = ctx.saved_tensors
        d = dout.to(torch.bfloat16).contiguous()
        if bits is not None:   # dropout sits after the LayerNorm
            d = (d * F.unpack_keep_bits(bits, H) * scale).to(torch.bfloat16)
        dg = torch.zeros(H, dtype=torch.float32, device=g.device)
        db = torch.zeros_like(dg)
        dy, _ = F.layernorm_bwd(d, y, mean, rstd, g, dg, db)
        dsrcs = [torch.zeros(s, dtype=torch.bfloat16, device=g.device) for s in ctx.src_shapes]
        dtabs = [torch.zeros(s, dtype=torch.float32, device=g.device) for s in ctx.tab_shapes]
        if dsrcs:
            F.embed_scatter(dy, dsrcs=list(zip(dsrcs, rows)))
        for t, ix in zip(dtabs, idxs[1]):
            F.embed_scatter_sorted(dy, t, *F.sort_indices(ix))   # idxs already carry -1 at padding_idx rows
        grads = [t.to(dt) for t, dt in zip(dsrcs + dtabs + [dg, db], ctx.dtypes)]
        return (None,) + tuple(grads)


def compose_ln(M, H, srcs, tabs, ln_weight, ln_bias, eps=1e-12, p=0.0, training=False, dropout_state=None):
    """srcs: up to 2 (tensor [*, H], int32 rows [M]); tabs: up to 3 (table [V, H], int32 idx [M][, padding_idx]).
    The same table may appear in several slots.  Returns bf16 [M, H]."""
    if len(srcs) > 2 or len(tabs) > 3:
        raise ValueError("compose_ln: at most 2 dense sources and 3 table slots")
    bits, scale = None, 1.0
    if training and p > 0.0:
        from .modules import _fresh_dropout_state
        ds = dropout_state or _fresh_dropout_state()
        bits, scale = ds.bits((M,), H, p, ln_weight.device), 1.0 / (1.0 - p)
    # a table slot may be (table, idx, padding_idx): the row is read in the forward but, like nn.Embedding(padding_idx=),
    # receives no gradient - the backward index gets -1 (= absent) there
    fwd_idx = [t[1] for t in tabs]
    bwd_idx = [t[1] if len(t) < 3 or t[2] is None else torch.where(t[1] == t[2], torch.full_like(t[1], -1), t[1])
               for t in tabs]
    meta = (M, H, len(srcs), len(tabs), [r for _, r in srcs], (fwd_idx, bwd_idx), float(eps), bits, scale)
    return _ComposeLN.apply(meta, *[t for t, _ in srcs], *[t[0] for t in tabs], ln_weight, ln_bias)


def i32(t):
    return t.reshape(-1).to(torch.int32).contiguous()


def linear_any(x2d, weight, bias=None):
    """`linear` for arbitrary out/in feature counts: the GEMM wants N and K in multiples of 8 (16-byte TMA row pitch), so a
    classifier with 2 labels or a 5-column location input gets zero-padded operands and a sliced result; autograd's
    pad / slice backward routes the gradients.  No-op wrapper when the sizes already fit."""
    N, K = weight.shape
    pn, pk = (-N) % 8, (-K) % 8
    if pk:
        x2d = torch.nn.functional.pad(x2d, (0, pk))
        weight = torch.nn.functional.pad(weight, (0, pk))
    if pn:
        weight = torch.nn.functional.pad(weight, (0, 0, 0, pn))
        if bias is not None:
            bias = torch.nn.functional.pad(bias, (0, pn))
    y = linear(x2d, weight, bias)
    return y[:, :N] if pn else y


class _LinearLoss(torch.autograd.Function):
    """A loss of the projection z = h W^T + b (W [N, K]), or z = h W + b with W stored [K, N] (weight_t, read MN-major),
    WITHOUT the [rows, N] tensor z: the rows are processed in chunks - GEMM -> row-loss kernel (loss + d(z) in place) ->
    dgrad, split-K weight gradient and bias column sum of the chunk (_linear_grads) - so at most `chunk_rows` x N values of
    z exist at a time (sized to stay L2-resident between the kernels that touch them).  Gradients are therefore computed
    in the FORWARD, already scaled; the backward multiplies them by the incoming scalar.  N need not be a multiple of 8:
    the weight and bias are padded, and the row kernels give the padding columns a zero gradient.

    kind "ce": mean cross-entropy against integer `target` labels (mmfb_ce_rows), rows labelled ignore_index excluded.
    Reference: prediction scores + CrossEntropyLoss(ignore_index) of mmf/models/visual_bert.py:269-277 and
    mmf/models/transformers/heads/mlm.py:83-88.  kind "kl" / "mse": the region heads' KL divergence from / squared error
    against the fp32 rows target[tgt_idx[r]] (mmfb_kl_rows_bounded, mmfb_mse_rows_bounded).

    count None (cross-entropy only): the scale 1 / n_active is read on the host, the loss goes to one fp32 sum.
    count (int32 [1] on the device): static-rows mode, the rows are a fixed capacity of which the first `count` are live
    and the rest hold zero features (and ignore_index labels), as a CUDA graph can capture it (mmf_b200.graphs).  Every
    kernel of a chunk takes the chunk's share of `count` as a device bound, so a chunk that starts past `count` costs
    launches whose CTAs exit at once, and inside a chunk only the rows below `count` rounded up to a 128-row tile are
    computed; chunk_rows None runs one chunk bounded by `count` itself.  The loss is scaled by `scale` (fp32 [1] on the
    device): no host read.  The row losses are summed over the whole capacity in one fixed-order sum, for the
    cross-entropy only in deterministic mode."""

    @staticmethod
    def forward(ctx, h, weight, bias, target, tgt_idx, count, scale, kind, ignore_index, weight_t, chunk_rows):
        hb, wb = _bf16(h), _bf16(weight)
        M, N = hb.shape[0], wb.shape[1 if weight_t else 0]
        pad = (-N) % 8
        if pad:                     # zero weight rows; for the softmax of the cross-entropy a -inf-like bias as well, so
            wb = torch.nn.functional.pad(wb, (0, 0, 0, pad))                 # that the padded logits vanish
        bb = _bf16(bias) if bias is not None else torch.zeros(N, dtype=torch.bfloat16, device=wb.device)
        if pad:
            fill = -30000.0 if kind == "ce" else 0.0
            bb = torch.cat([bb, torch.full((pad,), fill, dtype=torch.bfloat16, device=bb.device)])
        if count is None:
            scale = 1.0 / float(max(int((target != ignore_index).sum()), 1))    # the one host read (the mean reduction)
        need = need_h, need_w, need_b = ctx.needs_input_grad[:3]
        # in static-rows mode rows past count are never written by the bounded kernels: their gradients stay zero
        dh = (torch.empty_like if count is None else torch.zeros_like)(hb) if need_h else None
        dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device) if need_w else None
        db = torch.zeros(N + pad, dtype=torch.float32, device=wb.device) if need_b else None
        ordered = kind != "ce" or (count is not None and torch.are_deterministic_algorithms_enabled())
        loss_sum = torch.zeros((), dtype=torch.float32, device=wb.device)
        row_loss = torch.zeros(M, dtype=torch.float32, device=wb.device) if ordered else None
        if chunk_rows is None:
            chunk_rows, bounds = M, count
        elif count is not None:     # the live rows of chunk i: clamp(count - i * chunk_rows, 0, chunk_rows), one int32 each
            starts = torch.arange(0, M, chunk_rows, dtype=torch.int32, device=wb.device)
            bounds = (count.reshape(1) - starts).clamp_(0, chunk_rows)
        for i, r0 in enumerate(range(0, M, chunk_rows)):
            r1 = min(M, r0 + chunk_rows)
            nb = None if count is None else bounds[i:i + 1]
            z = F.gemm(hb[r0:r1], wb, b_mn=weight_t, epi=lib.EPI_BIAS, bias=bb, **_bnd("m_bound", nb))
            if kind == "kl":
                F.kl_rows_bounded(z, N, target, tgt_idx[r0:r1], nb, scale, row_loss[r0:r1])
            elif kind == "mse":
                F.mse_rows_bounded(z, target, tgt_idx[r0:r1], nb, scale, row_loss[r0:r1])
            elif count is None:
                F.ce_rows(z, target[r0:r1], ignore_index, scale, loss_sum)
            else:
                F.ce_rows_bounded(z, target[r0:r1], ignore_index, scale, nb, loss_sum=loss_sum,
                                  row_loss=row_loss[r0:r1] if ordered else None)
            _linear_grads(need, z, hb[r0:r1], wb, weight_t, nb, dh[r0:r1] if need_h else None, dw, db)
        if ordered:
            loss_sum = row_loss.sum()
        ctx.save_for_backward(dh, dw if dw is None or weight_t else dw[:N], db if db is None else db[:N])
        ctx.dtypes = (h.dtype, weight.dtype, bias.dtype if bias is not None else None)
        return loss_sum * (scale if count is None else scale.reshape(()))

    @staticmethod
    def backward(ctx, g):
        grads = [t if t is None else (t.float() * g).to(dt) for t, dt in zip(ctx.saved_tensors, ctx.dtypes)]
        return tuple(grads) + (None,) * 8


def linear_cross_entropy(h2d, weight, bias, labels, ignore_index=-1, chunk_rows=2048, count=None, scale=None):
    """mean_i CE((h W^T + b)_i, labels_i) over the rows with labels_i != ignore_index (0 when there is none), fp32 scalar.
    Static-rows mode: `count` (int32 [1] on the device) is the number of labelled rows, which come first, and `scale`
    (fp32 [1] on the device) = 1 / max(count, 1); later rows must hold ignore_index labels."""
    if (count is None) != (scale is None):
        raise ValueError("linear_cross_entropy: count and scale go together")
    labels = labels.reshape(-1).to(torch.int64).contiguous()
    return _LinearLoss.apply(h2d, weight, bias, labels, None, count, scale, "ce", int(ignore_index), False,
                             int(chunk_rows))


class _GatherRows(torch.autograd.Function):
    """rows [M, H] = x[sel.pos] with zero rows past sel.count (mmfb_gather_rows by pos); backward: the same kernel by
    sel.inv writes the whole input gradient, the gathered gradient at the selected rows and zero elsewhere"""

    @staticmethod
    def forward(ctx, x, sel):
        ctx.sel, ctx.dtype = sel, x.dtype
        return F.gather_rows(_bf16(x), sel.pos)

    @staticmethod
    def backward(ctx, g):
        return F.gather_rows(g.to(torch.bfloat16).contiguous(), ctx.sel.inv).to(ctx.dtype), None


def gather_rows(x2d, sel):
    """the rows of x2d [M, H] that F.select_rows selected, as a fixed-capacity [M, H] bf16 tensor (zeros past count)"""
    return _GatherRows.apply(x2d, sel)


def region_loss_static(h2d, weight, bias, target, tgt_idx, count, scale, kind, weight_t=False):
    """kind "kl": scale * sum_r KL(target[tgt_idx[r]] || softmax(h_r W^T + b)); kind "mse": scale * sum_r
    ||h_r W + b - target[tgt_idx[r]]||^2 (weight_t=True, weight [K, N]) - over the rows r below `count` (int32 [1] on the
    device) of a fixed capacity whose later rows are zero, in one chunk (_LinearLoss).  target: fp32 [*, N]; tgt_idx:
    int32, one per row."""
    if kind not in ("kl", "mse"):
        raise ValueError("region_loss_static: kind must be 'kl' or 'mse', got %r" % (kind,))
    if weight_t and weight.shape[1] % 8:
        raise ValueError("region loss: a transposed weight needs N %% 8 == 0, got %d" % weight.shape[1])
    return _LinearLoss.apply(h2d, weight, bias, target, tgt_idx, count, scale, kind, None, bool(weight_t), None)


class _OptimalTransport(torch.autograd.Function):
    """dist [B] of mmfb_ot_fwd over two row ranges of one sequence buffer; the backward (mmfb_ot_bwd) writes both ranges of
    the sequence gradient in place.  The plan is a constant of the backward, as in the reference (ot.py:98-101)."""

    @staticmethod
    def forward(ctx, seq, T_len, R_len, x_len, y_len, beta, iteration, k):
        sb = seq.detach()
        if sb.dtype != torch.bfloat16 or sb.stride(-1) != 1 or sb.stride(0) % 8 or sb.stride(1) % 8:
            sb = sb.to(torch.bfloat16).contiguous()
        x, y = sb[:, :T_len], sb[:, T_len:T_len + R_len]
        dist, plan, saved = F.ot_fwd(x, y, x_len, y_len, beta, iteration, k)
        ctx.save_for_backward(sb, plan, saved)
        ctx.meta = (T_len, R_len, x_len, y_len, seq.dtype)
        return dist

    @staticmethod
    def backward(ctx, g):
        sb, plan, saved = ctx.saved_tensors
        T_len, R_len, x_len, y_len, dtype = ctx.meta
        full = T_len + R_len == sb.shape[1]
        dseq = (torch.empty if full else torch.zeros)(sb.shape, dtype=torch.bfloat16, device=sb.device)
        F.ot_bwd(g.float().contiguous(), plan, saved, sb[:, :T_len], sb[:, T_len:T_len + R_len], x_len, y_len,
                 dseq[:, :T_len], dseq[:, T_len:T_len + R_len])
        return (dseq.to(dtype),) + (None,) * 7


def optimal_transport_dist(seq, T_len, R_len, x_len, y_len, beta=0.5, iteration=50, k=1):
    """optimal_transport_dist(seq[:, :T_len].float(), seq[:, T_len:T_len + R_len].float(), txt_pad, img_pad) of
    mmf/modules/ot.py:80-102 for prefix pads: sample b's valid text rows are its first x_len[b], its valid regions the first
    y_len[b] (host integers).  seq [B, S >= T_len + R_len, H]; returns fp32 [B].  T_len, R_len <= 128, H % 64 == 0."""
    x_len = torch.as_tensor(x_len).reshape(-1).to(device="cpu", dtype=torch.int32)
    y_len = torch.as_tensor(y_len).reshape(-1).to(device="cpu", dtype=torch.int32)
    return _OptimalTransport.apply(seq, int(T_len), int(R_len), x_len, y_len, float(beta), int(iteration), int(k))
