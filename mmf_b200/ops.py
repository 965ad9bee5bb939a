"""Differentiable building blocks over the C-ABI kernels, for the front-ends around the encoder trunk
(MMBT modal embeddings, MMFTransformer per-modality embeddings, ViLBERT image embeddings).

Unlike the encoder/VisualBERT-embedding fast path (flat parameter pack, one autograd node per module), these are
ordinary `torch.autograd.Function`s taking the parameters as inputs: the front-ends are a few percent of the block's
FLOPs, so flexibility wins over launch count.  All arithmetic still runs in libmmfb200 kernels; activations bf16.
"""
import torch

from . import functional as F
from . import lib
from .engine import best_splits


def _bf16(t):
    return t.detach().to(torch.bfloat16).contiguous()


class _Linear(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM; backward: dgrad (MN-major W), split-K wgrad, column-sum bias gradient."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        xb, wb = _bf16(x), _bf16(weight)
        bb = _bf16(bias) if bias is not None else None
        y = F.gemm(xb, wb, epi=lib.EPI_BIAS, bias=bb)
        ctx.save_for_backward(xb, wb)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype if bias is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, wb = ctx.saved_tensors
        dyb = dy.to(torch.bfloat16).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = F.gemm(dyb, wb, b_mn=True, epi=lib.EPI_BIAS).to(ctx.dtypes[0])
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)
            F.gemm(dyb, xb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                   splits=best_splits(wb.shape[0], wb.shape[1], xb.shape[0]))
            dw = dw.to(ctx.dtypes[1])
        if ctx.dtypes[2] is not None and ctx.needs_input_grad[2]:
            db = torch.zeros(wb.shape[0], dtype=torch.float32, device=wb.device)
            F.colsum(dyb, db)
            db = db.to(ctx.dtypes[2])
        return dx, dw, db


def linear(x2d, weight, bias=None):
    """x2d [M, K] (any float dtype) -> bf16 [M, N].  K and N must be multiples of 8 (TMA row pitch)."""
    return _Linear.apply(x2d, weight, bias)


class _LinearReLU(torch.autograd.Function):
    """y = relu(x W^T + b): GEMM with the ReLU epilogue; backward masks dy with (y > 0) and reuses the Linear backward."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        xb, wb, bb = _bf16(x), _bf16(weight), _bf16(bias)
        y = F.gemm(xb, wb, epi=lib.EPI_BIAS_RELU, bias=bb)
        ctx.save_for_backward(xb, wb, y)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, wb, y = ctx.saved_tensors
        dz = F.relu_bwd(dy.to(torch.bfloat16).contiguous(), y)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = F.gemm(dz, wb, b_mn=True, epi=lib.EPI_BIAS).to(ctx.dtypes[0])
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)
            F.gemm(dz, xb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                   splits=best_splits(wb.shape[0], wb.shape[1], xb.shape[0]))
            dw = dw.to(ctx.dtypes[1])
        if ctx.needs_input_grad[2]:
            db = torch.zeros(wb.shape[0], dtype=torch.float32, device=wb.device)
            F.colsum(dz, db)
            db = db.to(ctx.dtypes[2])
        return dx, dw, db


def linear_relu(x2d, weight, bias):
    return _LinearReLU.apply(x2d, weight, bias)


class _LinearGELU(torch.autograd.Function):
    """h = gelu(x W^T + b): GEMM with the bias + GELU epilogue (it also writes the pre-activation u, saved for the
    backward); backward: du = dh * GELU'(u) (row kernel), then the Linear backward."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        xb, wb, bb = _bf16(x), _bf16(weight), _bf16(bias)
        u, h = F.gemm(xb, wb, epi=lib.EPI_BIAS_GELU, bias=bb)
        ctx.save_for_backward(xb, wb, u)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype)
        return h

    @staticmethod
    def backward(ctx, dh):
        xb, wb, u = ctx.saved_tensors
        du = F.gelu_bwd(dh.to(torch.bfloat16).contiguous(), u)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = F.gemm(du, wb, b_mn=True, epi=lib.EPI_BIAS).to(ctx.dtypes[0])
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)
            F.gemm(du, xb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                   splits=best_splits(wb.shape[0], wb.shape[1], xb.shape[0]))
            dw = dw.to(ctx.dtypes[1])
        if ctx.needs_input_grad[2]:
            db = torch.zeros(wb.shape[0], dtype=torch.float32, device=wb.device)
            F.colsum(du, db)
            db = db.to(ctx.dtypes[2])
        return dx, dw, db


def linear_gelu(x2d, weight, bias):
    return _LinearGELU.apply(x2d, weight, bias)


class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        xb, g, b = _bf16(x), _bf16(weight), _bf16(bias)
        y, mean, rstd = F.layernorm_fwd(xb, g, b, eps)
        ctx.save_for_backward(xb, mean, rstd, g)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, mean, rstd, g = ctx.saved_tensors
        dg = torch.zeros(g.shape, dtype=torch.float32, device=g.device)
        db = torch.zeros_like(dg)
        dx, _ = F.layernorm_bwd(dy.to(torch.bfloat16).contiguous(), xb, mean, rstd, g, dg, db)
        return dx.to(ctx.dtypes[0]), dg.to(ctx.dtypes[1]), db.to(ctx.dtypes[2]), None


def layer_norm(x2d, weight, bias, eps=1e-12):
    return _LayerNorm.apply(x2d, weight, bias, eps)


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


class _LinearCrossEntropy(torch.autograd.Function):
    """mean cross-entropy of (h W^T + b) against integer labels WITHOUT the [rows, V] logits tensor: the rows are processed
    in chunks - vocabulary GEMM -> mmfb_ce_rows (loss + d(logits) in place) -> dgrad and split-K wgrad of the chunk - so at
    most `chunk_rows` x V logits exist at a time (sized to stay L2-resident between the three kernels that touch them).
    Gradients are therefore computed in the FORWARD (scaled by 1 / n_active); the backward multiplies them by the incoming
    scalar.  Reference: prediction scores + CrossEntropyLoss(ignore_index) of mmf/models/visual_bert.py:269-277 and
    mmf/models/transformers/heads/mlm.py:83-88."""

    @staticmethod
    def forward(ctx, h, weight, bias, labels, ignore_index, chunk_rows):
        hb, wb = _bf16(h), _bf16(weight)
        V, K = wb.shape
        pad = (-V) % 8
        if pad:                                # V = 30522 is not a multiple of 8: zero rows, and a -inf-like bias so that
            wb = torch.nn.functional.pad(wb, (0, 0, 0, pad))      # the padded logits vanish from the softmax
        bb = _bf16(bias) if bias is not None else torch.zeros(V, dtype=torch.bfloat16, device=wb.device)
        if pad:
            bb = torch.cat([bb, torch.full((pad,), -30000.0, dtype=torch.bfloat16, device=bb.device)])
        M = hb.shape[0]
        labels = labels.reshape(-1).to(torch.int64).contiguous()
        n_active = (labels != ignore_index).sum()
        scale = 1.0 / float(max(int(n_active), 1))      # the one host read of the head (the reference's mean reduction)
        loss_sum = torch.zeros((), dtype=torch.float32, device=wb.device)
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_b = bias is not None and ctx.needs_input_grad[2]
        dh = torch.empty_like(hb) if need_h else None
        dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device) if need_w else None
        db = torch.zeros(wb.shape[0], dtype=torch.float32, device=wb.device) if need_b else None
        for r0 in range(0, M, chunk_rows):
            r1 = min(M, r0 + chunk_rows)
            z = F.gemm(hb[r0:r1], wb, epi=lib.EPI_BIAS, bias=bb)
            F.ce_rows(z, labels[r0:r1], ignore_index, scale, loss_sum)      # z now holds d(logits)
            if need_h:
                F.gemm(z, wb, b_mn=True, epi=lib.EPI_BIAS, out=dh[r0:r1])
            if need_w:
                F.gemm(z, hb[r0:r1], a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                       splits=best_splits(wb.shape[0], K, r1 - r0))
            if need_b:
                F.colsum(z, db)
        ctx.save_for_backward(*[t for t in (dh, dw, db) if t is not None])
        ctx.have = (need_h, need_w, need_b)
        ctx.V = V
        ctx.dtypes = (h.dtype, weight.dtype, bias.dtype if bias is not None else None)
        return loss_sum * scale

    @staticmethod
    def backward(ctx, g):
        saved = list(ctx.saved_tensors)
        need_h, need_w, need_b = ctx.have
        dh = saved.pop(0) if need_h else None
        dw = saved.pop(0) if need_w else None
        db = saved.pop(0) if need_b else None
        gh = (dh.float() * g).to(ctx.dtypes[0]) if need_h else None
        gw = (dw[:ctx.V] * g).to(ctx.dtypes[1]) if need_w else None
        gb = (db[:ctx.V] * g).to(ctx.dtypes[2]) if need_b else None
        return gh, gw, gb, None, None, None


def linear_cross_entropy(h2d, weight, bias, labels, ignore_index=-1, chunk_rows=2048):
    """mean_i CE((h W^T + b)_i, labels_i) over the rows with labels_i != ignore_index (0 when there is none), fp32 scalar."""
    return _LinearCrossEntropy.apply(h2d, weight, bias, labels, int(ignore_index), int(chunk_rows))


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


class _LinearCrossEntropyStatic(torch.autograd.Function):
    """_LinearCrossEntropy on a fixed capacity of rows of which the first `count` (a device int32) are labelled and the
    rest hold zero features and ignore_index labels - the static-rows mode a CUDA graph can capture (mmf_b200.graphs).

    The chunk loop runs over the whole capacity; every vocabulary-sized kernel of a chunk (the GEMM, ce_rows, the dgrad,
    the wgrad and the bias column sum) takes the chunk's share of `count` as a device bound, so a chunk that starts past
    `count` costs launches whose CTAs exit at once, and inside a chunk only the rows below `count` rounded up to a
    128-row tile are computed.  The loss is loss_sum * scale with `scale` = 1 / max(count, 1) in device memory: no host
    read.  In deterministic mode the row losses are summed over the whole capacity in one fixed-shape sum."""

    @staticmethod
    def forward(ctx, h, weight, bias, labels, count, scale, ignore_index, chunk_rows):
        hb, wb = _bf16(h), _bf16(weight)
        V, K = wb.shape
        pad = (-V) % 8
        if pad:
            wb = torch.nn.functional.pad(wb, (0, 0, 0, pad))
        bb = _bf16(bias) if bias is not None else torch.zeros(V, dtype=torch.bfloat16, device=wb.device)
        if pad:
            bb = torch.cat([bb, torch.full((pad,), -30000.0, dtype=torch.bfloat16, device=bb.device)])
        M = hb.shape[0]
        labels = labels.reshape(-1).to(torch.int64).contiguous()
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_b = bias is not None and ctx.needs_input_grad[2]
        # rows past count are never written by the bounded kernels: their gradients stay the zeros allocated here
        dh = torch.zeros_like(hb) if need_h else None
        dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device) if need_w else None
        db = torch.zeros(wb.shape[0], dtype=torch.float32, device=wb.device) if need_b else None
        ordered = torch.are_deterministic_algorithms_enabled()
        loss_sum = torch.zeros((), dtype=torch.float32, device=wb.device)
        row_loss = torch.zeros(M, dtype=torch.float32, device=wb.device) if ordered else None
        # the labelled rows of chunk i: clamp(count - i * chunk_rows, 0, chunk_rows), one device int32 per chunk
        starts = torch.arange(0, M, chunk_rows, dtype=torch.int32, device=wb.device)
        bounds = (count.reshape(1) - starts).clamp_(0, chunk_rows)
        for i, r0 in enumerate(range(0, M, chunk_rows)):
            r1 = min(M, r0 + chunk_rows)
            nb = bounds[i:i + 1]
            z = F.gemm(hb[r0:r1], wb, epi=lib.EPI_BIAS, bias=bb, m_bound=nb)
            F.ce_rows_bounded(z, labels[r0:r1], ignore_index, scale, nb, loss_sum=loss_sum,
                              row_loss=row_loss[r0:r1] if ordered else None)
            if need_h:
                F.gemm(z, wb, b_mn=True, epi=lib.EPI_BIAS, out=dh[r0:r1], m_bound=nb)
            if need_w:
                F.gemm(z, hb[r0:r1], a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                       splits=best_splits(wb.shape[0], K, r1 - r0), k_bound=nb)
            if need_b:
                F.colsum_bounded(z, db, nb)
        if ordered:
            loss_sum = row_loss.sum()
        ctx.save_for_backward(*[t for t in (dh, dw, db) if t is not None])
        ctx.have = (need_h, need_w, need_b)
        ctx.V = V
        ctx.dtypes = (h.dtype, weight.dtype, bias.dtype if bias is not None else None)
        return loss_sum * scale.reshape(())

    @staticmethod
    def backward(ctx, g):
        return _LinearCrossEntropy.backward(ctx, g) + (None, None)


def linear_cross_entropy_static(h2d, weight, bias, labels, count, scale, ignore_index=-1, chunk_rows=2048):
    """linear_cross_entropy over a fixed capacity of rows whose first `count` (int32 [1] on the device) are the labelled
    ones; `scale` (fp32 [1] on the device) = 1 / max(count, 1).  Rows past count must hold ignore_index labels."""
    return _LinearCrossEntropyStatic.apply(h2d, weight, bias, labels, count, scale, int(ignore_index), int(chunk_rows))


class _LinearT(torch.autograd.Function):
    """y = x W + b with W stored [K, N]: the GEMM reads the weight MN-major (the layout the dgrad calls use), so a weight
    that is another layer's nn.Linear weight - MRFR's projection back to the feature space, tied to UNITER's img_linear
    (heads/mrfr.py:48-49, 86-88) - is consumed as it lies and autograd sums both uses' gradients into the one parameter."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        xb, wb, bb = _bf16(x), _bf16(weight), _bf16(bias)
        y = F.gemm(xb, wb, b_mn=True, epi=lib.EPI_BIAS, bias=bb)
        ctx.save_for_backward(xb, wb)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, wb = ctx.saved_tensors
        dyb = dy.to(torch.bfloat16).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = F.gemm(dyb, wb, epi=lib.EPI_BIAS).to(ctx.dtypes[0])              # dy [M, N] @ W[K, N]^T
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)       # x^T dy: [K, N]
            F.gemm(xb, dyb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
                   splits=best_splits(wb.shape[0], wb.shape[1], xb.shape[0]))
            dw = dw.to(ctx.dtypes[1])
        if ctx.needs_input_grad[2]:
            db = torch.zeros(wb.shape[1], dtype=torch.float32, device=wb.device)
            F.colsum(dyb, db)
            db = db.to(ctx.dtypes[2])
        return dx, dw, db


def linear_t(x2d, weight_kn, bias):
    """F.linear(x, weight_kn.t(), bias): x2d [M, K], weight_kn [K, N] -> bf16 [M, N]; K and N multiples of 8."""
    return _LinearT.apply(x2d, weight_kn, bias)


class _LinearGELULayerNormStatic(torch.autograd.Function):
    """LayerNorm(gelu(x W^T + b)) - the region heads' transform - on a fixed capacity of rows of which the first `count`
    (int32 [1] on the device) are live and the rest zero: the GELU GEMM, the LayerNorm and their backward (LayerNorm,
    GELU', dgrad, weight gradient, bias column sum) are all bounded by the device count, so nothing is read on the host.
    Output rows past the count are zero."""

    @staticmethod
    def forward(ctx, x, weight, bias, ln_weight, ln_bias, eps, count):
        xb, wb, bb, g, be = _bf16(x), _bf16(weight), _bf16(bias), _bf16(ln_weight), _bf16(ln_bias)
        u, h = F.gemm(xb, wb, epi=lib.EPI_BIAS_GELU, bias=bb, m_bound=count)
        y, mean, rstd = F.layernorm_fwd(h, g, be, eps, m_bound=count)
        ctx.save_for_backward(xb, wb, u, h, mean, rstd, g, count)
        ctx.dtypes = (x.dtype, weight.dtype, bias.dtype, ln_weight.dtype, ln_bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, wb, u, h, mean, rstd, g, count = ctx.saved_tensors
        dg = torch.zeros(g.shape, dtype=torch.float32, device=g.device)
        dbeta = torch.zeros_like(dg)
        # rows at and past the count come back zero; u is finite up to the 128-row tile edge, which is as far as the
        # dgrad reads du (the weight gradient reads it to the 64-row k-block edge)
        dh, _ = F.layernorm_bwd(dy.to(torch.bfloat16).contiguous(), h, mean, rstd, g, dg, dbeta, m_bound=count)
        du = F.gelu_bwd(dh, u)
        dx = F.gemm(du, wb, b_mn=True, epi=lib.EPI_BIAS, m_bound=count)
        dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)
        F.gemm(du, xb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw,
               splits=best_splits(wb.shape[0], wb.shape[1], xb.shape[0]), k_bound=count)
        db = torch.zeros(wb.shape[0], dtype=torch.float32, device=wb.device)
        F.colsum_bounded(du, db, count)
        t = ctx.dtypes
        return dx.to(t[0]), dw.to(t[1]), db.to(t[2]), dg.to(t[3]), dbeta.to(t[4]), None, None


def linear_gelu_layer_norm_static(x2d, weight, bias, ln_weight, ln_bias, eps, count):
    """LayerNorm(gelu(x2d W^T + b)) on the rows below `count` (int32 [1] on the device) of a fixed capacity whose later rows
    are zero; bf16 [M, N], zero past the count"""
    return _LinearGELULayerNormStatic.apply(x2d, weight, bias, ln_weight, ln_bias, float(eps), count)


class _RegionLossStatic(torch.autograd.Function):
    """The region heads' output projection and loss on a fixed capacity of rows whose first `count` are the masked regions:
    z = h W^T + b (weight [N, K]) or h W + b (weight_t: W stored [K, N], MRFR's tied image projection, read MN-major), then
    mmfb_kl_rows_bounded (MRC) or mmfb_mse_rows_bounded (MRFR) against target[tgt_idx[r]], which write d(z) in place; the
    dgrad, weight gradient and bias column sum run in the forward too, every kernel bounded by the device count.  The loss
    is the fixed-order sum of the row losses times `scale` (fp32 [1] on the device), so the same bits on every run; the
    backward multiplies the saved gradients by the incoming scalar.  N need not be a multiple of 8: the weight and bias are
    zero-padded and the loss kernel zeroes the padding columns' gradient."""

    @staticmethod
    def forward(ctx, h, weight, bias, target, tgt_idx, count, scale, kind, weight_t):
        hb, wb, bb = _bf16(h), _bf16(weight), _bf16(bias)
        K, N = wb.shape if weight_t else wb.shape[::-1]
        pad = (-N) % 8
        if pad:
            if weight_t:
                raise ValueError("region loss: a transposed weight needs N %% 8 == 0, got %d" % N)
            wb = torch.nn.functional.pad(wb, (0, 0, 0, pad))
            bb = torch.nn.functional.pad(bb, (0, pad))
        M = hb.shape[0]
        z = F.gemm(hb, wb, b_mn=weight_t, epi=lib.EPI_BIAS, bias=bb, m_bound=count)
        row_loss = torch.zeros(M, dtype=torch.float32, device=hb.device)
        if kind == "kl":
            F.kl_rows_bounded(z, N, target, tgt_idx, count, scale, row_loss)
        else:
            F.mse_rows_bounded(z, target, tgt_idx, count, scale, row_loss)
        dh = F.gemm(z, wb, b_mn=not weight_t, epi=lib.EPI_BIAS, out=torch.zeros_like(hb), m_bound=count)
        dw = torch.zeros(wb.shape, dtype=torch.float32, device=wb.device)
        if weight_t:                                  # [K, N] = h^T z
            F.gemm(hb, z, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=best_splits(K, N + pad, M),
                   k_bound=count)
        else:                                         # [N, K] = z^T h
            F.gemm(z, hb, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=best_splits(N + pad, K, M),
                   k_bound=count)
        db = torch.zeros(N + pad, dtype=torch.float32, device=wb.device)
        F.colsum_bounded(z, db, count)
        ctx.save_for_backward(dh, dw[:N] if not weight_t else dw, db[:N])
        ctx.dtypes = (h.dtype, weight.dtype, bias.dtype)
        return row_loss.sum() * scale.reshape(())

    @staticmethod
    def backward(ctx, g):
        dh, dw, db = ctx.saved_tensors
        t = ctx.dtypes
        return ((dh.float() * g).to(t[0]), (dw * g).to(t[1]), (db * g).to(t[2])) + (None,) * 6


def region_loss_static(h2d, weight, bias, target, tgt_idx, count, scale, kind, weight_t=False):
    """kind "kl": scale * sum_r KL(target[tgt_idx[r]] || softmax(h_r W^T + b)); kind "mse": scale * sum_r
    ||h_r W + b - target[tgt_idx[r]]||^2 (weight_t=True, weight [K, N]) - over the rows r below `count` (int32 [1] on the
    device) of a fixed capacity whose later rows are zero.  target: fp32 [*, N]; tgt_idx: int32, one per row."""
    if kind not in ("kl", "mse"):
        raise ValueError("region_loss_static: kind must be 'kl' or 'mse', got %r" % (kind,))
    return _RegionLossStatic.apply(h2d, weight, bias, target, tgt_idx, count, scale, kind, bool(weight_t))


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
