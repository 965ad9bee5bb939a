"""Thin Python wrappers over the C ABI: one function per exported kernel entry point.

Each wrapper validates dtypes/devices, allocates outputs with torch (so the caching allocator and
autograd own every buffer) and enqueues the kernel on the current CUDA stream.  Nothing here
computes on the CPU.

Deterministic mode: while torch.use_deterministic_algorithms(True) is in effect, every wrapper whose kernel would add
fp32 values with atomics in arrival order - gemm with EPI_ATOMIC_F32 and splits > 1, colsum, layernorm_bwd's parameter
gradients, embed_scatter_sorted and ce_rows' loss sum - runs the ordered variant instead, whose summation order depends
only on the call's shapes and indices, so repeated steps give the same bits.  The flag is read on every call; this module
is the only one that knows about it.  A path that has no ordered variant (embed_scatter with table gradients) raises
RuntimeError, or warns under warn_only=True, as PyTorch's own non-deterministic ops do.
"""
import ctypes
import warnings

import torch

from . import lib
from .lib import (LIB, AdamWArgs, AttnArgs, ComposeArgs, GemmArgs, GradNormArgs, LnArgs, OtArgs, ScatterArgs, _ptr, _stream_ptr,
                  check)


def _req(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the B200 path has no CPU fallback" % name)
    if t.dtype != dtype:
        raise ValueError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if t.stride(-1) != 1:
        raise ValueError("%s must be contiguous in its last dimension" % name)


def _ordered():
    return torch.are_deterministic_algorithms_enabled()


def _workspace(nbytes, device):
    """fp32 scratch of an ordered reduction, from torch's caching allocator (capture-safe).  Dropping it right after the
    launch is safe: the allocator only hands the block to work enqueued later on the same stream."""
    return torch.empty((int(nbytes) + 3) // 4, dtype=torch.float32, device=device)


def _no_ordered_path(what):
    msg = ("%s does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. "
           "You can turn off determinism just for this operation, or you can use the 'warn_only=True' option" % what)
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
    else:
        raise RuntimeError(msg)


def _idx_len(idx, M, name):
    """the kernels read one index per output row and never check: a short index buffer is an out-of-bounds device read"""
    if idx.numel() != M or not idx.is_contiguous():
        raise ValueError("%s must be a contiguous vector of %d indices (one per row), got shape %s" % (name, M, tuple(idx.shape)))


def _bound(t, name):
    """a device bound: one int32 in CUDA memory (read by the kernel when it runs, never on the host)"""
    if t is None:
        return None
    _req(t, torch.int32, name)
    if t.numel() != 1:
        raise ValueError("%s must be a CUDA int32 tensor with one element" % name)
    return t.data_ptr()


def gemm(a, b, *, a_mn=False, b_mn=False, epi=lib.EPI_BIAS, bias=None, aux=None, drop_mask=None,
         drop_scale=1.0, out=None, out2=None, splits=1, block_n=0, cluster=0, m_bound=None, k_bound=None):
    """C[M,N] = epi(A[M,K] @ B[N,K]^T) on the wgmma GEMM.

    a: [M,K] (a_mn=False) or [K,M] (a_mn=True); b: [N,K] (b_mn=False) or [K,N] (b_mn=True); bf16.
    Returns C (and C2 for EPI_BIAS_GELU and EPI_BIAS_GELU_DROP).  For EPI_ATOMIC_F32 `out` (fp32 [M,N]) is accumulated into; in deterministic
    mode with splits > 1 the split partials go through a workspace and are added in split order.
    m_bound / k_bound: int32 [1] CUDA tensors bounding M / K on the device (include/mmfb200.h, "Device bounds"); only the
    row tiles below the rounded M bound are written, so `out` past it keeps what it held.
    """
    _req(a, torch.bfloat16, "a")
    _req(b, torch.bfloat16, "b")
    _req(bias, torch.bfloat16, "bias")
    _req(aux, torch.bfloat16, "aux")
    if a.dim() != 2 or b.dim() != 2:
        raise ValueError("gemm operands must be 2-D")
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    if K != Kb:
        raise ValueError("gemm: inner dimensions differ (%d vs %d)" % (K, Kb))
    if epi == lib.EPI_ATOMIC_F32:
        if out is None:
            out = torch.zeros(M, N, dtype=torch.float32, device=a.device)
        _req(out, torch.float32, "out")
    else:
        if out is None:
            out = torch.empty(M, N, dtype=torch.bfloat16, device=a.device)
        _req(out, torch.bfloat16, "out")
        if epi in (lib.EPI_BIAS_GELU, lib.EPI_BIAS_GELU_DROP) and out2 is None:
            out2 = torch.empty(M, N, dtype=torch.bfloat16, device=a.device)
    args = GemmArgs()
    args.A, args.lda, args.a_mn = a.data_ptr(), a.stride(0), int(a_mn)
    args.B, args.ldb, args.b_mn = b.data_ptr(), b.stride(0), int(b_mn)
    args.C, args.ldc = out.data_ptr(), out.stride(0)
    args.C2 = out2.data_ptr() if out2 is not None else None
    args.bias = bias.data_ptr() if bias is not None else None
    args.aux, args.ldaux = (aux.data_ptr(), aux.stride(0)) if aux is not None else (None, 0)
    if drop_mask is not None:
        _req(drop_mask, torch.int32, "drop_mask")
        args.drop_mask, args.ldmask = drop_mask.data_ptr(), drop_mask.stride(0)
    args.drop_scale = float(drop_scale)
    args.M, args.N, args.K = M, N, K
    args.epi, args.splits, args.block_n, args.cluster = int(epi), int(splits), int(block_n), int(cluster)
    ws = None
    if epi == lib.EPI_ATOMIC_F32 and splits > 1 and _ordered():
        nbytes = LIB.mmfb_gemm_workspace_bytes(M, N, K, int(splits))
        if nbytes > 0:
            ws = _workspace(nbytes, a.device)
            args.workspace, args.workspace_bytes = ws.data_ptr(), nbytes
    if m_bound is not None or k_bound is not None:
        check(LIB.mmfb_gemm_bounded(ctypes.byref(args), _bound(m_bound, "m_bound"), _bound(k_bound, "k_bound"),
                                    _stream_ptr()))
    else:
        check(LIB.mmfb_gemm(ctypes.byref(args), _stream_ptr()))
    if epi in (lib.EPI_BIAS_GELU, lib.EPI_BIAS_GELU_DROP):
        return out, out2
    return out


def _attn_args(q, k, v, B, heads, Sq, Skv, mask, drop_mask, drop_scale, causal_len=0):
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, torch.bfloat16, n)
    W = q.shape[-1]
    if W % heads:
        raise ValueError(
            "The hidden size (%d) is not a multiple of the number of attention heads (%d)" % (W, heads))
    if q.shape[0] != B * Sq or k.shape[0] != B * Skv or v.shape[0] != B * Skv:
        raise ValueError("attention: q/k/v row counts do not match B*Sq / B*Skv")
    a = AttnArgs()
    a.q, a.ldq = q.data_ptr(), q.stride(0)
    a.k, a.ldk = k.data_ptr(), k.stride(0)
    a.v, a.ldv = v.data_ptr(), v.stride(0)
    if mask is not None:
        _req(mask, torch.float32, "mask")
        if tuple(mask.shape) != (B, Skv) or not mask.is_contiguous():
            raise ValueError("attention: additive mask must be contiguous fp32 [B, Skv]")
        a.mask = mask.data_ptr()
    if drop_mask is not None:
        _req(drop_mask, torch.int32, "drop_mask")
        if tuple(drop_mask.shape) != (B, heads, Sq, (Skv + 31) // 32) or not drop_mask.is_contiguous():
            raise ValueError("attention: drop_mask must be contiguous int32 [B, heads, Sq, ceil(Skv/32)]")
        a.drop_mask, a.drop_scale = drop_mask.data_ptr(), float(drop_scale)
    a.B, a.heads, a.Sq, a.Skv, a.head_dim = B, heads, Sq, Skv, W // heads
    a.causal_len = int(causal_len)
    return a


def attention_fwd(q, k, v, B, heads, Sq, Skv, mask=None, drop_mask=None, drop_scale=1.0, out=None, save_lo=False,
                  causal_len=0):
    """ctx, lse2 (, ctx_lo) = fused softmax(QK^T/sqrt(d) + mask) V.  q [B*Sq, h*d], k/v [B*Skv, h*d] (views allowed).
    save_lo: also return ctx_lo = bf16(O - float(ctx)), the part of the fp32 output the bf16 ctx drops; the backward's
    delta = rowsum(dO * (ctx + ctx_lo)) then carries no common rounding bias per row.
    causal_len = T > 0 (self-attention, Sq == Skv): the last T keys are a causal tail - key k >= Skv - T takes 0 where
    k <= q and -10000 otherwise, in place of mask[:, k] (M4C's prefix-LM mask); 0 = none."""
    a = _attn_args(q, k, v, B, heads, Sq, Skv, mask, drop_mask, drop_scale, causal_len)
    W = q.shape[-1]
    ctx = out if out is not None else torch.empty(B * Sq, W, dtype=torch.bfloat16, device=q.device)
    lse2 = torch.empty(B, heads, Sq, dtype=torch.float32, device=q.device)
    a.ctx, a.ldo, a.lse2 = ctx.data_ptr(), ctx.stride(0), lse2.data_ptr()
    ctx_lo = None
    if save_lo:
        ctx_lo = torch.empty(B * Sq, W, dtype=torch.bfloat16, device=q.device)
        a.ctx_lo = ctx_lo.data_ptr()
    check(LIB.mmfb_attention_fwd(ctypes.byref(a), _stream_ptr()))
    if save_lo:
        return ctx, lse2, ctx_lo
    return ctx, lse2


def attention_bwd(dctx, q, k, v, ctx, lse2, B, heads, Sq, Skv, mask=None, drop_mask=None, drop_scale=1.0,
                  dq=None, dk=None, dv=None, ctx_lo=None, causal_len=0):
    """dq, dk, dv from the saved q, k, v, ctx and row statistics (probabilities are recomputed).  causal_len: the
    forward's."""
    a = _attn_args(q, k, v, B, heads, Sq, Skv, mask, drop_mask, drop_scale, causal_len)
    _req(dctx, torch.bfloat16, "dctx")
    _req(ctx, torch.bfloat16, "ctx")
    W = q.shape[-1]
    dq = dq if dq is not None else torch.empty(B * Sq, W, dtype=torch.bfloat16, device=q.device)
    dk = dk if dk is not None else torch.empty(B * Skv, W, dtype=torch.bfloat16, device=q.device)
    dv = dv if dv is not None else torch.empty(B * Skv, W, dtype=torch.bfloat16, device=q.device)
    delta = torch.empty(B, heads, Sq, dtype=torch.float32, device=q.device)
    a.ctx, a.ldo, a.lse2 = ctx.data_ptr(), ctx.stride(0), lse2.data_ptr()
    a.dctx, a.ld_dctx, a.delta = dctx.data_ptr(), dctx.stride(0), delta.data_ptr()
    if ctx_lo is not None:
        _req(ctx_lo, torch.bfloat16, "ctx_lo")
        if not ctx_lo.is_contiguous():
            raise ValueError("ctx_lo must be contiguous [B*Sq, heads*head_dim]")
        a.ctx_lo = ctx_lo.data_ptr()
    a.dq, a.ld_dq = dq.data_ptr(), dq.stride(0)
    a.dk, a.ld_dk = dk.data_ptr(), dk.stride(0)
    a.dv, a.ld_dv = dv.data_ptr(), dv.stride(0)
    check(LIB.mmfb_attention_bwd(ctypes.byref(a), _stream_ptr()))
    return dq, dk, dv


_PROBS_DTYPES = {torch.float32: lib.MMFB_PROBS_F32, torch.bfloat16: lib.MMFB_PROBS_BF16}


def attention_probs(q, k, lse2, B, heads, Sq, Skv, mask=None, drop_mask=None, drop_scale=1.0, dtype=torch.float32,
                    out=None):
    """The attention probabilities [B, heads, Sq, Skv] of one attention_fwd call, from that call's q, k, mask, keep bits
    and the lse2 it returned: softmax(QK^T/sqrt(d) + mask) with the mask clamped at -10000 as in the forward; with keep
    bits, the post-dropout probabilities (dropped entries 0, kept ones scaled by drop_scale).  dtype: torch.float32 or
    torch.bfloat16.  `out`, when given, must be a contiguous tensor of that shape and dtype."""
    # layouts first (ValueError), then the device (_attn_args: RuntimeError for a CPU tensor)
    if dtype not in _PROBS_DTYPES:
        raise ValueError("attention_probs: dtype must be torch.float32 or torch.bfloat16, got %s" % (dtype,))
    for t, n in ((q, "q"), (k, "k")):
        if t.dtype != torch.bfloat16 or t.dim() != 2 or t.stride(-1) != 1:
            raise ValueError("attention_probs: %s must be a 2-D bf16 head-column slice, contiguous in its last dimension" % n)
    if k.shape[1] != q.shape[1] or q.shape[1] % heads:
        raise ValueError("attention_probs: q and k must have the same width, a multiple of heads=%d" % heads)
    if q.shape[0] != B * Sq or k.shape[0] != B * Skv:
        raise ValueError("attention_probs: q/k row counts do not match B*Sq / B*Skv")
    if mask is not None and (mask.dtype != torch.float32 or tuple(mask.shape) != (B, Skv) or not mask.is_contiguous()):
        raise ValueError("attention_probs: additive mask must be contiguous fp32 [B, Skv]")
    if drop_mask is not None and (drop_mask.dtype != torch.int32 or not drop_mask.is_contiguous()
                                  or tuple(drop_mask.shape) != (B, heads, Sq, (Skv + 31) // 32)):
        raise ValueError("attention_probs: drop_mask must be contiguous int32 [B, heads, Sq, ceil(Skv/32)]")
    if (not isinstance(lse2, torch.Tensor) or lse2.dtype != torch.float32 or tuple(lse2.shape) != (B, heads, Sq)
            or not lse2.is_contiguous()):
        raise ValueError("attention_probs: lse2 must be contiguous fp32 [B, heads, Sq]")
    if out is not None and (out.dtype != dtype or tuple(out.shape) != (B, heads, Sq, Skv) or not out.is_contiguous()
                            or out.device != q.device):
        raise ValueError("attention_probs: out must be a contiguous %s tensor [B, heads, Sq, Skv] = %s on %s"
                         % (dtype, (B, heads, Sq, Skv), q.device))
    a = _attn_args(q, k, k, B, heads, Sq, Skv, mask, drop_mask, drop_scale)
    a.v, a.ldv = 0, 0
    if not lse2.is_cuda:
        raise RuntimeError("lse2 must be a CUDA tensor: the B200 path has no CPU fallback")
    if out is None:
        out = torch.empty(B, heads, Sq, Skv, dtype=dtype, device=q.device)
    a.lse2 = lse2.data_ptr()
    check(LIB.mmfb_attention_probs(ctypes.byref(a), out.data_ptr(), _PROBS_DTYPES[dtype], _stream_ptr()))
    return out


def _varlen_args(q, k, v, cu_seqlens, max_len, heads, drop_mask, drop_scale, causal_len=0):
    """packed self-attention operands: q/k/v [total, h*d] rows of B samples delimited by cu_seqlens (int32 [B+1])"""
    if not isinstance(cu_seqlens, torch.Tensor) or cu_seqlens.dtype != torch.int32:
        raise ValueError("cu_seqlens must be an int32 tensor")
    if cu_seqlens.dim() != 1 or cu_seqlens.numel() < 2 or not cu_seqlens.is_contiguous():
        raise ValueError("cu_seqlens must be a contiguous int32 vector [B+1] with B >= 1, got shape %s"
                         % (tuple(cu_seqlens.shape),))
    if not cu_seqlens.is_cuda:
        raise RuntimeError("cu_seqlens must be a CUDA tensor: the kernels read it on the device")
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, torch.bfloat16, n)
        if t.dim() != 2:
            raise ValueError("attention_varlen: %s must be 2-D [total, heads*head_dim]" % n)
    total, W = q.shape
    if k.shape[0] != total or v.shape[0] != total:
        raise ValueError("attention_varlen: q/k/v must all hold total=%d rows" % total)
    if W % heads:
        raise ValueError(
            "The hidden size (%d) is not a multiple of the number of attention heads (%d)" % (W, heads))
    B = cu_seqlens.numel() - 1
    max_len = int(max_len)
    a = AttnArgs()
    a.q, a.ldq = q.data_ptr(), q.stride(0)
    a.k, a.ldk = k.data_ptr(), k.stride(0)
    a.v, a.ldv = v.data_ptr(), v.stride(0)
    if drop_mask is not None:
        _req(drop_mask, torch.int32, "drop_mask")
        if tuple(drop_mask.shape) != (heads, total, (max_len + 31) // 32) or not drop_mask.is_contiguous():
            raise ValueError("attention_varlen: drop_mask must be contiguous int32 [heads, total, ceil(max_len/32)]")
        a.drop_mask, a.drop_scale = drop_mask.data_ptr(), float(drop_scale)
    a.B, a.heads, a.Sq, a.Skv, a.head_dim = B, heads, max_len, max_len, W // heads
    a.causal_len = int(causal_len)
    return a, total, W


def attention_varlen_fwd(q, k, v, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0, out=None, save_lo=False,
                         causal_len=0):
    """Packed self-attention: ctx, lse2 (, ctx_lo).  Sample b is rows [cu_seqlens[b], cu_seqlens[b+1]) of q/k/v
    [total, h*d] (views allowed) and attends to its own rows only; max_len bounds every length.  lse2 is fp32
    [heads, total].  The lengths stay on the device: nothing here synchronises.
    causal_len = T > 0: the last T rows of every sample are a causal tail - with P_b = max(len_b - T, 0) within the
    sample, key k >= P_b takes 0 for queries q >= k and -10000 for the others (attention_fwd's rule with len_b in place of
    Skv; a sample shorter than T is all tail).  0 = none."""
    a, total, W = _varlen_args(q, k, v, cu_seqlens, max_len, heads, drop_mask, drop_scale, causal_len)
    ctx = out if out is not None else torch.empty(total, W, dtype=torch.bfloat16, device=q.device)
    _req(ctx, torch.bfloat16, "out")
    lse2 = torch.empty(heads, total, dtype=torch.float32, device=q.device)
    a.ctx, a.ldo, a.lse2 = ctx.data_ptr(), ctx.stride(0), lse2.data_ptr()
    ctx_lo = None
    if save_lo:
        ctx_lo = torch.empty(total, W, dtype=torch.bfloat16, device=q.device)
        a.ctx_lo = ctx_lo.data_ptr()
    fn = LIB.mmfb_attention_varlen_causal_fwd if a.causal_len else LIB.mmfb_attention_varlen_fwd
    check(fn(ctypes.byref(a), cu_seqlens.data_ptr(), total, _stream_ptr()))
    if save_lo:
        return ctx, lse2, ctx_lo
    return ctx, lse2


def attention_varlen_bwd(dctx, q, k, v, ctx, lse2, cu_seqlens, max_len, heads, drop_mask=None, drop_scale=1.0,
                         dq=None, dk=None, dv=None, ctx_lo=None, causal_len=0):
    """dq, dk, dv of attention_varlen_fwd (packed rows, probabilities recomputed from the saved lse2 [heads, total]).
    causal_len: the forward's."""
    a, total, W = _varlen_args(q, k, v, cu_seqlens, max_len, heads, drop_mask, drop_scale, causal_len)
    _req(dctx, torch.bfloat16, "dctx")
    _req(ctx, torch.bfloat16, "ctx")
    if dctx.shape[0] != total or ctx.shape[0] != total:
        raise ValueError("attention_varlen: dctx and ctx must hold total=%d rows" % total)
    if not lse2.is_cuda or lse2.dtype != torch.float32 or tuple(lse2.shape) != (heads, total) or not lse2.is_contiguous():
        raise ValueError("attention_varlen: lse2 must be contiguous fp32 [heads, total]")
    dq = dq if dq is not None else torch.empty(total, W, dtype=torch.bfloat16, device=q.device)
    dk = dk if dk is not None else torch.empty(total, W, dtype=torch.bfloat16, device=q.device)
    dv = dv if dv is not None else torch.empty(total, W, dtype=torch.bfloat16, device=q.device)
    for t, n in ((dq, "dq"), (dk, "dk"), (dv, "dv")):
        _req(t, torch.bfloat16, n)
    delta = torch.empty(heads, total, dtype=torch.float32, device=q.device)
    a.ctx, a.ldo, a.lse2 = ctx.data_ptr(), ctx.stride(0), lse2.data_ptr()
    a.dctx, a.ld_dctx, a.delta = dctx.data_ptr(), dctx.stride(0), delta.data_ptr()
    if ctx_lo is not None:
        _req(ctx_lo, torch.bfloat16, "ctx_lo")
        if not ctx_lo.is_contiguous() or tuple(ctx_lo.shape) != (total, W):
            raise ValueError("ctx_lo must be contiguous [total, heads*head_dim]")
        a.ctx_lo = ctx_lo.data_ptr()
    a.dq, a.ld_dq = dq.data_ptr(), dq.stride(0)
    a.dk, a.ld_dk = dk.data_ptr(), dk.stride(0)
    a.dv, a.ld_dv = dv.data_ptr(), dv.stride(0)
    fn = LIB.mmfb_attention_varlen_causal_bwd if a.causal_len else LIB.mmfb_attention_varlen_bwd
    check(fn(ctypes.byref(a), cu_seqlens.data_ptr(), total, _stream_ptr()))
    return dq, dk, dv


def _cu_check(cu, name):
    if not isinstance(cu, torch.Tensor) or cu.dtype != torch.int32:
        raise ValueError("%s must be an int32 tensor" % name)
    if cu.dim() != 1 or cu.numel() < 2 or not cu.is_contiguous():
        raise ValueError("%s must be a contiguous int32 vector [B+1] with B >= 1, got shape %s" % (name, tuple(cu.shape)))
    if not cu.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: the kernels read it on the device" % name)


def _varlen_cross_args(q, k, v, cu_q, cu_kv, max_q, max_kv, heads, drop_mask, drop_scale):
    """packed cross-attention operands: q [total_q, h*d] rows delimited by cu_q, k/v [total_kv, h*d] rows delimited by cu_kv
    (int32 [B+1] each, same B)"""
    _cu_check(cu_q, "cu_q")
    _cu_check(cu_kv, "cu_kv")
    if cu_q.numel() != cu_kv.numel():
        raise ValueError("cu_q and cu_kv must describe the same number of samples (%d vs %d)"
                         % (cu_q.numel() - 1, cu_kv.numel() - 1))
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, torch.bfloat16, n)
        if t.dim() != 2:
            raise ValueError("attention_varlen_cross: %s must be 2-D [rows, heads*head_dim]" % n)
    total_q, W = q.shape
    total_kv = k.shape[0]
    if v.shape[0] != total_kv:
        raise ValueError("attention_varlen_cross: k and v must hold the same number of rows (%d vs %d)" % (total_kv, v.shape[0]))
    if k.shape[1] != W or v.shape[1] != W:
        raise ValueError("attention_varlen_cross: q, k and v must have the same width")
    if W % heads:
        raise ValueError(
            "The hidden size (%d) is not a multiple of the number of attention heads (%d)" % (W, heads))
    max_q, max_kv = int(max_q), int(max_kv)
    a = AttnArgs()
    a.q, a.ldq = q.data_ptr(), q.stride(0)
    a.k, a.ldk = k.data_ptr(), k.stride(0)
    a.v, a.ldv = v.data_ptr(), v.stride(0)
    if drop_mask is not None:
        _req(drop_mask, torch.int32, "drop_mask")
        if tuple(drop_mask.shape) != (heads, total_q, (max_kv + 31) // 32) or not drop_mask.is_contiguous():
            raise ValueError("attention_varlen_cross: drop_mask must be contiguous int32 [heads, total_q, ceil(max_kv/32)]")
        a.drop_mask, a.drop_scale = drop_mask.data_ptr(), float(drop_scale)
    a.B, a.heads, a.Sq, a.Skv, a.head_dim = cu_q.numel() - 1, heads, max_q, max_kv, W // heads
    return a, total_q, total_kv, W


def attention_varlen_cross_fwd(q, k, v, cu_q, cu_kv, max_q, max_kv, heads, drop_mask=None, drop_scale=1.0, out=None,
                               save_lo=False):
    """Packed cross-attention: ctx, lse2 (, ctx_lo).  Sample b's queries are rows [cu_q[b], cu_q[b+1]) of q [total_q, h*d]
    and attend to its keys, rows [cu_kv[b], cu_kv[b+1]) of k / v [total_kv, h*d] (views allowed); max_q / max_kv bound the
    lengths.  lse2 is fp32 [heads, total_q].  A sample without keys gets ctx = ctx_lo = 0.  Nothing here synchronises."""
    a, total_q, total_kv, W = _varlen_cross_args(q, k, v, cu_q, cu_kv, max_q, max_kv, heads, drop_mask, drop_scale)
    ctx = out if out is not None else torch.empty(total_q, W, dtype=torch.bfloat16, device=q.device)
    _req(ctx, torch.bfloat16, "out")
    if ctx.shape[0] != total_q:
        raise ValueError("attention_varlen_cross: out must hold total_q=%d rows" % total_q)
    lse2 = torch.empty(heads, total_q, dtype=torch.float32, device=q.device)
    a.ctx, a.ldo, a.lse2 = ctx.data_ptr(), ctx.stride(0), lse2.data_ptr()
    ctx_lo = None
    if save_lo:
        ctx_lo = torch.empty(total_q, W, dtype=torch.bfloat16, device=q.device)
        a.ctx_lo = ctx_lo.data_ptr()
    check(LIB.mmfb_attention_varlen_cross_fwd(ctypes.byref(a), cu_q.data_ptr(), total_q, cu_kv.data_ptr(), total_kv,
                                              _stream_ptr()))
    if save_lo:
        return ctx, lse2, ctx_lo
    return ctx, lse2


def attention_varlen_cross_bwd(dctx, q, k, v, ctx, lse2, cu_q, cu_kv, max_q, max_kv, heads, drop_mask=None, drop_scale=1.0,
                               dq=None, dk=None, dv=None, ctx_lo=None):
    """dq [total_q, h*d], dk, dv [total_kv, h*d] of attention_varlen_cross_fwd (probabilities recomputed from the saved lse2
    [heads, total_q]).  Key rows of a sample without queries get dk = dv = 0."""
    a, total_q, total_kv, W = _varlen_cross_args(q, k, v, cu_q, cu_kv, max_q, max_kv, heads, drop_mask, drop_scale)
    _req(dctx, torch.bfloat16, "dctx")
    _req(ctx, torch.bfloat16, "ctx")
    if dctx.shape[0] != total_q or ctx.shape[0] != total_q:
        raise ValueError("attention_varlen_cross: dctx and ctx must hold total_q=%d rows" % total_q)
    if not lse2.is_cuda or lse2.dtype != torch.float32 or tuple(lse2.shape) != (heads, total_q) or not lse2.is_contiguous():
        raise ValueError("attention_varlen_cross: lse2 must be contiguous fp32 [heads, total_q]")
    dq = dq if dq is not None else torch.empty(total_q, W, dtype=torch.bfloat16, device=q.device)
    dk = dk if dk is not None else torch.empty(total_kv, W, dtype=torch.bfloat16, device=q.device)
    dv = dv if dv is not None else torch.empty(total_kv, W, dtype=torch.bfloat16, device=q.device)
    for t, n, rows in ((dq, "dq", total_q), (dk, "dk", total_kv), (dv, "dv", total_kv)):
        _req(t, torch.bfloat16, n)
        if t.shape[0] != rows:
            raise ValueError("attention_varlen_cross: %s must hold %d rows" % (n, rows))
    delta = torch.empty(heads, total_q, dtype=torch.float32, device=q.device)
    a.ctx, a.ldo, a.lse2 = ctx.data_ptr(), ctx.stride(0), lse2.data_ptr()
    a.dctx, a.ld_dctx, a.delta = dctx.data_ptr(), dctx.stride(0), delta.data_ptr()
    if ctx_lo is not None:
        _req(ctx_lo, torch.bfloat16, "ctx_lo")
        if not ctx_lo.is_contiguous() or tuple(ctx_lo.shape) != (total_q, W):
            raise ValueError("ctx_lo must be contiguous [total_q, heads*head_dim]")
        a.ctx_lo = ctx_lo.data_ptr()
    a.dq, a.ld_dq = dq.data_ptr(), dq.stride(0)
    a.dk, a.ld_dk = dk.data_ptr(), dk.stride(0)
    a.dv, a.ld_dv = dv.data_ptr(), dv.stride(0)
    check(LIB.mmfb_attention_varlen_cross_bwd(ctypes.byref(a), cu_q.data_ptr(), total_q, cu_kv.data_ptr(), total_kv,
                                              _stream_ptr()))
    return dq, dk, dv


def pack_keep_bits(keep):
    """bool [..., n] -> int32 [..., ceil(n/32)] keep-bit words (bit j of word w = element 32*w + j)."""
    n = keep.shape[-1]
    pad = (-n) % 32
    if pad:
        keep = torch.nn.functional.pad(keep, (0, pad))
    k = keep.reshape(*keep.shape[:-1], -1, 32).to(torch.int64)
    weights = (1 << torch.arange(32, device=keep.device, dtype=torch.int64))
    words = (k * weights).sum(-1)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
    return words.to(torch.int32).contiguous()


LN_EPS = 1e-12


def layernorm_fwd(y, gamma, beta, eps=LN_EPS, drop_mask=None, drop_scale=1.0, out=None, m_bound=None):
    """x, mean, rstd = LayerNorm(y) over the last dim; y bf16 [M,H] (row stride allowed).
    m_bound: an int32 [1] CUDA tensor; only the rows below it are read and written (mmfb_layernorm_fwd_bounded), and the
    rows past it of the tensors this call allocates are zero."""
    _req(y, torch.bfloat16, "y"); _req(gamma, torch.bfloat16, "gamma"); _req(beta, torch.bfloat16, "beta")
    M, H = y.shape
    alloc = torch.empty if m_bound is None else torch.zeros
    x = out if out is not None else alloc(M, H, dtype=torch.bfloat16, device=y.device)
    mean = alloc(M, dtype=torch.float32, device=y.device)
    rstd = alloc(M, dtype=torch.float32, device=y.device)
    a = LnArgs()
    a.y, a.ldy, a.gamma, a.beta = y.data_ptr(), y.stride(0), gamma.data_ptr(), beta.data_ptr()
    a.x, a.ldx, a.mean, a.rstd = x.data_ptr(), x.stride(0), mean.data_ptr(), rstd.data_ptr()
    if drop_mask is not None:
        _req(drop_mask, torch.int32, "drop_mask")
        a.drop_mask, a.ldmask, a.drop_scale = drop_mask.data_ptr(), drop_mask.stride(0), float(drop_scale)
    a.eps, a.M, a.H = float(eps), M, H
    if m_bound is not None:
        check(LIB.mmfb_layernorm_fwd_bounded(ctypes.byref(a), _bound(m_bound, "m_bound"), _stream_ptr()))
    else:
        check(LIB.mmfb_layernorm_fwd(ctypes.byref(a), _stream_ptr()))
    return x, mean, rstd


def layernorm_bwd(dx, y, mean, rstd, gamma, dgamma, dbeta, dbias=None, dx2=None, drop_mask=None, drop_scale=1.0,
                  need_dz=True, m_bound=None):
    """Returns (dy, dz): dy = grad wrt y (goes to the residual branch), dz = grad wrt the dense output that was
    dropped before the residual add (dz is dy when there is no dropout).  dgamma/dbeta/dbias (fp32 [H]) are
    accumulated in place.  m_bound: an int32 [1] CUDA tensor; only the rows below it are read and written and summed
    (mmfb_layernorm_bwd_bounded), and dy / dz are zero past it."""
    _req(dx, torch.bfloat16, "dx"); _req(y, torch.bfloat16, "y"); _req(gamma, torch.bfloat16, "gamma")
    M, H = y.shape
    alloc = torch.empty if m_bound is None else torch.zeros
    dy = alloc(M, H, dtype=torch.bfloat16, device=y.device)
    a = LnArgs()
    a.dx, a.lddx = dx.data_ptr(), dx.stride(0)
    if dx2 is not None:
        _req(dx2, torch.bfloat16, "dx2")
        a.dx2, a.lddx2 = dx2.data_ptr(), dx2.stride(0)
    a.y, a.ldy, a.mean, a.rstd, a.gamma = y.data_ptr(), y.stride(0), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr()
    a.dy, a.lddy = dy.data_ptr(), dy.stride(0)
    dz = dy
    if drop_mask is not None:
        _req(drop_mask, torch.int32, "drop_mask")
        dz = alloc(M, H, dtype=torch.bfloat16, device=y.device)
        a.drop_mask, a.ldmask, a.drop_scale = drop_mask.data_ptr(), drop_mask.stride(0), float(drop_scale)
    a.dz, a.lddz = dz.data_ptr(), dz.stride(0)
    for name, t in (("dgamma", dgamma), ("dbeta", dbeta), ("dbias", dbias)):
        if t is not None:
            _req(t, torch.float32, name)
            setattr(a, name, t.data_ptr())
    a.M, a.H = M, H
    ws = None
    if (dgamma is not None or dbeta is not None or dbias is not None) and _ordered():
        nbytes = LIB.mmfb_layernorm_bwd_workspace_bytes(M, H)
        ws = _workspace(nbytes, y.device)
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    if m_bound is not None:
        check(LIB.mmfb_layernorm_bwd_bounded(ctypes.byref(a), _bound(m_bound, "m_bound"), _stream_ptr()))
    else:
        check(LIB.mmfb_layernorm_bwd(ctypes.byref(a), _stream_ptr()))
    return dy, dz


def colsum(x, out):
    """out[n] += sum_m x[m,n] (x bf16 [M,N], out fp32 [N])."""
    _req(x, torch.bfloat16, "x"); _req(out, torch.float32, "out")
    if _ordered():
        nbytes = LIB.mmfb_colsum_workspace_bytes(x.shape[0], x.shape[1])
        ws = _workspace(nbytes, x.device)
        check(LIB.mmfb_colsum_ordered(x.data_ptr(), x.stride(0), out.data_ptr(), x.shape[0], x.shape[1], ws.data_ptr(),
                                      nbytes, _stream_ptr()))
        return out
    check(LIB.mmfb_colsum(x.data_ptr(), x.stride(0), out.data_ptr(), x.shape[0], x.shape[1], _stream_ptr()))
    return out


_DROPOUT_EPOCH = {}      # device index -> int64 [1] step counter in device memory (set by mmf_b200.graphs)


def dropout_epoch(device, create=False):
    """The device-resident step counter mixed into every keep-bit draw on `device` once it exists (None otherwise).
    A CUDA-graph capture freezes the host-side (seed, offset) of each draw; the captured graph increments this counter,
    so every replay still draws fresh masks (mmf_b200/graphs.py)."""
    idx = torch.device(device).index
    if idx is None:
        idx = torch.cuda.current_device()
    if idx not in _DROPOUT_EPOCH and create:
        _DROPOUT_EPOCH[idx] = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", idx))
    return _DROPOUT_EPOCH.get(idx)


def dropout_bits(shape_rows, ncols, p, seed, offset, device):
    """int32 keep-bit words [*shape_rows, ceil(ncols/32)] for nn.Dropout(p)."""
    words = (ncols + 31) // 32
    out = torch.empty(*shape_rows, words, dtype=torch.int32, device=device)
    epoch = dropout_epoch(out.device)
    if epoch is None:
        check(LIB.mmfb_dropout_bits(out.data_ptr(), out.numel(), int(seed) & (2 ** 64 - 1), int(offset), float(p),
                                    _stream_ptr()))
    else:
        check(LIB.mmfb_dropout_bits_epoch(out.data_ptr(), out.numel(), int(seed) & (2 ** 64 - 1), int(offset),
                                          epoch.data_ptr(), float(p), _stream_ptr()))
    return out


def dropout_path_bits(batch, rows_per_sample, ncols, p, p_path, seed, offset, device):
    """int32 keep-bit words [batch * rows_per_sample, ceil(ncols/32)] for nn.Dropout(p) followed by timm's DropPath(p_path)
    over the batch's samples: the draws of dropout_bits at (seed, offset), with every row of a dropped sample cleared.  Kept
    values scale by 1 / ((1 - p)(1 - p_path)).  Uses the Philox counters [offset, offset + 4 * words + batch)."""
    M = int(batch) * int(rows_per_sample)
    out = torch.empty(M, (ncols + 31) // 32, dtype=torch.int32, device=device)
    epoch = dropout_epoch(out.device)
    args = (out.data_ptr(), M, int(ncols), int(rows_per_sample), int(seed) & (2 ** 64 - 1), int(offset))
    if epoch is None:
        check(LIB.mmfb_dropout_path_bits(*args, float(p), float(p_path), _stream_ptr()))
    else:
        check(LIB.mmfb_dropout_path_bits_epoch(*args, epoch.data_ptr(), float(p), float(p_path), _stream_ptr()))
    return out


def relu_bwd(dy, y):
    """dz = dy where y > 0 else 0 (bf16, contiguous)."""
    _req(dy, torch.bfloat16, "dy"); _req(y, torch.bfloat16, "y")
    if not (dy.is_contiguous() and y.is_contiguous()) or dy.numel() != y.numel():
        raise ValueError("relu_bwd: contiguous, equally sized buffers required")
    dz = torch.empty_like(dy)
    check(LIB.mmfb_relu_bwd(dy.data_ptr(), y.data_ptr(), dz.data_ptr(), dy.numel(), _stream_ptr()))
    return dz


def ce_rows(logits, labels, ignore_index, grad_scale, loss_sum, row_loss=None):
    """In place: logits [M, V] bf16 (V % 8 == 0, row stride allowed) -> d(logits) = (softmax - onehot) * grad_scale, zeros for
    rows whose label is ignore_index; the summed loss of the active rows is ADDED to loss_sum (fp32 scalar tensor)."""
    _req(logits, torch.bfloat16, "logits"); _req(labels, torch.int64, "labels")
    if not loss_sum.is_cuda or loss_sum.dtype != torch.float32 or loss_sum.numel() != 1:
        raise ValueError("ce_rows: loss_sum must be a CUDA fp32 tensor with one element")
    M, V = logits.shape
    if labels.numel() != M or not labels.is_contiguous():
        raise ValueError("ce_rows: one contiguous int64 label per row required")
    rl = None
    if row_loss is not None:
        _req(row_loss, torch.float32, "row_loss")
        rl = row_loss.data_ptr()
    if _ordered():
        # the kernel's loss_sum takes one atomic per row; here the loss is a fixed-order sum of the per-row losses instead
        rows = row_loss if row_loss is not None else torch.empty(M, dtype=torch.float32, device=logits.device)
        check(LIB.mmfb_ce_rows(logits.data_ptr(), logits.stride(0), labels.data_ptr(), int(ignore_index), M, V,
                               float(grad_scale), None, rows.data_ptr(), _stream_ptr()))
        loss_sum.add_(rows.sum())
        return logits
    check(LIB.mmfb_ce_rows(logits.data_ptr(), logits.stride(0), labels.data_ptr(), int(ignore_index), M, V, float(grad_scale),
                           loss_sum.data_ptr(), rl, _stream_ptr()))
    return logits


def ce_rows_bounded(logits, labels, ignore_index, scale, m_bound, loss_sum=None, row_loss=None):
    """ce_rows on the rows below m_bound rounded up to 128, with grad_scale read from `scale` (fp32 [1]), both on the
    device.  Rows at and past the rounded bound are untouched (row_loss included).  In deterministic mode the loss goes only
    to row_loss (required), which the caller sums in a fixed order; otherwise it is added to loss_sum with atomics."""
    _req(logits, torch.bfloat16, "logits"); _req(labels, torch.int64, "labels"); _req(scale, torch.float32, "scale")
    M, V = logits.shape
    if labels.numel() != M or not labels.is_contiguous():
        raise ValueError("ce_rows_bounded: one contiguous int64 label per row required")
    if row_loss is not None:
        _req(row_loss, torch.float32, "row_loss")
        if row_loss.numel() != M:
            raise ValueError("ce_rows_bounded: row_loss must have one element per row")
    if _ordered():
        if row_loss is None:
            raise ValueError("ce_rows_bounded: deterministic mode needs row_loss (summed by the caller in a fixed order)")
        loss_sum = None
    elif loss_sum is not None and (not loss_sum.is_cuda or loss_sum.dtype != torch.float32 or loss_sum.numel() != 1):
        raise ValueError("ce_rows_bounded: loss_sum must be a CUDA fp32 tensor with one element")
    check(LIB.mmfb_ce_rows_bounded(logits.data_ptr(), logits.stride(0), labels.data_ptr(), int(ignore_index), M, V,
                                   _bound(m_bound, "m_bound"), scale.data_ptr(), _ptr(loss_sum), _ptr(row_loss),
                                   _stream_ptr()))
    return logits


def colsum_bounded(x, out, m_bound):
    """out[n] += sum over the rows m < m_bound (int32 [1] on the device) of x[m, n]; ordered in deterministic mode."""
    _req(x, torch.bfloat16, "x"); _req(out, torch.float32, "out")
    M, N = x.shape
    ws, nbytes = None, 0
    if _ordered():
        nbytes = LIB.mmfb_colsum_workspace_bytes(M, N)
        ws = _workspace(nbytes, x.device)
    check(LIB.mmfb_colsum_bounded(x.data_ptr(), x.stride(0), out.data_ptr(), M, N, _bound(m_bound, "m_bound"), _ptr(ws),
                                  nbytes, _stream_ptr()))
    return out


def _region_rows(what, z, cols, target, tgt_idx, m_bound, scale, row_loss):
    _req(z, torch.bfloat16, "z"); _req(target, torch.float32, "target"); _req(tgt_idx, torch.int32, "tgt_idx")
    _req(scale, torch.float32, "scale"); _req(row_loss, torch.float32, "row_loss")
    if z.dim() != 2 or target.dim() != 2:
        raise ValueError("%s: z and target must be 2-D" % what)
    M = z.shape[0]
    if not 0 < cols <= z.shape[1] or target.shape[1] != cols:
        raise ValueError("%s: %d columns of z [%d, %d] against a target of %d columns"
                         % (what, cols, M, z.shape[1], target.shape[1]))
    _idx_len(tgt_idx, M, "tgt_idx")
    if row_loss.numel() != M or not row_loss.is_contiguous():
        raise ValueError("%s: row_loss must be a contiguous vector of %d" % (what, M))
    if scale.numel() != 1:
        raise ValueError("%s: scale must be a CUDA fp32 tensor with one element" % what)
    return (z.data_ptr(), z.stride(0), M, cols, target.data_ptr(), target.stride(0), tgt_idx.data_ptr(),
            _bound(m_bound, "m_bound"), scale.data_ptr(), row_loss.data_ptr(), _stream_ptr())


def kl_rows_bounded(logits, V, target, tgt_idx, m_bound, scale, row_loss):
    """In place: logits [M, >= round8(V)] bf16 -> d(logits) of the KL divergence of softmax(logits[:, :V]) from the target
    rows target[tgt_idx[r]] (fp32 [*, V]), times `scale` (fp32 [1]), for the rows below m_bound (int32 [1]); row_loss[r]
    gets the row's KL.  Rows between the bound and its 128-row tile edge are zeroed, later rows untouched
    (mmfb_kl_rows_bounded); the padding columns [V, round8(V)) get a zero gradient."""
    if logits.dim() == 2 and logits.shape[1] < -(-V // 8) * 8:
        raise ValueError("kl_rows_bounded: logits need %d columns (V rounded up to 8), got %d" % (-(-V // 8) * 8,
                                                                                                logits.shape[1]))
    check(LIB.mmfb_kl_rows_bounded(*_region_rows("kl_rows_bounded", logits, V, target, tgt_idx, m_bound, scale, row_loss)))
    return logits


def mse_rows_bounded(pred, target, tgt_idx, m_bound, scale, row_loss):
    """In place: pred [M, D] bf16 -> 2 (pred - target[tgt_idx[r]]) * scale for the rows below m_bound; row_loss[r] gets the
    row's summed squared error (mmfb_mse_rows_bounded, the same row rules as kl_rows_bounded)."""
    check(LIB.mmfb_mse_rows_bounded(*_region_rows("mse_rows_bounded", pred, pred.shape[-1], target, tgt_idx, m_bound,
                                                   scale, row_loss)))
    return pred


class SelectedRows:
    """Device state of mmfb_select_rows over M labels: `count` (int32 [1]), `scale` (fp32 [1], 1 / max(count, 1)),
    `pos` / `inv` (int32 [M]) and the gathered `labels` (int64 [M], ignore_index past count).  Nothing is read on the host."""

    def __init__(self, state, labels):
        M = labels.numel()
        self.state, self.labels = state, labels
        self.count = state[0:1]
        self.scale = state[1:2].view(torch.float32)
        self.pos, self.inv = state[2:2 + M], state[2 + M:]


def select_rows(labels, ignore_index):
    """the rows whose label != ignore_index, in row-major order, selected on the device (mmfb_select_rows)"""
    _req(labels, torch.int64, "labels")
    if not labels.is_contiguous():
        raise ValueError("select_rows: labels must be contiguous")
    M = labels.numel()
    state = torch.empty(2 + 2 * M, dtype=torch.int32, device=labels.device)
    out = torch.empty(M, dtype=torch.int64, device=labels.device)
    check(LIB.mmfb_select_rows(labels.data_ptr(), int(ignore_index), M, state.data_ptr(), out.data_ptr(), _stream_ptr()))
    return SelectedRows(state, out)


def gather_rows(x, idx, out=None):
    """out[r] = x[idx[r]] where idx[r] >= 0, else 0 (bf16 rows; idx int32 on the device)"""
    _req(x, torch.bfloat16, "x"); _req(idx, torch.int32, "idx")
    M, H = idx.numel(), x.shape[1]
    if out is None:
        out = torch.empty(M, H, dtype=torch.bfloat16, device=x.device)
    _req(out, torch.bfloat16, "out")
    if tuple(out.shape) != (M, H):
        raise ValueError("gather_rows: out must be [%d, %d]" % (M, H))
    check(LIB.mmfb_gather_rows(x.data_ptr(), x.stride(0), idx.data_ptr(), out.data_ptr(), out.stride(0), M, H,
                               _stream_ptr()))
    return out


def plan_packing(masks, B, lens, causal_len=0):
    """The packing of one or two streams planned on the device (mmfb_plan_packing): `masks` holds each stream's additive
    fp32 [B, S_k] CUDA mask, or None for an unpadded stream, and `lens` their S_k.  Returns one (cu int32 [B+1], pack_map
    int32 [B*S_k], unpack_map int32 [B*S_k]) per stream, None for a stream without a mask.  A position is kept where its
    mask is exactly 0, or inside the causal tail (the last causal_len positions, one stream only); with two streams a
    sample empty in one stream and not in the other keeps every position of the empty one.  Nothing is read on the host."""
    masks, lens = list(masks), [int(s) for s in lens]
    if len(masks) not in (1, 2) or len(lens) != len(masks):
        raise ValueError("plan_packing: one or two streams, each with its length")
    out, args = [], []
    for m, S in zip(masks, lens):
        if m is None:
            out.append(None)
            args += [None, S, None, None, None]
            continue
        _req(m, torch.float32, "mask")
        if tuple(m.shape) != (B, S) or not m.is_contiguous():
            raise ValueError("plan_packing: a mask must be contiguous fp32 [B=%d, S=%d], got %s" % (B, S, tuple(m.shape)))
        cu = torch.empty(B + 1, dtype=torch.int32, device=m.device)
        pack_map = torch.empty(B * S, dtype=torch.int32, device=m.device)
        unpack_map = torch.empty(B * S, dtype=torch.int32, device=m.device)
        out.append((cu, pack_map, unpack_map))
        args += [m.data_ptr(), S, cu.data_ptr(), pack_map.data_ptr(), unpack_map.data_ptr()]
    if len(masks) == 1:
        args += [None, 0, None, None, None]
    check(LIB.mmfb_plan_packing(*args, int(B), int(causal_len), _stream_ptr()))
    return out


def add(a, b):
    """a + b (bf16, contiguous, same size)."""
    _req(a, torch.bfloat16, "a"); _req(b, torch.bfloat16, "b")
    if not (a.is_contiguous() and b.is_contiguous()) or a.numel() != b.numel():
        raise ValueError("add: contiguous, equally sized buffers required")
    out = torch.empty_like(a)
    check(LIB.mmfb_add_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _stream_ptr()))
    return out


def dropout_apply(x, drop_mask, drop_scale):
    """keep-bit ? x * scale : 0 for x bf16 [M, H] and keep-bit words int32 [M, ceil(H/32)]."""
    _req(x, torch.bfloat16, "x"); _req(drop_mask, torch.int32, "drop_mask")
    M, H = x.shape
    out = torch.empty(M, H, dtype=torch.bfloat16, device=x.device)
    check(LIB.mmfb_dropout_apply(x.data_ptr(), x.stride(0), drop_mask.data_ptr(), drop_mask.stride(0), float(drop_scale),
                                 out.data_ptr(), out.stride(0), M, H, _stream_ptr()))
    return out


def gelu_bwd(dh, u):
    """du = dh * GELU'(u) (bf16, contiguous) - for a GELU that is followed by a LayerNorm instead of a GEMM."""
    _req(dh, torch.bfloat16, "dh"); _req(u, torch.bfloat16, "u")
    if not (dh.is_contiguous() and u.is_contiguous()) or dh.numel() != u.numel():
        raise ValueError("gelu_bwd: contiguous, equally sized buffers required")
    du = torch.empty_like(dh)
    check(LIB.mmfb_gelu_bwd(dh.data_ptr(), u.data_ptr(), du.data_ptr(), dh.numel(), _stream_ptr()))
    return du


def _req_scalar(t, what, name):
    """the device scalars of the optimizer launches: None or a one-element fp32 CUDA tensor; returns its pointer"""
    if t is None:
        return None
    if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32 or t.numel() != 1:
        raise ValueError("%s: %s must be a one-element fp32 CUDA tensor" % (what, name))
    return t.data_ptr()


def _req_active(active, n_slots, what):
    """the per-slot gate of include/mmfb200_active.h: None or a contiguous uint8 CUDA tensor [n_slots]"""
    if active is None:
        return None
    if not torch.is_tensor(active) or not active.is_cuda or active.dtype != torch.uint8 or active.dim() != 1 or \
            not active.is_contiguous() or active.numel() != n_slots:
        raise ValueError("%s: active must be a contiguous uint8 CUDA tensor with one entry per slot (%d)" % (what, n_slots))
    return ctypes.c_void_p(active.data_ptr())


def adamw(param, grad, exp_avg, exp_avg_sq, groups, *, beta1, beta2, eps, mode, grad_scale=1.0, group_of_block=None,
          param_bf16=None, grad_scale_dev=None, hp_dev=None, loss_scale_dev=None, found_inf=None, active=None):
    """One fused AdamW step over flat fp32 buffers (staged, include/mmfb200.h: mmfb_adamw).
    groups: list (<= 8) of dicts {lr, weight_decay, step_size, bc2_sqrt}; group_of_block: uint8 [n/8] or None;
    grad_scale_dev: None or a one-element fp32 CUDA tensor (grad_norm's clip coefficient) multiplied into grad_scale when
    the kernel runs.  hp_dev: None or an fp32 CUDA tensor [n_groups, 8] written by adamw_hparams; the kernel then reads
    every group's hyper-parameters and beta1 / beta2 / eps from it, and `groups` may be None.
    loss_scale_dev, found_inf: None or one-element fp32 CUDA tensors (GradScaler's scale and non-finite flag): the
    gradients are first multiplied by fp32(1 / fp64(scale)), as GradScaler.unscale_ does, and a non-zero found_inf makes
    the launch write nothing.
    active: None or a uint8 CUDA tensor with one entry per row of hp_dev (include/mmfb200_active.h: mmfb_adamw_active);
    the blocks of a group whose entry is 0 read and write nothing."""
    if active is not None and hp_dev is None:
        raise ValueError("adamw: active gates the rows of hp_dev; pass hp_dev as well")
    for t, n in ((param, "param"), (grad, "grad"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        _req(t, torch.float32, n)
        if not t.is_contiguous() or t.numel() != param.numel():
            raise ValueError("adamw: %s must be contiguous and as large as param" % n)
    a = AdamWArgs()
    a.param, a.grad, a.exp_avg, a.exp_avg_sq = param.data_ptr(), grad.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr()
    if param_bf16 is not None:
        _req(param_bf16, torch.bfloat16, "param_bf16")
        a.param_bf16 = param_bf16.data_ptr()
    if group_of_block is not None:
        _req(group_of_block, torch.uint8, "group_of_block")
        if group_of_block.numel() != param.numel() // 8:
            raise ValueError("adamw: group_of_block needs one entry per 8 elements")
        a.group = group_of_block.data_ptr()
    if hp_dev is not None:
        _req_hp(hp_dev, "adamw")
        n_groups = hp_dev.shape[0]
        a.hp_dev = hp_dev.data_ptr()
    else:
        n_groups = len(groups)
    a.n, a.n_groups = param.numel(), n_groups
    if not 1 <= n_groups <= 8:
        raise ValueError("adamw: between 1 and 8 hyper-parameter groups per launch")
    for i, g in enumerate(groups or ()):
        a.lr[i], a.weight_decay[i], a.step_size[i], a.bc2_sqrt[i] = g["lr"], g["weight_decay"], g["step_size"], g["bc2_sqrt"]
    a.beta1, a.beta2, a.eps, a.grad_scale, a.mode = float(beta1), float(beta2), float(eps), float(grad_scale), int(mode)
    if grad_scale_dev is not None:
        if not grad_scale_dev.is_cuda or grad_scale_dev.dtype != torch.float32 or grad_scale_dev.numel() != 1:
            raise ValueError("adamw: grad_scale_dev must be a one-element fp32 CUDA tensor")
        a.grad_scale_dev = grad_scale_dev.data_ptr()
    a.loss_scale_dev = _req_scalar(loss_scale_dev, "adamw", "loss_scale_dev")
    a.found_inf = _req_scalar(found_inf, "adamw", "found_inf")
    gate = _req_active(active, n_groups, "adamw")
    if gate is None:
        check(LIB.mmfb_adamw(ctypes.byref(a), _stream_ptr()))
    else:
        check(LIB.mmfb_adamw_active(ctypes.byref(a), gate, _stream_ptr()))


def _req_hp(hp, what):
    if not hp.is_cuda or hp.dtype != torch.float32 or hp.dim() != 2 or hp.shape[1] != lib.ADAMW_HP_FLOATS or \
            not hp.is_contiguous():
        raise ValueError("%s: the hyper-parameter table must be a contiguous fp32 CUDA tensor [slots, %d]"
                         % (what, lib.ADAMW_HP_FLOATS))


def adamw_hparams(groups, slots, step, hp, mode, found_inf=None, active=None):
    """Advance the step counts and write the AdamW hyper-parameter table on the device (include/mmfb200.h:
    mmfb_adamw_hparams).  groups: fp64 CUDA [n_groups, 5] (lr, weight_decay, beta1, beta2, eps); slots: the device
    table of adamw_slot_table; step: int64 CUDA [n_slots], advanced by one for every slot that is not frozen; hp: fp32
    CUDA [n_slots, 8], overwritten.  found_inf: None or a one-element fp32 CUDA tensor; when it is non-zero the launch
    changes nothing (a step GradScaler skips does not count).  Nothing is read on the host.
    active: None or a uint8 CUDA tensor [n_slots] (include/mmfb200_active.h: mmfb_adamw_hparams_active); a slot whose
    entry is 0 keeps its step count and gets a frozen slot's row."""
    if groups.dtype != torch.float64 or groups.dim() != 2 or groups.shape[1] != lib.ADAMW_GROUP_HP_DOUBLES or \
            not groups.is_contiguous():
        raise ValueError("adamw_hparams: groups must be a contiguous fp64 tensor [n_groups, %d]" % lib.ADAMW_GROUP_HP_DOUBLES)
    if step.dtype != torch.int64 or step.dim() != 1 or not step.is_contiguous():
        raise ValueError("adamw_hparams: step must be a contiguous int64 tensor")
    _req_hp(hp, "adamw_hparams")
    if hp.shape[0] != step.numel() or slots.numel() != step.numel() * 8:
        raise ValueError("adamw_hparams: slots, step and hp must have one entry per slot")
    for t in (groups, slots, step):
        if not t.is_cuda:
            raise RuntimeError("adamw_hparams: tensors must be CUDA tensors: the B200 path has no CPU fallback")
    a = lib.AdamWHparamsArgs()
    a.groups, a.slots, a.step, a.hp = groups.data_ptr(), slots.data_ptr(), step.data_ptr(), hp.data_ptr()
    a.n_slots, a.mode = step.numel(), int(mode)
    a.found_inf = _req_scalar(found_inf, "adamw_hparams", "found_inf")
    gate = _req_active(active, step.numel(), "adamw_hparams")
    if gate is None:
        check(LIB.mmfb_adamw_hparams(ctypes.byref(a), _stream_ptr()))
    else:
        check(LIB.mmfb_adamw_hparams_active(ctypes.byref(a), gate, _stream_ptr()))


def adamw_slot_table(slots, device):
    """DEVICE table of mmfb_adamw_slot for adamw_hparams: `slots` is a list of (group index, flags)."""
    arr = (lib.AdamWSlot * len(slots))(*[lib.AdamWSlot(*s) for s in slots])
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).pin_memory()
    return host.to(device, non_blocking=True)


def adamw_segment_rows(segments):
    """Host rows of the mmfb_adamw_segments table: `segments` is a list of (param, grad, exp_avg, exp_avg_sq, slot)
    with contiguous fp32 tensors of equal sizes.  Returns (rows, n_blocks), a row being (param_ptr, grad_ptr,
    exp_avg_ptr, exp_avg_sq_ptr, n, slot, first_block, head); empty tensors get no row."""
    rows, first = [], 0
    for p, g, m, v, slot in segments:
        for t, name in ((p, "param"), (g, "grad"), (m, "exp_avg"), (v, "exp_avg_sq")):
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError("adamw_segments: %s must be a contiguous fp32 tensor, got %s%s"
                                 % (name, t.dtype, "" if t.is_contiguous() else " (not contiguous)"))
            if t.numel() != p.numel():
                raise ValueError("adamw_segments: %s has %d elements, param %d" % (name, t.numel(), p.numel()))
        if p.numel() == 0:
            continue
        ptrs = (p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr())
        mis = {(x >> 2) & 3 for x in ptrs}
        head = (4 - mis.pop()) & 3 if len(mis) == 1 else -1
        lead = 8 - head if head > 0 else 0
        rows.append(ptrs + (p.numel(), int(slot), first, head))
        first += (p.numel() + lead + lib.MMFB_ADAMW_SEGMENT_BLOCK - 1) // lib.MMFB_ADAMW_SEGMENT_BLOCK
    if first >= 2 ** 31:
        raise ValueError("adamw_segments: too many elements (%d blocks)" % first)
    return rows, first


class AdamWSegmentTable:
    """The DEVICE table of mmfb_adamw_segments over a fixed list of tensors (see adamw_segment_table)."""

    def __init__(self, segments, rows, n_blocks):
        self.segments, self.rows, self.n_blocks = segments, rows, n_blocks


def adamw_segment_table(segments):
    """Segment table for adamw_segments (rows as adamw_segment_rows).  One host-to-device copy from pinned memory without
    a stream synchronisation; it stays valid while the tensors keep their storage."""
    for s in segments:
        for t in s[:4]:
            if not t.is_cuda:
                raise RuntimeError("adamw_segments: tensors must be CUDA tensors: the B200 path has no CPU fallback")
    rows, n_blocks = adamw_segment_rows(segments)
    if not rows:
        raise ValueError("adamw_segments: no non-empty tensor")
    arr = (lib.AdamWSegment * len(rows))(*[lib.AdamWSegment(*r, 0) for r in rows])
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).pin_memory()
    return AdamWSegmentTable(host.to(segments[0][0].device, non_blocking=True), rows, n_blocks)


def adamw_segments(table, hp, *, mode, grad_scale=1.0, grad_scale_dev=None, loss_scale_dev=None, found_inf=None,
                   active=None):
    """One AdamW launch over every tensor of `table` (include/mmfb200.h: mmfb_adamw_segments), each with the
    hyper-parameters of its slot in hp (fp32 CUDA [slots, 8], written by adamw_hparams).  Element for element the
    arithmetic of adamw; grad_scale_dev, loss_scale_dev and found_inf as there.  active: None or a uint8 CUDA tensor
    with one entry per row of hp (mmfb_adamw_segments_active); a segment whose slot's entry is 0 is left alone."""
    _req_hp(hp, "adamw_segments")
    a = lib.AdamWSegmentsArgs()
    a.segments, a.n_segments, a.n_blocks = table.segments.data_ptr(), len(table.rows), table.n_blocks
    a.hp, a.grad_scale, a.mode = hp.data_ptr(), float(grad_scale), int(mode)
    if grad_scale_dev is not None:
        if not grad_scale_dev.is_cuda or grad_scale_dev.dtype != torch.float32 or grad_scale_dev.numel() != 1:
            raise ValueError("adamw_segments: grad_scale_dev must be a one-element fp32 CUDA tensor")
        a.grad_scale_dev = grad_scale_dev.data_ptr()
    a.loss_scale_dev = _req_scalar(loss_scale_dev, "adamw_segments", "loss_scale_dev")
    a.found_inf = _req_scalar(found_inf, "adamw_segments", "found_inf")
    gate = _req_active(active, hp.shape[0], "adamw_segments")
    if gate is None:
        check(LIB.mmfb_adamw_segments(ctypes.byref(a), _stream_ptr()))
    else:
        check(LIB.mmfb_adamw_segments_active(ctypes.byref(a), gate, _stream_ptr()))


class GradNormTable:
    """The DEVICE segment table of mmfb_grad_norm over a fixed list of gradient buffers (see grad_norm_table)."""

    def __init__(self, segments, n_segments, n_blocks, device):
        self.segments, self.n_segments, self.n_blocks, self.device = segments, n_segments, n_blocks, device


def grad_norm_table(grads):
    """Segment table for grad_norm over `grads`: contiguous fp32 or bf16 CUDA tensors, one segment each (empty ones are
    skipped).  One host-to-device copy from pinned memory, without a stream synchronisation; the table stays valid while
    the tensors keep their storage, so callers build it once and reuse it."""
    segs, first = [], 0
    device = None
    for g in grads:
        if not g.is_cuda:
            raise RuntimeError("grad_norm: gradients must be CUDA tensors: the B200 path has no CPU fallback")
        if g.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("grad_norm: gradients must be fp32 or bf16, got %s" % g.dtype)
        if not g.is_contiguous():
            raise ValueError("grad_norm: gradients must be contiguous")
        if device is not None and g.device != device:
            raise ValueError("grad_norm: all gradients must be on one device")
        device = g.device
        if g.numel() == 0:
            continue
        segs.append((g.data_ptr(), g.numel(), lib.MMFB_GRAD_BF16 if g.dtype == torch.bfloat16 else lib.MMFB_GRAD_F32, first))
        first += (g.numel() + lib.MMFB_GRAD_NORM_BLOCK - 1) // lib.MMFB_GRAD_NORM_BLOCK
    if not segs:
        raise ValueError("grad_norm: no non-empty gradient")
    if first >= 2 ** 31:
        raise ValueError("grad_norm: too many elements (%d partial-sum blocks)" % first)
    arr = (lib.GradSegment * len(segs))(*[lib.GradSegment(*s) for s in segs])
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).pin_memory()
    return GradNormTable(host.to(device, non_blocking=True), len(segs), first, device)


def grad_norm(table, max_norm, norm_type=2.0, max_norm_scale_dev=None):
    """Global L2 norm of the gradients of `table` and torch's clip coefficient min(max_norm / (norm + 1e-6), 1), both
    computed on the device (include/mmfb200.h: mmfb_grad_norm).  Returns fp32 [2] = (total_norm, clip_coef) without a host
    synchronisation; the summation order is fixed, so the bits repeat in every mode.  Only norm_type 2 is supported.
    max_norm_scale_dev: None or a one-element fp32 CUDA tensor S; the threshold is then fp32(max_norm) * S in fp32, read
    when the kernel runs (the clip of loss-scaled gradients)."""
    if float(norm_type) != 2.0:
        raise ValueError("grad_norm: only norm_type 2 is supported, got %s" % (norm_type,))
    out = torch.empty(2, dtype=torch.float32, device=table.device)
    partials = torch.empty(table.n_blocks, dtype=torch.float64, device=table.device)
    a = GradNormArgs()
    a.segments, a.n_segments, a.n_blocks = table.segments.data_ptr(), table.n_segments, table.n_blocks
    a.partials, a.out = partials.data_ptr(), out.data_ptr()
    a.max_norm, a.norm_type = float(max_norm), float(norm_type)
    a.max_norm_scale_dev = _req_scalar(max_norm_scale_dev, "grad_norm", "max_norm_scale_dev")
    check(LIB.mmfb_grad_norm(ctypes.byref(a), _stream_ptr()))
    return out


def grad_norm_check(table, max_norm, found_inf, norm_type=2.0, max_norm_scale_dev=None):
    """grad_norm, and GradScaler's non-finite check of the same gradients in the same read (include/mmfb200.h:
    mmfb_grad_norm_check): found_inf, a one-element fp32 CUDA tensor, is overwritten with 1.0 when any element is inf or
    NaN and 0.0 otherwise.  The test is per element, not on the norm.  Returns fp32 [2] as grad_norm."""
    if float(norm_type) != 2.0:
        raise ValueError("grad_norm_check: only norm_type 2 is supported, got %s" % (norm_type,))
    out = torch.empty(2, dtype=torch.float32, device=table.device)
    partials = torch.empty(2 * table.n_blocks, dtype=torch.float64, device=table.device)
    a = GradNormArgs()
    a.segments, a.n_segments, a.n_blocks = table.segments.data_ptr(), table.n_segments, table.n_blocks
    a.partials, a.out = partials.data_ptr(), out.data_ptr()
    a.max_norm, a.norm_type = float(max_norm), float(norm_type)
    a.max_norm_scale_dev = _req_scalar(max_norm_scale_dev, "grad_norm_check", "max_norm_scale_dev")
    fi = _req_scalar(found_inf, "grad_norm_check", "found_inf")
    if fi is None:
        raise ValueError("grad_norm_check: found_inf must be a one-element fp32 CUDA tensor")
    check(LIB.mmfb_grad_norm_check(ctypes.byref(a), fi, _stream_ptr()))
    return out


def grad_check(table, found_inf):
    """GradScaler's non-finite check alone over the gradients of a grad_norm table (include/mmfb200.h: mmfb_grad_check):
    found_inf is overwritten with 1.0 when any element is inf or NaN and 0.0 otherwise, nothing read on the host."""
    fi = _req_scalar(found_inf, "grad_check", "found_inf")
    if fi is None:
        raise ValueError("grad_check: found_inf must be a one-element fp32 CUDA tensor")
    flags = torch.empty(table.n_blocks, dtype=torch.float64, device=table.device)
    check(LIB.mmfb_grad_check(table.segments.data_ptr(), table.n_segments, table.n_blocks, flags.data_ptr(), fi,
                              _stream_ptr()))


def lr_schedule(counter, base_lr, lr, desc, advance, lr_stride=1):
    """One launch of MMF's learning-rate schedule on the device (include/mmfb200.h: mmfb_lr_schedule): with t = counter
    (+ 1 when advancing), lr[g * lr_stride] = base_lr[g] * f(t) in fp64, and the counter is stored advanced.
    counter: int64 CUDA [1]; base_lr: fp64 CUDA [n_groups]; lr: fp64 CUDA, typically the optimizer's group table;
    desc: a lib.LrScheduleDesc."""
    if counter.dtype != torch.int64 or counter.numel() != 1 or not counter.is_cuda:
        raise ValueError("lr_schedule: counter must be a one-element int64 CUDA tensor")
    if base_lr.dtype != torch.float64 or base_lr.dim() != 1 or not base_lr.is_contiguous() or not base_lr.is_cuda:
        raise ValueError("lr_schedule: base_lr must be a contiguous fp64 CUDA tensor [n_groups]")
    if lr.dtype != torch.float64 or not lr.is_contiguous() or not lr.is_cuda or \
            lr.numel() < (base_lr.numel() - 1) * lr_stride + 1:
        raise ValueError("lr_schedule: lr must be a contiguous fp64 CUDA tensor holding n_groups entries %d apart"
                         % lr_stride)
    a = lib.LrScheduleArgs()
    a.counter, a.base_lr, a.lr = counter.data_ptr(), base_lr.data_ptr(), lr.data_ptr()
    a.n_groups, a.lr_stride, a.advance = base_lr.numel(), int(lr_stride), 1 if advance else 0
    a.desc = desc
    check(LIB.mmfb_lr_schedule(ctypes.byref(a), _stream_ptr()))


def cast_f32_bf16(src, dst):
    _req(src, torch.float32, "src"); _req(dst, torch.bfloat16, "dst")
    if src.numel() != dst.numel() or not src.is_contiguous() or not dst.is_contiguous():
        raise ValueError("cast: buffers must be contiguous and equally sized")
    check(LIB.mmfb_cast_f32_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), _stream_ptr()))
    return dst


def embed_compose(M, H, srcs=(), tabs=(), device=None):
    """y[r] = sum_k src_k[row_k[r]] + sum_k tab_k[idx_k[r]].
    srcs: up to 2 of (bf16 [*,H] tensor, int32 [M] rows); tabs: up to 3 of (bf16 [V,H] table, int32 [M] idx).
    Negative indices drop the term for that row."""
    a = ComposeArgs()
    keep = []
    for k, (t, rows) in enumerate(srcs):
        _req(t, torch.bfloat16, "src%d" % k); _req(rows, torch.int32, "src_row%d" % k)
        _idx_len(rows, M, "src_row%d" % k)
        a.src[k], a.ldsrc[k], a.src_row[k] = t.data_ptr(), t.stride(0), rows.data_ptr()
        device = t.device
    for k, (t, idx) in enumerate(tabs):
        _req(t, torch.bfloat16, "tab%d" % k); _req(idx, torch.int32, "tab_idx%d" % k)
        _idx_len(idx, M, "tab_idx%d" % k)
        if t.shape[1] != H or not t.is_contiguous():
            raise ValueError("embedding table %d must be contiguous [V, %d]" % (k, H))
        a.tab[k], a.tab_idx[k] = t.data_ptr(), idx.data_ptr()
        device = t.device
    y = torch.empty(M, H, dtype=torch.bfloat16, device=device)
    a.y, a.ldy, a.M, a.H = y.data_ptr(), y.stride(0), M, H
    check(LIB.mmfb_embed_compose(ctypes.byref(a), _stream_ptr()))
    return y


def embed_scatter(dy, dsrcs=(), dtabs=()):
    """Backward of embed_compose: dsrcs (bf16 tensor, rows) get plain row stores, dtabs (fp32 table grad, idx) get
    atomic accumulation (no ordered variant: refused in deterministic mode; embed_scatter_sorted has one)."""
    _req(dy, torch.bfloat16, "dy")
    if len(dtabs) and _ordered():
        _no_ordered_path("mmf_b200.functional.embed_scatter with table gradients (dtabs)")
    M, H = dy.shape
    a = ScatterArgs()
    for k, (t, rows) in enumerate(dsrcs):
        _req(t, torch.bfloat16, "dsrc%d" % k)
        _idx_len(rows, M, "src_row%d" % k)
        a.dsrc[k], a.ldsrc[k], a.src_row[k] = t.data_ptr(), t.stride(0), rows.data_ptr()
    for k, (t, idx) in enumerate(dtabs):
        _req(t, torch.float32, "dtab%d" % k)
        _idx_len(idx, M, "tab_idx%d" % k)
        a.dtab[k], a.tab_idx[k] = t.data_ptr(), idx.data_ptr()
    a.dy, a.lddy, a.M, a.H = dy.data_ptr(), dy.stride(0), M, H
    check(LIB.mmfb_embed_scatter(ctypes.byref(a), _stream_ptr()))


def sort_indices(idx):
    """(sorted_idx, order) int32 for embed_scatter_sorted; a stable device sort of the [M] index vector."""
    sorted_idx, order = torch.sort(idx.to(torch.int64), stable=True)
    return sorted_idx.to(torch.int32).contiguous(), order.to(torch.int32).contiguous()


def embed_scatter_sorted(dy, dtab, sorted_idx, order):
    """dtab[sorted_idx[k]] += dy[order[k]] with run aggregation (fp32 table gradient)."""
    _req(dy, torch.bfloat16, "dy"); _req(dtab, torch.float32, "dtab")
    _req(sorted_idx, torch.int32, "sorted_idx"); _req(order, torch.int32, "order")
    M, H = dy.shape
    _idx_len(sorted_idx, M, "sorted_idx"); _idx_len(order, M, "order")
    if _ordered():
        nbytes = LIB.mmfb_embed_scatter_sorted_workspace_bytes(M, H)
        ws = _workspace(nbytes, dy.device)
        check(LIB.mmfb_embed_scatter_sorted_ordered(dy.data_ptr(), dy.stride(0), order.data_ptr(), sorted_idx.data_ptr(),
                                                    dtab.data_ptr(), M, H, ws.data_ptr(), nbytes, _stream_ptr()))
        return
    check(LIB.mmfb_embed_scatter_sorted(dy.data_ptr(), dy.stride(0), order.data_ptr(), sorted_idx.data_ptr(),
                                        dtab.data_ptr(), M, H, _stream_ptr()))


def unpack_keep_bits(words, n):
    """int32 [..., W] -> bool [..., n] (test helper / oracle interop; runs on the words' device)."""
    w = words.to(torch.int64) & 0xFFFFFFFF
    bits = (w.unsqueeze(-1) >> torch.arange(32, device=words.device, dtype=torch.int64)) & 1
    return bits.reshape(*words.shape[:-1], -1)[..., :n].bool()


def _ot_args(x, y, x_len, y_len):
    """x [B, M, H], y [B, N, H]: bf16 views with a contiguous last dimension (e.g. two row ranges of one encoder output);
    x_len / y_len: one int per sample, on the host (the library validates them and passes them as launch parameters)"""
    _req(x, torch.bfloat16, "x"); _req(y, torch.bfloat16, "y")
    if x.dim() != 3 or y.dim() != 3 or x.shape[0] != y.shape[0] or x.shape[2] != y.shape[2]:
        raise ValueError("optimal transport: x [B, M, H] and y [B, N, H] required, got %s and %s" % (tuple(x.shape), tuple(y.shape)))
    B = x.shape[0]
    lens = []
    for t, name in ((x_len, "x_len"), (y_len, "y_len")):
        t = torch.as_tensor(t).reshape(-1).to(device="cpu", dtype=torch.int32).contiguous()
        if t.numel() != B:
            raise ValueError("optimal transport: %s must hold one length per sample (%d), got %d" % (name, B, t.numel()))
        lens.append(t)
    a = OtArgs()
    a.x, a.ldx, a.bsx = x.data_ptr(), x.stride(1), x.stride(0)
    a.y, a.ldy, a.bsy = y.data_ptr(), y.stride(1), y.stride(0)
    a.x_len, a.y_len = lens[0].data_ptr(), lens[1].data_ptr()
    a.B, a.M, a.N, a.H = B, x.shape[1], y.shape[1], x.shape[2]
    return a, lens


def ot_fwd(x, y, x_len, y_len, beta=0.5, iterations=50, k=1, want_cost=False):
    """dist [B], plan T [B, N, M], saved [B, 2 (M + N)] (, cost [B, M, N]) of mmfb_ot_fwd: cosine cost + IPOT + trace(C T),
    one CTA per sample (mmf/modules/ot.py:80-102)."""
    a, lens = _ot_args(x, y, x_len, y_len)
    B, M, N = a.B, a.M, a.N
    dist = torch.empty(B, dtype=torch.float32, device=x.device)
    plan = torch.empty(B, N, M, dtype=torch.float32, device=x.device)
    saved = torch.empty(B, 2 * (M + N), dtype=torch.float32, device=x.device)
    cost = torch.empty(B, M, N, dtype=torch.float32, device=x.device) if want_cost else None
    a.dist, a.plan, a.saved, a.cost = dist.data_ptr(), plan.data_ptr(), saved.data_ptr(), _ptr(cost)
    a.beta, a.iterations, a.k = float(beta), int(iterations), int(k)
    check(LIB.mmfb_ot_fwd(ctypes.byref(a), _stream_ptr()))
    return (dist, plan, saved, cost) if want_cost else (dist, plan, saved)


def ot_bwd(g, plan, saved, x, y, x_len, y_len, dx, dy):
    """dx, dy (bf16 views addressed like x, y; every row is written, padded rows with zeros) from g = d loss / d dist [B]"""
    a, lens = _ot_args(x, y, x_len, y_len)
    _req(g, torch.float32, "g"); _req(plan, torch.float32, "plan"); _req(saved, torch.float32, "saved")
    _req(dx, torch.bfloat16, "dx"); _req(dy, torch.bfloat16, "dy")
    if dx.shape != x.shape or dy.shape != y.shape:
        raise ValueError("optimal transport: dx / dy must have the shapes of x / y")
    if not (g.is_contiguous() and plan.is_contiguous() and saved.is_contiguous()) or g.numel() != a.B or \
            tuple(plan.shape) != (a.B, a.N, a.M) or tuple(saved.shape) != (a.B, 2 * (a.M + a.N)):
        raise ValueError("optimal transport: g [B], plan [B, N, M] and saved [B, 2 (M + N)] must be the forward's, contiguous")
    a.g, a.plan, a.saved = g.data_ptr(), plan.data_ptr(), saved.data_ptr()
    a.dx, a.lddx, a.bsdx = dx.data_ptr(), dx.stride(1), dx.stride(0)
    a.dy, a.lddy, a.bsdy = dy.data_ptr(), dy.stride(1), dy.stride(0)
    check(LIB.mmfb_ot_bwd(ctypes.byref(a), _stream_ptr()))
    return dx, dy
