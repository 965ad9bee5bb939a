"""Every compute entry point of include/mmfb200.h with NaN in the memory it must not read and sentinels around what it
must not write (tests/guarded.py).

Each case runs the call twice on the same values: once on tight, freshly allocated buffers, once with every input inside
a poisoned allocation (NaN rows before and after, NaN slack columns, NaN capacity rows past the logical row count, keep-bit
slack of all ones, index slack holding valid but wrong indices) and every output inside a sentinel-filled one.  A pure
output view starts at the sentinel too (a NaN), so an element the kernel should write and does not shows up; only where
the contract says rows keep what they held (past a device bound, the rows a scatter does not index) does the view start
at zero.  The guarded outputs must hold no NaN, equal the tight call bit for bit, and every element outside the views
must keep its fill.  That comparison is what exposes a poison read or a guard write; it is not an accuracy check.  The
accuracy of these kernels is checked against fp64 by the edge tests, and here directly for the GEMM sweep (every
epilogue), dense attention, LayerNorm forward, the column sums, embedding compose and scatter, the element-wise kernels
and the gradient norm; the other cases (causal, probs, varlen, cross-entropy and region losses, dropout_apply, AdamW)
rely on the tight comparison, at shapes that are not all those of the edge tests.

CASES maps every compute entry point to the tests that poison it (tests/test_guarded_cpu.py checks that it is complete).
"""
import contextlib
import ctypes

import pytest
import torch

import guarded as G
import kernel_check as kc

pytestmark = pytest.mark.gpu

CASES = {
    "mmfb_gemm": ["test_gemm_epilogues_poisoned", "test_gemm_split_k_workspace_poisoned", "test_gemm_bench_size_poisoned"],
    "mmfb_gemm_bounded": ["test_gemm_bounded_poisoned", "test_gemm_k_bounded_wgrad_poisoned"],
    "mmfb_attention_fwd": ["test_dense_attention_poisoned", "test_causal_attention_poisoned"],
    "mmfb_attention_bwd": ["test_dense_attention_poisoned", "test_causal_attention_poisoned"],
    "mmfb_attention_probs": "test_attention_probs_poisoned",
    "mmfb_attention_varlen_fwd": "test_varlen_attention_poisoned",
    "mmfb_attention_varlen_bwd": "test_varlen_attention_poisoned",
    "mmfb_attention_varlen_causal_fwd": "test_varlen_attention_poisoned",
    "mmfb_attention_varlen_causal_bwd": "test_varlen_attention_poisoned",
    "mmfb_attention_varlen_cross_fwd": "test_varlen_cross_attention_poisoned",
    "mmfb_attention_varlen_cross_bwd": "test_varlen_cross_attention_poisoned",
    "mmfb_layernorm_fwd": "test_layernorm_poisoned",
    "mmfb_layernorm_bwd": "test_layernorm_poisoned",
    "mmfb_layernorm_fwd_bounded": "test_layernorm_poisoned",
    "mmfb_layernorm_bwd_bounded": "test_layernorm_poisoned",
    "mmfb_colsum": "test_colsum_poisoned",
    "mmfb_colsum_ordered": "test_colsum_poisoned",
    "mmfb_colsum_bounded": "test_colsum_poisoned",
    "mmfb_ce_rows": "test_ce_rows_poisoned",
    "mmfb_ce_rows_bounded": "test_ce_rows_poisoned",
    "mmfb_kl_rows_bounded": "test_region_rows_poisoned",
    "mmfb_mse_rows_bounded": "test_region_rows_poisoned",
    "mmfb_select_rows": "test_select_and_gather_rows_poisoned",
    "mmfb_gather_rows": "test_select_and_gather_rows_poisoned",
    "mmfb_embed_compose": "test_embed_compose_poisoned",
    "mmfb_embed_scatter": "test_embed_scatter_poisoned",
    "mmfb_embed_scatter_sorted": "test_embed_scatter_sorted_poisoned",
    "mmfb_embed_scatter_sorted_ordered": "test_embed_scatter_sorted_poisoned",
    "mmfb_dropout_apply": "test_dropout_apply_poisoned",
    "mmfb_dropout_bits": "test_dropout_bits_poisoned",
    "mmfb_dropout_bits_epoch": "test_dropout_bits_poisoned",
    "mmfb_dropout_path_bits": "test_dropout_bits_poisoned",
    "mmfb_dropout_path_bits_epoch": "test_dropout_bits_poisoned",
    "mmfb_relu_bwd": "test_elementwise_poisoned",
    "mmfb_gelu_bwd": "test_elementwise_poisoned",
    "mmfb_add_bf16": "test_elementwise_poisoned",
    "mmfb_cast_f32_bf16": "test_elementwise_poisoned",
    "mmfb_adamw": "test_adamw_poisoned",
    "mmfb_adamw_hparams": "test_adamw_hparams_and_segments_poisoned",
    "mmfb_adamw_segments": "test_adamw_hparams_and_segments_poisoned",
    "mmfb_grad_norm": "test_grad_norm_poisoned",
    "mmfb_ot_fwd": "covered by tests/test_ot_gpu.py, which puts NaN in padded rows and guards its outputs",
    "mmfb_ot_bwd": "covered by tests/test_ot_gpu.py, which puts NaN in padded rows and guards its outputs",
}

DEV = "cuda"
NAN = G.NAN
ROWS_BEFORE, ROWS_AFTER, SLACK = 2, 3, 8      # guard rows before / after every 2-D view, and slack columns past it


class Bufs:
    """The buffers of one call: tight (guarded=False) or inside guarded allocations (guarded=True)."""

    def __init__(self, guarded):
        self.guarded = guarded
        self.guards = []                          # (base, [views], fill)
        self.outs = []                            # float output views that must be finite

    def _put(self, shape, dtype, fill, flat, rows_after=ROWS_AFTER):
        if flat or len(shape) != 2:
            n = 1
            for s in shape:
                n *= int(s)
            v, base = G.embed((n,), dtype, rows_before=ROWS_BEFORE * 8, rows_after=rows_after * 8 + 5, fill=fill)
            v = v.view(tuple(shape))
        else:
            v, base = G.embed(tuple(shape), dtype, rows_before=ROWS_BEFORE, rows_after=rows_after, slack_cols=SLACK,
                              fill=fill)
        self.guards.append((base, [v], fill))
        return v

    def inp(self, t, fill=NAN, flat=False, rows_after=ROWS_AFTER):
        """an input: a copy of t, tight or inside an allocation whose other elements hold `fill` (NaN by default)"""
        if not self.guarded:
            return t.clone().contiguous()
        if fill is NAN and not t.dtype.is_floating_point:
            raise ValueError("an index or bit input needs an explicit, harmless fill")
        v = self._put(t.shape, t.dtype, fill, flat or t.dim() != 2, rows_after)
        v.copy_(t)
        return v

    def out(self, shape, dtype, init=None, flat=False, finite=True):
        """an output inside a sentinel-filled allocation.  init=None: a pure output, whose guarded view starts at the
        sentinel as well (the tight one at zero), so an element the kernel leaves unwritten differs; a number or a
        tensor: an in-place operand, or rows the contract keeps as they were, starting at that value in both runs"""
        if not self.guarded:
            v = torch.zeros(tuple(shape), dtype=dtype, device=DEV)
        else:
            v = self._put(shape, dtype, None, flat or len(shape) != 2)
            if init is None:
                _bits(v).fill_(G.fill_bits(dtype))
        if isinstance(init, (int, float)):
            v.fill_(init)
        elif init is not None:
            v.copy_(init)
        if finite:
            self.outs.append(v)
        return v

    def check(self, what):
        torch.cuda.synchronize()
        for base, views, fill in self.guards:
            G.untouched(base, *views, fill=fill, what=what)
        for v in self.outs:
            G.assert_finite(v, what)


def _bits(t):
    t = t.detach()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def poisoned_equals_tight(run, what):
    """run(bufs) -> {name: output view}; the guarded call must equal the tight one bit for bit"""
    want = run(Bufs(False))
    torch.cuda.synchronize()
    bufs = Bufs(True)
    got = run(bufs)
    bufs.check(what)
    for k, w in want.items():
        g = got[k]
        assert g.shape == w.shape, (what, k)
        if not torch.equal(_bits(g), _bits(w)):
            bad = (_bits(g) != _bits(w)).nonzero()
            idx = tuple(int(i) for i in bad[0])
            raise AssertionError("%s: %s differs from the tight call at %d element(s); first at %s: %r, tight %r"
                                 % (what, k, bad.shape[0], idx, g[idx].item(), w[idx].item()))
    return got


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _bf16(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(torch.bfloat16)


def _words(*shape, g):
    return torch.randint(-2 ** 31, 2 ** 31, shape, generator=g, device=DEV, dtype=torch.int64).to(torch.int32)


def _lib():
    from mmf_b200 import lib
    return lib


def _stream():
    return _lib()._stream_ptr()


@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


@contextlib.contextmanager
def _guarded_workspace(bufs):
    """functional's ordered-reduction scratch, placed inside a sentinel-filled allocation of `bufs`"""
    from mmf_b200 import functional as F
    orig = F._workspace

    def ws(nbytes, device):
        if not bufs.guarded:
            return orig(nbytes, device)
        return bufs.out(((int(nbytes) + 3) // 4,), torch.float32, flat=True, finite=False)
    F._workspace = ws
    try:
        yield
    finally:
        F._workspace = orig


# ---------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("a_mn,b_mn,epi", [(0, 0, 0), (0, 0, 1), (0, 0, 2), (0, 0, 6), (0, 1, 0), (0, 1, 3), (0, 1, 4),
                                           (1, 1, 5), (1, 0, 0), (1, 1, 0), (0, 0, 7), (0, 1, 8)])
def test_gemm_epilogues_poisoned(a_mn, b_mn, epi, bn):
    """every epilogue with every (a_mn, b_mn) dispatch() accepts, on the M / N / K tails of test_gemm_edges_gpu.py, with
    NaN around A, B (rows past K for MN-major operands), bias and aux, all-ones keep-bit slack, and C / C2 guarded"""
    import test_gemm_edges_gpu as GE
    Ms = GE.M_MN if a_mn else GE.M_ANY
    Ks = GE.K_FREE if (a_mn and b_mn) else GE.K_KMAJ
    for i, (M, N, K) in enumerate(zip(Ms, GE.N_ALL, Ks)):
        gd = Bufs(True)
        GE.run_and_check(a_mn, b_mn, epi, M, N, K, bn, seed=100 * i + epi, with_bias=(i % 3 != 2),
                         with_aux=(i % 4 != 3), guard=gd)
        gd.check("gemm a_mn=%d b_mn=%d epi=%d M=%d N=%d K=%d bn=%d" % (a_mn, b_mn, epi, M, N, K, bn))


@pytest.mark.parametrize("M,N,K", [(256, 264, 457), (64, 776, 65)])
def test_gemm_split_k_workspace_poisoned(M, N, K):
    """epilogue 5 with splits > 1, with vector reductions and with the ordered workspace, the workspace guarded"""
    import test_gemm_edges_gpu as GE
    for ordered in (False, True):
        gd = Bufs(True)
        with _deterministic(ordered), _guarded_workspace(gd):
            GE.run_and_check(1, 1, 5, M, N, K, 128, seed=K, splits=3, guard=gd)
        assert len(gd.guards) == (4 if ordered else 3), "the ordered call must use exactly one (guarded) workspace"
        gd.check("split-K M=%d N=%d K=%d ordered=%s" % (M, N, K, ordered))


def test_gemm_bench_size_poisoned():
    """one bench-sized call: the bert-base FFN input projection of 37 848 rows with its GELU output, both guarded"""
    import test_gemm_edges_gpu as GE
    gd = Bufs(True)
    GE.run_and_check(0, 0, 1, 37848 // 4, 3072, 768, 256, seed=5, guard=gd)
    gd.check("bench-size gemm")


def _rounded(b, M):
    return min(M, -(-b // 128) * 128)


@pytest.mark.parametrize("epi,a_mn,b_mn", [(0, 0, 0), (0, 0, 1), (1, 0, 0), (2, 0, 0), (3, 0, 1), (4, 0, 1)])
def test_gemm_bounded_poisoned(epi, a_mn, b_mn):
    """mmfb_gemm_bounded with an M bound: A, aux and the keep bits are NaN / all ones from the rounded bound on (their
    rows between the bound and the tile edge are zeros, as the header makes the caller keep them), C and C2 are guarded
    there, and rows below the bound equal the unbounded call on the first b rows"""
    from mmf_b200 import functional as F
    M, N, K = 300, 264, 136
    g = _gen(epi)
    a = _bf16(M, K, g=g, scale=0.5)
    b = _bf16(K, N, g=g, scale=0.5) if b_mn else _bf16(N, K, g=g, scale=0.5)
    bias = _bf16(N, g=g) if epi in (0, 1, 2) else None
    aux = _bf16(M, N, g=g) if epi in (2, 3, 4) else None
    words = _words(M, (N + 31) // 32, g=g) if epi == 2 else None
    kw = dict(b_mn=bool(b_mn), epi=epi, drop_scale=1.0 / 0.9)
    for bnd in (0, 1, 127, 129, M):
        r = _rounded(bnd, M)
        gd = Bufs(True)

        def staged(t, fill):
            """t with zeros in [bnd, r) and `fill` from r on (a copy inside a guarded allocation)"""
            s = t.clone()
            s[bnd:r] = 0
            s[r:] = fill
            return gd.inp(s, fill=fill)
        a_p = staged(a, NAN)
        aux_p = staged(aux, NAN) if aux is not None else None
        w_p = staged(words, -1) if words is not None else None
        b_p = gd.inp(b)
        bias_p = gd.inp(bias) if bias is not None else None
        out = gd.out((M, N), torch.bfloat16, init=torch.full((M, N), NAN, dtype=torch.bfloat16, device=DEV), finite=False)
        out2 = gd.out((M, N), torch.bfloat16, init=torch.full((M, N), NAN, dtype=torch.bfloat16, device=DEV),
                      finite=False) if epi == 1 else None
        F.gemm(a_p, b_p, bias=bias_p, aux=aux_p, drop_mask=w_p, out=out, out2=out2,
               m_bound=torch.tensor([bnd], dtype=torch.int32, device=DEV), **kw)
        gd.check("bounded gemm epi=%d bound=%d" % (epi, bnd))
        for o in [out] + ([out2] if out2 is not None else []):
            assert torch.isnan(o[r:].float()).all(), (epi, bnd, "rows past the rounded bound were written")
            G.assert_finite(o[:r], "bounded gemm epi=%d bound=%d" % (epi, bnd))
        if bnd:
            want = F.gemm(a[:bnd].contiguous(), b, bias=bias, aux=aux[:bnd].contiguous() if aux is not None else None,
                          drop_mask=words[:bnd].contiguous() if words is not None else None, **kw)
            want = want if isinstance(want, tuple) else (want,)
            for o, w in zip([out] + ([out2] if out2 is not None else []), want):
                assert torch.equal(_bits(o[:bnd]), _bits(w)), (epi, bnd)


def test_gemm_k_bounded_wgrad_poisoned():
    """the weight gradient of a static-rows head: EPI_ATOMIC_F32 with (1, 1) bounded on K (the row count), with and
    without an ordered workspace; operand rows past the rounded bound are NaN, rows between the bound and the k-block
    edge zeros, and the result equals the unbounded call on the first b rows"""
    from mmf_b200 import functional as F
    Kcap, M, N = 700, 264, 136
    g = _gen(11)
    x = _bf16(Kcap, M, g=g, scale=0.5)
    dy = _bf16(Kcap, N, g=g, scale=0.5)
    c0 = torch.randn(M, N, generator=g, device=DEV)
    for ordered in (False, True):
        for bnd in (0, 1, 63, 65, 640, Kcap):
            r = min(Kcap, -(-bnd // 64) * 64)
            gd = Bufs(True)

            def staged(t):
                s = t.clone()
                s[bnd:r] = 0
                s[r:] = NAN
                return gd.inp(s)
            splits = 3 if ordered else 1
            out = gd.out((M, N), torch.float32, init=c0)
            with _deterministic(ordered), _guarded_workspace(gd):
                F.gemm(staged(x), staged(dy), a_mn=True, b_mn=True, epi=_lib().EPI_ATOMIC_F32, out=out, splits=splits,
                       k_bound=torch.tensor([bnd], dtype=torch.int32, device=DEV))
                want = c0.clone()
                if bnd:
                    F.gemm(x[:bnd].contiguous(), dy[:bnd].contiguous(), a_mn=True, b_mn=True, epi=_lib().EPI_ATOMIC_F32,
                           out=want, splits=splits)
            gd.check("k-bounded wgrad ordered=%s bound=%d" % (ordered, bnd))
            if ordered or splits == 1:
                assert torch.equal(_bits(out), _bits(want)), (ordered, bnd)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def _attn_fields(a, o):
    """output / saved-state pointers of an AttnArgs from the dict o"""
    a.ctx, a.ldo, a.lse2 = o["ctx"].data_ptr(), o["ctx"].stride(0), o["lse2"].data_ptr()
    if o.get("ctx_lo") is not None:
        a.ctx_lo = o["ctx_lo"].data_ptr()
    if "dctx" in o:
        a.dctx, a.ld_dctx, a.delta = o["dctx"].data_ptr(), o["dctx"].stride(0), o["delta"].data_ptr()
        a.dq, a.ld_dq = o["dq"].data_ptr(), o["dq"].stride(0)
        a.dk, a.ld_dk = o["dk"].data_ptr(), o["dk"].stride(0)
        a.dv, a.ld_dv = o["dv"].data_ptr(), o["dv"].stride(0)


def _qkv(bufs, q, k, v, self_attn, cap_q=5, cap_kv=7):
    """q / k / v as column slices of fused buffers with NaN columns after v and NaN capacity rows past the last row"""
    W = q.shape[1]
    if self_attn:
        fused = bufs.inp(torch.cat([q, k, v], 1), rows_after=cap_q)
        return fused[:, :W], fused[:, W:2 * W], fused[:, 2 * W:]
    kv = bufs.inp(torch.cat([k, v], 1), rows_after=cap_kv)
    return bufs.inp(q, rows_after=cap_q), kv[:, :W], kv[:, W:]


def _attention_outputs(bufs, rows_q, rows_kv, W, heads, lse_shape, lse_finite=True):
    o = {"ctx": bufs.out((rows_q, W), torch.bfloat16), "ctx_lo": bufs.out((rows_q, W), torch.bfloat16, flat=True),
         "lse2": bufs.out(lse_shape, torch.float32, flat=True, finite=lse_finite)}
    o.update({"delta": bufs.out(lse_shape, torch.float32, flat=True, finite=False),
              "dq": bufs.out((rows_q, W), torch.bfloat16), "dk": bufs.out((rows_kv, W), torch.bfloat16),
              "dv": bufs.out((rows_kv, W), torch.bfloat16)})
    return o


def _dense_run(B, heads, Sq, Skv, d, seed, lens=None, p_drop=0.0, causal=0, inputs=None):
    """run(bufs) of one dense forward + backward through the C ABI with every buffer from bufs"""
    from mmf_b200 import functional as F
    lib = _lib()
    g = _gen(seed)
    W = heads * d
    q, k, v = _bf16(B * Sq, W, g=g, scale=0.8), _bf16(B * Skv, W, g=g, scale=0.8), _bf16(B * Skv, W, g=g, scale=0.8)
    mask = None
    if lens is not None:
        lt = torch.tensor(lens, device=DEV)
        mask = torch.where(torch.arange(Skv, device=DEV)[None] < lt[:, None], 0.0, -10000.0).float().contiguous()
    keep = words = None
    if p_drop:
        keep = torch.rand(B, heads, Sq, Skv, generator=g, device=DEV) >= p_drop
        words = F.pack_keep_bits(keep)
    dctx = _bf16(B * Sq, W, g=g)
    if inputs is not None:
        inputs.update(q=q, k=k, v=v, mask=mask, keep=keep, p_drop=p_drop, dctx=dctx, lo_used=True)

    def run(bufs):
        qq, kk, vv = _qkv(bufs, q, k, v, Sq == Skv)
        m = bufs.inp(mask, flat=True) if mask is not None else None
        w = bufs.inp(words, fill=-1, flat=True) if words is not None else None
        a = F._attn_args(qq, kk, vv, B, heads, Sq, Skv, m, w, 1.0 / (1.0 - p_drop), causal)
        o = _attention_outputs(bufs, B * Sq, B * Skv, W, heads, (B, heads, Sq))
        o["dctx"] = bufs.inp(dctx)
        _attn_fields(a, o)
        lib.check(lib.LIB.mmfb_attention_fwd(ctypes.byref(a), _stream()))
        lib.check(lib.LIB.mmfb_attention_bwd(ctypes.byref(a), _stream()))
        res = {k_: o[k_] for k_ in ("ctx", "ctx_lo", "lse2", "dq", "dk", "dv")}
        if not causal:                             # mmfb_attention_probs refuses a causal tail
            res["probs"] = bufs.out((B, heads, Sq, Skv), torch.float32, flat=True)
            lib.check(lib.LIB.mmfb_attention_probs(ctypes.byref(a), res["probs"].data_ptr(), lib.MMFB_PROBS_F32,
                                                   _stream()))
        return res
    return run


# the SELF / CROSS shapes of tests/test_attention_edges_gpu.py's sweeps: (B, heads, Sq, Skv, d, key lengths, p_drop)
DENSE = [(2, 3, 65, 65, 64, [65, 1], 0.1), (1, 2, 129, 129, 128, None, 0.0), (3, 2, 1, 200, 64, [200, 7, 33], 0.1),
         (2, 1, 130, 17, 128, [17, 1], 0.0), (2, 2, 384, 384, 64, [384, 100], 0.1)]


@pytest.mark.parametrize("B,heads,Sq,Skv,d,lens,p_drop", DENSE)
def test_dense_attention_poisoned(B, heads, Sq, Skv, d, lens, p_drop):
    """dense self and cross attention with fused q/k/v slices, NaN columns after v, NaN capacity rows, the mask in a NaN
    guard and keep-bit slack: ctx, ctx_lo, lse2, delta, dq / dk / dv and probs guarded, and against fp64"""
    import test_attention_edges_gpu as AE
    inp = {}
    run = _dense_run(B, heads, Sq, Skv, d, seed=Sq + Skv, lens=lens, p_drop=p_drop, inputs=inp)
    got = poisoned_equals_tight(run, "dense attention %s" % ((B, heads, Sq, Skv, d),))
    ref = AE.reference(inp, B, heads, Sq, Skv)
    AE._check_all(got, ref, B, heads, Sq, Skv, d, "poisoned dense attention")


def test_dense_attention_bench_size_poisoned():
    """one bench-sized case: 16 samples of 228 tokens, 12 heads of 64"""
    poisoned_equals_tight(_dense_run(16, 12, 228, 228, 64, seed=1, lens=[228 - 7 * i for i in range(16)], p_drop=0.1),
                          "bench-size attention")


@pytest.mark.parametrize("S,d,T", [(13, 64, 5), (65, 64, 30), (200, 128, 64)])
def test_causal_attention_poisoned(S, d, T):
    poisoned_equals_tight(_dense_run(2, 2, S, S, d, seed=S, lens=[S, S - 3], p_drop=0.1, causal=T),
                          "causal attention S=%d d=%d T=%d" % (S, d, T))


@pytest.mark.parametrize("d", [64, 128])
def test_attention_probs_poisoned(d):
    """mmfb_attention_probs reads the forward's q, k, mask, lse2 and keep bits from guarded buffers"""
    poisoned_equals_tight(_dense_run(2, 3, 65, 129, d, seed=d, lens=[129, 64], p_drop=0.2), "attention probs d=%d" % d)


def _cu(lens):
    c = [0]
    for n in lens:
        c.append(c[-1] + n)
    return torch.tensor(c, dtype=torch.int32, device=DEV)


def _varlen_run(lens_q, lens_kv, heads, d, seed, p_drop, causal=0, cross=False):
    from mmf_b200 import functional as F
    lib = _lib()
    g = _gen(seed)
    W = heads * d
    tq, tk = sum(lens_q), sum(lens_kv)
    mq, mk = max(lens_q + [1]), max(lens_kv + [1])
    q, k, v = _bf16(tq, W, g=g, scale=0.8), _bf16(tk, W, g=g, scale=0.8), _bf16(tk, W, g=g, scale=0.8)
    words = _words(heads, tq, (mk + 31) // 32, g=g) if p_drop else None
    dctx = _bf16(tq, W, g=g)
    cu_q, cu_kv = _cu(lens_q), _cu(lens_kv)

    def run(bufs):
        qq, kk, vv = _qkv(bufs, q, k, v, not cross)
        w = bufs.inp(words, fill=-1, flat=True) if words is not None else None
        # cu_seqlens slack: a valid offset (the total), never an address past the rows
        cq = bufs.inp(cu_q, fill=tq, flat=True)
        if cross:
            ck = bufs.inp(cu_kv, fill=tk, flat=True)
            a, _, _, _ = F._varlen_cross_args(qq, kk, vv, cq, ck, mq, mk, heads, w, 1.0 / (1.0 - p_drop))
        else:
            a, _, _ = F._varlen_args(qq, kk, vv, cq, mq, heads, w, 1.0 / (1.0 - p_drop), causal)
        o = _attention_outputs(bufs, tq, tk, W, heads, (heads, tq), lse_finite=not cross or min(lens_kv) > 0)
        o["dctx"] = bufs.inp(dctx)
        _attn_fields(a, o)
        if cross:
            lib.check(lib.LIB.mmfb_attention_varlen_cross_fwd(ctypes.byref(a), cq.data_ptr(), tq, ck.data_ptr(), tk,
                                                              _stream()))
            lib.check(lib.LIB.mmfb_attention_varlen_cross_bwd(ctypes.byref(a), cq.data_ptr(), tq, ck.data_ptr(), tk,
                                                              _stream()))
        else:
            fw = lib.LIB.mmfb_attention_varlen_causal_fwd if causal else lib.LIB.mmfb_attention_varlen_fwd
            bw = lib.LIB.mmfb_attention_varlen_causal_bwd if causal else lib.LIB.mmfb_attention_varlen_bwd
            lib.check(fw(ctypes.byref(a), cq.data_ptr(), tq, _stream()))
            lib.check(bw(ctypes.byref(a), cq.data_ptr(), tq, _stream()))
        return {k_: o[k_] for k_ in ("ctx", "ctx_lo", "lse2", "dq", "dk", "dv")}
    return run


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("causal", [0, 12])
def test_varlen_attention_poisoned(d, causal):
    lens = [65, 1, 0, 128, 37] if d == 64 else [129, 7, 0, 64]
    poisoned_equals_tight(_varlen_run(lens, lens, 2, d, seed=d + causal, p_drop=0.1, causal=causal),
                          "varlen attention d=%d causal=%d" % (d, causal))


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kind", ["ragged", "keys_without_queries", "queries_without_keys", "no_queries"])
def test_varlen_cross_attention_poisoned(d, kind):
    """packed cross-attention, including a sample that has keys but no queries (its dk / dv rows must be written) and a
    whole empty query side"""
    lq, lk = {"ragged": ([65, 1, 30], [100, 17, 1]), "keys_without_queries": ([40, 0, 9], [33, 50, 70]),
              "queries_without_keys": ([40, 12, 9], [33, 0, 70]), "no_queries": ([0, 0], [20, 65])}[kind]
    poisoned_equals_tight(_varlen_run(lq, lk, 2, d, seed=d, p_drop=0.1, cross=True),
                          "varlen cross d=%d %s" % (d, kind))


# ---------------------------------------------------------------------------------------------------------------------
# row kernels
# ---------------------------------------------------------------------------------------------------------------------
def _bound_t(b):
    return torch.tensor([b], dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("H", [768, 1032])
@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("ordered", [False, True])
def test_layernorm_poisoned(H, bounded, ordered):
    """forward and backward, bounded and not, ordered and not: y is inf outside its view (the kernel squares it), dx, dx2,
    mean, rstd are NaN there, keep bits all ones; x, mean, rstd, dy, dz, the parameter sums and the workspace guarded.
    Bounded: the rows at and past the bound, which the header says are neither read nor written, hold the same poison
    inside the views, and the output rows there start at zero and must stay zero"""
    from mmf_b200 import functional as F
    lib = _lib()
    M = 300
    g = _gen(H)
    y = (torch.randn(M, H, generator=g, device=DEV) * 2 + 0.3).to(torch.bfloat16)
    gam, bet = (1 + 0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16), _bf16(H, g=g, scale=0.1)
    dx, dx2 = _bf16(M, H, g=g), _bf16(M, H, g=g)
    words = _words(M, (H + 31) // 32, g=g)
    sums0 = torch.randint(-8, 8, (3, H), generator=g, device=DEV).float()
    def past(t, b, value):
        t = t.clone()
        t[b:] = value
        return t
    for bnd in ((0, 129, M) if bounded else (None,)):
        b0 = M if bnd is None else bnd
        keep = None if bnd is None else 0
        y_p, dx_p, dx2_p, w_p = past(y, b0, float("inf")), past(dx, b0, NAN), past(dx2, b0, NAN), past(words, b0, -1)

        def run(bufs):
            yy = bufs.inp(y_p, fill=float("inf"))
            a = lib.LnArgs()
            x = bufs.out((M, H), torch.bfloat16, init=keep)
            mean, rstd = bufs.out((M,), torch.float32, init=keep), bufs.out((M,), torch.float32, init=keep)
            w = bufs.inp(w_p, fill=-1)
            gg, bb = bufs.inp(gam), bufs.inp(bet)
            a.y, a.ldy, a.gamma, a.beta = yy.data_ptr(), yy.stride(0), gg.data_ptr(), bb.data_ptr()
            a.x, a.ldx, a.mean, a.rstd = x.data_ptr(), x.stride(0), mean.data_ptr(), rstd.data_ptr()
            a.eps, a.M, a.H = 1e-12, M, H
            mb = _bound_t(bnd) if bnd is not None else None
            lib.check(lib.LIB.mmfb_layernorm_fwd_bounded(ctypes.byref(a), mb.data_ptr(), _stream()) if mb is not None
                      else lib.LIB.mmfb_layernorm_fwd(ctypes.byref(a), _stream()))
            # backward from the saved statistics, re-read through poisoned copies
            b = lib.LnArgs()
            m2, r2 = bufs.inp(past(mean, b0, NAN), flat=True), bufs.inp(past(rstd, b0, NAN), flat=True)
            ddx, ddx2 = bufs.inp(dx_p), bufs.inp(dx2_p)
            dy, dz = bufs.out((M, H), torch.bfloat16, init=keep), bufs.out((M, H), torch.bfloat16, init=keep)
            sums = bufs.out((3, H), torch.float32, init=sums0)
            b.y, b.ldy, b.gamma, b.mean, b.rstd = yy.data_ptr(), yy.stride(0), gg.data_ptr(), m2.data_ptr(), r2.data_ptr()
            b.dx, b.lddx, b.dx2, b.lddx2 = ddx.data_ptr(), ddx.stride(0), ddx2.data_ptr(), ddx2.stride(0)
            b.dy, b.lddy, b.dz, b.lddz = dy.data_ptr(), dy.stride(0), dz.data_ptr(), dz.stride(0)
            b.drop_mask, b.ldmask, b.drop_scale = w.data_ptr(), w.stride(0), 1.0 / 0.9
            b.dgamma, b.dbeta, b.dbias = sums[0].data_ptr(), sums[1].data_ptr(), sums[2].data_ptr()
            b.M, b.H = M, H
            if ordered:
                nbytes = lib.LIB.mmfb_layernorm_bwd_workspace_bytes(M, H)
                ws = bufs.out(((nbytes + 3) // 4,), torch.float32, flat=True, finite=False)
                b.workspace, b.workspace_bytes = ws.data_ptr(), nbytes
            lib.check(lib.LIB.mmfb_layernorm_bwd_bounded(ctypes.byref(b), mb.data_ptr(), _stream()) if mb is not None
                      else lib.LIB.mmfb_layernorm_bwd(ctypes.byref(b), _stream()))
            out = {"x": x, "mean": mean, "rstd": rstd, "dy": dy, "dz": dz}
            if ordered:
                out["sums"] = sums
            return out
        got = poisoned_equals_tight(run, "layernorm H=%d bound=%s ordered=%s" % (H, bnd, ordered))
        if bnd is None:
            fw = kc.layernorm_ref(y, gam, bet)
            kc.assert_within(got["x"], fw["x"], fw["b_x"], kc.row_layout(), "poisoned layernorm x")


@pytest.mark.parametrize("M,N", [(1, 8), (129, 776), (1000, 2304)])
def test_colsum_poisoned(M, N):
    """colsum, ordered colsum and bounded colsum on exact small integers: X NaN outside its view, out and the ordered
    workspace guarded; out must equal the exact sum (so the atomic order does not matter)"""
    from mmf_b200 import functional as F
    lib = _lib()
    g = _gen(M + N)
    x = kc.exact_ints(M, N, gen=g, device=DEV)
    out0 = kc.exact_ints(N, gen=g, device=DEV).float()
    for mode in ("plain", "ordered", "bounded", "bounded_ordered"):
        for bnd in ((M // 2, M) if mode.startswith("bounded") else (M,)):
            bufs = Bufs(True)
            xx = bufs.inp(x)
            out = bufs.out((N,), torch.float32, init=out0)
            nbytes = lib.LIB.mmfb_colsum_workspace_bytes(M, N)
            ws = bufs.out(((nbytes + 3) // 4,), torch.float32, flat=True, finite=False)
            if mode == "plain":
                lib.check(lib.LIB.mmfb_colsum(xx.data_ptr(), xx.stride(0), out.data_ptr(), M, N, _stream()))
            elif mode == "ordered":
                lib.check(lib.LIB.mmfb_colsum_ordered(xx.data_ptr(), xx.stride(0), out.data_ptr(), M, N, ws.data_ptr(),
                                                      nbytes, _stream()))
            else:
                o = mode == "bounded_ordered"
                lib.check(lib.LIB.mmfb_colsum_bounded(xx.data_ptr(), xx.stride(0), out.data_ptr(), M, N,
                                                      _bound_t(bnd).data_ptr(), ws.data_ptr() if o else None,
                                                      nbytes if o else 0, _stream()))
            bufs.check("colsum %s M=%d N=%d" % (mode, M, N))
            kc.assert_equal(out, out0.double() + x[:bnd].double().sum(0), kc.colsum_layout(), "colsum " + mode)


@pytest.mark.parametrize("V", [8, 1000, 30528])
def test_ce_rows_poisoned(V):
    """ce_rows and ce_rows_bounded in place: the logits' slack columns and rows past M are NaN, label slack holds a valid
    label, row_loss guarded; rows past the rounded bound of the bounded call keep their (NaN-free) values"""
    lib = _lib()
    M = 300
    g = _gen(V)
    z = _bf16(M, V, g=g, scale=2.0)
    labels = torch.randint(0, V, (M,), generator=g, device=DEV)
    labels[::3] = -1
    for bnd in (None, 0, 1, 129):
        lab = labels.clone()
        if bnd is not None:
            lab[bnd:_rounded(bnd, M)] = -1                 # the header: rows up to the tile edge carry ignore_index

        def run(bufs):
            zz = bufs.out((M, V), torch.bfloat16, init=z)
            ll = bufs.inp(lab, fill=V - 1, flat=True)
            rl = bufs.out((M,), torch.float32, init=None if bnd is None else 0)   # rows past the rounded bound: kept
            if bnd is None:
                lib.check(lib.LIB.mmfb_ce_rows(zz.data_ptr(), zz.stride(0), ll.data_ptr(), -1, M, V, 0.5, None,
                                               rl.data_ptr(), _stream()))
            else:
                sc = bufs.inp(torch.tensor([0.5], device=DEV), flat=True)
                lib.check(lib.LIB.mmfb_ce_rows_bounded(zz.data_ptr(), zz.stride(0), ll.data_ptr(), -1, M, V,
                                                       _bound_t(bnd).data_ptr(), sc.data_ptr(), None, rl.data_ptr(),
                                                       _stream()))
            return {"dz": zz, "row_loss": rl}
        got = poisoned_equals_tight(run, "ce_rows V=%d bound=%s" % (V, bnd))
        if bnd is not None:
            r = _rounded(bnd, M)
            assert torch.equal(got["dz"][r:], z[r:]), (V, bnd, "rows past the rounded bound changed")


@pytest.mark.parametrize("kind", ["kl", "mse"])
def test_region_rows_poisoned(kind):
    """kl_rows_bounded / mse_rows_bounded: padding columns [V, round8(V)) and rows past M NaN in the logits, targets NaN
    outside their rows, tgt_idx slack a valid row; row_loss guarded"""
    lib = _lib()
    M, V, T = 300, 1601, 50                       # V % 8 != 0: kl's padding columns [V, round8(V)) hold NaN
    cols = -(-V // 8) * 8 if kind == "kl" else 600
    D = V if kind == "kl" else cols
    g = _gen(7)
    z = _bf16(M, cols, g=g)
    if kind == "kl":
        z[:, V:] = NAN
    tgt = torch.softmax(torch.randn(T, D, generator=g, device=DEV), 1) if kind == "kl" else torch.randn(T, D, generator=g, device=DEV)
    idx = torch.randint(0, T, (M,), generator=g, device=DEV, dtype=torch.int64).to(torch.int32)
    for bnd in (0, 1, 129, M):
        def run(bufs):
            zz = bufs.out((M, cols), torch.bfloat16, init=z, finite=False)
            tt = bufs.inp(tgt)
            ii = bufs.inp(idx, fill=T - 1, flat=True)
            rl = bufs.out((M,), torch.float32, init=0)         # rows past the rounded bound are not written
            sc = bufs.inp(torch.tensor([1.0 / 64], device=DEV), flat=True)
            fn = lib.LIB.mmfb_kl_rows_bounded if kind == "kl" else lib.LIB.mmfb_mse_rows_bounded
            lib.check(fn(zz.data_ptr(), zz.stride(0), M, D, tt.data_ptr(), tt.stride(0), ii.data_ptr(),
                         _bound_t(bnd).data_ptr(), sc.data_ptr(), rl.data_ptr(), _stream()))
            return {"dz": zz, "row_loss": rl}
        got = poisoned_equals_tight(run, "%s_rows bound=%d" % (kind, bnd))
        r = _rounded(bnd, M)
        G.assert_finite(got["dz"][:r], "%s gradient rows below the rounded bound" % kind)


def test_select_and_gather_rows_poisoned():
    """select_rows with label slack holding a selected label, state and labels_out guarded; gather_rows with x NaN outside
    its rows and idx slack a valid row, in both directions (pos and inv)"""
    lib = _lib()
    M, H = 777, 264
    g = _gen(3)
    labels = torch.randint(0, 50, (M,), generator=g, device=DEV)
    labels[torch.rand(M, generator=g, device=DEV) < 0.8] = -1
    x = _bf16(M, H, g=g)

    def run(bufs):
        ll = bufs.inp(labels, fill=5, flat=True)
        state = bufs.out((2 + 2 * M,), torch.int32, flat=True)
        lo = bufs.out((M,), torch.int64, flat=True)
        lib.check(lib.LIB.mmfb_select_rows(ll.data_ptr(), -1, M, state.data_ptr(), lo.data_ptr(), _stream()))
        xx = bufs.inp(x)
        res = {"state": state, "labels": lo}
        for name, part in (("pos", state[2:2 + M]), ("inv", state[2 + M:])):
            idx = bufs.inp(part.clone(), fill=M - 1, flat=True)
            o = bufs.out((M, H), torch.bfloat16)
            lib.check(lib.LIB.mmfb_gather_rows(xx.data_ptr(), xx.stride(0), idx.data_ptr(), o.data_ptr(), o.stride(0), M,
                                               H, _stream()))
            res[name] = o
        return res
    got = poisoned_equals_tight(run, "select / gather rows")
    sel = (labels != -1).nonzero().flatten()
    assert int(got["state"][0]) == sel.numel()
    assert torch.equal(got["pos"][:sel.numel()], x[sel]) and not got["pos"][sel.numel():].any()


def test_embed_compose_poisoned():
    """two dense sources and three tables, sources and tables NaN outside their rows, index slack a valid row, y guarded;
    exact small integers, so y equals the fp64 sum"""
    from mmf_b200 import lib as L
    M, H, V = 300, 776, 40
    g = _gen(4)
    srcs = [kc.exact_ints(M + 5, H, gen=g, device=DEV) for _ in range(2)]
    tabs = [kc.exact_ints(V, H, gen=g, device=DEV) for _ in range(3)]
    idx = [torch.randint(-1, V, (M,), generator=g, device=DEV, dtype=torch.int64).to(torch.int32) for _ in range(5)]

    def run(bufs):
        a = L.ComposeArgs()
        keep = []
        for k in range(2):
            s, r = bufs.inp(srcs[k]), bufs.inp(idx[k], fill=0, flat=True)
            keep += [s, r]
            a.src[k], a.ldsrc[k], a.src_row[k] = s.data_ptr(), s.stride(0), r.data_ptr()
        for k in range(3):
            t, i = bufs.inp(tabs[k], flat=True), bufs.inp(idx[2 + k], fill=0, flat=True)
            keep += [t, i]
            a.tab[k], a.tab_idx[k] = t.data_ptr(), i.data_ptr()
        y = bufs.out((M, H), torch.bfloat16)
        a.y, a.ldy, a.M, a.H = y.data_ptr(), y.stride(0), M, H
        L.check(L.LIB.mmfb_embed_compose(ctypes.byref(a), _stream()))
        return {"y": y}
    got = poisoned_equals_tight(run, "embed_compose")
    ref, _ = kc.compose_ref(M, H, list(zip(srcs, idx[:2])), list(zip(tabs, idx[2:])), DEV)
    kc.assert_equal(got["y"], ref, kc.row_layout(), "poisoned compose")


def test_embed_scatter_poisoned():
    """dsrc rows stored and table rows accumulated: dy NaN outside its rows, index slack a valid row, dsrc / dtab
    guarded; exact small integers"""
    from mmf_b200 import lib as L
    M, H, V = 300, 776, 40
    g = _gen(5)
    dy = kc.exact_ints(M, H, gen=g, device=DEV)
    rows = torch.randperm(M + 9, generator=torch.Generator().manual_seed(1))[:M].to(DEV, torch.int32)
    tidx = torch.randint(-1, V, (M,), generator=g, device=DEV, dtype=torch.int64).to(torch.int32)
    dtab0 = kc.exact_ints(V, H, gen=g, device=DEV).float()

    def run(bufs):
        a = L.ScatterArgs()
        dd = bufs.inp(dy)
        r, i = bufs.inp(rows, fill=0, flat=True), bufs.inp(tidx, fill=0, flat=True)
        ds = bufs.out((M + 9, H), torch.bfloat16, init=0)          # only the indexed rows are stored
        dt = bufs.out((V, H), torch.float32, init=dtab0, flat=True)
        a.dsrc[0], a.ldsrc[0], a.src_row[0] = ds.data_ptr(), ds.stride(0), r.data_ptr()
        a.dtab[0], a.tab_idx[0] = dt.data_ptr(), i.data_ptr()
        a.dy, a.lddy, a.M, a.H = dd.data_ptr(), dd.stride(0), M, H
        L.check(L.LIB.mmfb_embed_scatter(ctypes.byref(a), _stream()))
        return {"dsrc": ds, "dtab": dt}
    got = poisoned_equals_tight(run, "embed_scatter")
    ref, _ = kc.scatter_table_ref(dtab0, dy, tidx)
    kc.assert_equal(got["dtab"], ref, kc.row_layout(), "poisoned scatter table")


@pytest.mark.parametrize("ordered", [False, True])
def test_embed_scatter_sorted_poisoned(ordered):
    """sorted scatter and its ordered variant: dy NaN outside its rows, order / sorted_idx slack valid, dtab and the
    workspace guarded; exact small integers"""
    from mmf_b200 import functional as F
    lib = _lib()
    M, H, V = 1001, 264, 30
    g = _gen(6)
    dy = kc.exact_ints(M, H, gen=g, device=DEV)
    idx = torch.randint(-1, V, (M,), generator=g, device=DEV, dtype=torch.int64).to(torch.int32)
    sidx, order = F.sort_indices(idx)
    dtab0 = kc.exact_ints(V, H, gen=g, device=DEV).float()

    def run(bufs):
        dd = bufs.inp(dy)
        si, od = bufs.inp(sidx, fill=V - 1, flat=True), bufs.inp(order, fill=0, flat=True)
        dt = bufs.out((V, H), torch.float32, init=dtab0, flat=True)
        if ordered:
            nbytes = lib.LIB.mmfb_embed_scatter_sorted_workspace_bytes(M, H)
            ws = bufs.out(((nbytes + 3) // 4,), torch.float32, flat=True, finite=False)
            lib.check(lib.LIB.mmfb_embed_scatter_sorted_ordered(dd.data_ptr(), dd.stride(0), od.data_ptr(), si.data_ptr(),
                                                                dt.data_ptr(), M, H, ws.data_ptr(), nbytes, _stream()))
        else:
            lib.check(lib.LIB.mmfb_embed_scatter_sorted(dd.data_ptr(), dd.stride(0), od.data_ptr(), si.data_ptr(),
                                                        dt.data_ptr(), M, H, _stream()))
        return {"dtab": dt}
    got = poisoned_equals_tight(run, "embed_scatter_sorted ordered=%s" % ordered)
    ref, _ = kc.scatter_table_ref(dtab0, dy, idx)
    kc.assert_equal(got["dtab"], ref, kc.scatter_sorted_layout(sidx), "poisoned sorted scatter")


@pytest.mark.parametrize("M,H", [(1, 8), (300, 328), (129, 776)])
def test_dropout_apply_poisoned(M, H):
    lib = _lib()
    g = _gen(M + H)
    x = _bf16(M, H, g=g)
    words = _words(M, (H + 31) // 32, g=g)

    def run(bufs):
        xx, w = bufs.inp(x), bufs.inp(words, fill=-1)
        o = bufs.out((M, H), torch.bfloat16)
        lib.check(lib.LIB.mmfb_dropout_apply(xx.data_ptr(), xx.stride(0), w.data_ptr(), w.stride(0), 1.0 / 0.9,
                                             o.data_ptr(), o.stride(0), M, H, _stream()))
        return {"out": o}
    poisoned_equals_tight(run, "dropout_apply M=%d H=%d" % (M, H))


def test_dropout_bits_poisoned():
    """the keep-bit generators leave the words past nwords (and before the buffer) untouched"""
    lib = _lib()
    epoch = torch.tensor([3], dtype=torch.int64, device=DEV)
    for nwords in (1, 7, 1001):
        def run(bufs):
            a, b = bufs.out((nwords,), torch.int32, flat=True), bufs.out((nwords,), torch.int32, flat=True)
            lib.check(lib.LIB.mmfb_dropout_bits(a.data_ptr(), nwords, 99, 64, 0.1, _stream()))
            lib.check(lib.LIB.mmfb_dropout_bits_epoch(b.data_ptr(), nwords, 99, 64, epoch.data_ptr(), 0.1, _stream()))
            return {"bits": a, "epoch": b}
        poisoned_equals_tight(run, "dropout_bits nwords=%d" % nwords)
    for B, S, H in ((3, 5, 40), (7, 197, 328)):
        def run(bufs):
            a, b = (bufs.out((B * S, (H + 31) // 32), torch.int32, flat=True) for _ in range(2))
            lib.check(lib.LIB.mmfb_dropout_path_bits(a.data_ptr(), B * S, H, S, 7, 4096, 0.1, 0.2, _stream()))
            lib.check(lib.LIB.mmfb_dropout_path_bits_epoch(b.data_ptr(), B * S, H, S, 7, 4096, epoch.data_ptr(), 0.1, 0.2,
                                                           _stream()))
            return {"path": a, "path_epoch": b}
        poisoned_equals_tight(run, "dropout_path_bits %s" % ((B, S, H),))


@pytest.mark.parametrize("n", [1, 7, 8, 2047, 2053])
def test_elementwise_poisoned(n):
    """relu_bwd, gelu_bwd, add and cast with n not a multiple of the 8-element vector: NaN around the inputs, the element
    after n (and before 0) guarded in every output"""
    lib = _lib()
    g = _gen(n)
    a, b = _bf16(n, g=g), _bf16(n, g=g)
    f = torch.randn(n, generator=g, device=DEV) * 3

    def run(bufs):
        aa, bb, ff = bufs.inp(a, flat=True), bufs.inp(b, flat=True), bufs.inp(f, flat=True)
        outs = {k: bufs.out((n,), torch.bfloat16, flat=True) for k in ("relu", "gelu", "add", "cast")}
        lib.check(lib.LIB.mmfb_relu_bwd(aa.data_ptr(), bb.data_ptr(), outs["relu"].data_ptr(), n, _stream()))
        lib.check(lib.LIB.mmfb_gelu_bwd(aa.data_ptr(), bb.data_ptr(), outs["gelu"].data_ptr(), n, _stream()))
        lib.check(lib.LIB.mmfb_add_bf16(aa.data_ptr(), bb.data_ptr(), outs["add"].data_ptr(), n, _stream()))
        lib.check(lib.LIB.mmfb_cast_f32_bf16(ff.data_ptr(), outs["cast"].data_ptr(), n, _stream()))
        return outs
    got = poisoned_equals_tight(run, "element-wise n=%d" % n)
    lay = kc.flat8_layout(n)
    kc.assert_bits_equal(got["add"], (a.double() + b.double()).to(torch.float32).to(torch.bfloat16), lay, "add")
    kc.assert_bits_equal(got["cast"], f.to(torch.bfloat16), lay, "cast")
    kc.assert_bits_equal(got["relu"], torch.where(b > 0, a, torch.zeros_like(a)), lay, "relu_bwd")
    ref, bound = kc.gelu_bwd_ref(a, b)
    kc.assert_within(got["gelu"], ref, bound, lay, "gelu_bwd")


# ---------------------------------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------------------------------
SEG_LENS = [1, 7, 2047, 2049, 5000]                # the last one crosses MMFB_ADAMW_SEGMENT_BLOCK more than once


def _flat_segments(lens, gap=13):
    """offsets of segments inside one flat buffer, separated by `gap` neighbour elements"""
    offs, o = [], gap
    for n in lens:
        offs.append(o)
        o += n + gap
    return offs, o


def test_adamw_poisoned():
    """mmfb_adamw over a flat buffer of 8-element blocks, embedded among neighbours: grad NaN, param / moments / bf16 copy
    sentinel-guarded"""
    from mmf_b200 import functional as F
    lib = _lib()
    n = 8 * 1001
    g = _gen(8)
    p, gr = torch.randn(n, generator=g, device=DEV), torch.randn(n, generator=g, device=DEV)
    m, v = torch.randn(n, generator=g, device=DEV) * 0.1, torch.rand(n, generator=g, device=DEV) * 0.01
    groups = [{"lr": 1e-3, "weight_decay": 0.01, "step_size": 1e-3, "bc2_sqrt": 0.3}]

    def run(bufs):
        pp, mm, vv = (bufs.out((n,), torch.float32, init=t, flat=True) for t in (p, m, v))
        gg = bufs.inp(gr, flat=True)
        pb = bufs.out((n,), torch.bfloat16, flat=True)
        F.adamw(pp, gg, mm, vv, groups, beta1=0.9, beta2=0.999, eps=1e-8, mode=1, param_bf16=pb)
        return {"p": pp, "m": mm, "v": vv, "pb": pb}
    poisoned_equals_tight(run, "adamw")


def test_adamw_hparams_and_segments_poisoned():
    """mmfb_adamw_hparams into a guarded table, then mmfb_adamw_segments on segments of lengths 1, 7, 2047, 2049 and one
    that crosses the segment block, cut out of one flat buffer whose neighbours are NaN in grad and sentinel in param /
    exp_avg / exp_avg_sq"""
    from mmf_b200 import functional as F
    lib = _lib()
    offs, total = _flat_segments(SEG_LENS)
    g = _gen(9)
    p, gr = torch.randn(total, generator=g, device=DEV), torch.randn(total, generator=g, device=DEV)
    m, v = torch.randn(total, generator=g, device=DEV) * 0.1, torch.rand(total, generator=g, device=DEV) * 0.01
    inside = torch.zeros(total, dtype=torch.bool, device=DEV)
    for o, n in zip(offs, SEG_LENS):
        inside[o:o + n] = True
    groups = torch.tensor([[1e-3, 0.01, 0.9, 0.999, 1e-8]], dtype=torch.float64, device=DEV)
    slots = F.adamw_slot_table([(0, lib.MMFB_ADAMW_SLOT_CORRECT_BIAS)], DEV)

    def run(bufs):
        # neighbours: grad NaN, param / moments the sentinel, all inside the same allocations as the segments
        gg = bufs.inp(torch.where(inside, gr, torch.full_like(gr, NAN)), flat=True)
        sent = torch.full((total,), 0, dtype=torch.int32, device=DEV).fill_(G.fill_bits(torch.float32)).view(torch.float32)
        pp, mm, vv = (bufs.out((total,), torch.float32, init=torch.where(inside, t, sent), flat=True, finite=False)
                      for t in (p, m, v))
        step = bufs.out((1,), torch.int64, init=torch.tensor([4], device=DEV), flat=True)
        hp = bufs.out((1, lib.ADAMW_HP_FLOATS), torch.float32, flat=True)
        F.adamw_hparams(groups, slots, step, hp, mode=0)
        table = F.adamw_segment_table([(pp[o:o + n], gg[o:o + n], mm[o:o + n], vv[o:o + n], 0)
                                       for o, n in zip(offs, SEG_LENS)])
        F.adamw_segments(table, hp, mode=0)
        torch.cuda.synchronize()
        for t in (pp, mm, vv):                     # the neighbours inside the flat buffers keep the sentinel
            assert torch.equal(_bits(t[~inside]), _bits(sent[~inside])), "adamw_segments wrote a neighbour"
            G.assert_finite(t[inside], "adamw_segments")
        return {"p": pp, "m": mm, "v": vv, "step": step, "hp": hp}
    poisoned_equals_tight(run, "adamw_hparams / adamw_segments")


def test_grad_norm_poisoned():
    """mmfb_grad_norm over segments of one flat buffer whose neighbours are NaN (fp32) and inf (bf16): the norm is the fp64
    norm of the segments alone; partials and out guarded"""
    from mmf_b200 import functional as F
    lib = _lib()
    lens = SEG_LENS + [16384 + 3]
    offs, total = _flat_segments(lens)
    g = _gen(10)
    for dtype, fill in ((torch.float32, NAN), (torch.bfloat16, float("inf"))):
        x = torch.randn(total, generator=g, device=DEV).to(dtype)
        inside = torch.zeros(total, dtype=torch.bool, device=DEV)
        for o, n in zip(offs, lens):
            inside[o:o + n] = True
        bufs = Bufs(True)
        xx = bufs.inp(torch.where(inside, x, torch.full_like(x, fill)), fill=fill, flat=True)
        table = F.grad_norm_table([xx[o:o + n] for o, n in zip(offs, lens)])
        out = bufs.out((2,), torch.float32, flat=True)
        partials = bufs.out((table.n_blocks,), torch.float64, flat=True)
        a = lib.GradNormArgs()
        a.segments, a.n_segments, a.n_blocks = table.segments.data_ptr(), table.n_segments, table.n_blocks
        a.partials, a.out, a.max_norm, a.norm_type = partials.data_ptr(), out.data_ptr(), 1.0, 2.0
        lib.check(lib.LIB.mmfb_grad_norm(ctypes.byref(a), _stream()))
        bufs.check("grad_norm %s" % dtype)
        want = x[inside].double().pow(2).sum().sqrt()
        # the header: the fp32 norm is within one fp32 ulp of the exact norm
        assert abs(out[0].double() - want) <= 2.0 ** -23 * want, (dtype, out[0].item(), want.item())
        coef = min(1.0, 1.0 / (out[0].item() + 1e-6))
        assert abs(out[1].item() - coef) <= 2.0 ** -22 * coef, (dtype, out[1].item(), coef)
