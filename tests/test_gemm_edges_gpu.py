"""wgmma GEMM at the edges it branches on, every element against fp64 (tests/kernel_check.py): M, N, K around the 64 /
128 / 256 tile edges, the free K of MN-major operands, bias / aux absent, a dropout mask with N % 32 != 0 and padded
rows, strided operand / output views, split counts the host clamps, and the large many-tile case per tile."""
import math

import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu

EPI_NAMES = {0: "bias", 1: "bias_gelu", 2: "bias_drop_resid", 3: "gelu_bwd", 4: "add_aux", 5: "atomic_f32", 6: "bias_relu",
             7: "bias_gelu_drop", 8: "gelu_drop_bwd"}
# every (a_mn, b_mn, epi) that dispatch() accepts
COMBOS = [(0, 0, 0), (0, 0, 1), (0, 0, 2), (0, 0, 6), (0, 1, 0), (0, 1, 3), (0, 1, 4), (1, 1, 5), (1, 0, 0), (1, 1, 0),
          (0, 0, 7), (0, 1, 8)]
# curated (M, N, K) lists: every M, N and K of the sweep appears, not their product
M_ANY = [1, 8, 63, 64, 65, 127, 129, 1000]
M_MN = [8, 64, 72, 120, 136, 1000, 8, 256]                # MN-major A needs M % 8 == 0
N_ALL = [8, 120, 136, 248, 264, 776, 136, 264]
K_KMAJ = [8, 56, 72, 136, 3072, 72, 8, 136]
K_FREE = [1, 7, 63, 65, 457, 8, 136, 3072]                 # both operands MN-major: K is a row count


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf16(*shape, g, scale=0.5):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _operand(rows, K, mn, g):
    t = _bf16(rows, K, g=g)
    if not mn:
        return t, t
    # a fresh [K, rows] buffer: .contiguous() of the transposed view would keep stride 1 on a size-1 dimension (K = 1)
    st = torch.empty(K, rows, device="cuda", dtype=torch.bfloat16)
    st.copy_(t.t())
    return st, t


def _effective_splits(splits, K):
    """the host's clamp (gemm.cu launch()): at most one split per k-block, and every split owns at least one"""
    kb = (K + 63) // 64
    s = min(max(splits, 1), kb)
    while s > 1 and ((kb + s - 1) // s) * (s - 1) >= kb:
        s -= 1
    return s


def run_and_check(a_mn, b_mn, epi, M, N, K, bn, seed, with_bias=True, with_aux=True, splits=1, guard=None):
    """one launch through functional.gemm and the per-element check of each output; returns the worst |err|/bound.
    guard (tests/test_poison_guard_gpu.py): places every operand inside a poisoned allocation (guard.inp) and every
    output inside a sentinel-filled one (guard.out), to be checked by the caller afterwards"""
    from mmf_b200 import functional as F, lib
    g = _gen(seed)
    a_st, a = _operand(M, K, a_mn, g)
    b_st, b = _operand(N, K, b_mn, g)
    acc, absab = kc.gemm_ref(a, b)
    bias = _bf16(N, g=g) if with_bias and epi in (0, 1, 2, 6, 7) else None
    aux = _bf16(M, N, g=g, scale=1.0) if (with_aux or epi == 8) and epi in (2, 3, 4, 8) else None
    bias64 = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device="cuda")
    aux64 = aux.double() if aux is not None else None
    words, keep, dsc = None, None, 1.0
    if epi in (2, 7, 8):
        wpr = (N + 31) // 32 + (3 if epi == 2 else 0)                     # ldmask > ceil(N/32) for epi 2
        words = torch.randint(-2 ** 31, 2 ** 31, (M, wpr), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
        keep = F.unpack_keep_bits(words, N).double()
        dsc = 1.0 / 0.9
    out = out2 = None
    if guard is not None:
        a_st, b_st = guard.inp(a_st), guard.inp(b_st)
        bias = guard.inp(bias) if bias is not None else None
        aux = guard.inp(aux) if aux is not None else None
        words = guard.inp(words, fill=-1) if words is not None else None
        if epi != 5:
            out = guard.out((M, N), torch.bfloat16)
            out2 = guard.out((M, N), torch.bfloat16) if epi in (1, 7) else None
    lay = kc.gemm_layout(bn, _effective_splits(splits, K) if epi == 5 else 1)
    tag = "a_mn=%d b_mn=%d epi=%s M=%d N=%d K=%d bn=%d" % (a_mn, b_mn, EPI_NAMES[epi], M, N, K, bn)
    worst = 0.0
    if epi == 5:
        c0 = torch.randn(M, N, generator=g, device="cuda")
        out = c0.clone() if guard is None else guard.out((M, N), torch.float32, init=c0)
        F.gemm(a_st, b_st, a_mn=True, b_mn=True, epi=epi, out=out, splits=splits, block_n=bn)
        ref = c0.double() + acc
        s_eff = _effective_splits(splits, K)
        # fp32 output: accumulation (2^-20 sum|a||b|), plus one rounded atomic add per split of a partial sum
        bound = kc.gemm_bound(ref, absab, c0.double().abs(), bf16_out=False) + kc.U_F32 * s_eff * (absab + ref.abs())
        return kc.assert_within(out, ref, bound, lay, tag)
    res = F.gemm(a_st, b_st, a_mn=bool(a_mn), b_mn=bool(b_mn), epi=epi, bias=bias, aux=aux, drop_mask=words,
                 drop_scale=dsc, block_n=bn, out=out, out2=out2)
    if epi in (0, 6):
        ref = acc + bias64
        bound = kc.gemm_bound(ref, absab, bias64.abs())
        if epi == 6:
            ref = ref.clamp_min(0.0)                                       # relu is 1-Lipschitz: same bound
        worst = kc.assert_within(res, ref, bound, lay, tag)
    elif epi == 1:
        u, h = res
        uref = acc + bias64
        s = absab + bias64.abs()
        worst = kc.assert_within(u, uref, kc.gemm_bound(uref, absab, bias64.abs()), lay, tag + " (u)")
        href = kc.gelu64(uref)
        # h = gelu(u) of the fp32 u: u's error through gelu', the erf approximation (|Phi err| <= 2^-22, times |u|),
        # fp32 arithmetic, bf16 rounding of h
        hb = (kc.U_BF16 * href.abs() + kc.gelu_grad64(uref).abs() * kc.U_ACC * s + 2.0 ** -22 * uref.abs()
              + kc.U_ACC * href.abs())
        worst = max(worst, kc.assert_within(h, href, hb, lay, tag + " (gelu)"))
    elif epi == 2:
        pre = (acc + bias64) * (keep * dsc if keep is not None else 1.0)
        ref = pre + (aux64 if aux64 is not None else 0.0)
        extra = (absab + bias64.abs()) * (keep * dsc if keep is not None else 1.0)
        # (acc + bias) * dscale and + aux each round in fp32 (2^-20 of their terms); bf16 output
        bound = kc.U_BF16 * ref.abs() + kc.U_ACC * (extra + (aux64.abs() if aux64 is not None else 0.0) + ref.abs())
        worst = kc.assert_within(res, ref, bound, lay, tag)
    elif epi == 3:
        gp = kc.gelu_grad64(aux64) if aux64 is not None else torch.ones_like(acc)
        ref = acc * gp
        # gelu'(x) in fp32 with the erf / ex2 approximations: |err| <= 2^-21 (1 + |x|)
        gerr = 2.0 ** -21 * (1 + aux64.abs()) if aux64 is not None else 0.0
        bound = kc.U_BF16 * ref.abs() + kc.U_ACC * (absab * gp.abs() + ref.abs()) + acc.abs() * gerr
        worst = kc.assert_within(res, ref, bound, lay, tag)
    elif epi == 4:
        ref = acc + (aux64 if aux64 is not None else 0.0)
        worst = kc.assert_within(res, ref, kc.gemm_bound(ref, absab, aux64.abs() if aux64 is not None else 0.0), lay, tag)
    elif epi == 7:
        # the bounds of tests/test_albef_vit_kernels_gpu.py::test_bias_gelu_drop_vs_fp64
        u, h = res
        uref = acc + bias64
        worst = kc.assert_within(u, uref, kc.gemm_bound(uref, absab, bias64.abs()), lay, tag + " (u)")
        kept = keep.bool()
        href = torch.where(kept, kc.gelu64(uref) * dsc, torch.zeros_like(uref))
        hb = kc.U_BF16 * href.abs() + dsc * (kc.gelu_grad64(uref).abs() * kc.U_ACC * (absab + bias64.abs())
                                             + 2.0 ** -22 * uref.abs() + kc.U_F32 * href.abs())
        worst = max(worst, kc.assert_within(h, href, torch.where(kept, hb, torch.zeros_like(hb)), lay, tag + " (h)"))
        assert torch.equal(h[~kept], torch.zeros_like(h[~kept])), tag
    elif epi == 8:
        # the bound of tests/test_albef_vit_kernels_gpu.py::test_gelu_drop_bwd_vs_fp64
        kept = keep.bool()
        gg = kc.gelu_grad64(aux64)
        ref = torch.where(kept, acc * dsc * gg, torch.zeros_like(acc))
        bound = kc.U_BF16 * ref.abs() + dsc * (gg.abs() * kc.U_ACC * absab + acc.abs() * 2.0 ** -21 * (1 + aux64.abs())
                                               + 2 * kc.U_F32 * (acc * gg).abs())
        worst = kc.assert_within(res, ref, torch.where(kept, bound, torch.zeros_like(bound)), lay, tag)
        assert torch.equal(res[~kept], torch.zeros_like(res[~kept])), tag
    return worst


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("a_mn,b_mn,epi", COMBOS)
def test_gemm_shape_edges(a_mn, b_mn, epi, bn):
    Ms = M_MN if a_mn else M_ANY
    Ks = K_FREE if (a_mn and b_mn) else K_KMAJ
    worst = 0.0
    for i, (M, N, K) in enumerate(zip(Ms, N_ALL, Ks)):
        worst = max(worst, run_and_check(a_mn, b_mn, epi, M, N, K, bn, seed=100 * i + epi, with_bias=(i % 3 != 2),
                                         with_aux=(i % 4 != 3)))
    print("gemm a_mn=%d b_mn=%d epi=%s bn=%d: worst |err|/bound %.3f" % (a_mn, b_mn, EPI_NAMES[epi], bn, worst))


@pytest.mark.parametrize("epi", [0, 1, 2, 6, 3, 4])
def test_gemm_without_bias_and_aux(epi):
    a_mn, b_mn = (0, 1) if epi in (3, 4) else (0, 0)
    run_and_check(a_mn, b_mn, epi, 129, 264, 136, 256, seed=7, with_bias=False, with_aux=False)


def test_gemm_dropout_mask_with_partial_words_and_padded_rows():
    for N, bn in ((264, 256), (776, 128), (40, 128)):
        run_and_check(0, 0, 2, 65, N, 72, bn, seed=N)


def test_gemm_strided_views():
    """A is a column slice of a [M, 3K] buffer, C and aux are column slices of wider buffers (ldc, ldaux > N); the
    columns of C's buffer outside the view keep their sentinel"""
    from mmf_b200 import functional as F, lib
    g = _gen(3)
    M, N, K = 129, 264, 136
    abuf = _bf16(M, 3 * K, g=g)
    a = abuf[:, K:2 * K]
    w = _bf16(N, K, g=g)
    bias = _bf16(N, g=g)
    auxbuf = _bf16(M, N + 24, g=g, scale=1.0)
    aux = auxbuf[:, 8:8 + N]
    acc, absab = kc.gemm_ref(a, w)
    for epi in (0, 2):
        cbuf = torch.full((M, N + 16), 7.0, device="cuda", dtype=torch.bfloat16)
        out = cbuf[:, 8:8 + N]
        F.gemm(a, w, epi=epi, bias=bias, aux=aux if epi == 2 else None, out=out)
        ref = acc + bias.double() + (aux.double() if epi == 2 else 0.0)
        extra = bias.double().abs() + (aux.double().abs() if epi == 2 else 0.0)
        kc.assert_within(out, ref, kc.gemm_bound(ref, absab, extra), kc.gemm_layout(256), "strided epi=%d" % epi)
        assert torch.equal(cbuf[:, :8], torch.full_like(cbuf[:, :8], 7.0))
        assert torch.equal(cbuf[:, 8 + N:], torch.full_like(cbuf[:, 8 + N:], 7.0))
    # MN-major B as a column slice (dgrad of a fused projection) and ldc > N
    wbuf = _bf16(K, 3 * N, g=g)
    wt = wbuf[:, N:2 * N]                                         # [K, N] MN-major
    acc2, absab2 = kc.gemm_ref(a, wt.t())
    cbuf = torch.zeros(M, N + 8, device="cuda", dtype=torch.bfloat16)
    F.gemm(a, wt, b_mn=True, epi=lib.EPI_ADD_AUX, aux=aux, out=cbuf[:, :N])
    ref = acc2 + aux.double()
    kc.assert_within(cbuf[:, :N], ref, kc.gemm_bound(ref, absab2, aux.double().abs()), kc.gemm_layout(256), "strided b_mn")


@pytest.mark.parametrize("M,N,K", [(256, 264, 457), (1000, 136, 3072 + 40), (64, 776, 65)])
def test_gemm_split_k_counts_the_host_clamps(M, N, K):
    kb = (K + 63) // 64
    for splits in sorted({1, 2, 3, kb, kb + 5}):
        run_and_check(1, 1, 5, M, N, K, 128, seed=splits, splits=splits)


def test_gemm_large_persistent_per_tile():
    """14592 x 3072 x 768 (1368 tiles of 128 x 256, 12 k-blocks each) and a smaller call right after, per element"""
    from mmf_b200 import functional as F, lib
    g = _gen(7)
    M, N, K = 14592, 3072, 768
    a, w = _bf16(M, K, g=g), _bf16(N, K, g=g)
    c = F.gemm(a, w, epi=lib.EPI_BIAS)
    ref, absab = kc.gemm_ref(a, w)
    kc.assert_within(c, ref, kc.gemm_bound(ref, absab), kc.gemm_layout(256), "14592x3072x768")
    c2 = F.gemm(a[:1000], w[:512], epi=lib.EPI_BIAS)
    kc.assert_within(c2, ref[:1000, :512], kc.gemm_bound(ref[:1000, :512], absab[:1000, :512]), kc.gemm_layout(256),
                     "1000x512x768 after")
