"""The column-sum, embedding, dropout, element-wise and AdamW kernels at their edges, every element against fp64
(tests/kernel_check.py): partial 256-column slabs up to H = 2048, row counts around the grids, strided views, exact
small-integer inputs for every kernel that sums (the output must then equal the fp64 sum), bit-exact element-wise
kernels at every tail length and on special values, dropout keep-bits against a numpy model of the Philox stream, and
the host-side refusal of misaligned rows."""
import math

import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _maker(exact, g):
    """(rows, cols) -> bf16 CUDA tensor: integers in [-16, 16] (exact sums) or normals"""
    if exact:
        return lambda r, c: kc.exact_ints(r, c, gen=g, device="cuda")
    return lambda r, c: torch.randn(r, c, generator=g, device="cuda").to(torch.bfloat16)


def _drop_some(idx, g, frac=0.2):
    idx[torch.rand(idx.shape[0], generator=g, device="cuda") < frac] = -1
    return idx


def _M(kind):
    return 8 * _sms() + 1 if kind == "8sm+1" else int(kind)


# ------------------------------------------------------------------------------------------------------------------
# embedding compose and scatter
# ------------------------------------------------------------------------------------------------------------------
# H: partial and full last slabs for every NV up to 8
EMB_H = [8, 72, 264, 520, 776, 1032, 2040, 2048]
EMB_M = ["1", "7", "9", "8sm+1"]
# (dense sources, table slots, all slots read one table at different row offsets as in the vision-language embeddings)
EMB_CFG = [(0, 1, False), (1, 0, False), (2, 3, True), (1, 2, False), (2, 0, False), (0, 3, True), (1, 3, False), (0, 0, False)]
V = 37


def _emb_indices(M, n_src, n_tab, shared, g):
    """dense-source rows (unique, 20 % absent) and table indices (20 % absent in every other slot)"""
    rows = []
    for k in range(n_src):
        r = torch.randperm(M + 3, generator=g, device="cuda")[:M].to(torch.int32)
        rows.append(_drop_some(r, g))
    idx = []
    for k in range(n_tab):
        lo, hi = (k * V, (k + 1) * V) if shared else (0, V + k)
        i = torch.randint(lo, hi, (M,), generator=g, device="cuda", dtype=torch.int32)
        idx.append(_drop_some(i, g) if k % 2 == 0 else i)
    return rows, idx


def _emb_case(H, M_kind):
    i, j = EMB_H.index(H), EMB_M.index(M_kind)
    n_src, n_tab, shared = EMB_CFG[(i + j) % len(EMB_CFG)]
    return _M(M_kind), n_src, n_tab, shared


@pytest.mark.parametrize("H", EMB_H)
@pytest.mark.parametrize("M_kind", EMB_M)
def test_embed_compose(H, M_kind):
    from mmf_b200 import functional as F
    M, n_src, n_tab, shared = _emb_case(H, M_kind)
    g = torch.Generator(device="cuda").manual_seed(M * 10000 + H)
    rows, idx = _emb_indices(M, n_src, n_tab, shared, g)
    tag = "compose M%d H%d src=%d tab=%d shared=%d" % (M, H, n_src, n_tab, shared)
    lay = kc.row_layout()
    worst = 0.0
    for exact in (True, False):
        make = _maker(exact, g)
        # the last dense source is a row slice of a wider buffer (ldsrc > H)
        srcs = [(make(M + 3, H + (8 if k == n_src - 1 else 0))[:, :H], rows[k]) for k in range(n_src)]
        if shared:
            big = make(3 * V, H)
            tabs = [(big, idx[k]) for k in range(n_tab)]
        else:
            tabs = [(make(V + k, H), idx[k]) for k in range(n_tab)]
        y = F.embed_compose(M, H, srcs=srcs, tabs=tabs, device="cuda")
        torch.cuda.synchronize()
        ref, bound = kc.compose_ref(M, H, srcs, tabs, "cuda")
        if exact:
            kc.assert_equal(y, ref, lay, tag + " exact")
        else:
            worst = kc.assert_within(y, ref, bound, lay, tag)
    print("%s: worst %.3g" % (tag, worst))


@pytest.mark.parametrize("H", EMB_H)
@pytest.mark.parametrize("M_kind", EMB_M)
def test_embed_scatter(H, M_kind):
    from mmf_b200 import functional as F
    M, n_src, n_tab, shared = _emb_case(H, M_kind)
    n_src, n_tab = max(n_src, 1), max(n_tab, 1)
    g = torch.Generator(device="cuda").manual_seed(M * 10000 + H + 1)
    rows, idx = _emb_indices(M, n_src, n_tab, shared, g)
    tag = "scatter M%d H%d src=%d tab=%d shared=%d" % (M, H, n_src, n_tab, shared)
    lay = kc.row_layout()
    sentinel = 0.5
    worst = 0.0
    for exact in (True, False):
        make = _maker(exact, g)
        dy = make(M, H + 8)[:, :H] if M % 2 else make(M, H)          # odd M: dy is a row slice (lddy > H)
        bufs = [torch.full((M + 3, H + 8 * k), sentinel, device="cuda", dtype=torch.bfloat16) for k in range(n_src)]
        dsrcs = [(bufs[k][:, :H], rows[k]) for k in range(n_src)]
        # the gradients accumulate into non-zero tables (integers for the exact run, fp32 normals otherwise)
        grad0 = (lambda r: kc.exact_ints(r, H, gen=g, device="cuda").float()) if exact else \
            (lambda r: torch.randn(r, H, generator=g, device="cuda"))
        dtab0 = [grad0(3 * V)] * n_tab if shared else [grad0(V + k) for k in range(n_tab)]
        dtabs = [t.clone() for t in dtab0[:1]] * n_tab if shared else [t.clone() for t in dtab0]
        F.embed_scatter(dy, dsrcs=dsrcs, dtabs=list(zip(dtabs, idx)))
        torch.cuda.synchronize()
        # dense sources: the rows of dy stored bit for bit; every other row and column keeps the sentinel
        for k in range(n_src):
            want = torch.full_like(bufs[k], sentinel)
            ok = rows[k] >= 0
            want[rows[k][ok].long(), :H] = dy[ok]
            kc.assert_bits_equal(bufs[k], want, lay, tag + " dsrc%d" % k)
        # tables: fp32 atomics (one gradient table for all slots when they share the table)
        slots = [(dtabs[0], dtab0[0], list(range(n_tab)))] if shared else [(dtabs[k], dtab0[k], [k]) for k in range(n_tab)]
        for out, t0, ks in slots:
            ref, bound = t0.double(), torch.zeros_like(t0, dtype=torch.float64)
            for k in ks:
                ref, b = kc.scatter_table_ref(ref, dy, idx[k])
                bound = bound + b
            if exact:
                kc.assert_equal(out, ref, lay, tag + " dtab%s exact" % ks)
            else:
                worst = max(worst, kc.assert_within(out, ref, bound, lay, tag + " dtab%s" % ks))
    print("%s: worst %.3g" % (tag, worst))


# ------------------------------------------------------------------------------------------------------------------
# sorted scatter (type / position / word table gradients)
# ------------------------------------------------------------------------------------------------------------------
SS_KIND = ["one", "runs", "distinct", "pad", "allpad"]
SS_M = [1, 31, 33, 8191]
SS_H = [8, 264, 520, 776, 1024]           # NV = 1..4 with partial last slabs, and a full one


def _sorted_pattern(kind, M, g):
    if kind == "one":                                    # all rows one index (token type ids)
        return torch.full((M,), 1, dtype=torch.int32)
    if kind == "distinct":
        return torch.arange(M, dtype=torch.int32)
    if kind == "allpad":
        return torch.full((M,), -1, dtype=torch.int32)
    if kind == "pad":                                    # a leading -1 run (padding_idx rows), then sorted indices
        lead = min(M, 40)
        rest = torch.sort(torch.randint(0, 50, (M - lead,), generator=g)).values
        return torch.cat([torch.full((lead,), -1, dtype=torch.int64), rest]).to(torch.int32)
    # runs of 31, 32, 33, 255, 256 and 257 that start 5 positions in, so each straddles a warp (32) or block (256) end
    lengths = [5, 31, 32, 33, 255, 256, 257]
    while sum(lengths) < M:
        lengths.append(int(torch.randint(1, 10, (1,), generator=g)))
    s = torch.cat([torch.full((n,), k, dtype=torch.int32) for k, n in enumerate(lengths)])
    return s[:M]


@pytest.mark.parametrize("kind", SS_KIND)
@pytest.mark.parametrize("M", SS_M)
def test_embed_scatter_sorted(kind, M):
    from mmf_b200 import functional as F
    H = SS_H[(SS_KIND.index(kind) + SS_M.index(M)) % len(SS_H)]
    g = torch.Generator().manual_seed(M * 10 + SS_KIND.index(kind))
    gc = torch.Generator(device="cuda").manual_seed(M * 10 + SS_KIND.index(kind))
    s = _sorted_pattern(kind, M, g)
    idx = torch.empty(M, dtype=torch.int32)
    idx[torch.randperm(M, generator=g)] = s
    idx = idx.cuda()
    sorted_idx, order = F.sort_indices(idx)
    assert torch.equal(sorted_idx.cpu(), s)
    nV = max(int(s.max()) + 3, 3)
    tag = "scatter_sorted %s M%d H%d" % (kind, M, H)
    lay = kc.scatter_sorted_layout(sorted_idx)
    worst = 0.0
    for exact in (True, False):
        make = _maker(exact, gc)
        dy = make(M, H + 16)[:, :H]                                   # a row slice (lddy > H)
        # accumulates into a non-zero gradient
        dtab0 = kc.exact_ints(nV, H, gen=gc, device="cuda").float() if exact else torch.randn(nV, H, generator=gc, device="cuda")
        dtab = dtab0.clone()
        F.embed_scatter_sorted(dy, dtab, sorted_idx, order)
        torch.cuda.synchronize()
        ref, bound = kc.scatter_table_ref(dtab0, dy, idx)
        if exact:
            kc.assert_equal(dtab, ref, lay, tag + " exact")
        else:
            worst = kc.assert_within(dtab, ref, bound, lay, tag)
    print("%s: worst %.3g" % (tag, worst))


def test_compose_ln_padding_rows_get_exactly_zero_gradient():
    """ops.compose_ln end to end: the padding_idx row of the word table is read in the forward and gets no gradient"""
    from mmf_b200 import ops
    M, H, Vw, P = 300, 264, 30, 64
    g = torch.Generator(device="cuda").manual_seed(11)
    word = torch.randn(Vw, H, generator=g, device="cuda").requires_grad_(True)
    pos = torch.randn(P, H, generator=g, device="cuda").requires_grad_(True)
    lw = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).requires_grad_(True)
    lb = (0.1 * torch.randn(H, generator=g, device="cuda")).requires_grad_(True)
    ids = torch.randint(1, Vw, (M,), generator=g, device="cuda")
    ids[:45] = 0                                          # a run of pads longer than one warp's 32 sorted positions
    ids[100::7] = 0
    out = ops.compose_ln(M, H, [], [(word, ops.i32(ids), 0), (pos, ops.i32(torch.arange(M, device="cuda") % P))], lw, lb)
    w = torch.randn(M, H, generator=g, device="cuda")
    (out.float() * w).sum().backward()
    torch.cuda.synchronize()
    assert torch.equal(word.grad[0], torch.zeros(H, device="cuda"))
    used = torch.unique(ids[ids != 0])
    assert bool((word.grad[used].abs().sum(1) > 0).all())
    assert bool((pos.grad.abs().sum(1) > 0).all())


# ------------------------------------------------------------------------------------------------------------------
# column sums (bias gradients)
# ------------------------------------------------------------------------------------------------------------------
CS_N = [8, 248, 264, 2056, 30528]
CS_M = ["1", "7", "63", "64", "65", "cap", "cap+1", "3cap+17"]


@pytest.mark.parametrize("N", CS_N)
@pytest.mark.parametrize("M_kind", CS_M)
def test_colsum(N, M_kind):
    """row counts around one row block (64), where grid.y reaches its cap (about 4 blocks per SM) and beyond it"""
    from mmf_b200 import functional as F
    sms = _sms()
    gx = (N + 255) // 256
    cap = (4 * sms + gx - 1) // gx
    M = {"cap": 64 * cap, "cap+1": 64 * cap + 1, "3cap+17": 3 * 64 * cap + 17}.get(M_kind) or int(M_kind)
    strided = (CS_N.index(N) + CS_M.index(M_kind)) % 2 == 1
    g = torch.Generator(device="cuda").manual_seed(M * 100 + N)
    tag = "colsum M%d N%d grid.y=%d ldx%s" % (M, N, kc.colsum_grid_y(M, N, sms), ">N" if strided else "=N")
    lay = kc.colsum_layout()
    worst = 0.0
    for exact in (True, False):
        make = _maker(exact, g)
        x = make(M, N + 8)[:, :N] if strided else make(M, N)
        out0 = kc.exact_ints(N, gen=g, device="cuda").float() if exact else torch.randn(N, generator=g, device="cuda")
        out = out0.clone()
        F.colsum(x, out)
        torch.cuda.synchronize()
        ref, bound = kc.colsum_ref(x, out0, sms)
        if exact:
            kc.assert_equal(out, ref, lay, tag + " exact")
        else:
            worst = kc.assert_within(out, ref, bound, lay, tag)
    print("%s: worst %.3g" % (tag, worst))


# ------------------------------------------------------------------------------------------------------------------
# dropout keep-bits
# ------------------------------------------------------------------------------------------------------------------
P_VALUES = [0.0, 2.0 ** -16, 0.1, 0.25, 1.0 / 3.0, 0.5, 0.75, 0.9, 1.0 - 2.0 ** -16, 0.99999]
# (seed, offset, epoch): both key words, counters that carry from the low into the high word (and wrap), the epoch
DROP_VARIANTS = [(7, 0, None), (2 ** 32 + 5, 2 ** 32 - 6, None), (0xFEDCBA9876543210, (1 << 40) + 3, 5),
                 (1, 2 ** 64 - 10, 1)]


def _with_epoch(epoch, fn):
    from mmf_b200 import functional as F
    dev = torch.cuda.current_device()
    saved = dict(F._DROPOUT_EPOCH)
    try:
        if epoch is not None:
            F._DROPOUT_EPOCH[dev] = torch.full((1,), epoch, dtype=torch.int64, device="cuda")
        else:
            F._DROPOUT_EPOCH.pop(dev, None)
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        F._DROPOUT_EPOCH.clear()
        F._DROPOUT_EPOCH.update(saved)


@pytest.mark.parametrize("p", P_VALUES)
def test_dropout_bits_equal_the_model(p):
    from mmf_b200 import functional as F
    t = kc.dropout_thresh16(p)
    ip = P_VALUES.index(p)
    for j, nwords in enumerate([1, 255, 256, 257, 65537]):
        seed, offset, epoch = DROP_VARIANTS[(ip + j) % len(DROP_VARIANTS)]
        words = _with_epoch(epoch, lambda: F.dropout_bits((1,), 32 * nwords, p, seed, offset, "cuda"))
        kc.assert_keep_bits(words, kc.dropout_uniforms(nwords, seed, offset, epoch or 0), p,
                            "dropout_bits p=%r nwords=%d seed=%#x offset=%#x epoch=%s" % (p, nwords, seed, offset, epoch))
    # independently of the model: the keep fraction of the large draw is within 5 binomial sigma of 1 - thresh16 / 2^16
    keep = F.unpack_keep_bits(words.reshape(-1), 32 * nwords).double()
    q = 1.0 - t / 65536.0
    sigma = math.sqrt(q * (1 - q) / keep.numel())
    frac = keep.mean().item()
    print("dropout_bits p=%r thresh16=%d keep fraction %.6f expected %.6f (%.2f sigma)"
          % (p, t, frac, q, abs(frac - q) / sigma if sigma else 0.0))
    assert abs(frac - q) <= 5 * sigma, (p, frac, q, sigma)


def test_dropout_state_draws_equal_the_model_at_disjoint_counters():
    from mmf_b200.engine import DropoutState
    off0 = 2 ** 33 + 4
    ds = DropoutState(seed=0x5EED0000ABCD, offset=off0)
    a = _with_epoch(None, lambda: ds.bits((37,), 100, 0.1, "cuda"))           # 4 words per row
    off1 = ds.offset
    assert off1 == off0 + 4 * 37 * 4
    b = _with_epoch(None, lambda: ds.bits((5, 3), 776, 0.25, "cuda"))         # 25 words per row
    assert ds.offset == off1 + 4 * 15 * 25
    kc.assert_keep_bits(a, kc.dropout_uniforms(a.numel(), ds.seed, off0), 0.1, "first draw")
    kc.assert_keep_bits(b, kc.dropout_uniforms(b.numel(), ds.seed, off1), 0.25, "second draw")


DA_H = [8, 40, 264, 520, 1000, 2040]


@pytest.mark.parametrize("H", DA_H)
@pytest.mark.parametrize("M", [1, 7, 9, 300])
def test_dropout_apply(H, M):
    """keep ? bf16(x * scale) : 0 in fp32, bit for bit; H % 32 != 0, x a row slice (ldx > H), keep words a slice of wider
    rows (ldm > ceil(H / 32))"""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(M * 10000 + H)
    W = (H + 31) // 32
    x = torch.randn(M, H + 16, generator=g, device="cuda").to(torch.bfloat16)[:, :H]
    x[0, :8] = torch.tensor([3.3e38, -3.3e38, 0.0, -0.0, float("inf"), float("nan"), 1e-40, -2.5], device="cuda").to(torch.bfloat16)
    words = (torch.randint(0, 2 ** 32, (M, W + 3), generator=g, device="cuda") - 2 ** 31).to(torch.int32)[:, :W]
    scale = 1.0 / (1.0 - 0.1)
    out = F.dropout_apply(x, words, scale)
    torch.cuda.synchronize()
    keep = F.unpack_keep_bits(words, H)
    kept = (x.float() * torch.tensor(scale, dtype=torch.float32, device="cuda")).to(torch.bfloat16)
    ref = torch.where(keep, kept, torch.zeros_like(kept))
    kc.assert_bits_equal(out, ref, kc.row_layout(), "dropout_apply M%d H%d" % (M, H))


# ------------------------------------------------------------------------------------------------------------------
# element-wise kernels: every tail length, the grid edge, special values
# ------------------------------------------------------------------------------------------------------------------
EW_N = [1, 2, 3, 4, 5, 6, 7, 8, 9, 2047, 2048, 2049, 3 * 2048 - 1, 3 * 2048 + 7, 5 * 2048 - 8, 5 * 2048 + 1]

BF16_SPECIAL = [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0xFFC1, 0x7F81, 0x0001, 0x8001, 0x007F, 0x0080, 0x807F, 0x7F7F,
                0xFF7F, 0x3F80, 0xBF80]
# pairs (a, b) whose fp32 sum is a bf16 tie (1 + 2^-8 to even, 1 + 3 2^-8 up), overflows to +-inf in bf16 (max + half
# an ulp), mixes denormals, gives -0 / +0 or NaN
ADD_SPECIAL = [(0x3F80, 0x3B80), (0x3F81, 0x3B80), (0x7F7F, 0x7B00), (0xFF7F, 0xFB00), (0x0001, 0x0001),
               (0x0001, 0x8001), (0x8000, 0x8000), (0x8000, 0x0000), (0x7F80, 0xFF80), (0x7FC0, 0x3F80),
               (0x0080, 0x8001), (0x7F7F, 0x7A80), (0x4B80, 0x3F80)]
# fp32 ties (to even down / up), just above a tie, rounding to +-inf and to the bf16 maximum, fp32 denormals that
# round to zero, to a bf16 denormal (ties included) or up to the smallest normal, signalling and quiet NaNs
F32_SPECIAL = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC00001, 0x3F808000,
               0x3F818000, 0x3F808001, 0x7F7F8000, 0x7F7F7FFF, 0xFF7F8000, 0x00000001, 0x00008000, 0x00018000,
               0x00010000, 0x807FFFFF, 0x00800000, 0x007F8000, 0x80008001]


def _as_signed(vals, bits):
    return [v - (1 << bits) if v >= 1 << (bits - 1) else v for v in vals]


def _special_mix(n, g, specials, bits):
    """random bit patterns; about half of the elements, and the whole scalar tail, replaced by special values"""
    dt = {16: torch.int16, 32: torch.int32}[bits]
    x = torch.randint(-(1 << (bits - 1)), 1 << (bits - 1), (n,), generator=g, dtype=torch.int64).to(dt)
    sel = torch.rand(n, generator=g) < 0.5
    sel[n - n % 8:] = True
    sp = torch.tensor(_as_signed(specials, bits), dtype=dt)
    x[sel] = sp[torch.randint(0, len(specials), (int(sel.sum()),), generator=g)]
    return x


@pytest.mark.parametrize("n", EW_N)
def test_relu_bwd_bit_exact(n):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(n)
    y = _special_mix(n, g, BF16_SPECIAL, 16).view(torch.bfloat16)
    dy = _special_mix(n, g, BF16_SPECIAL, 16).view(torch.bfloat16)
    dz = F.relu_bwd(dy.cuda(), y.cuda()).cpu()
    ref = torch.where(y.float() > 0, dy, torch.zeros_like(dy))
    kc.assert_bits_equal(dz, ref, kc.flat8_layout(n), "relu_bwd n=%d" % n)


@pytest.mark.parametrize("n", EW_N)
def test_add_bf16_bit_exact(n):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(n + 1)
    a = torch.randint(-32768, 32768, (n,), generator=g, dtype=torch.int64).to(torch.int16)
    b = torch.randint(-32768, 32768, (n,), generator=g, dtype=torch.int64).to(torch.int16)
    sel = torch.rand(n, generator=g) < 0.5
    sel[n - n % 8:] = True
    pick = torch.randint(0, len(ADD_SPECIAL), (int(sel.sum()),), generator=g)
    pa, pb = (torch.tensor(_as_signed([p[k] for p in ADD_SPECIAL], 16), dtype=torch.int16) for k in (0, 1))
    a[sel], b[sel] = pa[pick], pb[pick]
    a, b = a.view(torch.bfloat16), b.view(torch.bfloat16)
    out = F.add(a.cuda(), b.cuda()).cpu()
    ref = (a.float() + b.float()).to(torch.bfloat16)
    kc.assert_bits_equal(out, ref, kc.flat8_layout(n), "add_bf16 n=%d" % n)


@pytest.mark.parametrize("n", EW_N)
def test_cast_f32_bf16_bit_exact(n):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(n + 2)
    src = _special_mix(n, g, F32_SPECIAL, 32).view(torch.float32)
    dst = torch.full((n,), 7.0, dtype=torch.bfloat16, device="cuda")
    F.cast_f32_bf16(src.cuda(), dst)
    kc.assert_bits_equal(dst.cpu(), src.to(torch.bfloat16), kc.flat8_layout(n), "cast_f32_bf16 n=%d" % n)


@pytest.mark.parametrize("n", EW_N)
def test_gelu_bwd(n):
    """u from -20 to 20 (ex2.approx.ftz underflows to 0 beyond |u| ~ 13)"""
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(n + 3)
    u = torch.rand(n, generator=g, dtype=torch.float64) * 40 - 20
    fixed = torch.tensor([-20, -13.5, -13, -5, -0.75, 0, 0.75, 5, 13, 20], dtype=torch.float64)
    u[-min(n, 10):] = fixed[:min(n, 10)]
    u = u.to(torch.bfloat16)
    dh = torch.randn(n, generator=g).to(torch.bfloat16)
    du = F.gelu_bwd(dh.cuda(), u.cuda()).cpu()
    ref, bound = kc.gelu_bwd_ref(dh, u)
    worst = kc.assert_within(du, ref, bound, kc.flat8_layout(n), "gelu_bwd n=%d" % n)
    print("gelu_bwd n=%d: worst %.3g" % (n, worst))


# ------------------------------------------------------------------------------------------------------------------
# AdamW
# ------------------------------------------------------------------------------------------------------------------
GROUPS = [{"lr": 1e-3 * (i + 1), "weight_decay": 0.0 if i % 3 == 0 else 0.01 * i, "step_size": 9e-4 * (i + 1) * (1 + 0.1 * i),
           "bc2_sqrt": math.sqrt(1 - 0.999 ** (i + 2))} for i in range(8)]
HP = dict(beta1=0.9, beta2=0.999, eps=1e-6, grad_scale=0.5)


@pytest.mark.parametrize("mode", [0, 1])
def test_adamw_update_per_element(mode):
    """8 groups with distinct lr, weight decay (zero and not), step size and bias correction, a random group per
    8-element block, n / 8 not a multiple of the 256-thread block, grad_scale != 1, three steps"""
    from mmf_b200 import functional as F
    n = 8 * (3 * 256 + 37)
    g = torch.Generator(device="cuda").manual_seed(40 + mode)
    p = torch.randn(n, generator=g, device="cuda")
    m = torch.randn(n, generator=g, device="cuda") * 0.01
    v = torch.rand(n, generator=g, device="cuda") * 1e-4 + 1e-8
    gid = torch.randint(0, 8, (n // 8,), generator=g, device="cuda").to(torch.uint8)
    st = kc.adamw_state(p, m, v)
    lay = kc.adamw_layout(gid)
    worst = {}
    for step in range(3):
        grad = torch.randn(n, generator=g, device="cuda") * 0.1
        F.adamw(p, grad, m, v, GROUPS, mode=mode, group_of_block=gid, **HP)
        torch.cuda.synchronize()
        kc.adamw_step_ref(st, grad, GROUPS, gid, mode=mode, **HP)
        for name, t in (("p", p), ("m", m), ("v", v)):
            worst[name] = max(worst.get(name, 0.0),
                              kc.assert_within(t, st[name], st["e_" + name], lay, "adamw mode %d step %d %s" % (mode, step, name)))
    print("adamw mode %d: %s" % (mode, " ".join("%s=%.3g" % kv for kv in worst.items())))


# ------------------------------------------------------------------------------------------------------------------
# misaligned rows are refused before anything is launched
# ------------------------------------------------------------------------------------------------------------------
def test_row_kernels_reject_unaligned_rows():
    """colsum, compose, scatter, the sorted scatter and dropout_apply read rows as 16-byte vectors: a row stride that is
    not a multiple of 8 elements, or a base that is not 16-byte aligned, is refused with ValueError naming the tensor"""
    from mmf_b200 import functional as F, lib
    M, H, Vt = 64, 264, 5
    bad = torch.randn(M, H + 4, device="cuda").to(torch.bfloat16)[:, :H]                  # ld = H + 4
    flat = torch.randn(M * H + 8, device="cuda").to(torch.bfloat16)
    shifted = flat[1:1 + M * H].view(M, H)                                                 # base 2 bytes off
    good = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    rows = torch.arange(M, device="cuda", dtype=torch.int32)
    tidx = torch.zeros(M, device="cuda", dtype=torch.int32)
    tab_shifted = flat[1:1 + Vt * H].view(Vt, H)
    out = torch.zeros(H, device="cuda")
    dtab = torch.zeros(Vt, H, device="cuda")
    sorted_idx, order = F.sort_indices(tidx)
    words = torch.zeros(M, (H + 31) // 32, device="cuda", dtype=torch.int32)
    dsrc_bad = torch.zeros(M, H + 4, device="cuda", dtype=torch.bfloat16)[:, :H]
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    with pytest.raises(ValueError, match="colsum: ldx"):
        F.colsum(bad, out)
    with pytest.raises(ValueError, match="colsum: x must be 16-byte aligned"):
        F.colsum(shifted, out)
    with pytest.raises(ValueError, match="embed_compose: ldsrc0"):
        F.embed_compose(M, H, srcs=[(bad, rows)], device="cuda")
    with pytest.raises(ValueError, match="embed_compose: tab0 must be 16-byte aligned"):
        F.embed_compose(M, H, tabs=[(tab_shifted, tidx)], device="cuda")
    with pytest.raises(ValueError, match="embed_scatter: lddy"):
        F.embed_scatter(bad, dtabs=[(dtab, tidx)])
    with pytest.raises(ValueError, match="embed_scatter: lddsrc0"):
        F.embed_scatter(good, dsrcs=[(dsrc_bad, rows)])
    with pytest.raises(ValueError, match="embed_scatter_sorted: lddy"):
        F.embed_scatter_sorted(bad, dtab, sorted_idx, order)
    with pytest.raises(ValueError, match="embed_scatter_sorted: dy must be 16-byte aligned"):
        F.embed_scatter_sorted(shifted, dtab, sorted_idx, order)
    with pytest.raises(ValueError, match="dropout_apply: ldx"):
        F.dropout_apply(bad, words, 1.0)
    assert lib.launch_count() == n0
