"""The kernels against fp64 at the operand scales of trained models (generators: tests/operand_scales.py), with the
bounds of tests/kernel_check.py:

  attention, every entry point (dense, causal tail, packed self, packed cross, probabilities), d = 64 and 128, key
  lengths across two or more 64-key blocks, with and without keep bits:
    peaked rows (scores spanning > 60 log2 units), the row max planted 40 or 140 log2 units above the rest in the last
    key block (the running correction ex2(m_old - m_new) is tiny, or exactly 0) or in the first (the later blocks' p
    underflow), one-hot rows (ctx is that key's v bit for bit, ctx_lo is 0, every other key's dk and dv exactly 0), exact
    ties (each p exactly 1/2), delta cancellation (dctx parallel to the dominant v, with and without ctx_lo), and peaked
    rows under a finfo.min padding mask (padded keys exactly 0);
  LayerNorm forward and backward, streaming (H <= 1024) and wide backward, unbounded / bounded / ordered, with dx2 and
    dropout: offset rows, outlier channels, constant rows (x = beta bit for bit, rstd = 1 / sqrt(eps)) and rows whose
    variance is within 10x of eps, for eps in {1e-12, 1e-6, 1e-5}; on the last two the fp64 result of another eps must
    miss the kernel by >= 5x its bound, so eps is observable; the same through the embeddings' compose + LayerNorm;
  the loss rows: cross-entropy with the label 60 above / below the rest, a row offset by 1000, the max in the last
    8-column vector and many tied maxima; KL with one-hot targets and 1e-30 entries; MSE at |z - t| ~ 1e3."""
import contextlib
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kernel_check as kc  # noqa: E402
import operand_scales as OS  # noqa: E402
import test_attention_causal_gpu as AC  # noqa: E402
import test_attention_edges_gpu as AE  # noqa: E402
import test_attention_probs_gpu as AP  # noqa: E402
import test_rowops_edges_gpu as RE  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
HEADS = 2
SEQ = {64: (65, 200, 384), 128: (65, 200, 256)}
CASES = {  # name: (generator kind, gap, where)
    "peaked": ("peaked", None, None),
    "max_last_40": ("planted", 40.0, "last"),
    "max_first_40": ("planted", 40.0, "first"),
    "max_last_140": ("planted", 140.0, "last"),
    "max_first_140": ("planted", 140.0, "first"),
    "onehot": ("onehot", None, "last"),
    "tie": ("tie", None, None),
    "delta": ("delta", None, "last"),
}
EXACT = ("onehot", "tie")      # p exactly 0, 1 or 1/2 in fp32


def _fmt(w):
    return " ".join("%s=%.3f" % kv for kv in w.items())


def _merge_worst(acc, w):
    return {k: max(acc.get(k, 0.0), v) for k, v in list(acc.items()) + list(w.items())}


def _sample(case, Sq, Skv, d, g):
    kind, gap, where = CASES[case]
    q, k, v, keys = OS.attention_sample(kind, Sq, Skv, HEADS, d, g, DEV, gap=gap, where=where or "last")
    dctx = OS.dctx_for(kind, Sq, v, keys, g, DEV)
    return q, k, v, keys, dctx


def _expected_ctx(v, keys, keep, dsc):
    """ctx and ctx_lo of one sample when every p is 0 except those of `keys`, equal in value (1 or 1/2): the fp32 output is
    (sum of the kept keys' v) * (fp32(dscale) / len(keys)), rounded to bf16; keep [heads, Sq, Skv] or None"""
    Skv, W = v.shape
    d = W // HEADS
    inv = torch.tensor(dsc, dtype=torch.float32, device=DEV) / len(keys)
    outs = []
    for h in range(HEADS):
        vs = v[:, h * d:(h + 1) * d].float()
        o = 0.0
        for j in keys:
            kj = torch.ones(1, device=DEV) if keep is None else keep[h, :, j].float()
            o = o + kj[:, None] * vs[j][None, :]
        outs.append(o * inv)
    o32 = torch.cat(outs, 1)
    hi = o32.to(torch.bfloat16)
    return hi, (o32 - hi.float()).to(torch.bfloat16)


def _check_exact(case, ctx, lo, dq, dk, dv, q, k, v, dctx, keys, keep, dsc, tag):
    """one-hot / tie rows: ctx bit for bit, ctx_lo, and exact zeros in dk / dv of every key whose p is 0.  One-hot rows
    without keep bits: dS is exactly 0 off the planted key and p (dP - delta) on it, where dP and delta are two fp32
    sums of the same d products dO v (delta from ctx + ctx_lo = v exactly): the tensor-core accumulation of dP (2^-20)
    and the sequential fp32 sum of delta (d 2^-24, its worst case) of sum |dO||v|.  So dq and the planted key's dk are zero
    up to that delta rounding alone: |dq| <= scale (2^-20 + d 2^-24) (|dO| . |v_j|) |k_j| per query, and dk_j the sum
    of the same terms over the queries (with |q|)."""
    Sq = ctx.shape[0]
    want, want_lo = _expected_ctx(v, keys, keep, dsc)
    want = want.expand(Sq, -1) if want.shape[0] == 1 else want
    want_lo = want_lo.expand(Sq, -1) if want_lo.shape[0] == 1 else want_lo
    kc.assert_bits_equal(ctx, want.contiguous(), kc.flat_layout(), tag + " ctx (bit for bit)")
    kc.assert_bits_equal(lo, want_lo.contiguous(), kc.flat_layout(), tag + " ctx_lo (bit for bit)")
    others = torch.ones(v.shape[0], dtype=torch.bool, device=DEV)
    others[keys] = False
    assert not dk[others].any() and not dv[others].any(), tag + ": a key with p = 0 got a nonzero dk / dv"
    if case != "onehot" or keep is not None:
        return
    W = v.shape[1]
    d = W // HEADS
    sc = 1.0 / math.sqrt(d)
    j = keys[0]
    heads = lambda t: t.double().abs().reshape(t.shape[0], HEADS, d)                  # [rows, heads, d]
    e = (kc.U_ACC + d * kc.U_F32) * (heads(dctx) * heads(v[j:j + 1])).sum(-1)         # [Sq, heads]
    b_dq = (sc * e[:, :, None] * heads(k[j:j + 1])).reshape(Sq, W)
    b_dk = (sc * (e[:, :, None] * heads(q)).sum(0)).reshape(1, W)
    lay = kc.flat_layout()
    kc.assert_within(dq, torch.zeros_like(b_dq), b_dq, lay, tag + " dq (delta rounding only)")
    kc.assert_within(dk[j:j + 1], torch.zeros_like(b_dk), b_dk, lay,
                     tag + " dk of the planted key (delta rounding only)")


def _keep(shape, p, g):
    return None if p == 0 else torch.rand(*shape, generator=g, device=DEV) >= p


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("case", list(CASES))
def test_dense_attention_at_scale(case, d):
    from mmf_b200 import functional as F
    worst = {}
    for S in SEQ[d]:
        for p in (0.0, 0.1):
            for use_lo in ((True, False) if case == "delta" else (True,)):
                g = torch.Generator(device=DEV).manual_seed(S * 10 + d + int(p * 10) + use_lo)
                B = 2
                parts = [_sample(case, S, S, d, g) for _ in range(B)]
                q, k, v, dctx = (torch.cat([pt[i] for pt in parts]) for i in (0, 1, 2, 4))
                keep = _keep((B, HEADS, S, S), p, g)
                dm = F.pack_keep_bits(keep) if keep is not None else None
                dsc = 1.0 / (1.0 - p)
                ctx, lse2, lo = F.attention_fwd(q, k, v, B, HEADS, S, S, drop_mask=dm, drop_scale=dsc, save_lo=True)
                dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, HEADS, S, S, drop_mask=dm, drop_scale=dsc,
                                             ctx_lo=lo if use_lo else None)
                torch.cuda.synchronize()
                tag = "dense %s S%d d%d p%.1f lo=%d" % (case, S, d, p, use_lo)
                out = {"ctx": ctx, "lse2": lse2, "ctx_lo": lo, "dq": dq, "dk": dk, "dv": dv}
                ref = kc.attention_ref(q, k, v, B, HEADS, S, S, keep=keep, p_drop=p, dctx=dctx, lo_used=use_lo)
                worst = _merge_worst(worst, AE._check_all(out, ref, B, HEADS, S, S, d, tag))
                if case in EXACT:
                    for b in range(B):
                        r = slice(b * S, (b + 1) * S)
                        _check_exact(case, ctx[r], lo[r], dq[r], dk[r], dv[r], q[r], k[r], v[r], dctx[r], parts[b][3],
                                     None if keep is None else keep[b], dsc, tag + " sample %d" % b)
    print("scale dense %s d%d: %s" % (case, d, _fmt(worst)))


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("case", list(CASES))
def test_causal_tail_attention_at_scale(case, d):
    from mmf_b200 import functional as F
    worst = {}
    for S in SEQ[d]:
        for p in (0.0, 0.1):
            g = torch.Generator(device=DEV).manual_seed(S * 10 + d + int(p * 10) + 1)
            B, T = 1, S // 3
            q, k, v, keys, dctx = _sample(case, S, S, d, g)
            enc = torch.ones(B, S - T, device=DEV)
            mask = torch.cat([torch.zeros(B, S - T, device=DEV), torch.full((B, T), float("nan"), device=DEV)], 1)
            keep = _keep((B, HEADS, S, S), p, g)
            dm = F.pack_keep_bits(keep) if keep is not None else None
            dsc = 1.0 / (1.0 - p)
            ctx, lse2, lo = F.attention_fwd(q, k, v, B, HEADS, S, S, mask=mask.contiguous(), drop_mask=dm, drop_scale=dsc,
                                            save_lo=True, causal_len=T)
            dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, HEADS, S, S, mask=mask.contiguous(), drop_mask=dm,
                                         drop_scale=dsc, ctx_lo=lo, causal_len=T)
            torch.cuda.synchronize()
            ref = AC.per_query_reference(q, k, v, B, HEADS, S, AC.reference_mask(enc, T), keep, p, dctx)
            out = {"ctx": ctx, "lse2": lse2, "dq": dq, "dk": dk, "dv": dv}
            worst = _merge_worst(worst, AC.check(out, ref, B, HEADS, S, d, "causal %s S%d d%d p%.1f" % (case, S, d, p)))
    print("scale causal %s d%d: %s" % (case, d, _fmt(worst)))


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("case", list(CASES))
def test_packed_self_attention_at_scale(case, d):
    from mmf_b200 import functional as F
    worst = {}
    S = SEQ[d][-1]
    lens = [S, 130, 65]
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    for p in (0.0, 0.1):
        g = torch.Generator(device=DEV).manual_seed(d + int(p * 10) + 2)
        parts = [_sample(case, n, n, d, g) for n in lens]
        q, k, v, dctx = (torch.cat([pt[i] for pt in parts]) for i in (0, 1, 2, 4))
        total = q.shape[0]
        keep = _keep((HEADS, total, S), p, g)
        dm = F.pack_keep_bits(keep) if keep is not None else None
        dsc = 1.0 / (1.0 - p)
        ctx, lse2, lo = F.attention_varlen_fwd(q, k, v, cu, S, HEADS, dm, dsc, save_lo=True)
        dq, dk, dv = F.attention_varlen_bwd(dctx, q, k, v, ctx, lse2, cu, S, HEADS, dm, dsc, ctx_lo=lo)
        torch.cuda.synchronize()
        s = 0
        for b, n in enumerate(lens):
            r = slice(s, s + n)
            kb = keep[:, r, :n].unsqueeze(0) if keep is not None else None
            ref = kc.attention_ref(q[r], k[r], v[r], 1, HEADS, n, n, keep=kb, p_drop=p, dctx=dctx[r], lo_used=True)
            out = {"ctx": ctx[r], "lse2": lse2[:, r].unsqueeze(0), "ctx_lo": lo[r], "dq": dq[r], "dk": dk[r], "dv": dv[r]}
            tag = "packed self %s d%d p%.1f sample %d (len %d)" % (case, d, p, b, n)
            worst = _merge_worst(worst, AE._check_all(out, ref, 1, HEADS, n, n, d, tag))
            if case in EXACT:
                _check_exact(case, ctx[r], lo[r], dq[r], dk[r], dv[r], q[r], k[r], v[r], dctx[r], parts[b][3],
                             None if kb is None else kb[0], dsc, tag)
            s += n
    print("scale packed self %s d%d: %s" % (case, d, _fmt(worst)))


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("case", list(CASES))
def test_packed_cross_attention_at_scale(case, d):
    from mmf_b200 import functional as F
    worst = {}
    S = SEQ[d][-1]
    lq, lk = [37, 100, 129], [S, 65, 200]
    cq = torch.tensor([0] + torch.tensor(lq).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    ck = torch.tensor([0] + torch.tensor(lk).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    for p in (0.0, 0.1):
        g = torch.Generator(device=DEV).manual_seed(d + int(p * 10) + 3)
        parts = [_sample(case, nq, nk, d, g) for nq, nk in zip(lq, lk)]
        q, k, v, dctx = (torch.cat([pt[i] for pt in parts]) for i in (0, 1, 2, 4))
        keep = _keep((HEADS, q.shape[0], max(lk)), p, g)
        dm = F.pack_keep_bits(keep) if keep is not None else None
        dsc = 1.0 / (1.0 - p)
        ctx, lse2, lo = F.attention_varlen_cross_fwd(q, k, v, cq, ck, max(lq), max(lk), HEADS, dm, dsc, save_lo=True)
        dq, dk, dv = F.attention_varlen_cross_bwd(dctx, q, k, v, ctx, lse2, cq, ck, max(lq), max(lk), HEADS, dm, dsc,
                                                  ctx_lo=lo)
        torch.cuda.synchronize()
        qs = ks = 0
        for b, (nq, nk) in enumerate(zip(lq, lk)):
            rq, rk = slice(qs, qs + nq), slice(ks, ks + nk)
            kb = keep[:, rq, :nk].unsqueeze(0) if keep is not None else None
            ref = kc.attention_ref(q[rq], k[rk], v[rk], 1, HEADS, nq, nk, keep=kb, p_drop=p, dctx=dctx[rq], lo_used=True)
            tag = "packed cross %s d%d p%.1f sample %d (q %d, kv %d)" % (case, d, p, b, nq, nk)
            lay_q, lay_k = kc.attn_layout(1, HEADS, nq, d, "query"), kc.attn_layout(1, HEADS, nk, d, "key")
            w = {"ctx": kc.assert_within(ctx[rq], ref["ctx"], ref["b_ctx"], lay_q, tag + " ctx"),
                 "lse2": kc.assert_within(lse2[:, rq].unsqueeze(0), ref["lse2"], ref["b_lse2"], lay_q, tag + " lse2"),
                 "ctx+lo": kc.assert_within(ctx[rq].double() + lo[rq].double(), ref["ctx"], ref["b_lo"], lay_q,
                                            tag + " ctx+ctx_lo"),
                 "dq": kc.assert_within(dq[rq], ref["dq"], ref["b_dq"], lay_q, tag + " dq"),
                 "dk": kc.assert_within(dk[rk], ref["dk"], ref["b_dk"], lay_k, tag + " dk"),
                 "dv": kc.assert_within(dv[rk], ref["dv"], ref["b_dv"], lay_k, tag + " dv")}
            worst = _merge_worst(worst, w)
            if case in EXACT:
                _check_exact(case, ctx[rq], lo[rq], dq[rq], dk[rk], dv[rk], q[rq], k[rk], v[rk], dctx[rq], parts[b][3],
                             None if kb is None else kb[0], dsc, tag)
            qs, ks = qs + nq, ks + nk
    print("scale packed cross %s d%d: %s" % (case, d, _fmt(worst)))


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("case", list(CASES))
def test_attention_probs_at_scale(case, d):
    from mmf_b200 import functional as F
    worst = 0.0
    for S in SEQ[d]:
        for p in (0.0, 0.1):
            g = torch.Generator(device=DEV).manual_seed(S * 10 + d + int(p * 10) + 4)
            Sq = 70
            q, k, v, keys, _ = _sample(case, Sq, S, d, g)
            keep = _keep((1, HEADS, Sq, S), p, g)
            dm = F.pack_keep_bits(keep) if keep is not None else None
            dsc = 1.0 / (1.0 - p)
            ctx, lse2 = F.attention_fwd(q, k, v, 1, HEADS, Sq, S, drop_mask=dm, drop_scale=dsc)
            out = F.attention_probs(q, k, lse2, 1, HEADS, Sq, S, drop_mask=dm, drop_scale=dsc)
            torch.cuda.synchronize()
            Pd, bound, _, _ = AP.probs_ref(q, k, 1, HEADS, Sq, S, keep=keep, p_drop=p)
            tag = "probs %s S%d d%d p%.1f" % (case, S, d, p)
            worst = max(worst, kc.assert_within(out, Pd, bound, AP.probs_layout(1, HEADS, Sq, S), tag))
            if keep is not None:
                assert (out[~keep] == 0).all(), tag + ": a dropped entry is not exactly 0"
            if case in EXACT:
                others = torch.ones(S, dtype=torch.bool, device=DEV)
                others[keys] = False
                assert not out[..., others].any(), tag + ": a key far below the row max has p != 0"
            if case == "tie":
                # l = 1 + 1 = 2, lse2 = max + 1 exactly, z - lse2 = -1 at both keys: p = 1/2 (* keep * dscale) in fp32
                kp = torch.ones(1, HEADS, Sq, len(keys), device=DEV) if keep is None else keep[..., keys].float()
                want = 0.5 * kp * torch.tensor(dsc, dtype=torch.float32, device=DEV)
                kc.assert_bits_equal(out[..., keys].contiguous(), want, kc.flat_layout(),
                                     tag + ": tied p is not exactly 1/2")
    print("scale probs %s d%d: probs=%.3f" % (case, d, worst))


@pytest.mark.parametrize("d", [64, 128])
def test_peaked_rows_under_a_dtype_min_padding_mask(d):
    """padded keys at finfo(fp32).min stay exactly 0 (probabilities, dk, dv) however large the real scores are, with and
    without keep bits; the samples match fp64 of the clamped mask"""
    from mmf_b200 import functional as F
    S = SEQ[d][-1]
    B = 2
    g = torch.Generator(device=DEV).manual_seed(d + 5)
    parts = [_sample("peaked", S, S, d, g) for _ in range(B)]
    q, k, v, dctx = (torch.cat([pt[i] for pt in parts]) for i in (0, 1, 2, 4))
    low = float(torch.finfo(torch.float32).min)
    mask = torch.zeros(B, S, device=DEV)
    mask[0, S - 37:] = low
    mask[1, :70] = low
    mask = mask.contiguous()
    padded = (mask == low)
    w = {}
    for p in (0.0, 0.1):
        keep = _keep((B, HEADS, S, S), p, g)
        dm = F.pack_keep_bits(keep) if keep is not None else None
        dsc = 1.0 / (1.0 - p)
        ctx, lse2, lo = F.attention_fwd(q, k, v, B, HEADS, S, S, mask=mask, drop_mask=dm, drop_scale=dsc, save_lo=True)
        dq, dk, dv = F.attention_bwd(dctx, q, k, v, ctx, lse2, B, HEADS, S, S, mask=mask, drop_mask=dm, drop_scale=dsc,
                                     ctx_lo=lo)
        probs = F.attention_probs(q, k, lse2, B, HEADS, S, S, mask=mask, drop_mask=dm, drop_scale=dsc)
        torch.cuda.synchronize()
        tag = "peaked dtype-min mask d%d p%.1f" % (d, p)
        assert not probs.permute(0, 3, 1, 2)[padded].any(), tag + ": a padded key has p != 0"
        rows = padded.reshape(-1)
        assert not dk[rows].any() and not dv[rows].any(), tag + ": a padded key has a nonzero dk / dv"
        ref = kc.attention_ref(q, k, v, B, HEADS, S, S, mask=mask.clamp_min(AE.MASK_FLOOR), keep=keep, p_drop=p,
                               dctx=dctx, lo_used=True)
        w = _merge_worst(w, AE._check_all({"ctx": ctx, "lse2": lse2, "ctx_lo": lo, "dq": dq, "dk": dk, "dv": dv}, ref,
                                          B, HEADS, S, S, d, tag))
    print("scale peaked dtype-min mask d%d: %s" % (d, _fmt(w)))


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
EPS = (1e-12, 1e-6, 1e-5)
LN_CASES = ["offset16", "offset64", "outlier", "constant", "near"]
LN_H = [264, 1024, 1032, 2040]         # streaming backward (H <= 1024), wide backward


def worst_ratio(out, ref, bound):
    """max |out - ref| / bound without asserting (the discrimination checks want it large)"""
    err = (out.detach().double() - ref.double()).abs()
    return (err / bound.double().expand_as(err).clamp_min(1e-300)).max().item()


def other_eps(eps):
    """the eps a misrouted call would use: the library default, or 1e-6 when eps is the default"""
    return 1e-6 if eps == 1e-12 else 1e-12


@contextlib.contextmanager
def _mode(mode):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "ordered")
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _ln_rows(case, M, H, eps, g):
    if case.startswith("offset"):
        return OS.ln_rows("offset", M, H, g, DEV, c=float(case[len("offset"):]))
    return OS.ln_rows(case, M, H, g, DEV, eps=eps)


@pytest.mark.parametrize("H", LN_H)
@pytest.mark.parametrize("case", LN_CASES)
def test_layernorm_at_scale(case, H):
    from mmf_b200 import functional as F
    M = 40
    lay = kc.row_layout()
    worst = {}
    for eps in EPS:
        for mode in ("plain", "bounded", "ordered"):
            i = EPS.index(eps) * 3 + ("plain", "bounded", "ordered").index(mode)
            with_dx2, with_drop = bool(i % 2), bool((i // 2) % 2)
            g = torch.Generator(device=DEV).manual_seed(H * 100 + i)
            y = _ln_rows(case, M, H, eps, g)
            gam = (1 + 0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16)
            bet = (0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16)
            rows = M - 3 if mode == "bounded" else M
            bnd = torch.tensor([rows], dtype=torch.int32, device=DEV) if mode == "bounded" else None
            dx = torch.randn(M, H, generator=g, device=DEV).to(torch.bfloat16)
            dx2 = torch.randn(M, H, generator=g, device=DEV).to(torch.bfloat16) if with_dx2 else None
            keep, bits, dsc = None, None, 1.0
            if with_drop:
                keep = torch.rand(M, H, generator=g, device=DEV) > 0.1
                bits, dsc = F.pack_keep_bits(keep), 1 / 0.9
            dgamma, dbeta, dbias = (torch.zeros(H, device=DEV) for _ in range(3))
            with _mode(mode):
                x, mean, rstd = F.layernorm_fwd(y, gam, bet, eps, m_bound=bnd)
                dy, dz = F.layernorm_bwd(dx, y, mean, rstd, gam, dgamma, dbeta, dbias=dbias, dx2=dx2, drop_mask=bits,
                                         drop_scale=dsc, m_bound=bnd)
            torch.cuda.synchronize()
            tag = "ln %s H%d eps%g %s dx2=%d drop=%d" % (case, H, eps, mode, with_dx2, with_drop)
            r = slice(0, rows)
            if rows < M:
                assert not x[rows:].any() and not dy[rows:].any() and not dz[rows:].any(), tag + ": rows past the bound"
            yr, dxr, dx2r = y[r], dx[r], (dx2[r] if dx2 is not None else None)
            keepr = keep[r] if keep is not None else None
            fw = kc.layernorm_ref(yr, gam, bet, eps)
            w = {"mean": kc.assert_within(mean[r], fw["mean"], fw["b_mean"], lay, tag + " mean"),
                 "rstd": kc.assert_within(rstd[r], fw["rstd"], fw["b_rstd"], lay, tag + " rstd"),
                 "x": kc.assert_within(x[r], fw["x"], fw["b_x"], lay, tag + " x")}
            n = RE._bwd_sum_terms(M)
            bw = kc.layernorm_bwd_ref(fw, dxr, gam, dx2=dx2r, keep=keepr, dscale=dsc, n_sum_terms=n)
            w["dy"] = kc.assert_within(dy[r], bw["dy"], bw["b_dy"], lay, tag + " dy")
            w["dz"] = kc.assert_within(dz[r], bw["dz"], bw["b_dz"], lay, tag + " dz")
            w["dgamma"] = kc.assert_within(dgamma, bw["dgamma"], bw["b_dgamma"], lay, tag + " dgamma")
            w["dbeta"] = kc.assert_within(dbeta, bw["dbeta"], bw["b_dbeta"], lay, tag + " dbeta")
            if with_drop and H <= 1024:      # the streaming kernel sums the bf16 dz it stores
                dz64 = dz[r].double()
                ref_b, b_b = dz64.sum(0), kc.U_F32 * n * dz64.abs().sum(0)
            else:
                ref_b, b_b = bw["dz"].sum(0), bw["e_dz_f32"].sum(0) + kc.U_F32 * n * bw["dz"].abs().sum(0)
            w["dbias"] = kc.assert_within(dbias, ref_b, b_b, lay, tag + " dbias")
            worst = _merge_worst(worst, w)
            if case == "constant":
                assert torch.equal(x[r], bet.expand(rows, H)), tag + ": x is not beta bit for bit"
                assert torch.isfinite(mean).all() and torch.isfinite(rstd).all(), tag
            if case in ("constant", "near"):
                # eps is observable: fp64 with another eps misses the kernel by far more than the bound
                fo = kc.layernorm_ref(yr, gam, bet, other_eps(eps))
                bo = kc.layernorm_bwd_ref(fo, dxr, gam, dx2=dx2r, keep=keepr, dscale=dsc, n_sum_terms=n)
                miss_rstd = worst_ratio(rstd[r], fo["rstd"], fw["b_rstd"])
                miss_dy = worst_ratio(dy[r], bo["dy"], bw["b_dy"])
                assert miss_rstd >= 5 * kc.SAFETY and miss_dy >= 5 * kc.SAFETY, (tag, miss_rstd, miss_dy)
                if case == "near":
                    miss_x = worst_ratio(x[r], fo["x"], fw["b_x"])
                    assert miss_x >= 5 * kc.SAFETY, (tag, miss_x)
    print("scale %s: %s" % ("ln %s H%d" % (case, H), _fmt(worst)))


@pytest.mark.parametrize("eps", [1e-6, 1e-5])
def test_compose_layernorm_takes_its_eps(eps):
    """the embeddings' compose + LayerNorm (ops.compose_ln) on rows whose variance is within 10x of eps: forward and the
    source gradient against fp64 with that eps, and far from fp64 with the default eps"""
    from mmf_b200 import ops
    M, H = 48, 768
    g = torch.Generator(device=DEV).manual_seed(int(-math.log10(eps)))
    y = OS.ln_rows("near", M, H, g, DEV, eps=eps)
    src = y.clone().requires_grad_(True)
    tab = torch.zeros(4, H, device=DEV, dtype=torch.bfloat16)
    rows = torch.arange(M, dtype=torch.int32, device=DEV)
    idx = (torch.arange(M, device=DEV) % 4).to(torch.int32)
    gam = (1 + 0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16)
    bet = (0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16)
    out = ops.compose_ln(M, H, [(src, rows)], [(tab, idx)], gam, bet, eps)
    dout = torch.randn(M, H, generator=g, device=DEV).to(torch.bfloat16)
    out.backward(dout)
    torch.cuda.synchronize()
    lay = kc.row_layout()
    fw = kc.layernorm_ref(y, gam, bet, eps)
    bw = kc.layernorm_bwd_ref(fw, dout, gam)
    w = {"x": kc.assert_within(out, fw["x"], fw["b_x"], lay, "compose_ln x eps %g" % eps),
         "dsrc": kc.assert_within(src.grad, bw["dy"], bw["b_dy"], lay, "compose_ln d(src) eps %g" % eps)}
    fo = kc.layernorm_ref(y, gam, bet, other_eps(eps))
    bo = kc.layernorm_bwd_ref(fo, dout, gam)
    assert worst_ratio(out, fo["x"], fw["b_x"]) >= 5 * kc.SAFETY
    assert worst_ratio(src.grad, bo["dy"], bw["b_dy"]) >= 5 * kc.SAFETY
    print("scale compose_ln eps %g: %s" % (eps, _fmt(w)))


# ------------------------------------------------------------------------------------------------------------------
# loss rows
# ------------------------------------------------------------------------------------------------------------------
def _ce_logits(V, g):
    """[6, V] rows: label 60 above the rest, label 60 below, the whole row + 1000, the max only in the last 8-column
    vector, 100 tied maxima, and a row with the tied maxima at the label"""
    z = torch.randn(6, V, generator=g, device=DEV)
    labels = torch.randint(0, V, (6,), generator=g, device=DEV)
    z[0, labels[0]] = 60.0
    z[1, labels[1]] = -60.0
    z[2] = 1000.0 + 16.0 * z[2]                 # bf16 ulp 4 at 1000: a spread of 16 keeps the row an offset N(0, 16^2)
    z[3, V - 8 + int(labels[3] % 8)] = 20.0
    for r in (4, 5):
        cols = torch.randperm(V, generator=g, device=DEV)[:100]
        z[r, cols] = 10.0
        if r == 5:
            labels[5] = cols[0]
    return z.to(torch.bfloat16), labels


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("V", [2056, 30528])
def test_ce_rows_at_scale(V, bounded):
    from mmf_b200 import functional as F
    g = torch.Generator(device=DEV).manual_seed(V + bounded)
    z, labels = _ce_logits(V, g)
    zin = z.clone()
    scale = 0.25
    M = z.shape[0]
    loss_sum = torch.zeros((), device=DEV)
    row_loss = torch.empty(M, device=DEV)
    if bounded:
        F.ce_rows_bounded(z, labels, -1, torch.tensor([scale], device=DEV), torch.tensor([M], dtype=torch.int32, device=DEV),
                          loss_sum, row_loss)
    else:
        F.ce_rows(z, labels, -1, scale, loss_sum, row_loss)
    torch.cuda.synchronize()
    loss, b_loss, grad, b_grad = RE._ce_ref(zin, labels, V, scale)
    lay = kc.row_layout()
    tag = "ce%s V%d" % ("_bounded" if bounded else "", V)
    w1 = kc.assert_within(row_loss, loss, b_loss, lay, tag + " row_loss")
    w2 = kc.assert_within(z, grad, b_grad, lay, tag + " d(logits)")
    print("scale %s: row_loss=%.3f d(logits)=%.3f" % (tag, w1, w2))


def _region_bounds(kind, z0, tgt, s, V):
    """fp64 gradient and row loss of the region rows and their bounds (test_uniter_graphs_gpu's derivation: fp32
    arithmetic of a few terms rounded once to bf16 for the gradient, fp32 sums of V terms for the loss)"""
    zz, q = z0[:, :V].double(), tgt.double()
    if kind == "kl":
        logp = torch.log_softmax(zz, dim=-1)
        Q = q.sum(-1, keepdim=True)
        loss_ref = (torch.xlogy(q, q) - q * logp).sum(-1)
        loss_abs = (torch.xlogy(q, q).abs() + (q * logp).abs()).sum(-1)
        grad_ref, grad_abs = (logp.exp() * Q - q) * s, (logp.exp() * Q + q) * s
    else:
        dd = zz - q
        loss_ref, loss_abs = (dd * dd).sum(-1), (dd * dd).sum(-1)
        grad_ref, grad_abs = 2 * dd * s, 2 * (zz.abs() + q.abs()) * s
    return (grad_ref, 2.0 ** -9 * grad_ref.abs() + 64 * kc.U_F32 * grad_abs,
            loss_ref, 2 * V * kc.U_F32 * loss_abs + 1e-30)


@pytest.mark.parametrize("kind", ["kl_onehot", "kl_tiny", "mse_far"])
def test_region_rows_at_scale(kind):
    from mmf_b200 import functional as F
    g = torch.Generator(device=DEV).manual_seed(len(kind))
    M, V = 24, 1601
    Vp = -(-V // 8) * 8
    z0 = (torch.randn(M, Vp, generator=g, device=DEV) * 4).to(torch.bfloat16)
    if kind == "kl_onehot":
        tgt = torch.nn.functional.one_hot(torch.randint(0, V, (M,), generator=g, device=DEV), V).float()
    elif kind == "kl_tiny":
        tgt = torch.softmax(torch.randn(M, V, generator=g, device=DEV) * 3, -1)
        tgt[torch.rand(M, V, generator=g, device=DEV) < 0.3] = 1e-30
    else:
        tgt = torch.randn(M, Vp, generator=g, device=DEV)
        z0 = (tgt + torch.where(torch.rand(M, Vp, generator=g, device=DEV) < 0.5, -1000.0, 1000.0)).to(torch.bfloat16)
    idx = torch.randperm(M, generator=g, device=DEV).to(torch.int32)
    s = 1.0 / M
    scale = torch.tensor([s], device=DEV)
    z, rl = z0.clone(), torch.full((M,), -5.0, device=DEV)
    bnd = torch.tensor([M], dtype=torch.int32, device=DEV)
    if kind.startswith("kl"):
        F.kl_rows_bounded(z, V, tgt, idx, bnd, scale, rl)
        cols = V
    else:
        F.mse_rows_bounded(z, tgt, idx, bnd, scale, rl)
        cols = Vp
    torch.cuda.synchronize()
    grad_ref, b_grad, loss_ref, b_loss = _region_bounds(kind.split("_")[0], z0, tgt.index_select(0, idx.long()), s, cols)
    lay = kc.row_layout()
    w1 = kc.assert_within(z[:, :cols], grad_ref, b_grad, lay, kind + " gradient")
    w2 = kc.assert_within(rl, loss_ref, b_loss, lay, kind + " row loss")
    print("scale %s: grad=%.3f loss=%.3f" % (kind, w1, w2))
