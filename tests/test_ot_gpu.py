"""mmfb_ot_fwd / mmfb_ot_bwd through the C ABI, element by element against the fp64 oracle
(oracle/ot_oracle.optimal_transport_dist, the restatement of mmf/modules/ot.py).

The bound.  The inputs are bf16, so the products of the dot products are exact in fp32 and the kernel differs from fp64
only by fp32 rounding: in the summation of the cost, in exp, and through `iterations` multiplicative updates of the
plan.  How far fp32 drifts over those updates depends on the problem (lengths, beta, how close the plan is to its fixed
point), so the test measures it instead of guessing: the same oracle runs in fp32 on the same inputs, and its worst
deviation from fp64 - relative to the largest entry of the tensor, which is how a plan of entries ~1/(M N) is judged -
is the yardstick.  The kernel must stay within SLACK times that drift plus FLOOR (1e-5 of the largest entry: the fp32
rounding of a 1024-term dot product, for the cases where the fp32 oracle happens to land on the fp64 value).  dx / dy are stored in bf16: their bound adds
half a bf16 ulp (at most 2^-8 of the fp64 value), element by element.  On an H100 the largest errors seen were at the
level of the fp32 oracle's own drift (plan 3.5e-6 against 3.0e-6, distance 3.4e-7, cost 1.8e-7 of the largest entry)."""
import ctypes
import os

import pytest
import torch

from oracle import ot_oracle as FO

pytestmark = pytest.mark.gpu

SLACK, FLOOR = 8.0, 1e-5
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _lens(kind, B, L, g):
    if kind == "one":
        return [1] * B
    if kind == "full":
        return [L] * B
    return [int(v) for v in torch.randint(1, L + 1, (B,), generator=g)]


def _pads(lens, L, device):
    return torch.arange(L, device=device).unsqueeze(0) >= torch.tensor(lens, device=device).unsqueeze(1)


def _oracle(x, y, xl, yl, dtype, beta, iteration, k, g_out):
    xr = x.detach().to(dtype).requires_grad_(True)
    yr = y.detach().to(dtype).requires_grad_(True)
    d, cost, T = FO.optimal_transport_dist(xr, yr, _pads(xl, x.shape[1], x.device), _pads(yl, y.shape[1], x.device), beta,
                                           iteration, k, return_all=True)
    (d * g_out.to(dtype)).sum().backward()
    return d.detach(), cost.detach(), T, xr.grad, yr.grad


def _scaled_err(got, ref):
    return ((got.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-30)).item()


def _run_case(B, M, N, H, lens_kind, iteration, k, seed, zero_row=False):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(seed)
    # text and regions are two row ranges of ONE buffer, with a row of slack between the samples' ranges
    buf = torch.randn(B, M + N + 1, H, generator=g).to(torch.bfloat16).cuda()
    xl, yl = _lens(lens_kind, B, M, g), _lens(lens_kind, B, N, g)
    if zero_row:
        buf[0, 0] = 0              # |x| below eps: x / eps, cost 1 against every region
        buf[0, M] = 0
    x, y = buf[:, :M], buf[:, M:M + N]
    # padded rows hold NaN: the kernels must not read them
    for b in range(B):
        buf[b, xl[b]:M] = float("nan")
        buf[b, M + yl[b]:M + N] = float("nan")
    g_out = (torch.randn(B, generator=g) + 2.0).cuda()
    dist, plan, saved, cost = F.ot_fwd(x, y, xl, yl, 0.5, iteration, k, want_cost=True)
    dbuf = torch.full_like(buf, 7.0)
    F.ot_bwd(g_out, plan, saved, x, y, xl, yl, dbuf[:, :M], dbuf[:, M:M + N])
    torch.cuda.synchronize()
    clean = torch.nan_to_num(buf, nan=0.0)
    cx, cy = clean[:, :M], clean[:, M:M + N]
    r64 = _oracle(cx, cy, xl, yl, torch.float64, 0.5, iteration, k, g_out)
    r32 = _oracle(cx, cy, xl, yl, torch.float32, 0.5, iteration, k, g_out)
    got = (dist, cost, plan, dbuf[:, :M], dbuf[:, M:M + N])
    worst = {}
    for name, gt, a, b32 in zip(("dist", "cost", "T", "dx", "dy"), got, r64, r32):
        assert torch.isfinite(gt).all(), name
        drift = _scaled_err(b32, a)
        bound = SLACK * drift + FLOOR
        if name in ("dx", "dy"):
            err = ((gt.double() - a).abs() - a.abs() * 2.0 ** -8).clamp_min(0).max().item() / a.abs().max().clamp_min(1e-30).item()
        else:
            err = _scaled_err(gt, a)
        worst[name] = (err, drift)
        assert err <= bound, "%s: error %.3e (of the largest entry) above %.1f x fp32 drift %.3e + %.0e" % (
            name, err, SLACK, drift, FLOOR)
    # exact zeros on padding; untouched memory outside the two row ranges
    xp, yp = _pads(xl, M, "cuda"), _pads(yl, N, "cuda")
    jp = yp.unsqueeze(-1) | xp.unsqueeze(-2)
    assert (plan[jp] == 0).all() and (cost[jp.transpose(1, 2)] == 0).all()
    assert (dbuf[:, :M][xp] == 0).all() and (dbuf[:, M:M + N][yp] == 0).all()
    assert (dbuf[:, M + N] == 7.0).all()
    return worst


@pytest.mark.parametrize("M,N", [(1, 1), (7, 1), (1, 100), (7, 7), (60, 100), (100, 60), (128, 128), (60, 128), (128, 7)])
@pytest.mark.parametrize("H", [64, 768, 1024])
def test_ot_against_fp64(M, N, H):
    worst = {}
    for lens_kind in ("one", "ragged", "full"):
        for iteration, k in ((1, 1), (50, 1), (50, 2)):
            w = _run_case(3, M, N, H, lens_kind, iteration, k, seed=M * 1000 + N * 10 + H)
            for name, (e, d) in w.items():
                if e >= worst.get(name, (-1, 0))[0]:
                    worst[name] = (e, d)
    print("\nOT M=%d N=%d H=%d: " % (M, N, H) + "  ".join("%s err %.2e (fp32 drift %.2e)" % (n, e, d)
                                                          for n, (e, d) in worst.items()))


def test_zero_row_and_many_samples():
    w = _run_case(5, 60, 100, 768, "ragged", 50, 1, seed=5, zero_row=True)
    print("\nOT zero row: " + "  ".join("%s err %.2e" % (n, e) for n, (e, _) in w.items()))
    w = _run_case(300, 16, 24, 64, "ragged", 50, 1, seed=6)        # more samples than one launch carries
    print("OT B=300: " + "  ".join("%s err %.2e" % (n, e) for n, (e, _) in w.items()))


def test_unsupported_arguments_are_refused_without_a_launch():
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    before = lib.launch_count()
    buf = torch.randn(2, 140, 72, device="cuda").to(torch.bfloat16)
    ok = torch.randn(2, 20, 64, device="cuda").to(torch.bfloat16)
    big = torch.randn(2, 133, 64, device="cuda").to(torch.bfloat16)
    with pytest.raises(ValueError, match="M, N <= 128"):
        F.ot_fwd(big[:, :129], big[:, 129:], [1, 1], [1, 1])
    with pytest.raises(ValueError, match="x_len"):
        F.ot_fwd(ok[:, :8], ok[:, 8:], [0, 3], [2, 2])
    with pytest.raises(ValueError, match="y_len"):
        F.ot_fwd(ok[:, :8], ok[:, 8:], [3, 3], [2, 13])
    with pytest.raises(ValueError, match="multiple of 64"):
        F.ot_fwd(buf[:, :8], buf[:, 8:16], [3, 3], [2, 2])
    with pytest.raises(ValueError, match="iterations"):
        F.ot_fwd(ok[:, :8], ok[:, 8:], [3, 3], [2, 2], iterations=0)
    assert lib.LIB.mmfb_ot_fwd(None, None) == lib.MMFB_ERR_ARG
    a = lib.OtArgs()
    assert lib.LIB.mmfb_ot_bwd(ctypes.byref(a), None) == lib.MMFB_ERR_ARG
    assert lib.launch_count() == before


def test_autograd_function_writes_both_row_ranges_of_the_sequence_gradient():
    from mmf_b200 import ops
    g = torch.Generator().manual_seed(11)
    T_len, R_len, H = 12, 20, 128
    seq = torch.randn(4, T_len + R_len + 3, H, generator=g).to(torch.bfloat16).cuda().requires_grad_(True)
    xl, yl = [12, 5, 12, 1], [20, 20, 3, 9]
    d = ops.optimal_transport_dist(seq, T_len, R_len, xl, yl)
    w = torch.tensor([1.0, -1.0, 0.5, 2.0], device="cuda")
    (d * w).sum().backward()
    s64 = seq.detach().double().requires_grad_(True)
    d64 = FO.optimal_transport_dist(s64[:, :T_len], s64[:, T_len:T_len + R_len], _pads(xl, T_len, "cuda"),
                                    _pads(yl, R_len, "cuda"))
    (d64 * w.double()).sum().backward()
    assert _scaled_err(d, d64) < 1e-4
    assert ((seq.grad.double() - s64.grad).abs() <= s64.grad.abs() * 2.0 ** -8 + 1e-5 * s64.grad.abs().max()).all()
    assert (seq.grad[:, T_len + R_len:] == 0).all()


def test_golden_wra_entry_is_reproduced():
    """the REFERENCE's own cost / ipot / distance (tools/make_golden_uniter_model.py) on the kernel"""
    from mmf_b200 import functional as F
    gold = torch.load(os.path.join(GOLD, "uniter_model.pt"), weights_only=False)["ot"]
    seq = gold["sequence_output"].to(torch.bfloat16).cuda()
    assert torch.equal(seq.float().cpu(), gold["sequence_output"])        # stored on the bf16 grid: nothing is lost
    T_len, R_len = gold["T_len"], gold["R_len"]
    xl = (~gold["txt_pad"]).sum(1).tolist()
    yl = (~gold["img_pad"]).sum(1).tolist()
    dist, plan, _, cost = F.ot_fwd(seq[:, :T_len], seq[:, T_len:T_len + R_len], xl, yl, want_cost=True)
    errs = {n: _scaled_err(a.cpu(), gold[n]) for n, a in (("cost", cost), ("T", plan), ("distance", dist))}
    print("\nOT golden: " + "  ".join("%s %.2e" % kv for kv in errs.items()))
    assert max(errs.values()) < 1e-4, errs
    jp = gold["img_pad"].unsqueeze(-1) | gold["txt_pad"].unsqueeze(-2)
    assert (plan.cpu()[jp] == 0).all()
