"""wgmma GEMM vs torch fp32 matmul of the same bf16 operands (bf16 tolerance 1e-2)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def _mk(rows, cols, mn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(rows, cols, generator=g, device="cuda", dtype=torch.float32) * 0.5
    t = t.to(torch.bfloat16)
    # logical [rows, K]; stored transposed when MN-major
    return (t.t().contiguous(), t) if mn else (t, t)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K,bn", [(128, 256, 64, 256), (256, 512, 256, 256), (200, 768, 1000, 256),
                                      (456, 2304, 768, 256), (456, 768, 3072, 128), (64, 128, 72, 128)])
def test_gemm_layouts(a_mn, b_mn, M, N, K, bn):
    from mmf_b200 import functional as F, lib
    if a_mn and M % 8:
        pytest.skip("MN-major A needs M % 8 == 0")
    a_st, a = _mk(M, K, a_mn, 1)
    b_st, b = _mk(N, K, b_mn, 2)
    c = F.gemm(a_st, b_st, a_mn=a_mn, b_mn=b_mn, epi=lib.EPI_BIAS, block_n=bn)
    ref = a.float() @ b.float().t()
    torch.cuda.synchronize()
    err = rel(c, ref)
    print("gemm a_mn=%d b_mn=%d %dx%dx%d bn=%d rel=%.3e" % (a_mn, b_mn, M, N, K, bn, err))
    assert err < 1e-2


def test_gemm_epilogues():
    from mmf_b200 import functional as F, lib
    M, N, K = 456, 768, 768
    _, a = _mk(M, K, False, 3)
    _, w = _mk(N, K, False, 4)
    bias = (torch.randn(N, device="cuda") * 0.5).to(torch.bfloat16)
    resid = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    acc = a.float() @ w.float().t()
    # bias
    c = F.gemm(a, w, epi=lib.EPI_BIAS, bias=bias)
    assert rel(c, acc + bias.float()) < 1e-2
    # bias + gelu (two outputs)
    u, h = F.gemm(a, w, epi=lib.EPI_BIAS_GELU, bias=bias)
    uref = acc + bias.float()
    assert rel(u, uref) < 1e-2
    assert rel(h, torch.nn.functional.gelu(uref)) < 1e-2
    # bias + dropout + residual
    keep = torch.rand(M, N, device="cuda") > 0.1
    words = torch.zeros(M, N // 32, dtype=torch.int64, device="cuda")
    kb = keep.view(M, N // 32, 32).to(torch.int64)
    for j in range(32):
        words |= kb[:, :, j] << j
    words = (words & 0xFFFFFFFF)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
    y = F.gemm(a, w, epi=lib.EPI_BIAS_DROP_RESID, bias=bias, aux=resid, drop_mask=words, drop_scale=1 / 0.9)
    yref = (acc + bias.float()) * keep.float() / 0.9 + resid.float()
    assert rel(y, yref) < 1e-2
    # dgrad with gelu' and with residual add: B is MN-major (W stored [K_out, N_in])
    _, dy = _mk(M, N, False, 5)
    wk = (torch.randn(N, 1024, device="cuda") * 0.05).to(torch.bfloat16)   # [out=N(K here), in=1024]
    pre = torch.randn(M, 1024, device="cuda").to(torch.bfloat16)
    dacc = dy.float() @ wk.float()
    du = F.gemm(dy, wk, b_mn=True, epi=lib.EPI_GELU_BWD, aux=pre)
    x = pre.float()
    gp = 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5
    assert rel(du, dacc * gp) < 1e-2
    dx = F.gemm(dy, wk, b_mn=True, epi=lib.EPI_ADD_AUX, aux=pre)
    assert rel(dx, dacc + x) < 1e-2
    # wgrad: dW[out,in] += dY^T X, split-K fp32 reductions
    xin = torch.randn(M, 1024, device="cuda").to(torch.bfloat16)
    for splits in (1, 3, 8):
        dw = torch.zeros(N, 1024, device="cuda", dtype=torch.float32)
        F.gemm(dy, xin, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=splits)
        F.gemm(dy, xin, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=splits)
        assert rel(dw, 2 * (dy.float().t() @ xin.float())) < 1e-2


def test_gemm_large_persistent():
    """many tiles and k-blocks: exercises the smem ring's barrier phase logic"""
    from mmf_b200 import functional as F, lib
    M, N, K = 14592, 3072, 768
    _, a = _mk(M, K, False, 7)
    _, w = _mk(N, K, False, 8)
    c = F.gemm(a, w, epi=lib.EPI_BIAS)
    ref = (a.float() @ w.float().t())
    assert rel(c, ref) < 1e-2
    # a second, different call right after (stale-barrier reuse across launches)
    c2 = F.gemm(a[:1000], w[:512], epi=lib.EPI_BIAS)
    assert rel(c2, ref[:1000, :512]) < 1e-2


def test_gemm_bad_args():
    from mmf_b200 import functional as F
    a = torch.zeros(16, 60, device="cuda", dtype=torch.bfloat16)
    b = torch.zeros(16, 60, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        F.gemm(a, b)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("M,N,K,bn", [(256, 512, 256, 256), (384, 768, 1000, 256), (456, 2304, 768, 256),
                                      (1160, 768, 3072, 128), (14592, 768, 768, 256)])
def test_gemm_cluster_multicast(a_mn, b_mn, M, N, K, bn):
    """the `cluster` field of the ABI (kept for compatibility) must not change results: even, odd and many-tile counts
    computed with cluster=1 and cluster=2 are equal bit for bit."""
    from mmf_b200 import functional as F, lib
    a_st, a = _mk(M, K, a_mn, 11)
    b_st, b = _mk(N, K, b_mn, 12)
    c1 = F.gemm(a_st, b_st, a_mn=a_mn, b_mn=b_mn, epi=lib.EPI_BIAS, block_n=bn, cluster=1)
    c2 = F.gemm(a_st, b_st, a_mn=a_mn, b_mn=b_mn, epi=lib.EPI_BIAS, block_n=bn, cluster=2)
    torch.cuda.synchronize()
    assert torch.equal(c1, c2)
    assert rel(c2, a.float() @ b.float().t()) < 1e-2


def test_gemm_cluster_epilogues_and_splitk():
    from mmf_b200 import functional as F, lib
    M, N, K = 1000, 768, 768
    _, a = _mk(M, K, False, 13)
    _, w = _mk(N, K, False, 14)
    bias = (torch.randn(N, device="cuda") * 0.5).to(torch.bfloat16)
    resid = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    u1, h1 = F.gemm(a, w, epi=lib.EPI_BIAS_GELU, bias=bias, cluster=1)
    u2, h2 = F.gemm(a, w, epi=lib.EPI_BIAS_GELU, bias=bias, cluster=2)
    assert torch.equal(u1, u2) and torch.equal(h1, h2)
    y1 = F.gemm(a, w, epi=lib.EPI_BIAS_DROP_RESID, bias=bias, aux=resid, cluster=1)
    y2 = F.gemm(a, w, epi=lib.EPI_BIAS_DROP_RESID, bias=bias, aux=resid, cluster=2)
    assert torch.equal(y1, y2)
    _, dy = _mk(M, N, False, 15)
    xin = torch.randn(M, 1024, device="cuda").to(torch.bfloat16)
    ref = dy.float().t() @ xin.float()
    for splits in (1, 3, 7):
        dw = torch.zeros(N, 1024, device="cuda", dtype=torch.float32)
        F.gemm(dy, xin, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=splits, cluster=2)
        assert rel(dw, ref) < 1e-2
