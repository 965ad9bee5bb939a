"""Row kernels through the C ABI vs torch fp32: LayerNorm fwd/bwd (with and without dropout / extra gradient term),
column sums, dropout-bit statistics and determinism, fp32->bf16 cast."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("M,H", [(1000, 768), (333, 1024), (50, 64), (4000, 256), (7, 512), (50, 128), (5000, 256),
                                 (37848, 768), (333, 1280), (100, 2048)])
@pytest.mark.parametrize("with_dx2", [False, True])
@pytest.mark.parametrize("with_drop", [False, True])
def test_layernorm_fwd_bwd(M, H, with_dx2, with_drop):
    from mmf_b200 import functional as F
    torch.manual_seed(M + H)
    y = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    g = (1 + 0.1 * torch.randn(H, device="cuda")).to(torch.bfloat16)
    b = (0.1 * torch.randn(H, device="cuda")).to(torch.bfloat16)
    x, mean, rstd = F.layernorm_fwd(y, g, b)
    yf = y.float().requires_grad_(True)
    gf, bf = g.float().requires_grad_(True), b.float().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(yf, (H,), gf, bf, 1e-12)
    assert rel(x, ref) < 1e-2
    dx = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    dx2 = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    ref.backward(dx.float() + dx2.float() if with_dx2 else dx.float())
    if not with_dx2:
        dx2 = None
    dgamma = torch.zeros(H, device="cuda"); dbeta = torch.zeros(H, device="cuda"); dbias = torch.zeros(H, device="cuda")
    bits = scale = None
    if with_drop:
        keep = torch.rand(M, H, device="cuda") > 0.1
        bits, scale = F.pack_keep_bits(keep), 1 / 0.9
    dy, dz = F.layernorm_bwd(dx, y, mean, rstd, g, dgamma, dbeta, dbias=dbias, dx2=dx2, drop_mask=bits,
                             drop_scale=scale or 1.0)
    assert rel(dy, yf.grad) < 1e-2
    dz_ref = yf.grad * keep.float() / 0.9 if with_drop else yf.grad
    assert rel(dz, dz_ref) < 1e-2
    assert rel(dgamma, gf.grad) < 1e-2 and rel(dbeta, bf.grad) < 1e-2
    # bias gradient = column sum of dz: the streaming kernel (H <= 1024) sums the STORED bf16 dz when there is dropout,
    # otherwise, and in the wide kernel, the fp32 values before rounding are summed - within bf16 rounding of each other
    assert rel(dbias, dz.float().sum(0)) < 4e-3 and rel(dbias, dz_ref.sum(0)) < 1e-2
    # accumulation semantics: a second call adds
    F.layernorm_bwd(dx, y, mean, rstd, g, dgamma, dbeta, dbias=dbias, dx2=dx2, drop_mask=bits, drop_scale=scale or 1.0)
    assert rel(dgamma, 2 * gf.grad) < 1e-2


@pytest.mark.parametrize("H", [768, 2048])
def test_layernorm_rejects_unaligned_rows(H):
    """Both LayerNorm kernels read rows as 16-byte vectors: a row stride that is not a multiple of 8 elements is refused
    with ValueError before anything is launched."""
    from mmf_b200 import functional as F, lib
    M = 64
    padded = torch.randn(M, H + 4, device="cuda").to(torch.bfloat16)
    y_bad = padded[:, :H]
    y = y_bad.contiguous()
    g = torch.ones(H, device="cuda", dtype=torch.bfloat16)
    b = torch.zeros(H, device="cuda", dtype=torch.bfloat16)
    _, mean, rstd = F.layernorm_fwd(y, g, b)
    dx = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    dgamma, dbeta = torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda")
    n0 = lib.launch_count()
    with pytest.raises(ValueError, match="ldy"):
        F.layernorm_fwd(y_bad, g, b)
    with pytest.raises(ValueError, match="ldy"):
        F.layernorm_bwd(dx, y_bad, mean, rstd, g, dgamma, dbeta)
    with pytest.raises(ValueError, match="lddx"):
        F.layernorm_bwd(y_bad, y, mean, rstd, g, dgamma, dbeta)
    assert lib.launch_count() == n0


def test_colsum_and_cast():
    from mmf_b200 import functional as F
    x = torch.randn(3000, 2304, device="cuda").to(torch.bfloat16)
    out = torch.ones(2304, device="cuda")
    F.colsum(x, out)
    assert rel(out, 1 + x.float().sum(0)) < 1e-4
    src = torch.randn(1000003, device="cuda")
    dst = torch.empty(1000003, device="cuda", dtype=torch.bfloat16)
    F.cast_f32_bf16(src, dst)
    assert torch.equal(dst, src.to(torch.bfloat16))


def test_dropout_bits_statistics_and_determinism():
    from mmf_b200 import functional as F
    a = F.dropout_bits((4096,), 768, 0.1, seed=7, offset=0, device="cuda")
    b = F.dropout_bits((4096,), 768, 0.1, seed=7, offset=0, device="cuda")
    c = F.dropout_bits((4096,), 768, 0.1, seed=8, offset=0, device="cuda")
    assert torch.equal(a, b) and not torch.equal(a, c)
    keep = F.unpack_keep_bits(a, 768).float()
    assert abs(keep.mean().item() - 0.9) < 2e-3
    assert abs(keep.mean(0).std().item() - (0.9 * 0.1 / 4096) ** 0.5) < 2e-3      # columns are independent draws
    assert torch.equal(F.pack_keep_bits(F.unpack_keep_bits(a, 768)), a)
