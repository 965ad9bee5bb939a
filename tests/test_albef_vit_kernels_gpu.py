"""The kernels the ALBEF ViT adds, element by element against fp64 (tests/kernel_check.py), at tile edges: M and N not
multiples of 128, N not a multiple of 32 (a partial keep word per row).
  * MMFB_EPI_BIAS_GELU_DROP:  C = u = acc + bias, C2 = keep * scale * gelu(u)
  * MMFB_EPI_GELU_DROP_BWD:   C = acc * keep * scale * gelu'(aux)
  * mmfb_dropout_path_bits / _epoch: bit for bit against a numpy model of the Philox stream, keep fractions of elements and
    samples within a binomial bound, and the epoch twin's draws."""
import math

import numpy as np
import pytest
import torch

import kernel_check as KC

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _operands(M, N, K, gen, b_mn=False):
    a = (torch.randn(M, K, generator=gen) * 0.5).to(torch.bfloat16).to(DEV)
    b = (torch.randn(K, N, generator=gen) * 0.5 if b_mn else torch.randn(N, K, generator=gen) * 0.5).to(torch.bfloat16)
    return a, b.to(DEV)


def _keep(M, N, p, gen):
    from mmf_b200 import functional as F
    keep = torch.rand(M, N, generator=gen) >= p
    return keep.to(DEV), F.pack_keep_bits(keep.to(DEV))


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(200, 328, 96), (130, 776, 200)])
def test_bias_gelu_drop_vs_fp64(M, N, K, block_n):
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    g = torch.Generator().manual_seed(M + N + K + block_n)
    a, b = _operands(M, N, K, g)
    bias = (torch.randn(N, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
    keep, bits = _keep(M, N, 0.3, g)
    scale = 1.0 / 0.7
    u, h = F.gemm(a, b, epi=lib.EPI_BIAS_GELU_DROP, bias=bias, drop_mask=bits, drop_scale=scale, block_n=block_n)
    ref, absab = KC.gemm_ref(a, b)
    ref = ref + bias.double()
    bu = KC.gemm_bound(ref, absab, bias.double().abs())
    KC.assert_within(u, ref, bu, KC.gemm_layout(block_n), "u")
    href = torch.where(keep, KC.gelu64(ref) * scale, torch.zeros_like(ref))
    # (as test_gemm_edges_gpu.py bounds the gelu epilogue: u's error through gelu', the erf approximation, |Phi err| <=
    # 2^-22 times |u|), then the fp32 product with scale and the bf16 rounding
    bh = KC.U_BF16 * href.abs() + scale * (KC.gelu_grad64(ref).abs() * KC.U_ACC * (absab + bias.double().abs()) +
                                           2.0 ** -22 * ref.abs() + KC.U_F32 * href.abs())
    KC.assert_within(h, href, torch.where(keep, bh, torch.zeros_like(bh)), KC.gemm_layout(block_n), "keep * scale * gelu(u)")
    assert torch.equal(h[~keep], torch.zeros_like(h[~keep]))                # dropped: exact zeros


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(200, 328, 96), (130, 776, 200)])
def test_gelu_drop_bwd_vs_fp64(M, N, K, block_n):
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    g = torch.Generator().manual_seed(7 * M + N + K + block_n)
    a, b = _operands(M, N, K, g, b_mn=True)
    u = (torch.randn(M, N, generator=g) * 1.5).to(torch.bfloat16).to(DEV)
    keep, bits = _keep(M, N, 0.5, g)
    scale = 2.0
    du = F.gemm(a, b, b_mn=True, epi=lib.EPI_GELU_DROP_BWD, aux=u, drop_mask=bits, drop_scale=scale, block_n=block_n)
    acc, absab = KC.gemm_ref(a, b.t())
    gg = KC.gelu_grad64(u.double())
    ref = torch.where(keep, acc * scale * gg, torch.zeros_like(acc))
    # the accumulation error through gelu'(u), gelu'(u) in fp32 with the erf / ex2 approximations (|err| <= 2^-21 (1 + |u|),
    # kernel_check.gelu_bwd_ref), the fp32 products and the bf16 rounding
    bound = KC.U_BF16 * ref.abs() + scale * (gg.abs() * KC.U_ACC * absab + acc.abs() * 2.0 ** -21 * (1 + u.double().abs())
                                             + 2 * KC.U_F32 * (acc * gg).abs())
    KC.assert_within(du, ref, torch.where(keep, bound, torch.zeros_like(bound)), KC.gemm_layout(block_n), "du")
    assert torch.equal(du[~keep], torch.zeros_like(du[~keep]))


def test_hidden_dropout_epilogues_refuse_bad_arguments():
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    g = torch.Generator().manual_seed(1)
    a, b = _operands(64, 96, 64, g)
    _, bits = _keep(64, 96, 0.1, g)
    with pytest.raises(ValueError, match="keep bits"):
        F.gemm(a, b, epi=lib.EPI_BIAS_GELU_DROP, drop_scale=1.1)
    with pytest.raises(ValueError, match="keep bits"):
        F.gemm(a, b, epi=lib.EPI_BIAS_GELU_DROP, drop_mask=bits[:, :2].contiguous(), drop_scale=1.1)        # ldmask 2 < ceil(96/32)
    with pytest.raises(ValueError, match="drop_scale"):
        F.gemm(a, b, epi=lib.EPI_BIAS_GELU_DROP, drop_mask=bits, drop_scale=0.0)
    at, bt = _operands(64, 96, 64, g, b_mn=True)
    with pytest.raises(ValueError, match="aux"):
        F.gemm(at, bt, b_mn=True, epi=lib.EPI_GELU_DROP_BWD, drop_mask=bits, drop_scale=1.1)
    with pytest.raises(ValueError, match="unsupported"):
        F.gemm(at, bt, b_mn=True, epi=lib.EPI_BIAS_GELU_DROP, drop_mask=bits, drop_scale=1.1)


def _sample_model(B, nwords, seed, offset, p_path, epoch=0):
    """sample keep of the model: high 16 bits of the first Philox output at offset + (epoch << 40) + 4 nwords + b"""
    ctr = np.uint64((offset + (epoch << 40) + 4 * nwords) % 2 ** 64) + np.arange(B, dtype=np.uint64)
    r = KC.philox4x32_7(seed, ctr)[0].astype(np.uint32)
    return (r >> np.uint32(16)) >= KC.dropout_thresh16(p_path)


def _epoch():
    """the device step counter functional.dropout_path_bits mixes in once a CUDA graph has been captured in this process"""
    from mmf_b200 import functional as F
    ep = F.dropout_epoch(DEV)
    return 0 if ep is None else int(ep.item())


def _expected_words(B, S, H, seed, offset, p, p_path, epoch=0):
    W = (H + 31) // 32
    n = B * S * W
    unif = KC.dropout_uniforms(n, seed, offset, epoch)
    elem = (unif >= KC.dropout_thresh16(p)).astype(np.uint64)
    words = (elem << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32).reshape(B, S * W)
    keep = _sample_model(B, n, seed, offset, p_path, epoch)
    return np.where(keep[:, None], words, 0).reshape(B * S, W), keep


@pytest.mark.parametrize("p,p_path", [(0.1, 0.1), (0.5, 0.5), (0.0, 0.3)])
def test_path_bits_match_the_philox_model(p, p_path):
    from mmf_b200 import functional as F
    B, S, H = 37, 197, 328                                   # H % 32 != 0: the last word of a row is partial
    seed, offset = 0x1234_5678_9ABC, 4096
    got = F.dropout_path_bits(B, S, H, p, p_path, seed, offset, DEV)
    assert tuple(got.shape) == (B * S, (H + 31) // 32)
    want, _ = _expected_words(B, S, H, seed, offset, p, p_path, epoch=_epoch())
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want)
    # the element words of the kept samples are mmfb_dropout_bits' words at the same counter
    plain = F.dropout_bits((B * S,), H, p, seed, offset, DEV).view(B, S, -1)
    kept = got.view(B, S, -1).ne(0).any(2).any(1)
    assert torch.equal(got.view(B, S, -1)[kept], plain[kept])


def _binomial_ok(k, n, q):
    """k successes of n with probability q: within 6 standard deviations"""
    return abs(k - n * q) <= 6.0 * math.sqrt(n * q * (1 - q)) + 1


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_path_bits_keep_fractions(p):
    from mmf_b200 import functional as F
    B, S, H = 4096, 3, 328
    words = F.dropout_path_bits(B, S, H, p, p, 99, 0, DEV)
    keep = F.unpack_keep_bits(words, H).view(B, S * H)
    sample_kept = keep.any(1)
    assert _binomial_ok(int(sample_kept.sum()), B, 1 - p)
    # every row of a dropped sample is cleared; a kept sample's elements are kept with 1 - p
    assert not keep[~sample_kept].any()
    assert _binomial_ok(int(keep[sample_kept].sum()), int(sample_kept.sum()) * S * H, 1 - p)


def test_path_bits_epoch_twin():
    from mmf_b200 import lib
    B, S, H = 64, 5, 200
    seed, offset = 7, 1 << 20
    W = (H + 31) // 32
    draws = []
    for e in (1, 2):
        out = torch.empty(B * S, W, dtype=torch.int32, device=DEV)
        epoch = torch.tensor([e], dtype=torch.int64, device=DEV)
        lib.check(lib.LIB.mmfb_dropout_path_bits_epoch(out.data_ptr(), B * S, H, S, seed, offset, epoch.data_ptr(), 0.5,
                                                        0.5, lib._stream_ptr()))
        torch.cuda.synchronize()
        want, _ = _expected_words(B, S, H, seed, offset, 0.5, 0.5, epoch=e)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want)
        draws.append(out)
        # the same counter without an epoch: the plain entry point at offset + (e << 40)
        same = torch.empty_like(out)
        lib.check(lib.LIB.mmfb_dropout_path_bits(same.data_ptr(), B * S, H, S, seed, offset + (e << 40), 0.5, 0.5,
                                                  lib._stream_ptr()))
        assert torch.equal(out, same)
    assert not torch.equal(draws[0], draws[1])


def test_path_bits_refuse_bad_arguments():
    from mmf_b200 import functional as F
    from mmf_b200 import lib
    with pytest.raises(ValueError, match="multiple"):
        out = torch.empty(10, 1, dtype=torch.int32, device=DEV)
        lib.check(lib.LIB.mmfb_dropout_path_bits(out.data_ptr(), 10, 32, 3, 1, 0, 0.1, 0.1, lib._stream_ptr()))
    with pytest.raises(ValueError, match="p_path"):
        F.dropout_path_bits(2, 3, 32, 0.1, 1.0, 1, 0, DEV)
    with pytest.raises(ValueError, match="p_path"):
        F.dropout_path_bits(2, 3, 32, -0.1, 0.1, 1, 0, DEV)
