"""The kernels the product library does NOT run by default but keeps for A/B timing (MMFB_LN_BWD=pair|tile|stream|lean)
against the default ones, in one process (the switches are read per call).  Part of the default `-m gpu` suite: a variant
that is kept must stay correct."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("variant,M,H", [("pair", 1000, 768), ("tile", 1000, 768), ("tile", 37848, 768), ("pair", 333, 1024),
                                         ("tile", 50, 128), ("pair", 7, 512), ("stream", 1000, 768), ("stream", 37848, 768),
                                         ("stream", 333, 1024), ("stream", 50, 128), ("stream", 7, 512), ("stream", 5000, 256),
                                         ("lean", 1000, 768)])
def test_layernorm_backward_variants_match_the_default(variant, M, H):
    from mmf_b200 import functional as F
    torch.manual_seed(0)
    dx = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    dx2 = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    y = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    g = (1.0 + 0.1 * torch.randn(H, device="cuda")).to(torch.bfloat16)
    b = torch.zeros(H, device="cuda", dtype=torch.bfloat16)
    _, mean, rstd = F.layernorm_fwd(y, g, b)
    bits = F.dropout_bits((M,), H, 0.1, 3, 0, "cuda")

    def run(variant, with_dx2, with_drop):
        if variant:
            os.environ["MMFB_LN_BWD"] = variant
        else:
            os.environ.pop("MMFB_LN_BWD", None)
        dg, db, dbias = (torch.zeros(H, device="cuda") for _ in range(3))
        dy, dz = F.layernorm_bwd(dx, y, mean, rstd, g, dg, db, dbias=dbias, dx2=dx2 if with_dx2 else None,
                                 drop_mask=bits if with_drop else None, drop_scale=1.0 / 0.9)
        torch.cuda.synchronize()
        return dy.float(), dz.float(), dg, db, dbias
    try:
        for with_dx2 in (False, True):
            for with_drop in (False, True):
                ref = run(None, with_dx2, with_drop)
                got = run(variant, with_dx2, with_drop)
                for r, t in zip(ref[:2], got[:2]):      # same row arithmetic; FMA contraction may flip a last bf16 bit
                    assert (r - t).abs().max() <= 1e-2 * r.abs().max() and (r != t).float().mean() < 0.01
                for r, t in zip(ref[2:], got[2:]):      # sums: different order; dbias from fp32 values instead of stored bf16
                    assert (r - t).abs().max() <= 4e-3 * r.abs().max().clamp_min(1.0)
    finally:
        os.environ.pop("MMFB_LN_BWD", None)
