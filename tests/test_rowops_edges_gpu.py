"""Row kernels at their edges, every element against fp64 (tests/kernel_check.py): LayerNorm forward / backward with a
partial last 256-column slab in every instantiation of both backward kernels and row counts around the persistent
grid; cross-entropy rows at vocabulary edges, extreme and constant logits, strided rows and out-of-range labels; the
AdamW bf16 parameter copy."""
import math

import pytest
import torch

import kernel_check as kc

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bwd_sum_terms(M):
    """depth of the fp32 column-sum chain of both LayerNorm backward kernels: rows per warp of the grid-strided loop,
    the 8-warp block sum, one atomic per block (grid <= 2 blocks per SM)"""
    grid = min((M + 7) // 8, 2 * _sms())
    return (M + 8 * grid - 1) // (8 * grid) + 8 + grid


# H: a partial last slab for NV = 1, 2, 3, 4 (streaming kernel) and 5, 6, 8 (wide kernel)
LN_H = [8, 72, 264, 520, 776, 1032, 1288, 2040]


@pytest.mark.parametrize("H", LN_H)
@pytest.mark.parametrize("M_kind", ["1", "7", "9", "grid+1"])
@pytest.mark.parametrize("with_dx2", [False, True])      # the streaming kernel has its own (NV, ST) instantiation for each
def test_layernorm_edges(H, M_kind, with_dx2):
    from mmf_b200 import functional as F
    M = 2 * _sms() * 8 + 1 if M_kind == "grid+1" else int(M_kind)
    i = LN_H.index(H)
    with_drop = bool((i // 2) % 2) ^ (M_kind == "9") ^ with_dx2
    g = torch.Generator(device="cuda").manual_seed(M * 10000 + H)
    y = (torch.randn(M, H, generator=g, device="cuda") * 2 + 0.5).to(torch.bfloat16)
    gam = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(torch.bfloat16)
    bet = (0.1 * torch.randn(H, generator=g, device="cuda")).to(torch.bfloat16)
    x, mean, rstd = F.layernorm_fwd(y, gam, bet)
    fw = kc.layernorm_ref(y, gam, bet)
    lay = kc.row_layout()
    tag = "ln M%d H%d dx2=%d drop=%d" % (M, H, with_dx2, with_drop)
    worst = {"mean": kc.assert_within(mean, fw["mean"], fw["b_mean"], lay, tag + " mean"),
             "rstd": kc.assert_within(rstd, fw["rstd"], fw["b_rstd"], lay, tag + " rstd"),
             "x": kc.assert_within(x, fw["x"], fw["b_x"], lay, tag + " x")}
    dx = torch.randn(M, H, generator=g, device="cuda").to(torch.bfloat16)
    dx2 = torch.randn(M, H, generator=g, device="cuda").to(torch.bfloat16) if with_dx2 else None
    bits = keep = None
    dsc = 1.0
    if with_drop:
        keep = torch.rand(M, H, generator=g, device="cuda") > 0.1
        bits, dsc = F.pack_keep_bits(keep), 1 / 0.9
    dgamma, dbeta, dbias = (torch.zeros(H, device="cuda") for _ in range(3))
    dy, dz = F.layernorm_bwd(dx, y, mean, rstd, gam, dgamma, dbeta, dbias=dbias, dx2=dx2, drop_mask=bits, drop_scale=dsc)
    torch.cuda.synchronize()
    n = _bwd_sum_terms(M)
    bw = kc.layernorm_bwd_ref(fw, dx, gam, dx2=dx2, keep=keep, dscale=dsc, n_sum_terms=n)
    worst["dy"] = kc.assert_within(dy, bw["dy"], bw["b_dy"], lay, tag + " dy")
    worst["dz"] = kc.assert_within(dz, bw["dz"], bw["b_dz"], lay, tag + " dz")
    worst["dgamma"] = kc.assert_within(dgamma, bw["dgamma"], bw["b_dgamma"], lay, tag + " dgamma")
    worst["dbeta"] = kc.assert_within(dbeta, bw["dbeta"], bw["b_dbeta"], lay, tag + " dbeta")
    if with_drop and H <= 1024:
        # the streaming kernel sums the bf16 dz it stores (what the consumer reads): check against those values
        dz64 = dz.double()
        ref_b, b_b = dz64.sum(0), kc.U_F32 * n * dz64.abs().sum(0)
    else:
        # otherwise the fp32 values before rounding are summed
        ref_b = bw["dz"].sum(0)
        b_b = bw["e_dz_f32"].sum(0) + kc.U_F32 * n * bw["dz"].abs().sum(0)
    worst["dbias"] = kc.assert_within(dbias, ref_b, b_b, lay, tag + " dbias")
    print("%s: %s" % (tag, " ".join("%s=%.3f" % kv for kv in worst.items())))


def _ce_ref(z, labels, V, scale):
    """fp64 loss per row and d(logits); bounds.  The kernel sums exp2(z log2e - max log2e) in fp32 over 8 ceil(V/2048)
    terms per thread and a 13-level block tree; each exponent is rounded (2^-24 (|z| + |max|) log2e) and evaluated by
    exp2f (2 ulp)."""
    z64 = z.double()
    mx = z64.amax(1, keepdim=True)
    lse = mx + torch.log(torch.exp(z64 - mx).sum(1, keepdim=True))
    lab = labels.clamp(0, V - 1)
    zl = z64.gather(1, lab[:, None])
    loss = (lse - zl).squeeze(1)
    nterm = 8 * ((V + 2047) // 2048) + 13
    e_exp = kc.U_F32 * kc.LOG2E * (z64.abs().amax(1, keepdim=True) + mx.abs()) * 2 + 2.0 ** -22
    rel_sum = kc.U_F32 * nterm + kc.LN2 * e_exp
    # loss = max + log(sum) - z[label]: relative error of the sum, logf (2 ulp of |log sum| <= 11), the two fp32 adds
    b_loss = (rel_sum + 2.0 ** -21 + kc.U_F32 * (mx.abs() + zl.abs() + (lse - zl).abs()) * 2).squeeze(1)
    p = torch.exp(z64 - lse)
    grad = (p - torch.nn.functional.one_hot(lab, V).double()) * scale
    # p * (scale / sum): relative error ln2 e_exp + the sum's + the division and product (2^-23); p - scale rounds once
    # (2^-24); values below fp32's normal range flush to zero (2^-126 absolute); bf16 output
    b_grad = (kc.U_BF16 * grad.abs() + scale * p * (rel_sum + kc.LN2 * e_exp + 2.0 ** -23) + kc.U_F32 * grad.abs()
              + scale * 2.0 ** -126)
    return loss, b_loss, grad, b_grad


@pytest.mark.parametrize("V", [8, 2056, 30528])
def test_ce_rows_edges(V):
    """labels 0 and V-1, ignored rows, logits of +-80, a constant row, rows of a wider buffer (ldz > V)"""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(V)
    M = 9
    buf = (torch.randn(M, V + 24, generator=g, device="cuda") * 3).to(torch.bfloat16)
    buf[2, :V] = torch.where(torch.rand(V, generator=g, device="cuda") < 0.5, 80.0, -80.0).to(torch.bfloat16)
    buf[3, :V] = 1.5                                                    # constant row: uniform softmax
    buf[4, V - 1] = 80.0                                                # one dominant logit at the label
    z = buf[:, :V]
    labels = torch.tensor([0, V - 1, V // 2, 0, V - 1, -1, 1 % V, V - 2, 3 % V], device="cuda")
    scale = 0.25
    zin, pad_before = z.clone(), buf[:, V:].clone()
    loss_sum = torch.zeros((), device="cuda")
    row_loss = torch.empty(M, device="cuda")
    F.ce_rows(z, labels, -1, scale, loss_sum, row_loss)
    torch.cuda.synchronize()
    loss, b_loss, grad, b_grad = _ce_ref(zin, labels, V, scale)
    act = labels != -1
    lay = kc.row_layout()
    w1 = kc.assert_within(row_loss[act], loss[act], b_loss[act], lay, "ce V%d row_loss" % V)
    w2 = kc.assert_within(z[act], grad[act], b_grad[act], lay, "ce V%d d(logits)" % V)
    assert torch.equal(z[~act].float(), torch.zeros_like(z[~act].float())) and torch.equal(row_loss[~act], torch.zeros(1, device="cuda").expand(int((~act).sum())))
    assert torch.equal(buf[:, V:], pad_before)                          # the columns past V of each row are untouched
    # loss_sum: one fp32 atomic add per row
    kc.assert_within(loss_sum.reshape(1), loss[act].sum().reshape(1),
                     (kc.U_F32 * M * loss[act].abs().sum() + b_loss[act].sum()).reshape(1), kc.flat_layout(),
                     "ce V%d loss_sum" % V)
    print("ce V%d: row_loss %.3f d(logits) %.3f" % (V, w1, w2))


def test_ce_rows_labels_outside_the_vocabulary_are_ignored():
    """A label outside [0, V) that is not ignore_index is treated like ignore_index (include/mmfb200.h): zero gradient,
    row_loss 0, nothing added to the summed loss."""
    from mmf_b200 import functional as F
    V = 2056
    g = torch.Generator(device="cuda").manual_seed(1)
    z = (torch.randn(4, V, generator=g, device="cuda") * 3).to(torch.bfloat16)
    labels = torch.tensor([V, -5, 5, V + 100], device="cuda")
    zin = z.clone()
    loss_sum = torch.zeros((), device="cuda")
    row_loss = torch.full((4,), 9.0, device="cuda")
    F.ce_rows(z, labels, -1, 1.0, loss_sum, row_loss)
    torch.cuda.synchronize()
    out = [0, 1, 3]
    assert torch.equal(z[out].float(), torch.zeros(3, V, device="cuda"))
    assert torch.equal(row_loss[out], torch.zeros(3, device="cuda"))
    loss, b_loss, _, _ = _ce_ref(zin[2:3], labels[2:3], V, 1.0)
    kc.assert_within(loss_sum.reshape(1), loss, b_loss, kc.flat_layout(), "loss_sum of the one valid row")


@pytest.mark.parametrize("n", [8, 2056, 8008])
@pytest.mark.parametrize("mode", [0, 1])
def test_adamw_bf16_copy_is_the_rounded_parameter(n, mode):
    """with 8 hyper-parameter groups, the bf16 compute copy equals p.to(bfloat16) bit for bit, for every element"""
    from mmf_b200 import functional as F
    g = torch.Generator(device="cuda").manual_seed(n + mode)
    p = torch.randn(n, generator=g, device="cuda")
    m = torch.randn(n, generator=g, device="cuda") * 0.01
    v = torch.rand(n, generator=g, device="cuda") * 1e-4
    grad = torch.randn(n, generator=g, device="cuda") * 0.1
    gid = torch.randint(0, 8, (n // 8,), generator=g, device="cuda").to(torch.uint8)
    groups = [{"lr": 1e-3 * (i + 1), "weight_decay": 0.01 * (i % 3), "step_size": 1e-3 * (i + 1) * 0.9,
               "bc2_sqrt": math.sqrt(1 - 0.999 ** (i + 1))} for i in range(8)]
    pb = torch.full((n,), 3.0, device="cuda", dtype=torch.bfloat16)
    p0 = p.clone()
    F.adamw(p, grad, m, v, groups, beta1=0.9, beta2=0.999, eps=1e-6, mode=mode, group_of_block=gid, param_bf16=pb)
    torch.cuda.synchronize()
    assert not torch.equal(p, p0)
    assert torch.equal(pb, p.to(torch.bfloat16))
