"""The references, bounds and exact checks of tests/kernel_check.py for the column-sum, embedding, dropout, element-wise
and AdamW kernels.  Runs on the CPU: a correctly rounded output stands for a correct kernel and must pass; each mutation
stands for one kind of kernel bug and must fail, naming the kernel coordinate where it happened.  The keep-bit model is
checked against a simulation of the kernel's bit-sliced comparison for every threshold."""
import math

import numpy as np
import pytest
import torch

import kernel_check as kc

SMS = 132            # H100 SXM: the grid shapes of the column sums below are those of a 132-SM device


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------
# column sums
# ------------------------------------------------------------------------------------------------------------------
def test_colsum_correct_output_passes_and_a_skipped_row_fails():
    M, N = 1000, 264                 # grid.y = 16: a warp's rows are 128 apart, 4 of them per step (512 rows)
    g = _gen(1)
    x = kc.exact_ints(M, N, gen=g)
    out0 = kc.exact_ints(N, gen=g).float()
    ref, bound = kc.colsum_ref(x, out0, SMS)
    lay = kc.colsum_layout()
    kc.assert_equal(ref.float(), ref, lay, "colsum exact")
    # block row 3, warp 5 skipped the row one 4-stride step on (row 29 + 512) in the partial last column block
    bad = ref.clone()
    bad[256:] -= x[541, 256:].double()
    assert x[541, 256:].abs().sum() > 0
    with pytest.raises(AssertionError, match=r"column block 1, lane 0"):
        kc.assert_equal(bad.float(), ref, lay, "colsum exact")
    # random inputs: the fp32 result passes the rounding bound
    xr = (torch.randn(M, N, generator=g, dtype=torch.float64)).to(torch.bfloat16)
    o0 = torch.randn(N, generator=g)
    ref, bound = kc.colsum_ref(xr, o0, SMS)
    assert kc.assert_within(ref.float(), ref, bound, lay, "colsum") <= kc.SAFETY


def test_colsum_grid_matches_the_launch():
    assert kc.colsum_grid_y(1, 8, SMS) == 1
    assert kc.colsum_grid_y(65, 8, SMS) == 2
    assert kc.colsum_grid_y(64 * 528, 8, SMS) == 528 and kc.colsum_grid_y(64 * 528 + 1, 8, SMS) == 528
    assert kc.colsum_grid_y(10 ** 6, 30528, SMS) == 5          # 120 column blocks: ceil(528 / 120)


# ------------------------------------------------------------------------------------------------------------------
# embedding compose and the sorted scatter
# ------------------------------------------------------------------------------------------------------------------
def test_compose_row_missing_its_last_partial_slab():
    M, H, V = 300, 776, 50           # slab 3 holds the 8 columns 768..775
    g = _gen(2)
    src = kc.exact_ints(M + 4, H + 8, gen=g)[:, :H]           # a row slice of a wider buffer
    rows = torch.randperm(M + 4, generator=g)[:M].to(torch.int32)
    rows[::7] = -1
    big = kc.exact_ints(3 * V, H, gen=g)                        # one table in three slots at different row offsets
    idx = [torch.randint(k * V, (k + 1) * V, (M,), generator=g, dtype=torch.int32) for k in range(3)]
    idx[1][::5] = -1
    y, bound = kc.compose_ref(M, H, [(src, rows)], [(big, i) for i in idx], "cpu")
    assert y.abs().max() <= 80
    lay = kc.row_layout()
    kc.assert_equal(y.to(torch.bfloat16), y, lay, "compose exact")
    bad = y.to(torch.bfloat16)
    bad[100, 768:] = 0
    with pytest.raises(AssertionError, match=r"row 100, slab 3, lane 0"):
        kc.assert_equal(bad, y, lay, "compose exact")
    # random inputs: bf16 of the fp32 sum is within the bound
    srcr = torch.randn(M + 4, H, generator=g).to(torch.bfloat16)
    bigr = torch.randn(3 * V, H, generator=g).to(torch.bfloat16)
    y, bound = kc.compose_ref(M, H, [(srcr, rows)], [(bigr, i) for i in idx], "cpu")
    kc.assert_within(y.float().to(torch.bfloat16), y, bound, lay, "compose")


def _sorted_runs(lengths, first=0):
    return torch.cat([torch.full((n,), first + k, dtype=torch.int32) for k, n in enumerate(lengths)])


def test_scatter_sorted_run_that_lost_the_row_at_a_warp_boundary():
    s = _sorted_runs([20, 41, 239, 300])                        # index 1: positions 20..60, across the warp 0/1 end
    M, H, V = s.numel(), 264, 8
    g = _gen(3)
    order = torch.randperm(M, generator=g).to(torch.int32)      # sorted position k reads dy row order[k]
    idx = torch.empty(M, dtype=torch.int32)
    idx[order.long()] = s
    dy = kc.exact_ints(M, H, gen=g)
    dtab0 = kc.exact_ints(V, H, gen=g).float()
    ref, bound = kc.scatter_table_ref(dtab0, dy, idx)
    lay = kc.scatter_sorted_layout(s)
    kc.assert_equal(ref.float(), ref, lay, "scatter_sorted exact")
    bad = ref.clone()
    bad[1] -= dy[order[32].item()].double()                     # the first row of warp 1 was not added
    with pytest.raises(AssertionError, match=r"table row 1, .*: run of 41 at sorted positions 20\.\.60, warps 0\.\.1"):
        kc.assert_equal(bad.float(), ref, lay, "scatter_sorted exact")
    dyr = torch.randn(M, H, generator=g).to(torch.bfloat16)
    ref, bound = kc.scatter_table_ref(dtab0, dyr, idx)
    kc.assert_within(ref.float(), ref, bound, lay, "scatter_sorted")


# ------------------------------------------------------------------------------------------------------------------
# AdamW
# ------------------------------------------------------------------------------------------------------------------
GROUPS = [{"lr": 1e-3 * (i + 1), "weight_decay": 0.0 if i % 3 == 0 else 0.01 * i, "step_size": 9e-4 * (i + 1) * (1 + 0.1 * i),
           "bc2_sqrt": math.sqrt(1 - 0.999 ** (i + 2))} for i in range(8)]
HP = dict(beta1=0.9, beta2=0.999, eps=1e-6, grad_scale=0.5)


def _adamw_fp32(p, m, v, g, gid, mode):
    """the kernel's operations in fp32 (without fused multiply-adds: one more rounding than the kernel per fma)"""
    f = lambda key: torch.tensor([gr[key] for gr in GROUPS], dtype=torch.float32)[gid.long().repeat_interleave(8)]
    lr, wd, step, bc2s = f("lr"), f("weight_decay"), f("step_size"), f("bc2_sqrt")
    b1, b2, eps = (torch.tensor(HP[k], dtype=torch.float32) for k in ("beta1", "beta2", "eps"))
    gr = g * torch.tensor(HP["grad_scale"], dtype=torch.float32)
    if mode == 1:
        p = p * (1 - lr * wd)
        m = (gr - m) * (1 - b1) + m
        v = gr * gr * (1 - b2) + v * b2
        p = p - step * (m / (v.sqrt() / bc2s + eps))
    else:
        m = gr * (1 - b1) + m * b1
        v = gr * gr * (1 - b2) + v * b2
        p = p - step * (m / (v.sqrt() + eps))
        p = torch.where(wd > 0, p + p * (-lr * wd), p)
    return p, m, v


@pytest.mark.parametrize("mode", [0, 1])
def test_adamw_fp32_steps_pass_and_the_neighbouring_blocks_group_fails(mode):
    n = 8 * 805
    g = _gen(4 + mode)
    p, m = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.01
    v = torch.rand(n, generator=g) * 1e-4 + 1e-8
    gid = torch.randint(0, 8, (n // 8,), generator=g, dtype=torch.uint8)
    st = kc.adamw_state(p, m, v)
    lay = kc.adamw_layout(gid)
    for step in range(3):
        grad = torch.randn(n, generator=g) * 0.1
        kc.adamw_step_ref(st, grad, GROUPS, gid, mode=mode, **HP)
        p, m, v = _adamw_fp32(p, m, v, grad, gid, mode)
        for name, t in (("p", p), ("m", m), ("v", v)):
            kc.assert_within(t, st[name], st["e_" + name], lay, "adamw step %d %s" % (step, name))
    # one step in which block b reads the group of block b + 1
    b = int(torch.nonzero(gid[:-1] != gid[1:])[5])
    shifted = gid.clone()
    shifted[b] = gid[b + 1]
    st = kc.adamw_state(p, m, v)
    grad = torch.randn(n, generator=g) * 0.1
    kc.adamw_step_ref(st, grad, GROUPS, gid, mode=mode, **HP)
    bad, _, _ = _adamw_fp32(p, m, v, grad, shifted, mode)
    with pytest.raises(AssertionError, match=r"8-element block %d \(CUDA block %d, thread %d\), group %d"
                       % (b, b // 256, b % 256, int(gid[b]))):
        kc.assert_within(bad, st["p"], st["e_p"], lay, "adamw p")


# ------------------------------------------------------------------------------------------------------------------
# element-wise kernels
# ------------------------------------------------------------------------------------------------------------------
def test_gelu_bwd_rounded_output_passes_and_the_tail_is_named():
    n = 2049
    u = torch.linspace(-20, 20, n, dtype=torch.float64).to(torch.bfloat16)
    dh = torch.randn(n, generator=_gen(6)).to(torch.bfloat16)
    ref, bound = kc.gelu_bwd_ref(dh, u)
    lay = kc.flat8_layout(n)
    kc.assert_within(kc.bf16_round(ref), ref, bound, lay, "gelu_bwd")
    bad = kc.bf16_round(ref)
    bad[2048] *= 1.05
    with pytest.raises(AssertionError, match=r"tail element 0 of 1 \(scalar loop of thread 0, block 1"):
        kc.assert_within(bad, ref, bound, lay, "gelu_bwd")


def test_bits_equal_tells_nan_and_the_sign_of_zero():
    ref = torch.tensor([0.0, -0.0, float("nan"), float("inf"), 1.0], dtype=torch.bfloat16)
    out = ref.clone()
    out.view(torch.int16)[2] = 0x7F81                            # another NaN payload: still NaN
    kc.assert_bits_equal(out, ref, kc.flat8_layout(5))
    out[1] = 0.0
    with pytest.raises(AssertionError, match=r"tail element 1 of 5"):
        kc.assert_bits_equal(out, ref, kc.flat8_layout(5))
    out = ref.clone()
    out[2] = float("inf")
    with pytest.raises(AssertionError, match=r"tail element 2 of 5"):
        kc.assert_bits_equal(out, ref, kc.flat8_layout(5))


# ------------------------------------------------------------------------------------------------------------------
# dropout keep-bits
# ------------------------------------------------------------------------------------------------------------------
P_VALUES = [0.0, 2.0 ** -16, 0.1, 0.25, 1.0 / 3.0, 0.5, 0.75, 0.9, 1.0 - 2.0 ** -16, 0.99999]


def test_thresholds():
    assert [kc.dropout_thresh16(p) for p in P_VALUES] == [0, 1, 6554, 16384, 21845, 32768, 49152, 58982, 65535, 65535]


def _bit_sliced(planes, thresh):
    """the kernel's comparison, restated: 16 planes, most significant first; a threshold bit of 1 keeps only the
    uniforms whose bit is 1 'equal so far', a 0 bit makes the equal-so-far uniforms with a 1 bit 'greater'; keep where
    greater or equal.  planes [16, W], thresh [T] -> words [T, W]"""
    T, W = thresh.shape[0], planes.shape[1]
    gt = np.zeros((T, W), dtype=np.uint32)
    eq = np.full((T, W), 0xFFFFFFFF, dtype=np.uint32)
    for i in range(4):
        for k in range(4):
            b = 15 - (i * 4 + k)
            r = planes[b][None, :]
            one = ((thresh >> np.uint32(b)) & np.uint32(1)).astype(bool)[:, None]
            gt = np.where(one, gt, gt | (eq & r))
            eq = np.where(one, eq & r, eq & ~r)
    return gt | eq


def _planes_of(uniforms):
    """[W, 32] sixteen-bit uniforms -> [16, W] bit-planes"""
    e = np.arange(32, dtype=np.uint32)
    return np.stack([(((uniforms >> np.uint32(b)) & np.uint32(1)) << e).sum(1, dtype=np.uint64).astype(np.uint32)
                     for b in range(16)])


def test_keep_bit_model_equals_the_bit_sliced_comparison_for_every_threshold():
    planes = kc.dropout_planes(6, seed=0x0123456789ABCDEF, offset=2 ** 32 - 9)
    edge = np.array([0, 1, 2, 3, 0x7FFF, 0x8000, 0x8001, 0xFFFE, 0xFFFF, 0x5555, 0xAAAA, 0x00FF, 0xFF00, 6553, 6554,
                     6555, 21845, 32767, 32768, 49152, 58982, 65535, 100, 1000, 10000, 20000, 30000, 40000, 50000, 60000,
                     65000, 65534], dtype=np.uint32)
    planes = np.concatenate([planes, _planes_of(edge[None, :])], axis=1)
    r = kc.uniforms_from_planes(planes)                                     # [W, 32]
    assert np.array_equal(_planes_of(r), planes)
    thresh = np.arange(65536, dtype=np.uint32)
    sliced = _bit_sliced(planes, thresh)                                    # [T, W]
    model = ((r[None, :, :] >= thresh[:, None, None]).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(
        -1, dtype=np.uint64).astype(np.uint32)
    bad = np.argwhere(sliced != model)
    if bad.size:
        t, w = (int(v) for v in bad[0])
        e = int(np.argwhere(((sliced[t, w] ^ model[t, w]) >> np.arange(32, dtype=np.uint32)) & 1)[0, 0])
        pytest.fail("word %d, bit %d, thresh16 %d (p = %r): bit-sliced %d, model %d (uniform %d)"
                    % (w, e, t, t / 65536.0, (int(sliced[t, w]) >> e) & 1, (int(model[t, w]) >> e) & 1, int(r[w, e])))


def test_keep_bit_check_names_word_bit_and_p():
    u = kc.dropout_uniforms(40, seed=5, offset=0)
    p = 0.5
    words = ((u >= kc.dropout_thresh16(p)).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)
    t = torch.from_numpy(words.view(np.int32).copy())
    kc.assert_keep_bits(t, u, p)
    t[17] ^= 1 << 9
    with pytest.raises(AssertionError, match=r"word 17, bit 9 at p = 0\.5"):
        kc.assert_keep_bits(t, u, p)


def test_philox_counters_carry_and_epoch_shift():
    """the counter is one 64-bit number: offset + 4 w + i carries from the low word into the high one, and the epoch
    adds 2^40 per step"""
    a = kc.dropout_planes(4, seed=3, offset=2 ** 32 - 8)
    b = kc.dropout_planes(2, seed=3, offset=2 ** 32)
    assert np.array_equal(a[:, 2:], b)
    assert np.array_equal(kc.dropout_planes(3, seed=3, offset=11, epoch=2), kc.dropout_planes(3, seed=3, offset=11 + 2 * 2 ** 40))
    assert not np.array_equal(kc.dropout_planes(3, seed=3, offset=0), kc.dropout_planes(3, seed=3 + 2 ** 32, offset=0))
