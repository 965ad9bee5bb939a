"""The persistent GEMM's schedule edges, every element against fp64 (tests/kernel_check.py through the checker of
test_gemm_edges_gpu): work-unit counts around the SM count (fewer units than SMs, one per SM, one or two more, several
per CTA with odd and even counts), one k-block and K tails, M and N tails in the last tile, split-K counts that do not
divide by the grid, back-to-back launches of different shapes in one stream and in one CUDA graph, and the bench shapes
of the four projections with their dgrad and wgrad."""
import pytest
import torch

from test_gemm_edges_gpu import COMBOS, EPI_NAMES, run_and_check

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _unit_counts():
    n = _sms()
    return [1, n - 1, n, n + 1, 2 * n, 2 * n + 1, 3 * n]


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("a_mn,b_mn,epi", COMBOS)
def test_gemm_work_unit_counts(a_mn, b_mn, epi, bn):
    """one n-tile with an N tail, M = 128 u - 40 (an M tail) so that there are exactly u work units"""
    N = bn - 56
    free_k = a_mn and b_mn
    worst = 0.0
    for i, u in enumerate(_unit_counts()):
        M = 128 * u - 40
        K = (64, 72, 40, 136, 200, 8, 64)[i] if not free_k else (64, 65, 1, 127, 200, 7, 64)[i]
        worst = max(worst, run_and_check(a_mn, b_mn, epi, M, N, K, bn, seed=1000 + 10 * i + epi,
                                         with_bias=(i % 3 != 2), with_aux=(i % 4 != 3)))
    print("persistent a_mn=%d b_mn=%d epi=%s bn=%d: worst |err|/bound %.3f" % (a_mn, b_mn, EPI_NAMES[epi], bn, worst))


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", [0, 1, 2])
def test_gemm_several_n_tiles_per_cta(epi, bn):
    """three n-tiles per m-tile with the N tail in the last, odd and even tiles per CTA"""
    n = _sms()
    N = 2 * bn + 136
    for i, tiles_m in enumerate((n // 3 + 1, (2 * n) // 3 + 1, n + 5)):
        run_and_check(0, 0, epi, 128 * tiles_m - 72, N, 200, bn, seed=50 + i)


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_split_k_not_dividing_the_grid(bn):
    """(tiles x splits) around and above the SM count, not a multiple of it"""
    n = _sms()
    N = bn
    for tiles_m, splits in ((n + 1, 3), (n // 2 + 1, 5), (2 * n - 1, 2)):
        run_and_check(1, 1, 5, 128 * tiles_m, N, 64 * 7 + 5, bn, seed=splits, splits=splits)


def _mk(rows, cols, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(rows, cols, generator=g, device="cuda") * 0.5).to(torch.bfloat16)


def _back_to_back_calls():
    """different shapes, epilogues and tile widths, launched without a synchronisation between them"""
    from mmf_b200 import functional as F, lib
    n = _sms()
    a1, w1 = _mk(128 * (2 * n + 1) - 24, 200, 1), _mk(3 * 256 + 8, 200, 2)
    a2, w2 = _mk(1000, 72, 3), _mk(136, 72, 4)
    a3, w3t = _mk(128 * (n - 1), 264, 5), _mk(264, 776, 6)          # w3t is MN-major [K, N]
    aux3 = _mk(128 * (n - 1), 776, 7)
    bias1 = _mk(1, 3 * 256 + 8, 8)[0]
    dy, xin = _mk(4096, 520, 9), _mk(4096, 264, 10)
    u1 = torch.empty(a1.shape[0], w1.shape[0], device="cuda", dtype=torch.bfloat16)
    h1 = torch.empty_like(u1)
    c2 = torch.empty(a2.shape[0], w2.shape[0], device="cuda", dtype=torch.bfloat16)
    c3 = torch.empty(a3.shape[0], w3t.shape[1], device="cuda", dtype=torch.bfloat16)
    dw = torch.zeros(520, 264, device="cuda")

    def run():
        F.gemm(a1, w1, epi=lib.EPI_BIAS_GELU, bias=bias1, out=u1, out2=h1)
        F.gemm(a2, w2, epi=lib.EPI_BIAS, out=c2, block_n=128)
        F.gemm(a3, w3t, b_mn=True, epi=lib.EPI_GELU_BWD, aux=aux3, out=c3)
        dw.zero_()
        F.gemm(dy, xin, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=3)

    refs = {
        "u": a1.double() @ w1.double().t() + bias1.double(),
        "c2": a2.double() @ w2.double().t(),
        "dw": dy.double().t() @ xin.double(),
    }
    return run, {"u": u1, "h": h1, "c2": c2, "c3": c3, "dw": dw}, refs


def _rel(a, b):
    return ((a.double() - b).norm() / b.norm()).item()


def test_gemm_back_to_back_launches_in_one_stream():
    run, outs, refs = _back_to_back_calls()
    run()
    torch.cuda.synchronize()
    assert _rel(outs["u"], refs["u"]) < 1e-2
    assert _rel(outs["h"], torch.nn.functional.gelu(refs["u"])) < 1e-2
    assert _rel(outs["c2"], refs["c2"]) < 1e-2
    assert _rel(outs["dw"], refs["dw"]) < 1e-4
    first = {k: v.clone() for k, v in outs.items() if k != "dw"}
    run()
    torch.cuda.synchronize()
    for k, v in first.items():
        assert torch.equal(outs[k], v), k


def test_gemm_back_to_back_launches_in_one_cuda_graph():
    run, outs, refs = _back_to_back_calls()
    run()
    torch.cuda.synchronize()
    eager = {k: v.clone() for k, v in outs.items()}
    for v in outs.values():
        v.fill_(7.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            run()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    for k, v in eager.items():
        if k == "dw":                            # split-K fp32 reductions: the order of the atomic adds varies
            assert _rel(outs[k], refs["dw"]) < 1e-4
        else:
            assert torch.equal(outs[k], v), k


# bench shapes (VisualBERT base, B = 166, S = 228): M = 37848 tokens, H = 768, I = 3072
M_BENCH, H, I = 166 * 228, 768, 3072


@pytest.mark.parametrize("a_mn,b_mn,epi,N,K", [
    (0, 0, 0, 3 * H, H),        # QKV
    (0, 0, 2, H, H),            # O-proj + dropout + residual
    (0, 0, 1, I, H),            # FFN-up + GELU, two outputs
    (0, 0, 2, H, I),            # FFN-down + dropout + residual
    (0, 1, 3, I, H),            # FFN-down dgrad x GELU'(u)
    (0, 1, 4, H, I),            # FFN-up dgrad + residual gradient
    (0, 1, 0, H, H),            # O-proj dgrad
    (0, 1, 4, H, 3 * H),        # QKV dgrad + residual gradient
], ids=["qkv", "oproj", "ffn_up", "ffn_down", "ffn_down_dgrad", "ffn_up_dgrad", "oproj_dgrad", "qkv_dgrad"])
def test_gemm_bench_shapes(a_mn, b_mn, epi, N, K):
    run_and_check(a_mn, b_mn, epi, M_BENCH, N, K, 256, seed=N + K + epi)     # block_n 256: the auto choice


@pytest.mark.parametrize("n_out,k_in", [(3 * H, H), (H, H), (I, H), (H, I)], ids=["qkv", "oproj", "ffn_up", "ffn_down"])
def test_gemm_bench_shapes_wgrad(n_out, k_in):
    from mmf_b200.engine import best_splits
    run_and_check(1, 1, 5, n_out, k_in, M_BENCH, 256, seed=n_out + k_in, splits=best_splits(n_out, k_in, M_BENCH))
