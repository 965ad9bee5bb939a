"""The GEMM epilogues that read a per-element operand (aux: residual, pre-activation or residual gradient) load it by
TMA into the output staging boxes.  Every element against fp64 (tests/kernel_check.py, with the bounds of
test_gemm_edges_gpu.run_and_check): M and N tails inside a box and wholly clipped boxes, aux as a strided view, several
work units per CTA, aux present and absent in consecutive launches (stream and CUDA graph), the output written over
aux in place, and the refusal of an aux that TMA cannot address."""
import pytest
import torch

import kernel_check as kc
from test_gemm_edges_gpu import run_and_check

pytestmark = pytest.mark.gpu

AUX_EPIS = [2, 3, 4]                  # bias + dropout + residual, GELU' x dgrad, + residual gradient


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf16(*shape, g, scale=0.5):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Case:
    """operands of one aux-epilogue GEMM (A K-major; B K-major for the forward epilogue, MN-major for the dgrads), its
    fp64 reference for a given aux, and the launch"""

    def __init__(self, epi, M, N, K, seed):
        from mmf_b200 import functional as F
        g = _gen(seed)
        self.epi, self.M, self.N = epi, M, N
        self.a = _bf16(M, K, g=g)
        w = _bf16(N, K, g=g)
        self.b_mn = epi != 2
        self.b = w.t().contiguous() if self.b_mn else w
        self.acc, self.absab = kc.gemm_ref(self.a, w)
        self.bias, self.words, self.keep, self.dsc = None, None, None, 1.0
        if epi == 2:
            self.bias = _bf16(N, g=g)
            wpr = (N + 31) // 32 + 3
            self.words = torch.randint(-2 ** 31, 2 ** 31, (M, wpr), generator=g, device="cuda",
                                       dtype=torch.int64).to(torch.int32)
            self.keep = F.unpack_keep_bits(self.words, N).double()
            self.dsc = 1.0 / 0.9

    def run(self, aux, out=None, with_mask=True):
        from mmf_b200 import functional as F
        return F.gemm(self.a, self.b, b_mn=self.b_mn, epi=self.epi, bias=self.bias, aux=aux,
                      drop_mask=self.words if with_mask else None, drop_scale=self.dsc, out=out)

    def check(self, out, aux64, tag, with_mask=True):
        """aux64: fp64 values of the aux the launch read, or None"""
        lay, acc, absab = kc.gemm_layout(256), self.acc, self.absab
        if self.epi == 2:
            bias64 = self.bias.double()
            scale = self.keep * self.dsc if with_mask else 1.0
            pre = (acc + bias64) * scale
            ref = pre + (aux64 if aux64 is not None else 0.0)
            extra = (absab + bias64.abs()) * scale
            bound = kc.U_BF16 * ref.abs() + kc.U_ACC * (extra + (aux64.abs() if aux64 is not None else 0.0) + ref.abs())
        elif self.epi == 3:
            gp = kc.gelu_grad64(aux64) if aux64 is not None else torch.ones_like(acc)
            ref = acc * gp
            gerr = 2.0 ** -21 * (1 + aux64.abs()) if aux64 is not None else 0.0
            bound = kc.U_BF16 * ref.abs() + kc.U_ACC * (absab * gp.abs() + ref.abs()) + acc.abs() * gerr
        else:
            ref = acc + (aux64 if aux64 is not None else 0.0)
            bound = kc.gemm_bound(ref, absab, aux64.abs() if aux64 is not None else 0.0)
        return kc.assert_within(out, ref, bound, lay, tag)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", AUX_EPIS)
def test_aux_tails_and_clipped_boxes(epi, bn):
    """M tails of 1 and 40 rows past a tile (the second warpgroup's rows wholly clipped at M = 65), N tails inside a box
    (40) and one box into the last tile with its other boxes clipped (264, 776); M = 128 * 140 + 40 gives more than three
    work units per CTA on 132 SMs, so unit u + 1's aux prefetch waits for unit u's stores"""
    a_mn, b_mn = (0, 0) if epi == 2 else (0, 1)
    for i, (M, N, K) in enumerate([(65, 40, 72), (129, 264, 136), (65, 776, 64), (128 * 140 + 40, 776, 136)]):
        run_and_check(a_mn, b_mn, epi, M, N, K, bn, seed=300 + 10 * i + epi)


@pytest.mark.parametrize("epi", AUX_EPIS)
def test_aux_strided_views(epi):
    """aux with ldaux > N at a 16-byte column offset into a wider buffer, and at offset 0 with ldaux > N"""
    M, N, K = 200, 264, 136
    c = Case(epi, M, N, K, seed=20 + epi)
    g = _gen(40 + epi)
    buf = _bf16(M, N + 40, g=g, scale=1.0)
    for off in (8, 0):
        aux = buf[:, off:off + N]
        assert aux.stride(0) == N + 40
        out = c.run(aux)
        c.check(out, aux.double(), "epi=%d aux column offset %d, ldaux %d" % (epi, off, N + 40))


@pytest.mark.parametrize("epi", AUX_EPIS)
def test_aux_written_over_in_place(epi):
    """out is aux itself: each aux box is loaded before the results of that box overwrite it"""
    n = _sms()
    M, N, K = 128 * (n + 7) - 24, 776, 200
    c = Case(epi, M, N, K, seed=60 + epi)
    aux = _bf16(M, N, g=_gen(70 + epi), scale=1.0)
    aux64 = aux.double()
    res = c.run(aux, out=aux)
    assert res.data_ptr() == aux.data_ptr()
    c.check(aux, aux64, "epi=%d in place" % epi)


def _mixed_launches():
    """the same three GEMMs, each with aux and then without it (and the forward without its keep bits too), launched
    back to back without a synchronisation"""
    n = _sms()
    M = 128 * (2 * n + 1) - 40
    cases = [Case(epi, M, 776 if epi != 2 else 264, 136, seed=80 + epi) for epi in AUX_EPIS]
    auxes = [_bf16(M, c.N, g=_gen(90 + c.epi), scale=1.0) for c in cases]
    outs = [[torch.empty(M, c.N, device="cuda", dtype=torch.bfloat16) for _ in range(2)] for c in cases]

    def run():
        for c, aux, (o_aux, o_none) in zip(cases, auxes, outs):
            c.run(aux, out=o_aux)
            c.run(None, out=o_none, with_mask=False)

    def check(tag):
        for c, aux, (o_aux, o_none) in zip(cases, auxes, outs):
            c.check(o_aux, aux.double(), "%s epi=%d with aux" % (tag, c.epi))
            c.check(o_none, None, "%s epi=%d without aux" % (tag, c.epi), with_mask=False)

    return run, check, [o for pair in outs for o in pair]


def test_aux_and_no_aux_back_to_back_in_one_stream():
    run, check, outs = _mixed_launches()
    run()
    torch.cuda.synchronize()
    check("stream")


def test_aux_and_no_aux_back_to_back_in_one_cuda_graph():
    run, check, outs = _mixed_launches()
    run()
    torch.cuda.synchronize()
    eager = [o.clone() for o in outs]
    for o in outs:
        o.fill_(7.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            run()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    check("graph")
    for o, e in zip(outs, eager):
        assert torch.equal(o, e)


@pytest.mark.parametrize("epi", AUX_EPIS)
def test_aux_that_tma_cannot_address_is_refused(epi):
    M, N, K = 64, 264, 64
    c = Case(epi, M, N, K, seed=5)
    buf = torch.zeros(M, N + 40, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="aux"):
        c.run(buf[:, 4:4 + N])                              # 8-byte but not 16-byte aligned
    buf2 = torch.zeros(M, N + 4, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="aux"):
        c.run(buf2[:, :N])                                  # ldaux = N + 4, not a multiple of 8
