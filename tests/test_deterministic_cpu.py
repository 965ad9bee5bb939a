"""Deterministic mode on the host: the ordered-reduction entry points of include/mmfb200.h, their workspace-size queries, and
mmf_b200.functional choosing the ordered path exactly while torch.use_deterministic_algorithms(True) is in effect.  The
library calls are recorded by a stand-in for functional.LIB; no kernel runs."""
import ctypes

import pytest
import torch

from mmf_b200 import functional as F, lib


@pytest.fixture
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()

    def set_mode(on, warn_only=False):
        torch.use_deterministic_algorithms(on, warn_only=warn_only)
    yield set_mode
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


class Recorder:
    """stands in for functional.LIB: records each entry point's name and arguments and returns MMFB_OK; the host-only size
    queries go to the real library"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        real = getattr(lib.LIB, name)
        if name.endswith("_workspace_bytes"):
            return real

        def call(*args):
            if args and isinstance(args[0], ctypes._Pointer) or (args and type(args[0]).__name__ == "CArgObject"):
                args = (ctypes.cast(args[0], ctypes.POINTER(type(args[0]._obj))).contents,) + args[1:]
            self.calls.append((name, args))
            return lib.MMFB_OK
        return call

    def names(self):
        return [n for n, _ in self.calls]


class _OnDevice(torch.Tensor):
    """a CPU tensor that passes functional's `is_cuda` checks (loss_sum)"""

    @property
    def is_cuda(self):
        return True


@pytest.fixture
def rec(monkeypatch):
    r = Recorder()
    monkeypatch.setattr(F, "LIB", r)
    monkeypatch.setattr(F, "_req", lambda t, dtype, name: None)
    monkeypatch.setattr(F, "_stream_ptr", lambda stream=None: None)
    return r


def test_ordered_symbols_exported_and_need_a_device():
    syms = lib.header_symbols()
    for s in ("mmfb_colsum_ordered", "mmfb_embed_scatter_sorted_ordered", "mmfb_gemm_workspace_bytes",
              "mmfb_layernorm_bwd_workspace_bytes", "mmfb_colsum_workspace_bytes",
              "mmfb_embed_scatter_sorted_workspace_bytes"):
        assert s in syms and hasattr(lib.LIB, s), s
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.LIB.mmfb_colsum_ordered(1, 8, 1, 4, 8, 1, 1024, None) == lib.MMFB_ERR_DEVICE
    assert "no CPU fallback" in lib.last_error()
    assert lib.LIB.mmfb_embed_scatter_sorted_ordered(1, 8, 1, 1, 1, 4, 8, 1, 1024, None) == lib.MMFB_ERR_DEVICE
    assert lib.LIB.mmfb_colsum_ordered(None, 8, 1, 4, 8, 1, 1024, None) == lib.MMFB_ERR_ARG
    # the appended fields sit at the end of both structs: a zero-initialised struct is the atomic path
    assert lib.GemmArgs._fields_[-2][0] == "workspace" and lib.LnArgs._fields_[-2][0] == "workspace"
    a = lib.GemmArgs()
    assert a.workspace is None and a.workspace_bytes == 0


def _splits(K, s):
    kb = (K + 63) // 64
    s = min(s, kb)
    while s > 1 and ((kb + s - 1) // s) * (s - 1) >= kb:
        s -= 1
    return s


@pytest.mark.parametrize("M,N,K,splits", [(768, 3072, 37848, 5), (768, 768, 37848, 7), (2304, 768, 37848, 2),
                                          (264, 136, 200, 7), (64, 64, 64, 3), (64, 64, 130, 3), (64, 64, 200, 5)])
def test_gemm_workspace_bytes(M, N, K, splits):
    s = _splits(K, splits)
    assert lib.LIB.mmfb_gemm_workspace_bytes(M, N, K, splits) == (s * M * N * 4 if s > 1 else 0)


def test_gemm_workspace_bytes_by_hand():
    assert lib.LIB.mmfb_gemm_workspace_bytes(768, 3072, 37848, 5) == 5 * 768 * 3072 * 4
    assert lib.LIB.mmfb_gemm_workspace_bytes(64, 64, 130, 3) == 3 * 64 * 64 * 4       # 3 k-blocks, one per split
    assert lib.LIB.mmfb_gemm_workspace_bytes(64, 64, 200, 5) == 4 * 64 * 64 * 4       # 4 k-blocks: at most 4 splits
    assert lib.LIB.mmfb_gemm_workspace_bytes(64, 64, 64, 3) == 0                      # one k-block: no split
    assert lib.LIB.mmfb_gemm_workspace_bytes(0, 64, 640, 3) == 0


def test_row_workspace_bytes_by_hand():
    assert lib.LIB.mmfb_layernorm_bwd_workspace_bytes(37848, 768) == 296 * 3 * 768 * 4
    assert lib.LIB.mmfb_layernorm_bwd_workspace_bytes(128, 2048) == 1 * 3 * 2048 * 4
    assert lib.LIB.mmfb_layernorm_bwd_workspace_bytes(129, 1024) == 2 * 3 * 1024 * 4
    assert lib.LIB.mmfb_colsum_workspace_bytes(37848, 3072) == 296 * 3072 * 4
    assert lib.LIB.mmfb_colsum_workspace_bytes(1, 8) == 8 * 4
    assert lib.LIB.mmfb_embed_scatter_sorted_workspace_bytes(37848, 768) == 1183 * 2 * 768 * 4
    assert lib.LIB.mmfb_embed_scatter_sorted_workspace_bytes(33, 64) == 2 * 2 * 64 * 4
    for fn in (lib.LIB.mmfb_layernorm_bwd_workspace_bytes, lib.LIB.mmfb_colsum_workspace_bytes,
               lib.LIB.mmfb_embed_scatter_sorted_workspace_bytes):
        assert fn(0, 768) == 0 and fn(16, 0) == 0


@pytest.mark.parametrize("on", [False, True])
def test_functional_picks_the_ordered_path_with_the_flag(rec, deterministic, on):
    deterministic(on)
    bf = torch.bfloat16
    dy = torch.zeros(300, 64, dtype=bf)
    x = torch.zeros(300, 96, dtype=bf)
    dw = torch.zeros(64, 96)

    F.gemm(dy, x, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=3)
    g = rec.calls[-1][1][0]
    assert rec.names()[-1] == "mmfb_gemm" and g.splits == 3
    want = lib.LIB.mmfb_gemm_workspace_bytes(64, 96, 300, 3)
    assert want == 3 * 64 * 96 * 4
    assert (g.workspace_bytes, bool(g.workspace)) == ((want, True) if on else (0, False))

    F.gemm(dy, x, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=dw, splits=1)   # one split: nothing to order
    assert rec.calls[-1][1][0].workspace_bytes == 0 and not rec.calls[-1][1][0].workspace
    F.gemm(x[:, :64].contiguous(), dy, epi=lib.EPI_BIAS)                               # no reduction at all
    assert rec.calls[-1][1][0].workspace_bytes == 0

    F.colsum(dy, torch.zeros(64))
    assert rec.names()[-1] == ("mmfb_colsum_ordered" if on else "mmfb_colsum")
    if on:
        assert rec.calls[-1][1][6] == lib.LIB.mmfb_colsum_workspace_bytes(300, 64) == 3 * 64 * 4

    y, mean, rstd, gam = torch.zeros(300, 64, dtype=bf), torch.zeros(300), torch.ones(300), torch.ones(64, dtype=bf)
    F.layernorm_bwd(dy, y, mean, rstd, gam, torch.zeros(64), torch.zeros(64))
    a = rec.calls[-1][1][0]
    assert rec.names()[-1] == "mmfb_layernorm_bwd"
    assert (a.workspace_bytes, bool(a.workspace)) == ((3 * 3 * 64 * 4, True) if on else (0, False))
    F.layernorm_bwd(dy, y, mean, rstd, gam, None, None)                                # no parameter gradients
    assert rec.calls[-1][1][0].workspace_bytes == 0

    idx = torch.zeros(300, dtype=torch.int32)
    F.embed_scatter_sorted(dy, torch.zeros(4, 64), *F.sort_indices(idx))
    assert rec.names()[-1] == ("mmfb_embed_scatter_sorted_ordered" if on else "mmfb_embed_scatter_sorted")
    if on:
        assert rec.calls[-1][1][8] == 10 * 2 * 64 * 4

    logits = torch.zeros(300, 64, dtype=bf)
    labels = torch.zeros(300, dtype=torch.int64)
    loss_sum = torch.zeros(1).as_subclass(_OnDevice)
    F.ce_rows(logits, labels, -1, 1.0, loss_sum)
    args = rec.calls[-1][1]
    assert rec.names()[-1] == "mmfb_ce_rows"
    if on:
        assert args[7] is None and args[8] is not None          # no atomic loss sum; the per-row losses are summed here
    else:
        assert args[7] == loss_sum.data_ptr() and args[8] is None


def test_ce_rows_ordered_sums_the_row_losses(rec, deterministic):
    deterministic(True)
    logits, labels = torch.zeros(5, 8, dtype=torch.bfloat16), torch.zeros(5, dtype=torch.int64)
    row_loss = torch.tensor([1.0, 2.0, 0.5, 0.25, 4.0])
    loss_sum = torch.full((1,), 10.0).as_subclass(_OnDevice)
    F.ce_rows(logits, labels, -1, 1.0, loss_sum, row_loss=row_loss)
    assert rec.calls[-1][1][8] == row_loss.data_ptr()
    assert loss_sum.item() == 17.75


def test_atomic_only_table_scatter_raises_or_warns(rec, deterministic):
    dy = torch.zeros(16, 64, dtype=torch.bfloat16)
    tab = (torch.zeros(4, 64), torch.zeros(16, dtype=torch.int32))
    deterministic(False)
    F.embed_scatter(dy, dtabs=[tab])
    assert rec.names()[-1] == "mmfb_embed_scatter"
    deterministic(True)
    n = len(rec.calls)
    with pytest.raises(RuntimeError, match="embed_scatter"):
        F.embed_scatter(dy, dtabs=[tab])
    assert len(rec.calls) == n
    F.embed_scatter(dy, dsrcs=[(torch.zeros(16, 64, dtype=torch.bfloat16), torch.arange(16, dtype=torch.int32))])
    assert rec.names()[-1] == "mmfb_embed_scatter"                   # plain row stores: nothing to order
    deterministic(True, warn_only=True)
    with pytest.warns(UserWarning, match="embed_scatter"):
        F.embed_scatter(dy, dtabs=[tab])
    assert rec.names()[-1] == "mmfb_embed_scatter"
