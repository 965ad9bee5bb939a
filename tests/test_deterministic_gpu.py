"""Deterministic mode on the H100: the ordered reductions give the same bits on every call and agree with fp64, the ordered
split-K GEMM equals its defined order restated in torch bit for bit, and whole training steps of the registered models
(forward, backward, B200AdamW) are bitwise reproducible under torch.use_deterministic_algorithms(True) and match the
default-mode step within the parity tolerances."""
import contextlib
import os
import sys

# model steps run torch matmuls (heads, poolers) next to the kernels: cuBLAS needs this before any CUDA context exists
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import pytest  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import kernel_check as KC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@contextlib.contextmanager
def flag(on):
    """torch.use_deterministic_algorithms(on) inside the block; the previous mode (and warn_only) is restored after it"""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.fixture
def deterministic():
    with flag(True):
        yield


def _bits(t):
    return t.detach().contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).clone()


def _three_calls_identical(run):
    outs = [run() for _ in range(3)]
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(_bits(a), _bits(b))
    return outs[0]


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [2, 3, 5, 7])
@pytest.mark.parametrize("M,N,K", [(264, 136, 845), (776, 392, 2196)])    # 14 and 35 k-blocks, the last one partial
def test_ordered_split_k(deterministic, S, M, N, K):
    from mmf_b200 import functional as F, lib
    g = torch.Generator().manual_seed(S * 1000 + M)
    a = torch.randn(K, M, generator=g).to(torch.bfloat16).to(DEV)       # MN-major A: dY [tokens, out]
    b = torch.randn(K, N, generator=g).to(torch.bfloat16).to(DEV)       # MN-major B: X [tokens, in]
    c0 = torch.randn(M, N, generator=g).to(DEV)
    kb = (K + 63) // 64
    assert ((kb + S - 1) // S) * (S - 1) < kb           # every split owns a k-block: the GEMM runs S splits as given
    assert lib.LIB.mmfb_gemm_workspace_bytes(M, N, K, S) == S * M * N * 4

    def run():
        c = c0.clone()
        F.gemm(a, b, a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=c, splits=S)
        return (c,)
    c, = _three_calls_identical(run)
    ref, absab = KC.gemm_ref(a.t().cpu(), b.t().cpu())
    ref = ref + c0.cpu().double()
    KC.assert_within(c.cpu(), ref, KC.gemm_bound(ref, absab + c0.cpu().double().abs(), bf16_out=False),
                     KC.gemm_layout(0, S))
    # the defined order: each split's product over its k-blocks into zeroed fp32, then C + P_0 + P_1 + ... in fp32
    per = (kb + S - 1) // S
    order = c0.clone()
    for s in range(S):
        k0, k1 = s * per * 64, min(K, (s + 1) * per * 64)
        part = torch.zeros(M, N, device=DEV)
        F.gemm(a[k0:k1], b[k0:k1], a_mn=True, b_mn=True, epi=lib.EPI_ATOMIC_F32, out=part, splits=1)
        order = order + part
    assert torch.equal(_bits(order), _bits(c))


def test_ordered_split_k_refuses_a_short_workspace():
    import ctypes
    from mmf_b200 import lib
    a = torch.zeros(640, 128, dtype=torch.bfloat16, device=DEV)
    c = torch.zeros(128, 128, device=DEV)
    ws = torch.zeros(10, device=DEV)
    args = lib.GemmArgs()
    args.A, args.lda, args.a_mn, args.B, args.ldb, args.b_mn = a.data_ptr(), 128, 1, a.data_ptr(), 128, 1
    args.C, args.ldc, args.M, args.N, args.K = c.data_ptr(), 128, 128, 128, 640
    args.epi, args.splits = lib.EPI_ATOMIC_F32, 3
    args.workspace, args.workspace_bytes = ws.data_ptr(), 40
    n0 = lib.launch_count()
    assert lib.LIB.mmfb_gemm(ctypes.byref(args), None) == lib.MMFB_ERR_ARG
    args.workspace, args.workspace_bytes = None, 3 * 128 * 128 * 4
    assert lib.LIB.mmfb_gemm(ctypes.byref(args), None) == lib.MMFB_ERR_ARG
    assert lib.launch_count() == n0


def test_ordered_row_reductions_refuse_a_bad_workspace():
    """a NULL, short or misaligned workspace is MMFB_ERR_ARG before anything is launched"""
    import ctypes
    from mmf_b200 import lib
    M, H = 300, 256
    x = torch.zeros(M, H, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(3, H, device=DEV)
    ws = torch.zeros(1 << 20, device=DEV)
    idx = torch.zeros(M, dtype=torch.int32, device=DEV)
    stats = torch.ones(M, device=DEV)
    gam = torch.ones(H, dtype=torch.bfloat16, device=DEV)
    sizes = {"colsum": lib.LIB.mmfb_colsum_workspace_bytes(M, H),
             "scatter": lib.LIB.mmfb_embed_scatter_sorted_workspace_bytes(M, H),
             "layernorm": lib.LIB.mmfb_layernorm_bwd_workspace_bytes(M, H)}

    def colsum(p, n):
        return lib.LIB.mmfb_colsum_ordered(x.data_ptr(), H, out.data_ptr(), M, H, p, n, None)

    def scatter(p, n):
        return lib.LIB.mmfb_embed_scatter_sorted_ordered(x.data_ptr(), H, idx.data_ptr(), idx.data_ptr(), out.data_ptr(),
                                                         M, H, p, n, None)

    def layernorm(p, n):
        a = lib.LnArgs()
        a.dx, a.lddx, a.y, a.ldy, a.mean, a.rstd, a.gamma = x.data_ptr(), H, x.data_ptr(), H, stats.data_ptr(), \
            stats.data_ptr(), gam.data_ptr()
        a.dy, a.lddy, a.dz, a.lddz = x.data_ptr(), H, x.data_ptr(), H
        a.dgamma, a.dbeta, a.M, a.H = out.data_ptr(), out.data_ptr() + 4 * H, M, H
        a.workspace, a.workspace_bytes = p, n
        return lib.LIB.mmfb_layernorm_bwd(ctypes.byref(a), None)

    for name, fn in (("colsum", colsum), ("scatter", scatter), ("layernorm", layernorm)):
        need = sizes[name]
        assert need > 0
        n0 = lib.launch_count()
        for p, n in ((None, need), (ws.data_ptr(), need - 4), (ws.data_ptr() + 4, need), (None, 0 if name != "layernorm" else 4)):
            assert fn(p, n) == lib.MMFB_ERR_ARG, (name, p, n)
            assert "workspace" in lib.last_error()
        assert lib.launch_count() == n0, name
        torch.cuda.synchronize()


@pytest.mark.parametrize("M,N", [(37848, 768), (37848, 3072), (1000, 2304), (5, 8)])
def test_ordered_colsum(deterministic, M, N):
    from mmf_b200 import functional as F
    g = torch.Generator().manual_seed(M + N)
    xi = KC.exact_ints(M, N, gen=g).to(DEV)               # small integers: every partial sum is exact
    out = F.colsum(xi, torch.zeros(N, device=DEV))
    assert torch.equal(out.cpu().double(), xi.cpu().double().sum(0))
    x = torch.randn(M, N, generator=g).to(torch.bfloat16).to(DEV)
    out0 = torch.randn(N, generator=g).to(DEV)
    got, = _three_calls_identical(lambda: (F.colsum(x, out0.clone()),))
    ref = x.cpu().double().sum(0) + out0.cpu().double()
    bound = KC.U_F32 * (M / 128 + 128 + 1) * (x.cpu().double().abs().sum(0) + out0.cpu().double().abs())
    KC.assert_within(got.cpu(), ref, bound, KC.flat_layout())


@pytest.mark.parametrize("H", [768, 1024, 2048])
@pytest.mark.parametrize("dropout,dx2", [(False, False), (True, True)])
def test_ordered_layernorm_bwd(deterministic, H, dropout, dx2):
    from mmf_b200 import functional as F
    M = 3000
    g = torch.Generator().manual_seed(H + 7 * dropout)
    y = torch.randn(M, H, generator=g).to(torch.bfloat16).to(DEV)
    gam = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).to(DEV)
    bet = torch.zeros(H, dtype=torch.bfloat16, device=DEV)
    dx = torch.randn(M, H, generator=g).to(torch.bfloat16).to(DEV)
    d2 = torch.randn(M, H, generator=g).to(torch.bfloat16).to(DEV) if dx2 else None
    keep = F.pack_keep_bits((torch.rand(M, H, generator=g) > 0.1).to(DEV)) if dropout else None
    _, mean, rstd = F.layernorm_fwd(y, gam, bet)

    def run():
        dg, db, dbias = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
        dy, dz = F.layernorm_bwd(dx, y, mean, rstd, gam, dg, db, dbias=dbias, dx2=d2, drop_mask=keep, drop_scale=1 / 0.9)
        return dy, dz, dg, db, dbias
    dy, dz, dg, db, dbias = _three_calls_identical(run)
    with flag(False):
        dy0, dz0, _, _, _ = run()
    assert torch.equal(_bits(dy), _bits(dy0)) and torch.equal(_bits(dz), _bits(dz0))     # row outputs: unchanged bits
    d = dx.cpu().double() + (d2.cpu().double() if dx2 else 0.0)
    xh = (y.cpu().double() - mean.cpu().double()[:, None]) * rstd.cpu().double()[:, None]
    scale = KC.U_F32 * (M / 128 + 128 + 8)
    KC.assert_within(dg.cpu(), (d * xh).sum(0), scale * (d * xh).abs().sum(0) + 1e-30, KC.flat_layout(), "dgamma")
    KC.assert_within(db.cpu(), d.sum(0), scale * d.abs().sum(0) + 1e-30, KC.flat_layout(), "dbeta")
    # dbias sums dz before its bf16 rounding where the kernel has the fp32 value: one bf16 rounding per term on top
    z = dz.cpu().double()
    KC.assert_within(dbias.cpu(), z.sum(0), (scale + KC.U_BF16) * z.abs().sum(0) + 1e-30, KC.flat_layout(), "dbias")


def _index_vectors(M):
    g = torch.Generator().manual_seed(M)
    S = 148
    return {"type": torch.zeros(M, dtype=torch.int32),
            "position": (torch.arange(M) % S).to(torch.int32),
            "word": torch.randint(0, 30522, (M,), generator=g).to(torch.int32),
            "word_padded": torch.where(torch.rand(M, generator=g) < 0.2, -1,
                                       torch.randint(0, 50, (M,), generator=g)).to(torch.int32)}


@pytest.mark.parametrize("kind", ["type", "position", "word", "word_padded"])
@pytest.mark.parametrize("M,H", [(37848, 768), (1001, 1024)])
def test_ordered_scatter_sorted(deterministic, kind, M, H):
    from mmf_b200 import functional as F
    idx = _index_vectors(M)[kind]
    V = 30522 if kind == "word" else max(int(idx.max()) + 1, 1)
    g = torch.Generator().manual_seed(M + H)
    srt, order = F.sort_indices(idx.to(DEV))
    dyi = KC.exact_ints(M, H, gen=g).to(DEV)
    tab = torch.zeros(V, H, device=DEV)
    F.embed_scatter_sorted(dyi, tab, srt, order)
    ok = idx >= 0
    ref = torch.zeros(V, H, dtype=torch.float64).index_add_(0, idx[ok].long(), dyi.cpu().double()[ok])
    assert torch.equal(tab.cpu().double(), ref)
    dy = torch.randn(M, H, generator=g).to(torch.bfloat16).to(DEV)
    tab0 = torch.randn(V, H, generator=g).to(DEV)

    def run():
        t = tab0.clone()
        F.embed_scatter_sorted(dy, t, srt, order)
        return (t,)
    got, = _three_calls_identical(run)
    ref = tab0.cpu().double().index_add_(0, idx[ok].long(), dy.cpu().double()[ok])
    absref = tab0.cpu().double().abs().index_add_(0, idx[ok].long(), dy.cpu().double().abs()[ok])
    KC.assert_within(got.cpu(), ref, KC.U_F32 * (M / 32 + 34) * absref + 1e-30, KC.flat_layout())


def test_ordered_ce_loss(deterministic):
    from mmf_b200 import functional as F
    M, V = 4000, 30528
    g = torch.Generator().manual_seed(5)
    z = (3 * torch.randn(M, V, generator=g)).to(torch.bfloat16).to(DEV)
    labels = torch.randint(0, V, (M,), generator=g)
    labels[torch.rand(M, generator=g) < 0.3] = -1
    labels = labels.to(DEV)

    def run():
        zz, loss = z.clone(), torch.zeros(1, device=DEV)
        F.ce_rows(zz, labels, -1, 1.0, loss)
        return loss, zz
    loss, dz = _three_calls_identical(run)
    with flag(False):
        loss0, dz0 = run()
    assert torch.equal(_bits(dz), _bits(dz0))
    zl = z.cpu().double()
    act = labels.cpu() >= 0
    li = torch.logsumexp(zl, 1) - zl.gather(1, labels.cpu().clamp_min(0)[:, None].long())[:, 0]
    ref = li[act].sum().item()
    assert abs(loss.item() - ref) <= 1e-5 * li[act].abs().sum().item() + 1e-3
    assert abs(loss.item() - loss0.item()) <= 1e-5 * li[act].abs().sum().item()


# ------------------------------------------------------------------------------------------------------------------
# whole training steps
# ------------------------------------------------------------------------------------------------------------------
def _step(model, batch_fn, loss_fn, state):
    """one forward + backward + B200AdamW step from `state` (parameters), with the dropout seeds reset"""
    from mmf_b200 import modules
    from mmf_b200.optim import B200AdamW
    with torch.no_grad():
        for k, p in model.named_parameters():
            p.copy_(state[k])
    model.zero_grad(set_to_none=True)
    torch.manual_seed(0)
    modules._SEED_COUNTER[0] = 0
    opt = B200AdamW(model.parameters(), lr=1e-4, weight_decay=0.01)
    losses = loss_fn(model, batch_fn())
    sum(v.float().sum() for v in losses.values()).backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
    opt.step()
    params = {k: p.detach().clone() for k, p in model.named_parameters()}
    torch.cuda.synchronize()
    return {k: v.detach().float().clone() for k, v in losses.items()}, grads, params


def _check_model(model, batch_fn, loss_fn=None):
    loss_fn = loss_fn or (lambda m, b: m(b)["losses"])
    state = {k: p.detach().clone() for k, p in model.named_parameters()}
    with flag(True):
        a = _step(model, batch_fn, loss_fn, state)
        b = _step(model, batch_fn, loss_fn, state)
    with flag(False):
        c = _step(model, batch_fn, loss_fn, state)
    for da, db in zip(a, b):
        assert da.keys() == db.keys()
        for k in da:
            assert torch.equal(_bits(da[k]), _bits(db[k])), k
    la, lc = a[0], c[0]
    for k in la:
        assert abs(la[k].sum().item() - lc[k].sum().item()) <= 1e-2 * max(1.0, abs(lc[k].sum().item())), k
    worst = 0.0
    for k, ga in a[1].items():
        gc = c[1][k].double()
        if gc.norm() > 1e-6:
            worst = max(worst, ((ga.double() - gc).norm() / gc.norm()).item())
    print("worst gradient difference to the default-mode step", worst)
    assert worst < 3e-2


def _visual_bert(B=192, skip=False):
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.visual_bert import B200VisualBERT
    import bench
    wl = bench.VisualBertWL()
    torch.manual_seed(0)
    model = B200VisualBERT(wl.config(0.1)).to(DEV).train()
    set_skip_padding(model, skip)
    batch = bench.to_device(wl.host_batch(B, 17), DEV)
    aux = wl.aux(B, DEV)
    return model, (lambda: batch), (lambda m, bt: {"loss": wl.loss(m, bt, aux)})


@pytest.mark.parametrize("skip", [False, True])
def test_visual_bert_steps_are_bitwise_reproducible(skip):
    sys.path.insert(0, os.path.dirname(HERE))
    model, batch_fn, loss_fn = _visual_bert(skip=skip)
    _check_model(model, batch_fn, loss_fn)


def test_vilbert_packed_steps_are_bitwise_reproducible():
    from bench_vilbert import vilbert_config, T_TOK, R_REG, FEAT, VOCAB
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.vilbert import B200ViLBERTBase
    torch.manual_seed(0)
    model = B200ViLBERTBase(vilbert_config(0.1)).to(DEV).train()
    set_skip_padding(model, True, two_stream=True)
    B = 256
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, VOCAB, (B, T_TOK), generator=g).to(DEV)
    lens = torch.randint(T_TOK // 2, T_TOK + 1, (B,), generator=g)
    tmask = (torch.arange(T_TOK)[None, :] < lens[:, None]).long().to(DEV)
    feats = torch.randn(B, R_REG, FEAT, generator=g).abs().to(DEV)
    loc = torch.rand(B, R_REG, 5, generator=g).to(DEV)
    nreg = torch.randint(R_REG // 2, R_REG + 1, (B,), generator=g)
    imask = (torch.arange(R_REG)[None, :] < nreg[:, None]).long().to(DEV)
    wt, wv = torch.randn(B, T_TOK, 768, generator=g).to(DEV), torch.randn(B, R_REG, 1024, generator=g).to(DEV)

    def loss_fn(m, _):
        t, v, _ = m(ids, feats, loc, attention_mask=tmask, image_attention_mask=imask)
        return {"loss": (t * wt).sum() + (v * wv).sum()}
    _check_model(model, lambda: None, loss_fn)


def test_lxmert_steps_are_bitwise_reproducible():
    from bench_lxmert import sample_list
    from mmf_b200 import models as MD
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("lxmert")).to(DEV).train()
    sl = sample_list(128, DEV, torch.Generator().manual_seed(3))
    _check_model(model, lambda: sl)


@pytest.mark.parametrize("task", ["mlm", "wra"])
def test_uniter_steps_are_bitwise_reproducible(task):
    import mmf_b200.mmft  # noqa: F401
    from bench_uniter import sample_list
    from mmf_b200 import models as MD
    torch.manual_seed(0)
    cfg = MD.load_model_config("uniter", overrides=dict(do_pretraining=True, tasks=task, mask_probability=0.15,
                                                        heads={task: {"type": task}}))
    model = MD.build_model(cfg).to(DEV).train()
    base = sample_list(128, DEV, torch.Generator().manual_seed(4))
    _check_model(model, lambda: type(base)(base))


def test_vinvl_pretraining_steps_are_bitwise_reproducible():
    from bench_vinvl import sample_list, PRE_TOK
    from mmf_b200 import models as MD
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("vinvl", overrides=dict(do_pretraining=True))).to(DEV).train()
    base = sample_list(128, PRE_TOK, DEV, torch.Generator().manual_seed(5))
    _check_model(model, lambda: type(base)(base))


def test_m4c_steps_are_bitwise_reproducible():
    from bench_m4c import sample_list, ANS, OCR_MAX
    from mmf_b200 import models as MD
    from mmf_b200.registry import registry
    registry.register("config", MD.ConfigNode({"datasets": "textvqa"}))
    registry.register("textvqa_num_final_outputs", ANS + OCR_MAX)
    registry.register("textvqa_answer_processor", MD.ConfigNode({"BOS_IDX": 1}))
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).to(DEV).train()
    sl = sample_list(128, DEV, torch.Generator().manual_seed(182))
    _check_model(model, lambda: sl, lambda m, b: {k: v.sum() for k, v in m(b)["losses"].items()})


def test_mmf_transformer_mlm_steps_are_bitwise_reproducible():
    import mmf_b200.mmft  # noqa: F401
    from mmf_b200 import engine, models as MD
    from mmf_b200.sample import SampleList
    B, T, R, FEAT, V = 96, 128, 100, 2048, 30522
    torch.manual_seed(0)
    cfg = MD.load_model_config("mmf_transformer", overrides={
        "modalities": [dict(type="text", key="text", embedding_dim=768, position_dim=512, segment_id=0),
                       dict(type="image", key="image", embedding_dim=FEAT, position_dim=R, segment_id=1,
                            encoder=dict(type="identity"))],
        "heads": [{"type": "mlm", "hidden_size": 768, "vocab_size": V}]})
    model = MD.build_model(cfg).to(DEV).train()
    g = torch.Generator().manual_seed(6)
    lens = torch.randint(T // 2, T + 1, (B,), generator=g)
    mask = (torch.arange(T)[None] < lens[:, None]).long()
    ids = torch.randint(1, V, (B, T), generator=g)
    labels = torch.where((torch.rand(B, T, generator=g) < 0.15) & (mask == 1), ids, torch.full_like(ids, -1))
    rows = B * (T + R)
    assert engine.best_splits(768, 768, rows) > 1 and engine.best_splits(3072, 768, rows) > 1

    def batch():
        return SampleList(input_ids=ids, input_mask=mask, lm_label_ids=labels,
                          image=torch.randn(B, R, FEAT, generator=torch.Generator().manual_seed(7)),
                          dataset_name="coco", dataset_type="train").to(DEV)
    _check_model(model, batch)


def test_graphed_visual_bert_steps_are_bitwise_reproducible(deterministic):
    sys.path.insert(0, os.path.dirname(HERE))
    from mmf_b200 import functional as F, modules
    from mmf_b200.graphs import GraphedStep
    model, batch_fn, loss_fn = _visual_bert(B=64)
    state = {k: p.detach().clone() for k, p in model.named_parameters()}
    grads = []
    for _ in range(2):
        with torch.no_grad():
            for k, p in model.named_parameters():
                p.copy_(state[k])
        torch.manual_seed(0)
        modules._SEED_COUNTER[0] = 0
        ep = F.dropout_epoch(DEV)
        if ep is not None:
            ep.zero_()
        step = GraphedStep(model, lambda b: loss_fn(model, b)["loss"], batch_fn())
        step()
        torch.cuda.synchronize()
        grads.append({k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None})
        del step
    assert grads[0].keys() == grads[1].keys() and len(grads[0]) > 0
    for k in grads[0]:
        assert torch.equal(_bits(grads[0][k]), _bits(grads[1][k])), k
