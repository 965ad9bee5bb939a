"""Skip-padding under static_rows() on the H100: the device-bounded GEMM epilogues of the encoder layer and the bounded
LayerNorm forward and backward against the unbounded calls on the rows below the bound, one bert-base encoder call planned
on the device against today's host-planned packed call, and registered VisualBERT and MMF-Transformer (masked-LM) steps
captured by GraphedStep(static_rows=True) against the eager static step, bit for bit under
torch.use_deterministic_algorithms."""
import contextlib
import copy
import os
import sys
import types

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import kernel_check as KC  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
TILE = 128
NAN = float("nan")


@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _bound(c):
    return torch.tensor([c], dtype=torch.int32, device=DEV)


def _rounded(c, M):
    return min(M, -(-c // TILE) * TILE)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _nan_cache():
    """leave NaN in freed blocks of torch's caching allocator: a buffer the static path reads without writing it first
    (rows past the count) then shows up as NaN instead of passing on stale finite values"""
    for n in (1 << 20, 1 << 24, 1 << 26, 1 << 28):
        for _ in range(4):
            torch.full((n,), NAN, dtype=torch.bfloat16, device=DEV)
    torch.cuda.synchronize()


def _poison(t, b, value=NAN):
    """t with rows at and past b set to `value` (a copy)"""
    t = t.clone()
    t[b:] = value
    return t


# ---------------------------------------------------------------------------------------------------------------------
# bounded GEMM epilogues
# ---------------------------------------------------------------------------------------------------------------------
M_GEMM = 384


@pytest.mark.parametrize("N", [128, 768])
@pytest.mark.parametrize("epi", ["bias_drop_resid", "bias_gelu", "gelu_bwd", "add_aux"])
def test_bounded_gemm_epilogues_equal_the_unbounded_call(epi, N):
    from mmf_b200 import functional as F, lib
    g = torch.Generator().manual_seed(3)
    M, K = M_GEMM, 256
    a = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    wt = w.t().contiguous()                                  # [K, N]: the dgrad's MN-major B
    bias = (torch.randn(N, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    aux = torch.randn(M, N, generator=g).to(torch.bfloat16).to(DEV)
    words = torch.randint(-2 ** 31, 2 ** 31 - 1, (M, (N + 31) // 32), generator=g, dtype=torch.int64).to(torch.int32).to(DEV)

    def call(a_, aux_, words_, M_, out=None, out2=None, m_bound=None):
        kw = {} if m_bound is None else {"m_bound": m_bound}
        if epi == "bias_drop_resid":
            return (F.gemm(a_, w, epi=lib.EPI_BIAS_DROP_RESID, bias=bias, aux=aux_, drop_mask=words_, drop_scale=1.0 / 0.9,
                           out=out, **kw),)
        if epi == "bias_gelu":
            return F.gemm(a_, w, epi=lib.EPI_BIAS_GELU, bias=bias, out=out, out2=out2, **kw)
        e = lib.EPI_GELU_BWD if epi == "gelu_bwd" else lib.EPI_ADD_AUX
        return (F.gemm(a_, wt, b_mn=True, epi=e, aux=aux_, out=out, **kw),)

    for b in sorted({0, 1, 127, 128, 129, M}):
        r = _rounded(b, M)
        # NaN in A and aux past the bound, and all-ones keep bits there: none of it may reach a row below the bound
        a_p, aux_p, words_p = _poison(a, b), _poison(aux, b), _poison(words, b, -1)
        outs = [torch.full((M, N), NAN, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
        got = call(a_p, aux_p, words_p, M, out=outs[0], out2=outs[1], m_bound=_bound(b))
        if b:
            want = call(a[:b].contiguous(), aux[:b].contiguous(), words[:b].contiguous(), b)
            for gt, wn in zip(got, want):
                assert torch.equal(_bits(gt[:b]), _bits(wn)), (epi, N, b)
                assert not torch.isnan(gt[:b].float()).any()
        for gt in got:
            assert torch.isnan(gt[r:].float()).all(), (epi, N, b, "rows past the rounded bound were written")


# ---------------------------------------------------------------------------------------------------------------------
# bounded LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
M_LN = 300


def _ln_inputs(H, seed):
    g = torch.Generator().manual_seed(seed)
    y = (torch.randn(M_LN, H, generator=g) * 2 + 0.3).to(torch.bfloat16).to(DEV)
    gam = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).to(DEV)
    bet = (0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).to(DEV)
    dx = torch.randn(M_LN, H, generator=g).to(torch.bfloat16).to(DEV)
    dx2 = torch.randn(M_LN, H, generator=g).to(torch.bfloat16).to(DEV)
    words = torch.randint(-2 ** 31, 2 ** 31 - 1, (M_LN, (H + 31) // 32), generator=g, dtype=torch.int64).to(torch.int32)
    return y, gam, bet, dx, dx2, words.to(DEV)


@pytest.mark.parametrize("H", [768, 1024, 2048])
def test_bounded_layernorm_forward_equals_the_unbounded_call(H):
    from mmf_b200 import functional as F
    y, gam, bet, _, _, words = _ln_inputs(H, 5)
    for drop in (False, True):
        for b in sorted({0, 1, 127, 128, 129, M_LN}):
            out = torch.full((M_LN, H), NAN, dtype=torch.bfloat16, device=DEV)
            y_p = _poison(y, b, float("inf"))
            x, mean, rstd = F.layernorm_fwd(y_p, gam, bet, out=out, m_bound=_bound(b),
                                            **({"drop_mask": _poison(words, b, -1), "drop_scale": 1.0 / 0.9} if drop else {}))
            assert torch.isnan(x[b:].float()).all() and not mean[b:].any() and not rstd[b:].any()
            if b:
                kw_b = {"drop_mask": words[:b].contiguous(), "drop_scale": 1.0 / 0.9} if drop else {}
                xr, mr, rr = F.layernorm_fwd(y[:b].contiguous(), gam, bet, **kw_b)
                assert torch.equal(_bits(x[:b]), _bits(xr)) and torch.equal(_bits(mean[:b]), _bits(mr))
                assert torch.equal(_bits(rstd[:b]), _bits(rr)), (H, drop, b)


@pytest.mark.parametrize("H", [768, 1024, 2048])
@pytest.mark.parametrize("ordered", [False, True])
def test_bounded_layernorm_backward_equals_the_unbounded_call(H, ordered):
    from mmf_b200 import functional as F
    y, gam, bet, dx, dx2, words = _ln_inputs(H, 7)
    _, mean, rstd = F.layernorm_fwd(y, gam, bet)
    for with_dx2 in (False, True):
        for drop in (False, True):
            for b in sorted({0, 1, 127, 128, 129, M_LN}):
                sums = [torch.zeros(H, dtype=torch.float32, device=DEV) for _ in range(6)]
                with _deterministic(ordered):
                    dy, dz = F.layernorm_bwd(
                        _poison(dx, b), _poison(y, b, float("inf")), _poison(mean, b), _poison(rstd, b), gam,
                        sums[0], sums[1], dbias=sums[2], dx2=_poison(dx2, b) if with_dx2 else None,
                        drop_mask=_poison(words, b, -1) if drop else None, drop_scale=1.0 / 0.9, m_bound=_bound(b))
                    if b:
                        dyr, dzr = F.layernorm_bwd(
                            dx[:b].contiguous(), y[:b].contiguous(), mean[:b].contiguous(), rstd[:b].contiguous(), gam,
                            sums[3], sums[4], dbias=sums[5], dx2=dx2[:b].contiguous() if with_dx2 else None,
                            drop_mask=words[:b].contiguous() if drop else None, drop_scale=1.0 / 0.9)
                what = (H, ordered, with_dx2, drop, b)
                assert not dy[b:].any() and not dz[b:].any(), what          # zero-allocated, never written
                for s in sums[:3]:
                    assert torch.isfinite(s).all(), what
                if not b:
                    assert not any(s.any() for s in sums[:3]), what
                    continue
                assert torch.equal(_bits(dy[:b]), _bits(dyr)) and torch.equal(_bits(dz[:b]), _bits(dzr)), what
                if ordered:
                    for s, r in zip(sums[:3], sums[3:]):
                        assert torch.equal(_bits(s), _bits(r)), what
                else:
                    keep = F.unpack_keep_bits(words[:b], H).cpu() if drop else None
                    fw = KC.layernorm_ref(y[:b].cpu(), gam.cpu(), bet.cpu())
                    ref = KC.layernorm_bwd_ref(fw, dx[:b].cpu(), gam.cpu(), dx2[:b].cpu() if with_dx2 else None, keep,
                                               1.0 / 0.9, n_sum_terms=b + 8 + 2 * 132)
                    assert bool(((sums[0].cpu().double() - ref["dgamma"]).abs() <= KC.SAFETY * ref["b_dgamma"]).all()), what
                    assert bool(((sums[1].cpu().double() - ref["dbeta"]).abs() <= KC.SAFETY * ref["b_dbeta"]).all()), what
                    # dbias sums dz in fp32, before (register kernel, streaming kernel without dropout) or after (streaming
                    # kernel with dropout) its bf16 rounding: b_dz covers both
                    bz = KC.SAFETY * (ref["b_dz"].sum(0) + KC.U_F32 * (b + 8 + 2 * 132) * ref["dz"].abs().sum(0))
                    assert bool(((sums[2].cpu().double() - ref["dz"].sum(0)).abs() <= bz).all()), what


# ---------------------------------------------------------------------------------------------------------------------
# one encoder call: static against today's packed call
# ---------------------------------------------------------------------------------------------------------------------
T_TXT, R_REG = 128, 100


def _valid(kind, B, g):
    S = T_TXT + R_REG
    if kind in ("bench", "short_text"):
        text = (64, 128) if kind == "bench" else (8, 24)
        regs = (50, 100) if kind == "bench" else (10, 100)
        lens = torch.randint(text[0], text[1] + 1, (B,), generator=g)
        nreg = torch.randint(regs[0], regs[1] + 1, (B,), generator=g)
        return torch.cat([torch.arange(T_TXT)[None] < lens[:, None], torch.arange(R_REG)[None] < nreg[:, None]], 1)
    v = torch.ones(B, S, dtype=torch.bool)
    if kind == "one_padding_sample":
        v[1] = False
    elif kind == "all_padding":
        v[:] = False
    return v


def _bert_base(p=0.0):
    from mmf_b200.modules import B200BertEncoder
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12,
                                hidden_dropout_prob=p, attention_probs_dropout_prob=p, layer_norm_eps=1e-12,
                                skip_padding=True)
    torch.manual_seed(0)
    return B200BertEncoder(cfg).to(DEV)


@pytest.mark.parametrize("kind", ["bench", "short_text", "all_valid", "one_padding_sample", "all_padding"])
def test_static_encoder_call_equals_todays_packed_call(kind):
    from mmf_b200.graphs import static_rows
    from mmf_b200.modules import run_bert_encoder
    enc = _bert_base().train()
    runner = enc._runner
    B = 16
    g = torch.Generator().manual_seed(11)
    valid = _valid(kind, B, g)
    mask = ((~valid).float() * -10000.0).to(DEV)
    x0 = torch.randn(B, T_TXT + R_REG, 768, generator=g).to(DEV)
    w = (torch.randn(B, T_TXT + R_REG, 768, generator=g) * valid[..., None]).to(DEV)

    def run(static):
        enc.zero_grad(set_to_none=True)
        x = x0.clone().requires_grad_(True)
        with static_rows() if static else contextlib.nullcontext():
            out = run_bert_encoder(runner, x, mask, True)[0]
        (out.float() * w).sum().backward()
        return out.detach(), x.grad, {k: p.grad.clone() for k, p in enc.named_parameters() if p.grad is not None}

    o_t, dx_t, g_t = run(False)
    _nan_cache()
    o_s, dx_s, g_s = run(True)
    assert torch.equal(o_s, o_t) and torch.equal(dx_s, dx_t), kind
    if kind == "all_padding":
        assert not o_s.any() and not dx_s.any() and all(not v.any() for v in g_s.values())
        return
    # parameter gradients: the weight gradients split their k-blocks by the capacity instead of the count, so they are
    # the same sums in another order; both must sit inside the fp32 accumulation bound of the same sum of |terms|
    assert g_s.keys() == g_t.keys() and len(g_s) == 16 * 12
    for k in g_t:
        scale = g_t[k].double().abs().max().item()
        err = (g_s[k].double() - g_t[k].double()).abs().max().item()
        assert err <= 1e-3 * scale + 1e-6, (kind, k, err, scale)


# ---------------------------------------------------------------------------------------------------------------------
# whole steps: GraphedStep(static_rows=True) replays against the eager static step
# ---------------------------------------------------------------------------------------------------------------------
def _visual_bert():
    import bench
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.visual_bert import B200VisualBERT
    wl = bench.VisualBertWL()
    torch.manual_seed(0)
    model = B200VisualBERT(wl.config(0.1)).to(DEV).train()
    assert set_skip_padding(model) >= 1
    B = 32
    base = bench.to_device(wl.host_batch(B, 17), DEV)
    aux = wl.aux(B, DEV)
    full = copy.deepcopy(base)
    full["input_mask"].fill_(1)
    full["image_info_0"]["max_features"].fill_(base["image_feature_0"].shape[1])
    one_empty = copy.deepcopy(base)
    one_empty["input_mask"][3] = 0
    return model, [base, full, one_empty], (lambda m: (lambda b: wl.loss(m, b, aux)))


def _mmf_transformer():
    import mmf_b200.mmft  # noqa: F401
    from mmf_b200 import models as MD
    from mmf_b200.patch import set_skip_padding
    from mmf_b200.sample import SampleList
    B, T, R, FEAT, V = 16, 128, 100, 2048, 30522
    torch.manual_seed(0)
    cfg = MD.load_model_config("mmf_transformer", overrides={
        "modalities": [dict(type="text", key="text", embedding_dim=768, position_dim=512, segment_id=0),
                       dict(type="image", key="image", embedding_dim=FEAT, position_dim=R, segment_id=1,
                            encoder=dict(type="identity"))],
        "heads": [{"type": "mlm", "hidden_size": 768, "vocab_size": V}]})
    model = MD.build_model(cfg).to(DEV).train()
    assert set_skip_padding(model) >= 1
    g = torch.Generator().manual_seed(6)
    batches = []
    for kind in ("random", "full", "one_empty"):
        lens = torch.randint(T // 2, T + 1, (B,), generator=g)
        if kind == "full":
            lens[:] = T
        mask = (torch.arange(T)[None] < lens[:, None]).long()
        if kind == "one_empty":
            mask[2] = 0
        ids = torch.randint(1, V, (B, T), generator=g)
        labels = torch.where((torch.rand(B, T, generator=g) < 0.15) & (mask == 1), ids, torch.full_like(ids, -1))
        batches.append({"input_ids": ids.to(DEV), "input_mask": mask.to(DEV), "lm_label_ids": labels.to(DEV),
                        "image": torch.randn(B, R, FEAT, generator=g).to(DEV),
                        "is_correct": torch.ones((), dtype=torch.long, device=DEV)})    # else made from a host value

    def loss_of(m):
        def run(b):
            out = m(SampleList(dict(b, dataset_name="coco", dataset_type="train")))
            return sum(v.sum() for v in out["losses"].values())
        return run
    return model, batches, loss_of


@pytest.mark.parametrize("name", ["visual_bert", "mmf_transformer"])
def test_graphed_static_packing_step_is_the_eager_step_bit_for_bit(name):
    from mmf_b200 import functional as F, modules
    from mmf_b200.graphs import GraphedStep, static_rows
    model, batches, loss_of = {"visual_bert": _visual_bert, "mmf_transformer": _mmf_transformer}[name]()

    def grads(m):
        return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}

    # torch's own dropout modules outside the encoder layers (embeddings, heads) draw from torch's generator, whose
    # offsets a graph replay advances differently from an eager step; the library's dropout (every encoder layer, p = 0.1)
    # is drawn from the frozen (seed, offset) and the dropout epoch, which the eager step below reproduces
    for n, m in model.named_modules():
        if isinstance(m, torch.nn.Dropout) and "layer" not in n:
            m.p = 0.0
    _nan_cache()
    with _deterministic():
        twin = copy.deepcopy(model)
        with static_rows():
            loss_of(twin)(batches[0]).backward()     # the twin's lazy engine state, outside the sync check
        c0 = modules._SEED_COUNTER[0]
        step = GraphedStep(model, loss_of(model), batches[0], warmup=3, static_rows=True)
        c1 = modules._SEED_COUNTER[0]
        per_step = (c1 - c0) // 4                    # fresh dropout streams per step (three warm-ups and the capture)
        assert per_step >= 1 and (c1 - c0) % 4 == 0
        epoch = F.dropout_epoch(DEV)
        for b in batches:
            loss = step(b)                           # advances the dropout epoch the eager step reads below
            twin.zero_grad(set_to_none=True)
            modules._SEED_COUNTER[0] = c1 - per_step  # the (seed, offset) the capture froze
            torch.cuda.set_sync_debug_mode("error")
            try:
                with static_rows():
                    ref = loss_of(twin)(b)
                ref.backward()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            assert epoch is not None
            assert torch.equal(loss.detach(), ref.detach()), (name, loss.item(), ref.item())
            got, want = grads(model), grads(twin)
            assert len(want) > 20 and got.keys() == want.keys()
            for n, gr in want.items():
                assert torch.equal(got[n], gr), (name, n)
