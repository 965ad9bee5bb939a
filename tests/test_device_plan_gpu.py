"""Device-planned packing on the H100: the planning kernel (mmfb_plan_packing) against the static single-stream plan and the
CPU restatement of its rules (tests/plan_ref.py), with guard words around its outputs and valid-looking zeros around its
masks; ViLBERT, LXMERT-encoder and M4C-MMT encoder calls planned on the device against today's host-planned packed calls
(bit for bit, with NaN left in torch's caching allocator so that a row past a count that reached a valid output would
show); one-sided samples against the dense path; and registered vilbert, m4c and m4c_captioner training steps captured by
GraphedStep(static_rows=True) and M4C greedy decodes captured by GraphedForward against the eager static ones, bit for
bit under torch.use_deterministic_algorithms."""
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
import guarded as G  # noqa: E402
import plan_ref as PR  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
PAD = 64                                     # guard elements on each side of every planner buffer


@contextlib.contextmanager
def _deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def _nan_cache():
    G.poison_cache(G.NAN, 1 << 28)


# ---------------------------------------------------------------------------------------------------------------------
# the planning kernel
# ---------------------------------------------------------------------------------------------------------------------
def _guarded(n, dtype, fill):
    base = torch.full((n + 2 * PAD,), fill, dtype=dtype, device=DEV)
    return base, base[PAD:PAD + n]


def _plan_guarded(masks, B, lens, causal_len=0):
    """mmfb_plan_packing on masks surrounded by zeros (a read past a mask would count a valid token) and outputs surrounded
    by sentinel words; checks the guards and returns the outputs on the host"""
    from mmf_b200 import lib
    from mmf_b200.lib import _stream_ptr
    sentinel = G._signed(G.SENTINEL_BITS[torch.int32], 4)
    args, outs, guards = [], [], []
    for m, S in zip(masks, lens):
        if m is None:
            args += [None, S, None, None, None]
            outs.append(None)
            continue
        mb, mv = _guarded(B * S, torch.float32, 0.0)
        mv.copy_(m.reshape(-1))
        bufs = [_guarded(n, torch.int32, sentinel) for n in (B + 1, B * S, B * S)]
        guards += [(mb, 0.0)] + [(b, sentinel) for b, _ in bufs]
        args += [mv.data_ptr(), S] + [v.data_ptr() for _, v in bufs]
        outs.append([v for _, v in bufs])
    if len(masks) == 1:
        args += [None, 0, None, None, None]
    lib.check(lib.LIB.mmfb_plan_packing(*args, B, causal_len, _stream_ptr()))
    torch.cuda.synchronize()
    for base, fill in guards:
        for part in (base[:PAD], base[-PAD:]):
            assert bool((part == fill).all()), "a guard element changed"
    return [None if o is None else [t.cpu() for t in o] for o in outs]


def _single_masks():
    g = torch.Generator().manual_seed(21)
    out = []
    for B, S in ((1, 1), (1, 77), (4, 64), (7, 130), (166, 228), (128, 182)):
        valid = PR.random_valid(B, S, g, kinds=[("empty", 0)] if B > 1 else ())
        out.append(("random", PR.masks_of(valid)))
        out.append(("all_valid", torch.zeros(B, S)))
        out.append(("all_padded", torch.full((B, S), -10000.0)))
        out.append(("soft", PR.masks_of(valid, soft=-1.0)))
        if B * S > 64:
            m = PR.masks_of(valid)
            m.view(-1)[::5] = float("nan")              # NaN is padding, as in the static plan
            out.append(("nan", m))
    return out


@pytest.mark.parametrize("case", range(len(_single_masks())))
def test_single_stream_plan_is_the_static_plan_bit_for_bit(case):
    from mmf_b200 import modules as M
    kind, mask = _single_masks()[case]
    B, S = mask.shape
    cu, pm, um = _plan_guarded([mask], B, [S])[0]
    st = M._plan_packing_static(mask.to(DEV), B, S)
    assert torch.equal(cu, st.varlen.cu_seqlens.cpu()), kind
    assert torch.equal(pm, st.pack_map.cpu()) and torch.equal(um, st.unpack_map.cpu()), kind
    # the functional wrapper returns the same
    (cu2, pm2, um2), = __import__("mmf_b200.functional", fromlist=["x"]).plan_packing([mask.to(DEV)], B, [S])
    assert torch.equal(cu2.cpu(), cu) and torch.equal(pm2.cpu(), pm) and torch.equal(um2.cpu(), um)


@pytest.mark.parametrize("B,S,T", [(1, 9, 1), (5, 70, 12), (3, 64, 64), (128, 182, 12)])
def test_causal_tail_plan_follows_the_rules(B, S, T):
    g = torch.Generator().manual_seed(B + S)
    mask = PR.masks_of(PR.random_valid(B, S, g, kinds=[("empty", 0)]))
    mask[:, S - T:] = torch.where(torch.rand(B, T, generator=g) < 0.5, -10000.0, 0.0)
    got = _plan_guarded([mask], B, [S], causal_len=T)[0]
    want = PR.plan([mask], B, [S], causal_len=T)[0]
    assert all(torch.equal(a, b) for a, b in zip(got, want))


@pytest.mark.parametrize("B,Sa,Sb,none", [(1, 5, 9, None), (9, 20, 37, None), (166, 128, 100, None), (64, 70, 36, 0),
                                          (64, 70, 36, 1)])
def test_two_stream_plan_follows_the_rules(B, Sa, Sb, none):
    g = torch.Generator().manual_seed(B * 7 + Sa)
    kinds_a = [("empty", 0), ("empty", B - 1)] if B > 1 else []
    kinds_b = [("empty", 0)] + ([("full", B - 1)] if B > 1 else [])
    masks = [PR.masks_of(PR.random_valid(B, Sa, g, kinds_a)), PR.masks_of(PR.random_valid(B, Sb, g, kinds_b))]
    if none is not None:
        masks[none] = None
    got = _plan_guarded(masks, B, [Sa, Sb])
    want = PR.plan(masks, B, [Sa, Sb])
    for k in range(2):
        assert (got[k] is None) == (want[k] is None)
        if got[k] is not None:
            assert all(torch.equal(a, b) for a, b in zip(got[k], want[k])), k


def test_argument_errors_launch_nothing():
    from mmf_b200 import functional as F, lib
    m = torch.zeros(2, 8, device=DEV)
    n0 = lib.launch_count()
    for masks, lens, T in (([m], [8], 9), ([m, m], [8, 8], 1), ([None], [8], 0), ([m], [7], 0)):
        with pytest.raises(ValueError):
            F.plan_packing(masks, 2, lens, T)
    with pytest.raises(ValueError):
        F.plan_packing([torch.zeros(4097, 1, device=DEV)], 4097, [1])
    assert lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------------
# encoder calls: planned on the device against today's host-planned packed call
# ---------------------------------------------------------------------------------------------------------------------
def _vilbert_encoder():
    from mmf_b200.modules import B200ViLBertEncoder
    cfg = types.SimpleNamespace(
        hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=4, v_hidden_size=1024,
        v_num_attention_heads=8, v_intermediate_size=1024, v_num_hidden_layers=3, bi_hidden_size=1024,
        bi_num_attention_heads=8, v_biattention_id=[0, 1], t_biattention_id=[2, 3], hidden_dropout_prob=0.0,
        v_hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, v_attention_probs_dropout_prob=0.0)
    torch.manual_seed(0)
    return B200ViLBertEncoder(cfg).to(DEV).train()


def _lxmert_encoder():
    from mmf_b200.lxmert import B200LXMERTEncoder
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, l_layers=2, x_layers=2,
                                r_layers=1, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, visual_feat_dim=64,
                                visual_pos_dim=4, skip_padding=True)
    torch.manual_seed(0)
    return B200LXMERTEncoder(cfg).to(DEV).train()


def _stream_valid(B, T, R, g, one_sided):
    vt = PR.random_valid(B, T, g, [("full", 1)])
    vr = PR.random_valid(B, R, g)
    vt[:, 0] = vr[:, 0] = True                      # every sample has tokens in both streams ...
    vt[3], vr[3] = False, False                     # ... or in neither
    if one_sided:
        vt[5] = False                               # image tokens, no text
        vr[6] = False                               # text tokens, no image
    return vt, vr


def _call(kind, model, x0, x1, m0, m1):
    if kind == "vilbert":
        t, v, _ = model(x0, x1, m0, None, m1, output_all_encoded_layers=False)
        return t[-1], v[-1]
    return model(x0, m0, (x1, None), m1)


def _run(kind, model, x0, x1, m0, m1, w0, w1, static):
    from mmf_b200.graphs import static_rows
    model.zero_grad(set_to_none=True)
    a, b = x0.clone().requires_grad_(True), x1.clone().requires_grad_(True)
    with static_rows() if static else contextlib.nullcontext():
        o0, o1 = _call(kind, model, a, b, m0, m1)
    ((o0.float() * w0).sum() + (o1.float() * w1).sum()).backward()
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    return o0.detach(), o1.detach(), a.grad, b.grad, grads


@pytest.mark.parametrize("kind", ["vilbert", "lxmert"])
def test_two_stream_encoder_call_equals_todays_packed_call(kind):
    from mmf_b200.patch import set_skip_padding
    model = _vilbert_encoder() if kind == "vilbert" else _lxmert_encoder()
    assert set_skip_padding(model, True, two_stream=True, device_plan=True) == 1
    B, T, R = 16, 40, 37
    g = torch.Generator().manual_seed(5)
    vt, vr = _stream_valid(B, T, R, g, one_sided=False)
    m0, m1 = PR.masks_of(vt).to(DEV), PR.masks_of(vr).to(DEV)
    H1 = 1024 if kind == "vilbert" else 64
    x0 = torch.randn(B, T, 768, generator=g).to(DEV)
    x1 = torch.randn(B, R, H1, generator=g).to(DEV)
    w0 = (torch.randn(B, T, 768, generator=g) * vt[..., None]).to(DEV)
    w1 = (torch.randn(B, R, 1024 if kind == "vilbert" else 768, generator=g) * vr[..., None]).to(DEV)
    with _deterministic():
        eager = _run(kind, model, x0, x1, m0, m1, w0, w1, False)
        _nan_cache()
        static = _run(kind, model, x0, x1, m0, m1, w0, w1, True)
    for e, s, what in zip(eager[:4], static[:4], ("out0", "out1", "dx0", "dx1")):
        assert torch.isfinite(s).all(), (kind, what)
        assert torch.equal(e, s), (kind, what, (e.double() - s.double()).abs().max().item())
    # the weight gradients split their k-blocks by the capacity instead of the count: the same sums in another order
    assert eager[4].keys() == static[4].keys()
    for k, ge in eager[4].items():
        gs = static[4][k]
        assert torch.isfinite(gs).all(), (kind, k)
        scale = ge.double().abs().max().item()
        assert (gs.double() - ge.double()).abs().max().item() <= 1e-3 * scale + 1e-6, (kind, k)


@pytest.mark.parametrize("kind", ["vilbert", "lxmert"])
def test_one_sided_samples_agree_with_the_dense_path(kind):
    from mmf_b200.patch import set_skip_padding
    model = _vilbert_encoder() if kind == "vilbert" else _lxmert_encoder()
    B, T, R = 12, 40, 37
    g = torch.Generator().manual_seed(8)
    vt, vr = _stream_valid(B, T, R, g, one_sided=True)
    m0, m1 = PR.masks_of(vt).to(DEV), PR.masks_of(vr).to(DEV)
    H1 = 1024 if kind == "vilbert" else 64
    x0 = torch.randn(B, T, 768, generator=g).to(DEV)
    x1 = torch.randn(B, R, H1, generator=g).to(DEV)
    w0 = (torch.randn(B, T, 768, generator=g) * vt[..., None]).to(DEV)
    w1 = (torch.randn(B, R, 1024 if kind == "vilbert" else 768, generator=g) * vr[..., None]).to(DEV)
    set_skip_padding(model, False, two_stream=True)
    dense = _run(kind, model, x0, x1, m0, m1, w0, w1, False)
    set_skip_padding(model, True, two_stream=True, device_plan=True)
    _nan_cache()
    static = _run(kind, model, x0, x1, m0, m1, w0, w1, True)
    for d, s, v, what in ((dense[0], static[0], vt, "out0"), (dense[1], static[1], vr, "out1"),
                          (dense[2], static[2], vt, "dx0"), (dense[3], static[3], vr, "dx1")):
        v = v.to(DEV)
        assert torch.isfinite(s).all(), (kind, what)
        d, s = d.float()[v], s.float()[v]
        # bf16 activations through several layers: the difference of two roundings of the same function
        tol = 3e-2 * d.abs().max().item() + 1e-3
        assert (d - s).abs().max().item() <= tol, (kind, what, (d - s).abs().max().item(), tol)


def test_m4c_mmt_call_with_a_causal_tail_equals_todays_packed_call():
    from mmf_b200.graphs import static_rows
    from mmf_b200.modules import B200BertEncoder, run_bert_encoder
    cfg = types.SimpleNamespace(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=4,
                                hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-12)
    torch.manual_seed(0)
    enc = B200BertEncoder(cfg).to(DEV).train()
    r = enc._runner
    r.skip_padding = r.pack_tail = r.device_plan = True
    B, S, D = 24, 182, 12
    g = torch.Generator().manual_seed(3)
    valid = PR.random_valid(B, S, g, [("empty", 2)])
    mask = PR.masks_of(valid)
    mask[:, S - D:] = 0.0
    mask = mask.to(DEV)
    x0 = torch.randn(B, S, 768, generator=g).to(DEV)
    keep = valid.clone()
    keep[:, S - D:] = True
    w = (torch.randn(B, S, 768, generator=g) * keep[..., None]).to(DEV)

    def run(static):
        enc.zero_grad(set_to_none=True)
        x = x0.clone().requires_grad_(True)
        with static_rows() if static else contextlib.nullcontext():
            out = run_bert_encoder(r, x, mask, True, causal_len=D)[0]
        (out.float() * w).sum().backward()
        return out.detach(), x.grad

    with _deterministic():
        o_e, d_e = run(False)
        _nan_cache()
        o_s, d_s = run(True)
    assert torch.isfinite(o_s).all() and torch.isfinite(d_s).all()
    assert torch.equal(o_s, o_e) and torch.equal(d_s, d_e)


# ---------------------------------------------------------------------------------------------------------------------
# captured steps and decodes
# ---------------------------------------------------------------------------------------------------------------------
def _registered(name):
    import test_graphed_forward_gpu as GF
    from mmf_b200.patch import set_skip_padding
    model, batch = GF._case(name)
    for m in model.modules():                       # dropout off: the captured and eager steps draw nothing
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    n = set_skip_padding(model, True, two_stream=True, causal=True, device_plan=True)
    assert n >= 1
    runners = [m.__dict__.get("_runner") for m in model.modules()]
    assert any(getattr(r, "pack_tail", False) or getattr(r, "pack_streams", False) for r in runners)
    return model, batch, GF


def _loss_of(GF):
    return lambda m: (lambda b: sum(v.sum() for v in m(GF._fresh(b))["losses"].values()))


@pytest.mark.parametrize("with_optimizer", [False, True])
@pytest.mark.parametrize("name", ["vilbert", "m4c", "m4c_captioner"])
def test_captured_step_is_the_eager_static_step_bit_for_bit(name, with_optimizer):
    from mmf_b200.graphs import GraphedStep, static_rows
    from mmf_b200.optim import B200AdamW
    model, batch, GF = _registered(name)
    model.train()
    loss_of = _loss_of(GF)
    with _deterministic():
        twin = copy.deepcopy(model)
        with static_rows():
            loss_of(twin)(batch).backward()         # the twin's lazy engine state
        twin.zero_grad(set_to_none=True)
        opt = opt_t = None
        if with_optimizer:
            opt = B200AdamW(model.parameters(), lr=1e-4, weight_decay=0.01, capturable=True)
            opt_t = B200AdamW(twin.parameters(), lr=1e-4, weight_decay=0.01, capturable=True)
        _nan_cache()
        step = GraphedStep(model, loss_of(model), batch, warmup=2, static_rows=True, optimizer=opt)
        for seed in (1, 2):
            b = GF._variant(batch, seed)
            loss = step(b)
            twin.zero_grad(set_to_none=True)
            with static_rows():
                ref = loss_of(twin)(b)
            ref.backward()
            if opt_t is not None:
                opt_t.step()
            torch.cuda.synchronize()
            assert torch.isfinite(loss).all()
            assert torch.equal(loss.detach(), ref.detach()), (name, seed, loss.item(), ref.item())
            for (n, p), q in zip(model.named_parameters(), twin.parameters()):
                assert (p.grad is None) == (q.grad is None), (name, n)
                assert p.grad is None or torch.equal(p.grad, q.grad), (name, seed, n)
                assert torch.equal(p.detach(), q.detach()), (name, seed, n)


@pytest.mark.parametrize("name", ["m4c", "m4c_captioner"])
def test_captured_greedy_decode_is_the_eager_decode(name):
    from mmf_b200.graphs import GraphedForward, static_rows
    model, batch, GF = _registered(name)
    model.eval()
    with torch.no_grad(), static_rows():
        model(GF._fresh(batch))                     # the lazy engine state
    fwd = GraphedForward(model, batch, static_rows=True)
    for seed in (1, 2):
        b = GF._variant(batch, seed)
        got = GF._snapshot(fwd(b))
        with torch.no_grad(), static_rows():
            want = model(GF._fresh(b))
        torch.cuda.synchronize()
        GF._assert_same(got, want, "%s/%d" % (name, seed))
