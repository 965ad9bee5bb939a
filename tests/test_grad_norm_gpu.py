"""mmfb_grad_norm and the clip coefficient AdamW reads from device memory, on the H100: exact sums at the block-partition
edges, the rounding bound on random gradients, repeatable bits, B200AdamW.clip_grad_norm + step() against
torch.nn.utils.clip_grad_norm_ + step() (VisualBERT trunk + head, non-finite gradients, no host synchronisation, CUDA-graph
capture, data-parallel ordering), and MMF's clip_gradients hook branch on the registered m4c model."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

BLOCK = 16384          # MMFB_GRAD_NORM_BLOCK
LENGTHS = [1, 7, 8, 9, BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK + 3, 5 * BLOCK - 8]


@pytest.fixture(scope="module")
def F():
    import mmf_b200.functional as F
    return F


def _fp64_norm(grads):
    return torch.linalg.vector_norm(torch.cat([g.reshape(-1).double() for g in grads])).float()


def _torch_coef(norm, max_norm):
    return torch.clamp(max_norm / (norm + 1e-6), max=1.0)


def _segments(kind, seed):
    """fp32 and bf16 segments alternating over LENGTHS, plus two views that start one element into their storage (the
    element-by-element path of the kernel); `exact`: small integers times 2^-4, so every sum of squares is exact"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for i, n in enumerate(LENGTHS + [BLOCK + 5, 300]):
        dt = torch.float32 if i % 2 == 0 else torch.bfloat16
        if kind == "exact":
            t = torch.randint(-8, 9, (n + 1,), generator=g, device="cuda").to(dt) * 0.0625
        else:
            t = (torch.randn(n + 1, generator=g, device="cuda") * 10.0 ** (i % 5 - 2)).to(dt)
        out.append(t[1:] if i >= len(LENGTHS) else t[:n])
    return out


def test_exact_sums_equal_the_fp64_norm_at_block_edges(F):
    grads = _segments("exact", 0)
    assert any(g.data_ptr() % 16 for g in grads)
    out = F.grad_norm(F.grad_norm_table(grads), 3.0)
    ref = _fp64_norm(grads)
    assert torch.equal(out[0], ref), (float(out[0]), float(ref))
    assert torch.equal(out[1], _torch_coef(ref, 3.0))
    for n in LENGTHS:                                   # one segment alone, either dtype
        for dt in (torch.float32, torch.bfloat16):
            t = (torch.arange(n, device="cuda") % 17 - 8).to(dt) * 0.25
            assert torch.equal(F.grad_norm(F.grad_norm_table([t]), 1.0)[0], _fp64_norm([t])), (n, dt)


def test_random_gradients_are_within_one_fp32_ulp_of_fp64(F):
    for seed in range(4):
        grads = _segments("random", seed)
        got = F.grad_norm(F.grad_norm_table(grads), 1.0)[0].double()
        exact = torch.linalg.vector_norm(torch.cat([g.reshape(-1).double() for g in grads]))
        assert abs(float(got - exact)) <= 2.0 ** -23 * float(exact), (seed, float(got), float(exact))


def test_two_calls_give_the_same_bits_in_both_modes(F):
    grads = _segments("random", 7)
    table = F.grad_norm_table(grads)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        outs = []
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            outs += [F.grad_norm(table, 0.5), F.grad_norm(F.grad_norm_table(grads), 0.5)]
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(o, outs[0]) for o in outs[1:])


def test_norm_type_other_than_2_is_refused_by_the_entry_point(F):
    import ctypes
    from mmf_b200 import lib
    t = torch.ones(8, device="cuda")
    table = F.grad_norm_table([t])
    out = torch.empty(2, device="cuda")
    part = torch.empty(1, dtype=torch.float64, device="cuda")
    a = lib.GradNormArgs(table.segments.data_ptr(), 1, 1, part.data_ptr(), out.data_ptr(), 1.0, 1.0)
    assert lib.LIB.mmfb_grad_norm(ctypes.byref(a), lib._stream_ptr()) == lib.MMFB_ERR_ARG
    with pytest.raises(ValueError):
        F.grad_norm(table, 1.0, norm_type=float("inf"))


# ---- B200AdamW.clip_grad_norm ---------------------------------------------------------------------------------------
class _Trunk(torch.nn.Module):
    """VisualBERT trunk (2 layers; its fusion layers live in a parameter pack) plus a head outside any pack"""

    def __init__(self):
        super().__init__()
        import bench
        from mmf_b200.visual_bert import B200VisualBERT
        self.trunk = B200VisualBERT(bench.bert_config(768, 12, 3072, 2, 0.0, visual_embedding_dim=2048))
        self.head = torch.nn.Linear(768, 5)

    def forward(self, batch):
        return self.head(self.trunk(batch)["sequence_output"])


def _batch(seed, B=4):
    import bench
    wl = bench.WORKLOADS["visual_bert"]()
    return bench.to_device(wl.host_batch(B, seed), torch.device("cuda"))


def _pair():
    torch.manual_seed(0)
    a = _Trunk().cuda().train()
    b = _Trunk().cuda().train()
    b.load_state_dict(a.state_dict())
    return a, b


def _backward(model, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed + 1000)
    out = model(_batch(seed))
    (out * torch.randn(out.shape, generator=g, device="cuda") * scale).sum().backward()


def _opt(model):
    from mmf_b200.optim import B200AdamW
    return B200AdamW(model.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01, arithmetic="torch")


def _close(a, b, what):
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        err = (p.detach() - q.detach()).abs().max() / q.detach().abs().max().clamp_min(1e-6)
        assert err < 2e-6, (what, n, float(err))


@pytest.fixture()
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)       # the two models' gradients are then equal bit for bit
    yield
    torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("max_norm", [0.05, 1e6])
def test_clip_and_step_match_torch_clip_grad_norm(deterministic, max_norm):
    a, b = _pair()
    oa, ob = _opt(a), _opt(b)
    for step in range(2):
        for m in (a, b):
            m.zero_grad(set_to_none=False)
            _backward(m, step)
        pack = a.trunk.bert.encoder._runner.pack          # packed and loose gradients are both in play
        assert all(p.grad.data_ptr() == pack.grad.data_ptr() + 4 * o for p, o in zip(pack.params, pack.offsets))
        assert a.head.weight.grad is not None
        na = oa.clip_grad_norm(max_norm)
        nb = torch.nn.utils.clip_grad_norm_(b.parameters(), max_norm)
        assert na.is_cuda and na.dim() == 0 and na.dtype == torch.float32
        assert torch.allclose(na, nb, rtol=2e-6, atol=0), (float(na), float(nb))
        coef = float(_torch_coef(na, max_norm))
        assert (coef < 0.5) if max_norm < 1 else (coef == 1.0)
        oa.step()
        ob.step()
        _close(a, b, "step %d" % step)


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_non_finite_gradients_follow_torch(deterministic, bad):
    a, b = _pair()
    oa, ob = _opt(a), _opt(b)
    for m in (a, b):
        _backward(m, 3)
        m.trunk.bert.encoder.layer[0].attention.self.query.weight.grad[0, 0] = bad     # a packed gradient
        m.head.bias.grad[1] = bad                                                         # a loose one
    na = oa.clip_grad_norm(1.0)
    nb = torch.nn.utils.clip_grad_norm_(b.parameters(), 1.0)
    assert torch.equal(na.isnan(), nb.isnan()) and torch.equal(na.isinf(), nb.isinf())
    oa.step()
    ob.step()
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=2e-6, atol=1e-7, equal_nan=True, msg=n)
    assert not torch.isfinite(a.head.bias).all()


def test_clip_and_step_do_not_synchronise_with_the_host():
    a, _ = _pair()
    oa = _opt(a)
    _backward(a, 4)
    oa.clip_grad_norm(0.1)                 # builds the segment table and the flat optimizer state
    oa.step()
    a.zero_grad(set_to_none=False)
    _backward(a, 5)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        norm = oa.clip_grad_norm(0.1)
        oa.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(norm)


def test_clip_and_step_capture_in_a_cuda_graph(deterministic):
    a, b = _pair()
    oa, ob = _opt(a), _opt(b)
    for m, o in ((a, oa), (b, ob)):       # eager first call: segment table, flat state
        _backward(m, 6)
        o.clip_grad_norm(0.1)
        o.step()
    _close(a, b, "eager")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = oa.clip_grad_norm(0.1)
        oa.step()
    g = torch.Generator(device="cuda").manual_seed(11)
    for p, q in zip(a.parameters(), b.parameters()):  # fresh gradients, written in place
        if p.grad is None:                             # the unused pooler
            assert q.grad is None
            continue
        fresh = torch.randn(p.shape, generator=g, device="cuda") * 1e-2
        p.grad.copy_(fresh)
        q.grad.copy_(fresh)
    graph.replay()
    eager = ob.clip_grad_norm(0.1)
    ob.step()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)
    for (n, p), q in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(p.detach(), q.detach()), n


@pytest.mark.parametrize("mode", ["bucket", "end"])
def test_data_parallel_norm_is_taken_after_the_all_reduce(deterministic, monkeypatch, mode):
    """The reduction is replaced by a halving that first sleeps ~0.1 s on the stream it is issued on (the side stream of
    the bucket all-reduces), with the wrapper told the world has two ranks.  The norm must be exactly half the local one:
    a norm launched before the end-of-backward join would read unreduced gradients."""
    import mmf_b200.ddp as D
    monkeypatch.setattr(D.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(D.dist, "get_world_size", lambda group=None: 1)
    a, b = _pair()
    dp = D.B200DataParallel(a, mode=mode, bucket_bytes=1 << 20)
    dp.world = 2

    def slow_half(flat):
        torch.cuda._sleep(200_000_000)
        flat.mul_(0.5)
    dp._avg_raw = slow_half
    oa, ob = _opt(a), _opt(b)
    g = torch.Generator(device="cuda").manual_seed(1000)
    out = dp(_batch(0))
    (out * torch.randn(out.shape, generator=g, device="cuda")).sum().backward()
    na = oa.clip_grad_norm(1.0)
    _backward(b, 0)
    nb = ob.clip_grad_norm(1.0)
    torch.cuda.synchronize()
    assert torch.equal(na, nb * 0.5), (float(na), float(nb))


# ---- the registered m4c model through MMF's clip_gradients ----------------------------------------------------------
def _clip_gradients(model, optimizer, max_grad_l2_norm, clip_norm_mode="all", scale=1.0):
    """mmf/utils/general.py clip_gradients (the writer left out)"""
    if max_grad_l2_norm is not None:
        if clip_norm_mode == "all":
            if hasattr(optimizer, "clip_grad_norm"):
                return optimizer.clip_grad_norm(max_grad_l2_norm * scale)
            return torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_l2_norm * scale)
        raise NotImplementedError("Clip norm mode %s not implemented" % clip_norm_mode)


def test_m4c_step_through_the_clip_gradients_hook_matches_the_fallback():
    import mmf_b200.models as MD
    from mmf_b200.models import ConfigNode
    from mmf_b200.optim import B200AdamW
    from mmf_b200.registry import registry
    from mmf_b200.sample import SampleList
    import test_m4c_model_cpu as C
    golden = torch.load(os.path.join(C.GOLD, "m4c_model.pt"), weights_only=False)
    C.register(golden)
    registry.register(golden["dataset"] + "_num_final_outputs", 5050)
    torch.manual_seed(0)
    model = MD.build_model(MD.load_model_config("m4c")).cuda().train()
    B, T, R, O, D = 8, 20, 100, 50, 12
    dev = "cuda"
    sl = SampleList(text=torch.randint(1, 30522, (B, T), device=dev), text_len=torch.randint(1, T + 1, (B,), device=dev),
                    image_feature_0=torch.randn(B, R, 2048, device=dev).relu(), obj_bbox_coordinates=torch.rand(B, R, 4, device=dev),
                    image_info_0={"max_features": torch.randint(10, R + 1, (B,), device=dev)},
                    context_feature_0=torch.randn(B, O, 300, device=dev), context_feature_1=torch.rand(B, O, 604, device=dev),
                    image_feature_1=torch.randn(B, O, 2048, device=dev).relu(), order_vectors=torch.zeros(B, O, 50, device=dev),
                    ocr_bbox_coordinates=torch.rand(B, O, 4, device=dev),
                    context_info_0={"max_features": torch.randint(0, O + 1, (B,), device=dev)},
                    train_prev_inds=torch.randint(0, 5050, (B, D), device=dev),
                    targets=(torch.rand(B, D, 5050, device=dev) < 0.01).float(),
                    train_loss_mask=(torch.rand(B, D, device=dev) < 0.7).float(), dataset_name="textvqa", dataset_type="train")
    C.loss_of(model(sl)).sum().backward()
    params0 = {n: p.detach().clone() for n, p in model.named_parameters()}
    grads0 = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    cfg = ConfigNode({"optimizer": {"type": "Adam", "params": {"lr": 1e-4, "eps": 1e-8, "weight_decay": 0}}})
    hp = dict(lr=1e-4, eps=1e-8, weight_decay=0.0)

    # hook branch: B200AdamW has clip_grad_norm
    opt = B200AdamW(model.get_optimizer_parameters(cfg), arithmetic="torch", **hp)
    norm_hook = _clip_gradients(model, opt, 0.25)
    opt.step()
    hooked = {n: p.detach().clone() for n, p in model.named_parameters()}
    # fallback branch on the same parameters and gradients: torch.optim.Adam has no clip_grad_norm
    for n, p in model.named_parameters():
        p.data.copy_(params0[n])
        if n in grads0:
            p.grad.copy_(grads0[n])
    ref = torch.optim.Adam(model.get_optimizer_parameters(cfg), **hp)
    assert not hasattr(ref, "clip_grad_norm")
    norm_ref = _clip_gradients(model, ref, 0.25)
    ref.step()
    assert norm_hook.is_cuda and float(norm_ref) > 0.25
    assert torch.allclose(norm_hook, norm_ref, rtol=2e-6, atol=0), (float(norm_hook), float(norm_ref))
    moved = 0
    for n, p in model.named_parameters():
        torch.testing.assert_close(hooked[n], p.detach(), rtol=1e-6, atol=1e-7, msg=n)
        moved += int(not torch.equal(p.detach(), params0[n]))
    assert moved > 0
