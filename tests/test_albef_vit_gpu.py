"""The registered `albef_vit_encoder` on the H100.
  * eval forward and backward against tests/golden/albef_vit.pt (the reference's own VisionTransformer in fp32), at a
    small geometry and at the default 224 px / patch 16 (197 positions);
  * a training step with drop_rate, attn_drop_rate and drop_path_rate > 0 against the fp64 restatement of
    tests/albef_vit_check.py fed the kernels' own keep bits, element by element: |product - fp64| <= 6 x (the bf16
    restatement's own error, at that element or as its row's rms) + 8 bf16 ulps + 3e-2 x rms(fp64 row), so one misrouted
    mask row or sample
    shows, and per tensor in relative L2 within 1.5 x the bf16 restatement's + 2e-3;
  * every sample a DropPath draw drops leaves its residual input unchanged, bit for bit;
  * one step under GraphedStep equals the eager step bit for bit under torch.use_deterministic_algorithms(True), and two
    replays draw different DropPath samples."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import albef_vit_check as AV  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def rel(a, b):
    a, b = kept(a, b.to(a.device))
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _encoder(cfg, **top):
    from mmf_b200.encoders import build_encoder
    return build_encoder({"type": "albef_vit_encoder", "params": dict(top, params=dict(cfg))}).to(DEV)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "albef_vit.pt"), weights_only=False)


@pytest.mark.parametrize("case", ["small", "default"])
def test_forward_backward_vs_reference_golden(golden, case):
    g = golden[case]
    enc = _encoder(g["config"]).eval()
    enc.vit.load_state_dict(g["state_dict"])
    images = g["images"].to(DEV).requires_grad_(True)
    out = enc(images)
    assert rel(out, g["out"]) < 2e-2
    (out * g["w_rand"].to(DEV)).sum().backward()
    assert rel(images.grad, g["grads"]["images"]) < 3e-2
    for n, p in enc.vit.named_parameters():
        assert rel(p.grad, g["grads"][n]) < 8e-2, n


TRAIN_CFG = dict(embed_dim=256, num_heads=4, depth=3, drop_rate=0.1, attn_drop_rate=0.1, drop_path_rate=0.4)


def _close(what, got, ref64, ref16):
    got, ref64, ref16 = got.detach().double(), ref64.detach().double(), ref16.detach().double()
    err, drift = (got - ref64).abs(), (ref16 - ref64).abs()
    # the scales are per row (last dimension): LayerNorm backward, attention and the GEMMs mix a row's errors, and one row
    # (the [CLS] position of pos_embed's gradient) can be 100x larger than the others.  The bf16 restatement's error is
    # taken at the element and as its row's rms (a single element's drift can be zero by chance)
    def row_rms(t):
        return t.square().mean(-1, keepdim=True).sqrt() if t.dim() > 1 else t.square().mean().sqrt()
    bound = 6.0 * torch.maximum(drift, row_rms(drift)) + 8 * 2.0 ** -8 * ref64.abs() + 3e-2 * row_rms(ref64)
    bad = err > bound
    i = int((err / bound).argmax())
    assert not bad.any(), "%s: %d element(s) off; worst at flat index %d: %g vs fp64 %g (bound %g)" % (
        what, int(bad.sum()), i, got.reshape(-1)[i].item(), ref64.reshape(-1)[i].item(), bound.reshape(-1)[i].item())


def test_training_step_vs_fp64_with_the_kernels_keep_bits(monkeypatch):
    torch.manual_seed(21)
    enc = _encoder(TRAIN_CFG).train()
    draws = AV.Draws().install(monkeypatch)
    pos = {}
    enc.vit.pos_drop.register_forward_hook(lambda m, i, o: pos.update(x=i[0].detach(), y=o.detach()))
    B, S = 8, 197
    images = torch.randn(B, 3, 224, 224, device=DEV).requires_grad_(True)
    out = enc(images)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    torch.cuda.synchronize()
    keeps = draws.blocks(TRAIN_CFG, B, S)
    assert any(not blk[s][0].view(B, -1).any(1).all() for blk in keeps for s in ("proj", "fc2"))   # a sample dropped
    pos_keep = ((pos["y"] != 0) | (pos["x"] == 0), 1.0 / (1.0 - TRAIN_CFG["drop_rate"]))
    res = {}
    for dt in (torch.float64, torch.bfloat16):
        sd = {k: v.detach().to(torch.bfloat16).to(dt).requires_grad_(True) for k, v in enc.vit.state_dict().items()}
        x = images.detach().to(torch.bfloat16).to(dt).requires_grad_(True)
        ref = AV.vit_ref(x, sd, TRAIN_CFG, keeps, pos_keep, dtype=dt)
        (ref * w.to(dt)).sum().backward()
        res[dt] = (ref, x.grad, {k: v.grad for k, v in sd.items()})
    (r64, dx64, g64), (r16, dx16, g16) = res[torch.float64], res[torch.bfloat16]
    _close("output", out, r64, r16)
    _close("d images", images.grad, dx64, dx16)
    for n, p in enc.vit.named_parameters():
        if n.endswith("attn.qkv.bias"):
            continue            # its key third is analytically zero; covered by the whole-tensor check below
        _close(n, p.grad, g64[n], g16[n])
    assert rel(out, r64) <= 1.5 * rel(r16, r64) + 2e-3
    assert rel(images.grad, dx64) <= 1.5 * rel(dx16, dx64) + 2e-3
    for n, p in enc.vit.named_parameters():
        assert rel(p.grad, g64[n]) <= 1.5 * rel(g16[n], g64[n]) + 2e-3 or g64[n].norm() < 1e-6, n


def test_dropped_samples_pass_their_residual_bit_for_bit(monkeypatch):
    """a sample whose DropPath draw drops a branch: h = x (attention branch) or out = h (MLP branch) exactly"""
    from mmf_b200 import albef_vit as AVT
    from mmf_b200 import engine as E
    seen = []
    orig = E.vit_layer_fwd

    def spy(x, add_mask, w, B, S, p_attn, p_hidden, p_mlp, p_path, ds, probs=None):
        out, saved = orig(x, add_mask, w, B, S, p_attn, p_hidden, p_mlp, p_path, ds, probs)
        seen.append((x, saved[7], out, saved[5], saved[13]))      # x, h, out, attention-branch bits, MLP-branch bits
        return out, saved
    monkeypatch.setattr(AVT.AlbefBlockW, "fwd", staticmethod(spy))
    torch.manual_seed(22)
    cfg = dict(TRAIN_CFG, drop_path_rate=0.8)
    enc = _encoder(cfg).train()
    B, S = 16, 197
    enc(torch.randn(B, 3, 224, 224, device=DEV))
    torch.cuda.synchronize()
    n_dropped = 0
    for x, h, out, b1, b2 in seen:
        if b1 is None:
            continue                                              # block 0: rate 0
        for before, after, bits in ((x, h, b1), (h, out, b2)):
            dropped = bits.view(B, -1).eq(0).all(1)
            n_dropped += int(dropped.sum())
            assert torch.equal(after.view(B, S, -1)[dropped], before.view(B, S, -1)[dropped])
            assert not torch.equal(after.view(B, S, -1)[~dropped], before.view(B, S, -1)[~dropped])
    assert n_dropped > 0


def test_graphed_step_equals_eager_and_replays_draw_fresh_samples(monkeypatch):
    from mmf_b200 import functional as F
    from mmf_b200 import modules
    from mmf_b200.graphs import GraphedStep
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        torch.manual_seed(23)
        enc = _encoder(TRAIN_CFG).train()
        enc.vit.pos_drop.p = 0.0            # torch's own dropout draws from torch's generator, not from the kernels' stream
        B = 4
        batch = {"images": torch.randn(B, 3, 224, 224, device=DEV), "w": torch.randn(B, 197, 256, device=DEV)}

        def loss_fn(b):
            return (enc(b["images"]) * b["w"]).sum()
        step = GraphedStep(enc, loss_fn, batch)
        seed_counter = modules._SEED_COUNTER[0]           # the captured forward drew from this seed
        epoch = F.dropout_epoch(DEV)
        losses, grads, epochs = [], [], []
        for _ in range(2):
            losses.append(step().detach().clone())
            torch.cuda.synchronize()
            grads.append({n: p.grad.detach().clone() for n, p in enc.named_parameters()})
            epochs.append(int(epoch.item()))
        assert not torch.equal(losses[0], losses[1])
        draws = AV.Draws().install(monkeypatch)
        for k in range(2):
            # the eager step with the captured seed and the epoch of replay k
            modules._SEED_COUNTER[0] = seed_counter - 1
            epoch.fill_(epochs[k])
            enc.zero_grad(set_to_none=True)
            loss = loss_fn(batch)
            loss.backward()
            torch.cuda.synchronize()
            assert torch.equal(loss.detach(), losses[k])
            for n, p in enc.named_parameters():
                assert torch.equal(p.grad, grads[k][n]), n
        paths = [d[5] for d in draws if d[0] == "path"]
        half = len(paths) // 2
        samples = [torch.stack([w.view(B, -1).ne(0).any(1) for w in paths[i * half:(i + 1) * half]]) for i in range(2)]
        assert not torch.equal(samples[0], samples[1])      # the two replays dropped different samples
    finally:
        torch.use_deterministic_algorithms(prev)
