"""The registered `albef_vit_encoder` (mmf_b200.encoders.B200AlbefVitEncoder) on the CPU: registry and config defaults,
state-dict keys and shapes, the refusals, `pretrained` loading, and the encoder run over the kernel test double
(tests/fake_kernels.py, extended below with the stochastic-depth keep bits and the hidden-dropout epilogues) against
tests/golden/albef_vit.pt - outputs and gradients of the REFERENCE's own VisionTransformer (tools/make_golden_albef_vit.py).
The kernels themselves are covered on the GPU (tests/test_albef_vit_gpu.py, tests/test_albef_vit_kernels_gpu.py)."""
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import albef_vit_check as AV  # noqa: E402
import fake_kernels as FK  # noqa: E402
from oracle.golden_format import kept  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel(a, b):
    a, b = kept(a, b)
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLD, "albef_vit.pt"), weights_only=False)


def _double():
    """tests/fake_kernels.py plus the contracts of the entry points this encoder adds (include/mmfb200.h)"""
    from mmf_b200 import lib
    d = types.SimpleNamespace(**{k: getattr(FK, k) for k in dir(FK) if not k.startswith("__")})

    def gemm(a, b, *, epi=lib.EPI_BIAS, bias=None, aux=None, drop_mask=None, drop_scale=1.0, **kw):
        if epi not in (lib.EPI_BIAS_GELU_DROP, lib.EPI_GELU_DROP_BWD):
            return FK.gemm(a, b, epi=epi, bias=bias, aux=aux, drop_mask=drop_mask, drop_scale=drop_scale, **kw)
        assert drop_mask is not None
        acc = FK.gemm(a, b, epi=lib.EPI_ATOMIC_F32, a_mn=kw.get("a_mn", False), b_mn=kw.get("b_mn", False))
        keep = FK.unpack_keep_bits(drop_mask, acc.shape[1])
        if epi == lib.EPI_BIAS_GELU_DROP:
            acc = acc + bias.float()
            h = torch.where(keep, FK._gelu(acc) * drop_scale, torch.zeros_like(acc))
            return acc.to(FK.BF), h.to(FK.BF)
        return torch.where(keep, acc * drop_scale * FK._gelu_grad(aux.float()), torch.zeros_like(acc)).to(FK.BF)

    def dropout_path_bits(batch, rows_per_sample, ncols, p, p_path, seed, offset, device):
        keep = FK.unpack_keep_bits(FK.dropout_bits((batch * rows_per_sample,), ncols, p, seed, offset, device), ncols)
        g = torch.Generator().manual_seed((int(seed) * 7919 + int(offset)) % (2 ** 63))
        sample = (torch.rand(batch, generator=g) >= p_path).repeat_interleave(rows_per_sample)
        return FK.pack_keep_bits(keep & sample[:, None])

    d.gemm, d.dropout_path_bits = gemm, dropout_path_bits
    return d


@pytest.fixture()
def cpu(monkeypatch):
    import mmf_b200.albef_vit as AVT
    import mmf_b200.engine as E
    import mmf_b200.modules as M
    import mmf_b200.ops as OPS
    double = _double()
    monkeypatch.setattr(E, "F", double)
    monkeypatch.setattr(OPS, "F", double)
    for mod in (M, AVT):
        monkeypatch.setattr(mod, "_require_cuda", lambda t, what: None)
    return double


def _encoder(cfg, **top):
    from mmf_b200.encoders import build_encoder
    return build_encoder({"type": "albef_vit_encoder", "params": dict(top, params=dict(cfg))})


def test_registry_and_defaults(golden):
    from mmf_b200.encoders import ALBEF_VIT_ENCODER_DEFAULTS, B200AlbefVitEncoder
    from mmf_b200.registry import registry
    assert registry.get_encoder_class("albef_vit_encoder") is B200AlbefVitEncoder
    assert ALBEF_VIT_ENCODER_DEFAULTS == dict(name="albef_vit_encoder", pretrained=False, out_dim=768)
    d = golden["defaults"]
    enc = _encoder({})                                          # every VisionTransformer default: ViT-B/16 at 224 px
    assert {k: getattr(enc.vit, k) for k in d["attrs"]} == d["attrs"]
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == {"vit." + k: s for k, s in
                                                                        d["state_dict_shapes"].items()}
    assert sorted(enc.vit.no_weight_decay()) == d["no_weight_decay"]
    assert [enc.vit.norm.eps] + [m.eps for b in enc.vit.blocks for m in (b.norm1, b.norm2)] == d["eps"]
    rates = _encoder(dict(embed_dim=64, num_heads=2, drop_path_rate=0.1))
    assert [float(getattr(b.drop_path, "drop_prob", 0.0)) for b in rates.vit.blocks] == d["drop_path_rates"]
    assert [rates.vit._runner.W.dropout_p(b)[3] for b in rates.vit.blocks] == d["drop_path_rates"]
    # a structured config (attribute access with get()) reads the same keys
    from mmf_b200.models import ConfigNode
    enc2 = _encoder(ConfigNode(dict(embed_dim=64, num_heads=2, depth=3, mlp_ratio=2.0, drop_rate=0.2)))
    assert (enc2.vit.depth, enc2.vit.blocks[0].mlp.fc1.out_features, enc2.vit.blocks[1].mlp.drop.p) == (3, 128, 0.2)


@pytest.mark.parametrize("case", ["small", "default"])
def test_state_dict_matches_reference(golden, case):
    g = golden[case]
    enc = _encoder(g["config"])
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == {"vit." + k: tuple(v.shape)
                                                                        for k, v in g["state_dict"].items()}
    enc.vit.load_state_dict(g["state_dict"])                    # ALBEF checkpoints load into .vit unchanged


def test_refusals():
    with pytest.raises(NotImplementedError, match="qk_scale"):
        _encoder(dict(embed_dim=64, num_heads=2, depth=1, qk_scale=0.125))
    with pytest.raises(NotImplementedError, match="norm_layer"):
        _encoder(dict(embed_dim=64, num_heads=2, depth=1, norm_layer="LayerNorm"))
    enc = _encoder(dict(img_size=32, patch_size=8, embed_dim=64, num_heads=2, depth=2))
    with pytest.raises(NotImplementedError, match="register_blk"):
        enc.vit(torch.zeros(1, 3, 32, 32), register_blk=1)


def test_image_size_is_asserted(cpu):
    enc = _encoder(dict(img_size=32, patch_size=8, embed_dim=64, num_heads=2, depth=1))
    with pytest.raises(AssertionError, match="doesn't match model"):
        enc(torch.zeros(1, 3, 48, 48))


def test_pretrained_loads_state_dict(golden, tmp_path):
    g = golden["small"]
    path = tmp_path / "vit.pth"
    torch.save(g["state_dict"], path)
    enc = _encoder(g["config"], pretrained=True, pretrained_path=str(path))
    assert not enc.vit.training
    for k, v in g["state_dict"].items():
        assert torch.equal(enc.vit.state_dict()[k], v), k


@pytest.mark.parametrize("case", ["small", "default"])
def test_encoder_vs_reference_golden(cpu, golden, case):
    """eval forward and backward over the double (bf16 operands, fp32 accumulation) against the reference in fp32"""
    g = golden[case]
    enc = _encoder(g["config"]).eval()
    enc.vit.load_state_dict(g["state_dict"])
    images = g["images"].clone().requires_grad_(True)
    out = enc(images)
    assert out.shape == g["out"].shape and out.dtype == torch.float32
    assert rel(out, g["out"]) < 2e-2
    (out * g["w_rand"]).sum().backward()
    assert rel(images.grad, g["grads"]["images"]) < 3e-2
    for n, p in enc.vit.named_parameters():
        assert rel(p.grad, g["grads"][n]) < 8e-2, n


def test_train_step_replays_with_the_drawn_masks(cpu, monkeypatch):
    """drop_rate, attn_drop_rate and drop_path_rate > 0: the draws (attention, proj + DropPath, after-GELU, fc2 +
    DropPath per block) fed to the fp64 restatement give the double's output and gradients"""
    cfg = dict(img_size=32, patch_size=8, embed_dim=64, num_heads=2, depth=3, drop_rate=0.2, attn_drop_rate=0.1,
               drop_path_rate=0.5)
    torch.manual_seed(5)
    enc = _encoder(cfg).train()
    draws = AV.Draws().install(monkeypatch)
    pos = {}
    enc.vit.pos_drop.register_forward_hook(lambda m, i, o: pos.update(x=i[0].detach(), y=o.detach()))
    images = torch.randn(4, 3, 32, 32).requires_grad_(True)
    out = enc(images)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    B, S = 4, 17
    keeps = draws.blocks(cfg, B, S)
    assert any(not blk["fc2"][0].view(B, -1).any(1).all() for blk in keeps)      # some sample dropped a branch
    sd = {k: v.detach().to(torch.bfloat16).double().requires_grad_(True) for k, v in enc.vit.state_dict().items()}
    x64 = images.detach().double().requires_grad_(True)
    pos_keep = ((pos["y"] != 0) | (pos["x"] == 0), 1.0 / (1.0 - cfg["drop_rate"]))
    ref = AV.vit_ref(x64, sd, cfg, keeps, pos_keep)
    (ref * w.double()).sum().backward()
    assert rel(out, ref) < 2e-2
    assert rel(images.grad, x64.grad) < 3e-2
    for n, p in enc.vit.named_parameters():
        assert rel(p.grad, sd[n].grad) < 8e-2, n
