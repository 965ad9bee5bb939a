#!/usr/bin/env python
"""TEST INFRASTRUCTURE - writes tests/golden/albef_vit.pt by running the REFERENCE's ALBEF vision transformer.

Needs the reference tree (MMF_REFERENCE_ROOT, see oracle/ref_loader.py):   python tools/make_golden_albef_vit.py
It needs a full checkout: mmf/models/albef/vit.py is not among the files oracle/build_ref.py stages.

Runs `VisionTransformer` (mmf/models/albef/vit.py:473-599), the reference's own file loaded unmodified by
oracle/ref_loader.py, in fp32, eval mode (dropout and stochastic depth off), on seeded weights on the int8 grid of
oracle/make_golden.py.  It writes that one fixture and nothing else.  Cases:
  small    - 32 px images, patch 8 (16 patches + [CLS] = 17 positions), embed 128 / 2 heads / depth 2, mlp_ratio 1,
             qkv_bias False, B = 3
  default  - the default geometry, 224 px / patch 16 (197 positions), embed 128 / 2 heads / depth 1, qkv_bias True, B = 1
(head size 64, as the attention kernels take; the random projection w_rand is stored on the int8 grid too)
Each: config, state dict, images, output, and the gradients of (out * w_rand).sum() wrt the images and every parameter.
Plus the reference's defaults: the VisionTransformer's attributes for an empty config, its stochastic-depth rates for
drop_path_rate 0.1, and the default model's state-dict keys and shapes.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden as MG  # noqa: E402
from oracle import ref_loader as R  # noqa: E402

CASES = {
    "small": (dict(img_size=32, patch_size=8, embed_dim=128, num_heads=2, depth=2, mlp_ratio=1.0, qkv_bias=False), 3, 11),
    "default": (dict(embed_dim=128, num_heads=2, depth=1), 1, 12),
}
DEFAULT_ATTRS = ["img_size", "patch_size", "in_chans", "num_classes", "embed_dim", "depth", "num_heads", "mlp_ratio",
                 "qkv_bias", "qk_scale", "representation_size", "drop_rate", "attn_drop_rate", "drop_path_rate", "norm_layer"]


def _vit():
    return R.load("mmf/models/albef/vit.py", "mmf.models.albef.vit")


def _seed_weights(model, seed):
    """normal 0.02 weights and biases, LayerNorm weights around 1: every value on the int8 grid of make_golden._q8"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            ln_weight = p.dim() == 1 and (".norm" in n or n.startswith("norm")) and n.endswith("weight")
            base = 1.0 if ln_weight else 0.0
            p.copy_(MG._q8(base + torch.randn(p.shape, generator=g) * 0.02, base))


def _case(cfg, B, seed):
    V = _vit()
    torch.manual_seed(seed)
    model = V.VisionTransformer(dict(cfg)).eval()
    _seed_weights(model, seed)
    g = torch.Generator().manual_seed(seed + 100)
    img = cfg.get("img_size", 224)
    images = MG._q8(torch.randn(B, cfg.get("in_chans", 3), img, img, generator=g) * 0.05, 0.0).requires_grad_(True)
    out = model(images)
    w_rand = MG._q8(torch.randn(out.shape, generator=g) * 0.05, 0.0)
    (out * w_rand).sum().backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()}
    grads["images"] = images.grad.detach().clone()
    return dict(config=dict(cfg), state_dict={k: v.detach().clone() for k, v in model.state_dict().items()},
                images=images.detach().clone(), out=out.detach().clone(), w_rand=w_rand, grads=grads)


def _defaults():
    V = _vit()
    torch.manual_seed(0)
    model = V.VisionTransformer({})
    attrs = {k: getattr(model, k) for k in DEFAULT_ATTRS}
    rates = V.VisionTransformer(dict(embed_dim=64, num_heads=2, drop_path_rate=0.1))
    dpr = [float(getattr(b.drop_path, "drop_prob", 0.0)) for b in rates.blocks]
    return dict(attrs=attrs, no_weight_decay=sorted(model.no_weight_decay()), drop_path_rates=dpr,
                eps=[float(model.norm.eps)] + [float(m.eps) for b in model.blocks for m in (b.norm1, b.norm2)],
                state_dict_shapes={k: tuple(v.shape) for k, v in model.state_dict().items()})


def main():
    obj = {name: _case(*spec) for name, spec in CASES.items()}
    obj["defaults"] = _defaults()
    MG._save("albef_vit", obj)


if __name__ == "__main__":
    main()
