"""A torch restatement of ALBEF's VisionTransformer (mmf/models/albef/vit.py:473-599) for the ALBEF ViT tests (a plain
module, imported by test_albef_vit_cpu.py and test_albef_vit_gpu.py).

`vit_ref` runs the reference's arithmetic in any dtype (fp64: the truth; bf16: the drift the product is allowed) on a
state dict of the reference's key names, with the keep masks of every dropout site given explicitly, so that a training
step can be replayed with the kernels' own draws.  `Draws` records those draws from engine.DropoutState and decodes them
into the masks `vit_ref` takes (layouts of include/mmfb200.h: element j of a row is bit j % 32 of word j // 32)."""
import math

import torch
import torch.nn.functional as TF


def unpack_bits(words, n):
    w = words.to(torch.int64) & 0xFFFFFFFF
    j = torch.arange(n, device=words.device)
    return ((w[..., j // 32] >> (j % 32)) & 1).bool()


class Draws(list):
    """every keep-bit draw of a forward, in order: (kind, rows, ncols, p, p_path, words)"""

    def install(self, monkeypatch):
        from mmf_b200 import engine as E
        bits, path_bits = E.DropoutState.bits, E.DropoutState.path_bits

        def spy_bits(ds, rows_shape, ncols, p, device):
            out = bits(ds, rows_shape, ncols, p, device)
            self.append(("bits", tuple(int(r) for r in rows_shape), int(ncols), float(p), 0.0, out.clone()))
            return out

        def spy_path(ds, batch, rows_per_sample, ncols, p, p_path, device):
            out = path_bits(ds, batch, rows_per_sample, ncols, p, p_path, device)
            self.append(("path", (int(batch), int(rows_per_sample)), int(ncols), float(p), float(p_path), out.clone()))
            return out
        monkeypatch.setattr(E.DropoutState, "bits", spy_bits)
        monkeypatch.setattr(E.DropoutState, "path_bits", spy_path)
        return self

    def blocks(self, cfg, B, S):
        """per block: dict site -> (bool keep mask in the reference's shape, scale) for the sites that drew, in the
        engine's order: attention probabilities, attn.proj (+ DropPath), mlp.drop after the GELU, mlp.fc2 (+ DropPath)"""
        H, heads = cfg["embed_dim"], cfg["num_heads"]
        inter = int(H * cfg.get("mlp_ratio", 4.0))
        p_drop, p_attn = cfg.get("drop_rate", 0.0), cfg.get("attn_drop_rate", 0.0)
        dpr = [x.item() for x in torch.linspace(0, cfg.get("drop_path_rate", 0.0), cfg["depth"])]
        it = iter(self)
        out = []
        for i in range(cfg["depth"]):
            blk = {}
            if p_attn > 0:
                kind, rows, n, p, _, w = next(it)
                assert (kind, rows, n, p) == ("bits", (B, heads, S), S, p_attn)
                blk["attn"] = (unpack_bits(w, S), 1.0 / (1.0 - p))
            for site, ncols, pp in (("proj", H, p_drop), ("mlp", inter, p_drop), ("fc2", H, p_drop)):
                if site == "mlp":
                    if pp > 0:
                        kind, rows, n, p, _, w = next(it)
                        assert (kind, rows, n, p) == ("bits", (B * S,), inter, pp)
                        blk[site] = (unpack_bits(w, n).view(B, S, n), 1.0 / (1.0 - p))
                    continue
                if dpr[i] > 0:
                    kind, rows, n, p, ppath, w = next(it)
                    assert (kind, rows, n, p) == ("path", (B, S), ncols, pp) and abs(ppath - dpr[i]) < 1e-12
                    blk[site] = (unpack_bits(w, n).view(B, S, n), 1.0 / ((1.0 - p) * (1.0 - ppath)))
                elif pp > 0:
                    kind, rows, n, p, _, w = next(it)
                    assert (kind, rows, n, p) == ("bits", (B * S,), ncols, pp)
                    blk[site] = (unpack_bits(w, n).view(B, S, n), 1.0 / (1.0 - p))
            out.append(blk)
        assert next(it, None) is None, "more draws than sites"
        return out


def _drop(t, site):
    if site is None:
        return t
    keep, scale = site
    return torch.where(keep.to(t.device), t * scale, torch.zeros_like(t))


def vit_ref(images, sd, cfg, keeps=None, pos=None, dtype=torch.float64):
    """VisionTransformer.forward in `dtype`.  sd: the reference's parameter names (no `vit.` prefix), tensors that may
    require grad; keeps: per block the dict of Draws.blocks, or None (eval); pos: (keep, scale) of pos_drop, or None."""
    p = {k: v.to(dtype) for k, v in sd.items()}
    patch = cfg.get("patch_size", 16)
    H, heads = cfg["embed_dim"], cfg["num_heads"]
    x = TF.conv2d(images.to(dtype), p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], stride=patch)
    x = x.flatten(2).transpose(1, 2)
    B = x.shape[0]
    x = torch.cat((p["cls_token"].expand(B, -1, -1), x), dim=1)
    x = _drop(x + p["pos_embed"][:, :x.shape[1]], pos)
    S, d = x.shape[1], H // heads
    for i in range(cfg["depth"]):
        k = keeps[i] if keeps is not None else {}
        pre = "blocks.%d." % i
        a = TF.layer_norm(x, (H,), p[pre + "norm1.weight"], p[pre + "norm1.bias"], 1e-6)
        qkv = TF.linear(a, p[pre + "attn.qkv.weight"], p.get(pre + "attn.qkv.bias"))
        q, kk, v = qkv.reshape(B, S, 3, heads, d).permute(2, 0, 3, 1, 4)
        att = torch.softmax(q @ kk.transpose(-2, -1) / math.sqrt(d), dim=-1)
        att = _drop(att, k.get("attn"))
        ctx = (att @ v).transpose(1, 2).reshape(B, S, H)
        x = x + _drop(TF.linear(ctx, p[pre + "attn.proj.weight"], p[pre + "attn.proj.bias"]), k.get("proj"))
        b = TF.layer_norm(x, (H,), p[pre + "norm2.weight"], p[pre + "norm2.bias"], 1e-6)
        g = _drop(TF.gelu(TF.linear(b, p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"])), k.get("mlp"))
        x = x + _drop(TF.linear(g, p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"]), k.get("fc2"))
    return TF.layer_norm(x, (H,), p["norm.weight"], p["norm.bias"], 1e-6)
