"""ALBEF's vision transformer on the fused pre-LN trunk.

  B200AlbefVisionTransformer  <->  VisionTransformer   mmf/models/albef/vit.py:473-599 (timm-style ViT)
  B200AlbefBlock              <->  Block               mmf/models/albef/vit.py:430-470

Parameter names are the reference's (`patch_embed.proj`, `cls_token`, `pos_embed`, `blocks.{i}.{norm1, attn.qkv, attn.proj,
norm2, mlp.fc1, mlp.fc2}`, `norm`), so ALBEF checkpoints load unchanged.  A block is engine.vit_layer_fwd / _bwd with the
fused qkv projection, LayerNorm eps 1e-6, dropout after the GELU (`mlp.drop`) and stochastic depth (`drop_path`) in the
kernels' keep bits.  The blocks' children are parameter holders: their own forward is never called.
"""
import torch
from torch import nn

from . import engine as E
from . import ops
from .modules import EncoderRunner, _Holder, _require_cuda, run_bert_encoder

# VisionTransformer's config keys and defaults (mmf/models/albef/vit.py:503-516)
ALBEF_VIT_DEFAULTS = dict(img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12, num_heads=12,
                          mlp_ratio=4.0, qkv_bias=True, qk_scale=None, representation_size=None, drop_rate=0.0,
                          attn_drop_rate=0.0, drop_path_rate=0.0, norm_layer=None)
LN_EPS = 1e-6


def _get(cfg, key, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    getter = getattr(cfg, "get", None)
    return getter(key, default) if callable(getter) else getattr(cfg, key, default)


def _pair(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x)


class _Attention(_Holder):
    def __init__(self, dim, num_heads, qkv_bias, attn_drop, proj_drop):
        super().__init__()
        if dim % num_heads:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)" % (dim, num_heads))
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)


class _Mlp(_Holder):
    def __init__(self, dim, hidden, drop):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)
        self.drop = nn.Dropout(drop)


class _DropPath(_Holder):
    """DropPath's rate (stochastic depth per sample); applied by the kernels through the residual branches' keep bits"""

    def __init__(self, drop_prob):
        super().__init__()
        self.drop_prob = drop_prob


class B200AlbefBlock(_Holder):
    def __init__(self, dim, num_heads, mlp_ratio, qkv_bias, drop, attn_drop, drop_path):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=LN_EPS)
        self.attn = _Attention(dim, num_heads, qkv_bias, attn_drop, drop)
        self.drop_path = _DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm2 = nn.LayerNorm(dim, eps=LN_EPS)
        self.mlp = _Mlp(dim, int(dim * mlp_ratio), drop)


class AlbefBlockW(E.ViTLayerW):
    """Handles of one B200AlbefBlock for vit_layer_fwd / _bwd.  Without a qkv bias (qkv_bias=False) the projection adds no
    bias and its column sums land in a scratch buffer that nothing reads."""

    @staticmethod
    def params(m):
        a = m.attn
        out = [a.qkv.weight] + ([a.qkv.bias] if a.qkv.bias is not None else [])
        return out + [a.proj.weight, a.proj.bias, m.norm1.weight, m.norm1.bias, m.norm2.weight, m.norm2.bias,
                      m.mlp.fc1.weight, m.mlp.fc1.bias, m.mlp.fc2.weight, m.mlp.fc2.bias]

    @staticmethod
    def dropout_p(m):
        """(p_attn, p_hidden, p_mlp, p_path) of vit_layer_fwd, read at every forward"""
        return (float(m.attn.attn_drop.p), float(m.attn.proj_drop.p), float(m.mlp.drop.p),
                float(getattr(m.drop_path, "drop_prob", 0.0)))

    def __init__(self, pack, m):
        p = self.params(m)
        self.wqkv = pack.handle(p[0])
        if m.attn.qkv.bias is not None:
            self.bqkv = pack.handle(p[1])
            p = p[2:]
        else:
            self.bqkv = E.Handle(None, torch.zeros(p[0].shape[0], dtype=torch.float32, device=pack.device))
            p = p[1:]
        (self.wo, self.bo, self.g1, self.be1, self.g2, self.be2, self.w1, self.b1, self.w2, self.b2) = (
            pack.handle(q) for q in p)
        self.heads = m.attn.num_heads
        self.hidden = p[0].shape[1]
        self.eps1, self.eps2 = float(m.norm1.eps), float(m.norm2.eps)


class AlbefVitRunner(EncoderRunner):
    W = AlbefBlockW


class _PatchEmbed(nn.Module):
    """PatchEmbed (vit.py:334-368): Conv2d(kernel = stride = patch) run as one GEMM over the unfolded patches"""

    def __init__(self, img_size, patch_size, in_chans, embed_dim):
        super().__init__()
        self.img_size, self.patch_size = _pair(img_size), _pair(patch_size)
        self.grid_size = (self.img_size[0] // self.patch_size[0], self.img_size[1] // self.patch_size[1])
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=self.patch_size, stride=self.patch_size)

    def forward(self, x):
        B, C, Hh, Ww = x.shape
        assert Hh == self.img_size[0] and Ww == self.img_size[1], (
            f"Input image size ({Hh}*{Ww}) doesn't match model ({self.img_size[0]}*{self.img_size[1]}).")
        ph, pw = self.patch_size
        # [B * n_patches, C * ph * pw] rows in the conv weight's (C, kh, kw) order; patches row-major over the grid
        rows = x.reshape(B, C, Hh // ph, ph, Ww // pw, pw).permute(0, 2, 4, 1, 3, 5).reshape(
            B * self.num_patches, C * ph * pw)
        w = self.proj.weight.reshape(self.proj.weight.shape[0], -1)
        return ops.linear_any(rows, w, self.proj.bias).view(B, self.num_patches, w.shape[0])


class B200AlbefVisionTransformer(nn.Module):
    """VisionTransformer (vit.py:473-599) from its config (a dict or any object with get()).  Refused, with
    NotImplementedError: `qk_scale` other than None (the attention kernels scale the scores by 1/sqrt(head_dim)),
    `norm_layer` (every LayerNorm is the eps-1e-6 one the kernels run), and register_blk >= 0 in forward (Grad-CAM's
    attention maps and their gradients: no gradient flows through the attention probabilities, DESIGN.md 7)."""

    def __init__(self, config):
        super().__init__()
        c = {k: _get(config, k, d) for k, d in ALBEF_VIT_DEFAULTS.items()}
        if c["qk_scale"] is not None:
            raise NotImplementedError("qk_scale=%r: the B200 attention kernels scale the scores by 1/sqrt(head_dim) only"
                                      % (c["qk_scale"],))
        if c["norm_layer"] is not None:
            raise NotImplementedError("norm_layer=%r: the B200 ViT runs LayerNorm(eps=1e-6) only" % (c["norm_layer"],))
        for k, v in c.items():
            setattr(self, k, v)
        self.num_features = self.embed_dim
        self.patch_embed = _PatchEmbed(self.img_size, self.patch_size, self.in_chans, self.embed_dim)
        num_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, self.embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, self.embed_dim))
        self.pos_drop = nn.Dropout(p=float(self.drop_rate))
        dpr = [x.item() for x in torch.linspace(0, float(self.drop_path_rate), int(self.depth))]   # stochastic depth decay
        self.blocks = nn.ModuleList([
            B200AlbefBlock(self.embed_dim, self.num_heads, self.mlp_ratio, self.qkv_bias, float(self.drop_rate),
                           float(self.attn_drop_rate), dpr[i])
            for i in range(int(self.depth))])
        self.norm = nn.LayerNorm(self.embed_dim, eps=LN_EPS)
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        nn.init.trunc_normal_(self.cls_token, std=0.02)
        self.apply(self._init_weights)
        self._runner = AlbefVitRunner(self.blocks)

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def no_weight_decay(self):
        return {"pos_embed", "cls_token"}

    def forward(self, images, register_blk=-1):
        if register_blk >= 0:
            raise NotImplementedError("register_blk=%d saves attention maps and their gradients (Grad-CAM): gradients "
                                      "through the attention probabilities are not computed on the B200 path" % register_blk)
        _require_cuda(images, "images")
        B = images.shape[0]
        x = self.patch_embed(images).to(self.pos_embed.dtype)
        x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
        x = self.pos_drop(x + self.pos_embed[:, :x.size(1), :])
        x = run_bert_encoder(self._runner, x, None, self.training)[0]
        shape = x.shape
        return ops.layer_norm(x.reshape(-1, shape[-1]), self.norm.weight, self.norm.bias, self.norm.eps).view(shape).to(
            self.norm.weight.dtype)
