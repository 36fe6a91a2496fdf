"""Host-side mirror of the reference ViT constructors, backed by the sm_90a engine.

Drop-in for ``classification/vision_transformer/vit_model.py`` of KKKSQJ/DeepLearning (VisionTransformer ``:164``,
Block ``:136``, Attention ``:71``, Mlp ``:114``, PatchEmbed ``:43``, ``vit_base_patch16_224_in21k`` ``:290`` ...): same
constructor signatures, attribute / state_dict names, shapes and initialisation RNG order (``trunc_normal_`` on pos/cls,
then ``apply(_init_vit_weights)``), so reference checkpoints load unchanged and ``torch.manual_seed(s)`` gives bit-identical
initial weights.  The sub-modules only hold parameters: ``VisionTransformer.forward`` runs the whole network through
``deeplearning_b200.engine.vit`` (fused patch-embed GEMM, LayerNorm, wgmma attention, GEMMs with bias/GELU/residual
epilogues) as one autograd Function.  No CPU path.
"""
from collections import OrderedDict
from functools import partial

import torch
import torch.nn as nn


class _EngineOnly(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter container; it runs inside VisionTransformer.forward")


class DropPath(nn.Module):
    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob


class PatchEmbed(_EngineOnly):
    def __init__(self, img_size=224, patch_size=16, in_c=3, embed_dim=768, norm_layer=None):
        super().__init__()
        self.img_size = (img_size, img_size)
        self.patch_size = (patch_size, patch_size)
        self.grid_size = (img_size // patch_size, img_size // patch_size)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_c, embed_dim, kernel_size=self.patch_size, stride=self.patch_size)
        self.norm = norm_layer(embed_dim) if norm_layer else nn.Identity()


class Attention(_EngineOnly):
    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop_ratio=0., proj_drop_ratio=0.):
        super().__init__()
        self.num_heads = num_heads
        self.scale = qk_scale or (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop_ratio)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop_ratio)


class Mlp(_EngineOnly):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features or in_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features)
        self.drop = nn.Dropout(drop)


class Block(_EngineOnly):
    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop_ratio=0., attn_drop_ratio=0.,
                 drop_path_ratio=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads, qkv_bias, qk_scale, attn_drop_ratio, drop_ratio)
        self.drop_path = DropPath(drop_path_ratio) if drop_path_ratio > 0. else nn.Identity()
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), act_layer=act_layer, drop=drop_ratio)


def _init_vit_weights(m):
    if isinstance(m, nn.Linear):
        nn.init.trunc_normal_(m.weight, std=.01)
        if m.bias is not None:
            nn.init.zeros_(m.bias)
    elif isinstance(m, nn.Conv2d):
        nn.init.kaiming_normal_(m.weight, mode="fan_out")
        if m.bias is not None:
            nn.init.zeros_(m.bias)
    elif isinstance(m, nn.LayerNorm):
        nn.init.zeros_(m.bias)
        nn.init.ones_(m.weight)


class VisionTransformer(nn.Module):
    def __init__(self, img_size=224, patch_size=16, in_c=3, num_classes=1000, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4.0, qkv_bias=True, qk_scale=None, representation_size=None, distilled=False, drop_ratio=0.,
                 attn_drop_ratio=0., drop_path_ratio=0., embed_layer=PatchEmbed, norm_layer=None, act_layer=None):
        super().__init__()
        self.num_classes = num_classes
        self.num_features = self.embed_dim = embed_dim
        self.num_tokens = 2 if distilled else 1
        norm_layer = norm_layer or partial(nn.LayerNorm, eps=1e-6)
        act_layer = act_layer or nn.GELU
        self.patch_embed = embed_layer(img_size=img_size, patch_size=patch_size, in_c=in_c, embed_dim=embed_dim)
        n_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.dist_token = nn.Parameter(torch.zeros(1, 1, embed_dim)) if distilled else None
        self.pos_embed = nn.Parameter(torch.zeros(1, n_patches + self.num_tokens, embed_dim))
        self.pos_drop = nn.Dropout(p=drop_ratio)
        dpr = [x.item() for x in torch.linspace(0, drop_path_ratio, depth)]
        self.blocks = nn.Sequential(*[Block(embed_dim, num_heads, mlp_ratio, qkv_bias, qk_scale, drop_ratio, attn_drop_ratio,
                                            dpr[i], act_layer, norm_layer) for i in range(depth)])
        self.norm = norm_layer(embed_dim)
        if representation_size and not distilled:
            self.has_logits = True
            self.num_features = representation_size
            self.pre_logits = nn.Sequential(OrderedDict([("fc", nn.Linear(embed_dim, representation_size)), ("act", nn.Tanh())]))
        else:
            self.has_logits = False
            self.pre_logits = nn.Identity()
        self.head = nn.Linear(self.num_features, num_classes) if num_classes > 0 else nn.Identity()
        self.head_dist = None
        if distilled:
            self.head_dist = nn.Linear(self.embed_dim, self.num_classes) if num_classes > 0 else nn.Identity()
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        if self.dist_token is not None:
            nn.init.trunc_normal_(self.dist_token, std=0.02)
        nn.init.trunc_normal_(self.cls_token, std=0.02)
        self.apply(_init_vit_weights)

    def forward(self, x):
        from deeplearning_b200.engine import vit as engine

        return engine.apply(self, x)


def _vit(patch, dim, depth, heads, num_classes, has_logits):
    return VisionTransformer(img_size=224, patch_size=patch, embed_dim=dim, depth=depth, num_heads=heads,
                             representation_size=dim if has_logits else None, num_classes=num_classes)


def vit_base_patch16_224_in21k(num_classes: int = 21843, has_logits: bool = True):
    return _vit(16, 768, 12, 12, num_classes, has_logits)


def vit_base_patch32_224_in21k(num_classes: int = 21843, has_logits: bool = True):
    return _vit(32, 768, 12, 12, num_classes, has_logits)


def vit_large_patch16_224_in21k(num_classes: int = 21843, has_logits: bool = True):
    return _vit(16, 1024, 24, 16, num_classes, has_logits)


def vit_large_patch32_224_in21k(num_classes: int = 21843, has_logits: bool = True):
    return _vit(32, 1024, 24, 16, num_classes, has_logits)


def vit_huge_patch14_224_in21k(num_classes: int = 21843, has_logits: bool = True):
    return _vit(14, 1280, 32, 16, num_classes, has_logits)
