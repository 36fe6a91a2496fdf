"""Host-side mirror of the reference Swin Transformer constructors, backed by the sm_90a engine.

Drop-in for ``classification/swin_transformer/models/swin_transformer.py`` of KKKSQJ/DeepLearning (SwinTransformer ``:478``,
BasicLayer ``:353``, SwinTransformerBlock ``:168``, WindowAttention ``:70``, PatchMerging ``:308``, PatchEmbed ``:430``,
Mlp ``:19``): same constructor signatures, parameter / buffer names (``relative_position_bias_table``,
``relative_position_index``, ``attn_mask`` ...), shapes and initialisation RNG order, so reference checkpoints load with
``strict=True``.  No timm dependency (``DropPath`` / ``to_2tuple`` / ``trunc_normal_`` are local).  Sub-modules only hold
parameters; ``SwinTransformer.forward`` runs the whole network through ``deeplearning_b200.engine.swin``: the cyclic shift,
window partition / reverse, relative-position bias and shift mask all live inside one wgmma window-attention kernel.
"""
import torch
import torch.nn as nn
from torch.nn.init import trunc_normal_


def to_2tuple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x)


class _EngineOnly(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter container; it runs inside SwinTransformer.forward")


class DropPath(nn.Module):
    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob


class Mlp(_EngineOnly):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features or in_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features)
        self.drop = nn.Dropout(drop)


def window_partition(x, window_size):
    """(B, H, W, C) -> (num_windows*B, window_size, window_size, C); kept for building ``attn_mask`` exactly as the reference."""
    B, H, W, C = x.shape
    x = x.view(B, H // window_size, window_size, W // window_size, window_size, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, window_size, window_size, C)


def window_reverse(windows, window_size, H, W):
    B = int(windows.shape[0] / (H * W / window_size / window_size))
    x = windows.view(B, H // window_size, W // window_size, window_size, window_size, -1)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, H, W, -1)


class WindowAttention(_EngineOnly):
    def __init__(self, dim, window_size, num_heads, qkv_bias=True, qk_scale=None, attn_drop=0., proj_drop=0.):
        super().__init__()
        self.dim, self.window_size, self.num_heads = dim, window_size, num_heads
        self.scale = qk_scale or (dim // num_heads) ** -0.5
        wh, ww = window_size
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * wh - 1) * (2 * ww - 1), num_heads))
        coords = torch.stack(torch.meshgrid([torch.arange(wh), torch.arange(ww)], indexing="ij")).flatten(1)
        rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += wh - 1
        rel[:, :, 1] += ww - 1
        rel[:, :, 0] *= 2 * ww - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)
        trunc_normal_(self.relative_position_bias_table, std=.02)
        self.softmax = nn.Softmax(dim=-1)


class SwinTransformerBlock(_EngineOnly):
    def __init__(self, dim, input_resolution, num_heads, window_size=7, shift_size=0, mlp_ratio=4., qkv_bias=True,
                 qk_scale=None, drop=0., attn_drop=0., drop_path=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm,
                 fused_window_process=False):
        super().__init__()
        self.dim, self.input_resolution, self.num_heads = dim, input_resolution, num_heads
        self.window_size, self.shift_size, self.mlp_ratio = window_size, shift_size, mlp_ratio
        if min(self.input_resolution) <= self.window_size:
            self.shift_size = 0
            self.window_size = min(self.input_resolution)
        assert 0 <= self.shift_size < self.window_size, "shift_size must in 0-window_size"
        self.norm1 = norm_layer(dim)
        self.attn = WindowAttention(dim, to_2tuple(self.window_size), num_heads, qkv_bias, qk_scale, attn_drop, drop)
        self.drop_path = DropPath(drop_path) if drop_path > 0. else nn.Identity()
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), act_layer=act_layer, drop=drop)
        attn_mask = None
        if self.shift_size > 0:
            H, W = self.input_resolution
            img_mask = torch.zeros((1, H, W, 1))
            spans = (slice(0, -self.window_size), slice(-self.window_size, -self.shift_size), slice(-self.shift_size, None))
            cnt = 0
            for h in spans:
                for w in spans:
                    img_mask[:, h, w, :] = cnt
                    cnt += 1
            mw = window_partition(img_mask, self.window_size).view(-1, self.window_size * self.window_size)
            attn_mask = mw.unsqueeze(1) - mw.unsqueeze(2)
            attn_mask = attn_mask.masked_fill(attn_mask != 0, float(-100.0)).masked_fill(attn_mask == 0, float(0.0))
        self.register_buffer("attn_mask", attn_mask)
        self.fused_window_process = fused_window_process  # always "fused" here: the permutations live in the attention kernel


class PatchMerging(_EngineOnly):
    def __init__(self, input_resolution, dim, norm_layer=nn.LayerNorm):
        super().__init__()
        self.input_resolution, self.dim = input_resolution, dim
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = norm_layer(4 * dim)


class BasicLayer(_EngineOnly):
    def __init__(self, dim, input_resolution, depth, num_heads, window_size, mlp_ratio=4., qkv_bias=True, qk_scale=None,
                 drop=0., attn_drop=0., drop_path=0., norm_layer=nn.LayerNorm, downsample=None, use_checkpoint=False,
                 fused_window_process=False):
        super().__init__()
        self.dim, self.input_resolution, self.depth, self.use_checkpoint = dim, input_resolution, depth, use_checkpoint
        self.blocks = nn.ModuleList([
            SwinTransformerBlock(dim, input_resolution, num_heads, window_size, 0 if (i % 2 == 0) else window_size // 2,
                                 mlp_ratio, qkv_bias, qk_scale, drop, attn_drop,
                                 drop_path[i] if isinstance(drop_path, list) else drop_path, norm_layer=norm_layer,
                                 fused_window_process=fused_window_process) for i in range(depth)])
        self.downsample = downsample(input_resolution, dim=dim, norm_layer=norm_layer) if downsample is not None else None


class PatchEmbed(_EngineOnly):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, embed_dim=96, norm_layer=None):
        super().__init__()
        self.img_size, self.patch_size = to_2tuple(img_size), to_2tuple(patch_size)
        self.patches_resolution = [self.img_size[0] // self.patch_size[0], self.img_size[1] // self.patch_size[1]]
        self.num_patches = self.patches_resolution[0] * self.patches_resolution[1]
        self.in_chans, self.embed_dim = in_chans, embed_dim
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=self.patch_size, stride=self.patch_size)
        self.norm = norm_layer(embed_dim) if norm_layer is not None else None


class SwinTransformer(nn.Module):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, num_classes=1000, embed_dim=96, depths=[2, 2, 6, 2],
                 num_heads=[3, 6, 12, 24], window_size=7, mlp_ratio=4., qkv_bias=True, qk_scale=None, drop_rate=0.,
                 attn_drop_rate=0., drop_path_rate=0.1, norm_layer=nn.LayerNorm, ape=False, patch_norm=True,
                 use_checkpoint=False, fused_window_process=False, **kwargs):
        super().__init__()
        self.num_classes, self.num_layers, self.embed_dim = num_classes, len(depths), embed_dim
        self.ape, self.patch_norm = ape, patch_norm
        self.num_features = int(embed_dim * 2 ** (self.num_layers - 1))
        self.mlp_ratio = mlp_ratio
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim, norm_layer if patch_norm else None)
        res = self.patches_resolution = self.patch_embed.patches_resolution
        if self.ape:
            self.absolute_pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches, embed_dim))
            trunc_normal_(self.absolute_pos_embed, std=.02)
        self.pos_drop = nn.Dropout(p=drop_rate)
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, sum(depths))]
        self.layers = nn.ModuleList()
        for i in range(self.num_layers):
            self.layers.append(BasicLayer(int(embed_dim * 2 ** i), (res[0] // (2 ** i), res[1] // (2 ** i)), depths[i],
                                          num_heads[i], window_size, self.mlp_ratio, qkv_bias, qk_scale, drop_rate,
                                          attn_drop_rate, dpr[sum(depths[:i]):sum(depths[:i + 1])], norm_layer,
                                          PatchMerging if (i < self.num_layers - 1) else None, use_checkpoint,
                                          fused_window_process))
        self.norm = norm_layer(self.num_features)
        self.avgpool = nn.AdaptiveAvgPool1d(1)
        self.head = nn.Linear(self.num_features, num_classes) if num_classes > 0 else nn.Identity()
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'absolute_pos_embed'}

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {'relative_position_bias_table'}

    def forward(self, x):
        from deeplearning_b200.engine import swin as engine

        return engine.apply(self, x)
