"""Drop-in for the reference's self-supervised/MAE/models/VIT.py: ``ViT``, ``Transformer``, ``PreNorm``, ``SelfAttention``
and ``FFN`` with the reference's module tree, parameter names and construction order, so a seeded constructor gives the
reference's parameters bit for bit.  The modules hold parameters only: the encoder and decoder stacks run inside
``MAE.forward`` on the GPU engine (engine/mae.py).  The classification ``ViT.forward`` (class token + ``mlp_head``) is not
built here; classification/vision_transformer trains that model."""
import torch
import torch.nn as nn


class _EngineOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} is a parameter container; it runs inside MAE.forward on the GPU engine")


class ViT(nn.Module):
    def __init__(self, image_size, patch_size, num_classes=1000, dim=1024, depth=6, num_heads=8, mlp_dim=2048, pool='cls',
                 channels=3, dim_per_head=64, dropout=0., embed_dropout=0.):
        super().__init__()
        img_h, img_w = image_size if isinstance(image_size, tuple) else (image_size, image_size)
        self.patch_h, self.patch_w = patch_size if isinstance(patch_size, tuple) else (patch_size, patch_size)
        assert not img_h % self.patch_h and not img_w % self.patch_w, \
            f'Image dimensions ({img_h},{img_w}) must be divisible by the patch size ({self.patch_h},{self.patch_w}).'
        num_patches = (img_h // self.patch_h) * (img_w // self.patch_w)
        assert pool in {'cls', 'mean'}, f'pool type must be either cls (cls token) or mean (mean pooling), got: {pool}'
        patch_dim = channels * self.patch_h * self.patch_w
        self.patch_embed = nn.Linear(patch_dim, dim)
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.pos_embed = nn.Parameter(torch.randn(1, num_patches + 1, dim))
        self.dropout = nn.Dropout(p=embed_dropout)
        self.pool = pool
        self.transformer = Transformer(dim, mlp_dim, depth=depth, num_heads=num_heads, dim_per_head=dim_per_head,
                                       dropout=dropout)
        self.mlp_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))

    def forward(self, x):
        raise NotImplementedError("the classification forward of the MAE ViT (class token + mlp_head) is not built on the "
                                  "GPU engine; train a classification ViT with "
                                  "deeplearning_b200.classification.vision_transformer")


class Transformer(_EngineOnly):
    def __init__(self, dim, mlp_dim, depth=6, num_heads=8, dim_per_head=64, dropout=0.):
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                PreNorm(dim, SelfAttention(dim, num_heads=num_heads, dim_per_head=dim_per_head, dropout=dropout)),
                PreNorm(dim, FFN(dim, mlp_dim, dropout=dropout)),
            ]))


class PreNorm(_EngineOnly):
    def __init__(self, dim, net):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.net = net


class SelfAttention(_EngineOnly):
    def __init__(self, dim, num_heads=8, dim_per_head=64, dropout=0.):
        super().__init__()
        self.num_heads = num_heads
        self.scale = dim_per_head ** -0.5
        inner_dim = dim_per_head * num_heads
        self.to_qkv = nn.Linear(dim, inner_dim * 3, bias=False)
        self.attend = nn.Softmax(dim=-1)
        project_out = not (num_heads == 1 and dim_per_head == dim)
        self.out = nn.Sequential(nn.Linear(inner_dim, dim), nn.Dropout(dropout)) if project_out else nn.Identity()


class FFN(_EngineOnly):
    def __init__(self, dim, hidden_dim, dropout=0.):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(dim, hidden_dim), nn.GELU(), nn.Dropout(p=dropout), nn.Linear(hidden_dim, dim),
                                 nn.Dropout(p=dropout))
