"""Host-side mirror of the reference ConvNeXt constructors, backed by the sm_90a engine.

Drop-in for ``classification/convNext/models/networks.py`` of KKKSQJ/DeepLearning (ConvNeXt ``:108``, Block ``:70``,
LayerNorm ``:41``, ``convnext_tiny`` ``:173`` ...): same constructor signatures, parameter names / shapes and the same
``apply(_init_weights)`` RNG order (trunc_normal std 0.2 on every conv / linear, as in the reference ``:155-158``), so
reference checkpoints load unchanged.  Sub-modules only hold parameters; ``ConvNeXt.forward`` runs the whole network through
``deeplearning_b200.engine.convnext`` (depthwise 7x7 kernel, LayerNorm, GEMMs with bias/GELU/layer-scale/residual epilogues,
2x2/s2 convs as 4-tap implicit GEMMs).  No CPU path.
"""
import torch
import torch.nn as nn


class _EngineOnly(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter container; it runs inside ConvNeXt.forward")


class DropPath(nn.Module):
    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob


class LayerNorm(_EngineOnly):
    """channels_last / channels_first LayerNorm container (the engine keeps activations NHWC, where both are the same op)."""

    def __init__(self, normalized_shape, eps=1e-6, data_format="channels_last"):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape), requires_grad=True)
        self.bias = nn.Parameter(torch.zeros(normalized_shape), requires_grad=True)
        self.eps = eps
        self.data_format = data_format
        if data_format not in ["channels_last", "channels_first"]:
            raise ValueError(f"not support data format '{data_format}'")
        self.normalized_shape = (normalized_shape,)


class Block(_EngineOnly):
    def __init__(self, dim, drop_rate=0., layer_scale_init_value=1e-6):
        super().__init__()
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = LayerNorm(dim, eps=1e-6, data_format="channels_last")
        self.pwconv1 = nn.Linear(dim, 4 * dim)
        self.act = nn.GELU()
        self.pwconv2 = nn.Linear(4 * dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones((dim,)), requires_grad=True) \
            if layer_scale_init_value > 0 else None
        self.drop_path = DropPath(drop_rate) if drop_rate > 0. else nn.Identity()


class ConvNeXt(nn.Module):
    def __init__(self, in_chans: int = 3, num_classes: int = 1000, depths: list = None, dims: list = None,
                 drop_path_rate: float = 0., layer_scale_init_value: float = 1e-6, head_init_scale: float = 1.):
        super().__init__()
        self.downsample_layers = nn.ModuleList()
        self.downsample_layers.append(nn.Sequential(nn.Conv2d(in_chans, dims[0], kernel_size=4, stride=4),
                                                    LayerNorm(dims[0], eps=1e-6, data_format="channels_first")))
        for i in range(3):
            self.downsample_layers.append(nn.Sequential(LayerNorm(dims[i], eps=1e-6, data_format="channels_first"),
                                                        nn.Conv2d(dims[i], dims[i + 1], kernel_size=2, stride=2)))
        self.stages = nn.ModuleList()
        dp_rates = [x.item() for x in torch.linspace(0, drop_path_rate, sum(depths))]
        cur = 0
        for i in range(4):
            self.stages.append(nn.Sequential(*[Block(dims[i], dp_rates[cur + j], layer_scale_init_value)
                                               for j in range(depths[i])]))
            cur += depths[i]
        self.norm = nn.LayerNorm(dims[-1], eps=1e-6)
        self.head = nn.Linear(dims[-1], num_classes)
        self.apply(self._init_weights)
        self.head.weight.data.mul_(head_init_scale)
        self.head.bias.data.mul_(head_init_scale)

    def _init_weights(self, m):
        if isinstance(m, (nn.Conv2d, nn.Linear)):
            nn.init.trunc_normal_(m.weight, std=0.2)
            nn.init.constant_(m.bias, 0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        from deeplearning_b200.engine import convnext as engine

        return engine.apply(self, x)


def convnext_tiny(num_classes: int):
    return ConvNeXt(depths=[3, 3, 9, 3], dims=[96, 192, 384, 768], num_classes=num_classes, drop_path_rate=0.2)


def convnext_small(num_classes: int):
    return ConvNeXt(depths=[3, 3, 27, 3], dims=[96, 192, 384, 768], num_classes=num_classes)


def convnext_base(num_classes: int):
    return ConvNeXt(depths=[3, 3, 27, 3], dims=[128, 256, 512, 1024], num_classes=num_classes)


def convnext_large(num_classes: int):
    return ConvNeXt(depths=[3, 3, 27, 3], dims=[192, 384, 768, 1536], num_classes=num_classes)


def convnext_xlarge(num_classes: int):
    return ConvNeXt(depths=[3, 3, 27, 3], dims=[256, 512, 1024, 2048], num_classes=num_classes)
