"""Drop-in for ``classification/efficientNet/models/network.py`` of KKKSQJ/DeepLearning: EfficientNet-B0..B7 on the sm_90a
engine.

The modules keep the reference's names, signatures, construction order and initialisation (``features`` = ``stem_conv``,
the MBConv blocks ``1a`` .. ``7x`` with ``block.expand_conv / dwconv / se / project_conv`` and ``dropout``, ``top``; then
``avgpool`` and ``classifier`` = Dropout + Linear), so ``torch.manual_seed(s); efficientnet_b0()`` gives the reference's
initial weights bit for bit and reference checkpoints load with ``strict=True``.  The reference's quirks are kept: the SE
squeeze width comes from the block's input width, both SE convolutions carry a bias, BatchNorm uses eps=1e-3, and the
drop-connect rate grows linearly with the block index from 0 at block 0.

``EfficientNet.forward`` hands the whole network to deeplearning_b200.engine.efficientnet; the blocks are never run one by
one.  ``torchsummary`` and ``torchvision`` are not needed.
"""
import copy
import math
from collections import OrderedDict
from functools import partial
from typing import Callable, Optional

import torch
import torch.nn as nn
from torch import Tensor

__all__ = ["_make_divisible", "DropPath", "ConvBNAction", "SELayer", "MBConvConfig", "MBConv", "EfficientNet",
           "efficientnet_b0", "efficientnet_b1", "efficientnet_b2", "efficientnet_b3", "efficientnet_b4",
           "efficientnet_b5", "efficientnet_b6", "efficientnet_b7"]


def _make_divisible(ch, divisor=8, min_ch=None):
    """Round ``ch`` to the nearest multiple of ``divisor`` (at least ``min_ch``), never more than 10% below ``ch``."""
    if min_ch is None:
        min_ch = divisor
    new_ch = max(min_ch, int(ch + divisor / 2) // divisor * divisor)
    if new_ch < 0.9 * ch:
        new_ch += divisor
    return new_ch


class DropPath(nn.Sequential):
    """Stochastic depth per sample: the branch is divided by keep = 1 - drop_prob and multiplied by floor(keep + U[0, 1))."""

    def __init__(self, drop_prob=None):
        super(DropPath, self).__init__()
        self.drop_prob = drop_prob

    def drop_path(self, x, drop_prob: float = 0, training: bool = False):
        if drop_prob == 0. or not training:
            return x
        keep_prob = 1 - drop_prob
        shape = (x.shape[0],) + (1,) * (x.ndim - 1)
        random_tensor = keep_prob + torch.rand(shape, dtype=x.dtype, device=x.device)
        random_tensor.floor_()
        return x.div(keep_prob) * random_tensor

    def forward(self, x):
        return self.drop_path(x, self.drop_prob, self.training)


class ConvBNAction(nn.Sequential):
    """Bias-free convolution (padding (k - 1) // 2), BatchNorm and activation (SiLU by default), as a Sequential."""

    def __init__(self,
                 in_planes: int,
                 out_planes: int,
                 kernel_size: int = 3,
                 stride: int = 1,
                 groups: int = 1,
                 norm_layer: Optional[Callable[..., nn.Module]] = None,
                 activation_layer: Optional[Callable[..., nn.Module]] = None):
        padding = (kernel_size - 1) // 2
        if norm_layer is None:
            norm_layer = nn.BatchNorm2d
        if activation_layer is None:
            activation_layer = nn.SiLU
        super(ConvBNAction, self).__init__(nn.Conv2d(in_channels=in_planes,
                                                     out_channels=out_planes,
                                                     kernel_size=kernel_size,
                                                     stride=stride,
                                                     padding=padding,
                                                     groups=groups,
                                                     bias=False),
                                           norm_layer(out_planes),
                                           activation_layer())


class SELayer(nn.Module):
    """Squeeze-and-excitation on ``outp`` channels with a squeeze width of _make_divisible(inp // reduction, 8)."""

    def __init__(self, inp: int, outp: int, reduction: int = 4):
        super(SELayer, self).__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(
            nn.Conv2d(outp, _make_divisible(inp // reduction, 8), 1),
            nn.SiLU(),
            nn.Conv2d(_make_divisible(inp // reduction, 8), outp, 1),
            nn.Sigmoid()
        )

    def forward(self, x: Tensor) -> Tensor:
        b, c, _, _ = x.size()
        y = self.avg_pool(x)
        y = self.fc(y).view(b, c, 1, 1)
        return x * y


class MBConvConfig:
    """Settings of one MBConv block: kernel 3 / 5, widths scaled by ``width_coefficient``, expand ratio 1 / 6, stride."""

    def __init__(self,
                 kernel: int,
                 input_c: int,
                 out_c: int,
                 expanded_ratio: int,
                 stride: int,
                 use_se: bool,
                 drop_rate: float,
                 index: str,
                 width_coefficient: float):
        self.kernel = kernel
        self.input_c = self.adjust_channels(input_c, width_coefficient)
        self.expanded_c = self.input_c * expanded_ratio
        self.out_c = self.adjust_channels(out_c, width_coefficient)
        self.use_se = use_se
        self.stride = stride
        self.drop_rate = drop_rate
        self.index = index

    @staticmethod
    def adjust_channels(channles: int, width_coefficient: float):
        return _make_divisible(channles * width_coefficient, 8)


class MBConv(nn.Module):
    """[expand 1x1 conv-BN-SiLU] -> depthwise conv-BN-SiLU -> SE -> project 1x1 conv-BN (-> DropPath + shortcut)."""

    def __init__(self, config: MBConvConfig, norm_layer: Callable[..., nn.Module]):
        super(MBConv, self).__init__()
        assert config.stride in [1, 2], "illegal stride value."
        self.use_res_connect = (config.stride == 1 and config.input_c == config.out_c)

        layers = OrderedDict()
        activation_layer = nn.SiLU
        if config.expanded_c != config.input_c:
            layers.update({"expand_conv": ConvBNAction(config.input_c, config.expanded_c, kernel_size=1, stride=1,
                                                       norm_layer=norm_layer, activation_layer=activation_layer)})
        layers.update({"dwconv": ConvBNAction(config.expanded_c, config.expanded_c, kernel_size=config.kernel,
                                              stride=config.stride, groups=config.expanded_c, norm_layer=norm_layer,
                                              activation_layer=activation_layer)})
        if config.use_se:
            layers.update({"se": SELayer(config.input_c, config.expanded_c)})
        layers.update({"project_conv": ConvBNAction(config.expanded_c, config.out_c, kernel_size=1, stride=1,
                                                    norm_layer=norm_layer, activation_layer=nn.Identity)})

        self.block = nn.Sequential(layers)
        self.out_channels = config.out_c
        self.is_stride = config.stride > 1
        if self.use_res_connect and config.drop_rate > 0:
            self.dropout = DropPath(config.drop_rate)
        else:
            self.dropout = nn.Identity()

    def forward(self, x):  # pragma: no cover - blocks are executed by the engine, not individually
        raise RuntimeError("deeplearning_b200 MBConv blocks run inside EfficientNet.forward (engine schedule)")


class EfficientNet(nn.Module):
    def __init__(self,
                 width_coefficient: float,
                 depth_coefficient: float,
                 num_classes: int = 1000,
                 dropout_rate: float = 0.2,
                 drop_connect_rate: float = 0.2,
                 block: Optional[Callable[..., nn.Module]] = None,
                 norm_layer: Optional[Callable[..., nn.Module]] = None):
        super(EfficientNet, self).__init__()

        # kernel_size, in_channel, out_channel, exp_ratio, strides, use_SE, drop_connect_rate, repeats (stages 2 - 8)
        default_cnf = [[3, 32, 16, 1, 1, True, drop_connect_rate, 1],
                       [3, 16, 24, 6, 2, True, drop_connect_rate, 2],
                       [5, 24, 40, 6, 2, True, drop_connect_rate, 2],
                       [3, 40, 80, 6, 2, True, drop_connect_rate, 3],
                       [5, 80, 112, 6, 1, True, drop_connect_rate, 3],
                       [5, 112, 192, 6, 2, True, drop_connect_rate, 4],
                       [3, 192, 320, 6, 1, True, drop_connect_rate, 1]]

        def round_repeats(repeats):
            return int(math.ceil(repeats * depth_coefficient))

        if block is None:
            block = MBConv
        if norm_layer is None:
            norm_layer = partial(nn.BatchNorm2d, eps=1e-3, momentum=0.1)

        adjust_channels = partial(MBConvConfig.adjust_channels, width_coefficient=width_coefficient)
        bneck_conf = partial(MBConvConfig, width_coefficient=width_coefficient)

        b = 0
        num_blocks = float(sum(round_repeats(i[-1]) for i in default_cnf))
        MBConv_setting = []
        for stage, args in enumerate(default_cnf):
            cnf = copy.copy(args)
            for i in range(round_repeats(cnf.pop(-1))):
                if i > 0:
                    cnf[-3] = 1        # stride: only the first block of a stage downsamples
                    cnf[1] = cnf[2]    # input channels = output channels
                cnf[-1] = args[-2] * b / num_blocks
                index = str(stage + 1) + chr(i + 97)   # 1a, 2a, 2b, ...
                MBConv_setting.append((bneck_conf(*cnf, index)))
                b += 1

        layers = OrderedDict()
        layers.update({"stem_conv": ConvBNAction(in_planes=3, out_planes=adjust_channels(32), kernel_size=3, stride=2,
                                                 norm_layer=norm_layer)})
        for cnf in MBConv_setting:
            layers.update({cnf.index: block(cnf, norm_layer)})
        last_conv_input_c = MBConv_setting[-1].out_c
        last_conv_output_c = adjust_channels(1280)
        layers.update({"top": ConvBNAction(in_planes=last_conv_input_c, out_planes=last_conv_output_c, kernel_size=1,
                                           norm_layer=norm_layer)})

        self.features = nn.Sequential(layers)
        self.avgpool = nn.AdaptiveAvgPool2d(1)

        classifier = []
        if dropout_rate > 0:
            classifier.append(nn.Dropout(p=dropout_rate, inplace=True))
        classifier.append(nn.Linear(last_conv_output_c, num_classes))
        self.classifier = nn.Sequential(*classifier)

        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
            elif isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.zeros_(m.bias)

    def forward(self, x: Tensor) -> Tensor:
        from deeplearning_b200.engine import efficientnet as engine

        return engine.apply(self, x)


def efficientnet_b0(num_classes=1000):
    # input image size 224x224
    return EfficientNet(width_coefficient=1.0, depth_coefficient=1.0, dropout_rate=0.2, num_classes=num_classes)


def efficientnet_b1(num_classes=1000):
    # input image size 240x240
    return EfficientNet(width_coefficient=1.0, depth_coefficient=1.1, dropout_rate=0.2, num_classes=num_classes)


def efficientnet_b2(num_classes=1000):
    # input image size 260x260
    return EfficientNet(width_coefficient=1.1, depth_coefficient=1.2, dropout_rate=0.3, num_classes=num_classes)


def efficientnet_b3(num_classes=1000):
    # input image size 300x300
    return EfficientNet(width_coefficient=1.2, depth_coefficient=1.4, dropout_rate=0.3, num_classes=num_classes)


def efficientnet_b4(num_classes=1000):
    # input image size 380x380
    return EfficientNet(width_coefficient=1.4, depth_coefficient=1.8, dropout_rate=0.4, num_classes=num_classes)


def efficientnet_b5(num_classes=1000):
    # input image size 456x456
    return EfficientNet(width_coefficient=1.6, depth_coefficient=2.2, dropout_rate=0.4, num_classes=num_classes)


def efficientnet_b6(num_classes=1000):
    # input image size 528x528
    return EfficientNet(width_coefficient=1.8, depth_coefficient=2.6, dropout_rate=0.5, num_classes=num_classes)


def efficientnet_b7(num_classes=1000):
    # input image size 600x600
    return EfficientNet(width_coefficient=2.0, depth_coefficient=3.1, dropout_rate=0.5, num_classes=num_classes)
