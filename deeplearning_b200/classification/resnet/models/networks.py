"""Host-side mirror of the reference ResNet constructors, backed by the sm_90a engine.

Drop-in for ``classification/resnet/models/networks.py`` of KKKSQJ/DeepLearning (ResNet ``:127``, Bottleneck ``:78``,
BasicBlock ``:38``, resnet50 ``:259``; the training script builds the identical torchvision model, train.py:14,74):
same constructor signatures, same parameter / buffer names and shapes, and the same RNG consumption order during
initialisation, so ``torch.manual_seed(s); resnet50()`` yields bit-identical initial weights and reference checkpoints
load with ``strict=True``.  The parameters are ordinary fp32 ``nn.Parameter`` tensors held by stock ``nn.Conv2d`` /
``nn.BatchNorm2d`` / ``nn.Linear`` containers; those containers' own ``forward`` is never used - ``ResNet.forward`` hands
the whole network to ``deeplearning_b200.engine.resnet`` which runs hand-written CUDA kernels through the C ABI and is
wired into autograd as a single Function.  There is no CPU path: a CPU tensor raises.
"""
import torch
import torch.nn as nn

__all__ = ["ResNet", "BasicBlock", "Bottleneck", "resnet18", "resnet34", "resnet50", "resnet101", "resnet152",
           "resnext50_32x4d", "resnext101_32x8d", "wide_resnet50_2", "wide_resnet101_2"]


def conv3x3(in_planes, out_planes, stride=1, groups=1, dilation=1):
    return nn.Conv2d(in_planes, out_planes, 3, stride, dilation, dilation, groups, bias=False)


def conv1x1(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, 1, stride, bias=False)


class _Block(nn.Module):
    """Parameter container for one residual block; the arithmetic lives in the engine."""
    expansion = 1

    def _finish(self, downsample, stride):
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):  # pragma: no cover - blocks are executed by the engine, not individually
        raise RuntimeError("deeplearning_b200 residual blocks run inside ResNet.forward (fused engine schedule)")


class BasicBlock(_Block):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None):
        super().__init__()
        norm_layer = norm_layer or nn.BatchNorm2d
        if groups != 1 or base_width != 64:
            raise ValueError("BasicBlock only supports groups=1 and base_width=64")
        if dilation > 1:
            raise NotImplementedError("Dilation > 1 not supported in BasicBlock")
        # registration order conv1,bn1,relu,conv2,bn2,downsample as in the reference (:51-57)
        self.conv1, self.bn1 = conv3x3(inplanes, planes, stride), norm_layer(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2, self.bn2 = conv3x3(planes, planes), norm_layer(planes)
        self.downsample = downsample
        self.stride = stride


class Bottleneck(_Block):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None):
        super().__init__()
        norm_layer = norm_layer or nn.BatchNorm2d
        width = int(planes * (base_width / 64.0)) * groups
        self.conv1, self.bn1 = conv1x1(inplanes, width), norm_layer(width)
        self.conv2, self.bn2 = conv3x3(width, width, stride, groups, dilation), norm_layer(width)  # stride on the 3x3 (v1.5)
        self.conv3, self.bn3 = conv1x1(width, planes * self.expansion), norm_layer(planes * self.expansion)
        self._finish(downsample, stride)


class ResNet(nn.Module):
    def __init__(self, block, layers, num_classes=1000, zero_init_residual=False, groups=1, width_per_group=64,
                 replace_stride_with_dilation=None, norm_layer=None):
        super().__init__()
        self._norm_layer = norm_layer = norm_layer or nn.BatchNorm2d
        self.inplanes, self.dilation = 64, 1
        rswd = [False, False, False] if replace_stride_with_dilation is None else replace_stride_with_dilation
        if len(rswd) != 3:
            raise ValueError("replace_stride_with_dilation should be None or a 3-element tuple, got {}".format(rswd))
        self.groups, self.base_width = groups, width_per_group
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = norm_layer(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        for i, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
            setattr(self, f"layer{i + 1}", self._make_layer(block, planes, n, stride=1 if i == 0 else 2,
                                                            dilate=False if i == 0 else rswd[i - 1]))
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        # same traversal order (hence same RNG stream) as the reference init loop (:163-168)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.constant_(m.bn3.weight, 0)
                elif isinstance(m, BasicBlock):
                    nn.init.constant_(m.bn2.weight, 0)

    def _make_layer(self, block, planes, blocks, stride=1, dilate=False):
        prev_dilation = self.dilation
        if dilate:
            self.dilation *= stride
            stride = 1
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(conv1x1(self.inplanes, planes * block.expansion, stride),
                                       self._norm_layer(planes * block.expansion))
        seq = [block(self.inplanes, planes, stride, downsample, self.groups, self.base_width, prev_dilation,
                     self._norm_layer)]
        self.inplanes = planes * block.expansion
        seq += [block(self.inplanes, planes, groups=self.groups, base_width=self.base_width, dilation=self.dilation,
                      norm_layer=self._norm_layer) for _ in range(1, blocks)]
        return nn.Sequential(*seq)

    def forward(self, x):
        from deeplearning_b200.engine import resnet as engine

        return engine.apply(self, x)

    _forward_impl = forward


def _resnet(arch, block, layers, pretrained, progress, **kwargs):
    if pretrained:
        raise RuntimeError("pretrained weights need network access; load a checkpoint with load_state_dict instead")
    return ResNet(block, layers, **kwargs)


def resnet18(pretrained=False, progress=True, **kwargs):
    return _resnet("resnet18", BasicBlock, [2, 2, 2, 2], pretrained, progress, **kwargs)


def resnet34(pretrained=False, progress=True, **kwargs):
    return _resnet("resnet34", BasicBlock, [3, 4, 6, 3], pretrained, progress, **kwargs)


def resnet50(pretrained=False, progress=True, **kwargs):
    return _resnet("resnet50", Bottleneck, [3, 4, 6, 3], pretrained, progress, **kwargs)


def resnet101(pretrained=False, progress=True, **kwargs):
    return _resnet("resnet101", Bottleneck, [3, 4, 23, 3], pretrained, progress, **kwargs)


def resnet152(pretrained=False, progress=True, **kwargs):
    return _resnet("resnet152", Bottleneck, [3, 8, 36, 3], pretrained, progress, **kwargs)


def resnext50_32x4d(pretrained=False, progress=True, **kwargs):
    kwargs["groups"], kwargs["width_per_group"] = 32, 4
    return _resnet("resnext50_32x4d", Bottleneck, [3, 4, 6, 3], pretrained, progress, **kwargs)


def resnext101_32x8d(pretrained=False, progress=True, **kwargs):
    kwargs["groups"], kwargs["width_per_group"] = 32, 8
    return _resnet("resnext101_32x8d", Bottleneck, [3, 4, 23, 3], pretrained, progress, **kwargs)


def wide_resnet50_2(pretrained=False, progress=True, **kwargs):
    kwargs["width_per_group"] = 64 * 2
    return _resnet("wide_resnet50_2", Bottleneck, [3, 4, 6, 3], pretrained, progress, **kwargs)


def wide_resnet101_2(pretrained=False, progress=True, **kwargs):
    kwargs["width_per_group"] = 64 * 2
    return _resnet("wide_resnet101_2", Bottleneck, [3, 4, 23, 3], pretrained, progress, **kwargs)
