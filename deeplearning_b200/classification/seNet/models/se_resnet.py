"""Drop-in for ``classification/seNet/models/se_resnet.py`` of KKKSQJ/DeepLearning: SE-ResNet on the sm_90a ResNet engine.

The reference builds torchvision's ``ResNet`` with ``SEBasicBlock`` / ``SEBottleneck`` (se_resnet.py:11-84, :87-134); here
the same blocks go into the engine-backed ``ResNet`` of ``classification/resnet/models/networks.py``, which has the same
constructor, module order and initialisation loop.  So ``torch.manual_seed(s); se_resnet50()`` gives the reference's initial
weights bit for bit and reference checkpoints load with ``strict=True``.

The blocks register their modules in the reference's order and always use ``nn.BatchNorm2d``; the bottleneck ignores
``groups`` / ``base_width`` as the reference does.  They do not derive from ``Bottleneck`` / ``BasicBlock``: the
``zero_init_residual`` option of ``ResNet`` only zeroes the last BatchNorm of those two types, and in the reference it never
touches an SE block either.
"""
import torch.nn as nn

from ...resnet.models.networks import ResNet, _Block, conv3x3
from .se_module import SELayer

__all__ = ["SELayer", "SEBasicBlock", "SEBottleneck", "se_resnet", "se_resnet34", "se_resnet50", "se_resnet101",
           "se_resnet152"]


class SEBasicBlock(_Block):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None,
                 reduction=16):
        super().__init__()
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(planes, planes, 1)
        self.bn2 = nn.BatchNorm2d(planes)
        self.se = SELayer(planes, reduction)
        self.downsample = downsample
        self.stride = stride


class SEBottleneck(_Block):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None,
                 reduction=16):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.se = SELayer(planes * 4, reduction)
        self.downsample = downsample
        self.stride = stride


def se_resnet(num_classes=1000):
    """SE-ResNet-18"""
    return ResNet(SEBasicBlock, [2, 2, 2, 2], num_classes=num_classes)


def se_resnet34(num_classes=1000):
    return ResNet(SEBasicBlock, [3, 4, 6, 3], num_classes=num_classes)


def se_resnet50(num_classes=1000, pretrained=False):
    if pretrained:
        raise RuntimeError("pretrained weights need network access; load a checkpoint with load_state_dict instead")
    return ResNet(SEBottleneck, [3, 4, 6, 3], num_classes=num_classes)


def se_resnet101(num_classes=1000):
    return ResNet(SEBottleneck, [3, 4, 23, 3], num_classes=num_classes)


def se_resnet152(num_classes=1000):
    return ResNet(SEBottleneck, [3, 8, 36, 3], num_classes=num_classes)
