"""Oracle: the SE-ResNet blocks of the reference (classification/seNet/models/se_module.py:4-19, se_resnet.py:11-84) restated
in fp32 PyTorch as a block pair that plugs into ``torchvision.models.ResNet``, the network the reference builds them into
(se_resnet.py:87-134).  The GPU tests use ``se_resnet_yardstick`` as their fp32 reference; tests/golden/make_senet_golden.py
pins it bit for bit against the reference's own ``se_resnet50()`` / ``se_resnet()``.

    SELayer:      gate = sigmoid(fc2(relu(fc1(avgpool(x))))),  out = x * gate                              se_module.py:15-19
    SEBottleneck: 1x1 -> BN -> ReLU -> 3x3(stride) -> BN -> ReLU -> 1x1 -> BN -> SE -> + identity -> ReLU  se_resnet.py:63-84
    SEBasicBlock: 3x3(stride) -> BN -> ReLU -> 3x3 -> BN -> SE -> + identity -> ReLU                      se_resnet.py:24-42
"""
import torch
import torch.nn as nn


class SELayer(nn.Module):
    def __init__(self, channel, reduction=16):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(nn.Linear(channel, channel // reduction, bias=False), nn.ReLU(inplace=True),
                                nn.Linear(channel // reduction, channel, bias=False), nn.Sigmoid())

    def forward(self, x):
        b, c = x.shape[:2]
        return x * self.fc(self.avg_pool(x).view(b, c)).view(b, c, 1, 1)


class SEBasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None,
                 reduction=16):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.se = SELayer(planes, reduction)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.se(self.bn2(self.conv2(out)))
        identity = x if self.downsample is None else self.downsample(x)
        return self.relu(out + identity)


class SEBottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, groups=1, base_width=64, dilation=1, norm_layer=None,
                 reduction=16):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.se = SELayer(planes * 4, reduction)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.relu(self.bn2(self.conv2(out)))
        out = self.se(self.bn3(self.conv3(out)))
        identity = x if self.downsample is None else self.downsample(x)
        return self.relu(out + identity)


def se_resnet_yardstick(state, layers, bottleneck=True, num_classes=1000):
    """torchvision ResNet with the SE blocks above, loaded with ``state`` (the reference's state_dict keys)."""
    import torchvision

    m = torchvision.models.ResNet(SEBottleneck if bottleneck else SEBasicBlock, list(layers), num_classes=num_classes)
    if state is not None:
        m.load_state_dict(state)
    return m
