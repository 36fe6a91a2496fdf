"""Drop-in for ``classification/seNet/models/se_module.py`` of KKKSQJ/DeepLearning: the squeeze-and-excitation layer.

``SELayer`` keeps the reference's submodule names and construction order (``avg_pool``, then ``fc`` = Linear(C, C // r,
bias=False), ReLU, Linear(C // r, C, bias=False), Sigmoid), so state_dict keys match and the two Linear layers draw their
default initialisation from the RNG stream in the reference's order.  Its arithmetic runs inside the ResNet engine
(deeplearning_b200.engine.resnet, csrc/se.cuh), fused with the BatchNorm passes of the block's tail.
"""
import torch.nn as nn


class SELayer(nn.Module):
    def __init__(self, channel, reduction=16):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(
            nn.Linear(channel, channel // reduction, bias=False),
            nn.ReLU(inplace=True),
            nn.Linear(channel // reduction, channel, bias=False),
            nn.Sigmoid(),
        )

    def forward(self, x):  # pragma: no cover - the gate is executed by the engine, not individually
        raise RuntimeError("deeplearning_b200 SE layers run inside ResNet.forward (fused engine schedule)")
