"""Host-side mirror of the reference's MNIST toy nets (classification/mnist/models/network.py:7 ``mnist_cnn``, :34 ``mnist_fcn``).

BASELINE.json's config 0 is *CPU plumbing, no GPU*: it exists to exercise the host loop (constructor -> forward -> loss ->
backward -> optimizer) end to end where no GPU is present, so these two nets are ordinary PyTorch modules with the
reference's layer structure, parameter names and initialisation order.  They are not part of the sm_90a hot path.
"""
import torch
import torch.nn as nn


def _stage(cin, cout):
    return nn.Sequential(nn.Conv2d(cin, cout, 3, 1, 1), nn.ReLU(inplace=True), nn.MaxPool2d(2, 2))


class mnist_cnn(nn.Module):
    def __init__(self, num_classes):
        super().__init__()
        layers = []
        for cin, cout in ((3, 32), (32, 64), (64, 64)):
            layers += list(_stage(cin, cout))
        self.backbone = nn.Sequential(*layers)
        self.fc = nn.Sequential(nn.Linear(64 * 3 * 3, 128), nn.ReLU(inplace=True), nn.Linear(128, num_classes))

    def forward(self, x):
        return self.fc(torch.flatten(self.backbone(x), 1))


class mnist_fcn(nn.Module):
    def __init__(self, num_classes):
        super().__init__()
        self.conv1, self.conv2, self.conv3 = _stage(3, 32), _stage(32, 64), _stage(64, 64)
        self.conv4 = nn.Sequential(nn.Conv2d(64, 128, 3, 1, 0), nn.ReLU(inplace=True))  # == Linear(576, 128)
        self.conv5 = nn.Sequential(nn.Conv2d(128, num_classes, 1, 1, 0))                # == Linear(128, classes)

    def forward(self, x):
        for stage in (self.conv1, self.conv2, self.conv3, self.conv4, self.conv5):
            x = stage(x)
        return torch.flatten(x, 1)
