"""Drop-in for ``classification/RepVGG/models/se_block.py`` of KKKSQJ/DeepLearning: the squeeze-and-excitation block of
RepVGG-D2se.

``SEBlock`` keeps the reference's submodule names and construction order (``down`` = Conv2d(C, internal, 1, bias=True), then
``up`` = Conv2d(internal, C, 1, bias=True)), so state_dict keys match and both convolutions draw their default
initialisation from the RNG stream in the reference's order.  The GPU engine does not run it yet
(deeplearning_b200.engine.repvgg rejects ``use_se`` models with NotImplementedError).
"""
import torch.nn as nn


class SEBlock(nn.Module):
    def __init__(self, input_channels, internal_neurons):
        super().__init__()
        self.down = nn.Conv2d(input_channels, internal_neurons, kernel_size=1, stride=1, bias=True)
        self.up = nn.Conv2d(internal_neurons, input_channels, kernel_size=1, stride=1, bias=True)
        self.input_channels = input_channels

    def forward(self, inputs):  # pragma: no cover - RepVGG blocks are executed by the engine, not individually
        raise RuntimeError("deeplearning_b200 RepVGG blocks run inside RepVGG.forward (engine schedule)")
