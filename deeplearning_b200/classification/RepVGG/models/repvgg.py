"""Drop-in for ``classification/RepVGG/models/repvgg.py`` of KKKSQJ/DeepLearning: RepVGG on the sm_90a engine.

The modules keep the reference's names, signatures and construction order (``stage0`` .. ``stage4`` of ``RepVGGBlock``s with
``nonlinearity``, ``se``, ``rbr_identity``, ``rbr_dense.conv / bn``, ``rbr_1x1.conv / bn`` or ``rbr_reparam``, then ``gap`` and
``linear``), and nothing re-initialises them, so ``torch.manual_seed(s); create_RepVGG_A0()`` gives the reference's initial
weights bit for bit and reference checkpoints (train form or converted) load with ``strict=True``.

``RepVGG.forward`` hands the whole network to deeplearning_b200.engine.repvgg: fused three-branch BatchNorm passes in train
mode, one conv + bias + ReLU GEMM per layer in eval mode (train form folded on the device, or the re-parameterised weights).
The re-parameterisation helpers (``get_equivalent_kernel_bias``, ``switch_to_deploy``, ``repvgg_model_convert``) and
``get_custom_L2`` are parameter arithmetic in PyTorch with the reference's semantics.  The grouped (g2 / g4) and SE (D2se)
variants construct as in the reference; the engine rejects them with NotImplementedError.
"""
import copy

import torch
import torch.nn as nn
import torch.nn.functional as F

from .se_block import SEBlock

__all__ = ["conv_bn", "RepVGGBlock", "RepVGG", "func_dict", "get_RepVGG_func_by_name", "repvgg_model_convert"]


def conv_bn(in_channels, out_channels, kernel_size, stride, padding, groups=1):
    """Bias-free convolution followed by BatchNorm2d, as ``Sequential(conv, bn)``."""
    result = nn.Sequential()
    result.add_module("conv", nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                                        groups=groups, bias=False))
    result.add_module("bn", nn.BatchNorm2d(out_channels))
    return result


class RepVGGBlock(nn.Module):
    """Train form: relu(se(bn(conv3x3(x)) + bn(conv1x1(x)) [+ bn(x)])); deploy form: relu(se(conv3x3_biased(x)))."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 padding_mode="zeros", deploy=False, use_se=False):
        super().__init__()
        assert kernel_size == 3 and padding == 1
        self.deploy = deploy
        self.groups = groups
        self.in_channels = in_channels
        self.nonlinearity = nn.ReLU()
        self.se = SEBlock(out_channels, internal_neurons=out_channels // 16) if use_se else nn.Identity()
        if deploy:
            self.rbr_reparam = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                                         dilation=dilation, groups=groups, bias=True, padding_mode=padding_mode)
        else:
            same = in_channels == out_channels and stride == 1
            self.rbr_identity = nn.BatchNorm2d(in_channels) if same else None
            self.rbr_dense = conv_bn(in_channels, out_channels, kernel_size, stride, padding, groups)
            self.rbr_1x1 = conv_bn(in_channels, out_channels, 1, stride, padding - kernel_size // 2, groups)

    def forward(self, inputs):  # pragma: no cover - blocks are executed by the engine, not individually
        raise RuntimeError("deeplearning_b200 RepVGG blocks run inside RepVGG.forward (engine schedule)")

    def get_custom_L2(self):
        """L2 term with the 3x3 kernel's centre replaced by the equivalent (BatchNorm-scaled) centre of both branches,
        normalised so its coefficient compares with plain weight decay (the reference's optional regulariser)."""
        k3, k1 = self.rbr_dense.conv.weight, self.rbr_1x1.conv.weight
        t3 = self._bn_scale(self.rbr_dense.bn).detach()
        t1 = self._bn_scale(self.rbr_1x1.bn).detach()
        centre = k3[:, :, 1:2, 1:2]
        circle = (k3 ** 2).sum() - (centre ** 2).sum()
        eq = centre * t3 + k1 * t1
        return (eq ** 2 / (t3 ** 2 + t1 ** 2)).sum() + circle

    @staticmethod
    def _bn_scale(bn):
        return (bn.weight / (bn.running_var + bn.eps).sqrt()).reshape(-1, 1, 1, 1)

    def _identity_kernel(self, device):
        per_group = self.in_channels // self.groups
        k = torch.zeros(self.in_channels, per_group, 3, 3, device=device)
        idx = torch.arange(self.in_channels, device=device)
        k[idx, idx % per_group, 1, 1] = 1.0
        return k

    def _fuse_bn_tensor(self, branch):
        """(kernel * gamma / std, beta - mean * gamma / std) of a conv_bn branch or of the identity BatchNorm; (0, 0) for
        None."""
        if branch is None:
            return 0, 0
        if isinstance(branch, nn.Sequential):
            kernel, bn = branch.conv.weight, branch.bn
        else:
            kernel, bn = self._identity_kernel(branch.weight.device), branch
        std = (bn.running_var + bn.eps).sqrt()
        return kernel * (bn.weight / std).reshape(-1, 1, 1, 1), bn.bias - bn.running_mean * bn.weight / std

    @staticmethod
    def _pad_1x1_to_3x3_tensor(kernel1x1):
        return 0 if kernel1x1 is None else F.pad(kernel1x1, [1, 1, 1, 1])

    def get_equivalent_kernel_bias(self):
        """Kernel and bias of the one 3x3 convolution equal to the block's three branches in eval mode (differentiable)."""
        k3, b3 = self._fuse_bn_tensor(self.rbr_dense)
        k1, b1 = self._fuse_bn_tensor(self.rbr_1x1)
        kid, bid = self._fuse_bn_tensor(self.rbr_identity)
        return k3 + self._pad_1x1_to_3x3_tensor(k1) + kid, b3 + b1 + bid

    def switch_to_deploy(self):
        """Replace the three branches by ``rbr_reparam``, the equivalent biased 3x3 convolution (no-op when converted)."""
        if hasattr(self, "rbr_reparam"):
            return
        kernel, bias = self.get_equivalent_kernel_bias()
        dense = self.rbr_dense.conv
        self.rbr_reparam = nn.Conv2d(dense.in_channels, dense.out_channels, dense.kernel_size, stride=dense.stride,
                                     padding=dense.padding, dilation=dense.dilation, groups=dense.groups, bias=True)
        self.rbr_reparam.weight.data = kernel
        self.rbr_reparam.bias.data = bias
        for p in self.parameters():
            p.detach_()
        del self.rbr_dense
        del self.rbr_1x1
        if hasattr(self, "rbr_identity"):
            del self.rbr_identity
        self.deploy = True


class RepVGG(nn.Module):
    def __init__(self, num_blocks, num_classes=1000, width_multiplier=None, override_groups_map=None, deploy=False,
                 use_se=False):
        super().__init__()
        assert len(width_multiplier) == 4
        self.deploy = deploy
        self.override_groups_map = override_groups_map or dict()
        self.use_se = use_se
        assert 0 not in self.override_groups_map
        self.in_planes = min(64, int(64 * width_multiplier[0]))
        self.stage0 = RepVGGBlock(3, self.in_planes, kernel_size=3, stride=2, padding=1, deploy=deploy, use_se=use_se)
        self.cur_layer_idx = 1
        self.stage1 = self._make_stage(int(64 * width_multiplier[0]), num_blocks[0], stride=2)
        self.stage2 = self._make_stage(int(128 * width_multiplier[1]), num_blocks[1], stride=2)
        self.stage3 = self._make_stage(int(256 * width_multiplier[2]), num_blocks[2], stride=2)
        self.stage4 = self._make_stage(int(512 * width_multiplier[3]), num_blocks[3], stride=2)
        self.gap = nn.AdaptiveAvgPool2d(output_size=1)
        self.linear = nn.Linear(int(512 * width_multiplier[3]), num_classes)

    def _make_stage(self, planes, num_blocks, stride):
        blocks = []
        for s in [stride] + [1] * (num_blocks - 1):
            groups = self.override_groups_map.get(self.cur_layer_idx, 1)
            blocks.append(RepVGGBlock(self.in_planes, planes, kernel_size=3, stride=s, padding=1, groups=groups,
                                      deploy=self.deploy, use_se=self.use_se))
            self.in_planes = planes
            self.cur_layer_idx += 1
        return nn.Sequential(*blocks)

    def forward(self, x):
        from deeplearning_b200.engine import repvgg as engine

        return engine.apply(self, x)


optional_groupwise_layers = [2, 4, 6, 8, 10, 12, 14, 16, 18, 20, 22, 24, 26]
g2_map = {layer: 2 for layer in optional_groupwise_layers}
g4_map = {layer: 4 for layer in optional_groupwise_layers}

_A = [2, 4, 14, 1]
_B = [4, 6, 16, 1]


def create_RepVGG_A0(deploy=False, num_classes=1000):
    return RepVGG(_A, num_classes, [0.75, 0.75, 0.75, 2.5], None, deploy)


def create_RepVGG_A1(deploy=False, num_classes=1000):
    return RepVGG(_A, num_classes, [1, 1, 1, 2.5], None, deploy)


def create_RepVGG_A2(deploy=False, num_classes=1000):
    return RepVGG(_A, num_classes, [1.5, 1.5, 1.5, 2.75], None, deploy)


def create_RepVGG_B0(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [1, 1, 1, 2.5], None, deploy)


def create_RepVGG_B1(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [2, 2, 2, 4], None, deploy)


def create_RepVGG_B1g2(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [2, 2, 2, 4], g2_map, deploy)


def create_RepVGG_B1g4(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [2, 2, 2, 4], g4_map, deploy)


def create_RepVGG_B2(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [2.5, 2.5, 2.5, 5], None, deploy)


def create_RepVGG_B2g2(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [2.5, 2.5, 2.5, 5], g2_map, deploy)


def create_RepVGG_B2g4(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [2.5, 2.5, 2.5, 5], g4_map, deploy)


def create_RepVGG_B3(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [3, 3, 3, 5], None, deploy)


def create_RepVGG_B3g2(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [3, 3, 3, 5], g2_map, deploy)


def create_RepVGG_B3g4(deploy=False, num_classes=1000):
    return RepVGG(_B, num_classes, [3, 3, 3, 5], g4_map, deploy)


def create_RepVGG_D2se(deploy=False, num_classes=1000):
    return RepVGG([8, 14, 24, 1], num_classes, [2.5, 2.5, 2.5, 5], None, deploy, use_se=True)


func_dict = {
    "RepVGG-A0": create_RepVGG_A0,
    "RepVGG-A1": create_RepVGG_A1,
    "RepVGG-A2": create_RepVGG_A2,
    "RepVGG-B0": create_RepVGG_B0,
    "RepVGG-B1": create_RepVGG_B1,
    "RepVGG-B1g2": create_RepVGG_B1g2,
    "RepVGG-B1g4": create_RepVGG_B1g4,
    "RepVGG-B2": create_RepVGG_B2,
    "RepVGG-B2g2": create_RepVGG_B2g2,
    "RepVGG-B2g4": create_RepVGG_B2g4,
    "RepVGG-B3": create_RepVGG_B3,
    "RepVGG-B3g2": create_RepVGG_B3g2,
    "RepVGG-B3g4": create_RepVGG_B3g4,
    "RepVGG-D2se": create_RepVGG_D2se,
}


def get_RepVGG_func_by_name(name):
    return func_dict[name]


def repvgg_model_convert(model: torch.nn.Module, save_path=None, do_copy=True):
    """Switch every block of ``model`` (or of a copy) to its deploy form; optionally save {"state_dict": ...}."""
    if do_copy:
        model = copy.deepcopy(model)
    for module in model.modules():
        if hasattr(module, "switch_to_deploy"):
            module.switch_to_deploy()
    if save_path is not None:
        torch.save({"state_dict": model.state_dict()}, save_path)
    return model
