"""Oracle: RepVGG (classification/RepVGG/models/repvgg.py) restated in fp32 PyTorch: the train form (three branches), the
deploy form (one biased 3x3 convolution per block) and the fold between them.  The GPU tests use it as their fp32 reference;
tests/golden/make_repvgg_golden.py pins it bit for bit against the reference's create_RepVGG_A0 / create_RepVGG_B0.

    block, train form:  relu(bn_d(conv3x3_s(x)) + bn_1(conv1x1_s(x)) + [bn_id(x) if in == out and s == 1])
    block, deploy form: relu(conv3x3_s(x) + b)
    fold:               K = W3 t3 + pad(W1 t1) + I t_id,  b = sum_b (beta_b - mean_b t_b),  t = gamma / sqrt(var + eps)
    network:            stage0 (3 -> min(64, 64 a0), s2), stage1..4 (first block s2), global average pool, linear
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

# name -> (blocks per stage, width multipliers) of the dense variants
ARCHS = {"RepVGG-A0": ([2, 4, 14, 1], [0.75, 0.75, 0.75, 2.5]), "RepVGG-A1": ([2, 4, 14, 1], [1, 1, 1, 2.5]),
         "RepVGG-A2": ([2, 4, 14, 1], [1.5, 1.5, 1.5, 2.75]), "RepVGG-B0": ([4, 6, 16, 1], [1, 1, 1, 2.5]),
         "RepVGG-B1": ([4, 6, 16, 1], [2, 2, 2, 4]), "RepVGG-B2": ([4, 6, 16, 1], [2.5, 2.5, 2.5, 5]),
         "RepVGG-B3": ([4, 6, 16, 1], [3, 3, 3, 5])}


def _branch(cin, cout, k, s):
    seq = nn.Sequential()
    seq.add_module("conv", nn.Conv2d(cin, cout, k, s, k // 2, bias=False))
    seq.add_module("bn", nn.BatchNorm2d(cout))
    return seq


class Block(nn.Module):
    def __init__(self, cin, cout, stride, deploy=False):
        super().__init__()
        self.nonlinearity = nn.ReLU()
        self.se = nn.Identity()
        if deploy:
            self.rbr_reparam = nn.Conv2d(cin, cout, 3, stride, 1, bias=True)
        else:
            self.rbr_identity = nn.BatchNorm2d(cin) if (cin == cout and stride == 1) else None
            self.rbr_dense = _branch(cin, cout, 3, stride)
            self.rbr_1x1 = _branch(cin, cout, 1, stride)

    def forward(self, x):
        if hasattr(self, "rbr_reparam"):
            return F.relu(self.rbr_reparam(x))
        # the identity branch is evaluated first, as in the reference: autograd then sums the three input gradients in
        # the same order, which keeps the gradients bit-identical
        ident = 0 if self.rbr_identity is None else self.rbr_identity(x)
        return F.relu(self.rbr_dense(x) + self.rbr_1x1(x) + ident)


class RepVGGOracle(nn.Module):
    def __init__(self, num_blocks, width_multiplier, num_classes=1000, deploy=False):
        super().__init__()
        c = min(64, int(64 * width_multiplier[0]))
        self.stage0 = Block(3, c, 2, deploy)
        widths = [int(64 * width_multiplier[0]), int(128 * width_multiplier[1]), int(256 * width_multiplier[2]),
                  int(512 * width_multiplier[3])]
        for i, (w, n) in enumerate(zip(widths, num_blocks), start=1):
            blocks = []
            for j in range(n):
                blocks.append(Block(c, w, 2 if j == 0 else 1, deploy))
                c = w
            setattr(self, f"stage{i}", nn.Sequential(*blocks))
        self.gap = nn.AdaptiveAvgPool2d(1)
        self.linear = nn.Linear(c, num_classes)

    def forward(self, x):
        for i in range(5):
            x = getattr(self, f"stage{i}")(x)
        return self.linear(torch.flatten(self.gap(x), 1))


def build(name, state=None, num_classes=1000, deploy=False):
    """The oracle of the dense variant ``name`` (a key of ARCHS), loaded with ``state`` (the reference's state_dict keys)."""
    num_blocks, wm = ARCHS[name]
    m = RepVGGOracle(num_blocks, wm, num_classes, deploy)
    if state is not None:
        m.load_state_dict(state)
    return m


def _fold_bn(kernel, bn):
    std = torch.sqrt(bn.running_var + bn.eps)
    return kernel * (bn.weight / std).view(-1, 1, 1, 1), bn.bias - bn.running_mean * bn.weight / std


def fold(block):
    """(K [O][I][3][3], b [O]) of the one biased 3x3 convolution equal to the train-form ``block`` in eval mode."""
    k, b = _fold_bn(block.rbr_dense.conv.weight, block.rbr_dense.bn)
    k1, b1 = _fold_bn(block.rbr_1x1.conv.weight, block.rbr_1x1.bn)
    k, b = k + F.pad(k1, [1, 1, 1, 1]), b + b1
    if block.rbr_identity is not None:
        C = block.rbr_identity.num_features
        eye = torch.zeros(C, C, 3, 3, dtype=k.dtype, device=k.device)
        eye[torch.arange(C), torch.arange(C), 1, 1] = 1.0
        ki, bi = _fold_bn(eye, block.rbr_identity)
        k, b = k + ki, b + bi
    return k, b


@torch.no_grad()
def convert(model):
    """A deploy-form copy of the train-form oracle ``model``: every block folded into its rbr_reparam."""
    import copy

    out = copy.deepcopy(model)
    for mod in out.modules():
        if isinstance(mod, Block) and not hasattr(mod, "rbr_reparam"):
            k, b = fold(mod)
            dense = mod.rbr_dense.conv
            mod.rbr_reparam = nn.Conv2d(dense.in_channels, dense.out_channels, 3, dense.stride, 1, bias=True)
            mod.rbr_reparam.weight.copy_(k)
            mod.rbr_reparam.bias.copy_(b)
            del mod.rbr_dense, mod.rbr_1x1, mod.rbr_identity
    return out
