"""Pieces shared by the ShuffleNet v1 and v2 schedules (engine/shufflenet.py, engine/shufflenetv2.py): layer admission,
the BatchNorm over a channel-padded tensor, the zero-padded depthwise weight, and the stem.

Both networks start with the same stem, conv1 = Conv 3x3/2 (3 -> C0) + BatchNorm + ReLU and a MaxPool2d(3, 2, 1).  It runs
as one GEMM over the im2col patch matrix of the image, then BatchNorm + ReLU + the max-pool in one pass; its backward is
the max-pool backward, the ReLU-masked reduce of shuffle_relu_bwd (mask from c * scale + shift), the BatchNorm backward
and the patch-matrix weight gradient.
"""
import torch
import torch.nn as nn

from .. import ops
from . import common

STEM_LDK = 32     # patch-matrix width of the 3x3 x 3-channel stem (27 columns, padded to a multiple of 8)


def pad8(n):
    return (n + 7) // 8 * 8


# --------------------------------------------------------------------------------------------------------- admission
def check_bn(name, bn, C):
    if not common.bn_ok(bn, C):
        raise NotImplementedError(f"{name}: expected an affine BatchNorm2d over {C} channels that tracks running statistics "
                                  f"(got {bn})")
    if common.bn_sync(bn) is not None:
        raise NotImplementedError(f"{name}: SyncBatchNorm in a multi-rank job is not implemented for ShuffleNet")


def check_conv(name, conv, k, stride, cin, cout, groups):
    if (type(conv) is not nn.Conv2d or conv.bias is not None or conv.dilation != (1, 1) or conv.padding_mode != "zeros"
            or conv.kernel_size != (k, k) or conv.stride != (stride, stride) or conv.padding != (k // 2, k // 2)
            or conv.in_channels != cin or conv.out_channels != cout or conv.groups != groups):
        raise NotImplementedError(f"{name}: expected a bias-free {k}x{k} Conv2d {cin} -> {cout}, stride {stride}, padding "
                                  f"{k // 2}, groups {groups} (got {conv})")


def check_stem(model):
    """Admission of conv1 = Sequential(Conv2d 3x3/2, BatchNorm2d, ReLU) and maxpool = MaxPool2d(3, 2, 1); returns
    (stem conv, stem bn, stem width)."""
    stem = model.conv1
    if not isinstance(stem, nn.Sequential) or len(stem) != 3 or type(stem[2]) is not nn.ReLU:
        raise NotImplementedError("conv1: expected the reference's Sequential(Conv2d, BatchNorm2d, ReLU)")
    c0 = getattr(stem[0], "out_channels", 0)
    check_conv("conv1.0", stem[0], 3, 2, 3, c0, 1)
    check_bn("conv1.1", stem[1], c0)
    mp = model.maxpool
    if (type(mp) is not nn.MaxPool2d or mp.kernel_size not in (3, (3, 3)) or mp.stride not in (2, (2, 2))
            or mp.padding not in (1, (1, 1)) or mp.dilation not in (1, (1, 1)) or mp.ceil_mode or mp.return_indices):
        raise NotImplementedError(f"maxpool: expected MaxPool2d(3, 2, 1) (got {mp})")
    return stem[0], stem[1], c0


# --------------------------------------------------------------------------------------------------- padded tensors
class PaddedBN:
    """A BatchNorm over a tensor stored with channel pitch Cp: stored channel n < b is the BatchNorm's channel src[n]; pad
    channels get gamma = beta = 0 (coefficients 0, so they stay 0).  Statistics, parameters and gradients of the real
    channels go to and from the module in its own order."""

    def __init__(self, bn, src, Cp, device):
        b = bn.num_features
        self.bn, self.b = bn, b
        idx = torch.full((Cp,), b, dtype=torch.int64)
        idx[:b] = torch.tensor(src, dtype=torch.int64)
        self.idx = idx.to(device)
        self.src = self.idx[:b]

    def _gather(self, v, fill):
        v = v.detach()
        return torch.cat([v, v.new_full((1,), fill)])[self.idx]

    def coeffs(self, stats, rows, train):
        bn = self.bn
        gamma, beta = self._gather(bn.weight, 0.0), self._gather(bn.bias, 0.0)
        rm, rv = self._gather(bn.running_mean, 0.0), self._gather(bn.running_var, 1.0)
        if not train:
            return ops.bn_eval_coeffs(gamma, beta, rm, rv, bn.eps)
        co = ops.bn_finalize(stats, rows, gamma, beta, bn.eps, bn.momentum, rm, rv, bn.num_batches_tracked)
        with torch.no_grad():
            bn.running_mean.index_copy_(0, self.src, rm[:self.b])
            bn.running_var.index_copy_(0, self.src, rv[:self.b])
        return co

    def scatter(self, v, out=None):
        """v fp32 [Cp] in stored order -> [b] in the module's order (into ``out`` when given)."""
        if out is None:
            out = torch.empty(self.b, dtype=v.dtype, device=v.device)
        return out.index_copy_(0, self.src, v[:self.b])

    def backward(self, grads, dz, partial, c, co):
        """dc of the train-mode BatchNorm from its masked gradient dz and partial sums; records the bias and then the
        weight gradient in the module's order."""
        dc, dg, db = ops.bn_backward_from_sums(dz, partial, c, co)
        grads.put(self.bn.bias, self.scatter(db, grads.dest(self.bn.bias)))
        grads.put(self.bn.weight, self.scatter(dg, grads.dest(self.bn.weight)))
        return dc


def padded_dw_weight(conv, Cp):
    """The depthwise weight [Cp, 1, k, k] fp32 of ``conv`` with zero pad channels."""
    w = conv.weight.detach()
    if Cp == w.shape[0]:
        return w.contiguous()
    return torch.cat([w, w.new_zeros(Cp - w.shape[0], *w.shape[1:])]).contiguous()


# ------------------------------------------------------------------------------------------------------------- stem
def stem_pack_spec(stem_conv):
    """engine.packing.ModelPack spec of the stem's [C0][STEM_LDK] patch-matrix operand."""
    return (stem_conv.weight, 0, STEM_LDK, stem_conv.out_channels)


def stem_forward(pack, stem_conv, stem_bn, x, train):
    """x fp32 NCHW [B, 3, H, W] -> (the max-pool output bf16 [B, H', W', C0], what stem_backward needs)."""
    B = x.shape[0]
    a, Ho, Wo = ops.im2col_nchw(x, 3, 3, 2, 1, ldk=STEM_LDK)
    patches = a.view(B, Ho, Wo, STEM_LDK)
    c_s, st = ops.conv2d_fwd(patches, pack.get(stem_conv.weight, 0), 1, 1, want_stats=train)
    co_s = common.bn_coeffs(stem_bn, st, common.rows(c_s), train)
    h, idx = ops.bn_relu_maxpool_fwd(c_s, co_s)
    return h, (patches, c_s, co_s, idx)


def stem_backward(grads, stem_conv, stem_bn, g, saved):
    """Records the stem's gradients from g = dL/d(max-pool output)."""
    patches, c_s, co_s, idx = saved
    g_act = ops.maxpool_bwd(g, idx, tuple(c_s.shape[1:3]))
    dz, part, _ = ops.shuffle_relu_bwd(g_act, c_s, co=co_s)
    dc = common.bn_backward_from_sums(grads, stem_bn, dz, part, c_s, co_s)
    C0 = c_s.shape[-1]
    gw = ops.conv2d_wgrad(dc, patches, 1, 1).view(C0, STEM_LDK)
    grads.put(stem_conv.weight, ops.stem_wgrad_relayout(gw, C0, 3, 9, out=grads.dest(stem_conv.weight)))
