"""Forward / backward schedule of the ResNet family on the sm_90a kernels.

The whole network is ONE autograd node (common.apply): forward runs conv(+BN statistics in the GEMM epilogue) -> finalize ->
apply(+ReLU)(+residual) per layer and records the tensors the backward needs on a tape; backward replays the tape with
BN-backward reduce/apply passes, wgmma dgrad and wgrad GEMMs.  Residual additions never get their own pass: the identity
gradient is added in the epilogue of the first conv's dgrad GEMM.

Mirrors ``ResNet._forward_impl`` / ``Bottleneck.forward`` / ``BasicBlock.forward`` of the reference
(classification/resnet/models/networks.py:204-220, :104-124, :59-75); activations are NHWC bf16, parameters fp32.

Bottleneck tail (conv3 1x1 -> bn3 -> + identity -> ReLU, :116-124) runs on the "algebra" path whenever conv3's input is
narrow (<= 256 channels; csrc/bn_algebra.cuh): train-mode BatchNorm is folded THROUGH the 1x1 convolution, so the 4x wider
conv3 output is never written, normalised or re-read -

    forward   G = y2^T y2, s = colsum(y2)  ->  batch statistics of conv3(y2)  ->  ONE GEMM: y = relu(acc*scale + shift + identity)
    backward  dz = relu'(y) * gradient comes out of the NEXT block's conv1 dgrad epilogue (mask + column sums);
              D = dz^T y2  ->  dgamma, dbeta, dW3, packed [a W3 | M] operand  ->  ONE GEMM over [dz | y2] gives dL/dy2

which removes the bn3 apply pass of the forward and both bn3 passes (reduce, apply) of the backward: 8 of the 17 passes a
bottleneck makes over its block-width tensors.  ``B200_RESNET_ALGEBRA=0`` selects the plain conv -> BN pass schedule.

A block with an ``se`` module (SEBottleneck / SEBasicBlock, classification/seNet/models/se_resnet.py:74-84 / :32-42) runs its
last unit as a squeeze-and-excitation tail (csrc/se.cuh) on the pass schedule under both settings:

    forward   c = conv(x) (+ statistics)  ->  squeeze: pool = mean_p bn(c)  ->  excite: gate = sigmoid(W2 relu(W1 pool))
              ->  y = relu(bn(c) * gate + identity)
    backward  reduce: dz = g * [y > 0], per-image sums of dz and dz * c  ->  SE / BN coefficients (dW1, dW2, dgamma, dbeta)
              ->  dc = BatchNorm backward of du = dz * gate + dpool / HW
"""
import os
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common
from .packing import weight_cache


_GROUP_WIDTHS = (4, 8, 16, 32, 64)


def _check_conv(conv, name):
    k = conv.kernel_size[0]
    if (conv.dilation != (1, 1) or conv.kernel_size[0] != conv.kernel_size[1] or conv.bias is not None
            or conv.padding != (k // 2, k // 2) or conv.stride[0] != conv.stride[1] or conv.stride[0] not in (1, 2)):
        raise NotImplementedError(f"{name}: only undilated k x k convolutions with pad=k//2, stride 1/2, no bias run on the "
                                  f"GPU engine (got {conv})")
    if conv.groups != 1:
        C = conv.in_channels
        if k != 3 or conv.out_channels != C or C % 64 != 0 or C // conv.groups not in _GROUP_WIDTHS:
            raise NotImplementedError(f"{name}: grouped convolutions run on the GPU engine as 3x3 with in_channels == "
                                      f"out_channels, a multiple of 64, and a group width in {_GROUP_WIDTHS} (got {conv})")


def _pack_modes(conv):
    """(forward, dgrad) packed-operand modes of a convolution weight (ops.pack_weight)."""
    return (3, 4) if conv.groups != 1 else (0, 1)


def _check_bn(bn, name):
    if (not isinstance(bn, (nn.BatchNorm2d, nn.SyncBatchNorm)) or not bn.affine or not bn.track_running_stats
            or bn.momentum is None):
        raise NotImplementedError(f"{name}: this engine implements affine nn.BatchNorm2d / nn.SyncBatchNorm with running "
                                  f"statistics (got {bn})")


def conv_pack_specs(net, stem):
    """Forward [O][taps*I] and dgrad [I][taps*O] bf16 operands of every convolution of ``net``; ``stem`` (the 7x7/2 stem
    convolution) gets the space-to-depth operand instead."""
    specs = []
    for mod in net.modules():
        if isinstance(mod, nn.Conv2d):
            w = mod.weight
            O, I, kh, kw = w.shape
            if mod is stem:
                specs.append((w, 2, 256, O, (O, I, kh * kw)))  # space-to-depth stem operand [64][256]
                continue
            if mod.groups != 1:   # block-diagonal operands of a grouped 3x3 convolution
                specs.append((w, 3, kh * kw * 64, O))
                specs.append((w, 4, kh * kw * 64, O))
                continue
            specs.append((w, 0, kh * kw * I, O))
            specs.append((w, 1, kh * kw * O, I))
    return specs


class _PackSpec:
    """Which bf16 operands a ResNet needs: forward [O][taps*I] and dgrad [I][taps*O] copies of every conv / fc weight."""

    @staticmethod
    def key(model):
        return (model.fc.out_features, id(model.fc))

    def __call__(self, model):
        return conv_pack_specs(model, model.conv1) + common.head_pack_specs(model.fc)


_pack_spec = _PackSpec()


class _Unit:
    """Saved state of one conv -> BN (-> ReLU) (-> + residual) application.  ``algebra`` units (bottleneck conv3 with the
    BatchNorm folded through the convolution) have no raw conv output ``c``; they keep the Gram matrix ``G`` and the column
    sums ``s`` of their input instead.  ``se`` holds (module, saved tensors) of a squeeze-and-excitation tail."""
    __slots__ = ("conv", "bn", "x", "c", "co", "y", "relu", "has_res", "algebra", "G", "s", "se")

    def __init__(self, conv, bn, x, c, co, y, relu, has_res, algebra=False, G=None, s=None, se=None):
        self.conv, self.bn, self.x, self.c, self.co, self.y = conv, bn, x, c, co, y
        self.relu, self.has_res, self.algebra, self.G, self.s, self.se = relu, has_res, algebra, G, s, se


def _algebra_enabled():
    return os.environ.get("B200_RESNET_ALGEBRA", "1") != "0"


def _algebra_ok(block, train, want_tape):
    """Bottleneck whose tail can run with bn3 folded through conv3 (train mode, or a forward that records no tape)."""
    if not _algebra_enabled() or not hasattr(block, "conv3") or not (train or not want_tape):
        return False
    if getattr(block, "se", None) is not None:   # the SE gate needs sum_p dz * u per image, hence the raw conv output
        return False
    if isinstance(block.bn3, nn.SyncBatchNorm) and train:
        return False
    c3, c1 = block.conv3, block.conv1
    return (c3.kernel_size == (1, 1) and c3.stride == (1, 1) and c3.groups == 1 and c3.bias is None and c3.dilation == (1, 1)
            and c3.in_channels % 64 == 0 and c3.in_channels <= 256 and c3.out_channels % 64 == 0
            and c1.kernel_size == (1, 1) and c1.stride == (1, 1) and c1.in_channels % 64 == 0 and c1.out_channels % 64 == 0)


def _conv3_bn_res_relu(pack, tape, y2, conv, bn, train, identity, name=""):
    """Algebra path of ``out = relu(bn3(conv3(y2)) + identity)``: statistics from the Gram matrix of y2, BN + add + ReLU in
    the GEMM epilogue."""
    _check_bn(bn, name)
    wp = pack.get(conv.weight, 0)
    G = s = None
    if train:
        G, s = ops.gram_colsum(y2)
        rows = y2.numel() // y2.shape[-1]
        co = ops.bn_gram_stats(G, s, wp, rows, bn.weight, bn.bias, bn.eps, bn.momentum, bn.running_mean, bn.running_var,
                               bn.num_batches_tracked)
    else:
        co = ops.bn_eval_coeffs(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
    y = ops.conv1x1_bn_act(y2, wp, co, identity)
    if tape is not None:
        tape.append(_Unit(conv, bn, y2, None, co, y, True, True, algebra=True, G=G, s=s))
    return y


def _ds_algebra_ok(block, train, want_tape):
    """Downsample branch (1x1 conv, stride 1 or 2 -> BatchNorm) of an algebra bottleneck that can run with its BatchNorm folded
    through the convolution too (train mode; input width <= 256)."""
    if not train or block.downsample is None or not _algebra_ok(block, train, want_tape):
        return False
    ds = block.downsample
    if len(ds) != 2 or not isinstance(ds[0], nn.Conv2d) or not isinstance(ds[1], nn.BatchNorm2d):
        return False
    c = ds[0]
    return (c.kernel_size == (1, 1) and c.stride in ((1, 1), (2, 2)) and c.groups == 1 and c.bias is None and c.padding == (0, 0)
            and c.in_channels % 64 == 0 and c.in_channels <= 256 and c.out_channels % 64 == 0)


def _ds_conv_bn_algebra(pack, tape, x_in, conv, bn, name=""):
    """identity = bn_ds(conv_ds(x_in)) with the batch statistics from the Gram matrix of the (compact) input: the raw conv output
    is never written.  A stride-2 branch runs on the compact copy of the even pixels it reads."""
    _check_bn(bn, name)
    xs = x_in if conv.stride == (1, 1) else ops.subsample2(x_in)
    wp = pack.get(conv.weight, 0)
    G, s = ops.gram_colsum(xs)
    rows = xs.numel() // xs.shape[-1]
    co = ops.bn_gram_stats(G, s, wp, rows, bn.weight, bn.bias, bn.eps, bn.momentum, bn.running_mean, bn.running_var,
                           bn.num_batches_tracked)
    ident = ops.conv1x1_bn(xs, wp, co)
    if tape is not None:
        tape.append(_Unit(conv, bn, xs, None, co, ident, False, False, algebra=True, G=G, s=s))
    return ident


def _conv_bn(pack, tape, x, conv, bn, train, relu, residual=None, name=""):
    _check_conv(conv, name)
    _check_bn(bn, name)
    k, s, g = conv.kernel_size[0], conv.stride[0], conv.groups
    wp = pack.get(conv.weight, _pack_modes(conv)[0])
    if not train and tape is None and conv.out_channels % 64 == 0 and _algebra_enabled():
        # eval forward (no tape): running statistics are constants, BatchNorm (+ identity) (+ ReLU) live in the conv epilogue
        co = ops.bn_eval_coeffs(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
        return ops.conv2d_bn_act(x, wp, co, k, s, relu=relu, residual=residual, groups=g)
    c, st = ops.conv2d_fwd(x, wp, k, s, want_stats=train, groups=g)
    co = common.bn_coeffs(bn, st, c.numel() // c.shape[-1], train)
    y = ops.bn_apply(c, co, relu=relu, residual=residual)
    if tape is not None:
        tape.append(_Unit(conv, bn, x, c, co, y, relu, residual is not None))
    return y


def _check_se(se, C, name):
    """SELayer(C, reduction) of the reference (classification/seNet/models/se_module.py:4-19): avg_pool, then
    fc = Linear(C, Cr, bias=False), ReLU, Linear(Cr, C, bias=False), Sigmoid, with C % 64 == 0 and 1 <= Cr <= 256."""
    fc, pool = getattr(se, "fc", None), getattr(se, "avg_pool", None)
    ok = (isinstance(pool, nn.AdaptiveAvgPool2d) and pool.output_size in (1, (1, 1))
          and isinstance(fc, nn.Sequential) and len(fc) == 4 and type(fc[0]) is nn.Linear and isinstance(fc[1], nn.ReLU)
          and type(fc[2]) is nn.Linear and isinstance(fc[3], nn.Sigmoid) and fc[0].bias is None and fc[2].bias is None)
    if ok:
        Cr = fc[0].out_features
        ok = (fc[0].in_features == C and fc[2].out_features == C and fc[2].in_features == Cr and C % 64 == 0
              and 1 <= Cr <= 256)
    if not ok:
        raise NotImplementedError(f"{name}: the GPU engine runs SELayer(C, reduction) as avg_pool -> Linear(C, Cr, bias=False) "
                                  f"-> ReLU -> Linear(Cr, C, bias=False) -> Sigmoid with C % 64 == 0 and 1 <= Cr <= 256 "
                                  f"on a {C}-channel tail (got {se})")


def _conv_bn_se(pack, tape, x, conv, bn, se, train, identity, name=""):
    """SE tail ``out = relu(bn(conv(x)) * gate + identity)``, gate = se(bn(conv(x))): conv (+ statistics) -> squeeze ->
    excite -> gated apply.  Eval mode runs the same kernels with the running-statistics coefficients."""
    _check_conv(conv, name)
    _check_bn(bn, name)
    _check_se(se, conv.out_channels, name)
    if train and common.bn_sync(bn) is not None:
        raise NotImplementedError(f"{name}: SyncBatchNorm in front of a squeeze-and-excitation gate is not implemented")
    wp = pack.get(conv.weight, _pack_modes(conv)[0])
    c, st = ops.conv2d_fwd(x, wp, conv.kernel_size[0], conv.stride[0], want_stats=train, groups=conv.groups)
    co = common.bn_coeffs(bn, st, c.numel() // c.shape[-1], train)
    csum, pool = ops.se_squeeze(c, co)
    h, gate = ops.se_excite(pool, se.fc[0].weight, se.fc[2].weight)
    y = ops.se_apply(c, co, gate, identity)
    if tape is not None:
        tape.append(_Unit(conv, bn, x, c, co, y, True, True, se=(se, csum, pool, h, gate)))
    return y


def _algebra_ok_dgrad(conv1):
    return (conv1.kernel_size == (1, 1) and conv1.stride == (1, 1) and conv1.in_channels % 64 == 0
            and conv1.out_channels % 64 == 0)


def _block_units(block):
    """(conv, bn) pairs of the residual branch, in order."""
    if hasattr(block, "conv3"):
        return [(block.conv1, block.bn1), (block.conv2, block.bn2), (block.conv3, block.bn3)]
    return [(block.conv1, block.bn1), (block.conv2, block.bn2)]


class Trunk:
    """Stem, stem BatchNorm and residual stages of a ResNet under the names its state_dict uses: the ResNet module itself
    (conv1, bn1, layer1 .. layer4), or the ``nn.Sequential`` of its children without ``fc`` that a SupCon encoder is
    (self-supervised/SupCon/models/model.py create_encoder: 0 = conv1, 1 = bn1, 2 = relu, 3 = maxpool, 4 .. 7 = layer1 ..
    layer4, 8 = avgpool).  ``prefix`` is the module's own name in error messages ("" for a ResNet)."""
    __slots__ = ("conv1", "bn1", "layers", "stem_name", "bn1_name", "layer_names")

    def __init__(self, net, prefix=""):
        if isinstance(net, nn.Sequential):
            kinds = (nn.Conv2d, nn.Module, nn.ReLU, nn.MaxPool2d, nn.Sequential, nn.Sequential, nn.Sequential, nn.Sequential,
                     nn.AdaptiveAvgPool2d)
            if len(net) != len(kinds) or not all(isinstance(m, k) for m, k in zip(net, kinds)):
                raise NotImplementedError(f"{prefix}: the GPU engine runs a ResNet trunk as the Sequential (conv1, bn1, relu, "
                                          f"maxpool, layer1 .. layer4, avgpool) of a ResNet's children without fc")
            self.conv1, self.bn1, self.layers = net[0], net[1], [net[i] for i in range(4, 8)]
            self.stem_name, self.bn1_name = f"{prefix}.0", f"{prefix}.1"
            self.layer_names = [f"{prefix}.{i}" for i in range(4, 8)]
        else:
            self.conv1, self.bn1 = net.conv1, net.bn1
            self.layers = [getattr(net, f"layer{li}") for li in range(1, 5)]
            self.stem_name, self.bn1_name = "stem", "bn1"
            self.layer_names = [f"layer{li}" for li in range(1, 5)]


def image_batch(x):
    """(x, (H, W), u8) of an image batch: an fp32 NCHW batch, or a decoded uint8 NHWC batch of the GPU input pipeline."""
    u8 = x.dtype == torch.uint8     # GPU input pipeline: decoded uint8 NHWC batch, ToTensor + Normalize fused into the stem operand
    if u8:
        if x.dim() != 4 or x.shape[3] != 3:
            raise ValueError(f"uint8 input must be a decoded NHWC batch [B,H,W,3], got {tuple(x.shape)}")
        x = x.contiguous()
        return x, (x.shape[1], x.shape[2]), True
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
    x = x.contiguous().float()
    return x, (x.shape[2], x.shape[3]), False


def trunk_forward(trunk, pack, x, x_hw, u8, train, want_tape, input_norm):
    """Stem through layer4 and the global average pool of ``trunk`` (a Trunk) on a batch from image_batch.
    Returns (pooled bf16 [B, F], tape or None).  ``train`` without ``want_tape`` runs train-mode BatchNorm (batch statistics,
    running statistics updated) and records nothing: the frozen encoder of SupCon's second stage."""
    B = x.shape[0]
    tape = {"stem": None, "blocks": [], "head": None, "pack": pack} if want_tape else None
    # ---- stem: 7x7/2 conv as a space-to-depth implicit GEMM, BN statistics in the epilogue, BN+ReLU+max-pool in one pass
    conv1, bn1 = trunk.conv1, trunk.bn1
    _check_bn(bn1, trunk.bn1_name)
    if conv1.kernel_size != (7, 7) or conv1.stride != (2, 2) or conv1.padding != (3, 3) or conv1.bias is not None:
        raise NotImplementedError(f"{trunk.stem_name} must be the 7x7/2 pad-3 bias-free convolution of the reference")
    if conv1.out_channels != 64 or x_hw[0] % 2 or x_hw[1] % 2:
        raise NotImplementedError(f"{trunk.stem_name}: 64 output channels and an even input size are required")
    # space-to-depth operand (108 MB at bs 256 instead of a 1 GB patch matrix); the conv reads it through overlapping TMA rows
    a = ops.stem_s2d_u8(x, *input_norm) if u8 else ops.stem_s2d(x)
    Ho, Wo = a.shape[1] - 3, a.shape[2] - 3
    c1, st = ops.stem_s2d_conv_fwd(a, pack.get(conv1.weight, 2), want_stats=train)
    co1 = common.bn_coeffs(bn1, st, B * Ho * Wo, train)
    h, idx = ops.bn_relu_maxpool_fwd(c1, co1)
    if want_tape:
        tape["stem"] = (a, c1, co1, idx, (Ho, Wo))
    # ---- residual stages
    for layer, lname in zip(trunk.layers, trunk.layer_names):
        for bi, block in enumerate(layer):
            units = [] if want_tape else None
            name = f"{lname}.{bi}"
            x_in = h
            pairs = _block_units(block)
            for j, (conv, bn) in enumerate(pairs[:-1]):
                h = _conv_bn(pack, units, h, conv, bn, train, relu=True, name=f"{name}.conv{j + 1}")
            ds_units = [] if want_tape else None
            if block.downsample is not None and _ds_algebra_ok(block, train, want_tape):
                identity = _ds_conv_bn_algebra(pack, ds_units, x_in, block.downsample[0], block.downsample[1],
                                               name=f"{name}.downsample")
            elif block.downsample is not None:
                identity = _conv_bn(pack, ds_units, x_in, block.downsample[0], block.downsample[1], train, relu=False,
                                    name=f"{name}.downsample")
            else:
                identity = x_in
            conv, bn = pairs[-1]
            se = getattr(block, "se", None)
            if se is not None:
                h = _conv_bn_se(pack, units, h, conv, bn, se, train, identity, name=f"{name}.conv{len(pairs)}")
            elif _algebra_ok(block, train, want_tape):
                _check_conv(conv, f"{name}.conv3")
                h = _conv3_bn_res_relu(pack, units, h, conv, bn, train, identity, name=f"{name}.conv3")
            else:
                h = _conv_bn(pack, units, h, conv, bn, train, relu=True, residual=identity, name=f"{name}.conv{len(pairs)}")
            if want_tape:
                tape["blocks"].append((units, ds_units[0] if ds_units else None, x_in))
    # ---- global average pool (bf16 features)
    pooled = ops.avgpool_fwd(h)
    if want_tape:
        tape["head"] = (pooled, h.shape[1:3])
    return pooled, tape


def forward(model, x, train, want_tape):
    """x: fp32 NCHW CUDA batch. Returns (logits fp32 [B, num_classes], tape or None)."""
    x, x_hw, u8 = image_batch(x)
    if not isinstance(model.fc, nn.Linear):
        raise NotImplementedError("model.fc must be an nn.Linear")
    pack = weight_cache.model_pack(model, _pack_spec)  # one launch repacks every bf16 operand if parameters changed
    pooled, tape = trunk_forward(Trunk(model), pack, x, x_hw, u8, train, want_tape,
                                 getattr(model, "input_norm", (ops.IMAGENET_MEAN, ops.IMAGENET_STD)))
    # ---- head: fc (fp32 logits)
    logits = common.head_forward(pack, model.fc, pooled)
    return logits, tape


def _unit_backward(u, g, grads, want_dz=False):
    """Backward of BN(+ReLU) of unit u for upstream gradient g; returns (dc, dz) and records BN param grads."""
    dc, dgamma, dbeta, dz = ops.bn_backward(g, u.c, u.co, relu=u.relu, y_out=u.y if (u.relu and u.has_res) else None,
                                            want_dz=want_dz, dgamma=grads.dest(u.bn.weight), dbeta=grads.dest(u.bn.bias),
                                            sync=common.bn_sync(u.bn))
    grads.put(u.bn.weight, dgamma)
    grads.put(u.bn.bias, dbeta)
    return dc, dz


def _se_unit_backward(u, g, grads):
    """Backward of an SE tail for the gradient g of its output; returns (dc, dz) like _unit_backward(want_dz=True) and
    records the gradients of the BatchNorm and of both SE weights."""
    se, csum, pool, h, gate = u.se
    w1, w2 = se.fc[0].weight, se.fc[2].weight
    dc, dz, dw1, dw2, dgamma, dbeta = ops.se_backward(
        g, u.y, u.c, u.co, csum, pool, h, gate, w1, w2, dw1=grads.dest(w1), dw2=grads.dest(w2),
        dgamma=grads.dest(u.bn.weight), dbeta=grads.dest(u.bn.bias))
    grads.put(w2, dw2)
    grads.put(w1, dw1)
    grads.put(u.bn.weight, dgamma)
    grads.put(u.bn.bias, dbeta)
    return dc, dz


def _fused_reduce_ok(u):
    """Can the dgrad GEMM that produces the gradient of unit u's output also do the reduce half of u's BN backward?
    (relu(bn(c)) without a residual, 64-channel multiples)"""
    return u.relu and not u.has_res and u.c.shape[-1] % 64 == 0


def _algebra_backward(u, dz, dz_stats, pack, grads):
    """Parameter gradients of an algebra unit (BatchNorm folded through its 1x1 convolution) from dz, the gradient of the
    BatchNorm output, and its column-sum partials; returns the packed operand ``wcat`` = [a W | M] and the bias ``wbias``
    of the ops.gemm_dual call over [dz | x] that gives the gradient of the unit's input."""
    D = ops.conv2d_wgrad(dz, u.x, 1, 1)                              # raw dz^T x [N, K, 1, 1]
    dgamma, dbeta, dW, wcat, wbias = ops.bn_conv1x1_bwd(
        dz_stats, D, u.G, u.s, pack.get(u.conv.weight, 0), u.conv.weight, dz.numel() // u.conv.out_channels, u.bn.weight,
        u.co, dgamma=grads.dest(u.bn.weight), dbeta=grads.dest(u.bn.bias), dW=grads.dest(u.conv.weight))
    grads.put(u.bn.weight, dgamma)
    grads.put(u.bn.bias, dbeta)
    grads.put(u.conv.weight, dW)
    return wcat, wbias


def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    grads = common.Grads(sink)
    pooled, _ = tape["head"]
    dpooled = common.head_backward(grads, tape["pack"], model.fc, pooled, dlogits)
    trunk_backward(Trunk(model), tape, dpooled, grads)
    return grads


def trunk_backward(trunk, tape, dpooled, grads):
    """Backward of trunk_forward for the gradient dpooled bf16 [B, F] of the pooled features; records every trunk
    parameter's gradient in ``grads`` (common.Grads)."""
    _, hw = tape["head"]
    pack = tape["pack"]
    g = ops.avgpool_bwd(dpooled, hw)

    # The gradient of a block output travels either as the raw gradient ``g`` (then the block masks it itself) or, when the
    # consumer's conv1 dgrad epilogue already applied this block's ReLU mask, as ``dz`` with its partial column sums.
    blocks = tape["blocks"]
    dz = dz_stats = None
    for bi in range(len(blocks) - 1, -1, -1):
        units, ds, x_in = blocks[bi]
        last = units[-1]
        has_ds = ds is not None
        if last.algebra:
            # out = relu(conv3(y2) * scale + shift + identity): BatchNorm backward folded through the 1x1 convolution
            if dz is None:
                dz, dz_stats = ops.relu_mask_sum(g, last.y)
            y2 = last.x
            wcat, wbias = _algebra_backward(last, dz, dz_stats, pack, grads)
            # dL/dy2 = [dz | y2] [a W3 | M]^T + k W3; its epilogue also masks with bn2's ReLU and sums for bn2's backward
            u2 = units[-2]
            if _fused_reduce_ok(u2):
                dz2, sums2 = ops.gemm_dual(dz, y2, wcat, wbias, bn_mask=(u2.c, u2.co))
                dc = common.bn_backward_from_sums(grads, u2.bn, dz2, sums2, u2.c, u2.co)
            else:
                g_prev = ops.gemm_dual(dz, y2, wcat, wbias)
                dc, _ = _unit_backward(u2, g_prev, grads)
            first = len(units) - 2
        elif last.se is not None:
            dc, dz = _se_unit_backward(last, g, grads)
            first = len(units) - 1
        else:
            # out = relu(bn_last(c) + identity): dz is the gradient of the pre-ReLU sum, shared by both branches
            dc, dz = _unit_backward(last, g, grads, want_dz=True)
            first = len(units) - 1
        # downsample branch on the algebra path: its data gradient gxs (on the compact even-pixel grid for stride 2) and all its
        # parameter gradients come from dz directly (no pass over a raw conv output, which does not exist)
        gxs = None
        if has_ds and ds.algebra:
            gxs = ops.gemm_dual(dz, ds.x, *_algebra_backward(ds, dz, dz_stats, pack, grads))
        # does the producer of x_in (the previous block) take its gradient pre-masked from this block's conv1 dgrad?
        prev_masked = (bi > 0 and not has_ds and blocks[bi - 1][0][-1].algebra and _algebra_ok_dgrad(units[0].conv))
        dz_prev = dz_prev_stats = None
        for j in range(first, -1, -1):
            u = units[j]
            k, s, gr = u.conv.kernel_size[0], u.conv.stride[0], u.conv.groups
            grads.put(u.conv.weight, ops.conv2d_wgrad(dc, u.x, k, s, out=grads.dest(u.conv.weight), groups=gr))
            wd = pack.get(u.conv.weight, _pack_modes(u.conv)[1])
            in_hw = tuple(u.x.shape[1:3])
            if j > 0 and s == 1 and _fused_reduce_ok(units[j - 1]):
                dzj, sumsj = ops.conv2d_dgrad(dc, wd, in_hw, k, s, bn_mask=(units[j - 1].c, units[j - 1].co), groups=gr)
                dc = common.bn_backward_from_sums(grads, units[j - 1].bn, dzj, sumsj, units[j - 1].c, units[j - 1].co)
            elif j > 0:
                g_prev = ops.conv2d_dgrad(dc, wd, in_hw, k, s, groups=gr)
                dc, _ = _unit_backward(units[j - 1], g_prev, grads)
            else:
                if has_ds and gxs is not None and ds.conv.stride == (1, 1):
                    gx = ops.conv2d_dgrad(dc, wd, in_hw, k, s, residual=gxs)   # + downsample-branch gradient (same grid)
                elif has_ds:
                    gx = ops.conv2d_dgrad(dc, wd, in_hw, k, s)
                    if gxs is not None:
                        ops.add_even_pixels_(gx, gxs)                            # stride-2 branch: onto the even pixels
                elif prev_masked:
                    # + identity-branch gradient, x_in's ReLU mask and the column sums the previous block needs, in the epilogue
                    dz_prev, dz_prev_stats = ops.conv1x1_dgrad_masked(dc, wd, residual=dz, mask_src=x_in)
                    gx = None
                else:
                    gx = ops.conv2d_dgrad(dc, wd, in_hw, k, s, residual=dz)  # + identity-branch gradient
        if has_ds and not ds.algebra:
            dcd, _ = _unit_backward(ds, dz, grads)
            kd, sd = ds.conv.kernel_size[0], ds.conv.stride[0]
            grads.put(ds.conv.weight, ops.conv2d_wgrad(dcd, x_in, kd, sd, out=grads.dest(ds.conv.weight)))
            wdd = pack.get(ds.conv.weight, 1)
            gx = ops.conv2d_dgrad(dcd, wdd, tuple(x_in.shape[1:3]), kd, sd, residual=gx, out=gx)
        g, dz, dz_stats = gx, dz_prev, dz_prev_stats

    a, c1, co1, idx, (Ho, Wo) = tape["stem"]
    g_act = ops.maxpool_bwd(g, idx, (Ho, Wo))
    bn1, conv1 = trunk.bn1, trunk.conv1
    dc, dgamma, dbeta, _ = ops.bn_backward(g_act, c1, co1, relu=True, sync=common.bn_sync(bn1), dgamma=grads.dest(bn1.weight),
                                           dbeta=grads.dest(bn1.bias))
    grads.put(bn1.weight, dgamma)
    grads.put(bn1.bias, dbeta)
    grads.put(conv1.weight, ops.stem_s2d_conv_wgrad(dc, a, out=grads.dest(conv1.weight)))


def apply(model, x):
    return common.apply(sys.modules[__name__], "ResNet", model, x)
