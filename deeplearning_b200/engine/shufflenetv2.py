"""Forward / backward schedule of ShuffleNet v2 (classification/ShuffleNet/models/shufflenetv2.py) on the sm_90a kernels.

The whole network is ONE autograd node (common.apply).  Activations are NHWC bf16, parameters fp32.  An InvertedResidual
of branch width b runs as

    branch2   ca = 1x1 GEMM (BatchNorm statistics in the epilogue)  ->  d2 = depthwise3x3(relu(bn(ca))) with the BatchNorm
              + ReLU applied on load and d2's statistics in the same kernel  ->  a2 = bn(d2)  ->  c3 = 1x1 GEMM (statistics)
    branch1   (stride 2 only) d1 = depthwise3x3/2(x) (statistics)  ->  a1 = bn(d1)  ->  cb1 = 1x1 GEMM (statistics)
    tail      channel_shuffle(cat(u, relu(bn(c3))), 2) in one pass (b200_shufflev2_tail_fwd), u = x's passthrough half
              (stride 1) or relu(bn(cb1)) (stride 2)
    backward  the tail backward un-interleaves the output gradient into bn(c3)'s masked dz (and branch1's, or the
              passthrough gradient) with the BatchNorm sums  ->  finalize + apply  ->  GEMM wgrad / dgrad  ->  bn2 reduce
              (tail_bwd_reduce) + apply  ->  depthwise wgrad, and dgrad times relu'(bn(ca)) with that BatchNorm's sums  ->
              finalize + apply  ->  GEMM wgrad / dgrad.  At stride 2 the block input gradient is branch2's dgrad added in
              the epilogue of branch1's depthwise dgrad.

Layout (DESIGN.md, ShuffleNet v2): the two-group shuffle of cat(u, v) is the interleave out[2i] = u[i], out[2i+1] = v[i], so
its chunk(2) halves are P' = zip(u[:b/2], v[:b/2]) and Q' = zip(u[b/2:], v[b/2:]).
- A block followed by a stride-1 block writes its output split, as the two tensors (P', Q') [B, H, W, bp]: the next
  block's branch2 reads Q' as a plain GEMM operand and passes P' through; its input gradient is (dP, dQ).
- Any other block (the last of each stage) writes one joined tensor [B, H, W, J] in reference order, as the stem's
  max-pool output is; stride-2 blocks and conv5 read it whole.
- Branch tensors have a channel pitch bp = b rounded up to a multiple of 8, joined tensors J = 2b rounded up likewise.  Pad
  rows / columns of the operands are zero and the pad channels' BatchNorm coefficients are 0, so those channels stay
  exactly 0 through every pass.

The stem is shared with ShuffleNet v1 (engine/shufflenet_parts.py); conv5 is a GEMM, BatchNorm + ReLU and the global mean,
then the shared classifier head.  Eval mode runs the same passes with running-statistics coefficients and records no
statistics or tape.
"""
import sys
import weakref

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from . import common
from . import shufflenet_parts as parts
from .packing import weight_cache
from .shufflenet_parts import PaddedBN, check_bn, check_conv, pad8


# --------------------------------------------------------------------------------------------------------- admission
class _Block:
    """Layers of one InvertedResidual as the schedule uses them: stride s, branch width b (pitch bp), real input width cin
    and input pitch xp (stride 2: the joined input; stride 1: one half), and whether the output is written split."""
    __slots__ = ("name", "s", "b", "bp", "cin", "xp", "split", "b1_dw", "b1_bn1", "b1_conv", "b1_bn2", "conv1", "bn1", "dw",
                 "bn2", "conv2", "bn3")


def _check_seq(name, seq, layers):
    """``seq`` is a Sequential of len(layers) modules with nn.ReLU where ``layers`` says "ReLU" (the convolutions and
    BatchNorms are checked one by one)."""
    if (not isinstance(seq, nn.Sequential) or len(seq) != len(layers)
            or any((type(m) is nn.ReLU) != (kind == "ReLU") for m, kind in zip(seq, layers))):
        raise NotImplementedError(f"{name}: expected the reference's Sequential({', '.join(layers)}) (got {seq})")


def _check_block(name, blk, cin, stride):
    from ..classification.ShuffleNet.models.shufflenetv2 import InvertedResidual

    if type(blk) is not InvertedResidual:
        raise NotImplementedError(f"{name}: expected the reference's InvertedResidual (got {type(blk).__name__})")
    if blk.stride not in (1, 2):
        raise NotImplementedError(f"{name}: stride {blk.stride} is not implemented by the GPU engine (strides 1 and 2 are)")
    if blk.stride != stride:
        raise NotImplementedError(f"{name}: expected stride {stride} (the first block of a stage has stride 2, the others 1)")
    keys = list(blk._modules)
    if keys != ["branch1", "branch2"]:
        raise NotImplementedError(f"{name}: expected the reference's modules ['branch1', 'branch2'] (got {keys})")
    _check_seq(f"{name}.branch2", blk.branch2, ["Conv2d", "BatchNorm2d", "ReLU", "Conv2d", "BatchNorm2d", "Conv2d",
                                                "BatchNorm2d", "ReLU"])
    b = getattr(blk.branch2[0], "out_channels", 0)
    if b % 2 != 0 or b < 2:
        raise NotImplementedError(f"{name}: the GPU engine needs an even branch width (got {b}): the shuffled output is "
                                  "interleaved in channel pairs")
    k = _Block()
    k.name, k.s, k.b, k.bp, k.cin = name, stride, b, pad8(b), cin
    br2 = blk.branch2
    if stride == 2:
        k.xp = pad8(cin)
        br1 = blk.branch1
        _check_seq(f"{name}.branch1", br1, ["Conv2d", "BatchNorm2d", "Conv2d", "BatchNorm2d", "ReLU"])
        check_conv(f"{name}.branch1.0", br1[0], 3, 2, cin, cin, cin)
        check_bn(f"{name}.branch1.1", br1[1], cin)
        check_conv(f"{name}.branch1.2", br1[2], 1, 1, cin, b, 1)
        check_bn(f"{name}.branch1.3", br1[3], b)
        k.b1_dw, k.b1_bn1, k.b1_conv, k.b1_bn2 = br1[0], br1[1], br1[2], br1[3]
        check_conv(f"{name}.branch2.0", br2[0], 1, 1, cin, b, 1)
    else:
        if not isinstance(blk.branch1, nn.Sequential) or len(blk.branch1) != 0:
            raise NotImplementedError(f"{name}.branch1: expected the empty Sequential of a stride-1 block")
        if cin != 2 * b:
            raise NotImplementedError(f"{name}: a stride-1 block needs input width 2 x branch width (got {cin}, b={b})")
        k.xp = k.bp
        k.b1_dw = k.b1_bn1 = k.b1_conv = k.b1_bn2 = None
        check_conv(f"{name}.branch2.0", br2[0], 1, 1, b, b, 1)
    check_bn(f"{name}.branch2.1", br2[1], b)
    check_conv(f"{name}.branch2.3", br2[3], 3, stride, b, b, b)
    check_bn(f"{name}.branch2.4", br2[4], b)
    check_conv(f"{name}.branch2.5", br2[5], 1, 1, b, b, 1)
    check_bn(f"{name}.branch2.6", br2[6], b)
    k.conv1, k.bn1, k.dw, k.bn2, k.conv2, k.bn3 = br2[0], br2[1], br2[3], br2[4], br2[5], br2[6]
    k.split = False
    return k, 2 * b


def check_model(model):
    """Admission of a whole ShuffleNetV2, without touching a device: raises NotImplementedError naming the first layer the
    engine does not run (anything but the reference's structure or block class; stride 3; an odd branch width or a stem
    width that is not a multiple of 8; BatchNorm that is not affine or keeps no running statistics; SyncBatchNorm in a
    multi-rank job).  Returns (stem conv, stem bn, [_Block], conv5 conv, conv5 bn, fc)."""
    names = list(model._modules)
    if names != ["conv1", "maxpool", "stage2", "stage3", "stage4", "conv5", "fc"]:
        raise NotImplementedError(f"ShuffleNetV2: expected the modules conv1, maxpool, stage2..4, conv5, fc (got {names})")
    stem_conv, stem_bn, c0 = parts.check_stem(model)
    if c0 % 8 != 0:
        raise NotImplementedError(f"conv1: the GPU engine needs a stem width that is a multiple of 8 (got {c0})")
    blocks = []
    cin = c0
    for sname in ("stage2", "stage3", "stage4"):
        stage = model._modules[sname]
        if not isinstance(stage, nn.Sequential) or len(stage) < 1:
            raise NotImplementedError(f"{sname}: expected a Sequential of InvertedResiduals")
        for i, blk in enumerate(stage):
            k, cin = _check_block(f"{sname}.{i}", blk, cin, 2 if i == 0 else 1)
            blocks.append(k)
    for k, nxt in zip(blocks, blocks[1:]):
        k.split = nxt.s == 1
    c5 = model.conv5
    if not isinstance(c5, nn.Sequential) or len(c5) != 3 or type(c5[2]) is not nn.ReLU:
        raise NotImplementedError("conv5: expected the reference's Sequential(Conv2d, BatchNorm2d, ReLU)")
    n5 = getattr(c5[0], "out_channels", 0)
    check_conv("conv5.0", c5[0], 1, 1, cin, n5, 1)
    check_bn("conv5.1", c5[1], n5)
    if n5 % 8 != 0:
        raise NotImplementedError(f"conv5: the GPU engine needs a width that is a multiple of 8 (got {n5})")
    fc = model.fc
    if type(fc) is not nn.Linear or fc.in_features != n5:
        raise NotImplementedError(f"fc: expected a Linear over the {n5} features of conv5 (got {fc})")
    return stem_conv, stem_bn, blocks, c5[0], c5[1], fc


# ---------------------------------------------------------------------------------------------------------- packing
class _PackSpec:
    """bf16 operands packed by weight_cache: the stem's [C0][32] patch-matrix operand and the classifier."""

    def key(self, model):
        return (id(model.fc), model.fc.out_features, id(model.conv1[0].weight))

    def __call__(self, model):
        return [parts.stem_pack_spec(model.conv1[0])] + common.head_pack_specs(model.fc)


_pack_spec = _PackSpec()


def _fwd_operand(conv, xp, bp):
    """[bp][xp] forward operand of a 1x1 convolution whose input has pitch xp and output pitch bp."""
    return weight_cache.get(conv.weight, 0, ld=xp, pad_rows=bp)


def _dgrad_operand(conv, xp, bp):
    """[xp][bp] dgrad operand of the same convolution."""
    return weight_cache.get(conv.weight, 1, pad_cols=bp, pad_rows=xp)


class _Plan:
    """Per-model device state of the schedule: a PaddedBN for every BatchNorm whose tensor has pad channels."""

    def __init__(self, key, blocks, device):
        self.key, self.device = key, device
        self.padded = {}
        for k in blocks:
            widths = [(k.bn1, k.b, k.bp), (k.bn2, k.b, k.bp), (k.bn3, k.b, k.bp)]
            if k.s == 2:
                widths += [(k.b1_bn1, k.cin, k.xp), (k.b1_bn2, k.b, k.bp)]
            for bn, C, Cp in widths:
                if Cp != C:
                    self.padded[bn] = PaddedBN(bn, list(range(C)), Cp, device)

    def coeffs(self, bn, stats, rows, train):
        pbn = self.padded.get(bn)
        return pbn.coeffs(stats, rows, train) if pbn is not None else common.bn_coeffs(bn, stats, rows, train)

    def bn_backward(self, grads, bn, dz, partial, c, co):
        pbn = self.padded.get(bn)
        if pbn is not None:
            return pbn.backward(grads, dz, partial, c, co)
        return common.bn_backward_from_sums(grads, bn, dz, partial, c, co)


_plans = weakref.WeakKeyDictionary()


def _plan(model, blocks, device):
    key = tuple(id(bn) for k in blocks for bn in (k.bn1, k.bn2, k.bn3, k.b1_bn1, k.b1_bn2))
    plan = _plans.get(model)
    if plan is None or plan.key != key or plan.device != device:
        plan = _Plan(key, blocks, device)
        _plans[model] = plan
    return plan


def tail_layout(u, v, b, split):
    """The channel map of the tail kernels in plain PyTorch (any device and dtype; the tests' reference): u, v [..., bp]
    with b real channels -> the joined output [..., J], or with ``split`` the halves (P', Q') [..., bp], of
    channel_shuffle(cat(u[..., :b], v[..., :b]), 2) along the last dimension, pad channels 0."""
    z = torch.stack([u[..., :b], v[..., :b]], -1).flatten(-2)
    if split:
        bp = u.shape[-1]
        return F.pad(z[..., :b], (0, bp - b)), F.pad(z[..., b:], (0, bp - b))
    return F.pad(z, (0, pad8(2 * b) - 2 * b))


def _put_wgrad(grads, conv, dy, x):
    """Records the weight gradient of a 1x1 convolution from its padded output gradient dy and input x."""
    O, I = conv.out_channels, conv.in_channels
    dst = grads.dest(conv.weight)
    if dy.shape[-1] == O and x.shape[-1] == I:
        grads.put(conv.weight, ops.conv2d_wgrad(dy, x, 1, 1, out=dst))
        return
    g = ops.conv2d_wgrad(dy, x, 1, 1)[:O, :I]
    grads.put(conv.weight, g if dst is None else dst.copy_(g))


def _put_dw_wgrad(grads, conv, gw):
    C = conv.out_channels
    dst = grads.dest(conv.weight)
    grads.put(conv.weight, gw[:C] if dst is None else dst.copy_(gw[:C]))


# ---------------------------------------------------------------------------------------------------------- forward
def forward(model, x, train, want_tape):
    """x: fp32 NCHW (or decoded uint8 NHWC) CUDA batch.  Returns (logits fp32 [B, num_classes], tape or None)."""
    stem_conv, stem_bn, blocks, conv5, bn5, fc = check_model(model)
    x = common.image_input(model, x)
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
    pack = weight_cache.model_pack(model, _pack_spec)
    plan = _plan(model, blocks, x.device)
    tape = {"blocks": [], "pack": pack, "plan": plan} if (train and want_tape) else None
    h, saved = parts.stem_forward(pack, stem_conv, stem_bn, x, train)
    if tape is not None:
        tape["stem"] = saved
    for k in blocks:
        t = {}
        if k.s == 2:
            t["x"] = h
            t["wd1"] = wd1 = parts.padded_dw_weight(k.b1_dw, k.xp)
            t["d1"], st = ops.dw_fwd(h, wd1, 3, 2, want_stats=train)
            t["co_d1"] = plan.coeffs(k.b1_bn1, st, common.rows(t["d1"]), train)
            t["a1"] = ops.bn_apply(t["d1"], t["co_d1"], relu=False)
            t["cb1"], st = ops.conv2d_fwd(t["a1"], _fwd_operand(k.b1_conv, k.xp, k.bp), 1, 1, want_stats=train)
            t["co_b1"] = plan.coeffs(k.b1_bn2, st, common.rows(t["cb1"]), train)
            x2 = h
        else:
            t["x"] = x2 = h[1]
        t["ca"], st = ops.conv2d_fwd(x2, _fwd_operand(k.conv1, k.xp, k.bp), 1, 1, want_stats=train)
        t["co_a"] = plan.coeffs(k.bn1, st, common.rows(t["ca"]), train)
        t["wd2"] = wd2 = parts.padded_dw_weight(k.dw, k.bp)
        t["d2"], st = ops.dw_relu_fwd(t["ca"], wd2, k.s, t["co_a"], want_stats=train)
        t["co_d2"] = plan.coeffs(k.bn2, st, common.rows(t["d2"]), train)
        t["a2"] = ops.bn_apply(t["d2"], t["co_d2"], relu=False)
        t["c3"], st = ops.conv2d_fwd(t["a2"], _fwd_operand(k.conv2, k.bp, k.bp), 1, 1, want_stats=train)
        t["co3"] = plan.coeffs(k.bn3, st, common.rows(t["c3"]), train)
        if k.s == 2:
            h = ops.shufflev2_tail_fwd(t["cb1"], t["c3"], t["co3"], k.b, co_u=t["co_b1"], split=k.split)
        else:
            h = ops.shufflev2_tail_fwd(h[0], t["c3"], t["co3"], k.b, split=k.split)
        if tape is not None:
            tape["blocks"].append(t)
    x5 = h
    xp5 = x5.shape[-1]
    c5, st = ops.conv2d_fwd(x5, weight_cache.get(conv5.weight, 0, ld=xp5), 1, 1, want_stats=train)
    co5 = common.bn_coeffs(bn5, st, common.rows(c5), train)
    pooled = ops.avgpool_fwd(ops.bn_apply(c5, co5, relu=True))
    logits = common.head_forward(pack, fc, pooled)
    if tape is not None:
        tape["conv5"] = (x5, c5, co5)
        tape["head"] = (pooled, tuple(c5.shape[1:3]))
    return logits, tape


# --------------------------------------------------------------------------------------------------------- backward
def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    stem_conv, stem_bn, blocks, conv5, bn5, fc = check_model(model)
    grads = common.Grads(sink)
    pack, plan = tape["pack"], tape["plan"]

    pooled, hw = tape["head"]
    g = ops.avgpool_bwd(common.head_backward(grads, pack, fc, pooled, dlogits), hw)
    x5, c5, co5 = tape["conv5"]
    dz, part, _ = ops.shuffle_relu_bwd(g, c5, co=co5)
    dc5 = common.bn_backward_from_sums(grads, bn5, dz, part, c5, co5)
    _put_wgrad(grads, conv5, dc5, x5)
    g = ops.conv2d_dgrad(dc5, weight_cache.get(conv5.weight, 1, pad_rows=x5.shape[-1]), hw, 1, 1)
    for i in range(len(blocks) - 1, -1, -1):
        k, t = blocks[i], tape["blocks"][i]
        if k.s == 2:
            dz3, p3, dzb1, pb1 = ops.shufflev2_tail_bwd(g, t["c3"], t["co3"], k.b, cu=t["cb1"], co_u=t["co_b1"])
        else:
            dz3, p3, dP, _ = ops.shufflev2_tail_bwd(g, t["c3"], t["co3"], k.b)
        dc3 = plan.bn_backward(grads, k.bn3, dz3, p3, t["c3"], t["co3"])
        _put_wgrad(grads, k.conv2, dc3, t["a2"])
        da2 = ops.conv2d_dgrad(dc3, _dgrad_operand(k.conv2, k.bp, k.bp), tuple(t["a2"].shape[1:3]), 1, 1)
        _, part = ops.tail_bwd_reduce(da2, t["d2"])
        dd2 = plan.bn_backward(grads, k.bn2, da2, part, t["d2"], t["co_d2"])
        _put_dw_wgrad(grads, k.dw, ops.dw_relu_wgrad(dd2, t["ca"], k.s, t["co_a"]))
        dza, part = ops.dw_relu_dgrad(dd2, t["wd2"], t["ca"], k.s, t["co_a"])
        dca = plan.bn_backward(grads, k.bn1, dza, part, t["ca"], t["co_a"])
        x = t["x"]
        _put_wgrad(grads, k.conv1, dca, x)
        gx2 = ops.conv2d_dgrad(dca, _dgrad_operand(k.conv1, k.xp, k.bp), tuple(x.shape[1:3]), 1, 1)
        if k.s == 1:
            g = (dP, gx2)
            continue
        dcb1 = plan.bn_backward(grads, k.b1_bn2, dzb1, pb1, t["cb1"], t["co_b1"])
        _put_wgrad(grads, k.b1_conv, dcb1, t["a1"])
        da1 = ops.conv2d_dgrad(dcb1, _dgrad_operand(k.b1_conv, k.xp, k.bp), tuple(t["a1"].shape[1:3]), 1, 1)
        _, part = ops.tail_bwd_reduce(da1, t["d1"])
        dd1 = plan.bn_backward(grads, k.b1_bn1, da1, part, t["d1"], t["co_d1"])
        _put_dw_wgrad(grads, k.b1_dw, ops.dw_wgrad(dd1, x, 3, 2))
        g, _ = ops.dw_dgrad(dd1, t["wd1"], x, 3, 2, residual=gx2)
    parts.stem_backward(grads, stem_conv, stem_bn, g, tape["stem"])
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "ShuffleNetV2", model, x)
