"""Forward / backward schedule of ShuffleNet v1 (classification/ShuffleNet/models/shufflenetv1.py) on the sm_90a kernels.

The whole network is ONE autograd node (common.apply).  Activations are NHWC bf16, parameters fp32.  A ResidualBlock runs as

    forward   c1 = group_conv1 GEMM (BatchNorm statistics in the epilogue)  ->  d = depthwise3x3(relu(bn1(c1))) with bn1 +
              ReLU applied on load and d's statistics in the same kernel  ->  a = bn2(d)  ->  c3 = group_conv GEMM
              (statistics)  ->  stride 1: y = relu(bn3(c3) + x);  stride 2: y = cat(relu(avg_pool(x)), relu(bn3(c3))),
              one pass writing the concatenated output
    backward  ReLU reduce (dz3 = g [y > 0], bn3's sums; stride 2 also writes the avg-pool backward gx in the same launch)
              ->  finalize + apply  ->  group_conv wgrad / dgrad (da)  ->  bn2 reduce (tail_bwd_reduce) + apply (dd)  ->
              depthwise wgrad, and dgrad times relu'(bn1(c1)) with bn1's sums  ->  finalize + apply  ->  group_conv1 wgrad,
              and dgrad with the shortcut gradient (dz3, or gx) added in its epilogue

Layout decisions (DESIGN.md section 3):
- The channel shuffle is a permutation of group_conv1's output channels; no pass runs it.  Stored channel n = c*g + j holds
  the reference's channel j*(b/g) + c, so the forward operand's rows are packed in that order and bn1's vectors are gathered
  the same way (running statistics and gradients scattered back).  After the shuffle, stored order is reference order.
- A grouped 1x1 convolution is the dense GEMM of a block-diagonal operand (zeros outside the groups): [Cout][Cin] forward,
  its transpose for dgrad.  Its weight gradient is the dense one with the in-group entries gathered.
- Bottleneck tensors have a channel pitch rounded up to a multiple of 8.  Pad rows / columns of the operands are zero and
  the pad channels' BatchNorm coefficients are 0, so those channels stay exactly 0 through every pass.

The stem is one GEMM over the im2col patch matrix of the image, then BatchNorm + ReLU + the 3x3/2 max-pool in one pass
(engine/shufflenet_parts.py, shared with ShuffleNet v2); the network ends with the global mean and the shared classifier head.  Eval mode runs the same passes with running-statistics
coefficients and records no statistics or tape.
"""
import sys
import weakref

import torch
import torch.nn as nn

from .. import ops
from . import common
from .packing import weight_cache
from .shufflenet_parts import PaddedBN, check_bn as _check_bn, check_conv as _check_conv, pad8 as _pad8
from . import shufflenet_parts as parts


# --------------------------------------------------------------------------------------------------------- admission
def _widths8(name, **widths):
    bad = {k: v for k, v in widths.items() if v % 8 != 0}
    if bad:
        raise NotImplementedError(f"{name}: the GPU engine needs stem, block and concat widths that are multiples of 8 "
                                  f"(got {', '.join(f'{k}={v}' for k, v in bad.items())}); pick a ratio that keeps them so")


class _Block:
    """Layers of one ResidualBlock as the schedule uses them: stride s, groups g, input width cin, bottleneck width b
    (pitch bp), conv-branch width cc (the block output is cin + cc wide at stride 2, cc at stride 1)."""
    __slots__ = ("name", "s", "g", "cin", "b", "bp", "cc", "conv1", "bn1", "dw", "bn2", "conv3", "bn3")


def _check_block(name, blk, cin, stride):
    from ..classification.ShuffleNet.models.shufflenetv1 import ResidualBlock

    if type(blk) is not ResidualBlock:
        raise NotImplementedError(f"{name}: expected the reference's ResidualBlock (got {type(blk).__name__})")
    if blk.stride != stride:
        raise NotImplementedError(f"{name}: expected stride {stride} (the first block of a stage has stride 2, the others 1)")
    keys = list(blk._modules)
    want = ["group_conv1", "bn1", "relu", "depthwise_conv3", "bn2", "group_conv", "bn3"]
    if stride == 2:
        want = ["avg_pool"] + want
    if keys != want:
        raise NotImplementedError(f"{name}: expected the reference's modules {want} (got {keys})")
    if type(blk.relu) is not nn.ReLU:
        raise NotImplementedError(f"{name}.relu: expected nn.ReLU (got {blk.relu})")
    if stride == 2:
        p = blk.avg_pool
        if (type(p) is not nn.AvgPool2d or p.kernel_size not in (3, (3, 3)) or p.stride not in (2, (2, 2))
                or p.padding not in (1, (1, 1)) or p.ceil_mode or not p.count_include_pad or p.divisor_override is not None):
            raise NotImplementedError(f"{name}.avg_pool: expected AvgPool2d(3, 2, 1) with count_include_pad (got {p})")
    b = getattr(blk.group_conv1, "out_channels", 0)
    cc = getattr(blk.group_conv, "out_channels", 0)
    g = blk.groups
    _check_conv(f"{name}.group_conv1", blk.group_conv1, 1, 1, cin, b, g)
    _check_bn(f"{name}.bn1", blk.bn1, b)
    _check_conv(f"{name}.depthwise_conv3", blk.depthwise_conv3, 3, stride, b, b, b)
    _check_bn(f"{name}.bn2", blk.bn2, b)
    _check_conv(f"{name}.group_conv", blk.group_conv, 1, 1, b, cc, g)
    _check_bn(f"{name}.bn3", blk.bn3, cc)
    if stride == 1 and cc != cin:
        raise NotImplementedError(f"{name}: a stride-1 block needs equal input and output widths (got {cin} -> {cc})")
    _widths8(name, input=cin, conv_branch=cc)
    k = _Block()
    k.name, k.s, k.g, k.cin, k.b, k.bp, k.cc = name, stride, g, cin, b, _pad8(b), cc
    k.conv1, k.bn1, k.dw, k.bn2, k.conv3, k.bn3 = (blk.group_conv1, blk.bn1, blk.depthwise_conv3, blk.bn2, blk.group_conv,
                                                  blk.bn3)
    return k, cin + cc if stride == 2 else cc


def check_model(model):
    """Admission of a whole ShuffleNetv1, without touching a device: raises NotImplementedError naming the first layer the
    engine does not run (anything but the reference's structure; stem, block or concat widths that are not multiples of
    8; BatchNorm that is not affine or keeps no running statistics; SyncBatchNorm in a multi-rank job).  Returns
    (stem conv, stem bn, [_Block], fc)."""
    names = list(model._modules)
    if names != ["conv1", "maxpool", "stage2", "stage3", "stage4", "fc"]:
        raise NotImplementedError(f"ShuffleNetv1: expected the modules conv1, maxpool, stage2..4, fc (got {names})")
    stem_conv, stem_bn, c0 = parts.check_stem(model)
    _widths8("conv1", stem=c0)
    blocks = []
    cin = c0
    for sname in ("stage2", "stage3", "stage4"):
        stage = model._modules[sname]
        if not isinstance(stage, nn.Sequential) or len(stage) < 1:
            raise NotImplementedError(f"{sname}: expected a Sequential of ResidualBlocks")
        for i, blk in enumerate(stage):
            k, cin = _check_block(f"{sname}.{i}", blk, cin, 2 if i == 0 else 1)
            blocks.append(k)
    fc = model.fc
    if type(fc) is not nn.Linear or fc.in_features != cin:
        raise NotImplementedError(f"fc: expected a Linear over the {cin} features of stage4 (got {fc})")
    return stem_conv, stem_bn, blocks, fc


# ---------------------------------------------------------------------------------------------------------- packing
class _PackSpec:
    """bf16 operands packed by weight_cache: the stem's [C0][32] patch-matrix operand and the classifier."""

    def key(self, model):
        return (id(model.fc), model.fc.out_features, id(model.conv1[0].weight))

    def __call__(self, model):
        stem = model.conv1[0]
        return [parts.stem_pack_spec(stem)] + common.head_pack_specs(model.fc)


_pack_spec = _PackSpec()


def shuffle_order(b, g):
    """Stored channel order of group_conv1's output: entry n is the reference channel stored at n (before the shuffle),
    n = c * g + j holding j * (b / g) + c, so that after shuffle_channels stored order is reference order."""
    bg = b // g
    return [(n % g) * bg + n // g for n in range(b)]


def dense_index(O, I, g, row_src, rows, cols):
    """int64 [rows][cols] index of the dense block-diagonal operand of a grouped 1x1 weight [O][I/g]: entry (n, i) is the
    flat weight index of output channel row_src[n] and input channel i when i lies in that channel's group, else O * I/g
    (the zero slot appended behind the weight).  Rows past len(row_src) and columns past I are padding (zero)."""
    Ig, Og = I // g, O // g
    idx = torch.full((rows, cols), O * Ig, dtype=torch.int64)
    for n, o in enumerate(row_src):
        go = o // Og
        idx[n, go * Ig:(go + 1) * Ig] = torch.arange(Ig) + o * Ig
    return idx


def gather_index(idx, numel):
    """int64 [numel]: for each weight element, its position in the flattened dense operand of ``idx`` (dense_index), so that
    dense_grad.flatten()[gather_index] is the grouped weight gradient."""
    flat = idx.flatten()
    live = flat < numel
    out = torch.empty(numel, dtype=torch.int64)
    out[flat[live]] = torch.nonzero(live).squeeze(1)
    return out


def dense_operand(w, idx):
    """fp32 dense [rows][cols] block-diagonal operand of the grouped 1x1 weight ``w`` through ``idx`` (dense_index)."""
    flat = w.detach().reshape(-1)
    return torch.cat([flat, flat.new_zeros(1)])[idx]


class _GroupedConv:
    """A grouped 1x1 convolution as a dense GEMM: index maps of its block-diagonal operand and of the weight-gradient
    gather, and the packed bf16 forward [rows][cols] / dgrad [cols][rows] operands, rebuilt when the weight changes."""

    def __init__(self, conv, row_src, rows, cols, device):
        self.w = conv.weight
        idx = dense_index(conv.out_channels, conv.in_channels, conv.groups, row_src, rows, cols)
        self.idx = idx.to(device)
        self.widx = gather_index(idx, conv.weight.numel()).to(device)
        self.stamp = None
        self.fwd = self.dgrad = None

    def operands(self):
        w = self.w
        stamp = (w._version, w.data_ptr(), weight_cache.generation)
        if stamp != self.stamp:
            dense = dense_operand(w, self.idx)
            self.fwd, self.dgrad = ops.pack_weight(dense, 0), ops.pack_weight(dense, 1)
            self.stamp = stamp
        return self.fwd, self.dgrad

    def weight_grad(self, dense_grad, out=None):
        """The grouped weight gradient from the dense one ([rows][cols] fp32), written into ``out`` when given."""
        g = dense_grad.reshape(-1)[self.widx].view(self.w.shape)
        if out is None:
            return g
        return out.copy_(g)


class _Plan:
    """Per-model device state of the schedule: the grouped convolutions and padded BatchNorms of every block."""

    def __init__(self, blocks, device):
        self.key = tuple((id(k.conv1.weight), id(k.conv3.weight), id(k.bn1), id(k.bn2)) for k in blocks)
        self.device = device
        self.conv1, self.conv3, self.bn1, self.bn2 = [], [], [], []
        for k in blocks:
            order = shuffle_order(k.b, k.g)
            self.conv1.append(_GroupedConv(k.conv1, order, k.bp, k.cin, device))
            self.conv3.append(_GroupedConv(k.conv3, list(range(k.cc)), k.cc, k.bp, device))
            self.bn1.append(PaddedBN(k.bn1, order, k.bp, device))
            self.bn2.append(PaddedBN(k.bn2, list(range(k.b)), k.bp, device))


_plans = weakref.WeakKeyDictionary()


def _plan(model, blocks, device):
    plan = _plans.get(model)
    key = tuple((id(k.conv1.weight), id(k.conv3.weight), id(k.bn1), id(k.bn2)) for k in blocks)
    if plan is None or plan.key != key or plan.device != device:
        plan = _Plan(blocks, device)
        _plans[model] = plan
    return plan


# ---------------------------------------------------------------------------------------------------------- forward
def forward(model, x, train, want_tape):
    """x: fp32 NCHW (or decoded uint8 NHWC) CUDA batch.  Returns (logits fp32 [B, num_classes], tape or None)."""
    stem_conv, stem_bn, blocks, fc = check_model(model)
    x = common.image_input(model, x)
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
    pack = weight_cache.model_pack(model, _pack_spec)
    plan = _plan(model, blocks, x.device)
    tape = {"blocks": [], "pack": pack, "plan": plan} if (train and want_tape) else None
    h, saved = parts.stem_forward(pack, stem_conv, stem_bn, x, train)
    if tape is not None:
        tape["stem"] = saved
    for i, k in enumerate(blocks):
        w1, _ = plan.conv1[i].operands()
        w3, _ = plan.conv3[i].operands()
        c1, st = ops.conv2d_fwd(h, w1, 1, 1, want_stats=train)
        co1 = plan.bn1[i].coeffs(st, common.rows(c1), train)
        wd = parts.padded_dw_weight(k.dw, k.bp)
        d, st = ops.dw_relu_fwd(c1, wd, k.s, co1, want_stats=train)
        co2 = plan.bn2[i].coeffs(st, common.rows(d), train)
        a = ops.bn_apply(d, co2, relu=False)
        c3, st = ops.conv2d_fwd(a, w3, 1, 1, want_stats=train)
        co3 = common.bn_coeffs(k.bn3, st, common.rows(c3), train)
        y = ops.bn_apply(c3, co3, relu=True, residual=h) if k.s == 1 else ops.shuffle_tail_s2_fwd(h, c3, co3)
        if tape is not None:
            tape["blocks"].append((h, c1, co1, wd, d, co2, a, c3, co3, y))
        h = y
    pooled = ops.avgpool_fwd(h)
    logits = common.head_forward(pack, fc, pooled)
    if tape is not None:
        tape["head"] = (pooled, tuple(h.shape[1:3]))
    return logits, tape


# --------------------------------------------------------------------------------------------------------- backward
def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    stem_conv, stem_bn, blocks, fc = check_model(model)
    grads = common.Grads(sink)
    pack, plan = tape["pack"], tape["plan"]

    pooled, hw = tape["head"]
    g = ops.avgpool_bwd(common.head_backward(grads, pack, fc, pooled, dlogits), hw)
    for i in range(len(blocks) - 1, -1, -1):
        k = blocks[i]
        x, c1, co1, wd, d, co2, a, c3, co3, y = tape["blocks"][i]
        if k.s == 1:
            dz3, part, _ = ops.shuffle_relu_bwd(g, c3, y=y)
            shortcut = dz3
        else:
            dz3, part, shortcut = ops.shuffle_relu_bwd(g, c3, y=y, in_hw=tuple(x.shape[1:3]))
        dc3 = common.bn_backward_from_sums(grads, k.bn3, dz3, part, c3, co3)
        gc3 = plan.conv3[i]
        grads.put(k.conv3.weight, gc3.weight_grad(ops.conv2d_wgrad(dc3, a, 1, 1), grads.dest(k.conv3.weight)))
        da = ops.conv2d_dgrad(dc3, gc3.operands()[1], tuple(a.shape[1:3]), 1, 1)
        _, part = ops.tail_bwd_reduce(da, d)
        dd = plan.bn2[i].backward(grads, da, part, d, co2)
        gw = ops.dw_relu_wgrad(dd, c1, k.s, co1)
        gwd = grads.dest(k.dw.weight)
        gw = gw[:k.b] if gwd is None else gwd.copy_(gw[:k.b])
        grads.put(k.dw.weight, gw)
        dz1, part = ops.dw_relu_dgrad(dd, wd, c1, k.s, co1)
        dc1 = plan.bn1[i].backward(grads, dz1, part, c1, co1)
        gc1 = plan.conv1[i]
        grads.put(k.conv1.weight, gc1.weight_grad(ops.conv2d_wgrad(dc1, x, 1, 1), grads.dest(k.conv1.weight)))
        g = ops.conv2d_dgrad(dc1, gc1.operands()[1], tuple(x.shape[1:3]), 1, 1, residual=shortcut)
    parts.stem_backward(grads, stem_conv, stem_bn, g, tape["stem"])
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "ShuffleNetv1", model, x)
