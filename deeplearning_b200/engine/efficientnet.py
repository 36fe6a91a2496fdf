"""Forward / backward schedule of EfficientNet (classification/efficientNet/models/network.py) on the sm_90a kernels.

The whole network is ONE autograd node (common.apply).  Activations are NHWC bf16, parameters fp32.  An MBConv block runs as

    forward   c_e = expand GEMM (BatchNorm statistics in the epilogue)  ->  d = depthwise(silu(bn_e(c_e))) with the BatchNorm
              + SiLU applied on load and d's statistics in the same kernel (the expanded activation is never stored)  ->
              pool = mean_p silu(bn_d(d))  ->  gate = excite(pool) (fp32, biased)  ->  a = silu(bn_d(d)) * gate  ->
              c_p = project GEMM (statistics)  ->  y = bn_p(c_p) * r_b (+ x), r_b the per-sample drop-connect multiplier
    backward  tail reduce (dz = g r_b)  ->  finalize + apply  ->  project wgrad / dgrad (da)  ->  gate reduce + excite
              backward (SE parameter gradients, dpool)  ->  SiLU-BN reduce (dz = (da gate + dpool / HW) silu'(u))  ->
              finalize + apply (dd)  ->  depthwise wgrad and dgrad (x silu'(u_e) with the expand BatchNorm's sums)  ->
              finalize + apply  ->  expand wgrad, and expand dgrad with the identity gradient added in its epilogue

An expand-ratio-1 block has no expand GEMM: its depthwise reads the stem's raw output with the stem BatchNorm + SiLU applied
on load (block 1a), or the previous block's y as is.  The stem is one GEMM over the im2col patch matrix of the image.  The
top 1x1 GEMM writes statistics, and the squeeze pass yields mean_p silu(bn(c_top)) times the classifier-dropout mask, the
bf16 [B, F] input of the shared head.

Eval mode runs the same passes with running-statistics coefficients (bn_eval_coeffs) and records no statistics, masks or
tape.  Drop-connect draws come from engine.droppath.sample_scale; the classifier-dropout mask is drawn with F.dropout on an
fp32 [B, F] tensor of ones in place, which consumes the generator exactly as the reference's ``nn.Dropout(p, inplace=True)``
on the pooled features does.  ``dropout_replay`` / ``dropout_record`` (engine.common, shared with VGG) are the mask's test
hooks, as droppath.replay / record are for the drop-connect multipliers.
"""
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common, droppath
from .common import dropout_record, dropout_replay  # noqa: F401  (the classifier-dropout test hooks)
from .packing import weight_cache

_STEM_LDK = 32     # patch-matrix width of the 3x3 x 3-channel stem (27 columns, padded to a multiple of 8)
_MAX_CR = 256      # widest SE squeeze the excite kernels take

# --------------------------------------------------------------------------------------------------------- admission
def _conv_bn_act(name, seq, k, stride, cin, cout, groups, act):
    """Checks a ConvBNAction (conv, bn, act); returns (conv, bn)."""
    def no(why):
        raise NotImplementedError(f"{name}: {why} (got {seq})")

    if not isinstance(seq, nn.Sequential) or len(seq) != 3:
        no("expected the reference's ConvBNAction (Conv2d, BatchNorm2d, activation)")
    conv, bn, a = seq[0], seq[1], seq[2]
    if type(conv) is not nn.Conv2d or conv.bias is not None or conv.dilation != (1, 1) or conv.padding_mode != "zeros":
        no("expected a bias-free Conv2d")
    if conv.kernel_size != (k, k) or conv.padding != (k // 2, k // 2) or conv.stride != (stride, stride):
        no(f"expected a {k}x{k} convolution with stride {stride} and padding {k // 2}")
    if (cin is not None and conv.in_channels != cin) or conv.out_channels != cout or conv.groups != groups:
        no("channel counts do not follow the block structure")
    if not common.bn_ok(bn, cout):
        no("expected an affine BatchNorm2d that tracks running statistics")
    if common.bn_sync(bn) is not None:
        no("SyncBatchNorm in a multi-rank job is not implemented for EfficientNet")
    if type(a) is not act:
        no(f"the GPU engine runs this layer with {act.__name__}")
    return conv, bn


class _Block:
    """Layers of one MBConv block as the schedule uses them."""
    __slots__ = ("name", "blk", "exp", "exp_bn", "dw", "dw_bn", "fc1", "fc2", "proj", "proj_bn", "k", "s", "res", "drop")


def _check_block(name, blk, cin):
    from ..classification.efficientNet.models.network import DropPath, MBConv, SELayer

    def no(why):
        raise NotImplementedError(f"{name}: {why}")

    if not isinstance(blk, MBConv) or not isinstance(getattr(blk, "block", None), nn.Sequential):
        no("expected the reference's MBConv block")
    keys = list(blk.block._modules)
    if keys not in (["expand_conv", "dwconv", "se", "project_conv"], ["dwconv", "se", "project_conv"]):
        no(f"the GPU engine runs MBConv blocks with [expand_conv,] dwconv, se, project_conv (got {keys}); a block without "
           f"SE is not implemented")
    b = _Block()
    b.name, b.blk = name, blk
    ce = cin
    b.exp = b.exp_bn = None
    if "expand_conv" in keys:
        conv = blk.block.expand_conv[0] if isinstance(blk.block.expand_conv, nn.Sequential) else None
        ce = getattr(conv, "out_channels", 0)
        b.exp, b.exp_bn = _conv_bn_act(f"{name}.expand_conv", blk.block.expand_conv, 1, 1, cin, ce, 1, nn.SiLU)
    dw = blk.block.dwconv
    conv = dw[0] if isinstance(dw, nn.Sequential) and len(dw) == 3 else None
    k = conv.kernel_size[0] if isinstance(conv, nn.Conv2d) else 0
    s = conv.stride[0] if isinstance(conv, nn.Conv2d) else 0
    if k not in (3, 5) or s not in (1, 2):
        no(f"the GPU engine runs depthwise convolutions of kernel size 3 or 5 at stride 1 or 2 (got {conv})")
    b.dw, b.dw_bn = _conv_bn_act(f"{name}.dwconv", dw, k, s, ce, ce, ce, nn.SiLU)
    se = blk.block.se
    fc = getattr(se, "fc", None)
    if (type(se) is not SELayer or not isinstance(fc, nn.Sequential) or len(fc) != 4 or type(fc[0]) is not nn.Conv2d
            or type(fc[1]) is not nn.SiLU or type(fc[2]) is not nn.Conv2d or type(fc[3]) is not nn.Sigmoid):
        no("expected the reference's SELayer (Conv2d, SiLU, Conv2d, Sigmoid)")
    cr = fc[0].out_channels
    for c, (i, o) in ((fc[0], (ce, cr)), (fc[2], (cr, ce))):
        if (c.in_channels, c.out_channels) != (i, o) or c.kernel_size != (1, 1) or c.groups != 1 or c.bias is None:
            no("SE convolutions must be biased 1x1 convolutions between the expanded width and the squeeze width")
    if not 1 <= cr <= _MAX_CR:
        no(f"the SE squeeze width must be in [1, {_MAX_CR}] (got {cr})")
    b.fc1, b.fc2 = fc[0], fc[2]
    conv = blk.block.project_conv[0] if isinstance(blk.block.project_conv, nn.Sequential) else None
    cout = getattr(conv, "out_channels", 0)
    b.proj, b.proj_bn = _conv_bn_act(f"{name}.project_conv", blk.block.project_conv, 1, 1, ce, cout, 1, nn.Identity)
    for c in (cin, ce, cout):
        if c % 8 != 0:
            no(f"channel counts must be multiples of 8 (got {cin} -> {ce} -> {cout})")
    b.res = bool(blk.use_res_connect)
    if b.res != (s == 1 and cin == cout):
        no("use_res_connect must hold exactly for stride-1 blocks with in_channels == out_channels")
    if isinstance(blk.dropout, DropPath):
        b.drop = float(blk.dropout.drop_prob or 0.0)
    elif isinstance(blk.dropout, nn.Identity):
        b.drop = 0.0
    else:
        no("dropout must be the reference's DropPath or nn.Identity")
    if b.drop > 0 and not b.res:
        no("drop-connect applies to residual blocks only")
    b.k, b.s = k, s
    return b, cout


def check_model(model):
    """Admission of a whole EfficientNet, without touching a device: raises NotImplementedError naming the first layer the
    engine does not run (anything but the reference's structure, depthwise kernels other than 3 / 5 or strides other than
    1 / 2, channel counts that are not multiples of 8, blocks without SE or with a non-SiLU activation, a shortcut around
    the first block, SyncBatchNorm in a multi-rank job).  Returns (stem conv, stem bn, [_Block], top conv, top bn, dropout p, head)."""
    feats = getattr(model, "features", None)
    if not isinstance(feats, nn.Sequential) or len(feats) < 3:
        raise NotImplementedError("features: expected the reference's Sequential(stem_conv, MBConv blocks..., top)")
    names = list(feats._modules)
    if names[0] != "stem_conv" or names[-1] != "top":
        raise NotImplementedError(f"features: expected stem_conv first and top last (got {names[0]}, {names[-1]})")
    stem = feats.stem_conv
    c0 = getattr(stem[0], "out_channels", 0) if isinstance(stem, nn.Sequential) and len(stem) else 0
    stem_conv, stem_bn = _conv_bn_act("features.stem_conv", stem, 3, 2, 3, c0, 1, nn.SiLU)
    if c0 % 8 != 0:
        raise NotImplementedError(f"features.stem_conv: channel counts must be multiples of 8 (got {c0})")
    blocks = []
    cin = c0
    for name in names[1:-1]:
        b, cin = _check_block(f"features.{name}", feats._modules[name], cin)
        if not blocks and b.exp is not None:
            raise NotImplementedError(f"features.{name}: the first block must have expand ratio 1 (it reads the stem's "
                                      f"BatchNorm + SiLU on load)")
        if not blocks and b.res:
            # its shortcut would be silu(bn(stem)), which the schedule never materialises (width coefficients below ~0.37
            # give the first block equal input and output widths)
            raise NotImplementedError(f"features.{name}: a shortcut around the first block (in_channels == out_channels, "
                                      f"stride 1) is not implemented on the GPU engine")
        blocks.append(b)
    top = feats.top
    cf = getattr(top[0], "out_channels", 0) if isinstance(top, nn.Sequential) and len(top) else 0
    top_conv, top_bn = _conv_bn_act("features.top", top, 1, 1, cin, cf, 1, nn.SiLU)
    if cf % 8 != 0:
        raise NotImplementedError(f"features.top: channel counts must be multiples of 8 (got {cf})")
    if not isinstance(getattr(model, "avgpool", None), nn.AdaptiveAvgPool2d) or model.avgpool.output_size not in (1, (1, 1)):
        raise NotImplementedError("avgpool: the GPU engine runs EfficientNet with AdaptiveAvgPool2d(1)")
    cls = getattr(model, "classifier", None)
    mods = list(cls) if isinstance(cls, nn.Sequential) else []
    p = 0.0
    if len(mods) == 2 and type(mods[0]) is nn.Dropout:
        p = float(mods[0].p)
        mods = mods[1:]
    if len(mods) != 1 or type(mods[0]) is not nn.Linear or mods[0].in_features != cf:
        raise NotImplementedError("classifier: expected the reference's [Dropout,] Linear")
    return stem_conv, stem_bn, blocks, top_conv, top_bn, p, mods[0]


# ---------------------------------------------------------------------------------------------------------- packing
class _PackSpec:
    """bf16 operands: forward [O][I] / dgrad [I][O] copies of every 1x1 convolution (expand, project, top), the stem's
    [C0][32] patch-matrix operand and the classifier."""

    @staticmethod
    def _convs(model):
        stem_conv, _, blocks, top_conv, _, _, head = check_model(model)
        convs = []
        for b in blocks:
            convs += ([b.exp] if b.exp is not None else []) + [b.proj]
        return stem_conv, convs + [top_conv], head

    def key(self, model):
        stem, convs, head = self._convs(model)
        return (id(head), head.out_features, id(stem.weight), tuple(id(c.weight) for c in convs))

    def __call__(self, model):
        stem, convs, head = self._convs(model)
        specs = [(stem.weight, 0, _STEM_LDK, stem.out_channels)]
        for c in convs:
            O, I = c.out_channels, c.in_channels
            specs += [(c.weight, 0, I, O), (c.weight, 1, O, I)]
        return specs + common.head_pack_specs(head)


_pack_spec = _PackSpec()


# ---------------------------------------------------------------------------------------------------------- forward
def forward(model, x, train, want_tape):
    """x: fp32 NCHW (or decoded uint8 NHWC) CUDA batch.  Returns (logits fp32 [B, num_classes], tape or None)."""
    stem_conv, stem_bn, blocks, top_conv, top_bn, p, head = check_model(model)
    x = common.image_input(model, x)
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
    pack = weight_cache.model_pack(model, _pack_spec)
    tape = {"blocks": [], "pack": pack} if (train and want_tape) else None
    B = x.shape[0]
    a, Ho, Wo = ops.im2col_nchw(x, 3, 3, 2, 1, ldk=_STEM_LDK)
    patches = a.view(B, Ho, Wo, _STEM_LDK)
    c_s, st = ops.conv2d_fwd(patches, pack.get(stem_conv.weight, 0), 1, 1, want_stats=train)
    co_s = common.bn_coeffs(stem_bn, st, common.rows(c_s), train)
    if tape is not None:
        tape["stem"] = (patches, c_s, co_s)
    h = None
    for i, b in enumerate(blocks):
        if b.exp is not None:
            c_e, st = ops.conv2d_fwd(h, pack.get(b.exp.weight, 0), 1, 1, want_stats=train)
            co_e = common.bn_coeffs(b.exp_bn, st, common.rows(c_e), train)
            dw_in, dw_co = c_e, co_e
        else:
            c_e = co_e = None
            dw_in, dw_co = (c_s, co_s) if i == 0 else (h, None)
        d, st = ops.dw_fwd(dw_in, b.dw.weight, b.k, b.s, co=dw_co, want_stats=train)
        co_d = common.bn_coeffs(b.dw_bn, st, common.rows(d), train)
        pool, _ = ops.silu_bn_squeeze(d, co_d)
        hpre, gate = ops.excite_fwd(pool, b.fc1.weight, b.fc1.bias, b.fc2.weight, b.fc2.bias)
        a = ops.gate_apply(d, co_d, gate)
        c_p, st = ops.conv2d_fwd(a, pack.get(b.proj.weight, 0), 1, 1, want_stats=train)
        co_p = common.bn_coeffs(b.proj_bn, st, common.rows(c_p), train)
        rs = droppath.sample_scale(b.drop if train else 0.0, B, 4, x.device)
        y = ops.tail_apply(c_p, co_p, rs, residual=h if b.res else None)
        if tape is not None:
            tape["blocks"].append((b, h, dw_in, dw_co, c_e, co_e, d, co_d, pool, hpre, gate, a, c_p, co_p, rs))
        h = y
    c_t, st = ops.conv2d_fwd(h, pack.get(top_conv.weight, 0), 1, 1, want_stats=train)
    co_t = common.bn_coeffs(top_bn, st, common.rows(c_t), train)
    Fc = c_t.shape[-1]
    if train and p > 0:
        mask = common.dropout_mask(p, B, Fc, x.device, inplace=True)
    else:
        mask = torch.ones(B, Fc, dtype=torch.float32, device=x.device)
    _, feat = ops.silu_bn_squeeze(c_t, co_t, mask=mask)
    logits = common.head_forward(pack, head, feat)
    if tape is not None:
        tape["top"] = (h, c_t, co_t, mask, feat)
    return logits, tape


# --------------------------------------------------------------------------------------------------------- backward
def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    stem_conv, stem_bn, blocks, top_conv, top_bn, _, head = check_model(model)
    grads = common.Grads(sink)
    pack = tape["pack"]

    h, c_t, co_t, mask, feat = tape["top"]
    dfeat = common.head_backward(grads, pack, head, feat, dlogits)
    dpool = ops.cast_f32(dfeat).mul_(mask)      # [B, F]: the classifier dropout's backward
    dz, part = ops.silu_bn_bwd_reduce(c_t, co_t, dpool)
    dc = common.bn_backward_from_sums(grads, top_bn, dz, part, c_t, co_t)
    grads.put(top_conv.weight, ops.conv2d_wgrad(dc, h, 1, 1, out=grads.dest(top_conv.weight)))
    g = ops.conv2d_dgrad(dc, pack.get(top_conv.weight, 1), tuple(h.shape[1:3]), 1, 1)

    for b, x, dw_in, dw_co, c_e, co_e, d, co_d, pool, hpre, gate, a, c_p, co_p, rs in reversed(tape["blocks"]):
        dz, part = ops.tail_bwd_reduce(g, c_p, rs)
        dc = common.bn_backward_from_sums(grads, b.proj_bn, dz, part, c_p, co_p)
        grads.put(b.proj.weight, ops.conv2d_wgrad(dc, a, 1, 1, out=grads.dest(b.proj.weight)))
        da = ops.conv2d_dgrad(dc, pack.get(b.proj.weight, 1), tuple(a.shape[1:3]), 1, 1)
        s = ops.gate_reduce(da, d, co_d)
        d1, d2 = grads.dest(b.fc1.weight), grads.dest(b.fc2.weight)
        dpool, dw1, db1, dw2, db2 = ops.excite_bwd(
            s, pool, hpre, gate, b.fc1.weight, b.fc2.weight,
            dw1=None if d1 is None else d1.view(d1.shape[0], -1), db1=grads.dest(b.fc1.bias),
            dw2=None if d2 is None else d2.view(d2.shape[0], -1), db2=grads.dest(b.fc2.bias))
        grads.put(b.fc2.bias, db2)
        grads.put(b.fc2.weight, dw2)
        grads.put(b.fc1.bias, db1)
        grads.put(b.fc1.weight, dw1)
        dz, part = ops.silu_bn_bwd_reduce(d, co_d, dpool, da=da, gate=gate)
        dd = common.bn_backward_from_sums(grads, b.dw_bn, dz, part, d, co_d)
        grads.put(b.dw.weight, ops.dw_wgrad(dd, dw_in, b.k, b.s, co=dw_co, out=grads.dest(b.dw.weight)))
        if dw_co is None:
            # the depthwise read the previous block's output as is
            g, _ = ops.dw_dgrad(dd, b.dw.weight, dw_in, b.k, b.s, residual=g if b.res else None)
            continue
        dz, part = ops.dw_dgrad(dd, b.dw.weight, dw_in, b.k, b.s, co=dw_co)
        if b.exp is None:
            # block 1a: its input is silu(bn(stem conv)), normalised on load
            patches, c_s, co_s = tape["stem"]
            dc = common.bn_backward_from_sums(grads, stem_bn, dz, part, c_s, co_s)
            C0 = c_s.shape[-1]
            gw = ops.conv2d_wgrad(dc, patches, 1, 1).view(C0, _STEM_LDK)
            grads.put(stem_conv.weight, ops.stem_wgrad_relayout(gw, C0, 3, 9, out=grads.dest(stem_conv.weight)))
            break
        dc = common.bn_backward_from_sums(grads, b.exp_bn, dz, part, c_e, co_e)
        grads.put(b.exp.weight, ops.conv2d_wgrad(dc, x, 1, 1, out=grads.dest(b.exp.weight)))
        g = ops.conv2d_dgrad(dc, pack.get(b.exp.weight, 1), tuple(x.shape[1:3]), 1, 1, residual=g if b.res else None)
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "EfficientNet", model, x)
