"""Forward / backward schedule of VGG (classification/vggNet/models/network.py) on the sm_90a kernels.

The whole network is ONE autograd node (common.apply).  Activations are NHWC bf16, parameters fp32.  A layer of ``features``
(Conv2d 3x3 / pad 1 with bias [, BatchNorm2d], ReLU [, MaxPool2d(2, 2)]) runs as

    plain     y = relu(conv(x) + b) in the GEMM epilogue; a pooled layer then runs the 2x2 pool over y (csrc/vgg.cuh)
    _bn       c = conv(x) + b with the BatchNorm statistics in the GEMM epilogue (the bias is inside the batch mean and
              running_mean, as in torch)  ->  finalize  ->  a pooled layer pools relu(c * scale + shift) straight from c, so
              its full-resolution activation is never stored; an unpooled layer writes y = relu(bn(c)) for the next conv
    backward  pooled: the pool backward scatters the pooled gradient to the arg-max pixel and applies the ReLU mask (plain:
              pooled y > 0; _bn: c * scale + shift > 0, with the BatchNorm-backward sums in the same pass); unpooled: the
              next layer's dgrad applies the mask in its epilogue (kEpiBnMask; the plain variant with scale 1 / shift 0,
              whose mask is then y > 0)  ->  (_bn: finalize + apply)  ->  wgrad with the bias gradient from the same kernel

The first convolution (3 input channels) is one 1x1 GEMM over the [B*H*W][32] im2col patch matrix of the image.
``avgpool`` + ``torch.flatten`` is one pass writing bf16 [B, C*49] in NCHW flatten order, so ``classifier.0.weight`` is used
as it is.  The classifier's Linear layers are GEMMs with bias + ReLU in the epilogue; the dropout after each multiplies by a
mask drawn with F.dropout on an fp32 tensor of ones, which consumes the generator as the reference's ``nn.Dropout()`` on
the fp32 [B, 4096] activation does; its backward needs only the stored h = dropout(relu(pre)): dpre = h > 0 ? dh / (1 - p) : 0.
``dropout_replay`` / ``dropout_record`` (engine.common, shared with EfficientNet) are the masks' test hooks.

Eval mode: plain layers run the same GEMMs and pools (without arg-max bytes); _bn layers run folded GEMMs
relu(conv * scale + shift') with shift' = beta - (running_mean - b) * scale, dropout is the identity and no tape is recorded.
"""
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common
from .common import dropout_record, dropout_replay  # noqa: F401  (the classifier-dropout test hooks)
from .packing import weight_cache

_STEM_LDK = 32     # patch-matrix width of the 3x3 x 3-channel first convolution (27 columns, padded to a multiple of 8)

# --------------------------------------------------------------------------------------------------------- admission
class _Layer:
    """One convolution of ``features`` as the schedule runs it."""
    __slots__ = ("name", "conv", "bn", "pool")


def _check_features(feats):
    if not isinstance(feats, nn.Sequential) or len(feats) == 0:
        raise NotImplementedError("features: expected the reference's make_layers Sequential")
    mods = list(feats._modules.items())
    layers = []
    cin = 3
    i = 0
    while i < len(mods):
        name, conv = mods[i]
        where = f"features.{name}"

        def no(why, m=conv, w=where):
            raise NotImplementedError(f"{w}: {why} (got {m})")

        if type(conv) is not nn.Conv2d:
            no("expected a Conv2d here (make_layers: Conv2d [, BatchNorm2d], ReLU [, MaxPool2d(2, 2)])")
        if (conv.kernel_size != (3, 3) or conv.stride != (1, 1) or conv.padding != (1, 1) or conv.dilation != (1, 1)
                or conv.groups != 1 or conv.bias is None or conv.padding_mode != "zeros"):
            no("the GPU engine runs VGG convolutions as 3x3, stride 1, padding 1, with bias")
        if conv.in_channels != cin:
            no(f"in_channels must be {cin}" + (" (3 input channels at the first convolution)" if not layers else ""))
        if conv.out_channels % 64 != 0:
            no("out_channels must be a multiple of 64")
        lay = _Layer()
        lay.name, lay.conv, lay.bn, lay.pool = where, conv, None, False
        i += 1
        if i < len(mods) and type(mods[i][1]) in (nn.BatchNorm2d, nn.SyncBatchNorm):
            bn_name, bn = mods[i]
            if not common.bn_ok(bn, conv.out_channels):
                raise NotImplementedError(f"features.{bn_name}: expected an affine BatchNorm2d that tracks running "
                                          f"statistics (got {bn})")
            if common.bn_sync(bn) is not None:
                raise NotImplementedError(f"features.{bn_name}: SyncBatchNorm in a multi-rank job is not implemented for VGG")
            lay.bn = bn
            i += 1
        if i >= len(mods) or type(mods[i][1]) is not nn.ReLU:
            m = mods[i] if i < len(mods) else (str(len(mods)), None)
            raise NotImplementedError(f"features.{m[0]}: expected a ReLU after the convolution{' and BatchNorm' if lay.bn else ''}"
                                      f" (got {m[1]})")
        i += 1
        if i < len(mods) and type(mods[i][1]) is nn.MaxPool2d:
            pname, pool = mods[i]
            if (pool.kernel_size not in (2, (2, 2)) or pool.stride not in (2, (2, 2)) or pool.padding not in (0, (0, 0))
                    or pool.dilation not in (1, (1, 1)) or pool.ceil_mode or pool.return_indices):
                raise NotImplementedError(f"features.{pname}: the GPU engine runs MaxPool2d(kernel_size=2, stride=2) only "
                                          f"(got {pool})")
            lay.pool = True
            i += 1
        elif i < len(mods) and type(mods[i][1]) is not nn.Conv2d:
            raise NotImplementedError(f"features.{mods[i][0]}: expected a Conv2d or MaxPool2d(2, 2) (got {mods[i][1]})")
        layers.append(lay)
        cin = conv.out_channels
    if not layers[-1].pool:
        raise NotImplementedError(f"{layers[-1].name}: the GPU engine needs features to end with MaxPool2d(2, 2)")
    return layers


def check_model(model):
    """Admission of a whole VGG, without touching a device: raises NotImplementedError naming the first layer the engine
    does not run (anything but make_layers' Conv2d(3x3, pad 1, bias) [, BatchNorm2d], ReLU [, MaxPool2d(2, 2)] structure,
    out_channels not a multiple of 64, SyncBatchNorm in a multi-rank job, an avgpool that is not an AdaptiveAvgPool2d, a
    classifier other than the reference's Linear, ReLU, Dropout, Linear, ReLU, Dropout, Linear).
    Returns ([_Layer], (fc0, fc3, fc6), (p0, p1))."""
    layers = _check_features(getattr(model, "features", None))
    if type(getattr(model, "avgpool", None)) is not nn.AdaptiveAvgPool2d or model.avgpool.output_size not in (7, (7, 7)):
        raise NotImplementedError(f"avgpool: the GPU engine runs VGG with AdaptiveAvgPool2d((7, 7)) "
                                  f"(got {getattr(model, 'avgpool', None)})")
    cls = getattr(model, "classifier", None)
    kinds = (nn.Linear, nn.ReLU, nn.Dropout, nn.Linear, nn.ReLU, nn.Dropout, nn.Linear)
    if not isinstance(cls, nn.Sequential) or len(cls) != 7:
        raise NotImplementedError("classifier: expected the reference's 7-module Sequential (Linear, ReLU, Dropout, Linear, "
                                  "ReLU, Dropout, Linear)")
    for k, (m, kind) in enumerate(zip(cls, kinds)):
        if type(m) is not kind:
            raise NotImplementedError(f"classifier.{k}: expected {kind.__name__} (got {m})")
    fc0, fc3, fc6 = cls[0], cls[3], cls[6]
    widths = (layers[-1].conv.out_channels * 49, fc0.out_features, fc3.out_features)
    for k, fc, fin in ((0, fc0, widths[0]), (3, fc3, widths[1]), (6, fc6, widths[2])):
        if fc.bias is None or fc.in_features != fin:
            raise NotImplementedError(f"classifier.{k}: expected a biased Linear with in_features {fin} (got {fc})")
    for k, fc in ((0, fc0), (3, fc3)):
        if fc.out_features % 8 != 0:
            raise NotImplementedError(f"classifier.{k}: out_features must be a multiple of 8 (got {fc})")
    ps = (float(cls[2].p), float(cls[5].p))
    for k, p in zip((2, 5), ps):
        if not 0.0 <= p < 1.0:
            raise NotImplementedError(f"classifier.{k}: the GPU engine runs dropout with 0 <= p < 1 (got {cls[k]})")
    return layers, (fc0, fc3, fc6), ps


# ---------------------------------------------------------------------------------------------------------- packing
class _PackSpec:
    """bf16 operands: the first convolution's [C0][32] patch-matrix operand, forward [O][9*I] / dgrad [I][9*O] copies of every
    other convolution, and forward / dgrad copies of the classifier's Linear layers (the last one class-padded)."""

    @staticmethod
    def key(model):
        layers, fcs, _ = check_model(model)
        return (tuple(id(l.conv.weight) for l in layers), tuple(id(f.weight) for f in fcs), fcs[2].out_features)

    def __call__(self, model):
        layers, (fc0, fc3, fc6), _ = check_model(model)
        first = layers[0].conv
        specs = [(first.weight, 0, _STEM_LDK, first.out_channels)]
        for l in layers[1:]:
            O, I = l.conv.out_channels, l.conv.in_channels
            specs += [(l.conv.weight, 0, 9 * I, O), (l.conv.weight, 1, 9 * O, I)]
        for fc in (fc0, fc3):
            specs += [(fc.weight, 0, fc.in_features, fc.out_features), (fc.weight, 1, fc.out_features, fc.in_features)]
        return specs + common.head_pack_specs(fc6)


_pack_spec = _PackSpec()

_ident = {}


def _identity_coeffs(C, device):
    """scale 1 / shift 0: the kEpiBnMask dgrad epilogue with these keeps the gradient where the stored ReLU output is > 0."""
    key = (C, device)
    co = _ident.get(key)
    if co is None:
        co = ops.BnCoeffs(C, device)
        co.scale.fill_(1.0)
        co.shift.zero_()
        co.mean.zero_()
        co.invstd.fill_(1.0)
        _ident[key] = co
    return co


def _linear(pack, fc, x2d, relu):
    B = x2d.shape[0]
    y, _ = ops.conv2d_fwd(x2d.view(B, 1, 1, x2d.shape[1]), pack.get(fc.weight, 0), bias=fc.bias.detach(), act=1 if relu else 0)
    return y.view(B, fc.out_features)


# ---------------------------------------------------------------------------------------------------------- forward
def forward(model, x, train, want_tape):
    """x: fp32 NCHW (or decoded uint8 NHWC) CUDA batch.  Returns (logits fp32 [B, num_classes], tape or None)."""
    layers, (fc0, fc3, fc6), (p0, p1) = check_model(model)
    x = common.image_input(model, x)
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
    pack = weight_cache.model_pack(model, _pack_spec)
    tape = {"layers": [], "pack": pack} if (train and want_tape) else None
    B, _, H, W = x.shape
    a, _, _ = ops.im2col_nchw(x, 3, 3, 1, 1, ldk=_STEM_LDK)
    h = a.view(B, H, W, _STEM_LDK)
    for li, l in enumerate(layers):
        conv, bn = l.conv, l.bn
        k = 1 if li == 0 else 3      # the first convolution is a 1x1 GEMM over the patch matrix
        w = pack.get(conv.weight, 0)
        Hc, Wc = h.shape[1], h.shape[2]
        if l.pool and (Hc < 2 or Wc < 2):
            raise ValueError(f"{l.name}: a {Hc}x{Wc} feature map is too small for MaxPool2d(2, 2)")
        if bn is None:
            y, _ = ops.conv2d_fwd(h, w, k, 1, bias=conv.bias.detach(), act=1)
            c = co = None
        elif train:
            c, st = ops.conv2d_fwd(h, w, k, 1, want_stats=True, bias=conv.bias.detach())
            co = common.bn_coeffs(bn, st, c.numel() // c.shape[-1], True)
            y = None if l.pool else ops.bn_apply(c, co, relu=True)
        else:
            # relu(bn(conv + b)) = relu(conv * scale + beta - (running_mean - b) * scale)
            fold = ops.bn_eval_coeffs(bn.weight, bn.bias, bn.running_mean - conv.bias.detach(), bn.running_var, bn.eps)
            y = ops.conv2d_bn_act(h, w, fold, k, 1, relu=True)
            c = co = None
        idx = None
        out = y
        if l.pool:
            out, idx = ops.vgg_pool_fwd(y if c is None else c, co, want_idx=tape is not None)
        if tape is not None:
            # y is kept only where the backward reads it: the ReLU mask of an unpooled plain layer (a pooled plain layer
            # masks on its pooled output, a _bn layer on c)
            tape["layers"].append((l, h, y if (bn is None and not l.pool) else None, c, co, idx, out))
        h = out
    feat = ops.vgg_avgpool7_fwd(h)
    d0 = _linear(pack, fc0, feat, True)
    if train and p0 > 0:
        d0 = ops.vgg_dropout_fwd(d0, common.dropout_mask(p0, B, d0.shape[1], x.device, inplace=False))
    d1 = _linear(pack, fc3, d0, True)
    if train and p1 > 0:
        d1 = ops.vgg_dropout_fwd(d1, common.dropout_mask(p1, B, d1.shape[1], x.device, inplace=False))
    logits = common.head_forward(pack, fc6, d1)
    if tape is not None:
        tape["head"] = (h.shape, feat, d0, d1)
    return logits, tape


# --------------------------------------------------------------------------------------------------------- backward
def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    _, (fc0, fc3, fc6), (p0, p1) = check_model(model)
    grads = common.Grads(sink)
    pack = tape["pack"]

    h_shape, feat, d0, d1 = tape["head"]
    g = ops.vgg_dropout_bwd(common.head_backward(grads, pack, fc6, d1, dlogits), d1, p1)
    common.linear_grads(grads, fc3, g, d0)
    g = ops.conv2d_dgrad(g.view(g.shape[0], 1, 1, -1), pack.get(fc3.weight, 1), (1, 1)).view(d0.shape)
    g = ops.vgg_dropout_bwd(g, d0, p0)
    common.linear_grads(grads, fc0, g, feat)
    g = ops.conv2d_dgrad(g.view(g.shape[0], 1, 1, -1), pack.get(fc0.weight, 1), (1, 1)).view(feat.shape)
    g = ops.vgg_avgpool7_bwd(g, tuple(h_shape))

    tl = tape["layers"]
    for li in range(len(tl) - 1, -1, -1):
        l, x, y, c, co, idx, out = tl[li]
        conv, bn = l.conv, l.bn
        # g: the gradient w.r.t. this layer's pooled output, or (unpooled) the masked gradient of its activation (plain:
        # dL/d(conv + b); _bn: (dz, partial) from the next layer's dgrad)
        if l.pool:
            hw = tuple(x.shape[1:3])   # (3x3 / stride 1 / pad 1: the conv output has its input's size)
            g = ops.vgg_pool_bwd(g, idx, hw, y=out) if bn is None else ops.vgg_pool_bwd(g, idx, hw, c=c, co=co)
        if bn is not None:
            dz, part = g
            dc = common.bn_backward_from_sums(grads, bn, dz, part, c, co)
        else:
            dc = g
        gb = grads.dest(conv.bias)
        if gb is None:
            gb = torch.empty(conv.out_channels, dtype=torch.float32, device=dc.device)
        if li == 0:
            C0 = conv.out_channels
            gw = ops.conv2d_wgrad(dc, x, 1, 1, bias_out=gb).view(C0, _STEM_LDK)
            grads.put(conv.bias, gb)
            grads.put(conv.weight, ops.stem_wgrad_relayout(gw, C0, 3, 9, out=grads.dest(conv.weight)))
            break
        gw = ops.conv2d_wgrad(dc, x, 3, 1, out=grads.dest(conv.weight), bias_out=gb)
        grads.put(conv.bias, gb)
        grads.put(conv.weight, gw)
        prev = tl[li - 1]
        wd = pack.get(conv.weight, 1)
        in_hw = tuple(x.shape[1:3])
        if prev[0].pool:
            g = ops.conv2d_dgrad(dc, wd, in_hw, 3, 1)
        elif prev[0].bn is None:
            g, _ = ops.conv2d_dgrad(dc, wd, in_hw, 3, 1, bn_mask=(prev[2], _identity_coeffs(x.shape[-1], x.device)))
        else:
            g = ops.conv2d_dgrad(dc, wd, in_hw, 3, 1, bn_mask=(prev[3], prev[4]))
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "VGG", model, x)
