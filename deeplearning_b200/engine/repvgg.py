"""Forward / backward schedule of RepVGG (classification/RepVGG/models/repvgg.py) on the sm_90a kernels.

The whole network is ONE autograd node (common.apply).  Activations are NHWC bf16, parameters fp32.

Train form, train mode - a block ``relu(bn_d(conv3x3(x)) + bn_1(conv1x1(x)) [+ bn_id(x)])`` runs as

    forward   c3, c1 = conv3x3(x), conv1x1(x) (BatchNorm statistics in the GEMM epilogues)  ->  finalize the two (three)
              BatchNorms  ->  ONE apply pass (csrc/repvgg.cuh) writes y; it also sums y and y^2 when the next block has an
              identity branch, whose batch statistics are then ready without another pass over its input
    backward  ONE reduce pass (dz = g [y > 0] and the per-branch sums)  ->  finalize per BatchNorm  ->  ONE apply pass writes
              dc3, dc1 and the identity branch's dx  ->  wgrad of both convolutions; dx = dgrad3(dc3) + dgrad1(dc1) + dx_id,
              the sums added in the dgrad epilogues

The stem (3x3/2 and 1x1/2 convolutions of the 3-channel image) runs as ONE 1x1 GEMM over the [B*Ho*Wo][32] patch matrix
with the combined [2*C0][32] operand: rows 0..C0-1 hold the 3x3 weight (k = tap*3 + c), rows C0..2*C0-1 the 1x1 weight at
the centre-tap columns 12-14, so [c3 | c1] comes out of one launch and the passes read the halves through a row pitch.

Eval mode folds every train-form block on the device on every forward (the running statistics change behind the tensors'
version counters, so a cached fold could go stale): each layer is one conv + bias + ReLU GEMM.  A block that has been
re-parameterised (``rbr_reparam``: ``deploy=True``, ``switch_to_deploy``, ``repvgg_model_convert``) runs the same GEMM from
its own weight and bias.  Eval forwards record no tape, and a deploy-form block cannot be trained.
"""
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common
from .packing import weight_cache

_STEM_LDK = 32     # patch-matrix width of the 3x3 x 3-channel stem (27 columns, padded to a multiple of 8)
_CENTRE = 12       # column of tap (1, 1), channel 0 in that matrix: what the 1x1/2 stem convolution reads


def _blocks(model):
    """(name, block) of every RepVGG block in execution order."""
    out = [("stage0", model.stage0)]
    for s in range(1, 5):
        out += [(f"stage{s}.{i}", b) for i, b in enumerate(getattr(model, f"stage{s}"))]
    return out


def _is_deploy(block):
    return hasattr(block, "rbr_reparam")


def _conv_ok(conv, k, stride, pad, bias):
    return (type(conv) is nn.Conv2d and conv.kernel_size == (k, k) and conv.stride == (stride, stride)
            and conv.padding == (pad, pad) and conv.dilation == (1, 1) and conv.groups == 1
            and (conv.bias is not None) == bias and conv.padding_mode == "zeros")


def _conv_bn_ok(branch, k, stride, pad, cin, cout):
    return (isinstance(branch, nn.Sequential) and list(branch._modules) == ["conv", "bn"]
            and _conv_ok(branch.conv, k, stride, pad, False) and branch.conv.in_channels == cin
            and branch.conv.out_channels == cout and common.bn_ok(branch.bn, cout))


def _check_block(name, blk, stem):
    """Admission of one RepVGGBlock; raises NotImplementedError naming the layer.  Returns the block's stride."""
    def no(why):
        raise NotImplementedError(f"{name}: {why} (got {blk})")

    if getattr(blk, "groups", 1) != 1:
        no("grouped RepVGG blocks (the g2 / g4 variants) are not implemented on the GPU engine")
    if not isinstance(getattr(blk, "se", None), nn.Identity):
        no("squeeze-and-excitation blocks (use_se, RepVGG-D2se) are not implemented on the GPU engine")
    if not isinstance(getattr(blk, "nonlinearity", None), nn.ReLU):
        no("the GPU engine runs RepVGG blocks with a ReLU nonlinearity")
    ref = blk.rbr_reparam if _is_deploy(blk) else getattr(blk, "rbr_dense", None)
    ref = ref.conv if isinstance(ref, nn.Sequential) else ref
    if not isinstance(ref, nn.Conv2d):
        no("expected the reference's rbr_dense / rbr_1x1 / rbr_identity or rbr_reparam structure")
    cin, cout, s = ref.in_channels, ref.out_channels, ref.stride[0]
    if s not in (1, 2) or ref.groups != 1:
        no("the GPU engine runs RepVGG blocks at stride 1 or 2 without groups")
    if (cin != 3 if stem else cin % 8 != 0) or cout % 8 != 0:
        no("channel counts must be multiples of 8 (3 input channels at the stem)")
    if _is_deploy(blk):
        if not _conv_ok(blk.rbr_reparam, 3, s, 1, True) or any(hasattr(blk, a) for a in ("rbr_dense", "rbr_1x1")):
            no("a re-parameterised block must be one biased 3x3 convolution with padding 1")
        return s
    ident = getattr(blk, "rbr_identity", None)
    if not (_conv_bn_ok(blk.rbr_dense, 3, s, 1, cin, cout) and _conv_bn_ok(getattr(blk, "rbr_1x1", None), 1, s, 0, cin, cout)):
        no("branches must be conv_bn(3x3, pad 1) and conv_bn(1x1, pad 0) at the block's stride")
    if ident is not None and not (cin == cout and s == 1 and common.bn_ok(ident, cin)):
        no("rbr_identity must be a BatchNorm2d of a stride-1 block with in_channels == out_channels")
    for bn in (blk.rbr_dense.bn, blk.rbr_1x1.bn) + ((ident,) if ident is not None else ()):
        if common.bn_sync(bn) is not None:
            no("SyncBatchNorm in a multi-rank job is not implemented for RepVGG")
    return s


def check_model(model):
    """Admission of a whole RepVGG, without touching a device: raises NotImplementedError naming the first layer the engine
    does not run (grouped blocks, SE blocks, channel counts that are not multiples of 8, SyncBatchNorm in a multi-rank job,
    anything but the reference's conv_bn / BatchNorm / ReLU structure).  Returns the blocks' strides."""
    if not isinstance(getattr(model, "gap", None), nn.AdaptiveAvgPool2d) or model.gap.output_size not in (1, (1, 1)):
        raise NotImplementedError("gap: the GPU engine runs RepVGG with AdaptiveAvgPool2d(1)")
    if type(getattr(model, "linear", None)) is not nn.Linear:
        raise NotImplementedError("linear: the classifier must be an nn.Linear")
    strides = []
    for name, blk in _blocks(model):
        strides.append(_check_block(name, blk, blk is model.stage0))
    return strides


class _PackSpec:
    """bf16 operands: forward [O][9*I] / dgrad [I][9*O] copies of every train-form conv weight (1x1: [O][I] / [I][O]), the
    stem's combined [2*C0][32] operand, the forward operands of re-parameterised convolutions and the classifier.  The key
    lists every conv weight, so a block that changes form rebuilds the pack."""

    @staticmethod
    def key(model):
        ws = []
        for _, blk in _blocks(model):
            ws += [id(blk.rbr_reparam.weight)] if _is_deploy(blk) else [id(blk.rbr_dense.conv.weight), id(blk.rbr_1x1.conv.weight)]
        return (id(model.linear), model.linear.out_features, tuple(ws))

    def __call__(self, model):
        specs = []
        for _, blk in _blocks(model):
            stem = blk is model.stage0
            if _is_deploy(blk):
                w = blk.rbr_reparam.weight
                O, I = w.shape[:2]
                specs.append((w, 0, _STEM_LDK if stem else 9 * I, O))
                continue
            w3, w1 = blk.rbr_dense.conv.weight, blk.rbr_1x1.conv.weight
            O, I = w3.shape[:2]
            if stem:
                specs.append((w3, 0, _STEM_LDK, O, None, None, ("stem", 0, 0, 2 * O)))
                specs.append((w1, 0, _STEM_LDK, O, None, None, ("stem", O, _CENTRE, 2 * O)))
                continue
            specs += [(w3, 0, 9 * I, O), (w3, 1, 9 * O, I), (w1, 0, I, O), (w1, 1, O, I)]
        return specs + common.head_pack_specs(model.linear)


_pack_spec = _PackSpec()


def forward(model, x, train, want_tape):
    """x: fp32 NCHW (or decoded uint8 NHWC) CUDA batch.  Returns (logits fp32 [B, num_classes], tape or None)."""
    strides = check_model(model)
    x = common.image_input(model, x)
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
    blocks = _blocks(model)
    if train and want_tape and any(_is_deploy(b) for _, b in blocks):
        raise NotImplementedError("training a re-parameterised (deploy-form) RepVGG is not implemented on the GPU engine: "
                                  "train the multi-branch form and convert it afterwards")
    pack = weight_cache.model_pack(model, _pack_spec)
    tape = {"blocks": [], "head": None, "pack": pack} if (train and want_tape) else None
    B = x.shape[0]
    a, Ho, Wo = ops.im2col_nchw(x, 3, 3, 2, 1, ldk=_STEM_LDK)
    h = a.view(B, Ho, Wo, _STEM_LDK)
    h_stats = None
    for bi, ((name, blk), s) in enumerate(zip(blocks, strides)):
        stem = bi == 0
        k, sk = (1, 1) if stem else (3, s)     # the stem's convolutions are one 1x1 GEMM over the patch matrix
        if _is_deploy(blk):
            conv = blk.rbr_reparam
            h, _ = ops.conv2d_fwd(h, pack.get(conv.weight, 0), k, sk, bias=conv.bias.detach(), act=1)
            h_stats = None
            continue
        ident = blk.rbr_identity
        if not train:
            wp, bias = ops.repvgg_fold(blk.rbr_dense.conv.weight, blk.rbr_1x1.conv.weight, blk.rbr_dense.bn, blk.rbr_1x1.bn,
                                       ident, ldk=_STEM_LDK if stem else None)
            h, _ = ops.conv2d_fwd(h, wp, k, sk, bias=bias, act=1)
            continue
        if ident is not None and h_stats is None:
            raise NotImplementedError(f"{name}: a train-mode identity branch needs the batch statistics of its input, which "
                                      f"only a multi-branch block in front of it provides")
        bn3, bn1 = blk.rbr_dense.bn, blk.rbr_1x1.bn
        if stem:
            C = bn3.num_features
            c, st = ops.conv2d_fwd(h, pack.shared("stem"), 1, 1, want_stats=True)
            c3, c1 = c[..., :C], c[..., C:]
            st3, st1 = st[:, :, :C].contiguous(), st[:, :, C:].contiguous()
        else:
            c = None
            c3, st3 = ops.conv2d_fwd(h, pack.get(blk.rbr_dense.conv.weight, 0), 3, s, want_stats=True)
            c1, st1 = ops.conv2d_fwd(h, pack.get(blk.rbr_1x1.conv.weight, 0), 1, s, want_stats=True)
        rows = c3.numel() // c3.shape[-1]
        co3, co1 = common.bn_coeffs(bn3, st3, rows, True), common.bn_coeffs(bn1, st1, rows, True)
        co_id = common.bn_coeffs(ident, h_stats, rows, True) if ident is not None else None
        nxt = blocks[bi + 1][1] if bi + 1 < len(blocks) else None
        want_stats = nxt is not None and not _is_deploy(nxt) and nxt.rbr_identity is not None
        y, h_stats = ops.repvgg_apply(c3, c1, co3, co1, x=h if ident is not None else None, co_id=co_id, want_stats=want_stats)
        if tape is not None:
            tape["blocks"].append((blk, s, h, c, c3, c1, co3, co1, co_id, y))
        h = y
    pooled = ops.avgpool_fwd(h)
    logits = common.head_forward(pack, model.linear, pooled)
    if tape is not None:
        tape["head"] = (pooled, h.shape[1:3])
    return logits, tape


def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    grads = common.Grads(sink)
    pack = tape["pack"]
    pooled, hw = tape["head"]
    g = ops.avgpool_bwd(common.head_backward(grads, pack, model.linear, pooled, dlogits), hw)

    for blk, s, x, c, c3, c1, co3, co1, co_id, y in reversed(tape["blocks"]):
        stem = c is not None
        C = y.shape[-1]
        rows = y.numel() // C
        ident = blk.rbr_identity if co_id is not None else None
        xi = x if ident is not None else None
        bn3, bn1 = blk.rbr_dense.bn, blk.rbr_1x1.bn
        w3, w1 = blk.rbr_dense.conv.weight, blk.rbr_1x1.conv.weight
        part = ops.repvgg_bwd_reduce(g, y, c3, c1, xi)
        dg1, db1, m1 = ops.bn_bwd_finalize(part[1], rows, co1, grads.dest(bn1.weight), grads.dest(bn1.bias))
        dg3, db3, m3 = ops.bn_bwd_finalize(part[0], rows, co3, grads.dest(bn3.weight), grads.dest(bn3.bias))
        m_id = None
        if ident is not None:
            dgi, dbi, m_id = ops.bn_bwd_finalize(part[2], rows, co_id, grads.dest(ident.weight), grads.dest(ident.bias))
        out = None
        if stem:
            dc = torch.empty_like(c)
            out = (dc[..., :C], dc[..., C:], None)
        dc3, dc1, dx_id = ops.repvgg_bwd_apply(g, y, c3, c1, co3, m3, co1, m1, x=xi, co_id=co_id, m_id=m_id, out=out)
        # gradients in reverse parameter order (rbr_identity, rbr_dense.conv / bn, rbr_1x1.conv / bn), for the bucketed
        # all-reduce that starts on completed stretches of the gradient arena
        grads.put(bn1.bias, db1)
        grads.put(bn1.weight, dg1)
        if stem:
            # one wgrad over [dc3 | dc1] and the patch matrix: rows 0..C-1 are the 3x3 gradient in patch layout, columns
            # 12..14 of rows C..2C-1 the 1x1 gradient
            gw = ops.conv2d_wgrad(dc, x, 1, 1).view(2 * C, _STEM_LDK)
            d1 = grads.dest(w1)
            g1 = gw[C:, _CENTRE:_CENTRE + 3].reshape(w1.shape)
            grads.put(w1, d1.copy_(g1) if d1 is not None else g1)
            grads.put(bn3.bias, db3)
            grads.put(bn3.weight, dg3)
            grads.put(w3, ops.stem_wgrad_relayout(gw[:C], C, 3, 9, out=grads.dest(w3)))
            break
        grads.put(w1, ops.conv2d_wgrad(dc1, x, 1, s, out=grads.dest(w1)))
        grads.put(bn3.bias, db3)
        grads.put(bn3.weight, dg3)
        grads.put(w3, ops.conv2d_wgrad(dc3, x, 3, s, out=grads.dest(w3)))
        if ident is not None:
            grads.put(ident.bias, dbi)
            grads.put(ident.weight, dgi)
        in_hw = tuple(x.shape[1:3])
        if s == 1:
            r = ops.conv2d_dgrad(dc1, pack.get(w1, 1), in_hw, 1, 1, residual=dx_id)
            g = ops.conv2d_dgrad(dc3, pack.get(w3, 1), in_hw, 3, 1, residual=r)
        else:
            # a 1x1 / stride-2 dgrad writes the even pixels only: it adds onto the 3x3 gradient in place
            g = ops.conv2d_dgrad(dc3, pack.get(w3, 1), in_hw, 3, 2)
            g = ops.conv2d_dgrad(dc1, pack.get(w1, 1), in_hw, 1, 2, residual=g, out=g)
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "RepVGG", model, x)
