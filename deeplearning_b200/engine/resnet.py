"""Forward / backward schedule of the ResNet family on the sm_90a kernels.

The whole network is ONE ``torch.autograd.Function``: forward runs conv(+BN statistics in the GEMM epilogue) -> finalize ->
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
"""
import os

import torch
import torch.nn as nn

from .. import ops
from .packing import weight_cache

BF16 = torch.bfloat16


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


def _bn_sync(bn):
    """(process_group, world_size) when ``bn`` is a SyncBatchNorm in a multi-rank job (the recipe converts every BatchNorm
    with ``nn.SyncBatchNorm.convert_sync_batchnorm``: others/train_with_DDP/train.py:190), else None.  Statistics and the
    two backward sums are then all-reduced per layer (ops._sync_sums); such layers stay on the plain conv -> BN schedule."""
    if not isinstance(bn, nn.SyncBatchNorm) or not bn.training:
        return None
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group if bn.process_group is not None else dist.group.WORLD
    world = dist.get_world_size(group)
    return (group, world) if world > 1 else None


class _PackSpec:
    """Which bf16 operands a ResNet needs: forward [O][taps*I] and dgrad [I][taps*O] copies of every conv / fc weight."""

    @staticmethod
    def key(model):
        return (model.fc.out_features, id(model.fc))

    def __call__(self, model):
        specs = []
        for name, mod in model.named_modules():
            if isinstance(mod, nn.Conv2d):
                w = mod.weight
                O, I, kh, kw = w.shape
                if name == "conv1":
                    specs.append((w, 2, 256, O, (O, I, kh * kw)))  # space-to-depth stem operand [64][256]
                    continue
                if mod.groups != 1:   # block-diagonal operands of a grouped 3x3 convolution
                    specs.append((w, 3, kh * kw * 64, O))
                    specs.append((w, 4, kh * kw * 64, O))
                    continue
                specs.append((w, 0, kh * kw * I, O))
                specs.append((w, 1, kh * kw * O, I))
        fc = model.fc
        n_pad = (fc.out_features + 7) // 8 * 8
        specs.append((fc.weight, 0, fc.in_features, n_pad))
        specs.append((fc.weight, 1, n_pad, fc.in_features))
        return specs


_pack_spec = _PackSpec()


class _Unit:
    """Saved state of one conv -> BN (-> ReLU) (-> + residual) application.  ``algebra`` units (bottleneck conv3 with the
    BatchNorm folded through the convolution) have no raw conv output ``c``; they keep the Gram matrix ``G`` and the column
    sums ``s`` of their input instead."""
    __slots__ = ("conv", "bn", "x", "c", "co", "y", "relu", "has_res", "algebra", "G", "s")


def _algebra_enabled():
    return os.environ.get("B200_RESNET_ALGEBRA", "1") != "0"


def _algebra_ok(block, train, want_tape):
    """Bottleneck whose tail can run with bn3 folded through conv3 (train mode, or a forward that records no tape)."""
    if not _algebra_enabled() or not hasattr(block, "conv3") or not (train or not want_tape):
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
        u = _Unit()
        u.conv, u.bn, u.x, u.c, u.co, u.y, u.relu, u.has_res = conv, bn, y2, None, co, y, True, True
        u.algebra, u.G, u.s = True, G, s
        tape.append(u)
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
        u = _Unit()
        u.conv, u.bn, u.x, u.c, u.co, u.y, u.relu, u.has_res = conv, bn, xs, None, co, ident, False, False
        u.algebra, u.G, u.s = True, G, s
        tape.append(u)
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
    if train:
        rows = c.numel() // c.shape[-1]
        co = ops.bn_finalize(st, rows, bn.weight, bn.bias, bn.eps, bn.momentum, bn.running_mean, bn.running_var,
                             bn.num_batches_tracked, sync=_bn_sync(bn))
    else:
        co = ops.bn_eval_coeffs(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
    y = ops.bn_apply(c, co, relu=relu, residual=residual)
    if tape is not None:
        u = _Unit()
        u.conv, u.bn, u.x, u.c, u.co, u.y, u.relu, u.has_res = conv, bn, x, c, co, y, relu, residual is not None
        u.algebra, u.G, u.s = False, None, None
        tape.append(u)
    return y


def _algebra_ok_dgrad(conv1):
    return (conv1.kernel_size == (1, 1) and conv1.stride == (1, 1) and conv1.in_channels % 64 == 0
            and conv1.out_channels % 64 == 0)


def _block_units(block):
    """(conv, bn) pairs of the residual branch, in order."""
    if hasattr(block, "conv3"):
        return [(block.conv1, block.bn1), (block.conv2, block.bn2), (block.conv3, block.bn3)]
    return [(block.conv1, block.bn1), (block.conv2, block.bn2)]


def forward(model, x, train, want_tape):
    """x: fp32 NCHW CUDA batch. Returns (logits fp32 [B, num_classes], tape or None)."""
    u8 = x.dtype == torch.uint8     # GPU input pipeline: decoded uint8 NHWC batch, ToTensor + Normalize fused into the stem operand
    if u8:
        if x.dim() != 4 or x.shape[3] != 3:
            raise ValueError(f"uint8 input must be a decoded NHWC batch [B,H,W,3], got {tuple(x.shape)}")
        x = x.contiguous()
        x_hw = (x.shape[1], x.shape[2])
    else:
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected an [B,3,H,W] image batch, got {tuple(x.shape)}")
        x = x.contiguous().float()
        x_hw = (x.shape[2], x.shape[3])
    B = x.shape[0]
    if not isinstance(model.fc, nn.Linear):
        raise NotImplementedError("model.fc must be an nn.Linear")
    pack = weight_cache.model_pack(model, _pack_spec)  # one launch repacks every bf16 operand if parameters changed
    tape = {"stem": None, "blocks": [], "head": None, "pack": pack} if want_tape else None
    # ---- stem: 7x7/2 conv as a space-to-depth implicit GEMM, BN statistics in the epilogue, BN+ReLU+max-pool in one pass
    conv1, bn1 = model.conv1, model.bn1
    _check_bn(bn1, "bn1")
    if conv1.kernel_size != (7, 7) or conv1.stride != (2, 2) or conv1.padding != (3, 3) or conv1.bias is not None:
        raise NotImplementedError("stem must be the 7x7/2 pad-3 bias-free convolution of the reference")
    if conv1.out_channels != 64 or x_hw[0] % 2 or x_hw[1] % 2:
        raise NotImplementedError("stem: 64 output channels and an even input size are required")
    # space-to-depth operand (108 MB at bs 256 instead of a 1 GB patch matrix); the conv reads it through overlapping TMA rows
    a = ops.stem_s2d_u8(x, *getattr(model, "input_norm", (ops.IMAGENET_MEAN, ops.IMAGENET_STD))) if u8 else ops.stem_s2d(x)
    Ho, Wo = a.shape[1] - 3, a.shape[2] - 3
    c1, st = ops.stem_s2d_conv_fwd(a, pack.get(conv1.weight, 2), want_stats=train)
    if train:
        co1 = ops.bn_finalize(st, B * Ho * Wo, bn1.weight, bn1.bias, bn1.eps, bn1.momentum, bn1.running_mean,
                              bn1.running_var, bn1.num_batches_tracked, sync=_bn_sync(bn1))
    else:
        co1 = ops.bn_eval_coeffs(bn1.weight, bn1.bias, bn1.running_mean, bn1.running_var, bn1.eps)
    h, idx = ops.bn_relu_maxpool_fwd(c1, co1)
    if want_tape:
        tape["stem"] = (a, c1, co1, idx, (Ho, Wo))
    # ---- residual stages
    for li in range(1, 5):
        for bi, block in enumerate(getattr(model, f"layer{li}")):
            units = [] if want_tape else None
            name = f"layer{li}.{bi}"
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
            if _algebra_ok(block, train, want_tape):
                _check_conv(conv, f"{name}.conv3")
                h = _conv3_bn_res_relu(pack, units, h, conv, bn, train, identity, name=f"{name}.conv3")
            else:
                h = _conv_bn(pack, units, h, conv, bn, train, relu=True, residual=identity, name=f"{name}.conv{len(pairs)}")
            if want_tape:
                tape["blocks"].append((units, ds_units[0] if ds_units else None, x_in))
    # ---- head: global average pool + fc (fp32 logits)
    pooled = ops.avgpool_fwd(h)
    fc = model.fc
    n_cls = fc.out_features
    n_pad = (n_cls + 7) // 8 * 8
    wfc = pack.get(fc.weight, 0)
    bias = None
    if fc.bias is not None:
        bias = fc.bias.detach()
        if n_pad != n_cls:
            bias = torch.cat([bias, bias.new_zeros(n_pad - n_cls)])
    logits, _ = ops.conv2d_fwd(pooled.view(B, 1, 1, -1), wfc, bias=bias, out_f32=True)
    logits = logits.view(B, n_pad)
    if want_tape:
        tape["head"] = (pooled, h.shape[1:3], n_cls, n_pad)
    return (logits[:, :n_cls] if n_pad != n_cls else logits), tape


class _Grads(dict):
    """{parameter.data_ptr(): fp32 gradient}. ``sink(param)`` may supply the destination buffer (a view of the flat
    gradient arena of engine.trainer) so gradients are produced in place instead of in fresh tensors."""

    def __init__(self, sink=None):
        super().__init__()
        self.sink = sink

    def dest(self, param):
        return self.sink(param) if self.sink is not None else None

    def put(self, param, value):
        """Record the (final) gradient of ``param``; a sink with a ``notify`` method is told so that the data-parallel
        trainer can start all-reducing completed stretches of the gradient arena while the backward pass continues."""
        self[param.data_ptr()] = value
        notify = getattr(self.sink, "notify", None)
        if notify is not None:
            notify(param)


def _unit_backward(u, g, grads, want_dz=False):
    """Backward of BN(+ReLU) of unit u for upstream gradient g; returns (dc, dz) and records BN param grads."""
    dc, dgamma, dbeta, dz = ops.bn_backward(g, u.c, u.co, relu=u.relu, y_out=u.y if (u.relu and u.has_res) else None,
                                            want_dz=want_dz, dgamma=grads.dest(u.bn.weight), dbeta=grads.dest(u.bn.bias),
                                            sync=_bn_sync(u.bn))
    grads.put(u.bn.weight, dgamma)
    grads.put(u.bn.bias, dbeta)
    return dc, dz


def _fused_reduce_ok(u):
    """Can the dgrad GEMM that produces the gradient of unit u's output also do the reduce half of u's BN backward?
    (relu(bn(c)) without a residual, 64-channel multiples)"""
    return u.relu and not u.has_res and u.c.shape[-1] % 64 == 0


def _unit_backward_from_sums(u, dz, sums, grads):
    dc, dgamma, dbeta = ops.bn_backward_from_sums(dz, sums, u.c, u.co, dgamma=grads.dest(u.bn.weight), dbeta=grads.dest(u.bn.bias),
                                                  sync=_bn_sync(u.bn))
    grads.put(u.bn.weight, dgamma)
    grads.put(u.bn.bias, dbeta)
    return dc


def backward(model, tape, dlogits, sink=None):
    """dlogits: fp32 [B, num_classes] (or the bf16 [B, n_pad] product of ops.softmax_xent).
    Returns {parameter.data_ptr(): fp32 gradient}; with ``sink`` the gradients are written into caller-owned buffers."""
    grads = _Grads(sink)
    pooled, hw, n_cls, n_pad = tape["head"]
    B = pooled.shape[0]
    fc = model.fc
    if dlogits.dtype == BF16 and dlogits.shape[1] == n_pad and dlogits.is_contiguous():
        dl16 = dlogits.view(B, 1, 1, n_pad)  # already produced by the fused soft-max/cross-entropy kernel
    else:
        dl = dlogits.contiguous().float()
        if n_pad != n_cls:
            dl = torch.cat([dl, dl.new_zeros(B, n_pad - n_cls)], 1).contiguous()
        dl16 = ops.cast_bf16(dl).view(B, 1, 1, n_pad)
    x_fc = pooled.view(B, 1, 1, -1)
    dst = grads.dest(fc.weight)
    if dst is not None and n_pad == n_cls:
        grads.put(fc.weight, ops.conv2d_wgrad(dl16, x_fc, out=dst.view(n_cls, -1, 1, 1)))
    else:
        gw = ops.conv2d_wgrad(dl16, x_fc).view(n_pad, -1)[:n_cls]
        if dst is not None:
            dst.copy_(gw)
            gw = dst
        grads.put(fc.weight, gw)
    if fc.bias is not None:
        grads.put(fc.bias, ops.colsum(dl16.view(B, n_pad), cols=n_cls, out=grads.dest(fc.bias)))
    pack = tape["pack"]
    wfc_d = pack.get(fc.weight, 1)
    dpooled = ops.conv2d_dgrad(dl16, wfc_d, (1, 1))
    g = ops.avgpool_bwd(dpooled.view(B, -1), hw)

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
            N, K = last.conv.out_channels, last.conv.in_channels
            D = ops.conv2d_wgrad(dz, y2, 1, 1)                       # raw dz^T y2 [N, K, 1, 1]
            count = dz.numel() // N
            dgamma, dbeta, dW, wcat, wbias = ops.bn_conv1x1_bwd(
                dz_stats, D, last.G, last.s, pack.get(last.conv.weight, 0), last.conv.weight, count, last.bn.weight, last.co,
                dgamma=grads.dest(last.bn.weight), dbeta=grads.dest(last.bn.bias), dW=grads.dest(last.conv.weight))
            grads.put(last.bn.weight, dgamma)
            grads.put(last.bn.bias, dbeta)
            grads.put(last.conv.weight, dW)
            # dL/dy2 = [dz | y2] [a W3 | M]^T + k W3; its epilogue also masks with bn2's ReLU and sums for bn2's backward
            u2 = units[-2]
            if _fused_reduce_ok(u2):
                dz2, sums2 = ops.gemm_dual(dz, y2, wcat, wbias, bn_mask=(u2.c, u2.co))
                dc = _unit_backward_from_sums(u2, dz2, sums2, grads)
            else:
                g_prev = ops.gemm_dual(dz, y2, wcat, wbias)
                dc, _ = _unit_backward(u2, g_prev, grads)
            first = len(units) - 2
        else:
            # out = relu(bn_last(c) + identity): dz is the gradient of the pre-ReLU sum, shared by both branches
            dc, dz = _unit_backward(last, g, grads, want_dz=True)
            first = len(units) - 1
        # downsample branch on the algebra path: its data gradient gxs (on the compact even-pixel grid for stride 2) and all its
        # parameter gradients come from dz directly (no pass over a raw conv output, which does not exist)
        gxs = None
        if has_ds and ds.algebra:
            Nd, Kd = ds.conv.out_channels, ds.conv.in_channels
            Dd = ops.conv2d_wgrad(dz, ds.x, 1, 1)
            dgd, dbd, dWd, wcat_d, wbias_d = ops.bn_conv1x1_bwd(
                dz_stats, Dd, ds.G, ds.s, pack.get(ds.conv.weight, 0), ds.conv.weight, dz.numel() // Nd, ds.bn.weight, ds.co,
                dgamma=grads.dest(ds.bn.weight), dbeta=grads.dest(ds.bn.bias), dW=grads.dest(ds.conv.weight))
            grads.put(ds.bn.weight, dgd)
            grads.put(ds.bn.bias, dbd)
            grads.put(ds.conv.weight, dWd)
            gxs = ops.gemm_dual(dz, ds.x, wcat_d, wbias_d)
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
                dc = _unit_backward_from_sums(units[j - 1], dzj, sumsj, grads)
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
    dc, dgamma, dbeta, _ = ops.bn_backward(g_act, c1, co1, relu=True, sync=_bn_sync(model.bn1), dgamma=grads.dest(model.bn1.weight),
                                           dbeta=grads.dest(model.bn1.bias))
    grads.put(model.bn1.weight, dgamma)
    grads.put(model.bn1.bias, dbeta)
    grads.put(model.conv1.weight, ops.stem_s2d_conv_wgrad(dc, a, out=grads.dest(model.conv1.weight)))
    return grads


class _ResNetFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, model, *params):
        want_tape = any(ctx.needs_input_grad[2:])
        logits, tape = forward(model, x, model.training, want_tape)
        ctx.model, ctx.tape, ctx.params = model, tape, params
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        if ctx.tape is None:
            raise RuntimeError("backward called on a forward that recorded no tape")
        grads = backward(ctx.model, ctx.tape, dlogits)
        ctx.tape = None
        out = []
        for p, need in zip(ctx.params, ctx.needs_input_grad[2:]):
            gp = grads.get(p.data_ptr()) if need else None
            out.append(gp.reshape(p.shape) if gp is not None else None)
        return (None, None, *out)


def apply(model, x):
    if not x.is_cuda:
        raise RuntimeError("deeplearning_b200 ResNet runs on CUDA (sm_90a) tensors only; there is no CPU fallback")
    params = tuple(model.parameters())
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        return _ResNetFunction.apply(x, model, *params)
    logits, _ = forward(model, x, model.training, False)
    return logits
