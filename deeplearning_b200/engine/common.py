"""Plumbing shared by the engine schedules: the class-padded classifier head, the gradient sink, the Linear / LayerNorm
gradient helpers, the BatchNorm admission / coefficient / backward helpers of the CNN engines, the classifier-dropout mask
and its test hooks, the image-input prefix and the autograd entry point ``apply``.

Classifier layout: the conv GEMMs take channel counts in multiples of 8, so the head runs with ``padded_classes(num_classes)``
output columns and the fused cross-entropy writes ``dlogits`` with that row stride; the logits a schedule returns are the
first ``num_classes`` columns of the head's output.
"""
import contextlib

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops

BF16 = torch.bfloat16
F32 = torch.float32


def padded_classes(n):
    """Column count of the classifier output for ``n`` classes (row stride of ``dlogits`` from ops.softmax_xent)."""
    return (n + 7) // 8 * 8


class Grads(dict):
    """{parameter.data_ptr(): fp32 gradient}. ``sink(param)`` may supply the destination buffer (a view of the flat
    gradient arena of engine.trainer) so gradients are produced in place instead of in fresh tensors."""

    def __init__(self, sink=None):
        super().__init__()
        self.sink = sink

    def dest(self, param):
        """The sink's buffer for ``param``'s gradient, viewed as the parameter's shape; None without a sink."""
        d = self.sink(param) if self.sink is not None else None
        return None if d is None else d.view(param.shape)

    def put(self, param, value):
        """Record the (final) gradient of ``param``; a sink with a ``notify`` method is told so that the data-parallel
        trainer can start all-reducing completed stretches of the gradient arena while the backward pass continues."""
        self[param.data_ptr()] = value
        notify = getattr(self.sink, "notify", None)
        if notify is not None:
            notify(param)


def head_pack_specs(head):
    """Forward [n_pad][F] and dgrad [F][n_pad] bf16 operands of the classifier ``head`` (engine.packing.ModelPack specs)."""
    n_pad = padded_classes(head.out_features)
    return [(head.weight, 0, head.in_features, n_pad), (head.weight, 1, n_pad, head.in_features)]


def head_forward(pack, head, feat):
    """fp32 logits [B, num_classes] of the classifier from bf16 features [B, F] (a view of the [B, n_pad] GEMM output)."""
    B, F = feat.shape
    n_cls = head.out_features
    n_pad = padded_classes(n_cls)
    bias = None
    if head.bias is not None:
        bias = head.bias.detach()
        if n_pad != n_cls:
            bias = torch.cat([bias, bias.new_zeros(n_pad - n_cls)])
    logits, _ = ops.conv2d_fwd(feat.view(B, 1, 1, F), pack.get(head.weight, 0), bias=bias, out_f32=True)
    logits = logits.view(B, n_pad)
    return logits[:, :n_cls] if n_pad != n_cls else logits


def head_backward(grads, pack, head, feat, dlogits):
    """Records the gradients of ``head.weight`` / ``head.bias`` and returns the bf16 gradient [B, F] of the features.
    dlogits: fp32 [B, num_classes], or the bf16 [B, n_pad] product of ops.softmax_xent."""
    B, F = feat.shape
    n_cls = head.out_features
    n_pad = padded_classes(n_cls)
    if dlogits.dtype == BF16 and dlogits.shape[1] == n_pad and dlogits.is_contiguous():
        dl16 = dlogits              # already produced by the fused soft-max / cross-entropy kernel
    else:
        dl = dlogits.contiguous().float()
        if n_pad != n_cls:
            dl = torch.cat([dl, dl.new_zeros(B, n_pad - n_cls)], 1).contiguous()
        dl16 = ops.cast_bf16(dl)
    dl4, x4 = dl16.view(B, 1, 1, n_pad), feat.view(B, 1, 1, F)
    dst = grads.dest(head.weight)
    if dst is not None and n_pad == n_cls:
        grads.put(head.weight, ops.conv2d_wgrad(dl4, x4, out=dst.view(n_cls, F, 1, 1)))
    else:
        # the padding rows of the [n_pad, F] gradient are dropped: a sink's [n_cls, F] buffer receives a copy
        gw = ops.conv2d_wgrad(dl4, x4).view(n_pad, F)[:n_cls]
        if dst is not None:
            dst.copy_(gw)
            gw = dst
        grads.put(head.weight, gw)
    if head.bias is not None:
        grads.put(head.bias, ops.colsum(dl16, cols=n_cls, out=grads.dest(head.bias)))
    return ops.conv2d_dgrad(dl4, pack.get(head.weight, 1), (1, 1)).view(B, F)


def linear_grads(grads, lin, dy2d, x2d, dy_stats=None):
    """Weight / bias gradient of a Linear layer from dy [M, N] and its input x [M, K] (both bf16).  Also serves a
    convolution whose weight is consumed as a flat [N][K] matrix (patch embeddings).
    dy_stats: epilogue column-sum partials of dy when the GEMM that produced dy already summed its columns."""
    M, N = dy2d.shape
    K = x2d.shape[1]
    dst = grads.dest(lin.weight)
    gb = None
    if lin.bias is not None and dy_stats is None:
        # bias gradient = column sums of dy: summed inside the wgrad kernel from the dy tiles it already holds
        gb = grads.dest(lin.bias)
        if gb is None:
            gb = torch.empty(N, dtype=F32, device=dy2d.device)
    gw = ops.conv2d_wgrad(dy2d.view(M, 1, 1, N), x2d.view(M, 1, 1, K), out=dst.view(N, K, 1, 1) if dst is not None else None,
                          bias_out=gb)
    grads.put(lin.weight, gw)
    if lin.bias is not None:
        if dy_stats is not None:
            grads.put(lin.bias, ops.stats_colsum(dy_stats, out=grads.dest(lin.bias)))
        else:
            grads.put(lin.bias, gb)


def check_layernorm_widths(named_widths, want_tape):
    """NotImplementedError naming the first LayerNorm (``(name, width)`` pairs) wider than the forward kernel takes, or,
    when a backward pass will follow (``want_tape``), wider than the backward kernel takes."""
    for name, C in named_widths:
        if C > ops.LAYERNORM_FWD_MAX_C:
            raise NotImplementedError(f"{name}: LayerNorm over {C} channels; the LayerNorm kernel takes at most "
                                      f"{ops.LAYERNORM_FWD_MAX_C}")
        if want_tape and C > ops.LAYERNORM_BWD_MAX_C:
            raise NotImplementedError(f"{name}: LayerNorm over {C} channels; the LayerNorm backward kernel takes at most "
                                      f"{ops.LAYERNORM_BWD_MAX_C}, so the GPU engine runs this model without gradients only")


def layernorm_backward(grads, norm, dy, x, mean, rstd, add=None):
    """bf16 dx (+ ``add``) of LayerNorm ``norm``; records the weight and then the bias gradient."""
    dx, dgamma, dbeta = ops.layernorm_bwd(dy, x, mean, rstd, norm.weight, add=add, dx_dtype=BF16,
                                          dgamma=grads.dest(norm.weight), dbeta=grads.dest(norm.bias))
    grads.put(norm.weight, dgamma)
    grads.put(norm.bias, dbeta)
    return dx


def rows(t):
    """Row count of an NHWC activation: the number of values per channel."""
    return t.numel() // t.shape[-1]


def bn_ok(bn, C):
    """``bn`` is an affine BatchNorm2d / SyncBatchNorm over C channels that tracks running statistics with a momentum."""
    return (type(bn) in (nn.BatchNorm2d, nn.SyncBatchNorm) and bn.num_features == C and bn.affine
            and bn.track_running_stats and bn.momentum is not None)


def bn_sync(bn):
    """(process_group, world_size) when ``bn`` is a SyncBatchNorm in a multi-rank job (the recipe converts every BatchNorm
    with ``nn.SyncBatchNorm.convert_sync_batchnorm``: others/train_with_DDP/train.py:190), else None.  Statistics and the
    two backward sums are then all-reduced per layer (ops._sync_sums)."""
    if not isinstance(bn, nn.SyncBatchNorm) or not bn.training:
        return None
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group if bn.process_group is not None else dist.group.WORLD
    world = dist.get_world_size(group)
    return (group, world) if world > 1 else None


def bn_coeffs(bn, stats, rows, train):
    """BatchNorm coefficients: from the batch statistics (``rows`` values per channel, running statistics updated) in
    train mode, from the running statistics in eval mode."""
    if train:
        return ops.bn_finalize(stats, rows, bn.weight, bn.bias, bn.eps, bn.momentum, bn.running_mean, bn.running_var,
                               bn.num_batches_tracked, sync=bn_sync(bn))
    return ops.bn_eval_coeffs(bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)


def bn_backward_from_sums(grads, bn, dz, partial, c, co):
    """dc of a train-mode BatchNorm over the raw input c from its masked gradient dz and partial sums {sum dz, sum dz * c};
    records the bias and then the weight gradient (reverse parameter order, as the overlapped all-reduce walks the arena)."""
    dc, dgamma, dbeta = ops.bn_backward_from_sums(dz, partial, c, co, dgamma=grads.dest(bn.weight),
                                                  dbeta=grads.dest(bn.bias), sync=bn_sync(bn))
    grads.put(bn.bias, dbeta)
    grads.put(bn.weight, dgamma)
    return dc


# ------------------------------------------------------------------------------------------- classifier-dropout masks
_mask_replay = None  # list of fp32 [B, F] classifier-dropout masks being consumed, or None
_mask_record = None  # list collecting the masks drawn, or None


@contextlib.contextmanager
def dropout_replay(masks):
    """Consume the given classifier-dropout masks (fp32 [B, F], already divided by 1 - p; call order) instead of drawing."""
    global _mask_replay
    prev, _mask_replay = _mask_replay, [m for m in masks]
    try:
        yield
    finally:
        _mask_replay = prev


@contextlib.contextmanager
def dropout_record():
    """Collect the classifier-dropout masks drawn inside the context (fp32 [B, F], call order)."""
    global _mask_record
    prev, _mask_record = _mask_record, []
    try:
        yield _mask_record
    finally:
        _mask_record = prev


def dropout_mask(p, B, F_, device, inplace):
    """fp32 [B, F_] dropout mask (0 or 1 / (1 - p)) drawn with F.dropout on a tensor of ones, so that it consumes the
    generator as the reference's nn.Dropout(p, inplace) does: the in-place path draws a Bernoulli noise tensor and
    multiplies by it, the out-of-place one runs the fused native_dropout kernel.  Replayed / recorded under
    dropout_replay / dropout_record."""
    if _mask_replay is not None:
        if not _mask_replay:
            raise RuntimeError("dropout_replay: more classifier-dropout draws than recorded masks")
        m = _mask_replay.pop(0).to(device=device, dtype=torch.float32).contiguous()
        if tuple(m.shape) != (B, F_):
            raise RuntimeError("dropout_replay: mask of the wrong shape")
    else:
        m = F.dropout(torch.ones(B, F_, dtype=torch.float32, device=device), p, True, inplace=inplace)
    if _mask_record is not None:
        _mask_record.append(m.detach().clone())
    return m


def image_input(model, x):
    """fp32 NCHW image batch; a decoded uint8 NHWC batch (GPU input pipeline) gets ToTensor + Normalize on the device."""
    if x.dtype == torch.uint8:
        x = ops.normalize_u8_nhwc(x, *getattr(model, "input_norm", (ops.IMAGENET_MEAN, ops.IMAGENET_STD)))
    return x.contiguous().float()


class _EngineFunction(torch.autograd.Function):
    """The whole network as one autograd node: ``engine.forward`` records a tape, ``engine.backward`` replays it."""

    @staticmethod
    def forward(ctx, x, engine, model, *params):
        want_tape = any(ctx.needs_input_grad[3:])
        logits, tape = engine.forward(model, x, model.training, want_tape)
        ctx.engine, ctx.model, ctx.tape, ctx.params = engine, model, tape, params
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        if ctx.tape is None:
            raise RuntimeError("backward called on a forward that recorded no tape")
        grads = ctx.engine.backward(ctx.model, ctx.tape, dlogits)
        ctx.tape = None
        out = []
        for p, need in zip(ctx.params, ctx.needs_input_grad[3:]):
            gp = grads.get(p.data_ptr()) if need else None
            out.append(gp.reshape(p.shape) if gp is not None else None)
        return (None, None, None, *out)


def apply(engine, family, model, x):
    """``model(x)`` through the schedule module ``engine``: an autograd node when any parameter needs a gradient, else a
    forward that records no tape.  ``family`` names the network in the error raised for CPU input."""
    if not x.is_cuda:
        raise RuntimeError(f"deeplearning_b200 {family} runs on CUDA (sm_90a) tensors only; there is no CPU fallback")
    params = tuple(model.parameters())
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        return _EngineFunction.apply(x, engine, model, *params)
    logits, _ = engine.forward(model, x, model.training, False)
    return logits
