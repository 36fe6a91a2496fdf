"""Forward / backward schedule of supervised contrastive learning on the sm_90a kernels (one autograd node for the network).

Mirrors ``SupConModel.forward`` of the reference (self-supervised/SupCon/models/model.py) with a ResNet encoder (the
``nn.Sequential`` of a ResNet's children without fc; engine/resnet.py runs it as a Trunk):

    stage 1   trunk -> pooled bf16 [B, F] -> head.0 GEMM (+bias, ReLU in the epilogue) -> head.2 GEMM (+bias, fp32 out)
              -> row L2 normalisation (fp32 unit embeddings); with the projection head off the pooled features are
              normalised directly
              loss (TrainStep): the SupCon loss over the 2B rows of cat(view1, view2) (ops.supcon_loss), whose backward
              writes the fp32 embedding gradient; the backward is the exact reverse, the head's ReLU as a mask pass
    stage 2   the encoder is frozen: the trunk runs with train-mode BatchNorm (running statistics updated) and records no
              tape; only ``classifier`` gets gradients.  Loss (TrainStep): the reference's LabelSmoothingLoss as the fused
              soft-target cross-entropy against 1 - s on the target class and s / (classes - 1) elsewhere
"""
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common, resnet
from .common import linear_grads
from .packing import weight_cache


def _trunk(model):
    return resnet.Trunk(model.encoder, "encoder")


class _PackSpec:
    @staticmethod
    def key(model):
        tail = (id(model.classifier), model.classifier.out_features) if model.second_stage else (id(model.head),)
        return (model.second_stage, id(model.encoder)) + tail

    def __call__(self, model):
        specs = resnet.conv_pack_specs(model.encoder, model.encoder[0])
        if model.second_stage:
            return specs + common.head_pack_specs(model.classifier)
        for lin in (model.head[0], model.head[2]):
            w = lin.weight
            specs.append((w, 0, w.shape[1], w.shape[0]))
            specs.append((w, 1, w.shape[0], w.shape[1]))
        return specs


_pack_spec = _PackSpec()


def params_without_grad(model):
    """The frozen encoder of the second stage: no gradient, optimizer state, decay or all-reduce."""
    return list(model.encoder.parameters()) if model.second_stage else []


def _check(model, want_tape):
    enc = list(model.encoder.parameters())
    frozen = [not p.requires_grad for p in enc]
    if any(frozen) and not all(frozen):
        raise NotImplementedError("encoder: a partially frozen encoder is not implemented on the GPU engine; freeze every "
                                  "encoder parameter (second stage) or none (first stage)")
    if model.second_stage:
        if not all(frozen):
            raise NotImplementedError("encoder: the second stage trains the classifier on a frozen encoder; set "
                                      "requires_grad=False on every encoder parameter")
        return
    if any(frozen) and want_tape:
        raise NotImplementedError("encoder: the first stage trains the encoder; a frozen encoder under a trainable "
                                  "projection head is not implemented")
    h0, relu, h2 = model.head
    if not (type(h0) is nn.Linear and isinstance(relu, nn.ReLU) and type(h2) is nn.Linear and h0.bias is not None
            and h2.bias is not None):
        raise NotImplementedError("head: the GPU engine runs the projection head Linear -> ReLU -> Linear with biases")
    for name, lin in (("head.0", h0), ("head.2", h2)):
        if lin.in_features % 8 or lin.out_features % 8:
            raise NotImplementedError(f"{name}: Linear {lin.in_features} -> {lin.out_features}; the GEMM kernels take "
                                      "widths that are multiples of 8")
    D = h2.out_features if model.projection_head else h0.in_features
    if want_tape and D > ops.supcon_max_dim():
        raise NotImplementedError(f"embedding width {D}; the SupCon loss kernels take at most {ops.supcon_max_dim()}")


def forward(model, x, train, want_tape):
    """Returns (stage 1: fp32 unit embeddings [B, embed_dim]; stage 2: fp32 logits [B, num_classes], tape or None)."""
    _check(model, want_tape)
    x, x_hw, u8 = resnet.image_batch(x)
    pack = weight_cache.model_pack(model, _pack_spec)
    trunk = _trunk(model)
    norm = getattr(model, "input_norm", (ops.IMAGENET_MEAN, ops.IMAGENET_STD))
    if model.second_stage:
        pooled, _ = resnet.trunk_forward(trunk, pack, x, x_hw, u8, train, False, norm)
        logits = common.head_forward(pack, model.classifier, pooled)
        return logits, ({"stage": 2, "pack": pack, "pooled": pooled} if want_tape else None)
    pooled, ttape = resnet.trunk_forward(trunk, pack, x, x_hw, u8, train, want_tape, norm)
    h1 = None
    if model.projection_head:
        h0, h2 = model.head[0], model.head[2]
        h1, _ = ops.gemm(pooled, pack.get(h0.weight, 0), bias=h0.bias, act=1)
        z, _ = ops.gemm(h1, pack.get(h2.weight, 0), bias=h2.bias, out_f32=True)
    else:
        z = ops.cast_f32(pooled)
    e, nrm = ops.supcon_normalize(z)
    tape = None
    if want_tape:
        tape = {"stage": 1, "pack": pack, "trunk": ttape, "pooled": pooled, "h1": h1, "e": e, "nrm": nrm}
    return e, tape


def row_labels(labels, bsz, n_views, device):
    """int32 labels [n_views * bsz] of the contrast rows cat(unbind(features, 1)) (row v * bsz + b is sample b); without
    labels every sample is its own class (SimCLR)."""
    if labels is None:
        base = torch.arange(bsz, dtype=torch.int32, device=device)
    else:
        if labels.numel() != bsz:
            raise ValueError(f"Num of labels does not match num of features ({labels.numel()} labels, {bsz} samples)")
        base = labels.reshape(bsz).to(device=device, dtype=torch.int32)
    return base.repeat(n_views)


def smoothed_target(labels, classes, smoothing, n_cols):
    """fp32 [B, classes] target of the reference's LabelSmoothingLoss: 1 - smoothing at the label, smoothing / (classes - 1)
    elsewhere."""
    if n_cols != classes:
        raise ValueError(f"LabelSmoothingLoss(classes={classes}) on logits with {n_cols} columns")
    t = torch.full((labels.shape[0], classes), smoothing / (classes - 1), dtype=torch.float32, device=labels.device)
    return t.scatter_(1, labels.reshape(-1, 1).long(), 1.0 - smoothing)


def check_criterion(model, criterion):
    """ValueError unless ``criterion`` is the loss of the model's stage: SupConLoss (stage 1), LabelSmoothingLoss or None
    (stage 2; None is plain cross-entropy)."""
    from ..self_supervised.SupCon.losses.LabelSmooth import LabelSmoothingLoss
    from ..self_supervised.SupCon.losses.SupConLoss import SupConLoss

    if model.second_stage:
        if criterion is not None and not isinstance(criterion, LabelSmoothingLoss):
            raise ValueError(f"a second-stage SupConModel trains with LabelSmoothingLoss or plain cross-entropy (None), "
                             f"got {type(criterion).__name__}")
        if criterion is not None and criterion.cls != model.classifier.out_features:
            raise ValueError(f"LabelSmoothingLoss(classes={criterion.cls}) for a classifier with "
                             f"{model.classifier.out_features} classes")
        return
    if not isinstance(criterion, SupConLoss):
        raise ValueError(f"a first-stage SupConModel trains with criterion=SupConLoss(...), got {type(criterion).__name__}")
    if criterion.contrast_mode != "all":
        raise NotImplementedError(f"SupConLoss: contrast_mode={criterion.contrast_mode!r} is not implemented on the GPU engine")


def train_loss(out, labels, loss_scale, criterion):
    """TrainStep's loss.  Stage 1: out are the embeddings of cat(view1, view2) [2B, D], labels [B] or None;
    returns (loss, fp32 embedding gradient, None).  Stage 2: (loss, bf16 logit gradient, correct)."""
    if criterion is not None and hasattr(criterion, "temperature"):   # SupConLoss
        rows = out.shape[0]
        if rows % 2:
            raise ValueError(f"SupCon step: {rows} images; the batch must be cat(view1, view2) of two views per sample")
        B = rows // 2
        if labels is not None and labels.numel() != B:
            raise ValueError(f"SupCon step: {rows} images need {B} labels (two views per sample), got {labels.numel()}")
        lab = row_labels(labels, B, 2, out.device)
        tau, base = float(criterion.temperature), float(criterion.base_temperature)
        loss, L, npos = ops.supcon_loss(out, lab, tau, base)
        one = torch.ones(1, dtype=torch.float32, device=out.device)
        de = ops.supcon_loss_bwd(out, lab, L, npos, one, tau, base, grad_scale=loss_scale)
        return loss, de, None
    n_cls = out.shape[1]
    target = labels if criterion is None else smoothed_target(labels, criterion.cls, criterion.smoothing, n_cls)
    return ops.softmax_xent(out, target, want_grad=True, ld_d=common.padded_classes(n_cls), loss_scale=loss_scale)


def backward(model, tape, dout, sink=None):
    grads = common.Grads(sink)
    pack = tape["pack"]
    if tape["stage"] == 2:
        common.head_backward(grads, pack, model.classifier, tape["pooled"], dout)
        return grads
    de = dout.contiguous().float()
    dz = ops.supcon_normalize_bwd(de, tape["e"], tape["nrm"])
    pooled, h1 = tape["pooled"], tape["h1"]
    if h1 is not None:
        h0, h2 = model.head[0], model.head[2]
        linear_grads(grads, h2, dz, h1)
        dh1, _ = ops.gemm(dz, pack.get(h2.weight, 1))
        dh1 = ops.relu_bwd(dh1, h1)
        linear_grads(grads, h0, dh1, pooled)
        dpooled, _ = ops.gemm(dh1, pack.get(h0.weight, 1))
    else:
        dpooled = dz
    resnet.trunk_backward(_trunk(model), tape["trunk"], dpooled, grads)
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "SupConModel", model, x)
