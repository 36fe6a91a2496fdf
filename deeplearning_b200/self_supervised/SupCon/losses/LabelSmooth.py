"""Drop-in for the reference's self-supervised/SupCon/losses/LabelSmooth.py: cross-entropy against the target
distribution 1 - smoothing on the target class and smoothing / (classes - 1) on every other class (not timm's
smoothing / classes), on the fused soft-target cross-entropy kernel (ops.softmax_xent)."""
import torch
import torch.nn as nn

from .... import ops


class _SoftXentFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target):
        loss, d, _ = ops.softmax_xent(logits.detach().float(), target, want_grad=True)
        ctx.save_for_backward(d)
        ctx.shape = logits.shape
        ctx.l_dtype = logits.dtype
        return loss.view(())

    @staticmethod
    def backward(ctx, g):
        (d,) = ctx.saved_tensors
        B, N = ctx.shape
        return (ops.cast_f32(d)[:, :N] * g).to(ctx.l_dtype), None


class LabelSmoothingLoss(nn.Module):
    def __init__(self, classes, smoothing=0.0, dim=-1):
        super().__init__()
        self.confidence = 1.0 - smoothing
        self.smoothing = smoothing
        self.cls = classes
        self.dim = dim

    def forward(self, pred, target):
        from ....engine.supcon import smoothed_target

        if not pred.is_cuda:
            raise RuntimeError("deeplearning_b200 LabelSmoothingLoss runs on CUDA (sm_90a) tensors only; there is no CPU "
                               "fallback")
        if pred.dim() != 2 or self.dim not in (-1, 1):
            raise NotImplementedError("LabelSmoothingLoss: [B, classes] logits smoothed over dim -1 only")
        return _SoftXentFunction.apply(pred, smoothed_target(target, self.cls, self.smoothing, pred.shape[1]))
