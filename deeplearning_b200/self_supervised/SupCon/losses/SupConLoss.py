"""Drop-in for the reference's self-supervised/SupCon/losses/SupConLoss.py: the supervised contrastive loss
(https://arxiv.org/abs/2004.11362), and its unsupervised SimCLR form without labels, on the sm_90a SupCon kernels
(ops.supcon_loss / ops.supcon_loss_bwd).  ``contrast_mode='one'`` and an explicit ``mask`` are not implemented."""
import torch
import torch.nn as nn

from .... import ops


class _SupConFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e, row_labels, temperature, base_temperature):
        e32 = e.detach().float().contiguous()
        loss, L, npos = ops.supcon_loss(e32, row_labels, temperature, base_temperature)
        ctx.save_for_backward(e32, row_labels, L, npos)
        ctx.hyper = (temperature, base_temperature)
        ctx.e_dtype = e.dtype
        return loss.view(())

    @staticmethod
    def backward(ctx, g):
        e32, row_labels, L, npos = ctx.saved_tensors
        # the upstream gradient stays on the device (GradScaler's scale, graph capture): the kernel reads it
        de = ops.supcon_loss_bwd(e32, row_labels, L, npos, g.detach().float().reshape(1), *ctx.hyper)
        return de.to(ctx.e_dtype), None, None, None


class SupConLoss(nn.Module):
    """Supervised Contrastive Learning: https://arxiv.org/pdf/2004.11362.pdf.
    It also supports the unsupervised contrastive loss in SimCLR"""

    def __init__(self, temperature=0.07, contrast_mode="all", base_temperature=0.07):
        super().__init__()
        self.temperature = temperature
        self.contrast_mode = contrast_mode
        self.base_temperature = base_temperature

    def forward(self, features, labels=None, mask=None):
        """features [bsz, n_views, ...] (CUDA), labels [bsz] or None (SimCLR).  Returns the scalar loss."""
        from ....engine.supcon import row_labels

        if len(features.shape) < 3:
            raise ValueError("`features` needs to be [bsz, n_views, ...],at least 3 dimensions are required")
        if labels is not None and mask is not None:
            raise ValueError("Cannot define both `labels` and `mask`")
        if mask is not None:
            raise NotImplementedError("SupConLoss: an explicit contrastive `mask` is not implemented on the GPU engine")
        if self.contrast_mode == "one":
            raise NotImplementedError("SupConLoss: contrast_mode='one' is not implemented on the GPU engine")
        if self.contrast_mode != "all":
            raise ValueError("Unknown mode: {}".format(self.contrast_mode))
        if not features.is_cuda:
            raise RuntimeError("deeplearning_b200 SupConLoss runs on CUDA (sm_90a) tensors only; there is no CPU fallback")
        bsz, n_views = features.shape[:2]
        features = features.reshape(bsz, n_views, -1)
        if labels is not None and labels.numel() != bsz:
            raise ValueError("Num of labels does not match num of features")
        contrast = torch.cat(torch.unbind(features, dim=1), dim=0)
        return _SupConFunction.apply(contrast, row_labels(labels, bsz, n_views, features.device), self.temperature,
                                     self.base_temperature)
