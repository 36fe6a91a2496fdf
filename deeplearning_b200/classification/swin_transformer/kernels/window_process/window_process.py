"""Drop-in for the reference's only first-party CUDA extension, ``kernels/window_process`` (SURVEY seam B2).

Replaces ``swin_window_process`` (the pybind module built by kernels/window_process/setup.py from swin_window_process.cpp:1-132
and swin_window_process_kernel.cu:1-354) and the two autograd Functions of kernels/window_process/window_process.py:11-63 with
the same names, argument order and semantics, on top of the 16-byte-vectorised sm_90a permutation kernels behind
``b200_window_partition`` / ``b200_window_merge`` (include/b200cls.h):

    roll_and_window_partition_forward(x, B, H, W, C, shift, ws)   == window_partition(torch.roll(x, (shift, shift), (1, 2)), ws)
    window_merge_and_roll_forward(xw, B, H, W, C, shift, ws)      == torch.roll(window_reverse(xw, ws, H, W), (shift, shift), (1, 2))
    *_backward(grad, B, H, W, C, shift, ws)                       == the inverse permutation of the matching forward

The training engine itself never calls these (engine/swin.py folds the roll + partition into the attention kernel's
addressing); they exist so that code written against the reference's fused_window_process API keeps working.
"""
import torch

from deeplearning_b200 import ops


def _chk(t):
    if not t.is_cuda:
        raise RuntimeError("swin_window_process: CUDA (sm_90a) tensors only; there is no CPU fallback")
    return t.contiguous()


class _SwinWindowProcess:
    """Namespace standing in for the compiled ``swin_window_process`` module."""

    @staticmethod
    def roll_and_window_partition_forward(input, B, H, W, C, shift_size, window_size):
        return ops.window_partition(_chk(input).view(B, H, W, C), shift_size, window_size)

    @staticmethod
    def roll_and_window_partition_backward(grad_in, B, H, W, C, shift_size, window_size):
        # inverse of out[win, wy, wx] = in[(h - shift) mod H, ...]: scatter back = merge with the same shift sign negated
        return ops.window_merge(_chk(grad_in), B, H, W, -shift_size, window_size)

    @staticmethod
    def window_merge_and_roll_forward(input, B, H, W, C, shift_size, window_size):
        return ops.window_merge(_chk(input), B, H, W, shift_size, window_size)

    @staticmethod
    def window_merge_and_roll_backward(grad_in, B, H, W, C, shift_size, window_size):
        return ops.window_partition(_chk(grad_in).view(B, H, W, C), -shift_size, window_size)


swin_window_process = _SwinWindowProcess()


class WindowProcess(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, B, H, W, C, shift_size, window_size):
        output = swin_window_process.roll_and_window_partition_forward(input, B, H, W, C, shift_size, window_size)
        ctx.B, ctx.H, ctx.W, ctx.C, ctx.shift_size, ctx.window_size = B, H, W, C, shift_size, window_size
        return output

    @staticmethod
    def backward(ctx, grad_in):
        grad_out = swin_window_process.roll_and_window_partition_backward(grad_in, ctx.B, ctx.H, ctx.W, ctx.C, ctx.shift_size,
                                                                          ctx.window_size)
        return grad_out, None, None, None, None, None, None, None


class WindowProcessReverse(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, B, H, W, C, shift_size, window_size):
        output = swin_window_process.window_merge_and_roll_forward(input, B, H, W, C, shift_size, window_size)
        ctx.B, ctx.H, ctx.W, ctx.C, ctx.shift_size, ctx.window_size = B, H, W, C, shift_size, window_size
        return output

    @staticmethod
    def backward(ctx, grad_in):
        grad_out = swin_window_process.window_merge_and_roll_backward(grad_in, ctx.B, ctx.H, ctx.W, ctx.C, ctx.shift_size,
                                                                      ctx.window_size)
        return grad_out, None, None, None, None, None, None, None
