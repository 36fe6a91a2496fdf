"""Epilogue options of the convolution entries are call arguments: a call that is rejected leaves nothing behind for the
next call on the same thread. A failed eval-mode conv + BatchNorm (unsupported kernel size, grouped shape out of scope) is
followed by plain convolutions that must reproduce their earlier outputs and statistics bit for bit. Only host-side
B200_EINVAL returns are provoked; nothing invalid is launched."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_rejected_bn_fold_does_not_reach_the_next_conv():
    from deeplearning_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(2, 8, 8, 64, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(64, 64, 3, 3, device="cuda", generator=g) * (64 * 9) ** -0.5
    wp = ops.pack_weight(w)
    co = ops.BnCoeffs(64, "cuda")
    co.scale.copy_(torch.rand(64, device="cuda", generator=g) + 0.5)
    co.shift.copy_(torch.randn(64, device="cuda", generator=g))

    y_ref, _ = ops.conv2d_fwd(x, wp, 3, 1)
    ys_ref, st_ref = ops.conv2d_fwd(x, wp, 3, 1, want_stats=True)
    rejected = [lambda: ops.conv2d_bn_act(x, wp, co, 5, 1),              # 5x5 is not supported
                lambda: ops.conv2d_bn_act(x, wp, co, 3, 1, groups=32)]   # group width 2 is out of the grouped scope
    for bad in rejected:
        with pytest.raises(RuntimeError):
            bad()
        y, _ = ops.conv2d_fwd(x, wp, 3, 1)
        torch.cuda.synchronize()
        assert torch.equal(y, y_ref)
        with pytest.raises(RuntimeError):
            bad()
        ys, st = ops.conv2d_fwd(x, wp, 3, 1, want_stats=True)
        torch.cuda.synchronize()
        assert torch.equal(ys, ys_ref) and torch.equal(st, st_ref)
