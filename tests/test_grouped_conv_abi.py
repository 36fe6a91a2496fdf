"""Grouped 3x3 convolution entries of the C ABI without a device: the host-side planners, and B200_EINVAL with a message for
shapes outside the grouped kernels' scope (checked before anything is launched). Also the engine's admission of grouped
convolutions."""
import pytest
import torch.nn as nn


def _lib():
    from deeplearning_b200 import _lib

    return _lib, _lib.load()


def test_grouped_stats_rows_follow_64_channel_tiles():
    # without a device the planners assume the 132 SMs of an H100 SXM; the grouped kernel always runs 64-channel tiles, so its
    # statistics rows are (132 // (C / 64)) CTA groups x 8 rows, which differs from the dense planner's 128-channel tiles
    _, lib = _lib()
    for C, groups in [(128, 32), (256, 32), (1024, 32), (1280, 40), (2048, 32)]:
        rows = lib.b200_conv2d_grouped_fwd_stats_rows(256, 56, 56, C, groups, 3, 1)
        assert rows == 132 // (C // 64) * 8, (C, rows)
    assert lib.b200_conv2d_grouped_fwd_stats_rows(256, 56, 56, 1280, 40, 3, 1) != lib.b200_conv2d_fwd_stats_rows(256, 56, 56, 1280, 3, 1)
    assert lib.b200_conv2d_grouped_fwd_stats_rows(1, 8, 8, 64, 16, 3, 1) == 8      # one tile: one CTA


def test_grouped_wgrad_workspace_is_split_diagonal_blocks():
    """workspace = splits x C x 9 taps x 64 columns x 4 bytes: only the diagonal 64-channel blocks, never C x C"""
    _, lib = _lib()
    for B, H, C, groups, s in [(256, 56, 128, 32, 1), (256, 56, 256, 32, 2), (256, 14, 1024, 32, 1), (256, 7, 2048, 32, 1),
                               (1, 7, 64, 16, 1)]:
        nbytes = lib.b200_conv2d_grouped_wgrad_workspace_bytes(B, H, H, C, groups, 3, s)
        unit = C * 9 * 64 * 4
        assert nbytes > 0 and nbytes % unit == 0, (C, nbytes)
        splits = nbytes // unit
        Ho = (H - 1) // s + 1
        assert 1 <= splits <= max(1, -(-B * Ho * Ho // 64) // 4), (C, splits)
        items = -(-C // 128) * 3 * splits
        assert items <= 2 * 132, ("more than two waves", C, splits)


@pytest.mark.parametrize("C,groups,ksize,stride,msg", [
    (64, 32, 3, 1, "group width"),       # Cg = 2
    (256, 2, 3, 1, "group width"),       # Cg = 128
    (96, 24, 3, 1, "multiple of 64"),    # C % 64 != 0
    (128, 32, 1, 1, "ksize"),
    (128, 32, 3, 3, "stride"),
    (128, 0, 3, 1, "multiple of 64"),    # groups = 0
])
def test_grouped_entries_reject_out_of_scope_shapes(C, groups, ksize, stride, msg):
    _l, lib = _lib()
    rc = lib.b200_conv2d_grouped_fwd(None, None, None, 2, 8, 8, C, groups, ksize, stride, None, 0, None, None, None)
    assert rc == -1 and msg in _l.last_error(), _l.last_error()
    rc = lib.b200_conv2d_grouped_dgrad(None, None, None, 2, 8, 8, C, groups, ksize, stride, None, None)
    assert rc == -1 and msg in _l.last_error(), _l.last_error()
    rc = lib.b200_conv2d_grouped_wgrad(None, None, None, None, 0, 2, 8, 8, C, groups, ksize, stride, 0, None)
    assert rc == -1 and msg in _l.last_error(), _l.last_error()
    assert lib.b200_conv2d_grouped_fwd_stats_rows(2, 8, 8, C, groups, ksize, stride) == -1
    assert lib.b200_conv2d_grouped_wgrad_workspace_bytes(2, 8, 8, C, groups, ksize, stride) == 0


def test_grouped_pack_modes_validate_shapes():
    _l, lib = _lib()
    assert lib.b200_pack_weight(None, None, 96, 4, 9, 3, 576, None) == -1 and "grouped" in _l.last_error()
    assert lib.b200_pack_weight(None, None, 128, 128, 9, 4, 576, None) == -1
    assert lib.b200_pack_weight(None, None, 128, 4, 9, 3, 500, None) == -1 and "ld_dst" in _l.last_error()


def test_engine_admits_resnext_convs_only_in_scope():
    from deeplearning_b200.classification.resnet.models.networks import resnext50_32x4d, resnext101_32x8d
    from deeplearning_b200.engine.resnet import _check_conv

    for m in (resnext50_32x4d(), resnext101_32x8d()):
        for name, mod in m.named_modules():
            if isinstance(mod, nn.Conv2d) and name != "conv1":
                _check_conv(mod, name)
    for bad in [nn.Conv2d(64, 64, 3, 1, 1, groups=32, bias=False),             # Cg = 2
                nn.Conv2d(256, 256, 3, 1, 1, groups=2, bias=False),            # Cg = 128
                nn.Conv2d(96, 96, 3, 1, 1, groups=24, bias=False),             # C % 64
                nn.Conv2d(128, 256, 3, 1, 1, groups=32, bias=False),           # C_in != C_out
                nn.Conv2d(128, 128, 1, 1, 0, groups=32, bias=False),           # 1x1
                nn.Conv2d(128, 128, 3, 1, 2, dilation=2, groups=32, bias=False),
                nn.Conv2d(128, 128, 3, 1, 2, dilation=2, bias=False)]:
        with pytest.raises(NotImplementedError):
            _check_conv(bad, "conv")
