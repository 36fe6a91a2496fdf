"""ShuffleNet v2 on the host, without a device: the four drop-in constructors (parameter names, stages, the split / joined
output of each block), get_model / model_dict, every rejected admission case with its message, the split / joined channel
maps of the block tails (with padding) against chunk / cat / channel_shuffle in fp32, the argument checks of the two C
entries, and loading torchvision's ShuffleNet v2 state_dict with strict=True."""
import pytest
import torch
import torch.nn as nn

from deeplearning_b200.classification.ShuffleNet.models import shufflenetv2 as sn
from deeplearning_b200.engine import common
from deeplearning_b200.engine import shufflenetv2 as eng

WIDTHS = {"x0_5": [48, 96, 192, 1024], "x1_0": [116, 232, 464, 1024], "x1_5": [176, 352, 704, 1024],
          "x2_0": [244, 488, 976, 2048]}


@pytest.mark.parametrize("name", list(WIDTHS))
def test_constructor_structure(name):
    outs = WIDTHS[name]
    m = getattr(sn, f"shufflenet_v2_{name}")(num_classes=7)
    assert [len(m.stage2), len(m.stage3), len(m.stage4)] == [4, 8, 4]
    names = [n for n, _ in m.named_parameters()]
    assert names[:3] == ["conv1.0.weight", "conv1.1.weight", "conv1.1.bias"] and names[-2:] == ["fc.weight", "fc.bias"]
    assert "stage2.0.branch1.2.weight" in names and "stage3.7.branch2.5.weight" in names
    assert "stage3.1.branch1.0.weight" not in names
    assert m.conv5[0].in_channels == outs[2] and m.conv5[0].out_channels == outs[3] and m.fc.in_features == outs[3]
    _, _, blocks, conv5, _, fc = eng.check_model(m)
    assert len(blocks) == 16 and conv5 is m.conv5[0] and fc is m.fc
    # a block writes split output iff the next block has stride 1: all but the last block of each stage
    assert [k.split for k in blocks] == [True] * 3 + [False] + [True] * 7 + [False] + [True] * 3 + [False]
    assert [k.b for k in blocks[::4]] == [outs[0] // 2, outs[1] // 2, outs[1] // 2, outs[2] // 2]


def test_get_model_and_exports():
    assert set(sn.model_dict) == {f"shufflenet_v2_{n}" for n in WIDTHS}
    assert sn.get_model("shufflenet_v2_x1_0") is sn.shufflenet_v2_x1_0
    assert set(sn.__all__) == {"ShuffleNetV2"} | {f"shufflenet_v2_{n}" for n in WIDTHS}
    assert sn.model_urls["shufflenetv2_x1.0"].endswith("shufflenetv2_x1-5666bf0f80.pth")
    with pytest.raises(AssertionError):
        sn.get_model("shufflenet_v2_x3_0")


def test_forward_refuses_cpu():
    m = sn.shufflenet_v2_x1_0(num_classes=5)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 3, 32, 32))


def test_block_forward_is_the_reference():
    """InvertedResidual.forward stays the reference's PyTorch code for direct callers"""
    torch.manual_seed(0)
    blk = sn.InvertedResidual(48, 48, 1).eval()
    x = torch.randn(2, 48, 5, 5)
    x1, x2 = x.chunk(2, dim=1)
    ref = sn.channel_shuffle(torch.cat((x1, blk.branch2(x2)), 1), 2)
    assert torch.equal(blk(x), ref)


def _raises(m, pattern):
    with pytest.raises(NotImplementedError, match=pattern):
        eng.check_model(m)


def test_admission_stride3():
    m = sn.shufflenet_v2_x1_0()
    m.stage3[0] = sn.InvertedResidual(116, 232, 3)
    _raises(m, r"^stage3\.0: stride 3 is not implemented")


def test_admission_odd_branch_width():
    m = sn.ShuffleNetV2([4, 8, 4], [24, 118, 236, 472, 1024])
    _raises(m, r"^stage2\.0: the GPU engine needs an even branch width \(got 59\)")


def test_admission_stem_width():
    m = sn.ShuffleNetV2([4, 8, 4], [20, 48, 96, 192, 1024])
    _raises(m, r"^conv1: the GPU engine needs a stem width that is a multiple of 8 \(got 20\)")


def test_admission_structure():
    m = sn.shufflenet_v2_x1_0()
    m.extra = nn.Identity()
    _raises(m, r"^ShuffleNetV2: expected the modules")

    class Other(nn.Module):
        def __init__(self, blk):
            super().__init__()
            self.branch1, self.branch2, self.stride = blk.branch1, blk.branch2, blk.stride

    m = sn.shufflenet_v2_x1_0()
    m.stage3[2] = Other(m.stage3[2])
    _raises(m, r"^stage3\.2: expected the reference's InvertedResidual \(got Other\)")
    m = sn.shufflenet_v2_x1_0()
    m.stage4[1].branch2[2] = nn.ReLU6()
    _raises(m, r"^stage4\.1\.branch2: expected the reference's Sequential")
    m = sn.shufflenet_v2_x1_0()
    m.stage2[0].branch1[0] = nn.Conv2d(24, 24, 5, 2, 2, groups=24, bias=False)
    _raises(m, r"^stage2\.0\.branch1\.0: expected a bias-free 3x3")
    m = sn.shufflenet_v2_x1_0()
    m.stage2[1].dropout = nn.Dropout()
    _raises(m, r"^stage2\.1: expected the reference's modules")
    m = sn.shufflenet_v2_x1_0()
    m.maxpool = nn.MaxPool2d(2, 2)
    _raises(m, r"^maxpool: expected MaxPool2d\(3, 2, 1\)")
    m = sn.shufflenet_v2_x1_0()
    m.conv5[2] = nn.GELU()
    _raises(m, r"^conv5: expected the reference's Sequential")
    m = sn.shufflenet_v2_x1_0()
    m.fc = nn.Sequential(nn.Dropout(), nn.Linear(1024, 5))
    _raises(m, r"^fc: expected a Linear")


def test_admission_batchnorm():
    m = sn.shufflenet_v2_x1_0()
    m.stage3[1].branch2[4] = nn.BatchNorm2d(116, affine=False)
    _raises(m, r"^stage3\.1\.branch2\.4: expected an affine BatchNorm2d")
    m = sn.shufflenet_v2_x1_0()
    m.stage2[0].branch1[1] = nn.BatchNorm2d(24, track_running_stats=False)
    _raises(m, r"^stage2\.0\.branch1\.1: expected an affine BatchNorm2d .*running statistics")
    m = sn.shufflenet_v2_x1_0()
    m.conv5[1] = nn.GroupNorm(8, 1024)
    _raises(m, r"^conv5\.1: expected an affine BatchNorm2d")


def test_admission_sync_batchnorm_multi_rank(monkeypatch):
    m = nn.SyncBatchNorm.convert_sync_batchnorm(sn.shufflenet_v2_x1_0())
    eng.check_model(m)            # one process: admitted
    monkeypatch.setattr(common, "bn_sync", lambda bn: (None, 2) if isinstance(bn, nn.SyncBatchNorm) else None)
    _raises(m, r"^conv1\.1: SyncBatchNorm in a multi-rank job is not implemented")


@pytest.mark.parametrize("b", [24, 58, 88, 116, 122, 232, 244, 488])
def test_tail_layout_is_chunk_cat_shuffle(b):
    """the joined output is channel_shuffle(cat(u, v), 2) in reference order; the split halves are its chunk(2), so a
    stride-1 block's (x1, x2) = (P', Q'); every pad channel is 0"""
    bp = (b + 7) // 8 * 8
    torch.manual_seed(b)
    u = torch.cat([torch.randn(2, 3, 4, b), torch.zeros(2, 3, 4, bp - b)], -1)
    v = torch.cat([torch.randn(2, 3, 4, b), torch.zeros(2, 3, 4, bp - b)], -1)
    ref = sn.channel_shuffle(torch.cat((u[..., :b], v[..., :b]), -1).permute(0, 3, 1, 2), 2)   # NCHW
    joined = eng.tail_layout(u, v, b, split=False)
    J = (2 * b + 7) // 8 * 8
    assert joined.shape[-1] == J
    assert torch.equal(joined[..., :2 * b].permute(0, 3, 1, 2), ref)
    assert torch.equal(joined[..., 2 * b:], torch.zeros_like(joined[..., 2 * b:]))
    P, Q = eng.tail_layout(u, v, b, split=True)
    x1, x2 = ref.chunk(2, dim=1)
    assert torch.equal(P[..., :b].permute(0, 3, 1, 2), x1) and torch.equal(Q[..., :b].permute(0, 3, 1, 2), x2)
    assert not P[..., b:].any() and not Q[..., b:].any()
    # the zip identities of the split halves
    h = b // 2
    assert torch.equal(P[..., 0:b:2], u[..., :h]) and torch.equal(P[..., 1:b:2], v[..., :h])
    assert torch.equal(Q[..., 0:b:2], u[..., h:b]) and torch.equal(Q[..., 1:b:2], v[..., h:b])


# --------------------------------------------------------------------------------------------------- C entry checks
F_ = 1 << 20    # 16-byte aligned, never dereferenced: every call below fails its argument checks first


def _rejects(call, msg):
    from deeplearning_b200 import _lib as L

    assert call(L.load()) == -1
    assert msg in L.last_error(), L.last_error()


def test_tail_entries_reject_arguments():
    fwd = lambda L, *a: L.b200_shufflev2_tail_fwd(*a, None)        # noqa: E731
    bwd = lambda L, *a: L.b200_shufflev2_tail_bwd(*a, None)        # noqa: E731
    ok = (F_, None, None, F_, F_, F_, F_, None)
    _rejects(lambda L: fwd(L, *ok, 64, 29, 32), "b must be even")
    _rejects(lambda L: fwd(L, *ok, 64, 0, 8), "b must be even")
    _rejects(lambda L: fwd(L, *ok, 64, 58, 60), "bp must be a multiple of 8 >= b")
    _rejects(lambda L: fwd(L, *ok, 64, 58, 56), "bp must be a multiple of 8 >= b")
    _rejects(lambda L: fwd(L, *ok, 0, 58, 64), "rows must be in")
    _rejects(lambda L: fwd(L, *ok, 64, 4098, 4104), "at most 8192")
    _rejects(lambda L: fwd(L, F_ + 2, None, None, F_, F_, F_, F_, None, 64, 58, 64), "16-byte aligned")
    _rejects(lambda L: fwd(L, F_, None, None, F_, F_, None, F_, None, 64, 58, 64), "16-byte aligned")
    _rejects(lambda L: fwd(L, F_, F_, None, F_, F_, F_, F_, None, 64, 58, 64), "given together")
    _rejects(lambda L: fwd(L, F_, None, None, F_, F_, F_, F_, F_ + 8, 64, 58, 64), "y1 must be 16-byte aligned")
    okb = (F_, None, F_, F_, F_, F_, F_, None, None, None, F_, None)
    _rejects(lambda L: bwd(L, *okb, 64, 61, 64), "b must be even")
    _rejects(lambda L: bwd(L, *okb, 64, 58, 63), "bp must be a multiple of 8 >= b")
    _rejects(lambda L: bwd(L, F_, None, F_, F_, F_, F_, None, None, None, None, F_, None, 64, 58, 64), "partial3 non-null")
    _rejects(lambda L: bwd(L, F_, None, F_, F_, F_, F_ + 4, F_, None, None, None, F_, None, 64, 58, 64), "16-byte aligned")
    _rejects(lambda L: bwd(L, F_, None, F_, F_, F_, F_, F_, F_, F_, F_, F_, None, 64, 58, 64), "given together")
    _rejects(lambda L: bwd(L, F_, None, F_, F_, F_, F_, F_, None, None, None, F_, F_, 64, 58, 64), "given together")
    _rejects(lambda L: bwd(L, F_, F_ + 8, F_, F_, F_, F_, F_, None, None, None, F_, None, 64, 58, 64),
             "g1 must be 16-byte aligned")


def test_torchvision_state_dict_loads_strict():
    """checkpoint compatibility: torchvision's shufflenet_v2_x1_0 (built without weights) loads into the drop-in with
    strict=True, and the parameters arrive in place"""
    tv = pytest.importorskip("torchvision")
    ref = tv.models.shufflenet_v2_x1_0(weights=None)
    m = sn.get_model("shufflenet_v2_x1_0")()
    sd = ref.state_dict()
    m.load_state_dict(sd, strict=True)
    mine = m.state_dict()
    assert list(mine) == list(sd) and all(torch.equal(mine[k], sd[k]) for k in sd)
    eng.check_model(m)
