"""ShuffleNet v1 on the host, without a device: the five drop-in constructors (parameter names, blocks + 1 stages, the
ungrouped stage2.0, init), get_model / model_dict, every rejected admission case with its message, and the host-side
packing of the grouped 1x1 convolutions in fp32 on the CPU (the shuffle-permuted, padded block-diagonal operand and the
weight-gradient gather)."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from deeplearning_b200.classification.ShuffleNet import models as pkg
from deeplearning_b200.classification.ShuffleNet.models import shufflenetv1 as sn
from deeplearning_b200.engine import common
from deeplearning_b200.engine import shufflenet as eng

WIDTHS = {"g1": (1, [144, 288, 576]), "g2": (2, [200, 400, 800]), "g3": (3, [240, 480, 960]),
          "g4": (4, [272, 544, 1088]), "g8": (8, [384, 768, 1536])}


@pytest.mark.parametrize("name", list(WIDTHS))
def test_constructor_structure(name):
    g, outs = WIDTHS[name]
    m = getattr(sn, f"shufflenet_v1_x1_{name}")(num_classes=7)
    assert [len(m.stage2), len(m.stage3), len(m.stage4)] == [4, 8, 4]
    names = [n for n, _ in m.named_parameters()]
    assert "stage2.3.bn3.bias" in names and "stage3.7.group_conv.weight" in names and "stage4.3.bn1.weight" in names
    assert names[:3] == ["conv1.0.weight", "conv1.1.weight", "conv1.1.bias"] and names[-2:] == ["fc.weight", "fc.bias"]
    assert m.stage2[0].group_conv1.groups == 1 and m.stage2[0].group_conv.groups == 1
    assert all(m.stage2[i].groups == g for i in range(1, 4)) and m.stage3[0].group_conv1.groups == g
    assert m.stage2[0].group_conv.out_channels == outs[0] - 24
    assert m.stage4[-1].bn3.num_features == outs[2] and m.fc.in_features == outs[2] and m.fc.out_features == 7
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            assert torch.equal(mod.weight, torch.ones_like(mod.weight)) and torch.equal(mod.bias, torch.zeros_like(mod.bias))
    # kaiming_normal_(fan_out, relu): std sqrt(2 / fan_out)
    w = m.stage3[1].group_conv.weight.detach()
    assert abs(float(w.std()) - (2.0 / w.shape[0]) ** 0.5) < 0.15 * (2.0 / w.shape[0]) ** 0.5
    eng.check_model(m)


def test_get_model():
    assert set(pkg.model_dict) == {f"shufflenet_v1_g{g}" for g in (1, 2, 3, 4, 8)}
    assert pkg.get_model("shufflenet_v1_g3") is sn.shufflenet_v1_x1_g3


def test_forward_refuses_cpu():
    m = sn.shufflenet_v1_x1_g3(num_classes=5)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(1, 3, 32, 32))


def _raises(m, pattern):
    with pytest.raises(NotImplementedError, match=pattern):
        eng.check_model(m)


def test_admission_ratio_half():
    _raises(sn.shufflenet_v1_x1_g3(ratio=0.5), r"conv1: .*multiples of 8 .*stem=12")


def test_admission_ratio_breaking_block_widths():
    # ratio 1.5 at g3: stem 36
    _raises(sn.shufflenet_v1_x1_g3(ratio=1.5), r"conv1: .*stem=36")


def test_admission_structure():
    m = sn.shufflenet_v1_x1_g3()
    m.stage3[2].relu = nn.ReLU6()
    _raises(m, r"stage3\.2\.relu: expected nn.ReLU")
    m = sn.shufflenet_v1_x1_g3()
    m.stage3[0].avg_pool = nn.AvgPool2d(3, 2, 1, count_include_pad=False)
    _raises(m, r"stage3\.0\.avg_pool: expected AvgPool2d")
    m = sn.shufflenet_v1_x1_g3()
    m.maxpool = nn.MaxPool2d(2, 2)
    _raises(m, r"maxpool: expected MaxPool2d\(3, 2, 1\)")
    m = sn.shufflenet_v1_x1_g3()
    m.stage4[1].depthwise_conv3 = nn.Conv2d(240, 240, 5, padding=2, groups=240, bias=False)
    _raises(m, r"stage4\.1\.depthwise_conv3: expected a bias-free 3x3")
    m = sn.shufflenet_v1_x1_g3()
    m.extra = nn.Identity()
    _raises(m, r"ShuffleNetv1: expected the modules")
    m = sn.shufflenet_v1_x1_g3()
    m.stage2[1].dropout = nn.Dropout()
    _raises(m, r"stage2\.1: expected the reference's modules")
    m = sn.shufflenet_v1_x1_g3()
    m.fc = nn.Sequential(nn.Dropout(), nn.Linear(960, 5))
    _raises(m, r"fc: expected a Linear")


def test_admission_batchnorm():
    m = sn.shufflenet_v1_x1_g3()
    m.stage3[1].bn2 = nn.BatchNorm2d(120, affine=False)
    _raises(m, r"stage3\.1\.bn2: expected an affine BatchNorm2d")
    m = sn.shufflenet_v1_x1_g3()
    m.stage2[0].bn1 = nn.BatchNorm2d(54, track_running_stats=False)
    _raises(m, r"stage2\.0\.bn1: expected an affine BatchNorm2d .*running statistics")
    m = sn.shufflenet_v1_x1_g3()
    m.conv1[1] = nn.GroupNorm(3, 24)
    _raises(m, r"conv1\.1: expected an affine BatchNorm2d")


def test_admission_sync_batchnorm_multi_rank(monkeypatch):
    m = nn.SyncBatchNorm.convert_sync_batchnorm(sn.shufflenet_v1_x1_g3())
    eng.check_model(m)            # one process: admitted
    monkeypatch.setattr(common, "bn_sync", lambda bn: (None, 2) if isinstance(bn, nn.SyncBatchNorm) else None)
    _raises(m, r"conv1\.1: SyncBatchNorm in a multi-rank job is not implemented")


@pytest.mark.parametrize("cin,b,groups", [(24, 30, 1), (240, 60, 3), (200, 50, 2), (272, 68, 4), (384, 96, 8),
                                          (768, 192, 8)])
def test_group_conv1_packing(cin, b, groups):
    """the block-diagonal, shuffle-permuted, padded operand applied to x == shuffle_channels(group_conv1(x)) with zero pad
    channels, and the weight-gradient gather inverts it"""
    torch.manual_seed(cin + b)
    conv = nn.Conv2d(cin, b, 1, groups=groups, bias=False)
    bp = (b + 7) // 8 * 8
    idx = eng.dense_index(b, cin, groups, eng.shuffle_order(b, groups), bp, cin)
    dense = eng.dense_operand(conv.weight, idx)
    assert dense.shape == (bp, cin)
    x = torch.randn(2, cin, 3, 4)
    got = F.conv2d(x, dense.view(bp, cin, 1, 1))
    ref = sn.shuffle_channels(conv(x), groups)
    assert torch.allclose(got[:, :b], ref, atol=1e-5) and torch.equal(got[:, b:], torch.zeros_like(got[:, b:]))
    # block-diagonal: zero outside each row's group
    assert int((dense != 0).sum()) == conv.weight.numel()
    widx = eng.gather_index(idx, conv.weight.numel())
    assert torch.equal(dense.flatten()[widx].view(conv.weight.shape), conv.weight.detach())
    # the dense weight gradient, gathered, is the grouped one
    gy = torch.randn_like(ref)
    gw_ref, = torch.autograd.grad(sn.shuffle_channels(F.conv2d(x, conv.weight, groups=groups), groups), conv.weight, gy)
    gy_p = torch.cat([gy, torch.zeros(2, bp - b, 3, 4)], 1)
    dense_gw = torch.einsum("bnhw,bihw->ni", gy_p, x)
    assert torch.allclose(dense_gw.flatten()[widx].view(conv.weight.shape), gw_ref, atol=1e-4)


@pytest.mark.parametrize("b,cout,groups", [(60, 240, 3), (30, 120, 1), (68, 272, 4), (90, 360, 1)])
def test_group_conv_packing(b, cout, groups):
    torch.manual_seed(b)
    conv = nn.Conv2d(b, cout, 1, groups=groups, bias=False)
    bp = (b + 7) // 8 * 8
    idx = eng.dense_index(cout, b, groups, list(range(cout)), cout, bp)
    dense = eng.dense_operand(conv.weight, idx)
    a = torch.randn(2, b, 3, 3)
    a_p = torch.cat([a, torch.randn(2, bp - b, 3, 3)], 1)     # pad columns are zero: pad channels are ignored
    assert torch.allclose(F.conv2d(a_p, dense.view(cout, bp, 1, 1)), conv(a), atol=1e-5)
    widx = eng.gather_index(idx, conv.weight.numel())
    assert torch.equal(dense.flatten()[widx].view(conv.weight.shape), conv.weight.detach())


def test_shuffle_order_is_the_shuffle():
    for b, g in ((60, 3), (96, 8), (50, 2), (30, 1)):
        order = eng.shuffle_order(b, g)
        x = torch.arange(b, dtype=torch.float32).view(1, b, 1, 1)
        assert sn.shuffle_channels(x, g).flatten().tolist() == [float(o) for o in order]
