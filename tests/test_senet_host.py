"""Device-free checks of SE-ResNet: the drop-in constructors' parameters, checkpoint round trip and options, the engine's
admission of SE layers, and the argument checks of the squeeze-and-excitation C entries (they reject a shape with
B200_EINVAL and a message before touching the device, so fake pointers are never dereferenced)."""
import pytest
import torch
import torch.nn as nn


def _nets():
    from deeplearning_b200.classification.seNet.models import networks

    return networks


def test_se_resnet50_state_dict_keys_and_shapes():
    m = _nets().se_resnet50()
    sd = m.state_dict()
    params = list(m.parameters())
    assert len(params) == 193 and sum(p.numel() for p in params) == 28_071_976
    assert list(m.layer1[0]._modules) == ["conv1", "bn1", "conv2", "bn2", "conv3", "bn3", "relu", "se", "downsample"]
    for li, (C, n) in enumerate([(256, 3), (512, 4), (1024, 6), (2048, 3)], start=1):
        for bi in range(n):
            p = f"layer{li}.{bi}.se.fc"
            assert sd[f"{p}.0.weight"].shape == (C // 16, C) and sd[f"{p}.2.weight"].shape == (C, C // 16)
            assert f"{p}.0.bias" not in sd and f"{p}.2.bias" not in sd


def test_se_resnet18_state_dict_keys_and_shapes():
    m = _nets().se_resnet()
    params = list(m.parameters())
    assert len(params) == 78 and sum(p.numel() for p in params) == 11_776_552
    assert list(m.layer2[0]._modules) == ["conv1", "bn1", "relu", "conv2", "bn2", "se", "downsample"]
    assert m.layer1[0].se.fc[0].weight.shape == (4, 64) and m.layer4[1].se.fc[2].weight.shape == (512, 32)


def test_strict_round_trip_and_pretrained_raises():
    nets = _nets()
    torch.manual_seed(3)
    a = nets.se_resnet50(num_classes=10)
    torch.manual_seed(4)
    b = nets.se_resnet50(num_classes=10)
    b.load_state_dict(a.state_dict(), strict=True)
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k
    with pytest.raises(RuntimeError):
        nets.se_resnet50(pretrained=True)


def test_zero_init_residual_leaves_se_blocks_alone():
    from deeplearning_b200.classification.resnet.models.networks import BasicBlock, Bottleneck, ResNet

    nets = _nets()
    for block, last in [(nets.SEBottleneck, "bn3"), (nets.SEBasicBlock, "bn2")]:
        assert not issubclass(block, (Bottleneck, BasicBlock))
        m = ResNet(block, [1, 1, 1, 1], zero_init_residual=True)
        for layer in (m.layer1, m.layer4):
            assert torch.equal(getattr(layer[0], last).weight, torch.ones_like(getattr(layer[0], last).weight))


def test_block_forward_raises():
    nets = _nets()
    m = nets.se_resnet()
    with pytest.raises(RuntimeError):
        m.layer1[0](torch.zeros(1, 64, 8, 8))
    with pytest.raises(RuntimeError):
        m.layer1[0].se(torch.zeros(1, 64, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 32, 32))


def test_engine_admission_rejects_malformed_se_layer():
    from deeplearning_b200.engine.resnet import _check_se
    from deeplearning_b200.classification.seNet.models.se_module import SELayer

    _check_se(SELayer(256), 256, "ok")
    _check_se(SELayer(64, 16), 64, "ok")
    bad = []
    se = SELayer(256)
    se.fc[0] = nn.Linear(256, 16, bias=True)               # biased squeeze
    bad.append((se, 256))
    se = SELayer(256)
    se.fc[3] = nn.Tanh()                                    # wrong gate nonlinearity
    bad.append((se, 256))
    se = SELayer(256)
    se.fc[1] = nn.GELU()
    bad.append((se, 256))
    se = SELayer(256)
    se.fc = nn.Sequential(*list(se.fc)[:3])                 # no sigmoid
    bad.append((se, 256))
    se = SELayer(256)
    se.fc[2] = nn.Linear(32, 256, bias=False)               # hidden widths do not match
    bad.append((se, 256))
    bad.append((SELayer(256), 512))                         # layer width differs from the tail's channels
    bad.append((SELayer(96, 16), 96))                       # C % 64 != 0
    bad.append((SELayer(2048, 4), 2048))                    # Cr = 512 > 256
    se = SELayer(256)
    se.avg_pool = nn.AdaptiveMaxPool2d(1)
    bad.append((se, 256))
    for se, C in bad:
        with pytest.raises(NotImplementedError):
            _check_se(se, C, "layer")


# ------------------------------------------------------------------------------------------- C entries, without a device
FAKE = 1 << 12   # 16-byte aligned, never dereferenced: every case below fails its shape check first


def _call(name, B=2, HW=49, C=256, Cr=16):
    from deeplearning_b200 import _lib

    lib = _lib.load()
    f = FAKE
    if name == "b200_se_squeeze":
        return lib.b200_se_squeeze(f, f, f, f, f, B, HW, C, None)
    if name == "b200_se_excite":
        return lib.b200_se_excite(f, f, f, f, f, B, C, Cr, None)
    if name == "b200_se_apply":
        return lib.b200_se_apply(f, f, f, f, f, f, B, HW, C, None)
    if name == "b200_se_bwd_reduce":
        return lib.b200_se_bwd_reduce(f, f, f, f, f, f, B, HW, C, None)
    if name == "b200_se_bwd_coeffs":
        return lib.b200_se_bwd_coeffs(*([f] * 12), B, HW, C, Cr, *([f] * 8), None)
    if name == "b200_se_bwd_apply":
        return lib.b200_se_bwd_apply(*([f] * 10), B, HW, C, None)
    raise AssertionError(name)


ENTRIES = ["b200_se_squeeze", "b200_se_excite", "b200_se_apply", "b200_se_bwd_reduce", "b200_se_bwd_coeffs",
           "b200_se_bwd_apply"]
WITH_HW = [e for e in ENTRIES if e != "b200_se_excite"]
WITH_CR = ["b200_se_excite", "b200_se_bwd_coeffs"]


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("C", [96, 32, 0])
def test_entries_reject_channel_count(entry, C):
    from deeplearning_b200 import _lib

    assert _call(entry, C=C) == -1
    assert "C must be a positive multiple of 64" in _lib.last_error(), _lib.last_error()


@pytest.mark.parametrize("entry", WITH_HW)
def test_entries_reject_empty_image(entry):
    from deeplearning_b200 import _lib

    assert _call(entry, HW=0) == -1
    assert "HW must be >= 1" in _lib.last_error(), _lib.last_error()


@pytest.mark.parametrize("entry", WITH_CR)
@pytest.mark.parametrize("Cr", [0, 257])
def test_entries_reject_hidden_width(entry, Cr):
    from deeplearning_b200 import _lib

    assert _call(entry, Cr=Cr) == -1
    assert "Cr must be in [1, 256]" in _lib.last_error(), _lib.last_error()


@pytest.mark.parametrize("entry", ENTRIES)
def test_entries_reject_empty_batch(entry):
    from deeplearning_b200 import _lib

    assert _call(entry, B=0) == -1
    assert "B must be in" in _lib.last_error(), _lib.last_error()


def test_entries_reject_misaligned_pointers():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    assert lib.b200_se_apply(FAKE + 4, FAKE, FAKE, FAKE, FAKE, FAKE, 2, 49, 256, None) == -1
    assert "16-byte aligned" in _lib.last_error()
    assert lib.b200_se_bwd_coeffs(*([FAKE] * 11), None, 2, 49, 256, 16, *([FAKE] * 8), None) == -1
    assert "every pointer" in _lib.last_error()
