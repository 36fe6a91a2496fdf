"""Device-free checks of the EfficientNet drop-in and its engine: the b0-b7 constructors' channel plans, module names and
block plan (against oracle/efficientnet.py's restatement of the reference's configuration), admission of every structure
the engine does not run, and the C entries of csrc/mbconv.cuh (each rejects a bad shape or pointer with B200_EINVAL and a
message before touching the device, so fake pointers are never dereferenced)."""
import pytest
import torch
import torch.nn as nn

NAMES = [f"b{i}" for i in range(8)]
# (stem width, widest expanded width, top width, blocks) of efficientnet_b0 .. b7
PLANS = {"b0": (32, 1152, 1280, 16), "b1": (32, 1920, 1280, 23), "b2": (32, 2112, 1408, 23), "b3": (40, 2304, 1536, 26),
         "b4": (48, 2688, 1792, 32), "b5": (48, 3072, 2048, 39), "b6": (56, 3456, 2304, 45), "b7": (64, 3840, 2560, 55)}


def _net(name="b0", **kw):
    from deeplearning_b200.classification.efficientNet.models import network

    torch.manual_seed(0)
    return getattr(network, f"efficientnet_{name}")(**kw)


@pytest.mark.parametrize("name", NAMES)
def test_constructor_plan(name):
    from deeplearning_b200.engine import efficientnet as engine
    from oracle.efficientnet import COEFFS, plan

    m = _net(name, num_classes=7)
    stem_conv, _, blocks, top_conv, _, p, head = engine.check_model(m)
    c0, widest, top, n = PLANS[name]
    assert stem_conv.out_channels == c0 and top_conv.out_channels == top and len(blocks) == n
    assert max(b.dw.out_channels for b in blocks) == widest
    assert p == COEFFS[name][2] and head.out_features == 7
    want = plan(name)
    assert [b.name for b in blocks] == [f"features.{idx}" for idx, *_ in want]
    for b, (idx, k, s, rate) in zip(blocks, want):
        assert (b.k, b.s) == (k, s), idx
        assert b.drop == (rate if b.res else 0.0), idx
        assert b.fc1.out_channels == max(8, int(b.fc1.out_channels))
    assert blocks[0].exp is None and blocks[0].drop == 0.0
    names = [n_ for n_, _ in m.named_parameters()]
    assert names[0] == "features.stem_conv.0.weight" and names[-1] == "classifier.1.bias"
    assert "features.2a.block.se.fc.0.bias" in names and "features.1a.block.expand_conv.0.weight" not in names


def test_se_width_comes_from_block_input():
    m = _net("b0")
    se = m.features._modules["2a"].block.se
    assert se.fc[0].in_channels == 96 and se.fc[0].out_channels == 8     # _make_divisible(16 // 4, 8), not 96 // 4
    assert m.features._modules["1a"].block.dwconv[1].eps == 1e-3
    assert isinstance(m.classifier[0], nn.Dropout) and m.classifier[0].inplace


def test_trainer_dispatches_efficientnet():
    from deeplearning_b200.engine import efficientnet, trainer

    assert trainer._engine_for(_net()) is efficientnet


def test_cpu_input_raises():
    with pytest.raises(RuntimeError, match="CUDA"):
        _net()(torch.zeros(1, 3, 32, 32))


def _set(m, path, mod):
    *parent, last = path.split(".")
    obj = m
    for p in parent:
        obj = obj._modules[p]
    obj._modules[last] = mod


@pytest.mark.parametrize("path,mod,where", [
    ("features.2a.block.dwconv.0", nn.Conv2d(96, 96, 7, 2, 3, groups=96, bias=False), "features.2a: the GPU engine runs "
     "depthwise convolutions of kernel size 3 or 5"),
    ("features.2a.block.dwconv.0", nn.Conv2d(96, 96, 3, 3, 1, groups=96, bias=False), "features.2a"),
    ("features.2a.block.dwconv.2", nn.ReLU(), "features.2a.dwconv"),
    ("features.top.2", nn.ReLU(), "features.top"),
    ("features.2a.block.se", nn.Identity(), "features.2a"),
    ("features.2a.block.se.fc.1", nn.ReLU(), "features.2a"),
    ("features.2a.block.project_conv.2", nn.SiLU(), "features.2a.project_conv"),
    ("features.3a.block.expand_conv.1", nn.GroupNorm(1, 144), "features.3a.expand_conv"),
    ("avgpool", nn.AdaptiveMaxPool2d(1), "avgpool"),
    ("classifier.1", nn.Identity(), "classifier"),
])
def test_rejects_foreign_structure(path, mod, where):
    from deeplearning_b200.engine import efficientnet as engine

    m = _net("b0")
    _set(m, path, mod)
    with pytest.raises(NotImplementedError, match=f"^{where}"):
        engine.check_model(m)


def test_rejects_channel_counts_not_multiple_of_8():
    from deeplearning_b200.classification.efficientNet.models.network import EfficientNet
    from deeplearning_b200.engine import efficientnet as engine

    m = EfficientNet(1.0, 1.0)
    blk = m.features._modules["2a"].block
    blk.expand_conv[0] = nn.Conv2d(16, 100, 1, bias=False)
    blk.expand_conv[1] = nn.BatchNorm2d(100)
    blk.dwconv[0] = nn.Conv2d(100, 100, 3, 2, 1, groups=100, bias=False)
    blk.dwconv[1] = nn.BatchNorm2d(100)
    blk.se.fc[0] = nn.Conv2d(100, 8, 1)
    blk.se.fc[2] = nn.Conv2d(8, 100, 1)
    blk.project_conv[0] = nn.Conv2d(100, 24, 1, bias=False)
    with pytest.raises(NotImplementedError, match="^features.2a: channel counts must be multiples of 8"):
        engine.check_model(m)


def test_rejects_shortcut_around_first_block():
    """Width coefficients below ~0.37 give block 1a equal input and output widths, so the reference adds a shortcut around
    it; the engine does not materialise that shortcut's input (silu(bn(stem))) and rejects the model"""
    from deeplearning_b200.classification.efficientNet.models.network import EfficientNet
    from deeplearning_b200.engine import efficientnet as engine

    m = EfficientNet(0.25, 1.0)
    assert m.features._modules["1a"].use_res_connect
    with pytest.raises(NotImplementedError, match="^features.1a: a shortcut around the first block"):
        engine.check_model(m)


def test_rejects_sync_batchnorm_in_multi_rank_job(monkeypatch):
    import torch.distributed as dist

    from deeplearning_b200.engine import efficientnet as engine

    m = nn.SyncBatchNorm.convert_sync_batchnorm(_net("b0")).train()
    engine.check_model(m)                    # no process group: a single-rank job
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "group", type("G", (), {"WORLD": object()}))
    with pytest.raises(NotImplementedError, match="^features.stem_conv: SyncBatchNorm in a multi-rank job"):
        engine.check_model(m)


def test_no_dropout_classifier_admitted():
    from deeplearning_b200.classification.efficientNet.models.network import EfficientNet
    from deeplearning_b200.engine import efficientnet as engine

    m = EfficientNet(1.0, 1.0, dropout_rate=0.0, drop_connect_rate=0.0)
    assert engine.check_model(m)[5] == 0.0
    assert all(b.drop == 0.0 for b in engine.check_model(m)[2])


# ------------------------------------------------------------------------------------------------------------ C entries
F_ = 1 << 20    # 16-byte aligned, never dereferenced: every call below fails its argument checks first


def _lib():
    from deeplearning_b200 import _lib as L

    return L


def _rejects(call, msg):
    L = _lib()
    assert call(L.load()) == -1
    assert msg in L.last_error(), L.last_error()


@pytest.mark.parametrize("C", [0, 4, 36, 8200])
def test_efficientnet_entries_reject_channel_count(C):
    m = "a multiple of 8 in [8, 8192]"
    _rejects(lambda L: L.b200_dw_fwd(F_, F_, None, None, F_, None, 2, 8, 8, C, 3, 1, None), m)
    _rejects(lambda L: L.b200_dw_dgrad(F_, F_, F_, None, None, None, F_, None, 2, 8, 8, C, 3, 1, None), m)
    _rejects(lambda L: L.b200_dw_wgrad(F_, F_, None, None, F_, F_, 1 << 30, 2, 8, 8, C, 3, 1, None), m)
    _rejects(lambda L: L.b200_silu_bn_squeeze(F_, F_, F_, None, F_, None, 2, 16, C, None), m)
    _rejects(lambda L: L.b200_excite_fwd(F_, F_, F_, F_, F_, F_, F_, 2, C, 8, None), m)
    _rejects(lambda L: L.b200_excite_bwd(*([F_] * 13), 2, C, 8, None), m)
    _rejects(lambda L: L.b200_gate_apply(F_, F_, F_, F_, F_, 2, 16, C, None), m)
    _rejects(lambda L: L.b200_gate_reduce(F_, F_, F_, F_, F_, 2, 16, C, None), m)
    _rejects(lambda L: L.b200_silu_bn_bwd_reduce(F_, F_, F_, F_, F_, F_, F_, F_, 2, 16, C, None), m)
    _rejects(lambda L: L.b200_tail_apply(F_, F_, F_, None, None, F_, 2, 16, C, None), m)
    _rejects(lambda L: L.b200_tail_bwd_reduce(F_, None, F_, None, F_, 2, 16, C, None), m)
    _rejects(lambda L: L.b200_bn_bwd_apply(F_, F_, None, 1, *([F_] * 7), 1, 32, C, None), m)
    L = _lib().load()
    assert L.b200_dw_partial_rows(32, C) == -1
    assert L.b200_dw_wgrad_workspace_bytes(2, 8, 8, C, 3, 1) == 0


def test_efficientnet_entries_reject_shapes_and_pointers():
    _rejects(lambda L: L.b200_dw_fwd(F_, F_, None, None, F_, None, 2, 8, 8, 64, 7, 1, None), "k must be 3 or 5")
    _rejects(lambda L: L.b200_dw_fwd(F_, F_, None, None, F_, None, 2, 8, 8, 64, 3, 3, None), "stride must be 1 or 2")
    _rejects(lambda L: L.b200_dw_fwd(F_, F_, None, None, F_, None, 2, 0, 8, 64, 3, 1, None), "H and W must be >= 1")
    _rejects(lambda L: L.b200_dw_fwd(F_, F_, None, None, F_, None, 0, 8, 8, 64, 3, 1, None), "B must be in")
    _rejects(lambda L: L.b200_dw_fwd(F_ + 2, F_, None, None, F_, None, 2, 8, 8, 64, 3, 1, None), "16-byte aligned")
    _rejects(lambda L: L.b200_dw_fwd(F_, F_, F_, None, F_, None, 2, 8, 8, 64, 3, 1, None), "both scale and shift")
    _rejects(lambda L: L.b200_dw_dgrad(F_, F_, F_, F_, F_, None, F_, None, 2, 8, 8, 64, 3, 1, None), "and partial")
    _rejects(lambda L: L.b200_dw_dgrad(F_, F_, F_, F_, F_, F_, F_, F_, 2, 8, 8, 64, 3, 1, None), "cannot be combined")
    _rejects(lambda L: L.b200_dw_wgrad(F_, F_, None, None, F_, F_, 16, 2, 8, 8, 64, 3, 1, None), "workspace of 16 bytes")
    _rejects(lambda L: L.b200_silu_bn_squeeze(F_, F_, F_, F_, F_, None, 2, 16, 64, None), "both mask and out16")
    _rejects(lambda L: L.b200_silu_bn_squeeze(F_, F_, F_, None, F_, None, 2, 0, 64, None), "HW must be >= 1")
    _rejects(lambda L: L.b200_excite_fwd(F_, F_, F_, F_, F_, F_, F_, 2, 64, 257, None), "Cr must be in [1, 256]")
    _rejects(lambda L: L.b200_excite_fwd(F_, F_, None, F_, F_, F_, F_, 2, 64, 8, None), "are required")
    _rejects(lambda L: L.b200_excite_bwd(*([F_] * 12), None, 2, 64, 8, None), "every pointer is required")
    _rejects(lambda L: L.b200_gate_apply(F_, F_, F_, None, F_, 2, 16, 64, None), "16-byte aligned")
    _rejects(lambda L: L.b200_gate_reduce(F_, F_, F_, F_, None, 2, 16, 64, None), "s non-null")
    _rejects(lambda L: L.b200_silu_bn_bwd_reduce(F_, None, F_, F_, F_, F_, F_, F_, 2, 16, 64, None), "come together")
    _rejects(lambda L: L.b200_tail_apply(F_, F_, F_, None, F_ + 8, F_, 2, 16, 64, None), "16-byte aligned")
    _rejects(lambda L: L.b200_tail_bwd_reduce(F_, F_, F_, None, F_, 2, 16, 64, None), "exactly when rs is given")
    _rejects(lambda L: L.b200_bn_bwd_apply(F_, F_, None, 1, *([F_] * 7), 1, 0, 64, None), "rows >= 1")
    _rejects(lambda L: L.b200_bn_bwd_apply(F_, F_ + 8, None, 1, *([F_] * 7), 1, 32, 64, None), "16-byte aligned")
    _rejects(lambda L: L.b200_bn_bwd_apply(F_, F_, F_ + 8, 0, *([F_] * 7), 1, 32, 64, None), "16-byte aligned")
    _rejects(lambda L: L.b200_bn_bwd_apply(F_, F_, None, 1, F_, F_, F_, F_, F_, None, F_, 1, 32, 64, None), "non-null")
    L = _lib().load()
    assert L.b200_dw_partial_rows(1000, 64) > 0
    assert L.b200_dw_wgrad_workspace_bytes(2, 8, 8, 64, 5, 2) % (25 * 64 * 4) == 0
