"""Device-free checks of RepVGG: every drop-in constructor's modules and parameters, the re-parameterisation helpers against
the oracle's fold, the engine's admission (it rejects what it does not run with a layer-named NotImplementedError before
touching a device), the stem's combined operand layout, and the argument checks of the RepVGG C entries (they reject a
shape with B200_EINVAL and a message before touching the device, so fake pointers are never dereferenced)."""
import pytest
import torch
import torch.nn as nn

# name -> (widths of stem, stage1..4; blocks per stage; grouped; SE)
VARIANTS = {"RepVGG-A0": ((48, 48, 96, 192, 1280), (2, 4, 14, 1)), "RepVGG-A1": ((64, 64, 128, 256, 1280), (2, 4, 14, 1)),
            "RepVGG-A2": ((64, 96, 192, 384, 1408), (2, 4, 14, 1)), "RepVGG-B0": ((64, 64, 128, 256, 1280), (4, 6, 16, 1)),
            "RepVGG-B1": ((64, 128, 256, 512, 2048), (4, 6, 16, 1)), "RepVGG-B2": ((64, 160, 320, 640, 2560), (4, 6, 16, 1)),
            "RepVGG-B3": ((64, 192, 384, 768, 2560), (4, 6, 16, 1))}


def _models():
    from deeplearning_b200.classification.RepVGG import models

    return models


def _randomise_bn(m, seed=0):
    g = torch.Generator().manual_seed(seed)
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            with torch.no_grad():
                mod.weight.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
                mod.bias.copy_(torch.rand(mod.num_features, generator=g) - 0.5)
                mod.running_mean.copy_(torch.rand(mod.num_features, generator=g) - 0.5)
                mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)


def test_package_exports():
    models = _models()
    assert len(models.func_dict) == 14
    assert models.get_RepVGG_func_by_name("RepVGG-B1g4") is models.func_dict["RepVGG-B1g4"]
    assert callable(models.repvgg_model_convert)


@pytest.mark.parametrize("name", sorted(_models().func_dict))
def test_constructor_structure(name):
    from deeplearning_b200.engine import repvgg as engine

    m = _models().func_dict[name](num_classes=7)
    blocks = engine._blocks(m)
    base = name[:-2] if name.endswith(("g2", "g4")) else name
    names = [n for n, _ in m.named_children()]
    assert names == ["stage0", "stage1", "stage2", "stage3", "stage4", "gap", "linear"]
    assert list(m.stage1[1]._modules) == ["nonlinearity", "se", "rbr_identity", "rbr_dense", "rbr_1x1"]
    assert m.stage1[0].rbr_identity is None and m.stage1[1].rbr_identity is not None
    assert m.linear.out_features == 7
    if base in VARIANTS:
        widths, nb = VARIANTS[base]
        assert [len(getattr(m, f"stage{i}")) for i in range(1, 5)] == list(nb)
        assert m.stage0.rbr_dense.conv.out_channels == widths[0]
        assert [getattr(m, f"stage{i}")[0].rbr_dense.conv.out_channels for i in range(1, 5)] == list(widths[1:])
        assert m.linear.in_features == widths[4]
    if name.endswith(("g2", "g4")):
        assert blocks[2][1].groups == int(name[-1]) and blocks[1][1].groups == 1
    if name == "RepVGG-D2se":
        assert isinstance(m.stage1[0].se.down, nn.Conv2d) and m.stage1[0].se.up.bias is not None


def test_deploy_constructor_keys():
    m = _models().func_dict["RepVGG-A0"](deploy=True, num_classes=5)
    keys = list(m.state_dict())
    assert keys[:2] == ["stage0.rbr_reparam.weight", "stage0.rbr_reparam.bias"]
    assert not any("rbr_dense" in k or "rbr_identity" in k for k in keys)


@pytest.mark.parametrize("name", ["RepVGG-A0", "RepVGG-B0"])
def test_switch_to_deploy_matches_oracle_fold(name):
    from oracle.repvgg import build, fold

    torch.manual_seed(0)
    m = _models().func_dict[name](num_classes=5)
    _randomise_bn(m)
    orc = build(name, m.state_dict(), 5)
    want = {}
    for (n, blk), (_, ob) in zip(m.named_modules(), orc.named_modules()):
        if hasattr(blk, "switch_to_deploy"):
            with torch.no_grad():
                want[n] = fold(ob)
    conv = _models().repvgg_model_convert(m)
    assert hasattr(m.stage1[1], "rbr_dense")      # do_copy=True left the original alone
    for n, blk in conv.named_modules():
        if n in want:
            k, b = want[n]
            assert torch.equal(blk.rbr_reparam.weight, k) and torch.equal(blk.rbr_reparam.bias, b), n
            assert not hasattr(blk, "rbr_dense") and not hasattr(blk, "rbr_identity") and blk.deploy
            assert not blk.rbr_reparam.weight.requires_grad
    d = _models().func_dict[name](deploy=True, num_classes=5)
    d.load_state_dict(conv.state_dict(), strict=True)


def test_custom_l2_matches_definition():
    torch.manual_seed(1)
    m = _models().func_dict["RepVGG-A0"](num_classes=5)
    _randomise_bn(m, 3)
    blk = m.stage2[1]
    k3, k1 = blk.rbr_dense.conv.weight, blk.rbr_1x1.conv.weight
    bd, b1 = blk.rbr_dense.bn, blk.rbr_1x1.bn
    t3 = (bd.weight / (bd.running_var + bd.eps).sqrt()).view(-1, 1, 1, 1)
    t1 = (b1.weight / (b1.running_var + b1.eps).sqrt()).view(-1, 1, 1, 1)
    eq = k3[:, :, 1:2, 1:2] * t3 + k1 * t1
    want = (eq ** 2 / (t3 ** 2 + t1 ** 2)).sum() + (k3 ** 2).sum() - (k3[:, :, 1:2, 1:2] ** 2).sum()
    got = blk.get_custom_L2()
    assert torch.allclose(got, want, rtol=1e-6)
    got.backward()
    assert k3.grad is not None and k1.grad is not None and bd.weight.grad is None


# ------------------------------------------------------------------------------------------------------------ admission
@pytest.mark.parametrize("name", ["RepVGG-A0", "RepVGG-A1", "RepVGG-A2", "RepVGG-B0", "RepVGG-B1", "RepVGG-B2", "RepVGG-B3"])
def test_dense_variants_admitted(name):
    from deeplearning_b200.engine import repvgg as engine

    strides = engine.check_model(_models().func_dict[name](num_classes=10))
    assert strides[:2] == [2, 2] and strides.count(2) == 5
    engine.check_model(_models().repvgg_model_convert(_models().func_dict[name](num_classes=10)))


@pytest.mark.parametrize("name, where, what", [("RepVGG-B1g2", "stage1.1", "grouped"), ("RepVGG-B2g4", "stage1.1", "grouped"),
                                               ("RepVGG-D2se", "stage0", "squeeze-and-excitation")])
def test_unsupported_variants_rejected(name, where, what):
    from deeplearning_b200.engine import repvgg as engine

    with pytest.raises(NotImplementedError, match=f"^{where}: .*{what}"):
        engine.check_model(_models().func_dict[name](num_classes=10))


def _a0():
    torch.manual_seed(0)
    return _models().func_dict["RepVGG-A0"](num_classes=10)


def test_rejects_odd_channel_count():
    from deeplearning_b200.classification.RepVGG.models.repvgg import RepVGG
    from deeplearning_b200.engine import repvgg as engine

    m = RepVGG([1, 1, 1, 1], 10, [0.75, 0.75, 0.75, 0.766], None)   # stage4: int(512 * 0.766) = 392 ... then 100 below
    engine.check_model(m)
    m = RepVGG([1, 1, 1, 1], 10, [0.75, 0.75, 0.75, 0.195], None)   # stage4: 99 channels
    with pytest.raises(NotImplementedError, match="^stage4.0: channel counts must be multiples of 8"):
        engine.check_model(m)


@pytest.mark.parametrize("mutate, where", [
    (lambda m: setattr(m.stage2[1], "nonlinearity", nn.GELU()), "stage2.1"),
    (lambda m: setattr(m.stage1[0].rbr_dense, "bn", nn.GroupNorm(4, 48)), "stage1.0"),
    (lambda m: setattr(m.stage3[2].rbr_1x1.conv, "padding", (1, 1)), "stage3.2"),
    (lambda m: setattr(m.stage1[1], "rbr_identity", nn.BatchNorm2d(48, affine=False)), "stage1.1"),
    (lambda m: setattr(m.stage2[0].rbr_dense.conv, "dilation", (2, 2)), "stage2.0"),
])
def test_rejects_foreign_structure(mutate, where):
    from deeplearning_b200.engine import repvgg as engine

    m = _a0()
    mutate(m)
    with pytest.raises(NotImplementedError, match=f"^{where}: "):
        engine.check_model(m)


def test_rejects_foreign_head():
    from deeplearning_b200.engine import repvgg as engine

    m = _a0()
    m.gap = nn.AdaptiveMaxPool2d(1)
    with pytest.raises(NotImplementedError, match="^gap: "):
        engine.check_model(m)


def test_rejects_sync_batchnorm_in_multi_rank_job(monkeypatch):
    import torch.distributed as dist

    from deeplearning_b200.engine import repvgg as engine

    m = nn.SyncBatchNorm.convert_sync_batchnorm(_a0()).train()
    engine.check_model(m.eval())             # eval mode: running statistics only, nothing to all-reduce
    engine.check_model(m.train())            # no process group: a single-rank job
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "group", type("G", (), {"WORLD": object()}))
    with pytest.raises(NotImplementedError, match="^stage0: SyncBatchNorm in a multi-rank job"):
        engine.check_model(m)


def test_trainer_dispatches_repvgg():
    from deeplearning_b200.engine import repvgg, trainer

    assert trainer._engine_for(_a0()) is repvgg


def test_cpu_input_raises():
    with pytest.raises(RuntimeError, match="CUDA"):
        _a0()(torch.zeros(1, 3, 32, 32))


def test_pack_spec_and_key_follow_the_block_form():
    from deeplearning_b200.engine import repvgg as engine

    m = _a0()
    specs = engine._pack_spec(m)
    stem = [s for s in specs if len(s) > 6]
    assert [s[6] for s in stem] == [("stem", 0, 0, 96), ("stem", 48, 12, 96)]
    assert stem[0][0] is m.stage0.rbr_dense.conv.weight and stem[1][0] is m.stage0.rbr_1x1.conv.weight
    k0 = engine._pack_spec.key(m)
    m.stage2[3].switch_to_deploy()
    assert engine._pack_spec.key(m) != k0
    assert any(s[0] is m.stage2[3].rbr_reparam.weight for s in engine._pack_spec(m))


# ------------------------------------------------------------------------------------------------------------ C entries
FAKE = 1 << 20   # 16-byte aligned, never dereferenced: every call below fails its argument checks first


def _call(name, rows=128, C=48, ld=None, f=FAKE):
    from deeplearning_b200 import _lib

    lib = _lib.load()
    ld = C if ld is None else ld
    if name == "b200_repvgg_apply":
        return lib.b200_repvgg_apply(f, ld, f, ld, f, ld, f, f, f, f, rows, C, None, None)
    if name == "b200_repvgg_bwd_reduce":
        return lib.b200_repvgg_bwd_reduce(f, f, f, ld, f, ld, f, ld, rows, C, f, None)
    if name == "b200_repvgg_bwd_apply":
        return lib.b200_repvgg_bwd_apply(f, f, f, ld, f, ld, f, ld, *([f] * 9), rows, C, None)
    raise AssertionError(name)


PASSES = ["b200_repvgg_apply", "b200_repvgg_bwd_reduce", "b200_repvgg_bwd_apply"]


@pytest.mark.parametrize("entry", PASSES)
@pytest.mark.parametrize("C", [0, 4, 36, 8200])
def test_passes_reject_channel_count(entry, C):
    from deeplearning_b200 import _lib

    assert _call(entry, C=C) == -1
    assert "C must be a multiple of 8 in [8, 8192]" in _lib.last_error(), _lib.last_error()


@pytest.mark.parametrize("entry", PASSES)
def test_passes_reject_empty_and_bad_pitch(entry):
    from deeplearning_b200 import _lib

    assert _call(entry, rows=0) == -1
    assert "rows must be >= 1" in _lib.last_error()
    assert _call(entry, C=48, ld=40) == -1
    assert "row pitches" in _lib.last_error()
    assert _call(entry, C=48, ld=100) == -1
    assert "row pitches" in _lib.last_error()


def test_passes_reject_pointers():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    assert lib.b200_repvgg_apply(FAKE + 4, 48, FAKE, 48, None, 0, FAKE, FAKE, None, FAKE, 128, 48, None, None) == -1
    assert "16-byte aligned" in _lib.last_error()
    assert lib.b200_repvgg_apply(FAKE, 48, FAKE, 48, FAKE, 48, FAKE, FAKE, None, FAKE, 128, 48, None, None) == -1
    assert "identity branch" in _lib.last_error()
    assert lib.b200_repvgg_bwd_apply(FAKE, FAKE, FAKE, 48, FAKE, 48, FAKE, 48, *([FAKE] * 4), FAKE, None, FAKE, FAKE, FAKE,
                                     128, 48, None) == -1
    assert "identity branch" in _lib.last_error()
    assert lib.b200_repvgg_bwd_reduce(FAKE, FAKE, FAKE, 48, FAKE, 48, None, 0, 128, 48, None, None) == -1
    assert "partial non-null" in _lib.last_error()


def test_partial_rows_and_fold_checks():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    assert lib.b200_repvgg_partial_rows(0, 48) == -1 and lib.b200_repvgg_partial_rows(100, 12) == -1
    T = lib.b200_repvgg_partial_rows(256 * 112 * 112, 48)
    assert 1 <= T <= 132 * 8
    assert lib.b200_repvgg_partial_rows(1, 2560) == 1
    f = FAKE
    bn = [f, f, f, f, 1e-5]
    assert lib.b200_repvgg_fold(f, f, *bn, *bn, None, None, None, None, 0.0, 48, 3, 24, f, f, None) == -1
    assert "ldk" in _lib.last_error()
    assert lib.b200_repvgg_fold(f, f, *bn, *bn, *bn, 48, 3, 32, f, f, None) == -1
    assert "O == I" in _lib.last_error()
    assert lib.b200_repvgg_fold(f, f, *bn, *bn, f, None, f, f, 1e-5, 48, 48, 432, f, f, None) == -1
    assert "all of gamma" in _lib.last_error()
    assert lib.b200_repvgg_fold(f, None, *bn, *bn, None, None, None, None, 0.0, 48, 48, 432, f, f, None) == -1
    assert "required" in _lib.last_error()
