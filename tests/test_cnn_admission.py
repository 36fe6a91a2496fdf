"""Admission of every CNN constructor the drop-in model packages export: each one either trains on the GPU engine, or is
rejected with a NotImplementedError that names the layer before any kernel runs.

``EXPECT`` has one entry per constructor of ResNet / ResNeXt / Wide-ResNet, SE-ResNet, VGG, EfficientNet, RepVGG
(``func_dict``) and ShuffleNet v1 / v2 (both ``get_model`` tables); a constructor added to one of those without an entry
fails here.  The device-free tests build every model on the meta device and run its engine's ``check_model``; the GPU test
reads the outcome of the batch-2 train steps that tests/test_gpu_cnn_gemm_calls.py records (one run serves both files)."""
import importlib

import pytest
import torch

# the modules that export the constructors, and the engine module whose check_model admits each family (ResNet and
# SE-ResNet have none: their schedule checks each layer as it reaches it)
_RESNET = "deeplearning_b200.classification.resnet.models.networks"
_SENET = "deeplearning_b200.classification.seNet.models.se_resnet"
_VGG = "deeplearning_b200.classification.vggNet.models.network"
_EFFNET = "deeplearning_b200.classification.efficientNet.models.network"
_REPVGG = "deeplearning_b200.classification.RepVGG.models.repvgg"
_SHUFFLE1 = "deeplearning_b200.classification.ShuffleNet.models.shufflenetv1"
_SHUFFLE2 = "deeplearning_b200.classification.ShuffleNet.models.shufflenetv2"
ENGINES = {"resnet": None, "senet": None, "vgg": "vgg", "efficientnet": "efficientnet", "repvgg": "repvgg",
           "shufflenet_v1": "shufflenet", "shufflenet_v2": "shufflenetv2"}

# the resolution each EfficientNet variant is trained at (efficientNet/train.py img_size)
EFFNET_HW = {"efficientnet_b0": 224, "efficientnet_b1": 240, "efficientnet_b2": 260, "efficientnet_b3": 300,
             "efficientnet_b4": 380, "efficientnet_b5": 456, "efficientnet_b6": 528, "efficientnet_b7": 600}

# what the engine does with each: "train", "eval" (runs without gradients only) or "reject" (not even a forward)
EXPECT = {
    "resnet18": "train", "resnet34": "train", "resnet50": "train", "resnet101": "train", "resnet152": "train",
    "resnext50_32x4d": "train", "resnext101_32x8d": "train", "wide_resnet50_2": "train", "wide_resnet101_2": "train",
    "se_resnet": "train", "se_resnet34": "train", "se_resnet50": "train", "se_resnet101": "train", "se_resnet152": "train",
    "vgg11": "train", "vgg11_bn": "train", "vgg13": "train", "vgg13_bn": "train", "vgg16": "train", "vgg16_bn": "train",
    "vgg19": "train", "vgg19_bn": "train",
    **{name: "train" for name in EFFNET_HW},
    "RepVGG-A0": "train", "RepVGG-A1": "train", "RepVGG-A2": "train", "RepVGG-B0": "train", "RepVGG-B1": "train",
    "RepVGG-B2": "train", "RepVGG-B3": "train",
    "RepVGG-B1g2": "reject", "RepVGG-B1g4": "reject", "RepVGG-B2g2": "reject", "RepVGG-B2g4": "reject",
    "RepVGG-B3g2": "reject", "RepVGG-B3g4": "reject",   # grouped 3x3 / 1x1 branches
    "RepVGG-D2se": "reject",                             # squeeze-and-excitation blocks
    "shufflenet_v1_g1": "train", "shufflenet_v1_g2": "train", "shufflenet_v1_g3": "train", "shufflenet_v1_g4": "train",
    "shufflenet_v1_g8": "train",
    "shufflenet_v2_x0_5": "train", "shufflenet_v2_x1_0": "train", "shufflenet_v2_x1_5": "train",
    "shufflenet_v2_x2_0": "train",
}
# what a rejection message starts with: the layer it names
REJECT_LAYER = {"RepVGG-B1g2": r"stage1\.1: grouped", "RepVGG-B1g4": r"stage1\.1: grouped",
                "RepVGG-B2g2": r"stage1\.1: grouped", "RepVGG-B2g4": r"stage1\.1: grouped",
                "RepVGG-B3g2": r"stage1\.1: grouped", "RepVGG-B3g4": r"stage1\.1: grouped",
                "RepVGG-D2se": r"stage0: squeeze-and-excitation"}


def _exported(modname):
    """Constructor functions a model module exports: the lower-case callables of its __all__."""
    mod = importlib.import_module(modname)
    return [n for n in mod.__all__ if not n.startswith("_") and n[0].islower() and callable(getattr(mod, n))
            and not isinstance(getattr(mod, n), type)]


def constructors():
    """{name: (family, zero-argument constructor, native resolution)} of every exported CNN constructor."""
    out = {}
    for fam, modname in (("resnet", _RESNET), ("senet", _SENET), ("vgg", _VGG), ("efficientnet", _EFFNET)):
        mod = importlib.import_module(modname)
        for n in _exported(modname):
            out[n] = (fam, getattr(mod, n), EFFNET_HW.get(n, 224))
    rep = importlib.import_module(_REPVGG)
    for n, fn in rep.func_dict.items():
        out[n] = ("repvgg", fn, 224)
    for fam, modname in (("shufflenet_v1", _SHUFFLE1), ("shufflenet_v2", _SHUFFLE2)):
        mod = importlib.import_module(modname)
        for n in mod.model_dict:
            out[n] = (fam, mod.get_model(n), 224)
    return out


CTORS = constructors()


def engine_of(family):
    name = ENGINES[family]
    return None if name is None else importlib.import_module(f"deeplearning_b200.engine.{name}")


def test_every_exported_constructor_has_an_entry():
    from deeplearning_b200.classification.ShuffleNet.models import get_model

    assert set(CTORS) == set(EXPECT), (sorted(set(CTORS) - set(EXPECT)), sorted(set(EXPECT) - set(CTORS)))
    assert set(REJECT_LAYER) == {n for n, w in EXPECT.items() if w == "reject"}
    # the package-level get_model is the ShuffleNet v1 table
    assert all(get_model(n) is CTORS[n][1] for n in CTORS if CTORS[n][0] == "shufflenet_v1")
    # every model of a family is dispatched to that family's engine schedule
    from deeplearning_b200.engine.trainer import _engine_for

    for n, (fam, fn, _) in CTORS.items():
        with torch.device("meta"):
            m = fn()
        assert _engine_for(m).__name__.split(".")[-1] == (ENGINES[fam] or "resnet"), n


@pytest.mark.parametrize("name", sorted(n for n, (fam, _, _) in CTORS.items() if ENGINES[fam] is not None))
def test_check_model_admits_or_names_the_layer(name):
    fam, fn, _ = CTORS[name]
    with torch.device("meta"):
        m = fn()
    check = engine_of(fam).check_model
    if EXPECT[name] == "reject":
        with pytest.raises(NotImplementedError, match="^" + REJECT_LAYER[name]) as e:
            check(m)
        print(f"{name}: {e.value}")
    else:
        check(m)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EXPECT))
def test_shipped_constructor_trains_or_is_rejected_before_launch(name):
    """The batch-2 train step at the native resolution (recorded with the GEMM calls): a "train" constructor finished it
    with finite logits and gradients; a "reject" one raised NotImplementedError before any kernel launched, in training
    and in eval mode."""
    import test_gpu_cnn_gemm_calls as calls

    outcome = calls.recording().outcome
    keys = [k for k in outcome if k[0] == name]
    assert keys, f"{name} was not stepped"
    for key in keys:
        got = outcome[key]
        print(key, got)
        assert got[0] == EXPECT[name], (key, got)
