"""Host-side checks of the SupCon drop-in and its GPU engine schedule (no GPU needed): constructor keys and shapes, the
meta-device admission of every BACKBONES entry, dispatch, CPU input, TrainStep's criterion validation, the frozen-encoder
arena of the second stage and the C-entry argument checks."""
import pytest
import torch
import torch.nn as nn

from deeplearning_b200.engine import resnet
from deeplearning_b200.engine import supcon as engine
from deeplearning_b200.self_supervised.SupCon.losses.LabelSmooth import LabelSmoothingLoss
from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss
from deeplearning_b200.self_supervised.SupCon.models.backbone import BACKBONES, RESNETS
from deeplearning_b200.self_supervised.SupCon.models.model import SupConModel, build_model, create_encoder

REJECTED = {"alexnet", "mobilenet_v2", "vgg11", "vgg11_bn", "vgg13", "vgg13_bn", "vgg16", "vgg16_bn", "vgg19", "vgg19_bn",
            "densenet121", "densenet169", "densenet161", "densenet201", "inception_v3"}


def test_constructor_keys_and_shapes():
    m = SupConModel("resnet18")
    sd = m.state_dict()
    names = list(sd)
    assert names[:2] == ["encoder.0.weight", "encoder.1.weight"] and "encoder.4.0.conv1.weight" in names
    assert names[-4:] == ["head.0.weight", "head.0.bias", "head.2.weight", "head.2.bias"]
    assert tuple(sd["head.0.weight"].shape) == (512, 512) and tuple(sd["head.2.weight"].shape) == (128, 512)
    assert not any(n.startswith(("encoder.2", "encoder.3", "encoder.8", "classifier")) for n in names)
    assert m.embed_dim == 128 and m.features_dim == 512
    m.use_projection_head(False)
    assert m.embed_dim == 512 and not m.projection_head
    m.use_projection_head(True)
    assert m.embed_dim == 128

    m = SupConModel("resnet50", second_stage=True, num_classes=10)
    sd = m.state_dict()
    assert list(sd)[-2:] == ["classifier.weight", "classifier.bias"] and tuple(sd["classifier.weight"].shape) == (10, 2048)
    assert not any(n.startswith("head") for n in sd)
    assert all(not p.requires_grad for p in m.encoder.parameters()) and m.classifier.weight.requires_grad


def test_create_encoder_and_build_model(tmp_path):
    enc, f = create_encoder("resnext50_32x4d")
    assert f == 2048 and len(enc) == 9 and isinstance(enc[8], nn.AdaptiveAvgPool2d)
    with pytest.raises(NotImplementedError, match="timm_resnet18"):
        create_encoder("timm_resnet18")
    with pytest.raises(RuntimeError, match="correct backbone name"):
        create_encoder("resnet19")
    src = SupConModel("resnet18")
    torch.save({"model_state_dict": src.state_dict()}, tmp_path / "ckpt.pt")
    m = build_model("resnet18", second_stage=True, num_classes=10, ckpt_pretrained=str(tmp_path / "ckpt.pt"))
    assert torch.equal(m.encoder[0].weight, src.encoder[0].weight)


@pytest.mark.parametrize("name", sorted(BACKBONES))
def test_meta_admission_of_every_backbone(name):
    assert set(BACKBONES) == set(RESNETS) | REJECTED
    with torch.device("meta"):
        if name in REJECTED:
            with pytest.raises(NotImplementedError, match=name):
                SupConModel(name)
            return
        for stage2 in (False, True):
            m = SupConModel(name, second_stage=stage2, num_classes=10)
            trunk = resnet.Trunk(m.encoder, "encoder")
            assert trunk.conv1 is m.encoder[0] and trunk.layers[3] is m.encoder[7]
            engine._check(m, want_tape=True)
            specs = resnet.conv_pack_specs(m.encoder, m.encoder[0])
            assert specs[0][0] is m.encoder[0].weight and specs[0][1] == 2   # space-to-depth stem operand


def test_admission_rejections():
    m = SupConModel("resnet18")
    for p in list(m.encoder.parameters())[:3]:
        p.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="partially frozen"):
        engine._check(m, want_tape=True)
    m = SupConModel("resnet18", second_stage=True, num_classes=10)
    for p in m.encoder.parameters():
        p.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="frozen encoder"):
        engine._check(m, want_tape=True)
    m = SupConModel("resnet18", projection_dim=100)
    with pytest.raises(NotImplementedError, match="head.2"):
        engine._check(m, want_tape=True)
    m = SupConModel("resnet18")
    m.encoder = nn.Sequential(*list(m.encoder)[:8])
    with pytest.raises(NotImplementedError, match="encoder"):
        resnet.Trunk(m.encoder, "encoder")


def test_dispatch_and_cpu_input():
    from deeplearning_b200.engine.trainer import _engine_for

    m = SupConModel("resnet18")
    assert _engine_for(m) is engine
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(2, 3, 32, 32))
    with pytest.raises(RuntimeError, match="CUDA"):
        SupConLoss()(torch.zeros(2, 2, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        LabelSmoothingLoss(10, 0.1)(torch.zeros(2, 10), torch.zeros(2, dtype=torch.long))


def test_supconloss_argument_checks():
    loss = SupConLoss()
    with pytest.raises(ValueError, match="at least 3 dimensions"):
        loss(torch.zeros(4, 8))
    with pytest.raises(ValueError, match="Cannot define both"):
        loss(torch.zeros(4, 2, 8), torch.zeros(4), torch.eye(4))
    with pytest.raises(NotImplementedError, match="mask"):
        loss(torch.zeros(4, 2, 8), mask=torch.eye(4))
    with pytest.raises(NotImplementedError, match="contrast_mode='one'"):
        SupConLoss(contrast_mode="one")(torch.zeros(4, 2, 8))
    with pytest.raises(ValueError, match="Unknown mode"):
        SupConLoss(contrast_mode="some")(torch.zeros(4, 2, 8))


def test_row_labels_and_smoothed_target():
    y = torch.tensor([3, 1, 3])
    assert engine.row_labels(y, 3, 2, "cpu").tolist() == [3, 1, 3, 3, 1, 3]
    assert engine.row_labels(None, 3, 3, "cpu").tolist() == [0, 1, 2] * 3
    with pytest.raises(ValueError, match="Num of labels"):
        engine.row_labels(y, 4, 2, "cpu")
    t = engine.smoothed_target(torch.tensor([0, 2]), 4, 0.3, 4)
    assert torch.allclose(t, torch.tensor([[0.7, 0.1, 0.1, 0.1], [0.1, 0.1, 0.7, 0.1]]))
    with pytest.raises(ValueError, match="classes=4"):
        engine.smoothed_target(torch.tensor([0]), 4, 0.1, 5)


def test_trainstep_criterion_validation():
    """TrainStep checks its criterion before it builds the arena or looks for a device."""
    from deeplearning_b200.classification.resnet.models.networks import resnet18
    from deeplearning_b200.engine.trainer import TrainStep

    s1 = SupConModel("resnet18")
    s2 = SupConModel("resnet18", second_stage=True, num_classes=10)
    for model, crit in ((s1, None), (s1, LabelSmoothingLoss(10, 0.1)), (s1, nn.CrossEntropyLoss()),
                        (s2, SupConLoss()), (s2, LabelSmoothingLoss(7, 0.1)), (resnet18(), SupConLoss()),
                        (resnet18(), LabelSmoothingLoss(1000, 0.1))):
        with pytest.raises(ValueError):
            TrainStep(model, criterion=crit)
    with pytest.raises(NotImplementedError, match="contrast_mode"):
        TrainStep(s1, criterion=SupConLoss(contrast_mode="one"))
    for model, crit in ((s1, SupConLoss(0.1)), (s2, LabelSmoothingLoss(10, 0.01)), (s2, None), (resnet18(), None)):
        with pytest.raises(RuntimeError, match="CUDA"):
            TrainStep(model, criterion=crit, momentum=0.0, weight_decay=0.0)


def test_second_stage_arena_holds_the_classifier_only():
    from deeplearning_b200.engine.trainer import TrainStep

    m = SupConModel("resnet18", second_stage=True, num_classes=10)
    step = TrainStep.__new__(TrainStep)
    with pytest.raises(RuntimeError, match="CUDA"):
        step.__init__(m, lr=0.01, momentum=0.0, weight_decay=0.0, criterion=LabelSmoothingLoss(10, 0.01))
    assert [id(p) for p in step.arena.params] == [id(m.classifier.weight), id(m.classifier.bias)]
    names = [n for n, _ in m.named_parameters()]
    assert [names[i] for i in step._pidx] == ["classifier.weight", "classifier.bias"]


def test_entries_reject_bad_arguments_before_launch():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    fake = 256   # never dereferenced: every check runs before a launch
    assert lib.b200_supcon_max_dim() == 2048
    assert lib.b200_supcon_normalize_fwd(fake, fake, fake, 4, 6, None) == -1 and "multiple of 4" in _lib.last_error()
    assert lib.b200_supcon_normalize_fwd(fake, fake, fake, 0, 8, None) == -1 and "N must be" in _lib.last_error()
    assert lib.b200_supcon_normalize_fwd(None, fake, fake, 4, 8, None) == -1 and "non-null" in _lib.last_error()
    assert lib.b200_supcon_normalize_bwd(fake, fake, fake, None, 4, 8, None) == -1 and "non-null" in _lib.last_error()
    assert lib.b200_supcon_loss_fwd(fake, fake, 4, 4096, 0.1, 0.07, fake, fake, fake, fake, None) == -1
    assert "[4, 2048]" in _lib.last_error()
    assert lib.b200_supcon_loss_fwd(fake, fake, 4, 128, 0.0, 0.07, fake, fake, fake, fake, None) == -1
    assert "temperature" in _lib.last_error()
    assert lib.b200_supcon_loss_fwd(fake, fake, 4, 128, 0.1, 0.07, fake, fake, None, fake, None) == -1
    assert "non-null" in _lib.last_error()
    assert lib.b200_supcon_loss_bwd(fake, fake, fake, fake, None, 1.0, 4, 128, 0.1, 0.07, fake, None) == -1
    assert "non-null" in _lib.last_error()
    assert lib.b200_supcon_loss_bwd(fake, fake, fake, fake, fake, float("inf"), 4, 128, 0.1, 0.07, fake, None) == -1
    assert "grad_scale" in _lib.last_error()
    assert lib.b200_supcon_loss_bwd(fake, fake, fake, fake, fake, 1.0, 4, 130, 0.1, 0.07, fake, None) == -1
    assert lib.b200_supcon_relu_bwd(fake, fake, fake, 0, None) == -1 and "n must be" in _lib.last_error()
    assert lib.b200_supcon_relu_bwd(fake, None, fake, 8, None) == -1 and "non-null" in _lib.last_error()


def test_wrappers_name_an_unsupported_width():
    from deeplearning_b200 import ops

    with pytest.raises(NotImplementedError, match="width 4096"):
        ops._supcon_rows(torch.zeros(4, 4096), "supcon_loss", 2048)
    with pytest.raises(NotImplementedError, match="width 130"):
        ops._supcon_rows(torch.zeros(4, 130), "supcon_loss", 2048)


def test_stage1_checkpoint_loads_into_stage2_like_the_reference():
    """The reference's second stage loads the first stage's state_dict with strict=False: the projection head is
    unexpected, the classifier missing."""
    s1 = SupConModel("resnet18")
    s2 = SupConModel("resnet18", second_stage=True, num_classes=10)
    res = s2.load_state_dict(s1.state_dict(), strict=False)
    assert res.missing_keys == ["classifier.weight", "classifier.bias"]
    assert res.unexpected_keys == ["head.0.weight", "head.0.bias", "head.2.weight", "head.2.bias"]
    assert torch.equal(s2.encoder[4][0].conv1.weight, s1.encoder[4][0].conv1.weight)
