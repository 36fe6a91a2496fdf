"""The fp32 ResNeXt yardstick of tests/test_gpu_resnext.py (torchvision's ResNet with groups=32, width_per_group=4) replayed
against the fixture tests/golden/make_resnext_golden.py wrote from the reference's own resnext50_32x4d(): constructor init
== reference init, yardstick forward / backward / running statistics == reference, fixture unchanged."""
import os

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
FX = torch.load(os.path.join(HERE, "golden", "resnext_golden.pt"), weights_only=False)["resnext50_32x4d"]


def _close(a, b, tol=2e-4):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


def _state():
    from deeplearning_b200.classification.resnet.models.networks import resnext50_32x4d

    torch.manual_seed(FX["seeds"]["init"])
    return {k: v.clone() for k, v in resnext50_32x4d().state_dict().items()}


def _yardstick(state):
    import torchvision

    m = torchvision.models.ResNet(torchvision.models.resnet.Bottleneck, [3, 4, 6, 3], groups=32, width_per_group=4)
    m.load_state_dict(state)
    return m


def test_resnext50_init_matches_reference():
    sd = _state()
    assert set(sd) >= set(FX["init_abs_sum"])
    for k, v in FX["init_abs_sum"].items():
        assert abs(float(sd[k].double().abs().sum()) - v) <= 1e-9 * (1 + abs(v)), k
    assert sd["layer1.0.conv2.weight"].shape == (128, 4, 3, 3)


def test_resnext50_yardstick_matches_reference_outputs():
    m = _yardstick(_state())
    x_eval = torch.randn(*FX["shapes"]["x_eval"], generator=torch.Generator().manual_seed(FX["seeds"]["x_eval"]))
    with torch.no_grad():
        _close(m.eval()(x_eval), FX["eval_logits"])
    x = torch.randn(*FX["shapes"]["x_train"], generator=torch.Generator().manual_seed(FX["seeds"]["x_train"]))
    y = torch.randint(0, 1000, (FX["shapes"]["x_train"][0],), generator=torch.Generator().manual_seed(FX["seeds"]["labels"]))
    out = m.train()(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    _close(out.detach(), FX["train_logits"])
    assert abs(float(loss.detach()) - FX["train_loss"]) <= 1e-4 * (1 + abs(FX["train_loss"]))
    for n, p in m.named_parameters():
        ref = FX["grad_norms"][n]
        assert abs(float(p.grad.double().norm()) - ref) <= 1e-3 * ref + 1e-8, n
    sd = m.state_dict()
    _close(sd["layer1.0.bn2.running_mean"], FX["running_mean_layer1_bn2"])
    _close(sd["layer4.2.bn2.running_var"], FX["running_var_layer4_bn2"])
