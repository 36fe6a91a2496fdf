"""The drop-in SE-ResNet constructors and the fp32 SE-ResNet yardstick of tests/test_gpu_senet.py (oracle/senet.py) replayed
against the fixture tests/golden/make_senet_golden.py wrote from the reference's own se_resnet50() / se_resnet():
constructor init == reference init, yardstick forward / backward / running statistics == reference."""
import os

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
FX = torch.load(os.path.join(HERE, "golden", "senet_golden.pt"), weights_only=False)
NETS = {"se_resnet50": ((3, 4, 6, 3), True), "se_resnet": ((2, 2, 2, 2), False)}


def _close(a, b, tol=2e-4):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


def _state(name):
    from deeplearning_b200.classification.seNet.models import networks

    torch.manual_seed(FX[name]["seeds"]["init"])
    return {k: v.clone() for k, v in getattr(networks, name)().state_dict().items()}


@pytest.mark.parametrize("name", list(NETS))
def test_init_matches_reference(name):
    fx, sd = FX[name], _state(name)
    assert list(sd) == list(fx["shapes_state"])
    for k, shape in fx["shapes_state"].items():
        assert list(sd[k].shape) == shape, k
    for k, v in fx["init_abs_sum"].items():
        assert abs(float(sd[k].double().abs().sum()) - v) <= 1e-9 * (1 + abs(v)), k


@pytest.mark.parametrize("name", list(NETS))
def test_yardstick_matches_reference_outputs(name):
    from oracle.senet import se_resnet_yardstick

    fx = FX[name]
    layers, bottleneck = NETS[name]
    m = se_resnet_yardstick(_state(name), layers, bottleneck)
    x_eval = torch.randn(*fx["shapes"]["x_eval"], generator=torch.Generator().manual_seed(fx["seeds"]["x_eval"]))
    with torch.no_grad():
        _close(m.eval()(x_eval), fx["eval_logits"])
    x = torch.randn(*fx["shapes"]["x_train"], generator=torch.Generator().manual_seed(fx["seeds"]["x_train"]))
    y = torch.randint(0, 1000, (fx["shapes"]["x_train"][0],), generator=torch.Generator().manual_seed(fx["seeds"]["labels"]))
    out = m.train()(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    _close(out.detach(), fx["train_logits"])
    assert abs(float(loss.detach()) - fx["train_loss"]) <= 1e-4 * (1 + abs(fx["train_loss"]))
    for n, p in m.named_parameters():
        ref = fx["grad_norms"][n]
        assert abs(float(p.grad.double().norm()) - ref) <= 1e-3 * ref + 1e-8, n
    sd = m.state_dict()
    for k, v in fx["running"].items():
        _close(sd[k], v)
