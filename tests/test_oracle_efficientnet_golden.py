"""The drop-in EfficientNet constructors and the fp32 EfficientNet oracle of tests/test_gpu_efficientnet.py
(oracle/efficientnet.py) replayed against the fixture tests/golden/make_efficientnet_golden.py wrote from the reference's
own efficientnet_b0 / efficientnet_b2: constructor init == reference init; oracle forward / backward / running statistics
with the fixture's drop-connect and dropout masks, and eval logits == reference."""
import os

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
FX = torch.load(os.path.join(HERE, "golden", "efficientnet_golden.pt"), weights_only=False)
NETS = ["b0", "b2"]


def _close(a, b, tol=2e-4):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


def _state(name):
    from deeplearning_b200.classification.efficientNet.models import network

    torch.manual_seed(FX[name]["seeds"]["init"])
    return {k: v.clone() for k, v in getattr(network, f"efficientnet_{name}")(num_classes=FX["num_classes"]).state_dict().items()}


@pytest.mark.parametrize("name", NETS)
def test_init_matches_reference(name):
    fx, sd = FX[name], _state(name)
    assert list(sd) == list(fx["shapes_state"])
    for k, shape in fx["shapes_state"].items():
        assert list(sd[k].shape) == shape, k
    for k, v in fx["init_abs_sum"].items():
        assert abs(float(sd[k].double().abs().sum()) - v) <= 1e-9 * (1 + abs(v)), k


@pytest.mark.parametrize("name", NETS)
def test_oracle_matches_reference_outputs(name):
    from oracle.efficientnet import efficientnet_forward, plan, train_step_grads

    fx = FX[name]
    state = _state(name)
    x = torch.randn(*fx["shapes"]["x_train"], generator=torch.Generator().manual_seed(fx["seeds"]["x_train"]))
    y = torch.randint(0, FX["num_classes"], (fx["shapes"]["x_train"][0],),
                      generator=torch.Generator().manual_seed(fx["seeds"]["labels"]))
    blocks = plan(name)
    out, loss, grads, after = train_step_grads(state, x, y, blocks, drop=fx["drop"], mask=fx["mask"])
    _close(out, fx["train_logits"])
    assert abs(float(loss) - fx["train_loss"]) <= 1e-4 * (1 + abs(fx["train_loss"]))
    assert set(grads) == set(fx["grad_norms"])
    for n, g in grads.items():
        ref = fx["grad_norms"][n]
        assert abs(float(g.double().norm()) - ref) <= 1e-3 * ref + 1e-8, n
    for k, v in fx["running"].items():
        _close(after[k], v)
    x_eval = torch.randn(*fx["shapes"]["x_eval"], generator=torch.Generator().manual_seed(fx["seeds"]["x_eval"]))
    with torch.no_grad():
        _close(efficientnet_forward(after, x_eval, blocks), fx["eval_logits"])
