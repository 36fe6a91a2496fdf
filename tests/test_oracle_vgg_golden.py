"""The drop-in VGG constructors and the fp32 VGG oracle of tests/test_gpu_vgg.py (oracle/vgg.py) replayed against the
fixture tests/golden/make_vgg_golden.py wrote from the reference's own vgg11 / vgg11_bn at 32 px and 64 px: constructor init
== reference init; oracle forward / backward / running statistics with the fixture's dropout masks, and eval logits ==
reference."""
import os

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
FX = torch.load(os.path.join(HERE, "golden", "vgg_golden.pt"), weights_only=False)
CASES = ["vgg11_32", "vgg11_64", "vgg11_bn_32", "vgg11_bn_64"]


def _close(a, b, tol=2e-4):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


def _name(case):
    return case.rsplit("_", 1)[0]


def _state(case):
    from deeplearning_b200.classification.vggNet.models import network

    torch.manual_seed(FX[case]["seeds"]["init"])
    return {k: v.clone() for k, v in getattr(network, _name(case))(num_classes=FX["num_classes"]).state_dict().items()}


@pytest.mark.parametrize("case", CASES)
def test_init_matches_reference(case):
    fx, sd = FX[case], _state(case)
    assert list(sd) == list(fx["shapes_state"])
    for k, shape in fx["shapes_state"].items():
        assert list(sd[k].shape) == shape, k
    for k, v in fx["init_abs_sum"].items():
        assert abs(float(sd[k].double().abs().sum()) - v) <= 1e-9 * (1 + abs(v)), k


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_outputs(case):
    from oracle.vgg import arch, train_step_grads, vgg_forward

    fx = FX[case]
    state = _state(case)
    x = torch.randn(*fx["shapes"]["x_train"], generator=torch.Generator().manual_seed(fx["seeds"]["x_train"]))
    y = torch.randint(0, FX["num_classes"], (fx["shapes"]["x_train"][0],),
                      generator=torch.Generator().manual_seed(fx["seeds"]["labels"]))
    masks = [bits.float() / (1.0 - p) for bits, p in zip(fx["mask_bits"], fx["p"])]
    cfg, bn = arch(_name(case))
    out, loss, grads, after = train_step_grads(state, x, y, cfg, bn, masks)
    _close(out, fx["train_logits"])
    assert abs(float(loss) - fx["train_loss"]) <= 1e-4 * (1 + abs(fx["train_loss"]))
    assert set(grads) == set(fx["grad_norms"])
    for n, g in grads.items():
        ref = fx["grad_norms"][n]
        assert abs(float(g.double().norm()) - ref) <= 1e-3 * ref + 1e-8, n
        _close(g.flatten()[:fx["grad_slices"][n].numel()], fx["grad_slices"][n], tol=1e-3 * (1 + ref))
    assert bn == bool(fx["running"])
    for k, v in fx["running"].items():
        _close(after[k], v)
    x_eval = torch.randn(*fx["shapes"]["x_eval"], generator=torch.Generator().manual_seed(fx["seeds"]["x_eval"]))
    with torch.no_grad():
        _close(vgg_forward(after, x_eval, cfg, bn), fx["eval_logits"])
