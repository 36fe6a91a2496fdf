"""The drop-in SupCon constructors and the fp32 SupCon oracle of tests/test_gpu_supcon.py (oracle/supcon.py) replayed against
the fixture tests/golden/make_supcon_golden.py wrote from the reference's own model and losses: constructor init ==
reference init (resnet18 / resnet50, both stages); oracle SupCon loss and feature gradient == reference over labels / none,
n_views 2 and 3, temperatures 0.07 and 0.1; a 32 px stage-1 step's loss, embeddings, gradients and running statistics ==
reference; label-smoothing loss == reference."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
FX = torch.load(os.path.join(HERE, "golden", "supcon_golden.pt"), weights_only=False)

from make_supcon_golden import LOSS_CASES, loss_inputs, step_inputs  # noqa: E402


def _close(a, b, tol=1e-5):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


@pytest.mark.parametrize("case", sorted(FX["ctor"]))
def test_init_matches_reference(case):
    from deeplearning_b200.self_supervised.SupCon.models.model import SupConModel

    bb, stage2 = case
    torch.manual_seed(0)
    sd = SupConModel(bb, second_stage=stage2, num_classes=10 if stage2 else None).state_dict()
    fx = FX["ctor"][case]
    assert list(sd) == fx["keys"]
    for k, v in fx["abs_sum"].items():
        assert abs(float(sd[k].double().abs().sum()) - v) <= 1e-9 * (1 + abs(v)), k


@pytest.mark.parametrize("case", LOSS_CASES)
def test_oracle_loss_matches_reference(case):
    from oracle.supcon import supcon_loss

    lab, v, t = case
    f, y = loss_inputs(lab, v)
    f.requires_grad_(True)
    loss = supcon_loss(f, y, t, 0.07)
    loss.backward()
    _close(loss.detach(), FX["loss"][case]["loss"])
    _close(f.grad, FX["loss"][case]["grad"])


def test_oracle_step_matches_reference():
    from deeplearning_b200.self_supervised.SupCon.models.model import SupConModel
    from oracle.supcon import train_step_grads

    torch.manual_seed(0)
    state = {k: v.clone() for k, v in SupConModel("resnet18").state_dict().items()}
    x, y = step_inputs()
    emb, loss, grads = train_step_grads(state, x, y, 0.1)
    fx = FX["step"]
    _close(loss, fx["loss"])
    _close(emb[:, :16], fx["emb_slice"])
    assert set(grads) == set(fx["grad_norm"])
    for n, g in grads.items():
        _close(g.double().norm(), fx["grad_norm"][n], 1e-4)
        _close(g.flatten()[:16], fx["grad_slice"][n], 1e-4)
    for k, v in fx["running_mean_sum"].items():
        _close(state[k].double().sum(), v)


def test_oracle_label_smoothing_matches_reference():
    from oracle.supcon import label_smoothing_loss

    g = torch.Generator().manual_seed(7)
    pred, tgt = torch.randn(5, 10, generator=g), torch.randint(0, 10, (5,), generator=g)
    for s, v in FX["smooth"].items():
        _close(label_smoothing_loss(pred, tgt, 10, s), v)
