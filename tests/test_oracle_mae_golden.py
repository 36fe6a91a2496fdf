"""The drop-in MAE constructor and the fp32 MAE oracle of tests/test_gpu_mae.py (oracle/mae.py) replayed against the
fixture tests/golden/make_mae_golden.py wrote from the reference's own models at 32 px (an enc_to_dec Linear and an
Identity): constructor init == reference init; oracle pred, mask_patches, loss and every gradient == reference."""
import os

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
FX = torch.load(os.path.join(HERE, "golden", "mae_golden.pt"), weights_only=False)
CASES = ["linear", "identity"]


def _close(a, b, tol=2e-4):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


def _state(case):
    from deeplearning_b200.self_supervised.MAE.models.MAE import MAEVisonTransformer

    torch.manual_seed(FX[case]["seeds"]["init"])
    m = MAEVisonTransformer(**FX[case]["config"])
    return {k: v.clone() for k, v in m.state_dict().items()}


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
    from oracle.mae import train_step_grads

    fx = FX[case]
    cfg = fx["config"]
    x = torch.randn(*fx["shapes"]["x"], generator=torch.Generator().manual_seed(fx["seeds"]["x"]))
    pred, mp, loss, grads = train_step_grads(_state(case), x, fx["shuffle"], cfg["patch_size"], cfg["num_encoder_head"],
                                             cfg["num_decoder_head"], cfg["mask_ratio"])
    _close(pred, fx["pred"])
    assert torch.equal(mp, fx["mask_patches"])
    assert abs(float(loss) - fx["loss"]) <= 1e-5 * (1 + abs(fx["loss"]))
    assert set(grads) == set(fx["grad_norms"])
    assert "encoder.cls_token" not in grads and not any(n.startswith("encoder.mlp_head") for n in grads)
    for n, g in grads.items():
        ref = fx["grad_norms"][n]
        assert abs(float(g.double().norm()) - ref) <= 1e-3 * ref + 1e-8, n
        _close(g.flatten()[:fx["grad_slices"][n].numel()], fx["grad_slices"][n], tol=1e-3 * (1 + ref))


def test_shuffle_is_the_stable_argsort_of_the_draw():
    """The fixture's shuffle came from torch.rand(B, P).argsort(); on a draw without ties it is the stable argsort the GPU
    engine computes."""
    for case in CASES:
        fx = FX[case]
        B, _, H, W = fx["shapes"]["x"]
        p = fx["config"]["patch_size"]
        torch.manual_seed(fx["seeds"]["shuffle"])
        keys = torch.rand(B, (H // p) * (W // p))
        assert torch.equal(keys.argsort(dim=1, stable=True), fx["shuffle"])
