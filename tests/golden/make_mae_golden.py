"""Pins the drop-in MAE constructor and the fp32 MAE oracle of the GPU tests (oracle/mae.py) against the reference itself and
writes tests/golden/mae_golden.pt, which tests/test_oracle_mae_golden.py replays on the CPU.

Run where a checkout of the reference exists; it is not available to the GPU tests:
    python tests/golden/make_mae_golden.py
For two tiny configurations (32 px, patch 8: an enc_to_dec Linear 64 -> 128 under an attention width of 128 over the
64-wide encoder, and an Identity at 128 / 128) it (1) builds the reference's ``MAEVisonTransformer`` under a fixed seed,
(2) checks that the drop-in constructor gives a bit-identical
state_dict under the same seed, (3) runs the reference's forward with a seeded CPU draw, recomputes the shuffle it used from
the same draw, and checks that the oracle fed that shuffle gives bit-identical pred, mask_patches, loss and every gradient,
and (4) stores small outputs only: the shuffle, pred, mask_patches, loss, per-parameter gradient norms and a fixed slice of
each gradient.  Weights are regenerated from the seed by the replay.
"""
import os
import sys
import types

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _load  # noqa: E402

B = 3
PX = 32
SLICE = 16   # leading elements of every flattened gradient kept in the fixture
CONFIGS = {
    "linear": dict(image_size=PX, patch_size=8, encoer_dim=64, mlp_dim=128, encoder_depth=2, num_encoder_head=2,
                   dim_per_head=64, decoder_dim=128, decoder_depth=2, num_decoder_head=2, mask_ratio=0.75),
    "identity": dict(image_size=PX, patch_size=8, encoer_dim=128, mlp_dim=256, encoder_depth=2, num_encoder_head=2,
                     dim_per_head=64, decoder_dim=128, decoder_depth=1, num_decoder_head=2, mask_ratio=0.75),
}


def _reference():
    """The reference's models/MAE.py, whose ``from models.VIT import ...`` resolves to the reference's VIT.py."""
    pkg = types.ModuleType("models")
    pkg.__path__ = []
    sys.modules["models"] = pkg
    sys.modules["models.VIT"] = _load(f"{REF}/self-supervised/MAE/models/VIT.py", "models.VIT")
    return _load(f"{REF}/self-supervised/MAE/models/MAE.py", "ref_mae")


def fixture(name, ref_mod):
    from deeplearning_b200.self_supervised.MAE.models.MAE import MAEVisonTransformer
    from oracle.mae import train_step_grads

    cfg = CONFIGS[name]
    torch.manual_seed(0)
    ref = ref_mod.MAEVisonTransformer(**cfg)
    torch.manual_seed(0)
    m = MAEVisonTransformer(**cfg)
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = m.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), f"{name}: ctor init differs"
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in m.named_parameters()], name
    assert isinstance(ref.enc_to_dec, torch.nn.Linear) == (name == "linear"), name

    x = torch.randn(B, 3, PX, PX, generator=torch.Generator().manual_seed(2))
    P = (PX // cfg["patch_size"]) ** 2
    torch.manual_seed(5)
    pred, mask_patches = ref(x)
    loss = F.mse_loss(pred, mask_patches)
    loss.backward()
    torch.manual_seed(5)
    shuffle = torch.rand(B, P).argsort()
    o_pred, o_mp, o_loss, grads = train_step_grads(sr, x, shuffle, cfg["patch_size"], cfg["num_encoder_head"],
                                                   cfg["num_decoder_head"], cfg["mask_ratio"])
    assert torch.equal(o_pred, pred.detach()) and torch.equal(o_mp, mask_patches), name
    assert float(o_loss) == float(loss.detach()), name
    with_grad = {n_: p_ for n_, p_ in ref.named_parameters() if p_.grad is not None}
    assert set(with_grad) == set(grads), (name, set(with_grad) ^ set(grads))
    assert not any(n_.startswith(("encoder.cls_token", "encoder.mlp_head")) for n_ in grads), name
    for n_, p_ in with_grad.items():
        assert torch.equal(p_.grad, grads[n_]), (name, n_)
    return {"config": cfg, "shuffle": shuffle.clone(), "init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items()},
            "shapes_state": {k: list(v.shape) for k, v in sr.items()},
            "pred": pred.detach().clone(), "mask_patches": mask_patches.clone(), "loss": float(loss.detach()),
            "grad_norms": {n_: float(p_.grad.double().norm()) for n_, p_ in with_grad.items()},
            "grad_slices": {n_: p_.grad.flatten()[:SLICE].clone() for n_, p_ in with_grad.items()},
            "seeds": {"init": 0, "x": 2, "shuffle": 5}, "shapes": {"x": [B, 3, PX, PX]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    ref_mod = _reference()
    path = os.path.join(HERE, "mae_golden.pt")
    fx = {name: fixture(name, ref_mod) for name in CONFIGS}
    torch.save({**fx, "torch": torch.__version__}, path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
