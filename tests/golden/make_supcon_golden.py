"""Pins the drop-in SupCon constructors and the fp32 SupCon oracle of the GPU tests (oracle/supcon.py) against the reference
itself and writes tests/golden/supcon_golden.pt, which tests/test_oracle_supcon_golden.py replays on the CPU.

Run where a checkout of the reference exists; it is not available to the GPU tests:
    python tests/golden/make_supcon_golden.py
The reference's models/model.py imports timm, which is stubbed, and builds its encoders with ``pretrained=True``: its
``BACKBONES`` entries are replaced with torchvision's constructors at random initialisation.  It checks, bit for bit:
(1) the drop-in's seeded state_dict against the reference's for resnet18 and resnet50 in stage 1 and stage 2;
(2) the oracle's SupCon loss and feature gradient against the reference's SupConLoss over labels / none, n_views 2 and 3
and temperatures 0.07 / 0.1; (3) a tiny 32 px stage-1 step of resnet18 (loss and every parameter gradient) against the
reference model and loss under autograd; (4) the oracle's label-smoothing loss against the reference's LabelSmoothingLoss.
It stores small outputs only (losses, norms and slices); inputs and weights are regenerated from the seeds by the replay.
"""
import os
import sys
import types

import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference/self-supervised/SupCon"
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _load  # noqa: E402

SLICE = 16
LOSS_CASES = [(lab, v, t) for lab in (True, False) for v in (2, 3) for t in (0.07, 0.1)]
BSZ, DIM = 6, 32


def _reference():
    sys.modules["timm"] = types.ModuleType("timm")
    pkg = types.ModuleType("models")
    pkg.__path__ = []
    sys.modules["models"] = pkg
    bb = _load(f"{REF}/models/backbone.py", "models.backbone")
    for k in list(bb.BACKBONES):
        ctor = getattr(torchvision.models, {"wide_resnet50": "wide_resnet50_2", "wide_resnet101": "wide_resnet101_2"}.get(k, k))
        bb.BACKBONES[k] = (lambda c: (lambda pretrained=True: c(weights=None)))(ctor)
    sys.modules["models.backbone"] = bb
    model = _load(f"{REF}/models/model.py", "ref_supcon_model")
    loss = _load(f"{REF}/losses/SupConLoss.py", "ref_supcon_loss")
    smooth = _load(f"{REF}/losses/LabelSmooth.py", "ref_label_smooth")
    return model, loss, smooth


def loss_inputs(labels, n_views, seed=3):
    g = torch.Generator().manual_seed(seed)
    f = torch.nn.functional.normalize(torch.randn(BSZ, n_views, DIM, generator=g), dim=-1)
    y = torch.randint(0, 3, (BSZ,), generator=g) if labels else None
    return f, y


def step_inputs(seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(8, 3, 32, 32, generator=g), torch.randint(0, 2, (4,), generator=g)


def main():
    from deeplearning_b200.self_supervised.SupCon.models.model import SupConModel
    from oracle.supcon import label_smoothing_loss, supcon_loss, train_step_grads

    ref_model, ref_loss, ref_smooth = _reference()
    fx = {"ctor": {}, "loss": {}, "step": {}, "smooth": {}}
    for bb in ("resnet18", "resnet50"):
        for stage2 in (False, True):
            kw = dict(backbone=bb, second_stage=stage2, num_classes=10 if stage2 else None)
            torch.manual_seed(0)
            r = ref_model.SupConModel(**kw).state_dict()
            torch.manual_seed(0)
            m = SupConModel(**kw).state_dict()
            assert list(r) == list(m) and all(torch.equal(r[k], m[k]) for k in r), f"{bb} stage2={stage2}: init differs"
            fx["ctor"][(bb, stage2)] = {"keys": list(m), "abs_sum": {k: float(v.double().abs().sum()) for k, v in m.items()}}
    for lab, v, t in LOSS_CASES:
        f, y = loss_inputs(lab, v)
        fr = f.clone().requires_grad_(True)
        lr = ref_loss.SupConLoss(temperature=t)(fr, y)
        lr.backward()
        fo = f.clone().requires_grad_(True)
        lo = supcon_loss(fo, y, t, 0.07)
        lo.backward()
        assert torch.equal(lr, lo) and torch.equal(fr.grad, fo.grad), (lab, v, t)
        fx["loss"][(lab, v, t)] = {"loss": float(lo.detach()), "grad": fo.grad.clone()}
    torch.manual_seed(0)
    ref = ref_model.SupConModel(backbone="resnet18", projection_dim=128)
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    x, y = step_inputs()
    ref.train()
    emb = ref(x)
    f1, f2 = torch.split(emb, [4, 4], dim=0)
    lr = ref_loss.SupConLoss(temperature=0.1)(torch.cat([f1.unsqueeze(1), f2.unsqueeze(1)], dim=1), y)
    lr.backward()
    emb_o, lo, grads = train_step_grads(state, x, y, 0.1)
    assert torch.equal(lr.detach(), lo) and torch.equal(emb.detach(), emb_o), (float(lr), float(lo))
    for n, p in ref.named_parameters():
        assert torch.equal(p.grad, grads[n]), n
    for k, v in ref.state_dict().items():
        assert torch.equal(v, state[k]), k
    fx["step"] = {"loss": float(lo), "emb_slice": emb_o[:, :SLICE].clone(),
                  "grad_norm": {n: float(g.double().norm()) for n, g in grads.items()},
                  "grad_slice": {n: g.flatten()[:SLICE].clone() for n, g in grads.items()},
                  "running_mean_sum": {k: float(v.double().sum()) for k, v in state.items() if "running_mean" in k}}
    g = torch.Generator().manual_seed(7)
    pred, tgt = torch.randn(5, 10, generator=g), torch.randint(0, 10, (5,), generator=g)
    for s in (0.0, 0.01, 0.1):
        r = ref_smooth.LabelSmoothingLoss(classes=10, smoothing=s)(pred, tgt)
        o = label_smoothing_loss(pred, tgt, 10, s)
        assert torch.equal(r, o), s
        fx["smooth"][s] = float(o)
    torch.save(fx, os.path.join(HERE, "supcon_golden.pt"))
    print("wrote supcon_golden.pt")


if __name__ == "__main__":
    main()
