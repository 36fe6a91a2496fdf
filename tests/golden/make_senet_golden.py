"""Pins the drop-in SE-ResNet constructors and the fp32 SE-ResNet yardstick of the GPU tests (oracle/senet.py) against the
reference itself and writes tests/golden/senet_golden.pt, which tests/test_oracle_senet_golden.py replays on the CPU.

Run where a checkout of the reference exists (it is not available to the GPU tests):
    python tests/golden/make_senet_golden.py
For se_resnet50() and se_resnet() it (1) builds the reference's model under a fixed seed, (2) checks that the drop-in
constructor gives a bit-identical state_dict under the same seed, (3) checks that the yardstick gives bit-identical eval
logits, train logits, loss, every gradient and the running statistics on the same weights and inputs, and (4) stores small
outputs only.  classification_golden.pt and oracle/resnet.py are not touched.
"""
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)

# name -> (layers, bottleneck, running-statistics keys to store)
NETS = {"se_resnet50": ((3, 4, 6, 3), True, ("layer1.0.bn3.running_mean", "layer4.2.bn3.running_var")),
        "se_resnet": ((2, 2, 2, 2), False, ("layer1.0.bn2.running_mean", "layer4.1.bn2.running_var"))}


def _reference_module():
    sys.path.insert(0, os.path.join(REF, "classification", "seNet"))
    import models.se_resnet as ref_mod   # the reference's own package layout (models/se_module.py)

    return ref_mod


def fixture(name, ref_mod):
    from deeplearning_b200.classification.seNet.models import networks as mine
    from oracle.senet import se_resnet_yardstick

    layers, bottleneck, keys = NETS[name]
    torch.manual_seed(0)
    ref = getattr(ref_mod, name)()
    torch.manual_seed(0)
    m = getattr(mine, name)()
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = m.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), f"{name}: ctor init differs"

    def yard():
        return se_resnet_yardstick({k: v.clone() for k, v in sr.items()}, layers, bottleneck)

    x_eval = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    ref.eval()
    with torch.no_grad():
        le = ref(x_eval)
        lo = yard().eval()(x_eval)
    assert torch.equal(le, lo), f"{name}: yardstick eval forward differs from the reference"
    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    y = torch.randint(0, 1000, (4,), generator=torch.Generator().manual_seed(3))
    ys = yard().train()
    ref.train()
    out = ref(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    out2 = ys(x)
    loss2 = F.cross_entropy(out2, y)
    loss2.backward()
    assert torch.equal(out, out2) and float(loss.detach()) == float(loss2.detach()), name
    yg = dict(ys.named_parameters())
    for n, p in ref.named_parameters():
        assert torch.equal(p.grad, yg[n].grad), (name, n)
    s2, s3 = ref.state_dict(), ys.state_dict()
    for k in s2:
        if "running" in k or "num_batches" in k:
            assert torch.equal(s2[k], s3[k]), (name, k)
    return {"init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items() if v.is_floating_point()},
            "shapes_state": {k: list(v.shape) for k, v in sr.items()},
            "eval_logits": le.clone(), "train_logits": out.detach().clone(), "train_loss": float(loss.detach()),
            "grad_norms": {n: float(p.grad.double().norm()) for n, p in ref.named_parameters()},
            "running": {k: s2[k].clone() for k in keys},
            "seeds": {"init": 0, "x_eval": 1, "x_train": 2, "labels": 3},
            "shapes": {"x_eval": [2, 3, 64, 64], "x_train": [4, 3, 64, 64]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    ref_mod = _reference_module()
    path = os.path.join(HERE, "senet_golden.pt")
    torch.save({**{name: fixture(name, ref_mod) for name in NETS}, "torch": torch.__version__}, path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
