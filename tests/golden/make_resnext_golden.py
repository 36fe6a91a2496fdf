"""Pins the fp32 ResNeXt yardstick of the GPU tests against the reference itself and writes tests/golden/resnext_golden.pt,
which tests/test_oracle_resnext_golden.py replays on the CPU.

Run in the build container (needs /root/reference, which does NOT exist on the GPU box):
    python tests/golden/make_resnext_golden.py
It (1) builds the reference's own ``resnext50_32x4d()`` under a fixed seed, (2) checks that the drop-in constructor gives a
bit-identical state_dict under the same seed, (3) checks that torchvision's fp32 ``ResNet(Bottleneck, groups=32,
width_per_group=4)`` - the oracle of tests/test_gpu_resnext.py - gives bit-identical eval logits, train logits, loss, every
gradient and the running statistics on the same weights and inputs, and (4) stores small outputs only.
classification_golden.pt is not touched.
"""
import importlib.util
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)

LAYERS, KW = [3, 4, 6, 3], dict(groups=32, width_per_group=4)


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def yardstick(state):
    import torchvision

    m = torchvision.models.ResNet(torchvision.models.resnet.Bottleneck, LAYERS, **KW)
    m.load_state_dict(state)
    return m


def resnext50_fixture():
    from deeplearning_b200.classification.resnet.models.networks import resnext50_32x4d as mine_ctor

    ref_mod = _load(f"{REF}/classification/resnet/models/networks.py", "ref_resnet_networks")
    torch.manual_seed(0)
    ref = ref_mod.resnext50_32x4d()
    torch.manual_seed(0)
    mine = mine_ctor()
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = mine.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), "ctor init differs"
    x_eval = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    ref.eval()
    with torch.no_grad():
        le = ref(x_eval)
        lo = yardstick({k: v.clone() for k, v in sr.items()}).eval()(x_eval)
    assert torch.equal(le, lo), "yardstick eval forward differs from the reference"
    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    y = torch.randint(0, 1000, (4,), generator=torch.Generator().manual_seed(3))
    ys = yardstick({k: v.clone() for k, v in sr.items()}).train()
    ref.train()
    out = ref(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    out2 = ys(x)
    loss2 = F.cross_entropy(out2, y)
    loss2.backward()
    assert torch.equal(out, out2) and float(loss.detach()) == float(loss2.detach())
    yg = dict(ys.named_parameters())
    for n, p in ref.named_parameters():
        assert torch.equal(p.grad, yg[n].grad), n
    s2, s3 = ref.state_dict(), ys.state_dict()
    for k in s2:
        if "running" in k or "num_batches" in k:
            assert torch.equal(s2[k], s3[k]), k
    return {"init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items() if v.is_floating_point()},
            "eval_logits": le.clone(), "train_logits": out.detach().clone(), "train_loss": float(loss.detach()),
            "grad_norms": {n: float(p.grad.double().norm()) for n, p in ref.named_parameters()},
            "running_mean_layer1_bn2": s2["layer1.0.bn2.running_mean"].clone(),
            "running_var_layer4_bn2": s2["layer4.2.bn2.running_var"].clone(),
            "seeds": {"init": 0, "x_eval": 1, "x_train": 2, "labels": 3}, "shapes": {"x_eval": [2, 3, 64, 64], "x_train": [4, 3, 64, 64]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    path = os.path.join(HERE, "resnext_golden.pt")
    torch.save({"resnext50_32x4d": resnext50_fixture(), "torch": torch.__version__}, path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
