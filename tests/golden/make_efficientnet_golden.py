"""Pins the drop-in EfficientNet constructors and the fp32 EfficientNet oracle of the GPU tests (oracle/efficientnet.py)
against the reference itself and writes tests/golden/efficientnet_golden.pt, which tests/test_oracle_efficientnet_golden.py
replays on the CPU.

Run where a checkout of the reference (and torchvision, which it imports) exists; it is not available to the GPU tests:
    python tests/golden/make_efficientnet_golden.py
For efficientnet_b0 and efficientnet_b2 at num_classes=5, batch 4, 72 px (36 -> 18 -> 9 -> 5 -> 3: stride 2 on odd sizes)
it (1) builds the reference's model under a fixed seed, (2) checks that the drop-in constructor gives a bit-identical
state_dict under the same seed, (3) runs a train step with the default drop-connect and dropout, ``torch.rand`` scripted as
in make_golden.py::droppath_fixture and the classifier-dropout mask reproduced from the generator state, and checks that
the oracle fed the same masks gives bit-identical logits, loss, every gradient and the running statistics, (4) checks the
eval logits, and (5) stores small outputs only.
"""
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _ScriptedRand, _load, _shim, drop_entries  # noqa: E402

NUM_CLASSES = 5
B, PX = 4, 72
NETS = {"b0": ("features.1a.block.dwconv.1.running_mean", "features.6c.block.project_conv.1.running_var"),
        "b2": ("features.1b.block.dwconv.1.running_var", "features.top.1.running_mean")}


def fixture(name, ref_mod):
    from deeplearning_b200.classification.efficientNet.models import network
    from oracle.efficientnet import efficientnet_forward, plan, train_step_grads

    torch.manual_seed(0)
    ref = getattr(ref_mod, f"efficientnet_{name}")(num_classes=NUM_CLASSES)
    torch.manual_seed(0)
    m = getattr(network, f"efficientnet_{name}")(num_classes=NUM_CLASSES)
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = m.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), f"{name}: ctor init differs"

    blocks = plan(name)
    x = torch.randn(B, 3, PX, PX, generator=torch.Generator().manual_seed(2))
    y = torch.randint(0, NUM_CLASSES, (B,), generator=torch.Generator().manual_seed(3))
    us = [torch.rand(B, generator=torch.Generator().manual_seed(100 + i)) for i in range(64)]
    drop_mod = ref.classifier[0]
    p = drop_mod.p
    saved = {}
    drop_mod.register_forward_pre_hook(lambda mod, inp: saved.update(rng=torch.get_rng_state()))
    torch.manual_seed(7)
    ref.train()
    with _ScriptedRand(us) as sc:
        out = ref(x)
        used = sc.i
    loss = F.cross_entropy(out, y)
    loss.backward()
    # the reference's nn.Dropout drew its Bernoulli mask from the generator state before the call
    after = torch.get_rng_state()
    torch.set_rng_state(saved["rng"])
    mask = F.dropout(torch.ones(B, ref.classifier[1].in_features), p, True, inplace=True)
    torch.set_rng_state(after)
    # the reference draws for the blocks that have a DropPath only
    probs = [r for idx, _, _, r in blocks if type(ref.features._modules[idx].dropout).__name__ == "DropPath"]
    drop, n = drop_entries(probs, us, 1)
    assert n == used and used > 0, (n, used)
    assert any(float(e[0].min()) == 0.0 for e in drop), "no sample was dropped: pick other seeds"
    assert float(mask.min()) == 0.0, "no feature was dropped: pick another seed"
    lg, lo, grads, s_after = train_step_grads(sr, x, y, blocks, drop=drop, mask=mask)
    assert torch.equal(lg, out.detach()) and float(lo) == float(loss.detach()), name
    for n_, p_ in ref.named_parameters():
        assert torch.equal(p_.grad, grads[n_]), (name, n_)
    s2 = ref.state_dict()
    for k in s2:
        if "running" in k or "num_batches" in k:
            assert torch.equal(s2[k], s_after[k]), (name, k)
    x_eval = torch.randn(2, 3, PX, PX, generator=torch.Generator().manual_seed(1))
    ref.eval()
    with torch.no_grad():
        le = ref(x_eval)
        lo_e = efficientnet_forward({k: v.clone() for k, v in s2.items()}, x_eval, blocks)
    assert torch.equal(le, lo_e), f"{name}: oracle eval forward differs from the reference"
    return {"init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items() if v.is_floating_point()},
            "shapes_state": {k: list(v.shape) for k, v in sr.items()},
            "train_logits": out.detach().clone(), "train_loss": float(loss.detach()),
            "grad_norms": {n_: float(p_.grad.double().norm()) for n_, p_ in ref.named_parameters()},
            "running": {k: s2[k].clone() for k in NETS[name]},
            "drop": drop, "mask": mask.clone(), "eval_logits": le.clone(),
            "seeds": {"init": 0, "x_eval": 1, "x_train": 2, "labels": 3, "u0": 100},
            "shapes": {"x_eval": [2, 3, PX, PX], "x_train": [B, 3, PX, PX]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    _shim("torchsummary", summary=lambda *a, **k: None)
    ref_mod = _load(f"{REF}/classification/efficientNet/models/network.py", "ref_efficientnet_network")
    path = os.path.join(HERE, "efficientnet_golden.pt")
    torch.save({**{name: fixture(name, ref_mod) for name in NETS}, "num_classes": NUM_CLASSES, "torch": torch.__version__},
               path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
