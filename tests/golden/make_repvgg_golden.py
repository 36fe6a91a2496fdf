"""Pins the drop-in RepVGG constructors and the fp32 RepVGG oracle of the GPU tests (oracle/repvgg.py) against the reference
itself and writes tests/golden/repvgg_golden.pt, which tests/test_oracle_repvgg_golden.py replays on the CPU.

Run where a checkout of the reference exists (it is not available to the GPU tests):
    python tests/golden/make_repvgg_golden.py
For create_RepVGG_A0 and create_RepVGG_B0 at num_classes=5 it (1) builds the reference's model under a fixed seed, (2) checks
that the drop-in constructor gives a bit-identical state_dict under the same seed, (3) checks that the oracle gives
bit-identical train logits, loss, every gradient, the running statistics, and eval logits before and after
repvgg_model_convert on the same weights and inputs, and (4) stores small outputs only.
"""
import contextlib
import io
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)

NUM_CLASSES = 5
# name -> running-statistics keys to store
NETS = {"RepVGG-A0": ("stage1.1.rbr_identity.running_mean", "stage3.13.rbr_dense.bn.running_var"),
        "RepVGG-B0": ("stage0.rbr_1x1.bn.running_mean", "stage2.5.rbr_identity.running_var")}


def _reference_module():
    sys.path.insert(0, os.path.join(REF, "classification", "RepVGG"))
    import models.repvgg as ref_mod   # the reference's own package layout (models/se_block.py)

    return ref_mod


def fixture(name, ref_mod):
    from deeplearning_b200.classification.RepVGG.models import func_dict
    from oracle.repvgg import build, convert

    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):   # the reference prints every block
        ref = ref_mod.func_dict[name](num_classes=NUM_CLASSES)
    torch.manual_seed(0)
    m = func_dict[name](num_classes=NUM_CLASSES)
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = m.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), f"{name}: ctor init differs"

    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    y = torch.randint(0, NUM_CLASSES, (4,), generator=torch.Generator().manual_seed(3))
    orc = build(name, {k: v.clone() for k, v in sr.items()}, NUM_CLASSES).train()
    ref.train()
    out = ref(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    out2 = orc(x)
    loss2 = F.cross_entropy(out2, y)
    loss2.backward()
    assert torch.equal(out, out2) and float(loss.detach()) == float(loss2.detach()), name
    og = dict(orc.named_parameters())
    for n, p in ref.named_parameters():
        assert torch.equal(p.grad, og[n].grad), (name, n)
    s2, s3 = ref.state_dict(), orc.state_dict()
    for k in s2:
        if "running" in k or "num_batches" in k:
            assert torch.equal(s2[k], s3[k]), (name, k)
    # eval logits with the running statistics of that step, before and after the re-parameterisation
    x_eval = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    ref.eval()
    orc.eval()
    with torch.no_grad():
        le, lo = ref(x_eval), orc(x_eval)
        assert torch.equal(le, lo), f"{name}: oracle eval forward differs from the reference"
        ld = ref_mod.repvgg_model_convert(ref)(x_eval)
        lod = convert(orc)(x_eval)
        assert torch.equal(ld, lod), f"{name}: oracle fold differs from repvgg_model_convert"
    return {"init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items() if v.is_floating_point()},
            "shapes_state": {k: list(v.shape) for k, v in sr.items()},
            "train_logits": out.detach().clone(), "train_loss": float(loss.detach()),
            "grad_norms": {n: float(p.grad.double().norm()) for n, p in ref.named_parameters()},
            "running": {k: s2[k].clone() for k in NETS[name]},
            "eval_logits": le.clone(), "deploy_logits": ld.clone(),
            "seeds": {"init": 0, "x_eval": 1, "x_train": 2, "labels": 3},
            "shapes": {"x_eval": [2, 3, 64, 64], "x_train": [4, 3, 64, 64]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    ref_mod = _reference_module()
    path = os.path.join(HERE, "repvgg_golden.pt")
    torch.save({**{name: fixture(name, ref_mod) for name in NETS}, "num_classes": NUM_CLASSES, "torch": torch.__version__},
               path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
