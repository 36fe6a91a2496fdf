"""Pins the drop-in ShuffleNet v2 constructors and the fp32 ShuffleNet v2 oracle of the GPU tests (oracle/shufflenetv2.py)
against the reference itself and writes tests/golden/shufflenetv2_golden.pt, which tests/test_oracle_shufflenetv2_golden.py
replays on the CPU.

Run where a checkout of the reference exists; it is not available to the GPU tests:
    python tests/golden/make_shufflenetv2_golden.py
For shufflenet_v2_x0_5 / x1_0 / x2_0 at num_classes=5, batch 4, 64 px it (1) builds the reference's model under a fixed
seed, (2) checks that the drop-in constructor gives a bit-identical state_dict under the same seed, (3) runs a train step
of the reference's own modules and checks that the oracle gives bit-identical logits, loss, every gradient and the running
statistics, (4) checks the eval logits after the step, and (5) stores small outputs only: logits, loss, per-parameter
gradient norms and a fixed slice of each gradient, and the running statistics.  Weights are regenerated from the seed by the
replay.
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

from make_golden import _load  # noqa: E402

NUM_CLASSES = 5
B = 4
PX = 64
NETS = ["x0_5", "x1_0", "x2_0"]
SLICE = 16   # leading elements of every flattened gradient kept in the fixture


def fixture(name, ref_mod):
    from deeplearning_b200.classification.ShuffleNet.models import shufflenetv2
    from oracle.shufflenetv2 import shufflenetv2_forward, train_step_grads

    ctor = f"shufflenet_v2_{name}"
    torch.manual_seed(0)
    ref = getattr(ref_mod, ctor)(num_classes=NUM_CLASSES)
    torch.manual_seed(0)
    m = getattr(shufflenetv2, ctor)(num_classes=NUM_CLASSES)
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = m.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), f"{name}: ctor init differs"
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in m.named_parameters()], name

    x = torch.randn(B, 3, PX, PX, generator=torch.Generator().manual_seed(2))
    y = torch.randint(0, NUM_CLASSES, (B,), generator=torch.Generator().manual_seed(3))
    ref.train()
    out = ref(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    lg, lo, grads, s_after = train_step_grads(sr, x, y)
    assert torch.equal(lg, out.detach()) and float(lo) == float(loss.detach()), name
    for n_, p_ in ref.named_parameters():
        assert torch.equal(p_.grad, grads[n_]), (name, n_)
    s2 = ref.state_dict()
    running = {}
    for k in s2:
        if "running" in k or "num_batches" in k:
            assert torch.equal(s2[k], s_after[k]), (name, k)
            running[k] = s2[k].clone()
    x_eval = torch.randn(B, 3, PX, PX, generator=torch.Generator().manual_seed(1))
    ref.eval()
    with torch.no_grad():
        le = ref(x_eval)
        lo_e = shufflenetv2_forward({k: v.clone() for k, v in s2.items()}, x_eval)
    assert torch.equal(le, lo_e), f"{name}: oracle eval forward differs from the reference"
    return {"init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items() if v.is_floating_point()},
            "shapes_state": {k: list(v.shape) for k, v in sr.items()},
            "train_logits": out.detach().clone(), "train_loss": float(loss.detach()),
            "grad_norms": {n_: float(p_.grad.double().norm()) for n_, p_ in ref.named_parameters()},
            "grad_slices": {n_: p_.grad.flatten()[:SLICE].clone() for n_, p_ in ref.named_parameters()},
            "running": running, "eval_logits": le.clone(),
            "seeds": {"init": 0, "x_eval": 1, "x_train": 2, "labels": 3},
            "shapes": {"x_eval": [B, 3, PX, PX], "x_train": [B, 3, PX, PX]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    ref_mod = _load(f"{REF}/classification/ShuffleNet/models/shufflenetv2.py", "ref_shufflenetv2")
    path = os.path.join(HERE, "shufflenetv2_golden.pt")
    fx = {name: fixture(name, ref_mod) for name in NETS}
    torch.save({**fx, "num_classes": NUM_CLASSES, "torch": torch.__version__}, path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
