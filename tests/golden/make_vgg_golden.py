"""Pins the drop-in VGG constructors and the fp32 VGG oracle of the GPU tests (oracle/vgg.py) against the reference itself
and writes tests/golden/vgg_golden.pt, which tests/test_oracle_vgg_golden.py replays on the CPU.

Run where a checkout of the reference (and torchvision, which it imports) exists; it is not available to the GPU tests:
    python tests/golden/make_vgg_golden.py
For vgg11 and vgg11_bn at num_classes=5, batch 2, at 32 px and 64 px (1x1 and 2x2 maps in front of the adaptive pool) it
(1) builds the reference's model under a fixed seed, (2) checks that the drop-in constructor gives a bit-identical
state_dict under the same seed, (3) runs a train step with the reference's two nn.Dropout() layers, their masks reproduced
from the generator state a forward pre-hook saves on each (CPU dropout draws a Bernoulli noise tensor of the input's shape
and multiplies by it, so F.dropout of a tensor of ones from that state is the mask), and checks that the oracle fed the same
masks gives bit-identical logits, loss, every gradient and the running statistics, (4) checks the eval logits after the
step, and (5) stores small outputs only: logits, loss, per-parameter gradient norms and a fixed slice of each gradient, the
running statistics and the masks (as bits).  Weights are regenerated from the seed by the replay.
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

from make_golden import _load, _shim  # noqa: E402

NUM_CLASSES = 5
B = 2
NETS = ("vgg11", "vgg11_bn")
PXS = (32, 64)
SLICE = 16   # leading elements of every flattened gradient kept in the fixture


def fixture(name, px, ref_mod):
    from deeplearning_b200.classification.vggNet.models import network
    from oracle.vgg import arch, train_step_grads, vgg_forward

    torch.manual_seed(0)
    ref = getattr(ref_mod, name)(num_classes=NUM_CLASSES)
    torch.manual_seed(0)
    m = getattr(network, name)(num_classes=NUM_CLASSES)
    sr = {k: v.clone() for k, v in ref.state_dict().items()}
    sm = m.state_dict()
    assert list(sr.keys()) == list(sm.keys()) and all(torch.equal(sr[k], sm[k]) for k in sr), f"{name}: ctor init differs"
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in m.named_parameters()], name

    x = torch.randn(B, 3, px, px, generator=torch.Generator().manual_seed(2))
    y = torch.randint(0, NUM_CLASSES, (B,), generator=torch.Generator().manual_seed(3))
    saved = []
    drops = [ref.classifier[2], ref.classifier[5]]
    for d in drops:
        d.register_forward_pre_hook(lambda mod, inp: saved.append((torch.get_rng_state(), tuple(inp[0].shape))))
    torch.manual_seed(7)
    ref.train()
    out = ref(x)
    loss = F.cross_entropy(out, y)
    loss.backward()
    after = torch.get_rng_state()
    masks = []
    for (state, shape), d in zip(saved, drops):
        torch.set_rng_state(state)
        masks.append(F.dropout(torch.ones(shape), d.p, True))
    torch.set_rng_state(after)
    assert all(float(mk.min()) == 0.0 for mk in masks), "no feature was dropped: pick another seed"
    cfg, bn = arch(name)
    lg, lo, grads, s_after = train_step_grads(sr, x, y, cfg, bn, masks)
    assert torch.equal(lg, out.detach()) and float(lo) == float(loss.detach()), (name, px)
    for n_, p_ in ref.named_parameters():
        assert torch.equal(p_.grad, grads[n_]), (name, px, n_)
    s2 = ref.state_dict()
    running = {}
    for k in s2:
        if "running" in k or "num_batches" in k:
            assert torch.equal(s2[k], s_after[k]), (name, px, k)
            running[k] = s2[k].clone()
    x_eval = torch.randn(B, 3, px, px, generator=torch.Generator().manual_seed(1))
    ref.eval()
    with torch.no_grad():
        le = ref(x_eval)
        lo_e = vgg_forward({k: v.clone() for k, v in s2.items()}, x_eval, cfg, bn)
    assert torch.equal(le, lo_e), f"{name} {px}px: oracle eval forward differs from the reference"
    return {"init_abs_sum": {k: float(v.double().abs().sum()) for k, v in sr.items() if v.is_floating_point()},
            "shapes_state": {k: list(v.shape) for k, v in sr.items()},
            "train_logits": out.detach().clone(), "train_loss": float(loss.detach()),
            "grad_norms": {n_: float(p_.grad.double().norm()) for n_, p_ in ref.named_parameters()},
            "grad_slices": {n_: p_.grad.flatten()[:SLICE].clone() for n_, p_ in ref.named_parameters()},
            "running": running, "mask_bits": [mk != 0 for mk in masks], "p": [float(d.p) for d in drops],
            "eval_logits": le.clone(),
            "seeds": {"init": 0, "x_eval": 1, "x_train": 2, "labels": 3},
            "shapes": {"x_eval": [B, 3, px, px], "x_train": [B, 3, px, px]}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    _shim("torchsummary", summary=lambda *a, **k: None)
    ref_mod = _load(f"{REF}/classification/vggNet/models/network.py", "ref_vgg_network")
    path = os.path.join(HERE, "vgg_golden.pt")
    fx = {f"{name}_{px}": fixture(name, px, ref_mod) for name in NETS for px in PXS}
    torch.save({**fx, "num_classes": NUM_CLASSES, "torch": torch.__version__}, path)
    print("golden fixture written:", path, os.path.getsize(path), "bytes")
