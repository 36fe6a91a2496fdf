"""Throughput of SupCon stage-1 training on the GPU engine, all in one invocation on one GPU: TrainStep graph step of the
recipe (SupConModel resnet18, bs 200 -> 400 images of two views at 224 px, SGD lr 0.1, SupConLoss temperature 0.1) and of
resnet50 at bs 128, the fp32 oracle (oracle/supcon.py) under bf16 autocast + cuDNN with torch.optim.SGD on the same
batches, and the normalisation + loss kernels on their own (forward + backward replayed from a CUDA graph, timed
with CUDA events) at N = 400 and N = 256, D = 128.

    python tools/supcon_step.py [--steps 10] [--warmup 3] [--out FILE]

The first line names the card, its power limit and max SM clock, read in the same call."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.senet_step import _device_line, _timed  # noqa: E402

TAU = 0.1


def _model(backbone):
    from deeplearning_b200.self_supervised.SupCon.models.model import SupConModel

    torch.manual_seed(0)
    return SupConModel(backbone)


def _data(B):
    g = torch.Generator(device="cuda").manual_seed(1234)
    return torch.randn(2 * B, 3, 224, 224, device="cuda", generator=g), torch.randint(0, 10, (B,), device="cuda", generator=g)


def engine_train(backbone, B, steps, warmup):
    from deeplearning_b200.engine.trainer import TrainStep
    from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss

    model = _model(backbone).cuda().train()
    tr = TrainStep(model, lr=0.1, momentum=0.0, weight_decay=0.0, criterion=SupConLoss(temperature=TAU))
    x, y = _data(B)
    tr.step_eager(x, y)
    tr.capture(x, y)
    ms = _timed(lambda: tr.step(x, y), steps, warmup)
    del tr, model
    torch.cuda.empty_cache()
    return ms


def oracle_train(backbone, B, steps, warmup):
    from oracle.supcon import supcon_forward, supcon_loss

    s = {k: v.cuda() for k, v in _model(backbone).state_dict().items()}
    params = [v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k]
    opt = torch.optim.SGD(params, lr=0.1)
    x, y = _data(B)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            emb = supcon_forward(s, x, True).float()
        f1, f2 = torch.split(emb, [B, B], dim=0)
        supcon_loss(torch.cat([f1.unsqueeze(1), f2.unsqueeze(1)], dim=1), y, TAU, 0.07).backward()
        opt.step()

    ms = _timed(step, steps, warmup)
    del s, opt
    torch.cuda.empty_cache()
    return ms


def loss_kernels(N, D=128, reps=200):
    from deeplearning_b200 import ops

    z = torch.randn(N, D, device="cuda")
    y = torch.randint(0, 10, (N // 2,), device="cuda").repeat(2).int()
    one = torch.ones(1, device="cuda")

    def run():
        e, nrm = ops.supcon_normalize(z)
        loss, L, npos = ops.supcon_loss(e, y, TAU, 0.07)
        de = ops.supcon_loss_bwd(e, y, L, npos, one, TAU, 0.07)
        ops.supcon_normalize_bwd(de, e, nrm)

    run()   # warm-up outside the graph (first-launch attribute calls)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):   # replayed, so the time is the kernels' and not the host's launch overhead
        run()
    return _timed(graph.replay, reps, 10)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("supcon_step.py measures on a CUDA device; none is available")
    lines = [f"device: {_device_line()}"]
    for backbone, B in (("resnet18", 200), ("resnet50", 128)):
        ms = engine_train(backbone, B, a.steps, a.warmup)
        lines.append(f"SupCon stage 1 {backbone} engine (graph, SGD) bs {B} ({2 * B} images) 224px: {ms:.1f} ms/step  "
                     f"{2 * B * 1e3 / ms:.0f} img/s")
        ms_o = oracle_train(backbone, B, a.steps, a.warmup)
        lines.append(f"SupCon stage 1 {backbone} oracle bf16 autocast bs {B}: {ms_o:.1f} ms/step  {2 * B * 1e3 / ms_o:.0f} img/s")
    for N in (400, 256):
        us = loss_kernels(N) * 1e3
        lines.append(f"normalise + SupCon loss, forward + backward, N {N} D 128: {us:.1f} us")
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
