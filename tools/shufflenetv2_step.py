"""Throughput of ShuffleNet v2 on the GPU engine, all in one invocation on one GPU:

  * training: TrainStep graph img/s of shufflenet_v2_x1_0 and _x2_0 (the recipe's SGD: momentum 0.9, weight decay 5e-4) and
    the fp32 oracle (oracle/shufflenetv2.py) under bf16 autocast with channels_last on cuDNN, same optimizer;
  * per-pass table of one x1_0 training step (ops.Profiler, CUDA events per C-ABI call): time per pass kind, and the HBM
    bandwidth achieved on the bytes each pass reads and writes once (computed from shapes), with its share of 3.35 TB/s.

    python tools/shufflenetv2_step.py [--batch 256] [--steps 10] [--warmup 3] [--out FILE]

The first line names the card, its power limit and max SM clock, read in the same call."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.senet_step import HBM_TBS, _device_line, _timed  # noqa: E402

NAMES = ["x1_0", "x2_0"]


def _data(B, hw=224):
    g = torch.Generator(device="cuda").manual_seed(1234)
    return torch.randn(B, 3, hw, hw, device="cuda", generator=g), torch.randint(0, 1000, (B,), device="cuda", generator=g)


def _model(name):
    from deeplearning_b200.classification.ShuffleNet.models import shufflenetv2

    torch.manual_seed(0)
    return getattr(shufflenetv2, f"shufflenet_v2_{name}")()


def engine_train(name, B, steps, warmup):
    from deeplearning_b200.engine.trainer import TrainStep

    model = _model(name).cuda().train()
    tr = TrainStep(model, lr=0.05, momentum=0.9, weight_decay=5e-4)
    x, y = _data(B)
    tr.step_eager(x, y)
    tr.capture(x, y)
    ms = _timed(lambda: tr.step(x, y), steps, warmup)
    del tr, model
    torch.cuda.empty_cache()
    return ms


def oracle_train(name, B, steps, warmup):
    from oracle.shufflenetv2 import shufflenetv2_forward

    s = {k: v.cuda() for k, v in _model(name).state_dict().items()}
    params = [v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k]
    opt = torch.optim.SGD(params, lr=0.05, momentum=0.9, weight_decay=5e-4)
    x, y = _data(B)
    x = x.to(memory_format=torch.channels_last)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(shufflenetv2_forward(s, x, True), y)
        loss.backward()
        opt.step()

    ms = _timed(step, steps, warmup)
    del s, params, opt
    torch.cuda.empty_cache()
    return ms


def pass_lines(name, B):
    """one eager engine step under ops.Profiler: per pass kind, calls, total ms, GB/s on its bytes and share of HBM"""
    from deeplearning_b200 import ops
    from deeplearning_b200.engine import shufflenetv2 as engine

    model = _model(name).cuda().train()
    x, y = _data(B)
    for _ in range(2):
        logits, tape = engine.forward(model, x, True, True)
        engine.backward(model, tape, ops.softmax_xent(logits, y, ld_d=1000)[1])
    torch.cuda.synchronize()
    with ops.Profiler(run_ahead_ms=50.0) as prof:
        logits, tape = engine.forward(model, x, True, True)
        engine.backward(model, tape, ops.softmax_xent(logits, y, ld_d=1000)[1])
    agg = prof.summary()
    total = sum(a["ms"] for a in agg.values())
    out = [f"per-pass {name} bs {B} 224px (one eager step, CUDA events per call; sum {total:.1f} ms):"]
    for nm, a in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
        gbs = a["bytes"] / a["ms"] / 1e6 if a["ms"] > 0 else 0.0
        tf = a["flops"] / a["ms"] / 1e9 if a["ms"] > 0 else 0.0
        out.append(f"  {nm:24s} calls {a['calls']:4d}  {a['ms']:8.2f} ms  {100 * a['ms'] / total:5.1f}%  "
                   f"{gbs:6.0f} GB/s ({100 * gbs / (HBM_TBS * 1e3):4.1f}% of HBM)  {tf:6.1f} TFLOP/s")
    del model, tape
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shufflenetv2_step.py measures on a CUDA device; none is available")
    B = a.batch
    lines = [f"device: {_device_line()}"]
    for name in NAMES:
        e = engine_train(name, B, a.steps, a.warmup)
        o = oracle_train(name, B, a.steps, a.warmup)
        lines.append(f"train shufflenet_v2_{name} engine (graph, SGD) bs {B} 224px: {e:.1f} ms/step  {B * 1e3 / e:.0f} img/s")
        lines.append(f"train shufflenet_v2_{name} oracle bf16 autocast channels_last cuDNN bs {B}: {o:.1f} ms/step  "
                     f"{B * 1e3 / o:.0f} img/s  (engine {o / e:.2f}x)")
    lines += pass_lines("x1_0", B)
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
