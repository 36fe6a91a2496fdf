"""Throughput of RepVGG on the GPU engine, all in one invocation on one GPU:

  * training: TrainStep graph img/s of RepVGG-A0 / B0 / B1 next to ResNet-50 on the same engine, and the fp32 oracle
    (oracle/repvgg.py) under bf16 autocast with channels_last on cuDNN;
  * inference: the converted (deploy-form) model on the engine against torch bf16 autocast on the converted oracle;
  * every RepVGG block pass (apply, backward reduce, backward apply) at every RepVGG-A0 block shape, CUDA events per call.

    python tools/repvgg_step.py [--batch 256] [--steps 30] [--warmup 5] [--iters 30] [--out FILE]

Engine training arms follow bench.py's protocol: TrainStep (SGD momentum 0.9, wd 5e-4 as in the recipe), the whole step
captured in a CUDA graph, >= 3 warm-up replays, then --steps replays between two CUDA events.  The cuDNN arm runs the same
SGD step eagerly under torch.autocast(bfloat16).  Inference arms time eager no-grad forwards.  Per-kernel lines give GB/s of
the tensors the pass reads and writes once, and that rate as a share of the H100 SXM's 3.35 TB/s."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.senet_step import HBM_TBS, _device_line, _timed  # noqa: E402


def _data(B, hw=224):
    g = torch.Generator(device="cuda").manual_seed(1234)
    return torch.randn(B, 3, hw, hw, device="cuda", generator=g), torch.randint(0, 1000, (B,), device="cuda", generator=g)


def engine_train(ctor, B, steps, warmup):
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    model = ctor().cuda().train()
    tr = TrainStep(model, lr=0.01, momentum=0.9, weight_decay=5e-4)
    x, y = _data(B)
    tr.step_eager(x, y)
    tr.capture(x, y)
    return _timed(lambda: tr.step(x, y), steps, warmup)


def oracle_train(name, B, steps, warmup):
    from oracle.repvgg import build

    torch.manual_seed(0)
    model = build(name).cuda().train().to(memory_format=torch.channels_last)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    x, y = _data(B)
    x = x.to(memory_format=torch.channels_last)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(model(x), y)
        loss.backward()
        opt.step()

    return _timed(step, steps, warmup)


def engine_infer(name, B, steps, warmup):
    from deeplearning_b200.classification.RepVGG.models import func_dict, repvgg_model_convert

    torch.manual_seed(0)
    model = repvgg_model_convert(func_dict[name]()).cuda().eval()
    x, _ = _data(B)
    with torch.no_grad():
        return _timed(lambda: model(x), steps, warmup)


def oracle_infer(name, B, steps, warmup):
    from oracle.repvgg import build, convert

    torch.manual_seed(0)
    model = convert(build(name)).cuda().eval().to(memory_format=torch.channels_last)
    x, _ = _data(B)
    x = x.to(memory_format=torch.channels_last)

    def fwd():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            model(x)

    return _timed(fwd, steps, warmup)


def pass_shapes(B):
    """(name, bytes read + written once, callable) of the three block passes at every RepVGG-A0 block shape"""
    from deeplearning_b200 import ops

    def nb(*ts):
        return float(sum(t.numel() * t.element_size() for t in ts if t is not None))

    out = []
    # (tag, H, C, identity, stem): stem 112 px x 48 (pitched [c3 | c1]), then stride-2 / stride-1 blocks of stage1..4
    for tag, H, C, ident, stem in [("stem", 112, 48, False, True), ("stage1 s2", 56, 48, False, False),
                                   ("stage1 s1", 56, 48, True, False), ("stage2 s1", 28, 96, True, False),
                                   ("stage3 s1", 14, 192, True, False), ("stage4 s2", 7, 1280, False, False)]:
        gen = torch.Generator(device="cuda").manual_seed(H + C)

        def r(*shape):
            return torch.randn(*shape, device="cuda", generator=gen).to(torch.bfloat16)

        if stem:
            c = r(B, H, H, 2 * C)
            c3, c1 = c[..., :C], c[..., C:]
        else:
            c3, c1 = r(B, H, H, C), r(B, H, H, C)
        x = r(B, H, H, C) if ident else None
        gy = r(B, H, H, C)
        cos = []
        for _ in range(3):
            co = ops.BnCoeffs(C, "cuda")
            co.mean.zero_()
            co.invstd.fill_(1.0)
            co.scale.fill_(0.5)
            co.shift.zero_()
            cos.append(co)
        m = torch.zeros(2, C, device="cuda")
        coi = cos[2] if ident else None
        y, _ = ops.repvgg_apply(c3, c1, cos[0], cos[1], x=x, co_id=coi, want_stats=True)
        name = f"{tag:9s} {H:3d}x{H:<3d} C={C:4d}{' +id' if ident else '    '}"
        out.append((f"{name} apply (+stats)", nb(c3, c1, x, y),
                    lambda a=(c3, c1, cos[0], cos[1], x, coi): ops.repvgg_apply(*a, want_stats=True)))
        out.append((f"{name} bwd_reduce", nb(gy, y, c3, c1, x), lambda a=(gy, y, c3, c1, x): ops.repvgg_bwd_reduce(*a)))
        out.append((f"{name} bwd_apply", nb(gy, y, c3, c1, x) * 2 - nb(gy, y),
                    lambda a=(gy, y, c3, c1, cos[0], m, cos[1], m, x, coi, m if ident else None): ops.repvgg_bwd_apply(*a)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the report to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("repvgg_step.py measures on a CUDA device; none is available")
    from deeplearning_b200.classification.RepVGG.models import func_dict
    from deeplearning_b200.classification.resnet.models.networks import resnet50

    lines = []

    def emit(s):
        print(s, flush=True)
        lines.append(s)

    B = args.batch
    emit(f"# {_device_line()}  batch {B}, 224 px, {args.steps} timed steps after {max(args.warmup, 3)} warm-up")
    emit("# training")
    arms = [("resnet50 (engine)", lambda: engine_train(resnet50, B, args.steps, args.warmup))]
    for name in ("RepVGG-A0", "RepVGG-B0", "RepVGG-B1"):
        arms.append((f"{name} (engine)", lambda n=name: engine_train(func_dict[n], B, args.steps, args.warmup)))
        arms.append((f"{name} oracle (torch bf16 autocast, channels_last, cuDNN)",
                     lambda n=name: oracle_train(n, B, args.steps, args.warmup)))
    for name, fn in arms:
        ms = fn()
        emit(f"{name:64s} {ms:8.2f} ms/step  {B * 1e3 / ms:8.0f} img/s")
        torch.cuda.empty_cache()
    emit("# inference, deploy form (repvgg_model_convert)")
    for name in ("RepVGG-A0", "RepVGG-B0", "RepVGG-B1"):
        for arm, fn in (("engine", engine_infer), ("oracle (torch bf16 autocast, channels_last, cuDNN)", oracle_infer)):
            ms = fn(name, B, args.steps, args.warmup)
            emit(f"{name + ' ' + arm:64s} {ms:8.2f} ms/fwd   {B * 1e3 / ms:8.0f} img/s")
            torch.cuda.empty_cache()
    emit(f"# RepVGG block passes at the RepVGG-A0 block shapes, bs {B} (CUDA events, per call; GB/s of tensors read / "
         f"written once, share of {HBM_TBS} TB/s)")
    for name, nbytes, fn in pass_shapes(B):
        fn()
        torch.cuda.synchronize()
        us = _timed(fn, args.iters, 3) * 1e3
        gbs = nbytes / us * 1e-3
        emit(f"{name:52s} {us:9.1f} us  {gbs:7.0f} GB/s  {gbs / (HBM_TBS * 1e3) * 100:5.1f}%")
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
