"""Training-step throughput of ResNeXt-50 32x4d on the GPU engine, next to ResNet-50 on the same engine and torchvision's
resnext50_32x4d under bf16 autocast with channels_last (cuDNN), all in one invocation on one GPU; then every grouped-conv
launch shape of the ResNeXt-50 step (forward + statistics, dgrad, wgrad), timed one shape at a time with CUDA events.

    python tools/resnext_step.py [--batch 256] [--steps 50] [--warmup 5] [--iters 30] [--out FILE]

Engine arms follow bench.py's protocol: TrainStep (SGD momentum 0.9, wd 5e-5), the whole step captured in a CUDA graph,
>= 3 warm-up replays, then --steps replays between two CUDA events. The cuDNN arm runs the same SGD step eagerly (forward,
loss, backward, optimizer step) under torch.autocast(bfloat16) with channels_last tensors. Per-shape lines give useful
TFLOP/s (the grouped convolution's own MACs), executed TFLOP/s (the 64-wide block-diagonal MACs the tensor cores run) and
GB/s of the operand and result tensors."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def _device_line():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return smi or torch.cuda.get_device_name()


def _timed(step, steps, warmup):
    for _ in range(max(warmup, 3)):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def engine_arm(ctor, B, steps, warmup):
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    model = ctor().cuda().train()
    tr = TrainStep(model, lr=0.01, momentum=0.9, weight_decay=5e-5)
    g = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.randn(B, 3, 224, 224, device="cuda", generator=g)
    y = torch.randint(0, 1000, (B,), device="cuda", generator=g)
    tr.step_eager(x, y)
    tr.capture(x, y)
    return _timed(lambda: tr.step(x, y), steps, warmup)


def cudnn_arm(B, steps, warmup):
    import torchvision

    torch.manual_seed(0)
    model = torchvision.models.resnext50_32x4d().cuda().train().to(memory_format=torch.channels_last)
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-5)
    g = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.randn(B, 3, 224, 224, device="cuda", generator=g).to(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (B,), device="cuda", generator=g)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(model(x), y)
        loss.backward()
        opt.step()

    return _timed(step, steps, warmup)


def grouped_shapes(B):
    """(name, useful flop, executed flop, bytes, callable) of every grouped-conv launch of a ResNeXt-50 32x4d step"""
    from deeplearning_b200 import ops

    def rnd(*shape, scale=1.0, seed=0):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        return (torch.randn(*shape, device="cuda", generator=gen) * scale).to(torch.bfloat16)

    def nb(*ts):
        return float(sum(t.numel() * t.element_size() for t in ts))

    out = []
    # (layer, input size, channels, stride): the first block of layers 2-4 carries the stride-2 3x3
    for lay, H, C, s in [(1, 56, 128, 1), (2, 56, 256, 2), (2, 28, 256, 1), (3, 28, 512, 2), (3, 14, 512, 1),
                         (4, 14, 1024, 2), (4, 7, 1024, 1)]:
        Cg, g = C // 32, 32
        Ho = (H - 1) // s + 1
        x = rnd(B, H, H, C, seed=1)
        w = rnd(C, Cg, 3, 3, scale=(9 * Cg) ** -0.5, seed=2).float()
        wp, wd = ops.pack_weight(w, mode=3), ops.pack_weight(w, mode=4)
        dy = rnd(B, Ho, Ho, C, seed=3)
        useful = 2.0 * B * Ho * Ho * C * Cg * 9
        executed = 2.0 * B * Ho * Ho * C * 64 * 9
        tag = f"L{lay} {C}ch Cg={Cg} s{s} @{H}"
        out.append((f"{tag} fwd+stats", useful, executed, nb(x, wp, dy),
                    lambda x=x, wp=wp, s=s, g=g: ops.conv2d_fwd(x, wp, 3, s, want_stats=True, groups=g)))
        if s == 1:
            co = ops.BnCoeffs(C, "cuda")
            co.scale.fill_(1.0)
            co.shift.fill_(0.0)
            out.append((f"{tag} dgrad+bnmask", useful, executed, nb(dy, wd, x, x),
                        lambda dy=dy, wd=wd, H=H, x=x, co=co, g=g: ops.conv2d_dgrad(dy, wd, (H, H), 3, 1, bn_mask=(x, co), groups=g)))
        else:
            out.append((f"{tag} dgrad", useful, executed, nb(dy, wd, x),
                        lambda dy=dy, wd=wd, H=H, s=s, g=g: ops.conv2d_dgrad(dy, wd, (H, H), 3, s, groups=g)))
        dw = torch.empty(C, Cg, 3, 3, device="cuda")
        out.append((f"{tag} wgrad", useful, executed, nb(dy, x, dw),
                    lambda dy=dy, x=x, s=s, g=g, dw=dw: ops.conv2d_wgrad(dy, x, 3, s, out=dw, groups=g)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the report to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resnext_step.py measures on a CUDA device; none is available")
    from deeplearning_b200.classification.resnet.models.networks import resnet50, resnext50_32x4d

    lines = []

    def emit(s):
        print(s, flush=True)
        lines.append(s)

    emit(f"# {_device_line()}  batch {args.batch}, {args.steps} timed steps after {max(args.warmup, 3)} warm-up")
    B = args.batch
    ms = {}
    for name, fn in [("resnet50 (engine)", lambda: engine_arm(resnet50, B, args.steps, args.warmup)),
                     ("resnext50_32x4d (engine)", lambda: engine_arm(resnext50_32x4d, B, args.steps, args.warmup)),
                     ("resnext50_32x4d (torch bf16 autocast, channels_last, cuDNN, eager)",
                      lambda: cudnn_arm(B, args.steps, args.warmup))]:
        ms[name] = fn()
        emit(f"{name:70s} {ms[name]:8.2f} ms/step  {B * 1e3 / ms[name]:8.0f} img/s")
        torch.cuda.empty_cache()
    r50, rx = ms["resnet50 (engine)"], ms["resnext50_32x4d (engine)"]
    emit(f"resnext50 / resnet50 img/s on the engine: {r50 / rx:.3f}")
    emit("# grouped-conv launches of the ResNeXt-50 step (CUDA events, per launch)")
    for name, useful, executed, nbytes, fn in grouped_shapes(B):
        fn()
        torch.cuda.synchronize()
        us = _timed(fn, args.iters, 3) * 1e3
        emit(f"{name:40s} {us:9.1f} us  useful {useful / us * 1e-6:6.1f} TFLOP/s  executed {executed / us * 1e-6:6.1f} TFLOP/s"
             f"  {nbytes / us * 1e-3:6.0f} GB/s")
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
