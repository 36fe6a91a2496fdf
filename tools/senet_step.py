"""Training-step throughput of SE-ResNet-50 on the GPU engine, next to ResNet-50 on the same engine and the fp32 SE-ResNet-50
yardstick (oracle/senet.py) under bf16 autocast with channels_last (cuDNN), all in one invocation on one GPU; then every
squeeze-and-excitation kernel at every SE-ResNet-50 tail shape, timed one shape at a time with CUDA events.

    python tools/senet_step.py [--batch 256] [--steps 50] [--warmup 5] [--iters 30] [--out FILE]

Engine arms follow bench.py's protocol: TrainStep (SGD momentum 0.9, wd 5e-5), the whole step captured in a CUDA graph,
>= 3 warm-up replays, then --steps replays between two CUDA events.  The cuDNN arm runs the same SGD step eagerly (forward,
loss, backward, optimizer step) under torch.autocast(bfloat16) with channels_last tensors.  Per-kernel lines give GB/s of the
tensors the kernel reads and writes once, and that rate as a share of the H100 SXM's 3.35 TB/s."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

HBM_TBS = 3.35


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
    from oracle.senet import se_resnet_yardstick

    torch.manual_seed(0)
    model = se_resnet_yardstick(None, (3, 4, 6, 3)).cuda().train().to(memory_format=torch.channels_last)
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


def se_shapes(B):
    """(name, bytes read + written once, callable) of every SE kernel entry at the four SE-ResNet-50 tail shapes"""
    from deeplearning_b200 import ops

    def nb(*ts):
        return float(sum(t.numel() * t.element_size() for t in ts))

    out = []
    for lay, HW, C in [(1, 3136, 256), (2, 784, 512), (3, 196, 1024), (4, 49, 2048)]:
        Cr = C // 16
        H = int(HW ** 0.5)
        gen = torch.Generator(device="cuda").manual_seed(lay)
        c = torch.randn(B, H, H, C, device="cuda", generator=gen).to(torch.bfloat16)
        ident = torch.randn(B, H, H, C, device="cuda", generator=gen).to(torch.bfloat16)
        gy = torch.randn(B, H, H, C, device="cuda", generator=gen).to(torch.bfloat16)
        w1 = torch.randn(Cr, C, device="cuda", generator=gen) * C ** -0.5
        w2 = torch.randn(C, Cr, device="cuda", generator=gen) * Cr ** -0.5
        co = ops.BnCoeffs(C, "cuda")
        co.mean.zero_()
        co.invstd.fill_(1.0)
        co.scale.fill_(1.0)
        co.shift.zero_()
        csum, pool = ops.se_squeeze(c, co)
        h, gate = ops.se_excite(pool, w1, w2)
        y = ops.se_apply(c, co, gate, ident)
        vec = B * C * 4.0
        tag = f"L{lay} HW={HW} C={C} Cr={Cr}"
        out.append((f"{tag} squeeze", nb(c) + 2 * vec, lambda c=c, co=co: ops.se_squeeze(c, co)))
        out.append((f"{tag} excite", nb(pool, w1, w2, h, gate), lambda p=pool, w1=w1, w2=w2: ops.se_excite(p, w1, w2)))
        out.append((f"{tag} apply", nb(c, ident, y), lambda c=c, co=co, g=gate, i=ident: ops.se_apply(c, co, g, i)))
        # the backward entry is three launches: reduce (g, y, c -> dz), coefficients, apply (dz, c -> dc)
        out.append((f"{tag} backward (reduce+coeffs+apply)", 7 * nb(c),
                    lambda a=(gy, y, c, co, csum, pool, h, gate, w1, w2): ops.se_backward(*a)))
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
        raise SystemExit("senet_step.py measures on a CUDA device; none is available")
    from deeplearning_b200 import ops
    from deeplearning_b200.classification.resnet.models.networks import resnet50
    from deeplearning_b200.classification.seNet.models.networks import se_resnet50

    lines = []

    def emit(s):
        print(s, flush=True)
        lines.append(s)

    emit(f"# {_device_line()}  batch {args.batch}, {args.steps} timed steps after {max(args.warmup, 3)} warm-up")
    B = args.batch
    ms = {}
    for name, fn in [("resnet50 (engine)", lambda: engine_arm(resnet50, B, args.steps, args.warmup)),
                     ("se_resnet50 (engine)", lambda: engine_arm(se_resnet50, B, args.steps, args.warmup)),
                     ("se_resnet50 yardstick (torch bf16 autocast, channels_last, cuDNN, eager)",
                      lambda: cudnn_arm(B, args.steps, args.warmup))]:
        ms[name] = fn()
        emit(f"{name:74s} {ms[name]:8.2f} ms/step  {B * 1e3 / ms[name]:8.0f} img/s")
        torch.cuda.empty_cache()
    emit(f"se_resnet50 / resnet50 img/s on the engine: {ms['resnet50 (engine)'] / ms['se_resnet50 (engine)']:.3f}")
    emit(f"# SE kernels at the SE-ResNet-50 tail shapes, bs {B} (CUDA events, per call; GB/s of tensors read / written once, "
         f"share of {HBM_TBS} TB/s)")
    for name, nbytes, fn in se_shapes(B):
        fn()
        torch.cuda.synchronize()
        us = _timed(fn, args.iters, 3) * 1e3
        gbs = nbytes / us * 1e-3
        emit(f"{name:52s} {us:9.1f} us  {gbs:7.0f} GB/s  {gbs / (HBM_TBS * 1e3) * 100:5.1f}%")
    # per-kernel split of the backward entry (profiler spans: every launch between CUDA events)
    emit("# SE backward entry split by launch (ops.Profiler spans, per call)")
    for name, _, fn in se_shapes(B):
        if "backward" not in name:
            continue
        with ops.Profiler(run_ahead_ms=2.0) as prof:
            for _ in range(args.iters):
                fn()
        agg = prof.summary()
        emit(f"{name.split(' backward')[0]:30s} " + "  ".join(f"{k} {v['ms'] * 1e3 / v['calls']:.1f} us"
                                                             for k, v in agg.items()))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
