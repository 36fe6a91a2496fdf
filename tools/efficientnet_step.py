"""Throughput of EfficientNet on the GPU engine, all in one invocation on one GPU:

  * training: TrainStep graph img/s of EfficientNet-B0 at 224 px and B1 at 240 px next to ResNet-50 on the same engine,
    and the fp32 oracle (oracle/efficientnet.py) under bf16 autocast with channels_last on cuDNN;
  * every new MBConv pass (csrc/mbconv.cuh) at every EfficientNet-B0 block shape, CUDA events per call.

    python tools/efficientnet_step.py [--batch 256] [--steps 30] [--warmup 5] [--iters 30] [--out FILE]

Engine training arms follow bench.py's protocol: TrainStep (SGD momentum 0.9, wd 5e-4), default drop-connect and dropout,
the whole step captured in a CUDA graph, >= 3 warm-up replays, then --steps replays between two CUDA events.  The cuDNN arm
runs the same SGD step eagerly under torch.autocast(bfloat16) without drop-connect or dropout masks.  Per-pass lines give
GB/s of the tensors the pass reads and writes once, and that rate as a share of the H100 SXM's 3.35 TB/s."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.senet_step import HBM_TBS, _device_line, _timed  # noqa: E402


def _data(B, hw):
    g = torch.Generator(device="cuda").manual_seed(1234)
    return torch.randn(B, 3, hw, hw, device="cuda", generator=g), torch.randint(0, 1000, (B,), device="cuda", generator=g)


def engine_train(ctor, B, hw, steps, warmup):
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    model = ctor().cuda().train()
    tr = TrainStep(model, lr=0.01, momentum=0.9, weight_decay=5e-4)
    x, y = _data(B, hw)
    tr.step_eager(x, y)
    tr.capture(x, y)
    return _timed(lambda: tr.step(x, y), steps, warmup)


def oracle_train(name, B, hw, steps, warmup):
    from deeplearning_b200.classification.efficientNet.models import network
    from oracle.efficientnet import efficientnet_forward, plan

    torch.manual_seed(0)
    s = {k: v.cuda() for k, v in getattr(network, f"efficientnet_{name}")().state_dict().items()}
    params = [v.requires_grad_(True) for k, v in s.items() if v.is_floating_point() and "running" not in k]
    opt = torch.optim.SGD(params, lr=0.01, momentum=0.9, weight_decay=5e-4)
    blocks = plan(name)
    x, y = _data(B, hw)
    x = x.contiguous(memory_format=torch.channels_last)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(efficientnet_forward(s, x, blocks, train=True), y)
        loss.backward()
        opt.step()

    return _timed(step, steps, warmup)


# (tag, H in, C expanded, k, stride, expand) of every distinct EfficientNet-B0 block at 224 px
B0_BLOCKS = [("1a", 112, 32, 3, 1, False), ("2a", 112, 96, 3, 2, True), ("2b", 56, 144, 3, 1, True),
             ("3a", 56, 144, 5, 2, True), ("3b", 28, 240, 5, 1, True), ("4a", 28, 240, 3, 2, True),
             ("4b", 14, 480, 3, 1, True), ("5a", 14, 480, 5, 1, True), ("5b", 14, 672, 5, 1, True),
             ("6a", 14, 672, 5, 2, True), ("6b", 7, 1152, 5, 1, True), ("7a", 7, 1152, 3, 1, True)]


def pass_shapes(B):
    """(name, bytes read + written once, callable) of every MBConv pass at every EfficientNet-B0 block shape"""
    from deeplearning_b200 import ops

    def nb(*ts):
        return float(sum(t.numel() * t.element_size() for t in ts if t is not None))

    out = []
    for tag, H, C, k, s, _ in B0_BLOCKS:
        gen = torch.Generator(device="cuda").manual_seed(H + C)

        def r(*shape):
            return torch.randn(*shape, device="cuda", generator=gen).to(torch.bfloat16)

        Ho = (H - 1) // s + 1
        x = r(B, H, H, C)
        w = torch.randn(C, 1, k, k, device="cuda") * 0.2
        co = ops.BnCoeffs(C, "cuda")
        co.mean.zero_()
        co.invstd.fill_(1.0)
        co.scale.fill_(0.5)
        co.shift.zero_()
        d, _ = ops.dw_fwd(x, w, k, s, co=co, want_stats=True)
        da = r(B, Ho, Ho, C)
        pool, _ = ops.silu_bn_squeeze(d, co)
        Cr = max(8, C // 24)
        w1, b1 = torch.randn(Cr, C, device="cuda") * 0.05, torch.zeros(Cr, device="cuda")
        w2, b2 = torch.randn(C, Cr, device="cuda") * 0.05, torch.zeros(C, device="cuda")
        hpre, gate = ops.excite_fwd(pool, w1, b1, w2, b2)
        sg = ops.gate_reduce(da, d, co)
        dpool = torch.randn(B, C, device="cuda")
        dz, part = ops.silu_bn_bwd_reduce(d, co, dpool, da=da, gate=gate)
        rs = torch.ones(B, device="cuda")
        name = f"{tag} {H:3d}->{Ho:<3d} C={C:4d} k{k}s{s}"
        out += [
            (f"{name} dw_fwd (+BN-SiLU on load, stats)", nb(x, d), lambda a=(x, w, k, s, co): ops.dw_fwd(*a[:4], co=a[4], want_stats=True)),
            (f"{name} dw_dgrad (x silu', sums)", nb(da, x, x), lambda a=(da, w, x, k, s, co): ops.dw_dgrad(*a[:5], co=a[5])),
            (f"{name} dw_wgrad", nb(da, x), lambda a=(da, x, k, s, co): ops.dw_wgrad(*a[:4], co=a[4])),
            (f"{name} silu_bn_squeeze", nb(d), lambda a=(d, co): ops.silu_bn_squeeze(*a)),
            (f"{name} excite_fwd", nb(pool, w1, w2, gate), lambda a=(pool, w1, b1, w2, b2): ops.excite_fwd(*a)),
            (f"{name} gate_apply", 2 * nb(d), lambda a=(d, co, gate): ops.gate_apply(*a)),
            (f"{name} gate_reduce", nb(da, d), lambda a=(da, d, co): ops.gate_reduce(*a)),
            (f"{name} excite_bwd", nb(pool, w1, w2, gate) * 2, lambda a=(sg, pool, hpre, gate, w1, w2): ops.excite_bwd(*a)),
            (f"{name} silu_bn_bwd_reduce", 3 * nb(d), lambda a=(d, co, dpool, da, gate): ops.silu_bn_bwd_reduce(*a[:3], da=a[3], gate=a[4])),
            (f"{name} tail_apply (+drop-connect, residual)", 3 * nb(d), lambda a=(d, co, rs, da): ops.tail_apply(*a[:3], residual=a[3])),
            (f"{name} tail_bwd_reduce (+drop-connect)", 3 * nb(d), lambda a=(da, d, rs): ops.tail_bwd_reduce(*a)),
            (f"{name} bn_bwd_apply (+finalize)", 3 * nb(d), lambda a=(dz, part, d, co): ops.bn_backward_from_sums(*a)),
        ]
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
        raise SystemExit("efficientnet_step.py measures on a CUDA device; none is available")
    from deeplearning_b200.classification.efficientNet.models.network import efficientnet_b0, efficientnet_b1
    from deeplearning_b200.classification.resnet.models.networks import resnet50

    lines = []

    def emit(s):
        print(s, flush=True)
        lines.append(s)

    B = args.batch
    emit(f"# {_device_line()}  batch {B}, {args.steps} timed steps after {max(args.warmup, 3)} warm-up")
    emit("# training")
    arms = [("resnet50 224 px (engine)", lambda: engine_train(resnet50, B, 224, args.steps, args.warmup))]
    for name, ctor, hw in (("b0", efficientnet_b0, 224), ("b1", efficientnet_b1, 240)):
        arms.append((f"efficientnet_{name} {hw} px (engine)", lambda c=ctor, h=hw: engine_train(c, B, h, args.steps, args.warmup)))
        arms.append((f"efficientnet_{name} {hw} px oracle (torch bf16 autocast, channels_last, cuDNN)",
                     lambda n=name, h=hw: oracle_train(n, B, h, args.steps, args.warmup)))
    for name, fn in arms:
        ms = fn()
        emit(f"{name:72s} {ms:8.2f} ms/step  {B * 1e3 / ms:8.0f} img/s")
        torch.cuda.empty_cache()
    emit(f"# MBConv passes at the EfficientNet-B0 block shapes, bs {B} (CUDA events, per call; GB/s of tensors read / "
         f"written once, share of {HBM_TBS} TB/s)")
    for name, nbytes, fn in pass_shapes(B):
        fn()
        torch.cuda.synchronize()
        us = _timed(fn, args.iters, 3) * 1e3
        gbs = nbytes / us * 1e-3
        emit(f"{name:62s} {us:9.1f} us  {gbs:7.0f} GB/s  {gbs / (HBM_TBS * 1e3) * 100:5.1f}%")
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
