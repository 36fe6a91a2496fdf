"""Throughput of VGG on the GPU engine, all in one invocation on one GPU:

  * training: TrainStep graph img/s of vgg16 and vgg16_bn (the recipe's Adam, lr 1e-3, weight decay 1e-3) and the fp32 oracle
    (oracle/vgg.py) under bf16 autocast with channels_last on cuDNN, same optimizer;
  * every distinct vgg16 convolution shape: forward GEMM time from CUDA events, achieved TFLOP/s and the share of the H100
    SXM's 989 TFLOP/s dense bf16 peak (the bound of these layers);
  * every 2x2 pool pass (plain and BatchNorm forward, both backwards) at vgg16's pooled shapes, and the adaptive pool: GB/s of
    the tensors each reads and writes once, and that rate as a share of 3.35 TB/s.

    python tools/vgg_step.py [--batch 256] [--steps 10] [--warmup 3] [--iters 20] [--out FILE]

The first line names the card, its power limit and max SM clock, read in the same call."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.senet_step import HBM_TBS, _device_line, _timed  # noqa: E402

BF16_TFLOPS = 989.0
VGG16 = [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M']


def _data(B, hw=224):
    g = torch.Generator(device="cuda").manual_seed(1234)
    return torch.randn(B, 3, hw, hw, device="cuda", generator=g), torch.randint(0, 1000, (B,), device="cuda", generator=g)


def engine_train(name, B, steps, warmup):
    from deeplearning_b200.classification.vggNet.models import network
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    model = getattr(network, name)().cuda().train()
    tr = TrainStep(model, lr=1e-3, optimizer="adam", weight_decay=1e-3)
    x, y = _data(B)
    tr.step_eager(x, y)
    tr.capture(x, y)
    ms = _timed(lambda: tr.step(x, y), steps, warmup)
    del tr, model
    torch.cuda.empty_cache()
    return ms


def oracle_train(name, B, steps, warmup):
    from deeplearning_b200.classification.vggNet.models import network
    from oracle.vgg import arch, vgg_forward

    torch.manual_seed(0)
    s = {k: v.cuda() for k, v in getattr(network, name)().state_dict().items()}
    params = [v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k]
    opt = torch.optim.Adam(params, lr=1e-3, weight_decay=1e-3)
    cfg, bn = arch(name)
    x, y = _data(B)
    x = x.to(memory_format=torch.channels_last)
    p = torch.full((B, 4096), 2.0, device="cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        masks = [F.dropout(torch.ones_like(p), 0.5, True) for _ in range(2)]
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(vgg_forward(s, x, cfg, bn, True, masks), y)
        loss.backward()
        opt.step()

    ms = _timed(step, steps, warmup)
    del s, params, opt
    torch.cuda.empty_cache()
    return ms


def _events(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def conv_lines(B, iters):
    from deeplearning_b200 import ops

    out, hw, cin, seen = [], 224, 3, set()
    for v in VGG16:
        if v == 'M':
            hw //= 2
            continue
        key = (hw, cin, v)
        if key not in seen:
            seen.add(key)
            if cin == 3:
                x = torch.randn(B, 3, hw, hw, device="cuda")
                a, _, _ = ops.im2col_nchw(x, 3, 3, 1, 1, ldk=32)
                h, k = a.view(B, hw, hw, 32), 1
                w = ops.pack_weight(torch.randn(v, 3, 3, 3, device="cuda"), 0, 32)
                flops = 2.0 * B * hw * hw * v * 27
            else:
                h, k = torch.randn(B, hw, hw, cin, device="cuda").to(torch.bfloat16), 3
                w = ops.pack_weight(torch.randn(v, cin, 3, 3, device="cuda") * 0.05)
                flops = 2.0 * B * hw * hw * v * cin * 9
            b = torch.zeros(v, device="cuda")
            ms = _events(lambda: ops.conv2d_fwd(h, w, k, 1, bias=b, act=1), iters)
            tf = flops / ms / 1e9
            out.append(f"conv fwd {hw}x{hw} {cin}->{v}: {ms:.3f} ms  {tf:.0f} TFLOP/s  {100 * tf / BF16_TFLOPS:.1f}% of peak")
            del h, w
        cin = v
    return out


def pool_lines(B, iters):
    from deeplearning_b200 import ops

    out = []
    for hw, C in ((224, 64), (112, 128), (56, 256), (28, 512), (14, 512)):
        c = torch.randn(B, hw, hw, C, device="cuda").to(torch.bfloat16)
        co = ops.BnCoeffs(C, "cuda")
        co.scale.fill_(1.0), co.shift.zero_(), co.mean.zero_(), co.invstd.fill_(1.0)
        y, idx = ops.vgg_pool_fwd(c, co)
        g = torch.randn_like(y)
        nb_in, nb_out = c.numel() * 2, y.numel() * 3
        arms = [("fwd plain", lambda: ops.vgg_pool_fwd(c), nb_in + nb_out),
                ("fwd bn", lambda: ops.vgg_pool_fwd(c, co), nb_in + nb_out),
                ("bwd plain", lambda: ops.vgg_pool_bwd(g, idx, (hw, hw), y=y), nb_in + y.numel() * 5),
                ("bwd bn", lambda: ops.vgg_pool_bwd(g, idx, (hw, hw), c=c, co=co), 2 * nb_in + y.numel() * 3)]
        for nm, fn, nb in arms:
            ms = _events(fn, iters)
            gbs = nb / ms / 1e6
            out.append(f"pool {nm} {hw}x{hw}x{C}: {ms:.3f} ms  {gbs:.0f} GB/s  {100 * gbs / (HBM_TBS * 1e3):.1f}% of HBM")
        del c, y, idx, g
    x = torch.randn(B, 7, 7, 512, device="cuda").to(torch.bfloat16)
    ms = _events(lambda: ops.vgg_avgpool7_fwd(x), iters)
    gbs = 2 * x.numel() * 2 / ms / 1e6
    out.append(f"avgpool7 fwd 7x7x512: {ms:.3f} ms  {gbs:.0f} GB/s  {100 * gbs / (HBM_TBS * 1e3):.1f}% of HBM")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vgg_step.py measures on a CUDA device; none is available")
    B = a.batch
    lines = [f"device: {_device_line()}"]
    for name in ("vgg16", "vgg16_bn"):
        ms = engine_train(name, B, a.steps, a.warmup)
        lines.append(f"train {name} engine (graph, Adam) bs {B} 224px: {ms:.1f} ms/step  {B * 1e3 / ms:.0f} img/s")
        ms = oracle_train(name, B, a.steps, a.warmup)
        lines.append(f"train {name} oracle bf16 autocast channels_last cuDNN bs {B}: {ms:.1f} ms/step  {B * 1e3 / ms:.0f} img/s")
    lines += conv_lines(B, a.iters)
    lines += pool_lines(B, a.iters)
    text = "\n".join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
