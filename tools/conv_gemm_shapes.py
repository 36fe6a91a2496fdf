"""Times the conv_gemm_kernel launches of the ResNet-50 (batch 256) and ViT-B/16 (batch 256) training steps one shape at a
time with CUDA events, and prints each one's TFLOP/s and GB/s next to the H100 SXM data-sheet peaks (989 TFLOP/s dense
bf16, 3.35 TB/s HBM3).

    python tools/conv_gemm_shapes.py [--iters 50] [--only SUBSTRING]

With a library built with -DCONV_PROFILE added to the Makefile's CXXFLAGS (make ... OUT=/elsewhere/libb200cls.so), pass
--profile: every shape then runs twice and CTA 0 of each launch prints its per-tile phase cycles instead.
Select another build of the library with B200_LIB=/path/to/libb200cls.so."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from deeplearning_b200 import ops  # noqa: E402

PEAK_TFLOPS = 989.0
PEAK_GBS = 3350.0


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _coeffs(C):
    co = ops.BnCoeffs(C, "cuda")
    co.scale.copy_(torch.rand(C, device="cuda") + 0.5)
    co.shift.copy_(torch.randn(C, device="cuda") * 0.1)
    return co


def cases(B=256, T=197):
    """(name, kind, flop, bytes, callable) of every launch shape."""
    out = []

    def nb(*ts):
        return sum(t.numel() * t.element_size() for t in ts)

    for lay, (H, Cin, C) in enumerate([(56, 256, 64), (28, 512, 128), (14, 1024, 256), (7, 2048, 512)], 1):
        x = _rand(B, H, H, Cin, seed=1)
        wp = ops.pack_weight(_rand(C, Cin, 1, 1, scale=Cin ** -0.5, seed=2).float())
        y = torch.empty(B, H, H, C, dtype=torch.bfloat16, device="cuda")
        out.append((f"L{lay} conv1 1x1 fwd +stats  {Cin}->{C} @{H}", 2.0 * B * H * H * Cin * C, nb(x, wp, y),
                    lambda x=x, wp=wp: ops.conv2d_fwd(x, wp, 1, 1, want_stats=True)))
    for lay, (H, C) in enumerate([(56, 64), (28, 128), (14, 256), (7, 512)], 1):
        x = _rand(B, H, H, C, seed=3)
        w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=4)
        wp, wd = ops.pack_weight(w.float()), ops.pack_weight(w.float(), mode=1)
        flop = 2.0 * B * H * H * C * C * 9
        if lay > 1:   # (layer 1's 3x3 forward runs conv_tap64)
            out.append((f"L{lay} conv2 3x3 fwd +stats  {C}->{C} @{H}", flop, 3 * nb(x),
                        lambda x=x, wp=wp: ops.conv2d_fwd(x, wp, 3, 1, want_stats=True)))
        xr, co = _rand(B, H, H, C, seed=5), _coeffs(C)
        out.append((f"L{lay} conv2 3x3 dgrad +bnmask {C}->{C} @{H}", flop, 4 * nb(x),
                    lambda x=x, wd=wd, xr=xr, co=co, H=H: ops.conv2d_dgrad(x, wd, (H, H), 3, 1, bn_mask=(xr, co))))
    for lay, (H, C) in enumerate([(56, 64), (28, 128), (14, 256)], 1):
        dz, y2 = _rand(B, H, H, 4 * C, seed=6), _rand(B, H, H, C, seed=7)
        wcat = _rand(C, 5 * C, scale=(5 * C) ** -0.5, seed=8)
        bias = torch.randn(C, device="cuda")
        xr, co = _rand(B, H, H, C, seed=9), _coeffs(C)
        out.append((f"L{lay} dual dgrad +bnmask  {5 * C}->{C} @{H}", 2.0 * B * H * H * 5 * C * C, nb(dz, y2) + 3 * nb(xr),
                    lambda dz=dz, y2=y2, wcat=wcat, bias=bias, xr=xr, co=co: ops.gemm_dual(dz, y2, wcat, bias, bn_mask=(xr, co))))
    M, D = B * T, 768
    a, h = _rand(M, D, seed=10), _rand(M, 4 * D, seed=11)
    res = torch.randn(M, D, device="cuda")
    for name, inp, N, kw in [("qkv +bias", a, 3 * D, {}), ("fc1 +bias gelu aux", a, 4 * D, {"act": 2, "aux_out": True}),
                             ("fc2 +bias +res f32", h, D, {"residual": res, "out_f32": True})]:
        K = inp.shape[-1]
        wp = ops.pack_weight(_rand(N, K, scale=K ** -0.5, seed=12).float())
        bias = torch.randn(N, device="cuda")
        ob = M * N * (4 if kw.get("out_f32") else 2) * (2 if kw.get("aux_out") or "residual" in kw else 1)
        out.append((f"ViT {name}  {K}->{N} x{M}", 2.0 * M * K * N, nb(inp, wp) + ob,
                    lambda inp=inp, wp=wp, bias=bias, kw=kw: ops.gemm(inp, wp, bias=bias, **kw)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--only", default="")
    ap.add_argument("--profile", action="store_true", help="run each shape once (a -DCONV_PROFILE build prints phase cycles)")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"# {smi}  lib={os.environ.get('B200_LIB', 'default')}")
    for name, flop, nbytes, fn in cases():
        if args.only not in name:
            continue
        fn()
        torch.cuda.synchronize()
        if args.profile:
            print(f"== {name}", flush=True)
            fn()
            torch.cuda.synchronize()
            continue
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / args.iters
        tf, gbs = flop / us * 1e-6, nbytes / us * 1e-3
        print(f"{name:44s} {us:9.1f} us  {tf:6.1f} TFLOP/s ({tf / PEAK_TFLOPS:5.1%})  {gbs:6.0f} GB/s ({gbs / PEAK_GBS:5.1%})",
              flush=True)


if __name__ == "__main__":
    main()
