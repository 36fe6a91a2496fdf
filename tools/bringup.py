"""Bring-up diagnostics for the wgmma kernels (run on an H100): python tools/bringup.py [fwd|wgrad|perf]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from deeplearning_b200 import ops

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*s, device="cuda", generator=g) * scale).to(torch.bfloat16)


def report(name, got, ref):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    rel = float(err.max()) / (float(ref.abs().max()) + 1e-9)
    print(f"[{name}] max_abs_err={float(err.max()):.5g} ref_max={float(ref.abs().max()):.5g} rel={rel:.3g} "
          f"nan={int(torch.isnan(got).sum())}", flush=True)
    return rel < 2e-2


def fwd():
    ok = True
    for (M, K, N) in [(128, 64, 64), (256, 128, 64), (256, 64, 128), (384, 256, 256), (1000, 200, 136), (4096, 512, 1000)]:
        x = rnd(M, 1, 1, K, seed=1)
        w = rnd(N, K, seed=2, scale=K ** -0.5)
        y, st = ops.conv2d_fwd(x, ops.pack_weight(w.float()), want_stats=True)
        torch.cuda.synchronize()
        ref = x.float().reshape(M, K) @ w.float().t()
        good = report(f"gemm M{M} K{K} N{N}", y.reshape(M, N), ref)
        if not good:
            d = (y.reshape(M, N).float() - ref)
            bad = d.abs() > 0.05
            rows = bad.any(1).nonzero().flatten()[:16].tolist()
            cols = bad.any(0).nonzero().flatten()[:16].tolist()
            print("   bad rows", rows, "bad cols", cols, "frac", float(bad.float().mean()))
            print("   got[0,:8]", y.reshape(M, N)[0, :8].float().tolist())
            print("   ref[0,:8]", ref[0, :8].tolist())
        ok &= good
    # 3x3 conv
    for (B, H, W, Cin, Cout, k, s) in [(2, 8, 8, 64, 64, 3, 1), (2, 56, 56, 64, 64, 3, 1), (2, 28, 28, 128, 128, 3, 2), (2, 28, 28, 64, 128, 1, 2)]:
        x = rnd(B, H, W, Cin, seed=3)
        w = rnd(Cout, Cin, k, k, seed=4, scale=(Cin * k * k) ** -0.5)
        y, _ = ops.conv2d_fwd(x, ops.pack_weight(w.float()), k, s)
        torch.cuda.synchronize()
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), stride=s, padding=k // 2).permute(0, 2, 3, 1)
        ok &= report(f"conv B{B} {H}x{W} {Cin}->{Cout} k{k}s{s}", y, ref)
    print("FWD", "OK" if ok else "FAILED", flush=True)
    return ok


def wgrad_case(B, H, W, Cin, Cout, k, s):
    x = rnd(B, H, W, Cin, seed=7)
    Ho, Wo = ops.out_hw(H, k, s), ops.out_hw(W, k, s)
    dy = rnd(B, Ho, Wo, Cout, seed=8)
    w = torch.zeros(Cout, Cin, k, k, device="cuda", requires_grad=True)
    yr = F.conv2d(x.float().permute(0, 3, 1, 2), w, stride=s, padding=k // 2)
    (gw,) = torch.autograd.grad(yr, w, dy.float().permute(0, 3, 1, 2))
    dw = ops.conv2d_wgrad(dy, x, k, s)
    torch.cuda.synchronize()
    return report(f"wgrad B{B} {H}x{W} {Cin}->{Cout} k{k}s{s}", dw, gw)


def wgrad():
    cases = [(1, 8, 8, 64, 64, 1, 1), (2, 8, 8, 64, 128, 1, 1), (2, 16, 16, 128, 256, 1, 1), (2, 8, 8, 64, 64, 3, 1), (2, 28, 28, 128, 128, 3, 2)]
    ok = all([wgrad_case(*c) for c in cases])
    print("WGRAD", "OK" if ok else "FAILED", flush=True)
    return ok


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def perf():
    B = 256
    layers = [(56, 56, 64, 64, 1, 1), (56, 56, 64, 64, 3, 1), (56, 56, 64, 256, 1, 1), (56, 56, 256, 64, 1, 1), (28, 28, 128, 128, 3, 1),
              (28, 28, 128, 512, 1, 1), (14, 14, 256, 256, 3, 1), (14, 14, 256, 1024, 1, 1), (14, 14, 1024, 256, 1, 1), (7, 7, 512, 512, 3, 1),
              (7, 7, 512, 2048, 1, 1), (56, 56, 128, 128, 3, 2)]
    for (H, W, Cin, Cout, k, s) in layers:
        x = rnd(B, H, W, Cin, seed=1)
        w = rnd(Cout, Cin, k, k, seed=2, scale=0.05)
        wp, wd = ops.pack_weight(w.float()), ops.pack_weight(w.float(), mode=1)
        Ho, Wo = ops.out_hw(H, k, s), ops.out_hw(W, k, s)
        dy = rnd(B, Ho, Wo, Cout, seed=3)
        flops = 2.0 * B * Ho * Wo * Cout * Cin * k * k
        byt = 2.0 * (x.numel() + dy.numel())
        t_f = timeit(lambda: ops.conv2d_fwd(x, wp, k, s, want_stats=True))
        t_d = timeit(lambda: ops.conv2d_dgrad(dy, wd, (H, W), k, s))
        t_w = timeit(lambda: ops.conv2d_wgrad(dy, x, k, s))
        print(f"conv {H}x{W} {Cin}->{Cout} k{k}s{s}: fwd {t_f:.3f} ms ({flops / t_f / 1e9:.0f} TF/s, {byt / t_f / 1e6:.0f} GB/s) "
              f"dgrad {t_d:.3f} ms ({flops / t_d / 1e9:.0f} TF/s) wgrad {t_w:.3f} ms ({flops / t_w / 1e9:.0f} TF/s)", flush=True)
    # big GEMM (ViT fc1 shape)
    M, K, N = 50432, 768, 3072
    x = rnd(M, 1, 1, K)
    wp = ops.pack_weight(rnd(N, K).float())
    t = timeit(lambda: ops.conv2d_fwd(x, wp))
    print(f"gemm {M}x{N}x{K}: {t:.3f} ms {2.0 * M * N * K / t / 1e9:.0f} TF/s", flush=True)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "fwd"
    t0 = time.time()
    r = {"fwd": fwd, "wgrad": wgrad, "perf": perf}[what]()
    print(f"done {what} in {time.time() - t0:.1f}s")
    sys.exit(0 if r in (True, None) else 1)
