"""L2-resident chunk scheduling probe (ResNet-50 bottleneck chains, bs 256).

Question: the big (256 / 512-channel) tensors of a bottleneck are written by one kernel and re-read by the next one or two.
If the chain is run per batch chunk (NHWC batch slices are contiguous) with the intermediate in a chunk-sized buffer that
is re-used by every chunk, does the 50 MB L2 keep the intermediate on chip (no HBM write, no HBM re-read)?

Chains (layer1: 56x56, 64/256 channels; layer2: 28x28, 128/512):
  tail : bn_bwd_apply(dz, c3 -> dc3)  ->  wgrad(dc3, y2)  ->  dgrad(dc3 -> g2)
  head : dgrad(dc1 + residual dz_next -> gx)  ->  bn_bwd_reduce(gx, c3, y -> dz)
  fwd  : bn_apply(c3 + identity -> y)  ->  conv1x1(y -> c1, stats)
Each variant is captured in a CUDA graph and replayed; time = CUDA events around 10 replays.
Also: plain L2 retention (fill S MB, then read it back) for S = 16..192 MB.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from deeplearning_b200 import _lib, ops

BF16, F32 = torch.bfloat16, torch.float32
dev = torch.device("cuda")
lib = _lib.load()


def p(t):
    return None if t is None else t.data_ptr()


def st():
    return torch.cuda.current_stream().cuda_stream


def timed_graph(fn, reps=10):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn()
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3  # us


def l2_retention():
    print("== L2 retention: fill S MB then sum it (read GB/s; HBM-speed ~6000, L2-speed higher)")
    for mb in (16, 32, 48, 64, 80, 96, 112, 128, 160, 192, 384):
        n = mb * (1 << 20) // 2
        buf = torch.empty(n, dtype=BF16, device=dev)
        out = torch.empty(1, dtype=F32, device=dev)

        def both():
            buf.fill_(1.0)
            out.copy_(buf.sum(dtype=F32))

        def fill_only():
            buf.fill_(1.0)

        tb, tf = timed_graph(both), timed_graph(fill_only)
        print(f"  {mb:4d} MB: fill {tf:7.1f} us ({mb * 1.048576 / tf * 1e3:6.0f} GB/s)  fill+sum {tb:7.1f} us  -> sum {tb - tf:7.1f} us "
              f"({mb * 1.048576 / max(tb - tf, 1e-3) * 1e3:6.0f} GB/s)")


def coeffs(C):
    co = ops.BnCoeffs(C, dev)
    co.mean.normal_(0, 0.1)
    co.invstd.fill_(1.0)
    co.scale.fill_(1.0)
    co.shift.fill_(0.0)
    return co


def chains(name, B, H, Cs, Cb):
    """Cs = narrow width (64/128), Cb = 4*Cs block width."""
    print(f"== {name}: B={B} {H}x{H} narrow {Cs} wide {Cb}")
    g = torch.Generator(device=dev).manual_seed(0)
    big = lambda: torch.randn(B, H, H, Cb, device=dev, generator=g).to(BF16)
    small = lambda: torch.randn(B, H, H, Cs, device=dev, generator=g).to(BF16)
    dz, c3, y, dzn = big(), big(), big().relu_(), big()
    y2, dc1 = small(), small()
    w3 = torch.randn(Cb, Cs, 1, 1, device=dev, generator=g) * 0.05      # conv3: Cs -> Cb
    w1 = torch.randn(Cs, Cb, 1, 1, device=dev, generator=g) * 0.05      # conv1 (next block): Cb -> Cs
    w3d = ops.pack_weight(w3, 1)    # dgrad operand [Cs][Cb]
    w1d = ops.pack_weight(w1, 1)    # [Cb][Cs]
    w1f = ops.pack_weight(w1, 0)    # [Cs][Cb]
    co = coeffs(Cb)
    m = torch.zeros(2, Cb, dtype=F32, device=dev)
    rows = B * H * H
    dw3 = torch.zeros(Cb, Cs, 1, 1, dtype=F32, device=dev)
    g2 = torch.empty(B, H, H, Cs, dtype=BF16, device=dev)
    dz_out = torch.empty_like(dz)
    y_out = torch.empty_like(y)

    for nch in (1, 2, 4, 8, 16, 32):
        if B % nch:
            continue
        b = B // nch
        r = b * H * H
        # ---------------- tail
        dc_full = torch.empty(B, H, H, Cb, dtype=BF16, device=dev) if nch == 1 else None
        dc_buf = torch.empty(b, H, H, Cb, dtype=BF16, device=dev)

        def tail():
            for i in range(nch):
                sl = slice(i * b, (i + 1) * b)
                dc = dc_full if nch == 1 else dc_buf
                _lib.check(lib.b200_bn_bwd_apply(p(dz[sl]), p(c3[sl]), None, 1, p(dc), p(co.scale), p(co.shift), p(co.mean),
                                                 p(co.invstd), p(m[0]), p(m[1]), 0, r, Cb, st()), "apply")
                ops.conv2d_wgrad(dc, y2[sl], 1, 1, out=dw3, accumulate=(i > 0))
                ops.conv2d_dgrad(dc, w3d, (H, H), 1, 1, out=g2[sl])

        t_tail = timed_graph(tail)
        # ---------------- head
        gx_full = torch.empty(B, H, H, Cb, dtype=BF16, device=dev) if nch == 1 else None
        gx_buf = torch.empty(b, H, H, Cb, dtype=BF16, device=dev)
        nblk = lib.b200_bn_bwd_blocks(r, Cb)
        partial = torch.empty(nch, nblk, 2, Cb, dtype=F32, device=dev)

        def head():
            for i in range(nch):
                sl = slice(i * b, (i + 1) * b)
                gx = gx_full if nch == 1 else gx_buf
                ops.conv2d_dgrad(dc1[sl], w1d, (H, H), 1, 1, residual=dzn[sl], out=gx)
                _lib.check(lib.b200_bn_bwd_reduce(p(gx), p(c3[sl]), p(y[sl]), p(dz_out[sl]), p(co.scale), p(co.shift), 1, r, Cb,
                                                  p(partial[i]), st()), "reduce")

        t_head = timed_graph(head)
        # ---------------- fwd
        T = lib.b200_conv2d_fwd_stats_rows(b, H, H, Cs, 1, 1)
        stats = torch.empty(nch, T, 2, Cs, dtype=F32, device=dev)
        c1 = torch.empty(B, H, H, Cs, dtype=BF16, device=dev)

        def fwd():
            for i in range(nch):
                sl = slice(i * b, (i + 1) * b)
                _lib.check(lib.b200_bn_apply(p(c3[sl]), p(dzn[sl]), p(y_out[sl]), p(co.scale), p(co.shift), r, Cb, 1, st()), "bn_apply")
                _lib.check(lib.b200_conv2d_fwd(p(y_out[sl]), p(w1f), p(c1[sl]), b, H, H, Cb, Cs, 1, 1, p(stats[i]), None, 0, None,
                                               None, 0, None, None, st()), "conv")

        t_fwd = timed_graph(fwd)
        chunk_mb = b * H * H * Cb * 2 / 1e6
        print(f"  chunks {nch:2d} (big chunk {chunk_mb:6.1f} MB): tail {t_tail:7.1f} us   head {t_head:7.1f} us   fwd {t_fwd:7.1f} us")


if __name__ == "__main__":
    torch.manual_seed(0)
    l2_retention()
    chains("layer1", 256, 56, 64, 256)
    chains("layer2", 256, 28, 128, 512)
    chains("layer3", 256, 14, 256, 1024)
