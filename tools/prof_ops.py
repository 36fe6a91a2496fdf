"""Runs single ops at their BASELINE shapes inside a cudaProfilerStart/Stop range (for `ncu --profile-from-start off`).
python tools/prof_ops.py attn_bwd|wattn_bwd|wattn_fwd|dwconv|dwconv_wgrad|ln96 ..."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from deeplearning_b200 import ops

BF16 = torch.bfloat16
dev = "cuda"


def rnd(*shape, dtype=BF16, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(dtype)


def attn_bwd():
    B, T, H = 256, 197, 12
    qkv = rnd(B, T, 3 * H * 64, scale=0.5)
    out, lse = ops.attention_fwd(qkv, H, 0.125)
    dout = rnd(B, T, H * 64)
    return lambda: ops.attention_bwd(qkv, out, dout, lse, H, 0.125)


def _wattn():
    B, Hh, W, nH = 128, 56, 56, 3
    qkv = rnd(B, Hh, W, 3 * nH * 32, scale=0.5)
    nW = 64
    index = torch.randint(0, 169, (49, 49), device=dev)
    bias = ops.window_bias_gather(torch.randn(169, nH, device=dev), index, nH, torch.zeros(nW, 49, 49, device=dev))
    return B, Hh, W, nH, qkv, bias, None


def wattn_fwd():
    B, Hh, W, nH, qkv, bias, mask = _wattn()
    return lambda: ops.window_attention_fwd(qkv, nH, bias, 3, 32 ** -0.5)


def wattn_bwd():
    B, Hh, W, nH, qkv, bias, mask = _wattn()
    out, lse = ops.window_attention_fwd(qkv, nH, bias, 3, 32 ** -0.5)
    dout = rnd(B, Hh, W, nH * 32)
    return lambda: ops.window_attention_bwd(qkv, out, dout, bias, lse, nH, 3, 32 ** -0.5)


def dwconv():
    x = rnd(256, 56, 56, 96, dtype=torch.float32)
    wt = ops.dwconv7_pack(torch.randn(96, 1, 7, 7, device=dev))
    b = torch.randn(96, device=dev)
    return lambda: ops.dwconv7(x, wt, b)


def dwconv_wgrad():
    x = rnd(256, 56, 56, 96, dtype=torch.float32)
    du = rnd(256, 56, 56, 96)
    return lambda: ops.dwconv7_wgrad(du, x)


def ln96():
    x = rnd(256 * 56 * 56, 96, dtype=torch.float32)
    g = torch.ones(96, device=dev)
    b = torch.zeros(96, device=dev)
    return lambda: ops.layernorm_fwd(x, g, b, 1e-6)


def _swin_gemm(kind):
    M, C = 128 * 56 * 56, 96
    if kind == "qkv":
        a = rnd(M, C); wp = ops.pack_weight(torch.randn(3 * C, C, device=dev) * 0.1); b = torch.randn(3 * C, device=dev)
        return lambda: ops.gemm(a, wp, bias=b)
    if kind == "proj":
        a = rnd(M, C); wp = ops.pack_weight(torch.randn(C, C, device=dev) * 0.1); b = torch.randn(C, device=dev)
        res = rnd(M, C, dtype=torch.float32)
        return lambda: ops.gemm(a, wp, bias=b, residual=res, out_f32=True)
    if kind == "fc1":
        a = rnd(M, C); wp = ops.pack_weight(torch.randn(4 * C, C, device=dev) * 0.1); b = torch.randn(4 * C, device=dev)
        return lambda: ops.gemm(a, wp, bias=b, act=2, aux_out=True)
    a = rnd(M, 4 * C); wp = ops.pack_weight(torch.randn(C, 4 * C, device=dev) * 0.05); b = torch.randn(C, device=dev)
    res = rnd(M, C, dtype=torch.float32)
    return lambda: ops.gemm(a, wp, bias=b, residual=res, out_f32=True)


def swin_qkv():
    return _swin_gemm("qkv")


def swin_proj():
    return _swin_gemm("proj")


def swin_fc1():
    return _swin_gemm("fc1")


def swin_fc2():
    return _swin_gemm("fc2")


def res_l1_conv3():   # ResNet layer1 conv3: 1x1 64 -> 256 at 56x56 (+BN statistics)
    x = rnd(256, 56, 56, 64)
    wp = ops.pack_weight(torch.randn(256, 64, 1, 1, device=dev) * 0.1)
    return lambda: ops.conv2d_fwd(x, wp, want_stats=True)


def res_l1_conv2():   # ResNet layer1 conv2: 3x3 64 -> 64
    x = rnd(256, 56, 56, 64)
    wp = ops.pack_weight(torch.randn(64, 64, 3, 3, device=dev) * 0.1)
    return lambda: ops.conv2d_fwd(x, wp, 3, 1, want_stats=True)


def res_l3_conv2():   # ResNet layer3 conv2: 3x3 256 -> 256 at 14x14
    x = rnd(256, 14, 14, 256)
    wp = ops.pack_weight(torch.randn(256, 256, 3, 3, device=dev) * 0.05)
    return lambda: ops.conv2d_fwd(x, wp, 3, 1, want_stats=True)


def vit_fc1():        # ViT-B/16 fc1: [50432, 768] x [3072, 768]^T + bias, GELU, second output GELU'(pre) for the backward
    a = rnd(256 * 197, 768, scale=0.5)
    wp = ops.pack_weight(torch.randn(3072, 768, device=dev) * 0.03)
    b = torch.randn(3072, device=dev) * 0.1
    return lambda: ops.gemm(a, wp, bias=b, act=2, aux_out=True)


def vit_qkv():
    a = rnd(256 * 197, 768, scale=0.5)
    wp = ops.pack_weight(torch.randn(2304, 768, device=dev) * 0.03)
    b = torch.randn(2304, device=dev) * 0.1
    return lambda: ops.gemm(a, wp, bias=b)


def vit_fc2_dgrad():  # d_pre = (g W2) * saved GELU'(pre) with column sums (fc1 bias gradient)
    g = rnd(256 * 197, 768, scale=0.1)
    wd = ops.pack_weight(torch.randn(768, 3072, device=dev) * 0.03, mode=1)
    pre = rnd(256 * 197, 3072)
    return lambda: ops.gemm(g, wd, act=3, aux_in=pre, want_stats=True)


def vit_ln_bwd():      # ViT-B/16 LayerNorm backward: x fp32 [50432, 768], dy / residual gradient bf16 (layernorm_bwd_kernel)
    x = rnd(256 * 197, 768, dtype=torch.float32)
    g = torch.rand(768, device=dev) + 0.5
    y, mean, rstd = ops.layernorm_fwd(x, g, torch.zeros(768, device=dev), 1e-6)
    dy, add = rnd(256 * 197, 768, scale=0.1), rnd(256 * 197, 768, scale=0.1)
    return lambda: ops.layernorm_bwd(dy, x, mean, rstd, g, add=add)


def vit_fc1_wgrad():
    dy = rnd(256 * 197, 1, 1, 3072, scale=0.1)
    x = rnd(256 * 197, 1, 1, 768)
    return lambda: ops.conv2d_wgrad(dy, x)


def vit_attn_fwd():
    qkv = rnd(256, 197, 3 * 768, scale=0.5)
    return lambda: ops.attention_fwd(qkv, 12, 0.125)


def res_l3_wgrad():   # ResNet layer3 conv2 weight gradient: 3x3 256 -> 256 at 14x14
    x = rnd(256, 14, 14, 256)
    dy = rnd(256, 14, 14, 256, scale=0.1)
    return lambda: ops.conv2d_wgrad(dy, x, 3, 1)


def res_l1_wgrad():   # ResNet layer1 conv2 weight gradient: 3x3 64 -> 64 at 56x56 (merged-tap mode, N = 192)
    x = rnd(256, 56, 56, 64)
    dy = rnd(256, 56, 56, 64, scale=0.1)
    return lambda: ops.conv2d_wgrad(dy, x, 3, 1)


def res_l4_wgrad():   # ResNet layer4 conv2 weight gradient: 3x3 512 -> 512 at 7x7 (72 output tiles x 2 splits: one wave)
    x = rnd(256, 7, 7, 512)
    dy = rnd(256, 7, 7, 512, scale=0.1)
    return lambda: ops.conv2d_wgrad(dy, x, 3, 1)


def res_l2_dgrad_res():   # ResNet layer2 conv1 dgrad (1x1 512 <- 128) + identity-branch gradient
    dy = rnd(256, 28, 28, 128, scale=0.1)
    wd = ops.pack_weight(torch.randn(128, 512, 1, 1, device=dev) * 0.05, mode=1)
    res = rnd(256, 28, 28, 512, scale=0.1)
    return lambda: ops.conv2d_dgrad(dy, wd, (28, 28), residual=res)


def _res_tail(H, K, N):
    y2 = rnd(256, H, H, K).relu_()
    wp = ops.pack_weight(torch.randn(N, K, 1, 1, device=dev) * K ** -0.5)
    ident = rnd(256, H, H, N)
    co = ops.BnCoeffs(N, dev)
    co.scale.fill_(1.0), co.shift.fill_(0.1)
    return y2, wp, ident, co


def res_l1_conv3_bn_add_relu():   # round 2: ResNet layer1 conv3 + BN + identity + ReLU in ONE streaming GEMM (K=64 -> N=256, 56x56)
    y2, wp, ident, co = _res_tail(56, 64, 256)
    return lambda: ops.conv1x1_bn_act(y2, wp, co, ident)


def res_l2_conv3_bn_add_relu():
    y2, wp, ident, co = _res_tail(28, 128, 512)
    return lambda: ops.conv1x1_bn_act(y2, wp, co, ident)


def res_l3_conv3_bn_add_relu():
    y2, wp, ident, co = _res_tail(14, 256, 1024)
    return lambda: ops.conv1x1_bn_act(y2, wp, co, ident)


def res_l1_dgrad_masked():        # round 2: conv1 dgrad + identity gradient + ReLU mask + column sums (K=64 -> N=256)
    dc = rnd(256, 56, 56, 64, scale=0.1)
    wd = ops.pack_weight(torch.randn(64, 256, 1, 1, device=dev) * 0.05, mode=1)
    res, y = rnd(256, 56, 56, 256, scale=0.1), rnd(256, 56, 56, 256).relu_()
    return lambda: ops.conv1x1_dgrad_masked(dc, wd, residual=res, mask_src=y)


def res_l1_gemm_dual():           # round 2: dL/dy2 = [dz | y2] [aW | M]^T + kW  (K = 256 + 64 -> N = 64)
    dz, y2 = rnd(256, 56, 56, 256, scale=0.1), rnd(256, 56, 56, 64).relu_()
    wcat = rnd(64, 320, scale=0.05)
    b = torch.zeros(64, device=dev)
    return lambda: ops.gemm_dual(dz, y2, wcat, b)


def res_l1_gram():                # round 2: G = y2^T y2 (wgrad kernel on the narrow tensor) + column sums
    y2 = rnd(256, 56, 56, 64).relu_()
    return lambda: ops.gram_colsum(y2)


def vit_qkv_wgrad_bias():         # round 2: qkv weight gradient with the bias gradient summed from the dY tiles
    dy = rnd(256 * 197, 1, 1, 2304, scale=0.1)
    x = rnd(256 * 197, 1, 1, 768)
    b = torch.empty(2304, device=dev)
    return lambda: ops.conv2d_wgrad(dy, x, bias_out=b)


def _bn_co(c):
    C = c.shape[-1]
    co = ops.BnCoeffs(C, c.device)
    cf = c.float().reshape(-1, C)
    co.mean.copy_(cf.mean(0))
    co.invstd.copy_((cf.var(0, unbiased=False) + 1e-5).rsqrt())
    co.scale.copy_(co.invstd)
    co.shift.copy_(-co.mean * co.invstd)
    return co


def res_l1_dgrad3x3_bn_reduce():  # round 2 (late): layer1 conv2 dgrad (3x3 64 <- 64) + ReLU mask of bn1 + sum dz, sum dz*x
    dc = rnd(256, 56, 56, 64, scale=0.1)
    wd = ops.pack_weight(torch.randn(64, 64, 3, 3, device=dev) * 0.05, mode=1)
    c = rnd(256, 56, 56, 64)
    co = _bn_co(c)
    return lambda: ops.conv2d_dgrad(dc, wd, (56, 56), 3, 1, bn_mask=(c, co))


def res_l2_dgrad3x3_bn_reduce():  # layer2 conv2 dgrad (3x3 128 <- 128 at 28x28) with the fused BN-backward reduce
    dc = rnd(256, 28, 28, 128, scale=0.1)
    wd = ops.pack_weight(torch.randn(128, 128, 3, 3, device=dev) * 0.05, mode=1)
    c = rnd(256, 28, 28, 128)
    co = _bn_co(c)
    return lambda: ops.conv2d_dgrad(dc, wd, (28, 28), 3, 1, bn_mask=(c, co))


def res_l1_gemm_dual_bn_reduce():  # dL/dy2 dual GEMM (K = 256 + 64 -> N = 64) + bn2's mask and backward sums in the epilogue
    dz, y2 = rnd(256, 56, 56, 256, scale=0.1), rnd(256, 56, 56, 64).relu_()
    wcat = rnd(64, 320, scale=0.05)
    b = torch.zeros(64, device=dev)
    c = rnd(256, 56, 56, 64)
    co = _bn_co(c)
    return lambda: ops.gemm_dual(dz, y2, wcat, b, bn_mask=(c, co))


def res_l1_conv2_tap64():         # layer1 conv2 forward 3x3 64 -> 64 with resident weights (conv_tap64.cuh) + BN statistics
    return res_l1_conv2()


def res_stem_conv():              # space-to-depth stem conv (4 taps x 64 -> 64 at 112x112, conv_tap64.cuh) + BN statistics
    x = torch.randn(256, 3, 224, 224, device=dev)
    a = ops.stem_s2d(x)
    wp = rnd(64, 256, scale=0.05)   # [Cout][4 y-taps x 64] (values are irrelevant for the profile)
    return lambda: ops.stem_s2d_conv_fwd(a, wp, want_stats=True)


def res_l3_algebra_small():       # layer3 BN-algebra kernels: statistics from the Gram matrix and the backward rows / M kernels
    y2 = rnd(256, 14, 14, 256).relu_()
    w3 = torch.randn(1024, 256, 1, 1, device=dev) * 0.05
    wp = ops.pack_weight(w3)
    G, s = ops.gram_colsum(y2)
    gamma, beta = torch.ones(1024, device=dev), torch.zeros(1024, device=dev)
    rows = 256 * 14 * 14
    co = ops.bn_gram_stats(G, s, wp, rows, gamma, beta, 1e-5, 0.1, None, None, None)
    dz = rnd(256, 14, 14, 1024, scale=0.1)
    D = ops.conv2d_wgrad(dz, y2, 1, 1)
    st = torch.zeros(4, 2, 1024, device=dev)

    def run():
        ops.bn_gram_stats(G, s, wp, rows, gamma, beta, 1e-5, 0.1, None, None, None)
        ops.bn_conv1x1_bwd(st, D, G, s, wp, w3, rows, gamma, co)
    return run


if __name__ == "__main__":
    fns = [(n, globals()[n]()) for n in sys.argv[1:]]
    for _, f in fns:
        f()
        f()
    torch.cuda.synchronize()
    for n, f in fns:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            f()
        e1.record()
        torch.cuda.synchronize()
        print(f"{n}: {e0.elapsed_time(e1) / 5 * 1e3:.1f} us per call")
    torch.cuda.profiler.start()
    for _, f in fns:
        f()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
