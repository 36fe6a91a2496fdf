"""Grouped 3x3 convolutions (ResNeXt conv2) on the implicit-GEMM kernels: forward and dgrad in channel-window mode, the
weight gradient in the grouped mode of the wgrad kernel. Every group width in scope (4 .. 64), 64 .. 2048 channels, stride 1
and 2, odd images (partial pixel boxes) and launches with several tiles per persistent CTA, against float64 PyTorch on the
same bf16-rounded operands. Statistics rows, the eval-mode BatchNorm fold, the fused BN-backward reduce of the dgrad, wgrad
accumulation and split-K are checked too, and a second identical launch must reproduce the first bit for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from deeplearning_b200 import ops

    return ops


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _close(a, b, rtol, atol, what):
    a, b = a.double(), b.double()
    err = (a - b).abs()
    bad = err > atol + rtol * b.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} bad, max abs err {float(err.max()):.4g} (ref max {float(b.abs().max()):.4g})"


def _same(run):
    a, b = run(), run()
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(x, y), "two identical launches differ"
    return a


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _coeffs(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    co = _ops().BnCoeffs(C, "cuda")
    co.scale.copy_(torch.rand(C, device="cuda", generator=g) + 0.5)
    co.shift.copy_(torch.randn(C, device="cuda", generator=g) * 0.5)
    return co


def _setup(C, Cg, B, H, W, seed=0):
    x = _rand(B, H, W, C, seed=seed + 1)
    w = _rand(C, Cg, 3, 3, scale=(9 * Cg) ** -0.5, seed=seed + 2)
    return x, w


# C, Cg, B, H, W, stride: every group width, 64 .. 2048 channels, odd images; the 28x28 rows give each of the 132 CTAs
# several tiles
SHAPES = [
    (64, 4, 2, 9, 11, 1), (64, 64, 3, 7, 7, 2), (128, 4, 32, 28, 28, 1), (128, 8, 4, 13, 13, 2), (256, 8, 32, 28, 28, 2),
    (256, 16, 4, 9, 11, 1), (512, 16, 2, 13, 13, 2), (1024, 32, 8, 7, 7, 1), (1024, 32, 4, 9, 11, 2), (2048, 64, 8, 7, 7, 1),
    (2048, 64, 2, 13, 13, 2),
]


@pytest.mark.parametrize("C,Cg,B,H,W,s", SHAPES)
def test_grouped_fwd_dgrad_wgrad(C, Cg, B, H, W, s):
    ops = _ops()
    g = C // Cg
    x, w = _setup(C, Cg, B, H, W)
    wp, wd = ops.pack_weight(w.float(), mode=3), ops.pack_weight(w.float(), mode=4)
    y, stats = _same(lambda: ops.conv2d_fwd(x, wp, 3, s, want_stats=True, groups=g))
    ref = _nhwc(F.conv2d(_nchw(x), w.double(), stride=s, padding=1, groups=g))
    assert y.shape == ref.shape
    _close(y, ref, 1e-2, 1e-2, "grouped fwd")
    yf = y.double().reshape(-1, C)
    _close(stats[:, 0].sum(0), yf.sum(0), 1e-3, 1e-2, "grouped fwd sum")
    _close(stats[:, 1].sum(0), (yf * yf).sum(0), 1e-3, 1e-2, "grouped fwd sumsq")

    dy = _rand(*y.shape, seed=7)
    (dx,) = _same(lambda: (ops.conv2d_dgrad(dy, wd, (H, W), 3, s, groups=g),))
    ref_dx = _nhwc(torch.nn.grad.conv2d_input((B, C, H, W), w.double(), _nchw(dy), stride=s, padding=1, groups=g))
    _close(dx, ref_dx, 1e-2, 2e-2, "grouped dgrad")

    (dw,) = _same(lambda: (ops.conv2d_wgrad(dy, x, 3, s, groups=g),))
    ref_dw = torch.nn.grad.conv2d_weight(_nchw(x), (C, Cg, 3, 3), _nchw(dy), stride=s, padding=1, groups=g)
    assert dw.shape == (C, Cg, 3, 3)
    _close(dw, ref_dw, 1e-4, 1e-4 * float(ref_dw.abs().max()), "grouped wgrad")


@pytest.mark.parametrize("C,Cg,s", [(128, 4, 1), (256, 8, 2), (1024, 32, 1), (2048, 64, 2)])
@pytest.mark.parametrize("relu", [True, False])
def test_grouped_eval_bn_fold(C, Cg, s, relu):
    ops = _ops()
    x, w = _setup(C, Cg, 16, 9, 11, seed=10)
    co = _coeffs(C, 13)
    (y,) = _same(lambda: (ops.conv2d_bn_act(x, ops.pack_weight(w.float(), mode=3), co, 3, s, relu=relu, groups=C // Cg),))
    want = _nhwc(F.conv2d(_nchw(x), w.double(), stride=s, padding=1, groups=C // Cg)) * co.scale.double() + co.shift.double()
    if relu:
        want = want.clamp_min(0)
    _close(y, want, 1e-2, 2e-2, "grouped conv + bn")


@pytest.mark.parametrize("C,Cg,B,H,W", [(128, 4, 32, 28, 28), (256, 8, 4, 9, 11), (512, 16, 8, 13, 13), (1024, 32, 16, 7, 7),
                                         (2048, 64, 4, 7, 7)])
def test_grouped_dgrad_bn_mask(C, Cg, B, H, W):
    """dz = relu'(bn1(x_raw)) * dgrad and the sums sum(dz), sum(dz * x_raw) of bn1's backward, from the grouped dgrad epilogue"""
    ops = _ops()
    g = C // Cg
    _, w = _setup(C, Cg, B, H, W, seed=20)
    dy = _rand(B, H, W, C, seed=22)
    x_raw, co = _rand(B, H, W, C, seed=23), _coeffs(C, 24)
    dz, stats = _same(lambda: ops.conv2d_dgrad(dy, ops.pack_weight(w.float(), mode=4), (H, W), 3, 1, bn_mask=(x_raw, co), groups=g))
    gref = _nhwc(torch.nn.grad.conv2d_input((B, C, H, W), w.double(), _nchw(dy), padding=1, groups=g))
    z = x_raw.double() * co.scale.double() + co.shift.double()
    clear = z.abs() > 1e-3
    _close(dz.double()[clear], torch.where(z > 0, gref, torch.zeros_like(gref))[clear], 1e-2, 2e-2, "grouped dgrad bn mask")
    dzf = dz.double().reshape(-1, C)
    _close(stats[:, 0].sum(0), dzf.sum(0), 1e-3, 1e-2, "sum(dz)")
    _close(stats[:, 1].sum(0), (dzf * x_raw.double().reshape(-1, C)).sum(0), 1e-3, 1e-2, "sum(dz x)")


@pytest.mark.parametrize("C,Cg,B,H,W,s,multi", [(128, 4, 1, 7, 7, 1, False), (128, 4, 64, 56, 56, 1, True),
                                               (256, 8, 64, 56, 56, 2, True), (1024, 32, 2, 7, 7, 1, False),
                                               (1024, 32, 128, 14, 14, 1, True)])
def test_grouped_wgrad_split_k_and_accumulate(C, Cg, B, H, W, s, multi):
    """one split at a handful of pixels, several at ResNeXt-sized ones (read back through the workspace size); accumulate=1
    adds onto the gradient buffer"""
    from deeplearning_b200 import _lib

    ops = _ops()
    g = C // Cg
    nbytes = _lib.load().b200_conv2d_grouped_wgrad_workspace_bytes(B, H, W, C, g, 3, s)
    splits = nbytes // (C * 9 * 64 * 4)
    assert nbytes % (C * 9 * 64 * 4) == 0 and (splits > 1) == multi, splits
    x, _ = _setup(C, Cg, B, H, W, seed=30)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    dy = _rand(B, Ho, Wo, C, seed=31)
    ref = torch.nn.grad.conv2d_weight(_nchw(x), (C, Cg, 3, 3), _nchw(dy), stride=s, padding=1, groups=g)
    base = torch.randn(C, Cg, 3, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(32))
    out = base.clone()
    ops.conv2d_wgrad(dy, x, 3, s, out=out, accumulate=True, groups=g)
    tol = 1e-4 * float(ref.abs().max())
    _close(out, base.double() + ref, 1e-4, tol, "grouped wgrad accumulate")
    (dw,) = _same(lambda: (ops.conv2d_wgrad(dy, x, 3, s, groups=g),))
    _close(dw, ref, 1e-4, tol, "grouped wgrad")


@pytest.mark.parametrize("C,Cg", [(64, 4), (128, 8), (256, 16), (1024, 32), (2048, 64)])
def test_grouped_pack_modes(C, Cg):
    """modes 3 / 4: block-diagonal [C][9*64] operands, from the single-tensor and the multi-tensor packing kernels"""
    from deeplearning_b200.engine.packing import ModelPack

    ops = _ops()
    w = torch.randn(C, Cg, 3, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(40))
    full = torch.zeros(C, C, 9, device="cuda")
    for grp in range(C // Cg):
        full[grp * Cg:(grp + 1) * Cg, grp * Cg:(grp + 1) * Cg] = w[grp * Cg:(grp + 1) * Cg].reshape(Cg, Cg, 9)
    blk = torch.arange(C, device="cuda") // 64 * 64
    cols = blk[:, None] + torch.arange(64, device="cuda")[None, :]                 # [C][64] channel of column j
    fwd = full[torch.arange(C, device="cuda")[:, None], cols]                       # [C][64][9] = W[o][c][tap]
    dgr = full[cols, torch.arange(C, device="cuda")[:, None]]                       # [C][64][9] = W[o = col][c = row][tap]
    want3 = fwd.permute(0, 2, 1).reshape(C, 9 * 64).to(torch.bfloat16)
    want4 = dgr.permute(0, 2, 1).reshape(C, 9 * 64).to(torch.bfloat16)
    assert torch.equal(ops.pack_weight(w, mode=3), want3)
    assert torch.equal(ops.pack_weight(w, mode=4), want4)
    pack = ModelPack([(w, 3, 9 * 64, C), (w, 4, 9 * 64, C)])
    pack.refresh(0)
    assert torch.equal(pack.get(w, 3), want3)
    assert torch.equal(pack.get(w, 4), want4)


def test_grouped_rejects_out_of_scope_shapes():
    """unsupported group widths / channel counts raise with the library's message; nothing is launched"""
    ops = _ops()
    x = _rand(2, 8, 8, 64)
    wp = torch.zeros(64, 9 * 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="group width"):
        ops.conv2d_fwd(x, wp, 3, 1, groups=32)    # Cg = 2
    with pytest.raises(RuntimeError, match="ksize"):
        ops.conv2d_fwd(x, wp, 1, 1, groups=16)
