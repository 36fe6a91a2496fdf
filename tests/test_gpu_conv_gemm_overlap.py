"""conv_gemm_kernel with several tiles per CTA: the MMA warpgroups hand each accumulator to the epilogue warpgroup through
the shared-memory image, so every launch here is sized to give each of the 132 persistent CTAs at least three tiles. Every
compile-time epilogue of the launcher (and the generic kernel) runs at 64- and 128-column tiles, with partial pixel boxes
(7x7 and 9x11 images, row counts that are not a multiple of 128) and channel counts that are not a multiple of the tile
width. Results are compared against an fp32 PyTorch reference with the tolerances of test_gpu_kernels.py, the statistics rows
against sums of the stored output, and a second identical launch must reproduce the first bit for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TILES_PER_CTA = 3
SMS = 132


def _ops():
    from deeplearning_b200 import ops

    return ops


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _close(a, b, rtol, atol, what):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    bad = err > atol + rtol * b.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} bad, max abs err {float(err.max()):.4g} (ref max {float(b.abs().max()):.4g})"


def _same(run):
    """run() twice: every returned tensor must be bit-identical."""
    a, b = run(), run()
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(x, y), "two identical launches differ"
    return a


def _coeffs(C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    co = _ops().BnCoeffs(C, "cuda")
    co.scale.copy_(torch.rand(C, device="cuda", generator=g) + 0.5)
    co.shift.copy_(torch.randn(C, device="cuda", generator=g) * 0.5)
    return co


def _rows(n_tiles):
    """flat row count giving >= TILES_PER_CTA tiles per CTA, with a partial last 128-row tile"""
    m_tiles = -(-TILES_PER_CTA * SMS // n_tiles)
    return m_tiles * 128 - 51


# (N, tile width): multiple of the tile, and partial column tiles (full_cols false)
WIDTHS = [(64, 64), (40, 64), (128, 128), (192, 128)]


def _stats_check(stats, y, what):
    yf = y.float().reshape(-1, y.shape[-1])
    _close(stats[:, 0].sum(0), yf.sum(0), 1e-3, 1e-2, what + " sum")
    _close(stats[:, 1].sum(0), (yf * yf).sum(0), 1e-3, 1e-2, what + " sumsq")


# ------------------------------------------------------------------------------------------------ GEMM-shaped epilogues
@pytest.mark.parametrize("N,bn", WIDTHS)
@pytest.mark.parametrize("epi", ["bias", "bias_res_f32_out_f32", "bias_colscale_res_f32_out_f32", "bias_gelu_aux",
                                 "gelu_bwd", "gelu_bwd_stats", "out_f32", "bias_out_f32", "stats", "rowscale_generic"])
def test_gemm_epilogues_many_tiles(N, bn, epi):
    ops = _ops()
    K = 192
    n_tiles = -(-N // bn)
    M = _rows(n_tiles)
    a = _rand(M, K, seed=1)
    w = _rand(N, K, scale=K ** -0.5, seed=2)
    wp = ops.pack_weight(w.float())
    g = torch.Generator(device="cuda").manual_seed(3)
    bias = torch.randn(N, device="cuda", generator=g)
    colscale = torch.rand(N, device="cuda", generator=g) + 0.5
    res32 = torch.randn(M, N, device="cuda", generator=g)
    aux_in = (torch.rand(M, N, device="cuda", generator=g) * 1.2).to(torch.bfloat16)
    rps = 97
    rs = torch.rand(-(-M // rps), device="cuda", generator=g) * 2.0
    ref = a.float() @ w.float().t()
    kw, want = {}, None
    if epi == "bias":
        kw, want = dict(bias=bias), ref + bias
    elif epi == "bias_res_f32_out_f32":
        kw, want = dict(bias=bias, residual=res32, out_f32=True), ref + bias + res32
    elif epi == "bias_colscale_res_f32_out_f32":
        kw, want = dict(bias=bias, colscale=colscale, residual=res32, out_f32=True), (ref + bias) * colscale + res32
    elif epi == "bias_gelu_aux":
        kw, want = dict(bias=bias, act=2, aux_out=True), F.gelu(ref + bias)
    elif epi.startswith("gelu_bwd"):
        kw, want = dict(act=3, aux_in=aux_in, want_stats=epi.endswith("stats")), ref * aux_in.float()
    elif epi == "out_f32":
        kw, want = dict(out_f32=True), ref
    elif epi == "bias_out_f32":
        kw, want = dict(bias=bias, out_f32=True), ref + bias
    elif epi == "stats":
        kw, want = dict(want_stats=True), ref
    elif epi == "rowscale_generic":
        kw = dict(bias=bias, rowscale=(rs, rps))
        want = (ref + bias) * rs.repeat_interleave(rps)[:M, None]
    res = _same(lambda: ops.gemm(a, wp, **kw))
    out = res[0]
    if out.dtype == torch.float32:
        _close(out, want, 1e-4, 1e-3, epi)
    else:
        _close(out, want, 1e-2, 1e-2, epi)
    if epi == "bias_gelu_aux":
        x = (ref + bias).requires_grad_(True)
        (gd,) = torch.autograd.grad(F.gelu(x).sum(), x)
        _close(res[1], gd, 1e-2, 1e-2, "GELU'(pre)")
    if kw.get("want_stats"):
        _stats_check(res[2], out, epi)


# ------------------------------------------------------------------------------------------------ convolution epilogues
def _conv_ref(x, w, k):
    return F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=k // 2).permute(0, 2, 3, 1)


# (H, W, B): 7x7 images are boxed 8x8x2 (two images per tile), 9x11 ones 16x4x2 (three tiles per two images): both leave
# rows of every tile outside the image
IMAGES = [(7, 7, 2 * TILES_PER_CTA * SMS), (9, 11, TILES_PER_CTA * SMS)]


@pytest.mark.parametrize("H,W,B", IMAGES)
@pytest.mark.parametrize("Cin,Cout", [(64, 64), (64, 40), (128, 128), (64, 192)])
@pytest.mark.parametrize("k", [1, 3])
def test_conv_fwd_stats_many_tiles(H, W, B, Cin, Cout, k):
    ops = _ops()
    x = _rand(B, H, W, Cin, seed=11)
    w = _rand(Cout, Cin, k, k, scale=(Cin * k * k) ** -0.5, seed=12)
    wp = ops.pack_weight(w.float())
    y, stats = _same(lambda: ops.conv2d_fwd(x, wp, k, 1, want_stats=True))
    _close(y, _conv_ref(x, w, k), 1e-2, 1e-2, "conv fwd")
    _stats_check(stats, y, "conv fwd")


@pytest.mark.parametrize("H,W,B", IMAGES)
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("relu,with_res", [(True, True), (True, False), (False, False)])
def test_conv_bn_affine_many_tiles(H, W, B, C, relu, with_res):
    ops = _ops()
    x = _rand(B, H, W, C, seed=13)
    w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=14)
    wp = ops.pack_weight(w.float())
    co = _coeffs(C, 15)
    res = _rand(B, H, W, C, seed=16) if with_res else None
    (y,) = _same(lambda: (ops.conv2d_bn_act(x, wp, co, 3, 1, relu=relu, residual=res),))
    want = _conv_ref(x, w, 3) * co.scale + co.shift
    if with_res:
        want = want + res.float()
    if relu:
        want = want.clamp_min(0)
    _close(y, want, 1e-2, 2e-2, "conv + bn")


@pytest.mark.parametrize("H,W,B", IMAGES)
@pytest.mark.parametrize("Cin,Cout", [(64, 64), (40, 64), (128, 128), (192, 64)])
@pytest.mark.parametrize("with_res", [False, True])
def test_conv_dgrad_many_tiles(H, W, B, Cin, Cout, with_res):
    ops = _ops()
    w = _rand(Cout, Cin, 3, 3, scale=(9 * Cout) ** -0.5, seed=21)
    dy = _rand(B, H, W, Cout, seed=22)
    wd = ops.pack_weight(w.float(), mode=1)
    res = _rand(B, H, W, Cin, seed=23) if with_res else None
    (dx,) = _same(lambda: (ops.conv2d_dgrad(dy, wd, (H, W), 3, 1, residual=res),))
    want = F.conv_transpose2d(dy.float().permute(0, 3, 1, 2), w.float(), padding=1).permute(0, 2, 3, 1)
    if with_res:
        want = want + res.float()
    _close(dx, want, 1e-2, 2e-2, "conv dgrad")


def _bn_mask_check(dz, g, x_raw, co, what):
    """dz = relu'(bn(x_raw)) * g, compared where bn(x_raw) is clearly away from 0 (the kernel evaluates it with one fma)"""
    z = x_raw.float() * co.scale + co.shift
    want = torch.where(z > 0, g, torch.zeros_like(g))
    clear = z.abs() > 1e-3
    _close(dz.float()[clear], want[clear], 1e-2, 2e-2, what)


def _bn_sums_check(dz, stats, x_raw, what):
    C = dz.shape[-1]
    dzf = dz.float().reshape(-1, C)
    _close(stats[:, 0].sum(0), dzf.sum(0), 1e-3, 1e-2, what + " sum(dz)")
    _close(stats[:, 1].sum(0), (dzf * x_raw.float().reshape(-1, C)).sum(0), 1e-3, 1e-2, what + " sum(dz x)")


@pytest.mark.parametrize("H,W,B", IMAGES)
@pytest.mark.parametrize("C", [64, 128, 192])
def test_dgrad_bn_mask_many_tiles(H, W, B, C):
    ops = _ops()
    w = _rand(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=31)
    dy = _rand(B, H, W, C, seed=32)
    wd = ops.pack_weight(w.float(), mode=1)
    x_raw, co = _rand(B, H, W, C, seed=33), _coeffs(C, 34)
    dz, stats = _same(lambda: ops.conv2d_dgrad(dy, wd, (H, W), 3, 1, bn_mask=(x_raw, co)))
    g = F.conv_transpose2d(dy.float().permute(0, 3, 1, 2), w.float(), padding=1).permute(0, 2, 3, 1)
    _bn_mask_check(dz, g, x_raw, co, "dgrad bn mask")
    _bn_sums_check(dz, stats, x_raw, "dgrad bn mask")


@pytest.mark.parametrize("C", [64, 128, 192])
def test_dual_gemm_bn_mask_many_tiles(C):
    ops = _ops()
    M = _rows(-(-C // (64 if C <= 64 else 128)))
    a0, a1 = _rand(M, 4 * C, seed=41), _rand(M, C, seed=42)
    wcat = _rand(C, 5 * C, scale=(5 * C) ** -0.5, seed=43)
    bias = torch.randn(C, device="cuda", generator=torch.Generator(device="cuda").manual_seed(44))
    x_raw, co = _rand(M, C, seed=45), _coeffs(C, 46)
    dz, stats = _same(lambda: ops.gemm_dual(a0, a1, wcat, bias, bn_mask=(x_raw, co)))
    g = torch.cat([a0, a1], 1).float() @ wcat.float().t() + bias
    _bn_mask_check(dz, g.reshape(dz.shape), x_raw, co, "dual gemm bn mask")
    _bn_sums_check(dz, stats, x_raw, "dual gemm bn mask")


@pytest.mark.parametrize("Cin", [64, 192])
def test_conv1x1_dgrad_masked_many_tiles(Cin):
    ops = _ops()
    Cout = 128
    M = _rows(-(-Cin // (64 if Cin <= 64 else 128)))   # (not a multiple of 128 rows: the implicit-GEMM kernel, not the stream one)
    dy = _rand(M, 1, 1, Cout, seed=51)
    w = _rand(Cout, Cin, 1, 1, scale=Cout ** -0.5, seed=52)
    wd = ops.pack_weight(w.float(), mode=1)
    res = _rand(M, 1, 1, Cin, seed=53)
    mask = _rand(M, 1, 1, Cin, seed=54).clamp_min(0)
    dz, stats = _same(lambda: ops.conv1x1_dgrad_masked(dy, wd, res, mask))
    want = (dy.float().reshape(M, Cout) @ w.float().reshape(Cout, Cin) + res.float().reshape(M, Cin))
    want = torch.where(mask.reshape(M, Cin) > 0, want, torch.zeros_like(want))
    _close(dz.reshape(M, Cin), want, 1e-2, 2e-2, "masked dgrad")
    _close(stats[:, 0].sum(0), dz.float().reshape(M, Cin).sum(0), 1e-3, 1e-2, "masked dgrad sum(dz)")
