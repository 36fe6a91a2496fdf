"""The small kernels of the training step (optimizers, column / row reductions, casts, copies, pooling, the stride-2 helpers of
the BatchNorm-algebra downsample branch) against float64 PyTorch restatements of the same op, on the exact inputs the kernel
received (bf16-rounded where it reads bf16).

Tolerances follow tests/test_gpu_se_kernels.py.  An fp32 output must be within 2^-20 of the sum of the magnitudes of the terms
it combines (a sum of n fp32 terms is off by far less than that at the sizes used here, while a dropped term, a lost
`accumulate` or a misplaced factor is off by a whole term).  A bf16 output must be within one bf16 rounding of the exact value
plus the fp32 rounding of its terms.  Copies, casts, layout ops and sums of exactly representable data must match exactly,
and every reduction must give bit-identical results on two identical launches."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_ULP = 2.0 ** -8
FP32_SUM = 2.0 ** -20


def _ops():
    from deeplearning_b200 import ops

    return ops


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(*shape, seed, dtype=torch.float32, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=_gen(seed)) * scale).to(dtype)


def _fp32_close(got, ref, mag, what, rel=FP32_SUM):
    """|got - ref| <= rel * mag elementwise (mag: sum of the magnitudes of the terms behind each output)"""
    err = (got.double() - ref.double()).abs()
    bound = rel * mag.double() + 1e-30
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())}/{bad.numel()} out of bound, worst excess {float((err - bound).max()):.3g}"


def _bf16_close(got, ref, terms, what):
    """|got - ref| <= one bf16 ulp of ref + fp32 rounding of the terms (|terms| = sum of the magnitudes combined)"""
    ref = ref.double()
    err = (got.double() - ref).abs()
    bound = BF16_ULP * ref.abs() + 1e-6 * terms.double() + 1e-30
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements out of one bf16 rounding, worst {float((err - bound).max()):.3g}"


def _twice(fn):
    """run a reduction twice on identical inputs: the results must be bit-identical"""
    a = fn().clone()
    b = fn()
    assert torch.equal(a, b), "two identical launches differ"
    return a


# ------------------------------------------------------------------------------------------- stride-2 downsample helpers
@pytest.mark.parametrize("B,H,W,C", [(2, 49, 49, 256), (3, 25, 13, 64), (2, 56, 56, 64), (1, 13, 8, 16), (4, 1, 1, 8)])
def test_subsample2_and_add_even_pixels(B, H, W, C):
    """xs = x[:, ::2, ::2] on odd and even grids (49 x 49 is layer2.0's input at 196 px); gx[:, ::2, ::2] += gs in place on
    small integers (exact in bf16), odd rows / columns untouched"""
    ops = _ops()
    x = _randn(B, H, W, C, seed=1, dtype=torch.bfloat16)
    xs = ops.subsample2(x)
    assert torch.equal(xs, x[:, ::2, ::2])
    gx = torch.randint(-8, 9, (B, H, W, C), device="cuda", generator=_gen(2)).to(torch.bfloat16)
    gs = torch.randint(-8, 9, tuple(xs.shape), device="cuda", generator=_gen(3)).to(torch.bfloat16)
    want = gx.clone()
    want[:, ::2, ::2] += gs
    assert ops.add_even_pixels_(gx, gs) is gx
    assert torch.equal(gx, want)


@pytest.mark.parametrize("B,H,W,K,N", [
    (4, 16, 16, 64, 256), (2, 25, 25, 64, 256),      # pixels % 128 == 0: streaming kernel / not: implicit-GEMM kernel
    (2, 16, 16, 128, 512), (2, 28, 28, 128, 512),
    (8, 8, 8, 256, 512), (2, 25, 25, 256, 512)])      # 25 x 25: layer2.0's compact even-pixel grid at 196 px
def test_conv1x1_bn(B, H, W, K, N):
    """y = conv1x1(x, w) * scale + shift, both sides of the streaming-kernel dispatch, against float64"""
    ops = _ops()
    x = _randn(B, H, W, K, seed=4, dtype=torch.bfloat16)
    w = _randn(N, K, seed=5, scale=K ** -0.5)
    wb = w.to(torch.bfloat16)
    co = ops.BnCoeffs(N, "cuda")
    co.scale.copy_(torch.rand(N, device="cuda", generator=_gen(6)) * 2 + 0.25)
    co.shift.copy_(_randn(N, seed=7))
    y = ops.conv1x1_bn(x, ops.pack_weight(w), co)
    xd, wd = x.double().reshape(-1, K), wb.double()
    ref = (xd @ wd.t()) * co.scale.double() + co.shift.double()
    terms = (xd.abs() @ wd.abs().t()) * co.scale.double() + co.shift.double().abs()
    _bf16_close(y.reshape(-1, N), ref, terms, "conv1x1_bn")


# ------------------------------------------------------------------------------------------------------ column sums
@pytest.mark.parametrize("rows,ld,cols", [(1, 64, 64), (37, 72, 40), (1000, 256, 256), (5000, 1000, 1000), (300, 136, 130)])
def test_colsum(rows, ld, cols):
    """colsum of the first `cols` columns of a [rows, ld] bf16 matrix, fresh and accumulated onto `out`"""
    ops = _ops()
    m = _randn(rows, ld, seed=8, dtype=torch.bfloat16)
    md = m.double()[:, :cols]
    ref, mag = md.sum(0), md.abs().sum(0)
    got = _twice(lambda: ops.colsum(m, cols))
    _fp32_close(got, ref, mag, "colsum")
    base = _randn(cols, seed=9, scale=10.0)
    out = base.clone()
    ops.colsum(m, cols, out=out, accumulate=True)
    _fp32_close(out, base.double() + ref, mag + base.double().abs(), "colsum accumulate")


# rows = 592 * 64 + 1: the slice count hits its cap of 592 with 65 rows per slice, so the last nine slices are empty
TALL = [(5, 64, 64), (63, 72, 40), (37889, 64, 64), (37889, 72, 40), (300, 2056, 2056), (4097, 768, 768)]


@pytest.mark.parametrize("rows,ld,cols", TALL)
def test_colsum_tall(rows, ld, cols):
    ops = _ops()
    m = _randn(rows, ld, seed=10, dtype=torch.bfloat16)
    md = m.double()[:, :cols]
    got = _twice(lambda: ops.colsum_tall(m, cols))
    _fp32_close(got, md.sum(0), md.abs().sum(0), "colsum_tall")


@pytest.mark.parametrize("rows,C", [(5, 64), (63, 40), (37889, 200), (4097, 768)])
def test_colsum_prod(rows, C):
    ops = _ops()
    a = _randn(rows, C, seed=11, dtype=torch.bfloat16)
    b = _randn(rows, C, seed=12, dtype=torch.bfloat16)
    ad, bd = a.double(), b.double()
    got = _twice(lambda: ops.colsum_prod(a, b))
    _fp32_close(got, (ad * bd).sum(0), (ad * bd).abs().sum(0), "colsum_prod")
    got = _twice(lambda: ops.colsum_prod(a))
    _fp32_close(got, ad.sum(0), ad.abs().sum(0), "colsum_prod without b")


@pytest.mark.parametrize("T,C", [(1, 8), (3, 40), (100, 256), (5000, 40), (5000, 1000)])
def test_stats_colsum(T, C):
    """column sums of plane 0 of [T, 2, C] epilogue partials; plane 1 is ignored"""
    ops = _ops()
    stats = _randn(T, 2, C, seed=13, scale=100.0)
    sd = stats.double()[:, 0]
    got = _twice(lambda: ops.stats_colsum(stats))
    _fp32_close(got, sd.sum(0), sd.abs().sum(0), "stats_colsum")


# ------------------------------------------------------------------------------------------------ rows of a batch
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_batch_rowsum(dtype):
    """out[d] (+)= sum_b g.flat[offset + b * stride_b + d]: the class-token row (offset 0) and one token row of every image"""
    ops = _ops()
    B, T, D = 5, 7, 200
    g = _randn(B, T, D, seed=14, dtype=dtype)
    gd = g.double()
    for tok in (0, 3):
        ref = gd[:, tok].sum(0)
        mag = gd[:, tok].abs().sum(0)
        got = _twice(lambda: ops.batch_rowsum(g, T * D, B, D, offset=tok * D))
        _fp32_close(got, ref, mag, f"batch_rowsum row {tok}")
        base = _randn(D, seed=15, scale=10.0)
        out = base.clone()
        ops.batch_rowsum(g, T * D, B, D, out=out, accumulate=True, offset=tok * D)
        _fp32_close(out, base.double() + ref, mag + base.double().abs(), f"batch_rowsum row {tok} accumulate")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_copy_rows(dtype):
    """rows of 48 bytes between buffers with different pitches and offsets; every byte outside them keeps its value"""
    ops = _ops()
    per16 = 16 // torch.tensor([], dtype=dtype).element_size()
    cols, sp, dp, rows = 3 * per16, 5 * per16, 7 * per16, 9
    src = _randn(rows + 2, sp, seed=16, dtype=dtype)
    dst = torch.full((rows + 3, dp), 7.0, dtype=dtype, device="cuda")
    want = dst.clone()
    so, do = sp + per16, 2 * dp + 2 * per16
    want.view(-1)[do:do + rows * dp].view(rows, dp)[:, :cols] = src.view(-1)[so:so + rows * sp].view(rows, sp)[:, :cols]
    ops.copy_rows(src, so, sp, dst, do, dp, rows, cols)
    assert torch.equal(dst, want)


# ------------------------------------------------------------------------------------------- element-wise kernels
def test_rowscale():
    """drop_path's backward multiplier: 168 elements per sample (a multiple of 8, not of 64), dropped samples (scale 0) exact 0"""
    ops = _ops()
    x = _randn(6, 3, 7, 8, seed=17, dtype=torch.bfloat16)
    scale = torch.tensor([0.0, 1.25, 0.0, 1 / 0.9, 2.0, 0.7], device="cuda")
    y = ops.rowscale(x, scale)
    # the fp32 product of a bf16 and an fp32 value is exact in float64: rounding it to fp32, then to bf16, is the kernel's op
    want = (x.double() * scale.double().view(-1, 1, 1, 1)).float().to(torch.bfloat16)
    assert torch.equal(y, want)
    assert float(y[scale == 0].float().abs().max()) == 0.0


def test_tanh_fwd_bwd():
    ops = _ops()
    n = 1001
    u = _randn(n, seed=18, scale=3.0)
    u[:8] = torch.tensor([0.0, -0.0, 1e-30, -1e-6, 20.0, -20.0, 1e4, -3e38], device="cuda")
    t, t16 = ops.tanh_fwd(u)
    ref = torch.tanh(u.double())
    _fp32_close(t, ref, ref.abs(), "tanh", rel=2.0 ** -21)
    assert torch.equal(t16, t.to(torch.bfloat16))
    dt = _randn(n, seed=19, dtype=torch.bfloat16)
    du = ops.tanh_bwd(dt, t)
    td = t.double()
    _bf16_close(du, dt.double() * (1 - td * td), dt.double().abs() * (1 + td * td), "tanh backward")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("HW,C", [(1, 36), (49, 36), (49, 768), (3136, 100)])
def test_avgpool_any(dtype, HW, C):
    ops = _ops()
    x = _randn(3, HW, 1, C, seed=20, dtype=dtype)
    got = _twice(lambda: ops.avgpool_any(x))
    xd = x.double()
    _fp32_close(got, xd.mean((1, 2)), xd.abs().mean((1, 2)), "avgpool_any")


def test_cast_bf16_and_cast_f32():
    """bf16 -> fp32 of every bf16 bit pattern; fp32 -> bf16 round-to-nearest-even: ties, +-inf, overflow, NaN, signed zero,
    subnormals, and a length that is no multiple of any vector width"""
    ops = _ops()
    every = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.bfloat16)
    f = ops.cast_f32(every)
    ref = every.float()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(f), nan)
    assert torch.equal(f[~nan].view(torch.int32), ref[~nan].view(torch.int32))
    assert torch.equal(ops.cast_bf16(ref[~nan]).view(torch.int16), every[~nan].view(torch.int16))
    one = 1.0
    special = [one + 2 ** -8, one + 3 * 2 ** -8, -(one + 2 ** -8), 2 ** -8 + 2 ** -16, 3.0e38, -3.4028234e38, 1e-40, -1e-45,
               float("inf"), float("-inf"), 0.0, -0.0, float("nan"), one + 2 ** -8 + 2 ** -20]
    x = torch.cat([torch.tensor(special, device="cuda"), _randn(1003 - len(special), seed=21, scale=100.0)])
    y = ops.cast_bf16(x)
    want = x.to(torch.bfloat16)
    xn = torch.isnan(x)
    assert torch.equal(torch.isnan(y), xn)
    assert torch.equal(y[~xn].view(torch.int16), want[~xn].view(torch.int16))


def test_bn_eval_coeffs():
    """scale / shift of eval-mode BatchNorm against F.batch_norm(training=False), running variances from 1e-7 to 1e3"""
    import torch.nn.functional as F

    ops = _ops()
    C = 1000
    gamma = 1.0 + 0.3 * _randn(C, seed=22)
    beta = _randn(C, seed=23)
    rm = _randn(C, seed=24, scale=2.0)
    rv = 10.0 ** (torch.rand(C, device="cuda", generator=_gen(25)) * 10 - 7)
    eps = 1e-5
    co = ops.bn_eval_coeffs(gamma, beta, rm, rv, eps)
    scale = gamma.double() / (rv.double() + eps).sqrt()
    _fp32_close(co.scale, scale, scale.abs(), "scale", rel=2.0 ** -21)
    shift = beta.double() - rm.double() * scale
    _fp32_close(co.shift, shift, beta.double().abs() + (rm.double() * scale).abs(), "shift", rel=2.0 ** -21)
    x = _randn(16, C, seed=26, scale=3.0).double()
    want = F.batch_norm(x, rm.double(), rv.double(), gamma.double(), beta.double(), False, 0.0, eps)
    got = x * co.scale.double() + co.shift.double()
    _fp32_close(got, want, (x * scale).abs() + shift.abs() + (rm.double() * scale).abs(), "eval batch_norm", rel=2.0 ** -20)


# ------------------------------------------------------------------------------------------------ gradient clipping
@pytest.mark.parametrize("n", [1, 2, 3, 5, 4099, 1000003])
def test_grad_clip_coef(n):
    """{min(1, max_norm / (gscale * ||g|| + 1e-6)), gscale * ||g||}: n % 4 tails (added by block 0 only), a zero gradient, and
    max_norm far above and below the norm"""
    ops = _ops()
    g = _randn(n, seed=27)
    g[-1] = 1e3   # the last element belongs to the tail whenever n % 4 != 0
    for gscale in (1.0, 0.125):
        norm = gscale * float(g.double().norm())
        for max_norm in (1e-3 * norm, 1e3 * norm):
            out = _twice(lambda: ops.grad_clip_coef(g, max_norm, gscale=gscale))
            assert abs(float(out[1]) - norm) <= 2.0 ** -20 * norm, (float(out[1]), norm)
            coef = min(1.0, max_norm / (norm + 1e-6))
            assert abs(float(out[0]) - coef) <= 2.0 ** -20 * coef, (float(out[0]), coef)
    out = ops.grad_clip_coef(torch.zeros(n, device="cuda"), 1.0)
    assert float(out[0]) == 1.0 and float(out[1]) == 0.0


# ------------------------------------------------------------------------------------------------------------ AdamW
def test_adamw_many_steps():
    """1000 AdamW steps over two parameter arenas that share one hyper vector (the second call does not tick), with a
    per-element weight-decay mask, gscale, a global-norm clip coefficient, a learning rate that changes every step, and
    gradients of magnitude 1, 1e-8 (where eps matters) and 0.

    hyper[1..4] (1 - beta^t, beta^t, advanced in fp32 on the device) must stay within t * 2^-23 of the float64 values: each tick
    rounds beta^t once (2^-24) and the fp32 betas differ from the float64 ones by < 3e-8 relative.

    Parameter bound, per element: |p - p_ref| <= 2^-22 * sum_t |p_t| + 2^-12 * sum_t |u_t|, with p_t, u_t the float64
    parameter and update (lr_t * m_hat / (sqrt(v_hat) + eps)) of step t.  The first term covers the three fp32 roundings of
    p per step (the decay factor, its product with p, the subtraction of the update).  The second covers the relative error of
    an fp32 update, at most ~1e-4 = 2^-13.3: the bias corrections from the hyper bound above (<= 7.3e-5 relative for
    1 - beta2^t over t <= 1000, halved by the square root), the fp32 moment EMAs (<= 2^-24 / (1 - beta2) = 6e-5 relative for v,
    halved again) and a few roundings of the quotient."""
    ops = _ops()
    T, nA, nB = 1000, 2053, 1030
    n = nA + nB
    b1, b2, eps, gscale, max_norm = 0.9, 0.999, 1e-8, 0.5, 20.0
    p = _randn(n, seed=30)
    decay = float(torch.tensor(0.05))   # the fp32 value the kernel reads, for the float64 references too
    wd = (torch.rand(n, device="cuda", generator=_gen(31)) < 0.7).float() * decay
    gmag = torch.ones(n, device="cuda")
    gmag[torch.rand(n, device="cuda", generator=_gen(32)) < 0.15] = 1e-8
    gmag[torch.rand(n, device="cuda", generator=_gen(33)) < 0.05] = 0.0
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    hyper = torch.tensor([0.0, 0.0, 0.0, 1.0, 1.0], device="cuda")
    hist = torch.empty(T, 5, device="cuda")
    # float64 restatement, and torch.optim.AdamW on float64 copies (decayed / undecayed elements in two parameter groups)
    pd, md, vd = p.double(), torch.zeros(n, device="cuda", dtype=torch.float64), torch.zeros(n, device="cuda", dtype=torch.float64)
    sum_p, sum_u = torch.zeros_like(pd), torch.zeros_like(pd)
    dec = wd > 0
    q_dec, q_nodec = pd[dec].clone().requires_grad_(True), pd[~dec].clone().requires_grad_(True)
    opt = torch.optim.AdamW([{"params": [q_dec], "weight_decay": decay}, {"params": [q_nodec], "weight_decay": 0.0}],
                            lr=1.0, betas=(b1, b2), eps=eps)
    gen = _gen(34)
    for t in range(1, T + 1):
        lr = 1e-5 + 1e-3 * 0.5 * (1 + math.cos(math.pi * t / T))
        g = torch.randn(n, device="cuda", generator=gen) * gmag * (4.0 if t % 7 == 0 else 1.0)
        clip = ops.grad_clip_coef(g, max_norm, gscale=gscale)
        hyper[0] = lr
        ops.adamw_(p[:nA], g[:nA], m[:nA], v[:nA], wd[:nA], hyper, b1, b2, eps, gscale=gscale, clip=clip)
        ops.adamw_(p[nA:], g[nA:], m[nA:], v[nA:], wd[nA:], hyper, b1, b2, eps, gscale=gscale, tick=False, clip=clip)
        hist[t - 1] = hyper
        gd = g.double()
        norm = gscale * gd.norm()
        gd = gd * gscale * torch.clamp(max_norm / (norm + 1e-6), max=1.0)
        md = b1 * md + (1 - b1) * gd
        vd = b2 * vd + (1 - b2) * gd * gd
        u = lr * (md / (1 - b1 ** t)) / ((vd / (1 - b2 ** t)).sqrt() + eps)
        pd = pd * (1 - lr * wd.double()) - u
        sum_p += pd.abs()
        sum_u += u.abs()
        q_dec.grad, q_nodec.grad = gd[dec], gd[~dec]
        for group in opt.param_groups:
            group["lr"] = lr
        opt.step()
    assert torch.allclose(q_dec.detach(), pd[dec], rtol=1e-10, atol=1e-12)
    assert torch.allclose(q_nodec.detach(), pd[~dec], rtol=1e-10, atol=1e-12)
    ts = torch.arange(1, T + 1, device="cuda", dtype=torch.float64)
    for i, ref in ((1, 1 - b1 ** ts), (2, 1 - b2 ** ts), (3, b1 ** ts), (4, b2 ** ts)):
        err = (hist[:, i].double() - ref).abs()
        assert bool((err <= ts * 2.0 ** -23).all()), f"hyper[{i}]: worst err / t = {float((err / ts).max()):.3g}"
    err = (p.double() - pd).abs()
    bound = 2.0 ** -22 * sum_p + 2.0 ** -12 * sum_u
    bad = err > bound
    assert not bool(bad.any()), f"adamw: {int(bad.sum())}/{n} parameters out of bound, worst excess {float((err - bound).max()):.3g}"
