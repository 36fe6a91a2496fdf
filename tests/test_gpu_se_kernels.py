"""Squeeze-and-excitation tail kernels (csrc/se.cuh) against float64 PyTorch on the same bf16 inputs.

fp32 outputs must agree within 1e-5 of the largest reference value; bf16 outputs within one bf16 rounding of the exact value
(plus the fp32 rounding of the terms it is computed from, which matters where those terms cancel).  Shapes cover every tail
of SE-ResNet-50 (HW 3136 / 784 / 196 / 49, C 256 - 2048, Cr 16 - 128), SE-ResNet-18 (C 64, Cr 4) and tiny images (B = 3,
HW 1 and 4); batch sizes that are not multiples of 8 exercise the partial image tiles of the small kernels."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(4, 3136, 256, 16), (10, 784, 512, 32), (10, 196, 1024, 64), (11, 49, 2048, 128), (5, 3136, 64, 4),
          (3, 1, 256, 16), (3, 4, 128, 8), (1, 1, 64, 1), (9, 49, 512, 256)]
EPS = 1e-5
BF16_ULP = 2.0 ** -8


def _inputs(B, HW, C, Cr, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    H = W = int(round(HW ** 0.5))
    shape = (B, H, W, C) if H * W == HW else (B, HW, 1, C)
    c = (torch.randn(*shape, device="cuda", generator=g) + 0.1).to(torch.bfloat16)
    ident = torch.randn(*shape, device="cuda", generator=g).to(torch.bfloat16)
    gy = torch.randn(*shape, device="cuda", generator=g).to(torch.bfloat16)
    gamma = 1.0 + 0.2 * torch.randn(C, device="cuda", generator=g)
    beta = 0.2 * torch.randn(C, device="cuda", generator=g)
    w1 = torch.randn(Cr, C, device="cuda", generator=g) * C ** -0.5
    w2 = torch.randn(C, Cr, device="cuda", generator=g) * Cr ** -0.5
    return c, ident, gy, gamma, beta, w1, w2


def _coeffs(c, gamma, beta):
    """train-mode BatchNorm coefficients from the batch statistics of c (fp32, computed in float64)"""
    from deeplearning_b200 import ops

    C = c.shape[-1]
    x = c.double().reshape(-1, C)
    mean, var = x.mean(0), x.var(0, unbiased=False)
    invstd = (var + EPS).rsqrt()
    co = ops.BnCoeffs(C, c.device)
    co.mean.copy_(mean)
    co.invstd.copy_(invstd)
    co.scale.copy_(gamma.double() * invstd)
    co.shift.copy_(beta.double() - mean * gamma.double() * invstd)
    return co


def _fp32_close(got, ref, what, tol=1e-5):
    ref = ref.double()
    err = float((got.double() - ref).abs().max())
    assert err <= tol * float(ref.abs().max()) + 1e-30, f"{what}: max err {err:.3g} vs max |ref| {float(ref.abs().max()):.3g}"


def _bf16_close(got, ref, terms, what):
    """|got - ref| <= one bf16 ulp of ref + fp32 rounding of the terms (|terms| = sum of the magnitudes combined)"""
    ref = ref.double()
    err = (got.double() - ref).abs()
    bound = BF16_ULP * ref.abs() + 1e-6 * terms.double() + 1e-30
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements out of one bf16 rounding, worst {float((err - bound).max()):.3g}"


def _forward_ref(c, ident, co, w1, w2):
    B, C = c.shape[0], c.shape[-1]
    c64 = c.double().reshape(B, -1, C)
    u = c64 * co.scale.double() + co.shift.double()
    csum = c64.sum(1)
    pool = u.mean(1)
    h = torch.relu(pool @ w1.double().t())
    gate = torch.sigmoid(h @ w2.double().t())
    pre = u * gate[:, None, :] + ident.double().reshape(B, -1, C)
    terms = (u * gate[:, None, :]).abs() + ident.double().reshape(B, -1, C).abs()
    return csum, pool, h, gate, torch.relu(pre).reshape(c.shape), terms.reshape(c.shape)


@pytest.mark.parametrize("B,HW,C,Cr", SHAPES)
def test_se_forward_kernels(B, HW, C, Cr):
    from deeplearning_b200 import ops

    c, ident, _, gamma, beta, w1, w2 = _inputs(B, HW, C, Cr)
    co = _coeffs(c, gamma, beta)
    csum, pool = ops.se_squeeze(c, co)
    h, gate = ops.se_excite(pool, w1, w2)
    y = ops.se_apply(c, co, gate, ident)
    r_csum, r_pool, r_h, r_gate, r_y, terms = _forward_ref(c, ident, co, w1, w2)
    _fp32_close(csum, r_csum, "csum")
    _fp32_close(pool, r_pool, "pool")
    # the excite and apply kernels on exactly the inputs they were given
    _fp32_close(h, torch.relu(pool.double() @ w1.double().t()), "h")
    _fp32_close(gate, torch.sigmoid(h.double() @ w2.double().t()), "gate")
    _fp32_close(gate, r_gate, "gate (composed)", tol=1e-5)
    u = c.double() * co.scale.double() + co.shift.double()
    g4 = gate.double()[:, None, None, :] if c.dim() == 4 else gate.double()
    pre = u * g4 + ident.double()
    _bf16_close(y, torch.relu(pre), (u * g4).abs() + ident.double().abs(), "y")
    _bf16_close(y, r_y, terms, "y (composed)")
    # identical launches agree bit for bit
    csum2, pool2 = ops.se_squeeze(c, co)
    h2, gate2 = ops.se_excite(pool2, w1, w2)
    y2 = ops.se_apply(c, co, gate2, ident)
    assert torch.equal(csum, csum2) and torch.equal(pool, pool2) and torch.equal(h, h2) and torch.equal(gate, gate2)
    assert torch.equal(y, y2)


@pytest.mark.parametrize("B,HW,C,Cr", SHAPES)
def test_se_backward_kernels(B, HW, C, Cr):
    from deeplearning_b200 import _lib, ops

    c, ident, gy, gamma, beta, w1, w2 = _inputs(B, HW, C, Cr, seed=1)
    co = _coeffs(c, gamma, beta)
    csum, pool = ops.se_squeeze(c, co)
    h, gate = ops.se_excite(pool, w1, w2)
    y = ops.se_apply(c, co, gate, ident)
    torch.cuda.synchronize()
    outs = [ops.se_backward(gy, y, c, co, csum, pool, h, gate, w1, w2) for _ in range(2)]
    for a, b in zip(*outs):
        assert torch.equal(a, b), "two identical backward launches differ"
    dc, dz, dw1, dw2, dgamma, dbeta = outs[0]

    # reduce kernel on its own: dz, A = sum_p dz, R = sum_p dz * c
    mask = (y > 0).double()
    r_dz = gy.double() * mask
    assert torch.equal(dz.double(), r_dz)
    sums = torch.empty(2, B, C, device="cuda")
    dz2 = torch.empty_like(c)
    lib = _lib.load()
    _lib.check(lib.b200_se_bwd_reduce(gy.data_ptr(), y.data_ptr(), c.data_ptr(), dz2.data_ptr(), sums[0].data_ptr(),
                                      sums[1].data_ptr(), B, HW, C, torch.cuda.current_stream().cuda_stream), "se_bwd_reduce")
    _fp32_close(sums[0], r_dz.reshape(B, -1, C).sum(1), "A")
    _fp32_close(sums[1], (r_dz * c.double()).reshape(B, -1, C).sum(1), "R")

    # float64 autograd of the train-mode tail: BatchNorm with batch statistics -> SE gate -> + identity, masked like y
    c64 = c.double().reshape(B, -1, C).requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    w164, w264 = w1.double().requires_grad_(True), w2.double().requires_grad_(True)
    mean = c64.mean((0, 1))
    var = c64.var((0, 1), unbiased=False)
    u = (c64 - mean) * (var + EPS).rsqrt() * g64 + b64
    gate64 = torch.sigmoid(torch.relu(u.mean(1) @ w164.t()) @ w264.t())
    pre = u * gate64[:, None, :]
    (pre * r_dz.reshape(B, -1, C)).sum().backward()
    _fp32_close(dw1, w164.grad, "dW1")
    _fp32_close(dw2, w264.grad, "dW2")
    _fp32_close(dgamma, g64.grad, "dgamma")
    _fp32_close(dbeta, b64.grad, "dbeta")
    r_dc = c64.grad.reshape(c.shape)
    err = (dc.double() - r_dc).abs()
    # fp32 rounding of the terms scale * (dz * gate + dp / HW - m1 - xhat * m2), which cancel where BatchNorm normalises
    # only a few values per channel (B * HW = 1 makes dc exactly zero)
    term = float((r_dz.reshape(B, -1, C) * co.scale.double() * gate.double()[:, None, :]).abs().max())
    bound = BF16_ULP * r_dc.abs() + 1e-5 * max(float(r_dc.abs().max()), term)
    assert not bool((err > bound).any()), f"dc: worst excess {float((err - bound).max()):.3g}"
