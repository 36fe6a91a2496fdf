"""The EfficientNet MBConv passes (csrc/mbconv.cuh) against float64 PyTorch restatements of their ops, at every distinct
depthwise shape of EfficientNet-B0 (224 px, batch 2), B2 widths that are not multiples of 64, odd and 1x1 grids, k3 / k5 x
stride 1 / 2, with and without the on-load BatchNorm + SiLU and the residual.  Reductions must also be bit-identical
across two launches."""
import pytest
import torch
import torch.nn.functional as F

from deeplearning_b200 import ops

pytestmark = pytest.mark.gpu

# (B, H, W, C, k, stride): the depthwise layers of EfficientNet-B0 at 224 px (1a, 2a, 2b, 3a, 3b, 4a, 4b, 5a, 5b, 6a, 6b, 7a),
# B2 widths (88 -> 528, 120 -> 720, 208 -> 1248), odd grids (B1's 15 -> 8 stride-2 stage, 5 -> 3) and 1x1
DW_SHAPES = [(2, 112, 112, 32, 3, 1), (2, 112, 112, 96, 3, 2), (2, 56, 56, 144, 3, 1), (2, 56, 56, 144, 5, 2),
             (2, 28, 28, 240, 5, 1), (2, 28, 28, 240, 3, 2), (2, 14, 14, 480, 3, 1), (2, 14, 14, 480, 5, 1),
             (2, 14, 14, 672, 5, 1), (2, 14, 14, 672, 5, 2), (2, 7, 7, 1152, 5, 1), (2, 7, 7, 1152, 3, 1),
             (3, 9, 9, 528, 3, 1), (3, 9, 9, 720, 5, 2), (2, 5, 5, 1248, 5, 1), (3, 15, 15, 40, 5, 2), (2, 5, 7, 24, 3, 2),
             (2, 1, 1, 64, 3, 1), (2, 1, 1, 8, 5, 2), (1, 3, 3, 3840, 3, 1)]
ROW_SHAPES = [(2, 112 * 112, 16), (2, 56 * 56, 24), (4, 81, 88), (3, 25, 120), (2, 49, 1152), (2, 9, 2112), (3, 1, 8),
              (2, 4, 3840), (5, 13, 8192)]


def _bf16(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _co(C, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed + 100)
    co = ops.BnCoeffs(C, "cuda")
    co.mean.copy_(torch.randn(C, generator=g, device="cuda") * 0.2)
    co.invstd.copy_(torch.rand(C, generator=g, device="cuda") + 0.5)
    co.scale.copy_(torch.randn(C, generator=g, device="cuda"))
    co.shift.copy_(torch.randn(C, generator=g, device="cuda") * 0.5)
    return co


def _d(t):
    return t.double()


def _silu_in(x, co):
    return F.silu(_d(x) * _d(co.scale) + _d(co.shift))


def _dsilu(u):
    s = torch.sigmoid(u)
    return s * (1 + u * (1 - s))


def _close(got, ref, rel=1.5e-2, what=""):
    got, ref = got.detach().double(), ref.detach().double()
    err = float((got - ref).abs().max())
    lim = rel * float(ref.abs().max()) + 1e-6
    assert err <= lim, f"{what}: max err {err:.4g} > {lim:.4g}"


def _dwconv64(a, w, k, s):
    """float64 depthwise conv of NHWC a with w [C,1,k,k] -> NHWC"""
    C = a.shape[-1]
    return F.conv2d(a.permute(0, 3, 1, 2), _d(w), None, s, k // 2, 1, C).permute(0, 2, 3, 1)


@pytest.mark.parametrize("shape", DW_SHAPES)
@pytest.mark.parametrize("pre", [False, True])
def test_dw_fwd(shape, pre):
    B, H, W, C, k, s = shape
    x = _bf16(B, H, W, C)
    w = torch.randn(C, 1, k, k, device="cuda") * 0.3
    co = _co(C) if pre else None
    d, st = ops.dw_fwd(x, w, k, s, co=co, want_stats=True)
    a = _silu_in(x, co) if pre else _d(x)
    ref = _dwconv64(a, w, k, s)
    assert d.shape == ref.shape
    _close(d, ref, what="d")
    dd = _d(d).reshape(-1, C)
    _close(st.double().sum(0)[0], dd.sum(0), rel=1e-5, what="sum d")
    _close(st.double().sum(0)[1], (dd * dd).sum(0), rel=1e-5, what="sum d^2")
    d2, st2 = ops.dw_fwd(x, w, k, s, co=co, want_stats=True)
    assert torch.equal(d, d2) and torch.equal(st, st2)


@pytest.mark.parametrize("shape", DW_SHAPES)
@pytest.mark.parametrize("mode", ["plain", "residual", "pre"])
def test_dw_backward(shape, mode):
    B, H, W, C, k, s = shape
    x = _bf16(B, H, W, C, seed=1)
    w = torch.randn(C, 1, k, k, device="cuda") * 0.3
    co = _co(C, seed=2) if mode == "pre" else None
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    dd = _bf16(B, Ho, Wo, C, seed=3)
    res = _bf16(B, H, W, C, seed=4) if mode == "residual" else None
    a = (_silu_in(x, co) if co is not None else _d(x)).requires_grad_(True)
    w64 = _d(w).requires_grad_(True)
    F.conv2d(a.permute(0, 3, 1, 2), w64, None, s, k // 2, 1, C).permute(0, 2, 3, 1).backward(_d(dd))
    g_in = a.grad
    dx, part = ops.dw_dgrad(dd, w, x, k, s, co=co, residual=res)
    if co is not None:
        ref = g_in * _dsilu(_d(x) * _d(co.scale) + _d(co.shift))
        _close(dx, ref, what="dz_in")
        z = _d(dx).reshape(-1, C)
        _close(part.double().sum(0)[0], z.sum(0), rel=1e-5, what="sum dz")
        _close(part.double().sum(0)[1], (z * _d(x).reshape(-1, C)).sum(0), rel=1e-5, what="sum dz x")
    else:
        _close(dx, g_in + (_d(res) if res is not None else 0), what="dx")
        assert part is None
    gw = ops.dw_wgrad(dd, x, k, s, co=co)
    _close(gw, w64.grad, rel=1e-4, what="dW")
    assert torch.equal(gw, ops.dw_wgrad(dd, x, k, s, co=co))


@pytest.mark.parametrize("shape", ROW_SHAPES)
def test_squeeze_gate_passes(shape):
    B, HW, C = shape
    d = _bf16(B, HW, 1, C, seed=5)
    co = _co(C, seed=6)
    u = _silu_in(d, co).reshape(B, HW, C)
    pool, none = ops.silu_bn_squeeze(d, co)
    assert none is None
    _close(pool, u.mean(1), rel=1e-5, what="pool")
    mask = (torch.rand(B, C, device="cuda") > 0.3).float() / 0.7
    pool2, f16 = ops.silu_bn_squeeze(d, co, mask=mask)
    assert torch.equal(pool, pool2)
    assert torch.equal(f16, (pool * mask).to(torch.bfloat16))
    gate = torch.rand(B, C, device="cuda")
    a = ops.gate_apply(d, co, gate)
    _close(a.reshape(B, HW, C), u * _d(gate)[:, None], rel=1e-2, what="gate_apply")
    da = _bf16(B, HW, 1, C, seed=7)
    s = ops.gate_reduce(da, d, co)
    _close(s, (_d(da).reshape(B, HW, C) * u).sum(1), rel=1e-5, what="gate_reduce")
    assert torch.equal(s, ops.gate_reduce(da, d, co))


@pytest.mark.parametrize("B,C,Cr", [(2, 32, 8), (4, 144, 8), (3, 1152, 48), (2, 528, 24), (5, 3840, 160), (1, 8, 1),
                                    (2, 8192, 256)])
def test_excite(B, C, Cr):
    g = torch.Generator(device="cuda").manual_seed(8)
    pool = torch.randn(B, C, generator=g, device="cuda")
    w1 = torch.randn(Cr, C, 1, 1, generator=g, device="cuda") * C ** -0.5
    b1 = torch.randn(Cr, generator=g, device="cuda") * 0.1
    w2 = torch.randn(C, Cr, 1, 1, generator=g, device="cuda") * Cr ** -0.5
    b2 = torch.randn(C, generator=g, device="cuda") * 0.1
    hpre, gate = ops.excite_fwd(pool, w1, b1, w2, b2)
    p64 = [_d(t).requires_grad_(True) for t in (pool, w1, b1, w2, b2)]
    h64 = F.conv2d(p64[0].view(B, C, 1, 1), p64[1], p64[2])
    g64 = torch.sigmoid(F.conv2d(F.silu(h64), p64[3], p64[4])).view(B, C)
    _close(hpre, h64.view(B, Cr), rel=1e-5, what="hpre")
    _close(gate, g64, rel=1e-5, what="gate")
    s = torch.randn(B, C, generator=g, device="cuda")
    g64.backward(_d(s))
    dpool, dw1, db1, dw2, db2 = ops.excite_bwd(s, pool, hpre, gate, w1, w2)
    for got, ref, n in ((dpool, p64[0].grad, "dpool"), (dw1, p64[1].grad.view(Cr, C), "dw1"), (db1, p64[2].grad, "db1"),
                        (dw2, p64[3].grad.view(C, Cr), "dw2"), (db2, p64[4].grad, "db2")):
        _close(got, ref, rel=1e-4, what=n)
    again = ops.excite_bwd(s, pool, hpre, gate, w1, w2)
    assert all(torch.equal(a, b) for a, b in zip((dpool, dw1, db1, dw2, db2), again))


@pytest.mark.parametrize("shape", ROW_SHAPES)
@pytest.mark.parametrize("with_da", [False, True])
def test_silu_bn_bwd_reduce(shape, with_da):
    B, HW, C = shape
    d = _bf16(B, HW, 1, C, seed=9)
    co = _co(C, seed=10)
    dpool = torch.randn(B, C, device="cuda")
    da = _bf16(B, HW, 1, C, seed=11) if with_da else None
    gate = torch.rand(B, C, device="cuda") if with_da else None
    dz, part = ops.silu_bn_bwd_reduce(d, co, dpool, da=da, gate=gate)
    v = _d(dpool)[:, None] / HW
    if with_da:
        v = v + _d(da).reshape(B, HW, C) * _d(gate)[:, None]
    ref = v * _dsilu(_d(d).reshape(B, HW, C) * _d(co.scale) + _d(co.shift))
    _close(dz.reshape(B, HW, C), ref, what="dz")
    z = _d(dz).reshape(-1, C)
    _close(part.double().sum(0)[0], z.sum(0), rel=1e-5, what="sum dz")
    _close(part.double().sum(0)[1], (z * _d(d).reshape(-1, C)).sum(0), rel=1e-5, what="sum dz d")


@pytest.mark.parametrize("shape", ROW_SHAPES)
@pytest.mark.parametrize("rs_on,res_on", [(False, False), (True, False), (False, True), (True, True)])
def test_tail_passes_and_bn_backward_from_sums(shape, rs_on, res_on):
    B, HW, C = shape
    c = _bf16(B, HW, 1, C, seed=12)
    co = _co(C, seed=13)
    rs = (torch.rand(B, device="cuda") > 0.4).float() / 0.8 if rs_on else None
    res = _bf16(B, HW, 1, C, seed=14) if res_on else None
    y = ops.tail_apply(c, co, rs, residual=res)
    ref = (_d(c) * _d(co.scale) + _d(co.shift)).reshape(B, HW, C)
    if rs_on:
        ref = ref * _d(rs)[:, None, None]
    if res_on:
        ref = ref + _d(res).reshape(B, HW, C)
    _close(y.reshape(B, HW, C), ref, what="tail_apply")
    g = _bf16(B, HW, 1, C, seed=15)
    dz, part = ops.tail_bwd_reduce(g, c, rs)
    ref_dz = _d(g).reshape(B, HW, C) * (_d(rs)[:, None, None] if rs_on else 1.0)
    _close(dz.reshape(B, HW, C), ref_dz, what="tail dz")
    z = _d(dz).reshape(-1, C)
    _close(part.double().sum(0)[0], z.sum(0), rel=1e-5, what="sum dz")
    _close(part.double().sum(0)[1], (z * _d(c).reshape(-1, C)).sum(0), rel=1e-5, what="sum dz c")
    dc, dgamma, dbeta = ops.bn_backward_from_sums(dz, part, c, co)
    xhat = (_d(c).reshape(-1, C) - _d(co.mean)) * _d(co.invstd)
    db_ref, dg_ref = z.sum(0), (z * xhat).sum(0)
    _close(dbeta, db_ref, rel=1e-5, what="dbeta")
    _close(dgamma, dg_ref, rel=1e-4, what="dgamma")
    m1, m2 = db_ref / z.shape[0], dg_ref / z.shape[0]
    _close(dc.reshape(-1, C), _d(co.scale) * (z - m1 - xhat * m2), what="bn_backward_from_sums dx")


@pytest.mark.parametrize("C", [240, 3840])
@pytest.mark.parametrize("source", ["dz", "mask_x", "mask_y"])
def test_bn_bwd_apply_sources(C, source):
    """b200_bn_bwd_apply at widths that are not 8 * 2^k (one channel chunk, and two) for each gradient source: g is dz
    already, or g masked where x * scale + shift > 0, or where the stored output y > 0"""
    from deeplearning_b200 import _lib

    rows = 196
    g, x = _bf16(rows, C, seed=20), _bf16(rows, C, seed=21)
    y = _bf16(rows, C, seed=22) if source == "mask_y" else None
    co = _co(C, seed=23)
    m = torch.randn(2, C, device="cuda") * 0.1
    dx = torch.empty_like(x)
    ptr = [t.data_ptr() for t in (co.scale, co.shift, co.mean, co.invstd, m[0], m[1])]
    rc = _lib.load().b200_bn_bwd_apply(g.data_ptr(), x.data_ptr(), None if y is None else y.data_ptr(),
                                       1 if source == "dz" else 0, dx.data_ptr(), *ptr, 1, rows, C,
                                       torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "b200_bn_bwd_apply")
    z = _d(g)
    if source == "mask_x":   # (exact in float64: the product of a bf16 and an fp32 value, then one rounding)
        z = z * (_d(x) * _d(co.scale) + _d(co.shift) > 0)
    elif source == "mask_y":
        z = z * (_d(y) > 0)
    xhat = (_d(x) - _d(co.mean)) * _d(co.invstd)
    _close(dx, _d(co.scale) * (z - _d(m[0]) - xhat * _d(m[1])), what=f"bn_bwd_apply {source}")
