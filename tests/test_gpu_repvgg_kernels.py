"""The RepVGG block passes (csrc/repvgg.cuh) against float64 PyTorch: the fused three-branch apply (with the statistics of its
own output), the backward reduce and apply, the eval fold, and the stem's combined [3x3 | 1x1] operand in the ModelPack.
Channel counts cover every RepVGG width class (48 .. 2560), the stem's pitched [c3 | c1] halves, odd row counts and the
row counts of stride-2 grids; two identical launches must agree bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

CHANNELS = [48, 96, 160, 1280, 1408, 2048, 2560]


def _ops():
    from deeplearning_b200 import ops

    return ops


def _bf(shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _co(C, g):
    co = _ops().BnCoeffs(C, "cuda")
    co.mean.copy_(torch.randn(C, generator=g, device="cuda") * 0.3)
    co.invstd.copy_(torch.rand(C, generator=g, device="cuda") + 0.5)
    co.scale.copy_(torch.randn(C, generator=g, device="cuda"))
    co.shift.copy_(torch.randn(C, generator=g, device="cuda") * 0.5)
    return co


def _branches(shape, C, ident, pitched, g):
    """(c3, c1, x): pitched = the stem's layout, both conv outputs as halves of one [..., 2C] tensor"""
    if pitched:
        c = _bf(tuple(shape) + (2 * C,), g)
        c3, c1 = c[..., :C], c[..., C:]
    else:
        c3, c1 = _bf(tuple(shape) + (C,), g), _bf(tuple(shape) + (C,), g)
    x = _bf(tuple(shape) + (C,), g).relu() if ident else None
    return c3, c1, x


def _d(t):
    return None if t is None else t.double()


CASES = [(C, (4, 7, 5), True, False) for C in CHANNELS] + [
    (48, (8, 17, 17), False, True),      # stem at 34 x 34 input: pitched halves, no identity
    (64, (3, 13, 11), True, True),       # pitched halves with an identity branch
    (96, (5, 25, 25), False, False),     # stride-2 grid of 49 x 49
    (1280, (2, 3, 3), False, False),     # stage4 at 96 px
    (2560, (1, 1, 1), False, False),     # a single row
]


@pytest.mark.parametrize("C, shape, ident, pitched", CASES)
def test_apply_and_output_statistics(C, shape, ident, pitched):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(C + len(shape))
    c3, c1, x = _branches(shape, C, ident, pitched, g)
    co3, co1 = _co(C, g), _co(C, g)
    coi = _co(C, g) if ident else None
    y, st = ops.repvgg_apply(c3, c1, co3, co1, x=x, co_id=coi, want_stats=True)
    want = _d(c3) * _d(co3.scale) + _d(c1) * _d(co1.scale) + _d(co3.shift) + _d(co1.shift)
    if ident:
        want = want + _d(x) * _d(coi.scale) + _d(coi.shift)
    want = want.relu()
    assert y.shape == c3.shape and y.is_contiguous()
    err = (y.double() - want).abs()
    assert float((err - 2 ** -7 * want.abs()).max()) <= 1e-4, float(err.max())
    rows = y.numel() // C
    assert st.shape == (ops.repvgg_partial_rows(rows, C), 2, C)
    yd = y.double().reshape(rows, C)
    s = st.double().sum(0)
    assert torch.allclose(s[0], yd.sum(0), rtol=1e-5, atol=1e-3)
    assert torch.allclose(s[1], (yd * yd).sum(0), rtol=1e-5, atol=1e-3)
    y2, st2 = ops.repvgg_apply(c3, c1, co3, co1, x=x, co_id=coi, want_stats=True)
    assert torch.equal(y, y2) and torch.equal(st, st2)
    y3, none = ops.repvgg_apply(c3, c1, co3, co1, x=x, co_id=coi)
    assert none is None and torch.equal(y, y3)


@pytest.mark.parametrize("C, shape, ident, pitched", CASES)
def test_backward_reduce_and_apply(C, shape, ident, pitched):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(7 * C + len(shape))
    c3, c1, x = _branches(shape, C, ident, pitched, g)
    y = _bf(tuple(shape) + (C,), g).relu()          # about half of the ReLU mask closed
    gy = _bf(tuple(shape) + (C,), g)
    part = ops.repvgg_bwd_reduce(gy, y, c3, c1, x)
    rows = y.numel() // C
    T = ops.repvgg_partial_rows(rows, C)
    assert part.shape == (3 if ident else 2, T, 2, C)
    dz = torch.where(y.double() > 0, gy.double(), torch.zeros((), dtype=torch.float64, device="cuda")).reshape(rows, C)
    ins = [c3, c1] + ([x] if ident else [])
    for b, inp in enumerate(ins):
        s = part[b].double().sum(0)
        assert torch.allclose(s[0], dz.sum(0), rtol=1e-5, atol=1e-3), b
        assert torch.allclose(s[1], (dz * inp.double().reshape(rows, C)).sum(0), rtol=1e-5, atol=1e-3), b
    assert torch.equal(part, ops.repvgg_bwd_reduce(gy, y, c3, c1, x))

    cos = [_co(C, g) for _ in ins]
    ms = [torch.randn(2, C, generator=g, device="cuda") * 0.1 for _ in ins]
    out = None
    if pitched:
        dc = torch.empty(c3.shape[:-1] + (2 * C,), dtype=torch.bfloat16, device="cuda")
        out = (dc[..., :C], dc[..., C:], torch.empty_like(x) if ident else None)
    res = ops.repvgg_bwd_apply(gy, y, c3, c1, cos[0], ms[0], cos[1], ms[1], x=x, co_id=cos[2] if ident else None,
                               m_id=ms[2] if ident else None, out=out)
    for b, inp in enumerate(ins):
        co, m = cos[b], ms[b].double()
        xhat = (inp.double().reshape(rows, C) - _d(co.mean)) * _d(co.invstd)
        want = _d(co.scale) * (dz - m[0] - xhat * m[1])
        got = res[b].double().reshape(rows, C)
        assert float(((got - want).abs() - 2 ** -7 * want.abs()).max()) <= 1e-3, (b, float((got - want).abs().max()))
    if not ident:
        assert res[2] is None
    res2 = ops.repvgg_bwd_apply(gy, y, c3, c1, cos[0], ms[0], cos[1], ms[1], x=x, co_id=cos[2] if ident else None,
                                m_id=ms[2] if ident else None)
    for a, b in zip(res, res2):
        assert (a is None and b is None) or torch.equal(a, b)


def _block(cin, cout, stride, seed):
    from deeplearning_b200.classification.RepVGG.models.repvgg import RepVGGBlock

    torch.manual_seed(seed)
    blk = RepVGGBlock(cin, cout, 3, stride=stride, padding=1)
    g = torch.Generator().manual_seed(seed)
    for mod in blk.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            with torch.no_grad():
                mod.weight.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
                mod.bias.copy_(torch.rand(mod.num_features, generator=g) - 0.5)
                mod.running_mean.copy_(torch.rand(mod.num_features, generator=g) - 0.5)
                mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
    return blk


@pytest.mark.parametrize("cin, cout, stride, ldk", [(3, 48, 2, 32), (3, 64, 2, 32), (48, 48, 1, None), (96, 96, 1, None),
                                                    (160, 160, 1, None), (384, 1408, 2, None), (512, 2048, 2, None)])
def test_fold_matches_oracle(cin, cout, stride, ldk):
    from oracle.repvgg import fold

    blk = _block(cin, cout, stride, cin + cout)
    with torch.no_grad():
        k, b = fold(blk.double())
    blk = blk.float().cuda()
    bn_id = blk.rbr_identity
    wp, bias = _ops().repvgg_fold(blk.rbr_dense.conv.weight, blk.rbr_1x1.conv.weight, blk.rbr_dense.bn, blk.rbr_1x1.bn, bn_id,
                                  ldk=ldk)
    L = 9 * cin if ldk is None else ldk
    want = torch.zeros(cout, L, dtype=torch.float64)
    want[:, : 9 * cin] = k.permute(0, 2, 3, 1).reshape(cout, 9 * cin)       # k = tap * I + i
    got = wp.double().cpu()
    assert wp.shape == (cout, L)
    assert float(((got - want).abs() - 2 ** -8 * want.abs()).max()) <= 1e-6
    assert torch.allclose(bias.double().cpu(), b, rtol=1e-5, atol=1e-5)
    wp2, bias2 = _ops().repvgg_fold(blk.rbr_dense.conv.weight, blk.rbr_1x1.conv.weight, blk.rbr_dense.bn, blk.rbr_1x1.bn,
                                    bn_id, ldk=ldk)
    assert torch.equal(wp, wp2) and torch.equal(bias, bias2)


@pytest.mark.parametrize("name, C0", [("RepVGG-A0", 48), ("RepVGG-B0", 64)])
def test_stem_combined_operand_follows_the_weights(name, C0):
    """ModelPack's shared [2*C0][32] stem operand: 3x3 weight in rows 0..C0-1 (k = tap * 3 + c), 1x1 weight at columns 12-14 of
    rows C0..2*C0-1, zeros elsewhere; refreshed when the weights change in place"""
    from deeplearning_b200.classification.RepVGG.models import func_dict
    from deeplearning_b200.engine import repvgg as engine
    from deeplearning_b200.engine.packing import weight_cache

    torch.manual_seed(0)
    m = func_dict[name](num_classes=5).cuda()

    def want():
        w3, w1 = m.stage0.rbr_dense.conv.weight.detach(), m.stage0.rbr_1x1.conv.weight.detach()
        t = torch.zeros(2 * C0, 32, device="cuda")
        t[:C0, :27] = w3.permute(0, 2, 3, 1).reshape(C0, 27)
        t[C0:, 12:15] = w1.reshape(C0, 3)
        return t.to(torch.bfloat16)

    pack = weight_cache.model_pack(m, engine._pack_spec)
    assert torch.equal(pack.shared("stem"), want())
    with torch.no_grad():
        m.stage0.rbr_dense.conv.weight.mul_(-2.0)
        m.stage0.rbr_1x1.conv.weight.add_(1.0)
    pack2 = weight_cache.model_pack(m, engine._pack_spec)
    assert pack2 is pack
    torch.cuda.synchronize()
    assert torch.equal(pack.shared("stem"), want())
