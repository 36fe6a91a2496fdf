"""The ShuffleNet v2 block tails (csrc/shufflenet.cuh shufflev2_tail_*) against float64, in all four modes (u passthrough or
relu(bn(cu)); split or joined output), at the branch widths of every variant and their stage boundaries
(b = 24 / 58 / 88 / 116 / 122 / 232 / 244 / 488: half offsets b / 2 odd, 2 mod 4 and 0 mod 4), on even and odd maps.  Every
pad channel of every output is exactly 0, the mask at exactly c * scale + shift = 0 passes no gradient (torch's ReLU), and
the partial rows sum to the float64 BatchNorm sums."""
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = [24, 58, 88, 116, 122, 232, 244, 488]
MAPS = [(5, 7), (4, 6)]


def _pad8(n):
    return (n + 7) // 8 * 8


def _act(B, H, W, b, bp, gen):
    t = torch.randn(B, H, W, b, generator=gen)
    return torch.cat([t, torch.zeros(B, H, W, bp - b)], -1).to(torch.bfloat16).cuda()


def _coeffs(b, bp, gen):
    from deeplearning_b200 import ops

    co = ops.BnCoeffs(bp, "cuda")
    s = torch.zeros(bp)
    t = torch.zeros(bp)
    s[:b] = torch.rand(b, generator=gen) + 0.5
    t[:b] = torch.randn(b, generator=gen) * 0.5
    s[0], t[0] = 0.5, -0.25          # c = 0.5 gives c * scale + shift = 0 exactly
    co.scale.copy_(s)
    co.shift.copy_(t)
    co.mean.zero_()
    co.invstd.fill_(1.0)
    return co


def _with_zero_mask(c):
    c = c.clone()
    c.view(-1, c.shape[-1])[::2, 0] = 0.5     # every other row of channel 0 sits exactly on the ReLU threshold
    return c


def _relu_bn64(c, co):
    return (c.double() * co.scale.double() + co.shift.double()).clamp_min(0.0)


def _mask64(c, co):
    return (c.double() * co.scale.double() + co.shift.double()) > 0


@pytest.mark.parametrize("hw", MAPS)
@pytest.mark.parametrize("b", WIDTHS)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("bn_u", [False, True])
def test_tail_fwd_bwd(bn_u, split, b, hw):
    from deeplearning_b200 import ops
    from deeplearning_b200.engine.shufflenetv2 import tail_layout

    B, (H, W) = 3, hw
    bp = _pad8(b)
    gen = torch.Generator().manual_seed(b * 10 + H + 2 * split + bn_u)
    c3 = _with_zero_mask(_act(B, H, W, b, bp, gen))
    u = _with_zero_mask(_act(B, H, W, b, bp, gen))
    co3 = _coeffs(b, bp, gen)
    co_u = _coeffs(b, bp, gen) if bn_u else None

    # ---- forward
    got = ops.shufflev2_tail_fwd(u, c3, co3, b, co_u=co_u, split=split)
    u64 = _relu_bn64(u, co_u) if bn_u else u.double()
    ref = tail_layout(u64, _relu_bn64(c3, co3), b, split)
    gots, refs = (got, ref) if split else ((got,), (ref,))
    for g_, r_ in zip(gots, refs):
        assert g_.shape == r_.shape
        lim = b if split else 2 * b
        assert not g_[..., lim:].any(), "pad channels must be exactly 0"
        err = (g_.double() - r_).abs()
        assert float((err - r_.abs() * 2.0 ** -8).max()) <= 1e-30, float(err.max())

    # ---- backward: random gradient, pad channels included (they must be ignored)
    if split:
        g = tuple(torch.randn(B, H, W, bp, generator=gen).to(torch.bfloat16).cuda() for _ in range(2))
    else:
        g = torch.randn(B, H, W, _pad8(2 * b), generator=gen).to(torch.bfloat16).cuda()
    dz3, p3, du, pu = ops.shufflev2_tail_bwd(g, c3, co3, b, cu=u if bn_u else None, co_u=co_u)
    a64 = torch.zeros(B, H, W, bp, dtype=torch.float64, device="cuda", requires_grad=True)
    v64 = torch.zeros_like(a64, requires_grad=True)
    out = tail_layout(a64, v64, b, split)
    gu, gv = torch.autograd.grad(out, (a64, v64), tuple(x.double() for x in g) if split else g.double())
    m3 = _mask64(c3, co3)
    assert not bool(m3.view(-1, bp)[::2, 0].any())
    ref_dz3 = gv * m3
    assert torch.equal(dz3.double(), ref_dz3)
    assert not dz3[..., b:].any() and not du[..., b:].any()
    T = ops.repvgg_partial_rows(B * H * W, bp)
    assert tuple(p3.shape) == (T, 2, bp)

    def sums_ok(part, dz, c):
        s = part.double().sum(0)
        ref = torch.stack([dz.reshape(-1, bp).sum(0), (dz * c.double()).reshape(-1, bp).sum(0)])
        assert not s[:, b:].any()
        assert float((s - ref).abs().max()) <= 1e-5 * (1.0 + float(ref.abs().max()))

    sums_ok(p3, ref_dz3, c3)
    if bn_u:
        ref_du = gu * _mask64(u, co_u)
        assert torch.equal(du.double(), ref_du)
        sums_ok(pu, ref_du, u)
    else:
        assert pu is None
        assert torch.equal(du.double(), gu)
