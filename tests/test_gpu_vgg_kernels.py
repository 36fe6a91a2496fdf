"""The VGG passes (csrc/vgg.cuh) against float64 PyTorch at VGG's shapes: the 2x2 max-pool forward / backward (plain and
BatchNorm + ReLU, odd H / W, positive bf16 ties, exact-zero ties) and the BatchNorm-backward sums of its backward, the
adaptive 7x7 pool + flatten and its backward at 1x1 / 2x2 / 7x7 / 14x14 / odd maps, the classifier dropout, the epilogue
combinations the schedule adds (bias + ReLU, bias + statistics), and torch.optim.Adam over many steps."""
import pytest
import torch
import torch.nn.functional as F

from deeplearning_b200 import ops

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def _co(C, seed):
    g = torch.Generator().manual_seed(seed)
    co = ops.BnCoeffs(C, "cuda")
    co.scale.copy_((torch.rand(C, generator=g) + 0.5).cuda())
    co.shift.copy_((torch.randn(C, generator=g) * 0.5).cuda())
    co.mean.zero_()
    co.invstd.fill_(1.0)
    return co


def _act(B, H, W, C, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g)
    if ties:
        # values on a coarse grid: many equal (bf16-exact) maxima in a window, including exact zeros after the ReLU
        x = torch.randint(-2, 3, (B, H, W, C), generator=g).float() * 0.5
    return x.to(BF16).cuda().contiguous()


def _ref_pool(v):
    """torch max-pool (float64, NCHW) of v [B,H,W,C] -> pooled NHWC and the arg-max window tap (row-major)."""
    y, ind = F.max_pool2d(_nchw(v), 2, 2, return_indices=True)
    W = v.shape[2]
    tap = (ind // W % 2) * 2 + (ind % W % 2)
    return y.permute(0, 2, 3, 1), tap.permute(0, 2, 3, 1)


@pytest.mark.parametrize("shape", [(2, 8, 8, 64), (3, 7, 9, 128), (2, 14, 14, 512), (1, 5, 5, 256)])
@pytest.mark.parametrize("bn", [False, True])
@pytest.mark.parametrize("ties", [False, True])
def test_pool_fwd_bwd(shape, bn, ties):
    B, H, W, C = shape
    x = _act(B, H, W, C, 1, ties)
    co = _co(C, 2) if bn else None
    if not bn:
        x = torch.relu(x)   # the plain pool reads relu(conv + b), written by the GEMM
    v = torch.relu(x.double() * co.scale.double() + co.shift.double()) if bn else x.double()
    y, idx = ops.vgg_pool_fwd(x, co)
    ry, rtap = _ref_pool(v)
    if bn:   # (fp32 fma in the kernel, then one bf16 rounding)
        assert torch.allclose(y.double(), ry, rtol=2 ** -8, atol=1e-6)
    else:
        assert torch.equal(y.double(), ry)
        assert torch.equal(idx.long(), rtap)   # ties to the first maximum, as torch
    g = _act(B, H // 2, W // 2, C, 3)
    # reference gradient w.r.t. the pre-activation: through torch's pool (its own arg-max) and the ReLU mask
    pre = (x.double() * co.scale.double() + co.shift.double()) if bn else x.double()
    pre_n = _nchw(pre).requires_grad_()
    out = F.max_pool2d(torch.relu(pre_n), 2, 2)
    out.backward(_nchw(g))
    ref = pre_n.grad.permute(0, 2, 3, 1)
    if bn:
        dz, part = ops.vgg_pool_bwd(g, idx, (H, W), c=x, co=co)
        # partial sums of the stored dz and dz * c
        s = part.double().sum(0)
        c64 = x.double().reshape(-1, C)
        d64 = dz.double().reshape(-1, C)
        assert torch.allclose(s[0], d64.sum(0), rtol=1e-5, atol=1e-3)
        assert torch.allclose(s[1], (d64 * c64).sum(0), rtol=1e-5, atol=1e-3)
        # the arg-max of relu(c * scale + shift), ties to the first: checked wherever the float64 ordering of the window and
        # the fp32 one (torch's mul + add; the kernel's fma agrees with it on the tie grid, where c * scale is exact) agree
        _, tap32 = _ref_pool(torch.relu(x.float() * co.scale + co.shift))
        agree = tap32 == rtap
        assert float(agree.double().mean()) > 0.99
        assert torch.equal(idx.long()[agree], rtap[agree])
        # dz: g at the kernel's own arg-max where the activation there is positive, 0 elsewhere (also where a whole window
        # is <= 0, the exact-zero ties of the ReLU)
        Ho, Wo = H // 2, W // 2
        expect = torch.zeros(B, H, W, C, dtype=torch.float64, device="cuda")
        t = idx.long()
        for tap in range(4):
            dh, dw = tap // 2, tap % 2
            sel = (t == tap) & (pre[:, dh:2 * Ho:2, dw:2 * Wo:2] > 0)
            expect[:, dh:2 * Ho:2, dw:2 * Wo:2] = torch.where(sel, g.double(), 0.0)
        assert torch.equal(dz.double(), expect)
        if not ties:
            assert torch.equal(dz.double(), ref.to(BF16).double())
        dx = dz
    else:
        dx = ops.vgg_pool_bwd(g, idx, (H, W), y=y)
        assert torch.equal(dx.double(), ref.to(BF16).double())
    if H % 2 or W % 2:
        assert dx[:, (H // 2) * 2:].abs().sum() == 0 and dx[:, :, (W // 2) * 2:].abs().sum() == 0


@pytest.mark.parametrize("hw", [(1, 1), (2, 2), (7, 7), (14, 14), (5, 9), (3, 17)])
def test_avgpool7_fwd_bwd(hw):
    B, C = 3, 512
    H, W = hw
    x = _act(B, H, W, C, 4)
    y = ops.vgg_avgpool7_fwd(x)
    xn = _nchw(x).requires_grad_()
    ref = torch.flatten(F.adaptive_avg_pool2d(xn, (7, 7)), 1)
    assert y.shape == (B, C * 49)
    err = (y.double() - ref.detach()).abs().max()
    assert err <= 2 ** -8 * ref.detach().abs().max() + 1e-6, float(err)
    gy = _act(B, 1, 1, C * 49, 5).view(B, C * 49)
    ref.backward(gy.double())
    gx = ops.vgg_avgpool7_bwd(gy, (B, H, W, C))
    rg = xn.grad.permute(0, 2, 3, 1)
    err = (gx.double() - rg).abs().max()
    assert err <= 2 ** -8 * rg.abs().max() + 1e-6, float(err)


@pytest.mark.parametrize("p", [0.5, 0.1, 0.0])
def test_dropout_fwd_bwd(p):
    B, N = 8, 4096
    pre = _act(B, 1, 1, N, 6).view(B, N)
    r = torch.relu(pre)
    torch.manual_seed(7)
    m = F.dropout(torch.ones(B, N, device="cuda"), p, True)
    h = ops.vgg_dropout_fwd(r, m) if p > 0 else r
    ref = r.double() * m.double()
    assert torch.equal(h.double(), ref.to(BF16).double())
    g = _act(B, 1, 1, N, 8).view(B, N)
    dx = ops.vgg_dropout_bwd(g, h, p)
    ref_dx = g.double() * m.double() * (pre.double() > 0)
    assert torch.equal(dx.double(), ref_dx.to(BF16).double())


@pytest.mark.parametrize("bn", [False, True])
def test_conv_bias_epilogues(bn):
    """conv + bias + ReLU (plain layers, classifier) and conv + bias with statistics (the _bn layers)"""
    B, H, W, Cin, Cout = 2, 12, 10, 128, 256
    x = _act(B, H, W, Cin, 9)
    w = torch.randn(Cout, Cin, 3, 3, generator=torch.Generator().manual_seed(10)).cuda() * 0.05
    b = torch.randn(Cout, generator=torch.Generator().manual_seed(11)).cuda()
    ref = F.conv2d(_nchw(x), w.double(), b.double(), padding=1).permute(0, 2, 3, 1)
    if bn:
        y, st = ops.conv2d_fwd(x, ops.pack_weight(w), 3, 1, want_stats=True, bias=b)
        s = st.double().sum(0)
        r2 = ref.reshape(-1, Cout)
        assert torch.allclose(s[0], y.double().reshape(-1, Cout).sum(0), rtol=1e-4, atol=1e-2)
        assert torch.allclose(s[0] / r2.shape[0], r2.mean(0), atol=2e-2)
    else:
        y, _ = ops.conv2d_fwd(x, ops.pack_weight(w), 3, 1, bias=b, act=1)
        ref = torch.relu(ref)
    err = (y.double() - ref).abs().max()
    assert err <= 1e-2 * ref.abs().max(), float(err)


def test_adam_matches_torch():
    n = 10007
    g0 = torch.Generator().manual_seed(12)
    p = torch.randn(n, generator=g0).cuda()
    ref = p.double().clone().requires_grad_()
    opt = torch.optim.Adam([ref], lr=1e-2, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-3)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    hyper = torch.tensor([1e-2, 0.0, 0.0, 1.0, 1.0], device="cuda")
    gscale, max_norm = 0.5, 30.0
    for step in range(40):
        g = torch.randn(n, generator=g0).cuda()
        clip = ops.grad_clip_coef(g, max_norm, gscale=gscale)
        ops.adam_(p, g, m, v, hyper, 0.9, 0.99, 1e-8, 1e-3, gscale=gscale, clip=clip)
        ref.grad = g.double() * gscale * clip[0].double()
        opt.step()
    err = (p.double() - ref.detach()).abs().max()
    assert err <= 1e-5, float(err)
    assert torch.allclose(m.double(), opt.state[ref]["exp_avg"], atol=1e-5)
    assert torch.allclose(v.double(), opt.state[ref]["exp_avg_sq"], rtol=1e-4, atol=1e-7)
