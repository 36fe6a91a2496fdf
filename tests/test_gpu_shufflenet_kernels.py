"""The ShuffleNet v1 passes against float64 PyTorch restatements of their ops: the ReLU-on-load depthwise convolution
(forward with statistics, data gradient with bn1's partial rows, weight gradient) at stride 1 and 2, the stride-2 tail's
concatenated forward and its one-pass backward (divide-by-9 at borders, zero-average ReLU mask), the stride-1 and stem ReLU
reduces, and the dense block-diagonal grouped 1x1 forward / dgrad / gathered wgrad against F.conv2d(groups=g).  Bottleneck
widths that need padding (30, 54, 60, 90) run at their padded pitch with zero pad coefficients, and the pad channels must
come out exactly 0."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _bf(t):
    return t.to(BF16).cuda().contiguous()


def _co(scale, shift):
    from deeplearning_b200 import ops

    co = ops.BnCoeffs(scale.numel(), "cuda")
    co.scale.copy_(scale)
    co.shift.copy_(shift)
    co.mean.zero_()
    co.invstd.fill_(1.0)
    return co


def _padded(b, seed):
    """bf16-exact inputs of a bottleneck of width b at pitch bp: scale / shift with zero pad entries"""
    bp = (b + 7) // 8 * 8
    g = torch.Generator().manual_seed(seed)
    sc = torch.zeros(bp)
    sh = torch.zeros(bp)
    sc[:b] = torch.rand(b, generator=g) + 0.5
    sh[:b] = torch.randn(b, generator=g) * 0.5
    return bp, sc, sh, g


def _close(a, ref, rel=2e-2):
    a, ref = a.double().cpu(), ref.double().cpu()
    err = float((a - ref).abs().max())
    assert err <= rel * float(ref.abs().max()) + 1e-6, (err, float(ref.abs().max()))


@pytest.mark.parametrize("b", [30, 54, 60, 90])
@pytest.mark.parametrize("stride", [1, 2])
def test_dw_relu_passes(b, stride):
    from deeplearning_b200 import ops

    bp, sc, sh, g = _padded(b, b + stride)
    B, H, W = 3, 13, 11
    c1 = torch.randn(B, H, W, bp, generator=g)
    c1[..., b:] = 0
    c1 = c1.to(BF16).float()
    w = torch.zeros(bp, 1, 3, 3)
    w[:b] = torch.randn(b, 1, 3, 3, generator=g) * 0.3
    co = _co(sc.cuda(), sh.cuda())
    d, st = ops.dw_relu_fwd(_bf(c1), w.cuda(), stride, co, want_stats=True)
    u = torch.relu(c1.double() * sc.double() + sh.double()).permute(0, 3, 1, 2)
    ref = F.conv2d(u, w.double(), stride=stride, padding=1, groups=bp).permute(0, 2, 3, 1)
    _close(d.float(), ref)
    assert torch.equal(d[..., b:].float().cpu(), torch.zeros_like(ref[..., b:]).float())
    dq = d.float().cpu().double()
    _close(st.sum(0)[0], dq.sum((0, 1, 2)), 1e-4)
    _close(st.sum(0)[1], (dq * dq).sum((0, 1, 2)), 1e-4)

    dd = torch.randn(*d.shape, generator=g)
    dd[..., b:] = 0
    dd = dd.to(BF16).float()
    dz, part = ops.dw_relu_dgrad(_bf(dd), w.cuda(), _bf(c1), stride, co)
    v = torch.zeros(B, bp, H, W, dtype=torch.float64, requires_grad=True)
    (gin,) = torch.autograd.grad(F.conv2d(v, w.double(), stride=stride, padding=1, groups=bp), v,
                                 dd.double().permute(0, 3, 1, 2))
    mask = (c1.double() * sc.double() + sh.double()) > 0
    ref = gin.permute(0, 2, 3, 1) * mask
    _close(dz.float(), ref)
    assert torch.equal(dz[..., b:].float().cpu(), torch.zeros(B, H, W, bp - b))
    dzq = dz.float().cpu().double()
    _close(part.sum(0)[0], dzq.sum((0, 1, 2)), 1e-4)
    _close(part.sum(0)[1], (dzq * c1.double()).sum((0, 1, 2)), 1e-4)

    gw = ops.dw_relu_wgrad(_bf(dd), _bf(c1), stride, co)
    ref = torch.nn.grad.conv2d_weight(u, (bp, 1, 3, 3), dd.double().permute(0, 3, 1, 2), stride=stride, padding=1,
                                      groups=bp)
    _close(gw, ref, 1e-3)
    assert torch.equal(gw[b:].cpu(), torch.zeros(bp - b, 1, 3, 3))


@pytest.mark.parametrize("hw", [(8, 8), (7, 9)])
def test_tail_s2_forward_and_backward(hw):
    """the pool half divides by 9 at the borders too (count_include_pad); a pooled value of exactly 0 gets no gradient"""
    from deeplearning_b200 import ops

    B, Cin, Cc = 2, 24, 40
    H, W = hw
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, H, W, Cin, generator=g)
    x[:, :, :, :8] = 0.0        # channels whose pooled average is exactly 0 everywhere
    x = x.to(BF16).float()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    c3 = torch.randn(B, Ho, Wo, Cc, generator=g).to(BF16).float()
    sc, sh = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g) * 0.3
    y = ops.shuffle_tail_s2_fwd(_bf(x), _bf(c3), _co(sc.cuda(), sh.cuda()))
    pool = F.avg_pool2d(x.double().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    ref = torch.relu(torch.cat([pool, c3.double() * sc.double() + sh.double()], -1))
    _close(y.float(), ref, 1e-2)
    assert torch.equal(y[..., :8].float().cpu(), torch.zeros(B, Ho, Wo, 8))

    gy = torch.randn(B, Ho, Wo, Cin + Cc, generator=g).to(BF16).float()
    dz, part, gx = ops.shuffle_relu_bwd(_bf(gy), _bf(c3), y=y, in_hw=(H, W))
    yq = y.float().cpu().double()
    gm = gy.double() * (yq > 0)
    _close(dz.float(), gm[..., Cin:], 1e-2)
    dzq = dz.float().cpu().double()
    _close(part.sum(0)[0], dzq.sum((0, 1, 2)), 1e-4)
    _close(part.sum(0)[1], (dzq * c3.double()).sum((0, 1, 2)), 1e-4)
    xd = x.double().permute(0, 3, 1, 2).requires_grad_()
    (ref_gx,) = torch.autograd.grad(F.avg_pool2d(xd, 3, 2, 1), xd, gm[..., :Cin].permute(0, 3, 1, 2))
    _close(gx.float(), ref_gx.permute(0, 2, 3, 1), 1e-2)
    assert torch.equal(gx[..., :8].float().cpu(), torch.zeros(B, H, W, 8))
    # the corner pixel is read by one window only: its gradient is that window's masked gradient / 9
    _close(gx[:, 0, 0, 8:].float(), gm[:, 0, 0, 8:Cin] / 9.0, 1e-2)


def test_relu_reduce_stride1_and_stem():
    from deeplearning_b200 import ops

    B, H, W, C = 2, 9, 10, 48
    g = torch.Generator().manual_seed(9)
    c = torch.randn(B, H, W, C, generator=g).to(BF16).float()
    y = torch.relu(torch.randn(B, H, W, C, generator=g)).to(BF16).float()
    gy = torch.randn(B, H, W, C, generator=g).to(BF16).float()
    dz, part, gx = ops.shuffle_relu_bwd(_bf(gy), _bf(c), y=_bf(y))
    assert gx is None
    ref = gy.double() * (y > 0)
    assert torch.equal(dz.float().cpu().double(), ref)
    _close(part.sum(0)[0], ref.sum((0, 1, 2)), 1e-4)
    _close(part.sum(0)[1], (ref * c.double()).sum((0, 1, 2)), 1e-4)
    sc, sh = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    dz, part, _ = ops.shuffle_relu_bwd(_bf(gy), _bf(c), co=_co(sc.cuda(), sh.cuda()))
    ref = gy.double() * ((c * sc + sh) > 0)
    assert torch.equal(dz.float().cpu().double(), ref)
    _close(part.sum(0)[1], (ref * c.double()).sum((0, 1, 2)), 1e-4)
    # fixed-order sums: two launches agree bit for bit
    _, part2, _ = ops.shuffle_relu_bwd(_bf(gy), _bf(c), co=_co(sc.cuda(), sh.cuda()))
    assert torch.equal(part, part2)


@pytest.mark.parametrize("cin,b,groups", [(24, 30, 1), (240, 60, 3), (480, 136, 4), (384, 96, 8), (192, 90, 3)])
def test_block_diagonal_group_conv1(cin, b, groups):
    """group_conv1 as a dense GEMM on the shuffle-permuted, padded block-diagonal operand: forward == shuffle_channels of
    F.conv2d(groups=g) with zero pad channels; dgrad == F.conv2d's input gradient; the gathered dense wgrad == its weight
    gradient"""
    from deeplearning_b200 import ops
    from deeplearning_b200.classification.ShuffleNet.models.shufflenetv1 import shuffle_channels
    from deeplearning_b200.engine import shufflenet as eng

    conv = torch.nn.Conv2d(cin, b, 1, groups=groups, bias=False)
    bp = (b + 7) // 8 * 8
    gc = eng._GroupedConv(conv, eng.shuffle_order(b, groups), bp, cin, "cuda")
    gc.w = conv.weight.data.cuda()
    wf, wd = gc.operands()
    gen = torch.Generator().manual_seed(cin + b)
    x = torch.randn(2, 6, 5, cin, generator=gen).to(BF16).float()
    c, _ = ops.conv2d_fwd(_bf(x), wf, 1, 1)
    wq = conv.weight.detach().to(BF16).double()
    ref = shuffle_channels(F.conv2d(x.double().permute(0, 3, 1, 2), wq, groups=groups), groups).permute(0, 2, 3, 1)
    _close(c[..., :b].float(), ref)
    assert torch.equal(c[..., b:].float().cpu(), torch.zeros(2, 6, 5, bp - b))
    dy = torch.randn(2, 6, 5, bp, generator=gen)
    dy[..., b:] = 0
    dy = dy.to(BF16).float()
    # dy in stored (shuffled) order is the gradient of shuffle_channels(conv(x))
    xd = x.double().permute(0, 3, 1, 2).requires_grad_()
    wdd = wq.clone().requires_grad_()
    out = shuffle_channels(F.conv2d(xd, wdd, groups=groups), groups)
    gx_ref, gw_ref = torch.autograd.grad(out, (xd, wdd), dy[..., :b].double().permute(0, 3, 1, 2))
    dx = ops.conv2d_dgrad(_bf(dy), wd, (6, 5), 1, 1)
    _close(dx.float(), gx_ref.permute(0, 2, 3, 1))
    dense = ops.conv2d_wgrad(_bf(dy), _bf(x), 1, 1)
    _close(gc.weight_grad(dense), gw_ref, 1e-3)


@pytest.mark.parametrize("b,cout,groups", [(60, 240, 3), (90, 360, 1), (136, 544, 4), (96, 384, 8)])
def test_block_diagonal_group_conv(b, cout, groups):
    """group_conv (bottleneck -> block output) on the block-diagonal operand with zero pad columns"""
    from deeplearning_b200 import ops
    from deeplearning_b200.engine import shufflenet as eng

    conv = torch.nn.Conv2d(b, cout, 1, groups=groups, bias=False)
    bp = (b + 7) // 8 * 8
    gc = eng._GroupedConv(conv, list(range(cout)), cout, bp, "cuda")
    gc.w = conv.weight.data.cuda()
    wf, wd = gc.operands()
    gen = torch.Generator().manual_seed(b + cout)
    a = torch.randn(2, 4, 7, bp, generator=gen)
    a[..., b:] = 0
    a = a.to(BF16).float()
    c, _ = ops.conv2d_fwd(_bf(a), wf, 1, 1)
    wq = conv.weight.detach().to(BF16).double()
    ad = a[..., :b].double().permute(0, 3, 1, 2).requires_grad_()
    out = F.conv2d(ad, wq, groups=groups)
    _close(c.float(), out.detach().permute(0, 2, 3, 1))
    dy = torch.randn(2, 4, 7, cout, generator=gen).to(BF16).float()
    wdd = wq.clone().requires_grad_()
    ga, gw = torch.autograd.grad(F.conv2d(ad, wdd, groups=groups), (ad, wdd), dy.double().permute(0, 3, 1, 2))
    da = ops.conv2d_dgrad(_bf(dy), wd, (4, 7), 1, 1)
    _close(da[..., :b].float(), ga.permute(0, 2, 3, 1))
    assert torch.equal(da[..., b:].float().cpu(), torch.zeros(2, 4, 7, bp - b))
    _close(gc.weight_grad(ops.conv2d_wgrad(_bf(dy), _bf(a), 1, 1)), gw, 1e-3)
