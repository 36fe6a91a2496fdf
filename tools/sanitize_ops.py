"""One small launch of every wgmma / TMA kernel family, for `compute-sanitizer --tool {memcheck,racecheck,synccheck}`:
implicit-GEMM conv (forward + statistics, dgrad + residual, affine / mask epilogues, dual-source K), the streaming 1x1 kernel
(both modes), wgrad, ViT attention forward / backward, window attention forward / backward, BN-algebra kernels, the VGG passes, the ShuffleNet v1 passes, the ShuffleNet v2 tails.
usage: compute-sanitizer --tool racecheck python tools/sanitize_ops.py [family ...]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deeplearning_b200 import ops

dev = torch.device("cuda")
BF = torch.bfloat16
fam = set(sys.argv[1:]) or {"conv", "stream", "wgrad", "attn", "attn2", "ln", "wattn", "algebra", "vgg", "shufflenet",
                               "shufflenetv2"}


def r(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(BF)


if "conv" in fam:
    x = r(2, 16, 16, 64)
    w = torch.randn(128, 64, 3, 3, device=dev) * 0.05
    y, st = ops.conv2d_fwd(x, ops.pack_weight(w), 3, 1, want_stats=True)
    dx = ops.conv2d_dgrad(y, ops.pack_weight(w, 1), (16, 16), 3, 1, residual=x)
    w1 = torch.randn(64, 128, 1, 1, device=dev) * 0.05
    z = ops.gemm_dual(y, x, torch.randn(64, 192, device=dev).to(BF), torch.zeros(64, device=dev))
    print("conv ok", float(y.float().abs().mean()), float(dx.float().abs().mean()), float(z.float().abs().mean()))
    # round 2, late: resident-weight 64 -> 64 kernel (conv_tap64.cuh: forward with statistics, plain dgrad) and the dgrad /
    # dual-GEMM epilogue that masks with relu'(bn(x)) and sums dz, dz * x (kEpiBnMask)
    x64 = r(4, 16, 16, 64)
    w64 = torch.randn(64, 64, 3, 3, device=dev) * 0.05
    y64, st64 = ops.conv2d_fwd(x64, ops.pack_weight(w64), 3, 1, want_stats=True)
    d64 = ops.conv2d_dgrad(y64, ops.pack_weight(w64, 1), (16, 16), 3, 1)
    co = ops.bn_finalize(st64, 1024, torch.ones(64, device=dev), torch.zeros(64, device=dev), 1e-5, 0.1, None, None, None)
    dzm, sums = ops.conv2d_dgrad(y64, ops.pack_weight(w64, 1), (16, 16), 3, 1, bn_mask=(y64, co))
    dxm, dgm, dbm = ops.bn_backward_from_sums(dzm, sums, y64, co)
    zm, sums2 = ops.gemm_dual(y, x, torch.randn(64, 192, device=dev).to(BF), torch.zeros(64, device=dev), bn_mask=(x, co))
    print("tap64 / bn-mask ok", float(d64.float().abs().mean()), float(dxm.float().abs().mean()), float(zm.float().abs().mean()))
if "stream" in fam or "algebra" in fam:
    y2 = r(4, 16, 16, 64).relu_()
    w3 = torch.randn(256, 64, 1, 1, device=dev) * 0.1
    wp = ops.pack_weight(w3)
    ident = r(4, 16, 16, 256)
    G, s = ops.gram_colsum(y2)
    gamma, beta = torch.ones(256, device=dev), torch.zeros(256, device=dev)
    co = ops.bn_gram_stats(G, s, wp, 1024, gamma, beta, 1e-5, 0.1, None, None, None)
    out = ops.conv1x1_bn_act(y2, wp, co, ident)                      # streaming kernel, kStreamBnRelu (1024 pixels)
    w1 = torch.randn(64, 256, 1, 1, device=dev) * 0.05
    dz, stats = ops.conv1x1_dgrad_masked(r(4, 16, 16, 64), ops.pack_weight(w1, 1), residual=ident, mask_src=out)
    D = ops.conv2d_wgrad(dz, y2, 1, 1)
    dg, db, dW, wcat, wb = ops.bn_conv1x1_bwd(stats, D, G, s, wp, w3, 1024, gamma, co)
    g2 = ops.gemm_dual(dz, y2, wcat, wb)
    print("stream/algebra ok", float(out.float().abs().mean()), float(dz.float().abs().mean()), float(g2.float().abs().mean()))
if "wgrad" in fam:
    dy, x = r(2, 16, 16, 128), r(2, 16, 16, 64)
    print("wgrad ok", float(ops.conv2d_wgrad(dy, x, 3, 1).abs().mean()))
if "attn" in fam:
    qkv = r(2, 197, 3 * 2 * 64, scale=0.5)
    o, lse = ops.attention_fwd(qkv, 2, 0.125)
    dq = ops.attention_bwd(qkv, o, r(2, 197, 128), lse, 2, 0.125)
    print("attn ok", float(o.float().abs().mean()), float(dq.float().abs().mean()))
if "wattn" in fam:
    B, H, W, C, nH = 2, 14, 14, 96, 3
    qkv = r(B, H, W, 3 * C, scale=0.5)
    table = torch.randn(169, nH, device=dev) * 0.1
    coords = torch.stack(torch.meshgrid(torch.arange(7), torch.arange(7), indexing="ij")).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += 6
    rel[:, :, 1] += 6
    rel[:, :, 0] *= 13
    index = rel.sum(-1).to(dev)
    bias = ops.window_bias_gather(table, index, nH, None)
    o, lse = ops.window_attention_fwd(qkv, nH, bias, 0, 32 ** -0.5)
    dqkv, dbias = ops.window_attention_bwd(qkv, o, r(B, H, W, C), bias, lse, nH, 0, 32 ** -0.5)
    print("wattn ok", float(o.float().abs().mean()), float(dqkv.float().abs().mean()))
if "attn2" in fam:
    # persistent attention forward (attention_fwd2.cuh): 300 (batch, head) items on 132 CTAs, i.e. two or three items per CTA
    # (buffer reuse, barrier phases of the two query-block warpgroups), checked against PyTorch soft-max attention
    qkv = r(100, 197, 3 * 3 * 64, scale=0.5)
    o, lse = ops.attention_fwd(qkv, 3, 0.125)
    q, k, v = qkv[:2].float().view(2, 197, 3, 3, 64).permute(2, 0, 3, 1, 4)
    ref = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v
    err = (o[:2].float().view(2, 197, 3, 64).permute(0, 2, 1, 3) - ref).abs().max()
    print("attn2 ok", float(o.float().abs().mean()), "max|err|", float(err))
if "ln" in fam:
    # LayerNorm backward v2 (transformer.cuh): fp32 / bf16 rows with and without the residual-gradient operand
    for rows, C, dt in ((3000, 768, torch.float32), (5000, 96, torch.float32), (2000, 384, BF)):
        x = torch.randn(rows, C, device=dev).to(dt)
        g = torch.rand(C, device=dev) + 0.5
        y, mean, rstd = ops.layernorm_fwd(x, g, torch.zeros(C, device=dev), 1e-6)
        dx, dg, db = ops.layernorm_bwd(r(rows, C, scale=0.1), x, mean, rstd, g, add=r(rows, C, scale=0.1) if dt != BF else None)
        print("ln ok", rows, C, float(dx.float().abs().mean()), float(dg.abs().mean()))
if "vgg" in fam:
    # VGG passes (vgg.cuh): 2x2 pool forward / backward, plain and BatchNorm (odd H / W), adaptive 7x7 pool, dropout, Adam
    c = r(2, 9, 7, 128)
    co = ops.BnCoeffs(128, dev)
    co.scale.fill_(1.0), co.shift.fill_(0.1), co.mean.zero_(), co.invstd.fill_(1.0)
    for cc in (None, co):
        y, idx = ops.vgg_pool_fwd(c if cc is not None else torch.relu(c), cc)
        g = r(*y.shape)
        d = ops.vgg_pool_bwd(g, idx, (9, 7), y=y) if cc is None else ops.vgg_pool_bwd(g, idx, (9, 7), c=c, co=cc)[0]
    f = ops.vgg_avgpool7_fwd(r(2, 5, 9, 128))
    gx = ops.vgg_avgpool7_bwd(f, (2, 5, 9, 128))
    h = ops.vgg_dropout_fwd(r(4, 64), torch.full((4, 64), 2.0, device=dev))
    dh = ops.vgg_dropout_bwd(r(4, 64), h, 0.5)
    p, gg = torch.randn(1001, device=dev), torch.randn(1001, device=dev)
    ops.adam_(p, gg, torch.zeros_like(p), torch.zeros_like(p), torch.tensor([1e-3, 0, 0, 1, 1.0], device=dev), weight_decay=1e-3)
    print("vgg ok", float(d.float().abs().mean()), float(gx.float().abs().mean()), float(dh.float().abs().mean()))
if "shufflenet" in fam:
    # ShuffleNet passes (shufflenet.cuh, mbconv.cuh's ReLU mode): depthwise forward / dgrad / wgrad at a padded width,
    # the stride-2 tail forward and its backward with the pool half (odd H / W), the stride-1 and stem ReLU reduces
    c1 = r(2, 9, 7, 32)
    co = ops.BnCoeffs(32, dev)
    co.scale.fill_(1.0), co.shift.fill_(0.1), co.mean.zero_(), co.invstd.fill_(1.0)
    for s in (1, 2):
        d, _ = ops.dw_relu_fwd(c1, torch.randn(32, 1, 3, 3, device=dev), s, co, want_stats=True)
        dz, _ = ops.dw_relu_dgrad(r(*d.shape), torch.randn(32, 1, 3, 3, device=dev), c1, s, co)
        gw = ops.dw_relu_wgrad(r(*d.shape), c1, s, co)
    c3 = r(2, 5, 4, 40)
    co3 = ops.BnCoeffs(40, dev)
    co3.scale.fill_(1.0), co3.shift.fill_(0.1), co3.mean.zero_(), co3.invstd.fill_(1.0)
    y = ops.shuffle_tail_s2_fwd(r(2, 9, 7, 24), c3, co3)
    dz3, _, gx = ops.shuffle_relu_bwd(r(*y.shape), c3, y=y, in_hw=(9, 7))
    dz1, _, _ = ops.shuffle_relu_bwd(r(2, 9, 7, 32), c1, y=torch.relu(r(2, 9, 7, 32)))
    dzs, _, _ = ops.shuffle_relu_bwd(r(2, 9, 7, 32), c1, co=co)
    print("shufflenet ok", float(dz.float().abs().mean()), float(gw.abs().mean()), float(gx.float().abs().mean()))
if "shufflenetv2" in fam:
    # ShuffleNet v2 tails (shufflenet.cuh shufflev2_tail_*): all four modes at b = 58 (pitch 64, joined pitch 120, the
    # second half starting at the odd channel 29), forward and backward, joined and split gradients
    b, bp = 58, 64
    cos = []
    for _ in range(2):
        c = ops.BnCoeffs(bp, dev)
        c.scale.fill_(1.0), c.shift.fill_(0.1), c.mean.zero_(), c.invstd.fill_(1.0)
        cos.append(c)
    c3, u = r(2, 5, 3, bp), r(2, 5, 3, bp)
    for co_u in (None, cos[1]):
        for split in (False, True):
            y = ops.shufflev2_tail_fwd(u, c3, cos[0], b, co_u=co_u, split=split)
            g = tuple(r(*t.shape) for t in y) if split else r(*y.shape)
            dz3, _, du, _ = ops.shufflev2_tail_bwd(g, c3, cos[0], b, cu=None if co_u is None else u, co_u=co_u)
    print("shufflenetv2 ok", float(dz3.float().abs().mean()), float(du.float().abs().mean()))
torch.cuda.synchronize()
print("done")
