"""GPU parity tests of the ConvNeXt path: depthwise 7x7 kernels, 2x2/s2 convs, layer-scale bookkeeping, end-to-end net."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from deeplearning_b200 import ops

    return ops


def _rand(*shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


def _close(a, b, rtol, atol, what):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    bad = err > atol + rtol * b.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} bad, max abs err {float(err.max()):.4g} (ref max {float(b.abs().max()):.4g})"


@pytest.mark.parametrize("B,H,W,C", [(2, 56, 56, 96), (3, 28, 14, 192), (5, 14, 14, 384), (3, 7, 7, 768), (2, 14, 9, 192)])
def test_dwconv7_fwd_bwd(B, H, W, C):
    ops = _ops()
    x = _rand(B, H, W, C, seed=1, dtype=torch.float32)
    w = torch.randn(C, 1, 7, 7, device="cuda") * 0.1
    b = torch.randn(C, device="cuda") * 0.1
    wt = ops.dwconv7_pack(w)
    u = ops.dwconv7(x, wt, b)
    xr = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    wr, br = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, br, padding=3, groups=C)
    _close(u, ref.permute(0, 2, 3, 1), 1e-2, 1e-2, "dwconv fwd")
    du = _rand(B, H, W, C, seed=2)
    g = _rand(B, H, W, C, seed=3)
    gx, gw, gb = torch.autograd.grad(ref, (xr, wr, br), du.float().permute(0, 3, 1, 2))
    dx = ops.dwconv7(du, wt, add=g, out_dtype=torch.bfloat16, flip=True)
    _close(dx, gx.permute(0, 2, 3, 1) + g.float(), 1e-2, 2e-2, "dwconv bwd data (+add)")
    dw = ops.dwconv7_wgrad(du, x)
    sc = float(gw.abs().max())
    _close(dw / sc, gw / sc, 1e-3, 1e-3, "dwconv wgrad")
    _close(ops.colsum_tall(du.view(-1, C)), gb, 1e-3, 1e-2, "dwconv bias grad")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 56, 56, 96, 192), (2, 14, 14, 384, 768), (1, 8, 6, 64, 64)])
def test_conv2x2_stride2(B, H, W, Cin, Cout):
    ops = _ops()
    x = _rand(B, H, W, Cin, seed=1)
    w = _rand(Cout, Cin, 2, 2, seed=2, scale=(4 * Cin) ** -0.5)
    bias = torch.randn(Cout, device="cuda")
    y = ops.conv2d_fwd_f32(x, ops.pack_weight(w.float()), 2, 2, bias=bias)
    xr = x.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    wr = w.float().clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, bias, stride=2)
    _close(y, ref.permute(0, 2, 3, 1), 1e-3, 1e-2, "conv2x2 fwd (fp32 out)")
    dy = _rand(B, H // 2, W // 2, Cout, seed=3)
    gx, gw = torch.autograd.grad(ref, (xr, wr), dy.float().permute(0, 3, 1, 2))
    dx = ops.conv2d_dgrad(dy, ops.pack_weight(w.float(), mode=1), (H, W), 2, 2)
    _close(dx, gx.permute(0, 2, 3, 1), 1e-2, 2e-2, "conv2x2 dgrad")
    dw = ops.conv2d_wgrad(dy, x, 2, 2)
    sc = float(gw.abs().max())
    _close(dw / sc, gw / sc, 1e-3, 2e-3, "conv2x2 wgrad")


def test_layerscale_block_tail():
    """x' = x + gamma*(post W2^T + b2): forward epilogue and the gradient bookkeeping derived from the unscaled wgrad."""
    ops = _ops()
    M, C = 1000, 96
    post = _rand(M, 4 * C, seed=1)
    x = _rand(M, C, seed=2, dtype=torch.float32)
    W2 = (torch.randn(C, 4 * C, device="cuda") * 0.05)
    b2 = torch.randn(C, device="cuda") * 0.1
    gamma = torch.rand(C, device="cuda") + 0.5
    out, _ = ops.gemm(post, ops.pack_weight(W2), bias=b2, colscale=gamma, residual=x, out_f32=True)
    pr = post.float().requires_grad_(True)
    Wr, br, gr = W2.to(torch.bfloat16).float().requires_grad_(True), b2.clone().requires_grad_(True), gamma.clone().requires_grad_(True)
    ref = x + gr * (pr @ Wr.t() + br)
    _close(out, ref, 1e-3, 1e-2, "layer-scale epilogue")
    g = _rand(M, C, seed=3)
    gp, gW, gb, gg = torch.autograd.grad(ref, (pr, Wr, br, gr), g.float())
    gsum = ops.colsum_tall(g)
    G = ops.conv2d_wgrad(g.view(M, 1, 1, C), post.view(M, 1, 1, 4 * C)).view(C, 4 * C)
    dW2, db2, dgam = ops.layerscale_grads(G, Wr.detach(), b2, gsum, gamma)
    _close(dW2, gW, 2e-3, 2e-3 * float(gW.abs().max()), "dW2")
    _close(db2, gb, 2e-3, 2e-3 * float(gb.abs().max()), "db2")
    _close(dgam, gg, 5e-3, 5e-3 * float(gg.abs().max()), "dgamma")


def _build(depths=(3, 3, 9, 3), std=None, gamma_init=None, seed=0, dims=(96, 192, 384, 768)):
    from deeplearning_b200.classification.convNext.models.networks import ConvNeXt

    torch.manual_seed(seed)
    m = ConvNeXt(depths=list(depths), dims=list(dims), num_classes=1000, drop_path_rate=0.0)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    if std is not None:  # SURVEY D5: the reference init (std 0.2) gives |logit| ~ 20; also test a std 0.02 re-init
        g = torch.Generator().manual_seed(7)
        for k, v in state.items():
            if v.dim() >= 2:
                state[k] = torch.randn(v.shape, generator=g) * std
            elif k.endswith("gamma") and gamma_init is not None:
                state[k] = torch.full_like(v, gamma_init)
        m.load_state_dict(state)
    return m.cuda(), state


@pytest.mark.parametrize("std,gamma", [(None, None), (0.02, 0.5)])
def test_convnext_tiny_eval_parity(std, gamma):
    from oracle.convnext import convnext_forward

    m, state = _build(std=std, gamma_init=gamma)
    m.eval()
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = convnext_forward(state, x)
        got = m(x.cuda()).float().cpu()
    err = float((got - ref).abs().max())
    scale = float(ref.abs().max())
    print(f"ConvNeXt-T eval logits max-abs err {err:.4g} (|ref| max {scale:.3g}, init std {std})")
    assert err <= 1e-2 * max(1.0, scale)  # SURVEY D5: relative gate when the std=0.2 init inflates the logits


@pytest.mark.parametrize("depths,std,gamma", [((1, 1, 1, 1), 0.02, 0.5), ((3, 3, 9, 3), None, None), ((3, 3, 9, 3), 0.02, 0.5)])
def test_convnext_train_step_parity(depths, std, gamma):
    _train_step_parity(depths, std, gamma)


def test_convnext_base_widths_train_step_parity():
    """ConvNeXt-B widths (128 .. 1024: depthwise 7x7 and LayerNorm at 1024 channels), one block per stage - the kernel
    shapes depend only on the widths."""
    _train_step_parity((1, 1, 1, 1), 0.02, 0.5, dims=(128, 256, 512, 1024))


def _train_step_parity(depths, std, gamma, dims=(96, 192, 384, 768)):
    from oracle.convnext import train_step_grads

    m, state = _build(depths=depths, std=std, gamma_init=gamma, dims=dims)
    m.train()
    B = 8
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    ref_logits, ref_loss, ref_grads = train_step_grads(state, x, y)
    out = m(x.cuda())
    loss = F.cross_entropy(out, y.cuda())
    loss.backward()
    err = float((out.detach().float().cpu() - ref_logits).abs().max())
    scale = float(ref_logits.abs().max())
    print(f"depths {depths} dims {dims} std {std}: train logits err {err:.4g} (|ref| max {scale:.3g}); loss {float(loss.detach()):.4f} vs {float(ref_loss):.4f}")
    assert err <= 1e-2 * max(1.0, scale)
    assert abs(float(loss.detach()) - float(ref_loss)) <= 1e-2 * max(1.0, abs(float(ref_loss)))
    worst = (0.0, "")
    for name, p in m.named_parameters():
        assert p.grad is not None, name
        g, r = p.grad.float().cpu(), ref_grads[name]
        rel = float((g - r).norm() / (r.norm() + 1e-9))
        worst = max(worst, (rel, name))
        assert rel < 0.06, f"{name}: grad rel-L2 error {rel:.3g}"
    print(f"worst grad rel-L2 error {worst[0]:.3g} at {worst[1]}")


def test_convnext_tiny_default_ctor_runs_in_train_and_eval():
    """convnext_tiny(n) keeps the reference's hard-coded drop_path_rate 0.2 (:178) and trains (tests/test_gpu_droppath.py
    checks the numbers against the oracle with shared masks)."""
    from deeplearning_b200.classification.convNext.models.networks import convnext_tiny

    m = convnext_tiny(10).cuda().train()
    out = m(torch.randn(2, 3, 224, 224, device="cuda"))
    out.sum().backward()
    assert out.shape == (2, 10) and torch.isfinite(out).all() and torch.isfinite(m.head.weight.grad).all()
    m.eval()
    assert m(torch.randn(2, 3, 224, 224, device="cuda")).shape == (2, 10)
