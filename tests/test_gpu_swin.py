"""End-to-end parity of the GPU Swin-T path against the CPU oracle (fp32) on the same weights and inputs, plus the
kernels/window_process drop-in (SURVEY seam B2) against its torch definition (the reference's own unit_test.py protocol)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _build(depths=(2, 2, 6, 2), num_classes=1000, seed=0, embed_dim=96, num_heads=(3, 6, 12, 24)):
    from deeplearning_b200.classification.swin_transformer.models.swin_transformer import SwinTransformer

    torch.manual_seed(seed)
    m = SwinTransformer(embed_dim=embed_dim, depths=list(depths), num_heads=list(num_heads)[:len(depths)],
                        num_classes=num_classes, drop_path_rate=0.0)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    return m.cuda(), state


def _randomize(m, state, seed=5):
    """trunc_normal(std .02) + zero biases makes every block a near no-op: perturb so that all layers (and the relative
    position bias) matter."""
    g = torch.Generator().manual_seed(seed)
    for k, v in state.items():
        if "relative_position_index" in k or "attn_mask" in k:
            continue
        if "relative_position_bias_table" in k:
            state[k] = v + torch.randn(v.shape, generator=g) * 0.5
        elif v.dim() >= 2:
            state[k] = v + torch.randn(v.shape, generator=g) * (0.5 / v.shape[-1] ** 0.5 if v.dim() == 2 else 0.02)
        elif "bias" in k:
            state[k] = v + torch.randn(v.shape, generator=g) * 0.02
        elif "norm" in k and "weight" in k:
            state[k] = v + torch.randn(v.shape, generator=g) * 0.05
    m.load_state_dict(state)


@pytest.mark.parametrize("randomize", [False, True])
def test_swin_tiny_eval_logits_parity(randomize):
    from oracle.swin import swin_forward

    m, state = _build()
    if randomize:
        _randomize(m, state)
    m.eval()
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = swin_forward(state, x)
        got = m(x.cuda()).float().cpu()
    err = float((got - ref).abs().max())
    print(f"Swin-T eval logits max-abs err {err:.4g} (|ref| max {float(ref.abs().max()):.3g}, randomized={randomize})")
    assert err <= 1e-2 * max(1.0, float(ref.abs().max()))  # north_star: 1e-2 for bf16


@pytest.mark.parametrize("depths,randomize", [((2, 2), True), ((2, 2, 6, 2), False), ((2, 2, 6, 2), True)])
def test_swin_train_step_parity(depths, randomize):
    _train_step_parity(depths, randomize)


def test_swin_base_widths_train_step_parity():
    """Swin-B widths (embed 128, heads 4/8/16/32: LayerNorm up to 1024, patch merges up to 4C = 2048), one block per
    stage - the kernel shapes depend only on the widths."""
    _train_step_parity((1, 1, 1, 1), True, embed_dim=128, num_heads=(4, 8, 16, 32))


def _train_step_parity(depths, randomize, embed_dim=96, num_heads=(3, 6, 12, 24)):
    from oracle.swin import train_step_grads

    m, state = _build(depths=depths, embed_dim=embed_dim, num_heads=num_heads)
    if randomize:
        _randomize(m, state)
    m.train()
    B = 4
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    ref_logits, ref_loss, ref_grads = train_step_grads(state, x, y, depths=depths, num_heads=tuple(num_heads)[:len(depths)])
    out = m(x.cuda())
    loss = F.cross_entropy(out, y.cuda())
    loss.backward()
    err = float((out.detach().float().cpu() - ref_logits).abs().max())
    print(f"depths {depths} embed {embed_dim} rand={randomize}: train logits err {err:.4g} (|ref| max {float(ref_logits.abs().max()):.3g}); "
          f"loss {float(loss.detach()):.5f} vs {float(ref_loss):.5f}")
    assert err <= 1e-2 * max(1.0, float(ref_logits.abs().max()))
    assert abs(float(loss.detach()) - float(ref_loss)) < 1e-2
    worst = (0.0, "")
    for name, p in m.named_parameters():
        assert p.grad is not None, name
        g, r = p.grad.float().cpu(), ref_grads[name]
        rel = float((g - r).norm() / (r.norm() + 1e-9))
        worst = max(worst, (rel, name))
        assert rel < 0.05, f"{name}: grad rel-L2 error {rel:.3g}"
    print(f"worst grad rel-L2 error {worst[0]:.3g} at {worst[1]}")


def test_swin_small_head_and_cpu_raises():
    m, _ = _build(depths=(1, 1), num_classes=5)
    m.train()
    out = m(torch.randn(2, 3, 224, 224, device="cuda"))
    assert out.shape == (2, 5)
    out.sum().backward()
    assert m.head.weight.grad.shape == (5, 192)
    assert m.layers[0].blocks[0].attn.relative_position_bias_table.grad.shape == (169, 3)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 3, 224, 224))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_window_process_dropin_matches_torch(dtype):
    """Same protocol as the reference's kernels/window_process/unit_test.py: forward and backward of both Functions against
    roll + window_partition / window_reverse + roll in torch, exact (pure permutations)."""
    from deeplearning_b200.classification.swin_transformer.kernels.window_process.window_process import (WindowProcess,
                                                                                                        WindowProcessReverse)
    from deeplearning_b200.classification.swin_transformer.models.swin_transformer import window_partition, window_reverse

    B, H, W, C, shift, ws = 24, 56, 56, 96, 2, 7
    nW = (H // ws) * (W // ws)
    x = torch.randn(B, H, W, C, device="cuda").to(dtype)
    x1 = x.clone().requires_grad_(True)
    x2 = x.clone().requires_grad_(True)
    ref = window_partition(torch.roll(x1, shifts=(-shift, -shift), dims=(1, 2)), ws)
    got = WindowProcess.apply(x2, B, H, W, C, -shift, ws)
    assert torch.equal(ref, got)
    gout = torch.randn_like(ref)
    ref.backward(gout)
    got.backward(gout)
    assert torch.equal(x1.grad, x2.grad)
    w = torch.randn(B * nW, ws, ws, C, device="cuda").to(dtype)
    w1 = w.clone().requires_grad_(True)
    w2 = w.clone().requires_grad_(True)
    ref = torch.roll(window_reverse(w1, ws, H, W), shifts=(shift, shift), dims=(1, 2))
    got = WindowProcessReverse.apply(w2, B, H, W, C, shift, ws)
    assert torch.equal(ref, got)
    gout = torch.randn_like(ref)
    ref.backward(gout)
    got.backward(gout)
    assert torch.equal(w1.grad, w2.grad)
