"""End-to-end parity of the GPU ViT path against the CPU oracle (fp32) on the same weights and inputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _build(depth=12, num_classes=1000, seed=0, patch=16, embed_dim=768, num_heads=12):
    from deeplearning_b200.classification.vision_transformer.vit_model import VisionTransformer

    torch.manual_seed(seed)
    m = VisionTransformer(img_size=224, patch_size=patch, embed_dim=embed_dim, depth=depth, num_heads=num_heads,
                          num_classes=num_classes)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    return m.cuda(), state


def _randomize(m, state, seed=5):
    """The reference init (trunc_normal std .01, zero biases) makes every block a near no-op; perturb the weights so that
    parity is tested on a network whose layers all matter."""
    g = torch.Generator().manual_seed(seed)
    for k, v in state.items():
        if v.dim() >= 2 and "pos_embed" not in k and "cls_token" not in k:
            state[k] = v + torch.randn(v.shape, generator=g) * (0.5 / v.shape[-1] ** 0.5 if v.dim() == 2 else 0.02)
        elif "bias" in k:
            state[k] = v + torch.randn(v.shape, generator=g) * 0.02
        elif "norm" in k and "weight" in k:
            state[k] = v + torch.randn(v.shape, generator=g) * 0.05
    m.load_state_dict(state)


@pytest.mark.parametrize("randomize", [False, True])
def test_vit_b16_eval_logits_parity(randomize):
    from oracle.vit import vit_forward

    m, state = _build()
    if randomize:
        _randomize(m, state)
    m.eval()
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = vit_forward(state, x)
        got = m(x.cuda()).float().cpu()
    err = float((got - ref).abs().max())
    print(f"ViT-B/16 eval logits max-abs err {err:.4g} (|ref| max {float(ref.abs().max()):.3g}, randomized={randomize})")
    assert err <= 1e-2 * max(1.0, float(ref.abs().max()))  # north_star: 1e-2 for bf16


@pytest.mark.parametrize("depth,randomize", [(2, True), (12, False), (12, True)])
def test_vit_train_step_parity(depth, randomize):
    _train_step_parity(depth, randomize)


# ViT-L/16 (1024 wide, 16 heads: the 768 < C <= 1024 LayerNorm backward) and ViT-B/32 (50 tokens); the kernel shapes
# depend only on the widths, so two blocks are enough
@pytest.mark.parametrize("patch,embed_dim,num_heads", [(16, 1024, 16), (32, 768, 12)])
def test_vit_wide_and_patch32_train_step_parity(patch, embed_dim, num_heads):
    _train_step_parity(2, True, patch=patch, embed_dim=embed_dim, num_heads=num_heads)


def _train_step_parity(depth, randomize, **arch):
    from oracle.vit import train_step_grads

    m, state = _build(depth=depth, **arch)
    if randomize:
        _randomize(m, state)
    m.train()
    B = 8
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    kw = {k: arch[k] for k in ("patch", "num_heads") if k in arch}
    ref_logits, ref_loss, ref_grads = train_step_grads(state, x, y, **kw)
    out = m(x.cuda())
    loss = F.cross_entropy(out, y.cuda())
    loss.backward()
    err = float((out.detach().float().cpu() - ref_logits).abs().max())
    print(f"depth {depth} {arch} rand={randomize}: train logits err {err:.4g} (|ref| max {float(ref_logits.abs().max()):.3g}); loss {float(loss.detach()):.5f} vs {float(ref_loss):.5f}")
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


def test_vit_small_head_and_cpu_raises():
    m, _ = _build(depth=1, num_classes=5)
    m.train()
    out = m(torch.randn(2, 3, 224, 224, device="cuda"))
    assert out.shape == (2, 5)
    out.sum().backward()
    assert m.head.weight.grad.shape == (5, 768)
    assert m.cls_token.grad.shape == (1, 1, 768) and m.pos_embed.grad.shape == (1, 197, 768)
    with pytest.raises(RuntimeError):
        m(torch.randn(1, 3, 224, 224))
