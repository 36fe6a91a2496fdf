"""Stochastic depth (drop_path) and ViT pre_logits on the GPU engines, against the CPU oracle with SHARED per-sample masks
(SURVEY.md 7.3): the reference's default constructors - convnext_tiny() (rate 0.2), SwinTransformer() (0.1),
vit_base_patch16_224_in21k() (has_logits=True) - train on the drop-in without raising."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _masks(probs, per_block, batch, seed):
    """(engine multipliers r/keep, oracle entries (r, keep)) for blocks with the given drop probabilities."""
    scales, entries, i = [], [], 0
    for p in probs:
        for _ in range(per_block):
            if p and p > 0:
                keep = 1.0 - p
                r = (keep + torch.rand(batch, generator=torch.Generator().manual_seed(seed + i))).floor()
                i += 1
                scales.append((r / keep).float())
                entries.append((r, keep))
            else:
                entries.append(None)
    return scales, entries


def _rel(a, b):
    return float((a.float().cpu() - b.float()).norm() / (b.float().norm() + 1e-12))


def _check(model, state, x, y, scales, entries, oracle_grads, tol_logits, what):
    from deeplearning_b200.engine import droppath

    model = model.cuda().train()
    with droppath.replay(scales):
        out = model(x.cuda())
        loss = F.cross_entropy(out, y.cuda())
        loss.backward()
    torch.cuda.synchronize()
    ref_logits, ref_loss, ref_grads = oracle_grads(state, x, y, drop=entries)
    err = float((out.detach().float().cpu() - ref_logits).abs().max())
    scale = max(1.0, float(ref_logits.abs().max()))
    assert err <= tol_logits * scale, f"{what}: logits max abs err {err:.4g} (|logit|max {scale:.3g})"
    assert abs(float(loss.detach()) - float(ref_loss)) < 2e-2, (what, float(loss.detach()), float(ref_loss))
    bad = []
    for n, p in model.named_parameters():
        r = _rel(p.grad, ref_grads[n])
        if r > 0.08 and float(ref_grads[n].norm()) > 1e-6:
            bad.append((n, round(r, 4)))
    assert not bad, f"{what}: gradient rel-L2 above 8 %: {bad[:6]}"
    return err


def test_convnext_default_ctor_trains_with_droppath():
    from deeplearning_b200.classification.convNext.models.networks import convnext_tiny
    from oracle.convnext import train_step_grads

    torch.manual_seed(0)
    m = convnext_tiny(1000)                      # drop_path_rate 0.2 hard-coded, as in the reference (networks.py:178)
    # SURVEY D5: the reference init (std 0.2) drives |logit| to ~20 where bf16 cannot hold 1e-2 abs; re-init at std 0.02
    g = torch.Generator().manual_seed(7)
    state = {k: (torch.randn(v.shape, generator=g) * 0.02 if v.dim() >= 2 else v.clone()) for k, v in m.state_dict().items()}
    state = {k: (torch.full_like(v, 0.5) if k.endswith("gamma") else v) for k, v in state.items()}
    m.load_state_dict(state)
    B = 8
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    probs = [getattr(b.drop_path, "drop_prob", 0.0) for st in m.stages for b in st]
    scales, entries = _masks(probs, 1, B, 500)
    assert any(float(s.min()) == 0.0 for s in scales)
    _check(m, state, x, y, scales, entries, train_step_grads, 1e-2, "ConvNeXt-T drop_path 0.2")


def test_swin_default_ctor_trains_with_droppath():
    from deeplearning_b200.classification.swin_transformer.models.swin_transformer import SwinTransformer
    from oracle.swin import train_step_grads

    torch.manual_seed(0)
    m = SwinTransformer()                        # class default drop_path_rate 0.1
    state = {k: v.clone() for k, v in m.state_dict().items()}
    B = 8
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    probs = [getattr(b.drop_path, "drop_prob", 0.0) for l in m.layers for b in l.blocks]
    scales, entries = _masks(probs, 2, B, 600)
    assert any(float(s.min()) == 0.0 for s in scales)
    _check(m, state, x, y, scales, entries, train_step_grads, 1e-2, "Swin-T drop_path 0.1")


def test_vit_default_ctor_pre_logits_and_droppath():
    from deeplearning_b200.classification.vision_transformer.vit_model import VisionTransformer, vit_base_patch16_224_in21k
    from oracle.vit import train_step_grads, vit_forward

    # (1) the reference's default entry point: has_logits=True (Linear + Tanh pre_logits), eval + train
    torch.manual_seed(0)
    m = vit_base_patch16_224_in21k(num_classes=1000)      # has_logits=True is the constructor default (vit_model.py:290)
    assert m.has_logits
    state = {k: v.clone() for k, v in m.state_dict().items()}
    B = 4
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    m = m.cuda().eval()
    with torch.no_grad():
        out = m(x.cuda()).float().cpu()
        ref = vit_forward(state, x)
    err = float((out - ref).abs().max())
    assert err <= 1e-2 * max(1.0, float(ref.abs().max())), f"ViT pre_logits eval: {err}"
    _check(m, state, x, y, [], [None] * 24, train_step_grads, 1e-2, "ViT-B/16 pre_logits (train)")
    # (2) stochastic depth 0.1 on both branches of every block + pre_logits
    torch.manual_seed(0)
    m = VisionTransformer(img_size=224, patch_size=16, embed_dim=768, depth=12, num_heads=12, representation_size=768,
                          num_classes=1000, drop_path_ratio=0.1)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    probs = [getattr(b.drop_path, "drop_prob", 0.0) for b in m.blocks]
    scales, entries = _masks(probs, 2, B, 700)
    assert any(float(s.min()) == 0.0 for s in scales)
    _check(m, state, x, y, scales, entries, train_step_grads, 1e-2, "ViT-B/16 drop_path 0.1")


def test_droppath_draws_like_the_reference_and_survives_graph_capture():
    """Without the test hook the engine draws floor(keep + torch.rand(B,1,1)) per application from torch's CUDA generator
    (the reference's own call), and a captured training step redraws the masks on every replay."""
    from deeplearning_b200.classification.vision_transformer.vit_model import VisionTransformer
    from deeplearning_b200.engine import droppath
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    m = VisionTransformer(img_size=224, patch_size=16, embed_dim=768, depth=2, num_heads=12, num_classes=16,
                          drop_path_ratio=0.5).cuda().train()
    x = torch.randn(16, 3, 224, 224, device="cuda")
    torch.cuda.manual_seed(123)
    with droppath.record() as drawn:
        m(x)
    torch.cuda.manual_seed(123)
    expect = []
    for blk in m.blocks:
        p = getattr(blk.drop_path, "drop_prob", 0.0)
        for _ in range(2):
            if p > 0:
                keep = 1 - p
                expect.append(((keep + torch.rand((16, 1, 1), device="cuda")).floor_() / keep).view(-1))
    assert len(drawn) == len(expect) > 0
    for a, b in zip(drawn, expect):
        assert torch.equal(a, b)
    # graph replay: the losses of successive replays on the SAME batch differ because the masks are redrawn
    tr = TrainStep(m, lr=0.0, momentum=0.0, weight_decay=0.0)
    y = torch.randint(0, 16, (16,), device="cuda")
    tr.capture(x, y)
    losses = {round(float(tr.step(x, y)[0]), 6) for _ in range(4)}
    assert len(losses) > 1, losses
