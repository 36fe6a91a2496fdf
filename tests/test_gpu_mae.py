"""MAE pre-training end to end on the GPU engine, against the fp32 oracle (oracle/mae.py) fed the engine's shuffle on the
same weights and inputs, with PyTorch's own bf16 autocast run of the oracle as the measure of what bf16 storage costs:
train steps of both train.py configurations at 224 px, the reference's mask draw and generator state, the reference loop
(F.mse_loss + torch.optim.AdamW) against TrainStep, CUDA-graph capture, the uint8 input path and a bs 256 step."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PRETRAIN = dict(image_size=224, patch_size=16, encoer_dim=768, mlp_dim=1024, encoder_depth=12, num_encoder_head=12,
                dim_per_head=64, decoder_dim=512, decoder_depth=8, num_decoder_head=16, mask_ratio=0.75)
BRANCH = dict(image_size=224, patch_size=16, encoer_dim=512, mlp_dim=1024, encoder_depth=6, num_encoder_head=8,
              dim_per_head=64, decoder_dim=512, decoder_depth=6, num_decoder_head=8, mask_ratio=0.75)   # Identity enc_to_dec
SMALL = dict(image_size=64, patch_size=16, encoer_dim=128, mlp_dim=256, encoder_depth=2, num_encoder_head=2,
             dim_per_head=64, decoder_dim=64, decoder_depth=2, num_decoder_head=2, mask_ratio=0.75)
UNUSED = ("encoder.cls_token", "encoder.mlp_head.")


def _model(cfg, seed=0):
    from deeplearning_b200.self_supervised.MAE.models.MAE import MAEVisonTransformer

    torch.manual_seed(seed)
    m = MAEVisonTransformer(**cfg)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _draw(B, P, seed):
    """The engine's shuffle for a forward run right after torch.cuda.manual_seed(seed): the reference's torch.rand draw,
    sorted stably."""
    torch.cuda.manual_seed(seed)
    return torch.rand(B, P, device="cuda").argsort(dim=1, stable=True)


def _oracle(state, x, shuffle, cfg):
    """fp32 and bf16-autocast oracle runs on the GPU (TF32 off): (pred32, grads32, max |pred_ac - pred32|, grad rel-L2)."""
    from oracle.mae import mae_forward

    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    preds, grads = [], []
    try:
        for amp in (False, True):
            s = {k: v.clone().cuda().requires_grad_() for k, v in state.items()}
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                pred, mp = mae_forward(s, x.cuda(), shuffle, cfg["patch_size"], cfg["num_encoder_head"],
                                       cfg["num_decoder_head"], cfg["mask_ratio"])
            pred = pred.float()
            F.mse_loss(pred, mp).backward()
            preds.append((pred.detach(), mp))
            grads.append({k: v.grad for k, v in s.items() if v.grad is not None})
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    gerr = {n: float((grads[1][n] - grads[0][n]).norm() / (grads[0][n].norm() + 1e-12)) for n in grads[0]}
    return preds[0], grads[0], float((preds[1][0] - preds[0][0]).abs().max()), gerr


@pytest.mark.parametrize("name", ["pretrain", "branch"])
def test_train_step_against_oracle(name):
    cfg = PRETRAIN if name == "pretrain" else BRANCH
    m, state = _model(cfg)
    m = m.cuda().train()
    B, P = 4, 196
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda()
    shuffle = _draw(B, P, 7)
    torch.cuda.manual_seed(7)
    pred, mp = m(x)
    loss = F.mse_loss(pred, mp)
    loss.backward()
    torch.cuda.synchronize()
    assert pred.dtype == torch.float32 and pred.requires_grad and not mp.requires_grad
    (ref_pred, ref_mp), ref_grads, d_ac, g_ac = _oracle(state, x, shuffle, cfg)
    assert torch.equal(mp, ref_mp)
    d = float((pred.detach() - ref_pred).abs().max())
    assert d <= max(2.0 * d_ac, 0.02 * float(ref_pred.abs().max())), (d, d_ac)
    ref_loss = float(F.mse_loss(ref_pred, ref_mp))
    assert abs(float(loss.detach()) - ref_loss) <= 1e-2 * ref_loss
    for n, p in m.named_parameters():
        if n.startswith(UNUSED):
            assert p.grad is None, n
            continue
        r = ref_grads[n]
        rel = float((p.grad - r).norm() / (r.norm() + 1e-12))
        assert rel <= max(3.0 * g_ac[n], 0.03), (n, rel, g_ac[n])


def test_masks_and_generator_state_follow_the_reference_draw():
    """MAE.forward draws torch.rand(b, P, device) where the reference does: same masks on a draw without ties, same
    generator state afterwards."""
    from deeplearning_b200.engine import mae as engine

    m, _ = _model(SMALL)
    m = m.cuda().train()
    x = torch.randn(8, 3, 64, 64, device="cuda")
    torch.cuda.manual_seed(11)
    keys = torch.rand(8, 16, device="cuda")
    assert keys.unique().numel() == keys.numel()
    ref_after = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(11)
    (_, mp, ids), _ = engine.forward(m, x, True, False)
    assert torch.equal(torch.cuda.get_rng_state(), ref_after)
    assert torch.equal(ids.long(), keys.argsort())
    patches = x.view(8, 3, 4, 16, 4, 16).permute(0, 2, 4, 3, 5, 1).reshape(8, 16, -1)
    assert torch.equal(mp, patches[torch.arange(8, device="cuda").unsqueeze(-1), keys.argsort()[:, :12]])


def test_reference_loop_with_adamw_matches_trainstep():
    from deeplearning_b200.engine.trainer import TrainStep

    m1, _ = _model(SMALL)
    m2, _ = _model(SMALL)
    m1, m2 = m1.cuda().train(), m2.cuda().train()
    init = {n: p.detach().clone() for n, p in m1.named_parameters()}
    step = TrainStep(m1, lr=1e-3, optimizer="adamw", betas=(0.9, 0.95), weight_decay=0.05, no_decay=lambda n, p: False)
    opt = torch.optim.AdamW(m2.parameters(), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.05)
    g = torch.Generator().manual_seed(3)
    for i in range(3):
        x = torch.randn(16, 3, 64, 64, generator=g).cuda()
        torch.cuda.manual_seed(100 + i)
        loss1, correct = step.step(x)
        torch.cuda.manual_seed(100 + i)
        opt.zero_grad()
        loss2 = F.mse_loss(*m2(x))
        loss2.backward()
        opt.step()
        assert correct is None
        assert abs(float(loss1) - float(loss2)) <= 1e-3 * float(loss2), (i, float(loss1), float(loss2))
    torch.cuda.synchronize()
    for (n, p1), (_, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        if n.startswith(UNUSED):
            assert torch.equal(p1.detach(), init[n]) and torch.equal(p2.detach(), init[n]), n
            assert p1.grad is None and p2.grad is None, n
            continue
        # AdamW's first steps move every element by about lr: compare the updates, which bf16 rounding of the loss
        # gradient can only perturb where a gradient element is near zero
        u1, u2 = p1.detach() - init[n], p2.detach() - init[n]
        rel = float((u1 - u2).norm() / (u2.norm() + 1e-12))
        assert rel <= 0.05, (n, rel)
    sd = step.optimizer_state_dict()
    names = [n for n, _ in m1.named_parameters()]
    assert all(not names[i].startswith(UNUSED) for i in sd["state"])


def test_captured_step_equals_eager_step():
    from deeplearning_b200.engine.trainer import TrainStep

    m1, _ = _model(SMALL)
    m2, _ = _model(SMALL)
    m1, m2 = m1.cuda().train(), m2.cuda().train()
    kw = dict(lr=1e-3, optimizer="adamw", betas=(0.9, 0.95), weight_decay=0.05, no_decay=lambda n, p: False)
    s1, s2 = TrainStep(m1, **kw), TrainStep(m2, **kw)
    x = torch.randn(16, 3, 64, 64, generator=torch.Generator().manual_seed(4)).cuda()
    s1.capture(x)
    for i in range(2):
        torch.cuda.manual_seed(50 + i)
        l1, _ = s1.step(x)
        torch.cuda.manual_seed(50 + i)
        l2, _ = s2.step_eager(x)
        torch.cuda.synchronize()
        assert torch.equal(l1, l2), (i, float(l1), float(l2))
    assert torch.equal(s1.arena.flat_p, s2.arena.flat_p)


def test_uint8_input_matches_normalised_float():
    from deeplearning_b200 import ops

    m, _ = _model(SMALL)
    m = m.cuda().eval()
    x8 = torch.randint(0, 256, (4, 64, 64, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).cuda()
    mean = torch.tensor(ops.IMAGENET_MEAN, device="cuda").view(1, 3, 1, 1)
    std = torch.tensor(ops.IMAGENET_STD, device="cuda").view(1, 3, 1, 1)
    xf = (x8.permute(0, 3, 1, 2).float() / 255.0 - mean) / std
    with torch.no_grad():
        torch.cuda.manual_seed(6)
        p8, t8 = m(x8)
        torch.cuda.manual_seed(6)
        pf, tf = m(xf)
    assert torch.allclose(t8, tf, rtol=1e-5, atol=1e-5)
    assert torch.allclose(p8, pf, rtol=1e-2, atol=1e-2)


def test_bs256_pretraining_step_is_finite():
    from deeplearning_b200.engine.trainer import TrainStep

    m, _ = _model(PRETRAIN)
    m = m.cuda().train()
    step = TrainStep(m, lr=1.5e-4, optimizer="adamw", betas=(0.9, 0.95), weight_decay=0.05, no_decay=lambda n, p: False)
    x = torch.randn(256, 3, 224, 224, device="cuda")
    loss, _ = step.step_eager(x)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all() and torch.isfinite(step.arena.flat_g).all()
    assert torch.isfinite(step.arena.flat_p).all()
