"""SupCon training end to end on the GPU engine, against the fp32 oracle (oracle/supcon.py) on the same weights and inputs,
with PyTorch's own bf16 autocast run of the oracle as the measure of what bf16 storage costs: stage-1 train steps of
resnet18 and resnet50 at 224 px, the reference loop (model(cat) -> split -> cat(unsqueeze) -> SupConLoss -> SGD) against
TrainStep, CUDA-graph capture, the uint8 input path, eval embeddings with the projection head on and off, and the
second stage on a frozen encoder."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(backbone="resnet18", seed=0, **kw):
    from deeplearning_b200.self_supervised.SupCon.models.model import SupConModel

    torch.manual_seed(seed)
    m = SupConModel(backbone, **kw)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _views(B, px=224, seed=1):
    return torch.randn(2 * B, 3, px, px, generator=torch.Generator().manual_seed(seed)).cuda()


def _oracle(state, x, y, tau):
    """fp32 and bf16-autocast oracle steps on the GPU (TF32 off): (emb32, loss32, grads32, state32 after the step,
    max |emb_ac - emb32|, |loss_ac - loss32|, {name: rel-L2 of autocast's gradient, or of its running mean})."""
    from oracle.supcon import train_step_grads

    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    outs = []
    try:
        for amp in (False, True):
            s = {k: v.clone().cuda() for k, v in state.items()}
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                emb, loss, grads = train_step_grads(s, x, y, tau)
            outs.append((emb.float(), float(loss), {k: g.float() for k, g in grads.items()}, s))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    (e32, l32, g32, s32), (eac, lac, gac, sac) = outs
    gerr = {n: float((gac[n] - g32[n]).norm() / (g32[n].norm() + 1e-12)) for n in g32}
    gerr.update({k: _rel(sac[k], s32[k]) for k in s32 if "running_mean" in k})
    return e32, l32, g32, s32, float((eac - e32).abs().max()), abs(lac - l32), gerr


def _rel(a, ref):
    return float((a.float() - ref.float()).norm() / (ref.float().norm() + 1e-12))


@pytest.mark.parametrize("backbone,B", [("resnet18", 16), ("resnet50", 16)])
def test_stage1_train_step_against_oracle(backbone, B):
    from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss

    m, state = _model(backbone)
    m = m.cuda().train()
    x = _views(B)
    y = torch.randint(0, 4, (B,), generator=torch.Generator().manual_seed(2)).cuda()
    emb = m(x)
    f1, f2 = torch.split(emb, [B, B], dim=0)
    loss = SupConLoss(temperature=0.1)(torch.cat([f1.unsqueeze(1), f2.unsqueeze(1)], dim=1), y)
    loss.backward()
    torch.cuda.synchronize()
    assert emb.dtype == torch.float32 and emb.shape == (2 * B, 128)
    e32, l32, g32, s32, d_ac, l_ac, g_ac = _oracle(state, x, y, 0.1)
    d = float((emb.detach() - e32).abs().max())
    assert d <= max(2.0 * d_ac, 0.02), (d, d_ac)
    assert abs(float(loss.detach()) - l32) <= max(2.0 * l_ac, 1e-2 * l32), (float(loss), l32, l_ac)
    for n, p in m.named_parameters():
        r = g32[n]
        rel = float((p.grad - r).norm() / (r.norm() + 1e-12))
        assert rel <= max(3.0 * g_ac[n], 0.03), (n, rel, g_ac[n])
    for k, v in m.state_dict().items():
        if "running_mean" in k:
            rel = _rel(v, s32[k])
            assert rel <= max(3.0 * g_ac[k], 0.03), (k, rel, g_ac[k])


def _reference_loop_step(m, opt, x, y, crit):
    emb = m(x)
    B = x.shape[0] // 2
    f1, f2 = torch.split(emb, [B, B], dim=0)
    loss = crit(torch.cat([f1.unsqueeze(1), f2.unsqueeze(1)], dim=1), y)
    opt.zero_grad()
    loss.backward()
    opt.step()
    return loss.detach()


@pytest.mark.parametrize("labels", [True, False])
def test_reference_loop_matches_trainstep(labels):
    from deeplearning_b200.engine.trainer import TrainStep
    from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss

    B = 16
    a, _ = _model()
    b, _ = _model()
    a, b = a.cuda().train(), b.cuda().train()
    crit = SupConLoss(temperature=0.1)
    opt = torch.optim.SGD(a.parameters(), lr=0.1)
    step = TrainStep(b, lr=0.1, momentum=0.0, weight_decay=0.0, criterion=SupConLoss(temperature=0.1))
    for i in range(3):
        x = _views(B, seed=10 + i)
        y = torch.randint(0, 4, (B,), generator=torch.Generator().manual_seed(20 + i)).cuda() if labels else None
        la = _reference_loop_step(a, opt, x, y, crit)
        lb, correct = step.step(x, y)
        assert correct is None
        assert abs(float(la) - float(lb)) <= 1e-4 * abs(float(la)), (i, float(la), float(lb))
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        if sa[k].is_floating_point():
            assert torch.allclose(sa[k], sb[k], rtol=1e-3, atol=1e-5), k


def test_trainstep_ratio_check():
    from deeplearning_b200.engine.trainer import TrainStep
    from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss

    m, _ = _model()
    step = TrainStep(m.cuda(), lr=0.1, momentum=0.0, weight_decay=0.0, criterion=SupConLoss(0.1))
    with pytest.raises(ValueError, match="two views"):
        step.step(_views(4, px=64), torch.zeros(3, dtype=torch.long, device="cuda"))


def test_graph_capture_matches_eager_and_uint8_input():
    from deeplearning_b200.engine.trainer import TrainStep
    from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss

    B = 16
    a, _ = _model()
    b, _ = _model()
    a, b = a.cuda().train(), b.cuda().train()
    sa = TrainStep(a, lr=0.1, momentum=0.0, weight_decay=0.0, criterion=SupConLoss(0.1))
    sb = TrainStep(b, lr=0.1, momentum=0.0, weight_decay=0.0, criterion=SupConLoss(0.1))
    xs = [_views(B, seed=30 + i) for i in range(2)]
    ys = [torch.randint(0, 4, (B,), generator=torch.Generator().manual_seed(40 + i)).cuda() for i in range(2)]
    sb.capture(xs[0], ys[0])
    for x, y in zip(xs, ys):
        la, _ = sa.step_eager(x, y)
        lb, _ = sb.step(x, y)
        assert torch.equal(la, lb)
    for (k, va), vb in zip(a.state_dict().items(), b.state_dict().values()):
        assert torch.equal(va, vb), k
    # uint8 NHWC input: ToTensor + Normalize fused into the stem, against the fp32 batch the reference's transform makes
    u8 = torch.randint(0, 256, (2 * B, 224, 224, 3), dtype=torch.uint8, device="cuda")
    mean = torch.tensor([0.485, 0.456, 0.406], device="cuda").view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], device="cuda").view(1, 3, 1, 1)
    xf = (u8.permute(0, 3, 1, 2).float() / 255.0 - mean) / std
    a.eval()
    with torch.no_grad():
        e8, ef = a(u8), a(xf)
    assert float((e8 - ef).abs().max()) <= 2e-2


@pytest.mark.parametrize("head", [True, False])
def test_eval_embeddings_against_oracle(head):
    from oracle.supcon import supcon_forward

    m, state = _model("resnet50")
    m = m.cuda().eval()
    m.use_projection_head(head)
    x = _views(4)
    with torch.no_grad():
        e = m(x)
        ref = supcon_forward({k: v.cuda() for k, v in state.items()}, x, False, projection_head=head)
    assert e.shape == (8, 128 if head else 2048)
    assert float((e - ref).abs().max()) <= 2e-2 * float(ref.abs().max())
    assert torch.allclose(e.norm(dim=1), torch.ones(8, device="cuda"), atol=1e-5)


def test_stage2_trains_the_classifier_on_a_frozen_encoder():
    from deeplearning_b200.engine.trainer import TrainStep
    from deeplearning_b200.self_supervised.SupCon.losses.LabelSmooth import LabelSmoothingLoss
    from oracle.supcon import label_smoothing_loss, supcon_forward

    m, state = _model(second_stage=True, num_classes=10)
    m = m.cuda().train()
    B = 20
    x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda()
    y = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(4)).cuda()
    step = TrainStep(m, lr=0.01, momentum=0.0, weight_decay=0.0, criterion=LabelSmoothingLoss(10, 0.01))
    before = {k: v.clone() for k, v in m.state_dict().items()}
    loss, correct = step.step(x, y)
    torch.cuda.synchronize()
    assert correct is not None and correct.shape == (B,)
    s = {k: v.cuda() for k, v in state.items()}
    logits = supcon_forward(s, x, True)
    ref_loss = float(label_smoothing_loss(logits, y, 10, 0.01))
    assert abs(float(loss) - ref_loss) <= 1e-2 * ref_loss, (float(loss), ref_loss)
    after = m.state_dict()
    for k, v in after.items():
        if k.startswith("classifier."):
            assert not torch.equal(v, before[k]), k
        elif "running_" in k or "num_batches" in k:
            assert torch.allclose(v, s[k], rtol=2e-2, atol=2e-3), k
            assert not torch.equal(v, before[k]) or "num_batches" in k, k
        else:
            assert torch.equal(v, before[k]), k
    # the LabelSmoothingLoss module: value and logit gradient against the oracle's formula
    lg = (torch.randn(B, 10, device="cuda") * 3).requires_grad_(True)
    lo = LabelSmoothingLoss(10, 0.1)(lg, y)
    lo.backward()
    lr = lg.detach().double().requires_grad_(True)
    ref = label_smoothing_loss(lr, y, 10, 0.1)
    ref.backward()
    assert abs(float(lo.detach()) - float(ref.detach())) <= 1e-5 * abs(float(ref.detach()))
    assert float((lg.grad.double() - lr.grad).norm() / lr.grad.norm()) <= 1e-2
