"""ResNeXt (grouped 3x3 convolutions in every bottleneck) end to end on the GPU engine, against an fp32 CPU run of
torchvision's ResNet with the same groups / width on the same weights and inputs, with PyTorch's own bf16 autocast run as
the yardstick for what bf16 storage costs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

X32 = dict(groups=32, width_per_group=4)


def _tv(state, layers, kw):
    import torchvision

    ref = torchvision.models.ResNet(torchvision.models.resnet.Bottleneck, list(layers), **kw)
    ref.load_state_dict(state)
    return ref


def _oracle_train_step(state, x, labels, layers, kw):
    """fp32 CPU train step: (logits, loss, {param: grad}, state after the step's running-statistics update)"""
    ref = _tv(state, layers, kw).train()
    out = ref(x)
    loss = F.cross_entropy(out, labels)
    loss.backward()
    return out.detach(), loss.detach(), {n: p.grad for n, p in ref.named_parameters()}, ref.state_dict()


def _autocast_yardstick(state, x, train, labels, layers, kw):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    outs, grads = [], []
    for amp in (False, True):
        ref = _tv(state, layers, kw).cuda().train(train)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            with torch.set_grad_enabled(labels is not None):
                o = ref(x.cuda()).float()
        outs.append(o.detach())
        if labels is not None:
            F.cross_entropy(o, labels.cuda()).backward()
            grads.append({n: p.grad.detach().clone() for n, p in ref.named_parameters()})
    gerr = {}
    if labels is not None:
        gerr = {n: float((grads[1][n] - grads[0][n]).norm() / (grads[0][n].norm() + 1e-12)) for n in grads[0]}
    return float((outs[1] - outs[0]).abs().max()), gerr


def _model(layers, kw, seed=0):
    from deeplearning_b200.classification.resnet.models.networks import Bottleneck, ResNet

    torch.manual_seed(seed)
    m = ResNet(Bottleneck, list(layers), **kw)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _train_step_check(layers, B, hw, grad_slack, kw=X32):
    m, state = _model(layers, kw)
    m = m.cuda().train()
    x = torch.randn(B, 3, hw, hw, generator=torch.Generator().manual_seed(1))
    labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    ref_logits, ref_loss, ref_grads, ref_state = _oracle_train_step(state, x, labels, layers, kw)
    out = m(x.cuda())
    loss = F.cross_entropy(out, labels.cuda())
    loss.backward()
    err = float((out.detach().float().cpu() - ref_logits).abs().max())
    yard, gyard = _autocast_yardstick(state, x, True, labels, layers, kw)
    print(f"layers={layers}: train logits max-abs err {err:.4g} (torch-bf16 yardstick {yard:.4g}); loss "
          f"{float(loss.detach()):.5f} vs {float(ref_loss):.5f}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)
    assert abs(float(loss.detach()) - float(ref_loss)) <= 1e-2
    worst = (0.0, "")
    for name, p in m.named_parameters():
        g, r = p.grad.float().cpu(), ref_grads[name]
        assert g.shape == r.shape, name
        rel = float((g - r).norm() / (r.norm() + 1e-12))
        worst = max(worst, (rel / (gyard[name] + 1e-3), name))
        assert rel <= grad_slack * gyard[name] + 0.02, f"{name}: grad rel-L2 error {rel:.3g} vs torch-bf16 yardstick {gyard[name]:.3g}"
    print(f"worst grad error relative to the torch-bf16 yardstick: {worst[0]:.2f}x at {worst[1]}")
    sd = m.state_dict()
    shallow = sum(layers) <= 4
    for k in ref_state:
        if "running_" in k and (shallow or k.startswith(("bn1.", "layer1."))):
            assert torch.allclose(sd[k].cpu(), ref_state[k], rtol=2e-2, atol=2e-3), k
        if "num_batches" in k:
            assert int(sd[k]) == int(ref_state[k])


@pytest.mark.parametrize("algebra", ["0", "1"])
def test_resnext_shallow_train_step_parity(monkeypatch, algebra):
    """[1,1,1,1] ResNeXt 32x4d at bs 32, 128x128, on both bottleneck-tail schedules"""
    monkeypatch.setenv("B200_RESNET_ALGEBRA", algebra)
    _train_step_check((1, 1, 1, 1), 32, 128, grad_slack=2.0)


def test_resnext_shallow_odd_grid_train_step_parity():
    """196 px: the grouped 3x3/s2 and the downsample convolutions of layer2 .. layer4 read 49 x 49, 25 x 25 and 13 x 13 grids"""
    _train_step_check((1, 1, 1, 1), 32, 196, grad_slack=2.0)


def test_resnext50_train_step_parity():
    _train_step_check((3, 4, 6, 3), 64, 224, grad_slack=2.0)


@pytest.mark.parametrize("algebra", ["0", "1"])
def test_resnext50_eval_logits_parity(monkeypatch, algebra):
    """eval logits after calibrating the running statistics on one batch (momentum 1: running stats := batch stats)"""
    monkeypatch.setenv("B200_RESNET_ALGEBRA", algebra)
    layers = (3, 4, 6, 3)
    m, state = _model(layers, X32)
    ref = _tv(state, layers, X32)
    for mod in ref.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = 1.0
    with torch.no_grad():
        ref.train()(torch.randn(32, 3, 224, 224, generator=torch.Generator().manual_seed(3)))
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    m.load_state_dict(state)
    m = m.cuda().eval()
    x = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = ref.eval()(x)
        got = m(x.cuda()).float().cpu()
    err = float((got - want).abs().max())
    yard, _ = _autocast_yardstick(state, x, False, None, layers, X32)
    print(f"eval logits max-abs err {err:.4g} (|ref| max {float(want.abs().max()):.3g}); torch bf16 autocast: {yard:.4g}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)


@pytest.mark.parametrize("accum", [1, 2])
def test_resnext_trainstep_captured_equals_eager(accum):
    """CUDA-graph replay of the TrainStep reproduces eager stepping bit for bit (gradient accumulation included)"""
    from deeplearning_b200.engine.trainer import TrainStep

    a, _ = _model((1, 1, 1, 1), dict(X32, num_classes=16), seed=4)
    b, _ = _model((1, 1, 1, 1), dict(X32, num_classes=16), seed=4)
    a, b = a.cuda().train(), b.cuda().train()
    ta, tb = TrainStep(a, lr=0.02, accum_steps=accum), TrainStep(b, lr=0.02, accum_steps=accum)
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(8, 3, 64, 64, device="cuda", generator=g)
    y = torch.randint(0, 16, (8,), device="cuda", generator=g)
    tb.capture(x, y)
    for _ in range(2 * accum):
        la, _ = ta.step_eager(x, y)
        lb, _ = tb.step(x, y)
    assert ta.steps == tb.steps == 2
    assert float(la) == float(lb)
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(pa, pb), n
    for ba, bb in zip(a.buffers(), b.buffers()):
        assert torch.equal(ba, bb)


def test_resnext101_32x8d_step_has_finite_grads():
    """one train step of ResNeXt-101 32x8d (group width 8 .. 64, 256 .. 2048 grouped channels)"""
    from deeplearning_b200.classification.resnet.models.networks import resnext101_32x8d

    torch.manual_seed(0)
    m = resnext101_32x8d().cuda().train()
    x = torch.randn(8, 3, 128, 128, device="cuda")
    y = torch.randint(0, 1000, (8,), device="cuda")
    loss = F.cross_entropy(m(x), y)
    loss.backward()
    assert torch.isfinite(loss)
    for name, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and torch.isfinite(p.grad).all(), name
    assert m.layer4[0].conv2.weight.grad.shape == (2048, 64, 3, 3)
    assert float(m.layer4[0].conv2.weight.grad.abs().sum()) > 0
