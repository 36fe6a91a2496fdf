"""SE-ResNet (a squeeze-and-excitation gate in the tail of every block) end to end on the GPU engine, against an fp32 CPU run
of the in-tree yardstick (oracle/senet.py: the reference's SE blocks in torchvision's ResNet) on the same weights and
inputs, with PyTorch's own bf16 autocast run of the yardstick as the measure of what bf16 storage costs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _yard(state, layers, bottleneck, num_classes=1000):
    from oracle.senet import se_resnet_yardstick

    return se_resnet_yardstick(state, layers, bottleneck, num_classes)


def _oracle_train_step(state, x, labels, layers, bottleneck):
    """fp32 CPU train step: (logits, loss, {param: grad}, state after the step's running-statistics update)"""
    ref = _yard(state, layers, bottleneck).train()
    out = ref(x)
    loss = F.cross_entropy(out, labels)
    loss.backward()
    return out.detach(), loss.detach(), {n: p.grad for n, p in ref.named_parameters()}, ref.state_dict()


def _autocast_yardstick(state, x, train, labels, layers, bottleneck):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    outs, grads = [], []
    for amp in (False, True):
        ref = _yard(state, layers, bottleneck).cuda().train(train)
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


def _model(layers, bottleneck, seed=0, num_classes=1000):
    from deeplearning_b200.classification.resnet.models.networks import ResNet
    from deeplearning_b200.classification.seNet.models.se_resnet import SEBasicBlock, SEBottleneck

    torch.manual_seed(seed)
    m = ResNet(SEBottleneck if bottleneck else SEBasicBlock, list(layers), num_classes=num_classes)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _train_step_check(layers, B, hw, bottleneck=True, grad_slack=2.0):
    m, state = _model(layers, bottleneck)
    m = m.cuda().train()
    x = torch.randn(B, 3, hw, hw, generator=torch.Generator().manual_seed(1))
    labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    ref_logits, ref_loss, ref_grads, ref_state = _oracle_train_step(state, x, labels, layers, bottleneck)
    out = m(x.cuda())
    loss = F.cross_entropy(out, labels.cuda())
    loss.backward()
    err = float((out.detach().float().cpu() - ref_logits).abs().max())
    yard, gyard = _autocast_yardstick(state, x, True, labels, layers, bottleneck)
    print(f"layers={layers}: train logits max-abs err {err:.4g} (torch-bf16 yardstick {yard:.4g}); loss "
          f"{float(loss.detach()):.5f} vs {float(ref_loss):.5f}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)
    assert abs(float(loss.detach()) - float(ref_loss)) <= 1e-2
    worst = (0.0, "")
    names = [n for n, _ in m.named_parameters()]
    assert any(".se.fc.0." in n for n in names) and any(".se.fc.2." in n for n in names)
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
def test_senet_shallow_train_step_parity(monkeypatch, algebra):
    """[1,1,1,1] SE-bottleneck net at bs 32, 128x128: the SE tails and the downsample branches take the pass schedule
    under both settings, the other units keep theirs"""
    monkeypatch.setenv("B200_RESNET_ALGEBRA", algebra)
    _train_step_check((1, 1, 1, 1), 32, 128)


def test_senet_shallow_odd_grid_train_step_parity():
    """196 px: the stride-2 layers of layer2 .. layer4 read 49 x 49, 25 x 25 and 13 x 13 grids"""
    _train_step_check((1, 1, 1, 1), 32, 196)


def test_se_resnet50_train_step_parity():
    _train_step_check((3, 4, 6, 3), 64, 224)


def test_se_resnet18_train_step_parity():
    """SE basic blocks (se_resnet): 64 .. 512 channels, hidden widths 4 .. 32"""
    _train_step_check((2, 2, 2, 2), 32, 128, bottleneck=False)


@pytest.mark.parametrize("algebra", ["0", "1"])
def test_se_resnet50_eval_logits_parity(monkeypatch, algebra):
    """eval logits after calibrating the running statistics on one batch (momentum 1: running stats := batch stats)"""
    monkeypatch.setenv("B200_RESNET_ALGEBRA", algebra)
    layers = (3, 4, 6, 3)
    m, state = _model(layers, True)
    ref = _yard(state, layers, True)
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
    yard, _ = _autocast_yardstick(state, x, False, None, layers, True)
    print(f"eval logits max-abs err {err:.4g} (|ref| max {float(want.abs().max()):.3g}); torch bf16 autocast: {yard:.4g}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)


@pytest.mark.parametrize("accum", [1, 2])
def test_senet_trainstep_captured_equals_eager(accum):
    """CUDA-graph replay of the TrainStep reproduces eager stepping bit for bit (gradient accumulation included)"""
    from deeplearning_b200.engine.trainer import TrainStep

    a, _ = _model((1, 1, 1, 1), True, seed=4, num_classes=16)
    b, _ = _model((1, 1, 1, 1), True, seed=4, num_classes=16)
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
    # the SE weights moved: their gradients reached the optimizer through the arena
    _, fresh = _model((1, 1, 1, 1), True, seed=4, num_classes=16)
    assert not torch.equal(a.layer1[0].se.fc[0].weight.cpu(), fresh["layer1.0.se.fc.0.weight"])


def test_se_resnet101_step_has_finite_grads():
    from deeplearning_b200.classification.seNet.models.networks import se_resnet101

    torch.manual_seed(0)
    m = se_resnet101().cuda().train()
    x = torch.randn(8, 3, 128, 128, device="cuda")
    y = torch.randint(0, 1000, (8,), device="cuda")
    loss = F.cross_entropy(m(x), y)
    loss.backward()
    assert torch.isfinite(loss)
    for name, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and torch.isfinite(p.grad).all(), name
    for w in (m.layer3[22].se.fc[0].weight, m.layer4[0].se.fc[2].weight):
        assert float(w.grad.abs().sum()) > 0
