"""RepVGG end to end on the GPU engine, against an fp32 CPU run of the in-tree oracle (oracle/repvgg.py, pinned to the
reference by tests/golden/make_repvgg_golden.py) on the same weights and inputs, with PyTorch's own bf16 autocast run of the
oracle as the measure of what bf16 storage costs: train steps of RepVGG-A0 / B0, eval logits of the train form (folded on
the device) and of the converted deploy form, CUDA-graph capture, get_custom_L2, and a RepVGG-B1 step at 224 px."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _model(name, seed=0, num_classes=1000, deploy=False):
    from deeplearning_b200.classification.RepVGG.models import func_dict

    torch.manual_seed(seed)
    m = func_dict[name](deploy=deploy, num_classes=num_classes)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _oracle(name, state, num_classes=1000):
    from oracle.repvgg import build

    return build(name, {k: v.clone() for k, v in state.items()}, num_classes)


def _autocast_yardstick(make, x, train, labels):
    """(max |bf16-autocast - fp32| of the logits, {param: grad rel-L2 of autocast vs fp32}) of the oracle on the GPU"""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    outs, grads = [], []
    for amp in (False, True):
        ref = make().cuda().train(train).to(memory_format=torch.channels_last)
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


def _custom_l2(b):
    """RepVGGBlock.get_custom_L2 of the reference, on an oracle block"""
    def t(bn):
        return (bn.weight / (bn.running_var + bn.eps).sqrt()).reshape(-1, 1, 1, 1).detach()

    k3, k1 = b.rbr_dense.conv.weight, b.rbr_1x1.conv.weight
    t3, t1 = t(b.rbr_dense.bn), t(b.rbr_1x1.bn)
    eq = k3[:, :, 1:2, 1:2] * t3 + k1 * t1
    return (eq ** 2 / (t3 ** 2 + t1 ** 2)).sum() + (k3 ** 2).sum() - (k3[:, :, 1:2, 1:2] ** 2).sum()


def _train_step_check(name, B, hw, custom_l2=0.0):
    m, state = _model(name)
    m = m.cuda().train()
    x = torch.randn(B, 3, hw, hw, generator=torch.Generator().manual_seed(1))
    labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    ref = _oracle(name, state).train()
    ref_out = ref(x)
    ref_loss = F.cross_entropy(ref_out, labels)
    blocks_ref = [b for b in ref.modules() if hasattr(b, "rbr_1x1")]
    if custom_l2:
        ref_total = ref_loss + custom_l2 * 0.5 * sum(_custom_l2(b) for b in blocks_ref)
    else:
        ref_total = ref_loss
    ref_total.backward()
    ref_grads = {n: p.grad for n, p in ref.named_parameters()}
    out = m(x.cuda())
    loss = F.cross_entropy(out, labels.cuda())
    total = loss
    if custom_l2:
        total = loss + custom_l2 * 0.5 * sum(b.get_custom_L2() for b in m.modules() if hasattr(b, "rbr_1x1"))
    total.backward()
    err = float((out.detach().float().cpu() - ref_out.detach()).abs().max())
    yard, gyard = _autocast_yardstick(lambda: _oracle(name, state), x, True, labels)
    print(f"{name} bs {B} {hw}px: train logits max-abs err {err:.4g} (torch-bf16 yardstick {yard:.4g}); loss "
          f"{float(loss.detach()):.5f} vs {float(ref_loss.detach()):.5f}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)
    assert abs(float(loss.detach()) - float(ref_loss.detach())) <= 1e-2
    worst = (0.0, "")
    for pname, p in m.named_parameters():
        g, r = p.grad.float().cpu(), ref_grads[pname]
        assert g.shape == r.shape, pname
        rel = float((g - r).norm() / (r.norm() + 1e-12))
        worst = max(worst, (rel / (gyard[pname] + 1e-3), pname))
        assert rel <= 2.0 * gyard[pname] + 0.02, f"{pname}: grad rel-L2 error {rel:.3g} vs torch-bf16 yardstick {gyard[pname]:.3g}"
    print(f"worst grad error relative to the torch-bf16 yardstick: {worst[0]:.2f}x at {worst[1]}")
    sd, rsd = m.state_dict(), ref.state_dict()
    for k in rsd:
        if "running_" in k and k.startswith(("stage0.", "stage1.")):
            assert torch.allclose(sd[k].cpu(), rsd[k], rtol=2e-2, atol=2e-3), k
            assert not torch.equal(sd[k].cpu(), state[k]), k
        if "num_batches" in k:
            assert int(sd[k]) == int(rsd[k]) == 1, k


def test_repvgg_a0_train_step_parity():
    _train_step_check("RepVGG-A0", 32, 128)


def test_repvgg_b0_train_step_parity():
    _train_step_check("RepVGG-B0", 32, 128)


def test_repvgg_a0_odd_grid_train_step_parity():
    """100 px: the stem and stage1..4 read 100, 50, 25, 13 and 7 px grids (odd stride-2 inputs)"""
    _train_step_check("RepVGG-A0", 16, 100)


def test_custom_l2_gradients_match_oracle():
    _train_step_check("RepVGG-A0", 16, 96, custom_l2=5e-4 * 1000)


def _calibrated(name):
    """model + oracle state after one batch-statistics pass with momentum 1 (running stats := batch stats)"""
    m, state = _model(name)
    ref = _oracle(name, state)
    for mod in ref.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = 1.0
    with torch.no_grad():
        ref.train()(torch.randn(32, 3, 128, 128, generator=torch.Generator().manual_seed(3)))
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    m.load_state_dict(state)
    return m, state


@pytest.mark.parametrize("name", ["RepVGG-A0", "RepVGG-B0"])
def test_eval_logits_train_form_and_deploy_form(name):
    from deeplearning_b200.classification.RepVGG.models import repvgg_model_convert
    from oracle.repvgg import convert

    m, state = _calibrated(name)
    m = m.cuda().eval()
    ref = _oracle(name, state).eval()
    x = torch.randn(8, 3, 160, 160, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = ref(x)
        got = m(x.cuda()).float().cpu()
        dep = repvgg_model_convert(m)
        got_dep = dep(x.cuda()).float().cpu()
        want_dep = convert(ref)(x)
    yard, _ = _autocast_yardstick(lambda: _oracle(name, state), x, False, None)
    err, err_dep = float((got - want).abs().max()), float((got_dep - want_dep).abs().max())
    print(f"{name} eval logits max-abs err: train form {err:.4g}, deploy form {err_dep:.4g}; torch bf16 autocast: {yard:.4g}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)
    assert err_dep <= max(1e-2, 1.5 * yard), (err_dep, yard)
    # a forward with parameters that need gradients still records no tape in eval mode
    out = m(x[:2].cuda())
    with pytest.raises(RuntimeError, match="recorded no tape"):
        out.sum().backward()


def test_partially_converted_and_deploy_constructed_models():
    from deeplearning_b200.classification.RepVGG.models import func_dict
    from oracle.repvgg import convert

    m, state = _calibrated("RepVGG-A0")
    ref = _oracle("RepVGG-A0", state).eval()
    for blk in (m.stage0, m.stage2[1], m.stage3[5]):
        blk.switch_to_deploy()
    m = m.cuda().eval()
    x = torch.randn(4, 3, 96, 96, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = ref(x)
        got = m(x.cuda()).float().cpu()
        d = func_dict["RepVGG-A0"](deploy=True, num_classes=1000)
        d.load_state_dict(convert(ref).state_dict())
        got_d = d.cuda().eval()(x.cuda()).float().cpu()
    assert float((got - want).abs().max()) <= 0.05 * (1 + float(want.abs().max()))
    assert float((got_d - want).abs().max()) <= 0.05 * (1 + float(want.abs().max()))
    with pytest.raises(NotImplementedError, match="deploy-form"):
        m.train()(x.cuda())


def test_uint8_input_matches_normalised_float():
    from deeplearning_b200 import ops

    m, _ = _model("RepVGG-A0", num_classes=10)
    m = m.cuda().eval()
    u8 = torch.randint(0, 256, (4, 64, 64, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).cuda()
    mean = torch.tensor(ops.IMAGENET_MEAN, device="cuda").view(1, 3, 1, 1)
    std = torch.tensor(ops.IMAGENET_STD, device="cuda").view(1, 3, 1, 1)
    xf = (u8.permute(0, 3, 1, 2).float() / 255.0 - mean) / std
    with torch.no_grad():
        a, b = m(u8), m(xf)
    assert float((a - b).abs().max()) <= 2e-2 * (1 + float(b.abs().max()))


@pytest.mark.parametrize("accum", [1, 2])
def test_repvgg_trainstep_captured_equals_eager(accum):
    """CUDA-graph replay of the TrainStep reproduces eager stepping bit for bit (gradient accumulation included)"""
    from deeplearning_b200.engine.trainer import TrainStep

    a, _ = _model("RepVGG-A0", seed=4, num_classes=16)
    b, _ = _model("RepVGG-A0", seed=4, num_classes=16)
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
    _, fresh = _model("RepVGG-A0", seed=4, num_classes=16)
    for k in ("stage0.rbr_1x1.conv.weight", "stage0.rbr_dense.conv.weight", "stage1.1.rbr_identity.weight"):
        assert not torch.equal(a.state_dict()[k].cpu(), fresh[k]), k


def test_repvgg_b1_step_at_224_has_finite_grads():
    m, _ = _model("RepVGG-B1")
    m = m.cuda().train()
    x = torch.randn(16, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (16,), device="cuda")
    loss = F.cross_entropy(m(x), y)
    loss.backward()
    assert torch.isfinite(loss)
    for name, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and torch.isfinite(p.grad).all(), name
    assert float(m.stage4[0].rbr_1x1.conv.weight.grad.abs().sum()) > 0
