"""ShuffleNet v2 end to end on the GPU engine, against an fp32 CPU run of the in-tree oracle (oracle/shufflenetv2.py) on the
same weights and inputs, with PyTorch's own bf16 autocast run of the oracle as the measure of what bf16 storage costs: train
steps of all four variants and an x1_0 step at 72 px (odd maps 9 -> 5 -> 3 at the stride-2 blocks), running statistics,
eval logits, CUDA-graph capture, the recipe's SGD against torch.optim.SGD, the uint8 input path and an x1_0 step at 224 px
through the model get_model builds."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

NAMES = ["x0_5", "x1_0", "x1_5", "x2_0"]
# BatchNorms without a ReLU whose output feeds a 1x1 convolution and another BatchNorm: their bias gradient is analytically
# zero (the second BatchNorm removes any per-channel constant), so the reference holds rounding noise only
ZERO_BIAS = ("branch1.1.bias", "branch2.4.bias")


def _model(name, seed=0, num_classes=5):
    from deeplearning_b200.classification.ShuffleNet.models import shufflenetv2

    torch.manual_seed(seed)
    m = getattr(shufflenetv2, f"shufflenet_v2_{name}")(num_classes=num_classes)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _autocast_yardstick(state, x, labels):
    """(max |bf16-autocast - fp32| of the logits, {param: grad rel-L2 of autocast vs fp32}, {running statistic: max
    |autocast - fp32|}) of the oracle on the GPU"""
    from oracle.shufflenetv2 import shufflenetv2_forward

    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    outs, grads, states = [], [], []
    try:
        for amp in (False, True):
            s = {k: v.clone().cuda() for k, v in state.items()}
            params = {k: v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k}
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                o = shufflenetv2_forward(s, x.cuda().contiguous(memory_format=torch.channels_last), True).float()
            outs.append(o.detach())
            gs = torch.autograd.grad(F.cross_entropy(o, labels.cuda()), list(params.values()))
            grads.append(dict(zip(params, gs)))
            states.append({k: v.detach().cpu() for k, v in s.items() if "running_" in k})
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    gerr = {n: float((grads[1][n] - grads[0][n]).norm() / (grads[0][n].norm() + 1e-12)) for n in grads[0]}
    serr = {k: float((states[1][k] - states[0][k]).abs().max()) for k in states[0]}
    return float((outs[1] - outs[0]).abs().max()), gerr, serr


def _train_check(name, hw):
    from oracle.shufflenetv2 import train_step_grads

    B = 8
    m, state = _model(name)
    m = m.cuda().train()
    x = torch.randn(B, 3, hw, hw, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 5, (B,), generator=torch.Generator().manual_seed(2))
    out = m(x.cuda())
    F.cross_entropy(out, y.cuda()).backward()
    torch.cuda.synchronize()
    ref_logits, _, ref_grads, ref_state = train_step_grads(state, x, y)
    d_ac, g_ac, s_ac = _autocast_yardstick(state, x, y)
    d = float((out.detach().cpu() - ref_logits).abs().max())
    assert d <= max(2.0 * d_ac, 0.05 * float(ref_logits.abs().max()) + 1e-3), (d, d_ac)
    for n, p in m.named_parameters():
        r = ref_grads[n]
        if n.endswith(ZERO_BIAS):
            # the engine's bf16 noise is bounded against the same BatchNorm's weight gradient instead
            ref_w = ref_grads[n[:-4] + "weight"]
            assert float(p.grad.norm()) <= 0.02 * float(ref_w.norm()), n
            continue
        rel = float((p.grad.cpu() - r).norm() / (r.norm() + 1e-12))
        assert rel <= max(3.0 * g_ac[n], 0.03), (n, rel, g_ac[n])
    for k, v in m.state_dict().items():
        if "running_" in k:
            r = ref_state[k]
            err = float((v.cpu() - r).abs().max())
            assert err <= max(3.0 * s_ac[k], 2e-2 * float(r.abs().max()) + 2e-3), (k, err, s_ac[k])
        if "num_batches_tracked" in k:
            assert int(v) == int(ref_state[k]), k


@pytest.mark.parametrize("name", NAMES)
def test_train_step(name):
    _train_check(name, 64)


def test_train_step_odd_maps():
    """72 px: the stride-2 blocks see 18 -> 9, 9 -> 5 and 5 -> 3 maps"""
    _train_check("x1_0", 72)


@pytest.mark.parametrize("name", ["x0_5", "x1_0"])
def test_eval_logits(name):
    from oracle.shufflenetv2 import shufflenetv2_forward

    m, _ = _model(name)
    m = m.cuda().train()
    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        m(x.cuda())   # one train forward: running statistics move away from their init
    m.eval()
    state = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    with torch.no_grad():
        out = m(x.cuda()).cpu()
    ref = shufflenetv2_forward(state, x, False)
    err = float((out - ref).abs().max())
    assert err <= 0.03 * float(ref.abs().max()) + 1e-3, err


def test_graph_capture_equals_eager():
    """three SGD steps replayed from one captured CUDA graph equal three eager steps"""
    from deeplearning_b200.engine.trainer import TrainStep

    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(5)).cuda()
    y = torch.randint(0, 5, (4,), generator=torch.Generator().manual_seed(6)).cuda()
    res = []
    for graph in (False, True):
        m, _ = _model("x1_0")
        m = m.cuda().train()
        step = TrainStep(m, lr=0.05, momentum=0.9, weight_decay=5e-4)
        if graph:
            step.capture(x, y)
        losses = [float(step.step(x, y)[0]) for _ in range(3)]
        res.append((losses, torch.cat([p.detach().flatten() for p in m.parameters()]).cpu(),
                    torch.cat([b.detach().float().flatten() for b in m.buffers()]).cpu()))
    assert res[0][0] == pytest.approx(res[1][0], rel=1e-5, abs=1e-6)
    assert torch.allclose(res[0][1], res[1][1], rtol=1e-4, atol=1e-6)
    assert torch.allclose(res[0][2], res[1][2], rtol=1e-4, atol=1e-6)


def test_sgd_recipe_against_torch():
    """TrainStep's SGD (momentum 0.9, weight decay 5e-4, the recipe's) over four steps equals torch.optim.SGD applied to the
    engine's own gradients (each step's gradients are checked against the oracle by test_train_step)"""
    from deeplearning_b200.engine.trainer import TrainStep

    m, _ = _model("x1_0")
    m = m.cuda().train()
    step = TrainStep(m, lr=0.05, momentum=0.9, weight_decay=5e-4)
    mine = [p.detach().clone().double().requires_grad_() for p in m.parameters()]
    opt = torch.optim.SGD(mine, lr=0.05, momentum=0.9, weight_decay=5e-4)
    losses = []
    for i in range(4):
        x = torch.randn(8, 3, 64, 64, generator=torch.Generator().manual_seed(20 + i))
        y = torch.randint(0, 5, (8,), generator=torch.Generator().manual_seed(30 + i))
        losses.append(float(step.step(x.cuda(), y.cuda())[0]))
        for r, p in zip(mine, m.parameters()):
            r.grad = p.grad.detach().double().clone()
        opt.step()
    torch.cuda.synchronize()
    assert all(l == l for l in losses), losses
    for (n, p), r in zip(m.named_parameters(), mine):
        err = float((p.detach().double() - r.detach()).abs().max())
        assert err <= 1e-5 * (1 + float(r.detach().abs().max())), (n, err)


def test_uint8_input_path():
    from deeplearning_b200 import ops

    m, _ = _model("x1_0")
    m = m.cuda().eval()
    u8 = torch.randint(0, 256, (2, 64, 64, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(8)).cuda()
    x = ((u8.permute(0, 3, 1, 2).float() / 255.0) - torch.tensor(ops.IMAGENET_MEAN, device="cuda").view(1, 3, 1, 1)) \
        / torch.tensor(ops.IMAGENET_STD, device="cuda").view(1, 3, 1, 1)
    with torch.no_grad():
        a, b = m(u8), m(x)
    assert float((a - b).abs().max()) <= 0.02 * float(b.abs().max()) + 1e-4


def test_x1_0_step_224():
    """the model the recipe builds with --arch shufflenet_v2_x1_0 trains: the loss falls over three steps"""
    from deeplearning_b200.classification.ShuffleNet.models import shufflenetv2
    from deeplearning_b200.engine.trainer import TrainStep

    torch.manual_seed(0)
    m = shufflenetv2.get_model("shufflenet_v2_x1_0")(num_classes=1000).cuda().train()
    step = TrainStep(m, lr=0.05, momentum=0.9, weight_decay=5e-4)
    x = torch.randn(16, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (16,), device="cuda")
    losses = [float(step.step(x, y)[0]) for _ in range(3)]
    assert all(l == l and l < 20 for l in losses), losses
    assert losses[-1] < losses[0], losses
