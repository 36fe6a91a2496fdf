"""VGG end to end on the GPU engine, against an fp32 CPU run of the in-tree oracle (oracle/vgg.py) on the same weights,
inputs and dropout masks, with PyTorch's own bf16 autocast run of the oracle as the measure of what bf16 storage costs:
train steps of vgg11 / vgg11_bn / vgg16 / vgg16_bn, running statistics, eval logits (plain and BatchNorm-folded),
CUDA-graph capture, the Adam recipe against torch.optim.Adam, the uint8 input path and a vgg16 step at 224 px."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _model(name, seed=0, num_classes=5, conv_bias=False):
    """the constructor's model and state_dict; conv_bias: random conv biases instead of the init's zeros, so that a bias in
    front of a BatchNorm moves its batch mean, running_mean and the eval fold"""
    from deeplearning_b200.classification.vggNet.models import network

    torch.manual_seed(seed)
    m = getattr(network, name)(num_classes=num_classes)
    if conv_bias:
        g = torch.Generator().manual_seed(seed + 50)
        with torch.no_grad():
            for mod in m.features:
                if isinstance(mod, torch.nn.Conv2d):
                    mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.5)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _masks(B, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(B, 4096, generator=g) >= 0.5).float() * 2.0 for _ in range(2)]


def _autocast_yardstick(state, x, labels, cfg, bn, masks):
    """(max |bf16-autocast - fp32| of the logits, {param: grad rel-L2 of autocast vs fp32}) of the oracle on the GPU"""
    from oracle.vgg import vgg_forward

    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    outs, grads = [], []
    try:
        for amp in (False, True):
            s = {k: v.clone().cuda() for k, v in state.items()}
            params = {k: v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k}
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                o = vgg_forward(s, x.cuda().contiguous(memory_format=torch.channels_last), cfg, bn, True,
                                [m.cuda() for m in masks]).float()
            outs.append(o.detach())
            gs = torch.autograd.grad(F.cross_entropy(o, labels.cuda()), list(params.values()))
            grads.append(dict(zip(params, gs)))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    gerr = {n: float((grads[1][n] - grads[0][n]).norm() / (grads[0][n].norm() + 1e-12)) for n in grads[0]}
    return float((outs[1] - outs[0]).abs().max()), gerr


def _train_check(name, B, hw, seed=0, conv_bias=False):
    from deeplearning_b200.engine import vgg as engine
    from oracle.vgg import arch, train_step_grads

    m, state = _model(name, seed, conv_bias=conv_bias)
    m = m.cuda().train()
    x = torch.randn(B, 3, hw, hw, generator=torch.Generator().manual_seed(1))
    y = torch.randint(0, 5, (B,), generator=torch.Generator().manual_seed(2))
    masks = _masks(B, 3)
    with engine.dropout_replay([mk.cuda() for mk in masks]):
        out = m(x.cuda())
    F.cross_entropy(out, y.cuda()).backward()
    torch.cuda.synchronize()
    cfg, bn = arch(name)
    ref_logits, ref_loss, ref_grads, ref_state = train_step_grads(state, x, y, cfg, bn, masks)
    d_ac, g_ac = _autocast_yardstick(state, x, y, cfg, bn, masks)
    d = float((out.detach().cpu() - ref_logits).abs().max())
    assert d <= max(2.0 * d_ac, 0.05 * float(ref_logits.abs().max()) + 1e-3), (d, d_ac)
    for n, p in m.named_parameters():
        r = ref_grads[n]
        rel = float((p.grad.cpu() - r).norm() / (r.norm() + 1e-12))
        assert rel <= max(3.0 * g_ac[n], 0.03), (n, rel, g_ac[n])
    if bn:
        for k, v in m.state_dict().items():
            if "running_" in k:
                assert torch.allclose(v.cpu(), ref_state[k], rtol=2e-2, atol=2e-3), k
            if "num_batches_tracked" in k:
                assert int(v) == int(ref_state[k]), k
    return m


@pytest.mark.parametrize("name", ["vgg11", "vgg11_bn"])
@pytest.mark.parametrize("hw", [32, 64])
def test_train_step_vgg11(name, hw):
    _train_check(name, 4, hw)


@pytest.mark.parametrize("name", ["vgg16", "vgg16_bn"])
def test_train_step_vgg16(name):
    _train_check(name, 4, 48)


@pytest.mark.parametrize("name", ["vgg11", "vgg11_bn"])
def test_train_step_conv_bias(name):
    """non-zero conv biases: the plain epilogue bias, and a bias in front of BatchNorm inside the batch mean and
    running_mean"""
    _train_check(name, 4, 32, conv_bias=True)


@pytest.mark.parametrize("name", ["vgg11", "vgg13_bn"])
def test_eval_logits(name):
    from oracle.vgg import arch, vgg_forward

    m, _ = _model(name, conv_bias=True)
    m = m.cuda().train()
    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        m(x.cuda())   # one train forward: running statistics move away from their init
    m.eval()
    state = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    with torch.no_grad():
        out = m(x.cuda()).cpu()
    cfg, bn = arch(name)
    ref = vgg_forward(state, x, cfg, bn, False)
    err = float((out - ref).abs().max())
    assert err <= 0.03 * float(ref.abs().max()) + 1e-3, err


def test_graph_capture_equals_eager():
    """three Adam steps replayed from one captured CUDA graph equal three eager steps (dropout off: the masks of a replay
    come from the generator state at replay time, which an eager run does not share)"""
    from deeplearning_b200.engine.trainer import TrainStep

    x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(5)).cuda()
    y = torch.randint(0, 5, (4,), generator=torch.Generator().manual_seed(6)).cuda()
    res = []
    for graph in (False, True):
        m, _ = _model("vgg11_bn")
        m.classifier[2].p = m.classifier[5].p = 0.0
        m = m.cuda().train()
        step = TrainStep(m, lr=1e-3, optimizer="adam", weight_decay=1e-3)
        if graph:
            step.capture(x, y)
        losses = [float(step.step(x, y)[0]) for _ in range(3)]
        res.append((losses, torch.cat([p.detach().flatten() for p in m.parameters()]).cpu(),
                    torch.cat([b.detach().float().flatten() for b in m.buffers()]).cpu()))
    assert res[0][0] == pytest.approx(res[1][0], rel=1e-5, abs=1e-6)
    assert torch.allclose(res[0][1], res[1][1], rtol=1e-4, atol=1e-6)
    assert torch.allclose(res[0][2], res[1][2], rtol=1e-4, atol=1e-6)


def test_adam_recipe_and_state_dict():
    """three TrainStep(optimizer="adam", weight_decay=1e-3) steps equal torch.optim.Adam(lr, weight_decay=1e-3) applied to
    the engine's own gradients (the gradients themselves are checked against the oracle above: Adam's normalised step
    turns their bf16 noise into sign flips of near-zero elements), and the state dict round-trips through torch's Adam"""
    from deeplearning_b200.engine import vgg as engine
    from deeplearning_b200.engine.trainer import TrainStep

    m, _ = _model("vgg11_bn")
    m = m.cuda().train()
    step = TrainStep(m, lr=1e-3, optimizer="adam", weight_decay=1e-3)
    ref = [p.detach().clone().double().requires_grad_() for p in m.parameters()]
    opt = torch.optim.Adam(ref, lr=1e-3, weight_decay=1e-3)
    for i in range(3):
        x = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(20 + i))
        y = torch.randint(0, 5, (4,), generator=torch.Generator().manual_seed(30 + i))
        with engine.dropout_replay([mk.cuda() for mk in _masks(4, 40 + i)]):
            step.step(x.cuda(), y.cuda())
        for r, p in zip(ref, m.parameters()):
            r.grad = p.grad.detach().double().clone()
        opt.step()
    torch.cuda.synchronize()
    for (n, p), r in zip(m.named_parameters(), ref):
        err = float((p.detach().double() - r.detach()).abs().max())
        assert err <= 1e-6, (n, err)
    sd = step.optimizer_state_dict()
    ref_opt = torch.optim.Adam([p for p in m.parameters()], lr=1e-3, weight_decay=1e-3)
    ref_opt.load_state_dict(sd)
    back = ref_opt.state_dict()
    assert back["param_groups"][0]["weight_decay"] == 1e-3 and len(back["param_groups"]) == 1
    st2 = TrainStep(_model("vgg11_bn")[0].cuda().train(), lr=5e-4, optimizer="adam", weight_decay=1e-3)
    st2.load_optimizer_state_dict(back)
    assert st2.steps == 3
    assert torch.equal(st2.arena.flat_m, step.arena.flat_m) and torch.equal(st2.arena.flat_v, step.arena.flat_v)


def test_uint8_input_path():
    from deeplearning_b200 import ops

    m, _ = _model("vgg11")
    m = m.cuda().eval()
    u8 = torch.randint(0, 256, (2, 32, 32, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(8)).cuda()
    x = ((u8.permute(0, 3, 1, 2).float() / 255.0) - torch.tensor(ops.IMAGENET_MEAN, device="cuda").view(1, 3, 1, 1)) \
        / torch.tensor(ops.IMAGENET_STD, device="cuda").view(1, 3, 1, 1)
    with torch.no_grad():
        a, b = m(u8), m(x)
    assert float((a - b).abs().max()) <= 0.02 * float(b.abs().max()) + 1e-4


def test_vgg16_step_224():
    from deeplearning_b200.engine.trainer import TrainStep

    m, _ = _model("vgg16", num_classes=1000)
    m = m.cuda().train()
    step = TrainStep(m, lr=1e-4, optimizer="adam", weight_decay=1e-3)
    x = torch.randn(8, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (8,), device="cuda")
    losses = [float(step.step(x, y)[0]) for _ in range(3)]
    assert all(l == l and l < 20 for l in losses), losses
    assert losses[-1] < losses[0], losses
