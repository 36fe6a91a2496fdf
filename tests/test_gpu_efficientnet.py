"""EfficientNet end to end on the GPU engine, against an fp32 CPU run of the in-tree oracle (oracle/efficientnet.py, pinned
to the reference by tests/golden/make_efficientnet_golden.py) on the same weights, inputs and drop-connect / dropout masks,
with PyTorch's own bf16 autocast run of the oracle as the measure of what bf16 storage costs: train steps of B0 at 96 px and
B2 at 72 px with the default drop-connect and dropout, eval logits, CUDA-graph capture against eager stepping, the
reference's own train_one_epoch loop, and the classifier-dropout mask against nn.Dropout's."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _model(name, seed=0, num_classes=1000):
    from deeplearning_b200.classification.efficientNet.models import network

    torch.manual_seed(seed)
    m = getattr(network, f"efficientnet_{name}")(num_classes=num_classes)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _train_step_check(name, B, hw):
    from deeplearning_b200.engine import droppath, efficientnet as eng
    from oracle.efficientnet import efficientnet_forward, plan, train_step_grads

    m, state = _model(name)
    # DropPath members only exist on residual blocks: pair each recorded multiplier with its block's rate
    rates = [float(b.dropout.drop_prob) for b in m.features if type(b).__name__ == "MBConv"
             and type(b.dropout).__name__ == "DropPath"]
    m = m.cuda().train()
    x = torch.randn(B, 3, hw, hw, generator=torch.Generator().manual_seed(1))
    labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2))
    torch.manual_seed(5)
    with droppath.record() as scales, eng.dropout_record() as masks:
        out = m(x.cuda())
    loss = F.cross_entropy(out, labels.cuda())
    loss.backward()
    assert len(scales) == len(rates) and len(masks) == 1
    drop = [((s.cpu() > 0).float(), 1.0 - r) for s, r in zip(scales, rates)]
    mask = masks[0].cpu()
    blocks = plan(name)
    ref_out, ref_loss, ref_grads, ref_state = train_step_grads(state, x, labels, blocks, drop=drop, mask=mask)
    # torch bf16 autocast of the same oracle on the GPU: the yardstick
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    s_gpu = {k: v.cuda() for k, v in state.items()}
    runs = []
    for amp in (False, True):
        s = {k: v.clone() for k, v in s_gpu.items()}
        params = {k: v.requires_grad_(True) for k, v in s.items() if v.is_floating_point() and "running" not in k}
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            o = efficientnet_forward(s, x.cuda().contiguous(memory_format=torch.channels_last), blocks, train=True,
                                     drop=[(r.cuda(), k) for r, k in drop], mask=mask.cuda()).float()
        g = torch.autograd.grad(F.cross_entropy(o, labels.cuda()), list(params.values()))
        runs.append((o.detach(), dict(zip(params, g))))
    yard = float((runs[1][0] - runs[0][0]).abs().max())
    gyard = {n: float((runs[1][1][n] - runs[0][1][n]).norm() / (runs[0][1][n].norm() + 1e-12)) for n in runs[0][1]}
    err = float((out.detach().float().cpu() - ref_out).abs().max())
    print(f"efficientnet_{name} bs {B} {hw}px: train logits max-abs err {err:.4g} (torch-bf16 yardstick {yard:.4g}); "
          f"loss {float(loss):.5f} vs {float(ref_loss):.5f}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)
    assert abs(float(loss.detach()) - float(ref_loss)) <= 1e-2
    # The project-BatchNorm shift of a block whose output reaches the loss only through train-mode BatchNorms (the last block
    # of a stage, and its residual successors) has a gradient that is zero in exact arithmetic: what remains is rounding
    # noise, so those gradients are held to 1e-3 of the largest gradient norm instead of a relative error.
    gmax = max(float(r.norm()) for r in ref_grads.values())
    worst = (0.0, "")
    for pname, p in m.named_parameters():
        g, r = p.grad.float().cpu(), ref_grads[pname]
        assert g.shape == r.shape, pname
        err = float((g - r).norm())
        rel = err / (float(r.norm()) + 1e-12)
        if err <= 1e-3 * gmax and float(r.norm()) <= 1e-3 * gmax:
            continue
        worst = max(worst, (rel / (gyard[pname] + 1e-3), pname))
        assert rel <= 2.0 * gyard[pname] + 0.02, f"{pname}: grad rel-L2 error {rel:.3g} vs torch-bf16 yardstick {gyard[pname]:.3g}"
    print(f"worst grad error relative to the torch-bf16 yardstick: {worst[0]:.2f}x at {worst[1]}")
    sd = m.state_dict()
    for k in ref_state:
        if "running_" in k and k.startswith(("features.stem_conv.", "features.1a.", "features.top.")):
            assert torch.allclose(sd[k].cpu(), ref_state[k], rtol=2e-2, atol=2e-3), k
        if "num_batches" in k:
            assert int(sd[k]) == int(ref_state[k]) == 1, k


def test_b0_train_step_parity_96px():
    _train_step_check("b0", 16, 96)


def test_b2_train_step_parity_72px():
    """72 px: 36 -> 18 -> 9 -> 5 -> 3 (stride 2 on odd grids), widths that are not multiples of 64, block 1b"""
    _train_step_check("b2", 8, 72)


@pytest.mark.parametrize("name", ["b0", "b2"])
def test_eval_logits(name):
    from oracle.efficientnet import efficientnet_forward, plan

    m, state = _model(name)
    # running statistics of a calibration batch, so that eval differs from train mode
    s = {k: v.clone() for k, v in state.items()}
    for k in s:
        if k.endswith("num_batches_tracked"):
            s[k].zero_()
    with torch.no_grad():
        efficientnet_forward(s, torch.randn(16, 3, 96, 96, generator=torch.Generator().manual_seed(3)), plan(name),
                             train=True)
    m.load_state_dict(s)
    m = m.cuda().eval()
    x = torch.randn(8, 3, 96, 96, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = efficientnet_forward({k: v.clone() for k, v in s.items()}, x, plan(name))
        got = m(x.cuda()).float().cpu()
        s_gpu = {k: v.cuda() for k, v in s.items()}
        with torch.autocast("cuda", dtype=torch.bfloat16):
            amp = efficientnet_forward(s_gpu, x.cuda(), plan(name)).float().cpu()
    err, yard = float((got - want).abs().max()), float((amp - want).abs().max())
    print(f"efficientnet_{name} eval logits max-abs err {err:.4g}; torch bf16 autocast {yard:.4g}")
    assert err <= max(1e-2, 1.5 * yard), (err, yard)
    out = m(x[:2].cuda())
    with pytest.raises(RuntimeError, match="recorded no tape"):
        out.sum().backward()


def test_trainstep_captured_equals_eager_with_random_masks():
    """With the default drop-connect and classifier dropout, a CUDA-graph replay draws the same masks as an eager step from
    the same generator state (torch's graph-safe Philox offsets), so replay and eager stepping agree bit for bit"""
    from deeplearning_b200.engine import droppath, efficientnet as eng
    from deeplearning_b200.engine.trainer import TrainStep

    a, _ = _model("b0", seed=4, num_classes=16)
    b, _ = _model("b0", seed=4, num_classes=16)
    a, b = a.cuda().train(), b.cuda().train()
    ta, tb = TrainStep(a, lr=0.02), TrainStep(b, lr=0.02)
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(8, 3, 64, 64, device="cuda", generator=g)
    y = torch.randint(0, 16, (8,), device="cuda", generator=g)
    tb.capture(x, y)
    drawn = []
    for step in range(3):
        torch.cuda.manual_seed(1000 + step)
        with droppath.record() as scales, eng.dropout_record() as masks:
            la, _ = ta.step_eager(x, y)
        drawn.append((scales, masks))
        torch.cuda.manual_seed(1000 + step)
        lb, _ = tb.step(x, y)
        assert float(la) == float(lb), step
    # the masks are real draws: some samples and features are dropped, and they change from step to step
    assert any(float(s.min()) == 0.0 for scales, _ in drawn for s in scales)
    assert all(float(m[0].min()) == 0.0 for _, m in drawn)
    assert not torch.equal(drawn[0][1][0], drawn[1][1][0])
    for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
        assert torch.equal(pa, pb), n
    for ba, bb in zip(a.buffers(), b.buffers()):
        assert torch.equal(ba, bb)


def test_trainstep_with_default_dropout_trains():
    """efficientnet_b0() with its default drop-connect and dropout, captured: finite losses that go down on one batch"""
    from deeplearning_b200.engine.trainer import TrainStep

    m, _ = _model("b0", seed=1, num_classes=10)
    m = m.cuda().train()
    t = TrainStep(m, lr=0.05)
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(16, 3, 96, 96, device="cuda", generator=g)
    y = torch.randint(0, 10, (16,), device="cuda", generator=g)
    t.capture(x, y)
    losses = [float(t.step(x, y)[0]) for _ in range(12)]
    assert all(torch.isfinite(torch.tensor(losses)))
    assert sum(losses[-3:]) < sum(losses[:3]), losses


def test_reference_train_one_epoch_loop():
    """The reference's own utils.train_one_epoch loop (restated: forward, cross-entropy, backward, SGD step) on the
    drop-in with the default drop-connect and dropout"""
    m, _ = _model("b0", seed=2, num_classes=5)
    m = m.cuda()
    opt = torch.optim.SGD([p for p in m.parameters() if p.requires_grad], lr=0.01, momentum=0.9, weight_decay=1e-4)
    loss_function = torch.nn.CrossEntropyLoss()
    g = torch.Generator().manual_seed(8)
    data = [(torch.randn(8, 3, 64, 64, generator=g), torch.randint(0, 5, (8,), generator=g)) for _ in range(3)]
    m.train()
    opt.zero_grad()
    for images, labels in data:
        pred = m(images.cuda())
        loss = loss_function(pred, labels.cuda())
        loss.backward()
        assert torch.isfinite(loss)
        opt.step()
        opt.zero_grad()
    for n, p in m.named_parameters():
        assert torch.isfinite(p).all(), n


def test_dropout_mask_matches_nn_dropout():
    """With a seeded generator the engine's classifier-dropout mask is nn.Dropout(p, inplace=True)'s on fp32 [B, F]"""
    from deeplearning_b200.engine import efficientnet as eng

    m, _ = _model("b0", seed=3, num_classes=5)
    m = m.cuda().train()
    x = torch.randn(4, 3, 64, 64, device="cuda")
    n_drop = sum(1 for b in m.features if type(b).__name__ == "MBConv" and type(b.dropout).__name__ == "DropPath")
    torch.cuda.manual_seed(11)
    with eng.dropout_record() as masks, torch.no_grad():
        m(x)
    torch.cuda.manual_seed(11)
    for _ in range(n_drop):           # the drop-connect draws come first, as in the reference's forward
        torch.rand((4, 1, 1, 1), device="cuda")
    feats = torch.full((4, 1280), 0.75, device="cuda")      # the pooled features: no generator draw of their own
    kept = torch.nn.Dropout(p=0.2, inplace=True)(feats) != 0
    assert torch.equal(masks[0], kept.float() * (1.0 / 0.8))
    assert 0 < int(kept.sum()) < kept.numel()
