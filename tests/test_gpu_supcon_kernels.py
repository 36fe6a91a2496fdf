"""The SupCon kernels (csrc/supcon.cuh) against float64: the row normalisation forward and backward, the SupCon loss and its
feature gradient over N in {2, 6, 64, 400, 510, 2048}, D in {128, 512, 2048} and temperatures 0.07 / 0.1 / 1.0, labels with
few classes, all distinct (SimCLR) and one class, n_views 2 and 3, batches where a fixed shift of 1 / tau would underflow in
fp32, the no-positive NaN case, the device-side upstream gradient, and bitwise repeatability.

Tolerances: the loss and gradient are fp32 sums over N * D products of unit-row entries, the exponentials of fp32 logits of
size up to 1 / tau; 1e-5 relative on the loss and 1e-4 relative L2 on the gradient leave a margin over that rounding."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

LOSS_TOL, GRAD_TOL = 1e-5, 1e-4


def _ref(e64, rows, tau, base=0.07):
    """float64 loss and gradient of the contrast rows e64 [N, D] with int labels rows [N] (the formula of the reference's
    SupConLoss, written over all rows)."""
    e = e64.detach().clone().requires_grad_(True)
    N = e.shape[0]
    lg = e @ e.T / tau
    eye = torch.eye(N, dtype=torch.bool, device=e.device)
    pos = (rows[:, None] == rows[None, :]) & ~eye
    L = torch.logsumexp(lg.masked_fill(eye, float("-inf")), dim=1)
    mean_pos = (lg * pos).sum(1) / pos.sum(1)
    loss = (-(tau / base) * (mean_pos - L)).mean()
    loss.backward()
    return loss.detach(), e.grad


def _run(e32, rows32, tau, base=0.07, g=1.0):
    from deeplearning_b200 import ops

    loss, L, npos = ops.supcon_loss(e32, rows32, tau, base)
    gout = torch.full((1,), g, dtype=torch.float32, device="cuda")
    de = ops.supcon_loss_bwd(e32, rows32, L, npos, gout, tau, base)
    return loss, de


def _check(e32, rows, tau):
    ref_loss, ref_g = _ref(e32.double(), rows, tau)
    loss, de = _run(e32, rows.int().contiguous(), tau)
    torch.cuda.synchronize()
    # (N = 2: the only other row is the positive, so loss and gradient are exactly 0)
    d_loss, d_grad = abs(float(loss) - float(ref_loss)), float((de.double() - ref_g).norm())
    assert d_loss <= LOSS_TOL * abs(float(ref_loss)) and d_grad <= GRAD_TOL * float(ref_g.norm()), (d_loss, d_grad)


def _unit(N, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return F.normalize(torch.randn(N, D, device="cuda", generator=g), dim=1)


@pytest.mark.parametrize("N", [2, 6, 64, 400, 510, 2048])
@pytest.mark.parametrize("D", [128, 512, 2048])
def test_loss_and_gradient_against_float64(N, D):
    B = N // 2
    e = _unit(N, D, N * 7 + D)
    few = torch.randint(0, 5, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(N)).repeat(2)
    for tau in (0.07, 0.1, 1.0):
        _check(e, few, tau)
    simclr = torch.arange(B, device="cuda").repeat(2)
    _check(e, simclr, 0.1)
    _check(e, torch.zeros(N, dtype=torch.long, device="cuda"), 0.1)


def test_three_views():
    B = 50
    e = _unit(3 * B, 128, 1)
    y = torch.randint(0, 4, (B,), device="cuda").repeat(3)
    for tau in (0.07, 1.0):
        _check(e, y, tau)
    _check(e, torch.arange(B, device="cuda").repeat(3), 0.07)


def test_fixed_shift_underflow_cases():
    """tau = 0.01: one-hot orthogonal rows (every off-diagonal logit 0 against a diagonal of 100) and an antipodal positive
    pair (logit -100): a shift by the row maximum including the diagonal underflows exp() in fp32; the running maximum
    does not."""
    N, D = 8, 16
    e = torch.eye(D, device="cuda")[:N].contiguous()
    _check(e, torch.arange(4, device="cuda").repeat(2), 0.01)
    e = torch.eye(D, device="cuda")[:N].clone()
    e[4] = -e[0]
    loss, de = _run(e, torch.arange(4, device="cuda").repeat(2).int(), 0.01)
    assert torch.isfinite(loss).all() and torch.isfinite(de).all()
    _check(e, torch.arange(4, device="cuda").repeat(2), 0.01)


def test_anchor_without_positive_gives_nan():
    e = _unit(6, 128, 3)
    loss, de = _run(e, torch.arange(6, device="cuda").int(), 0.1)   # n_views 1, distinct labels: no positives
    assert torch.isnan(loss).all() and torch.isnan(de).all()


def test_upstream_gradient_read_from_device_and_bitwise_repeatable():
    e = _unit(400, 128, 5)
    y = torch.randint(0, 10, (200,), device="cuda").repeat(2).int()
    l1, d1 = _run(e, y, 0.1)
    l2, d2 = _run(e, y, 0.1)
    assert torch.equal(l1, l2) and torch.equal(d1, d2)
    _, d3 = _run(e, y, 0.1, g=1024.0)
    assert torch.equal(d3, d1 * 1024.0)   # a power of two: exact


def test_supconloss_module_autograd_and_graph_capture():
    from deeplearning_b200.self_supervised.SupCon.losses.SupConLoss import SupConLoss
    from oracle.supcon import supcon_loss

    f = F.normalize(torch.randn(64, 2, 128, device="cuda"), dim=-1)
    y = torch.randint(0, 5, (64,), device="cuda")
    crit = SupConLoss(temperature=0.1)
    fa = f.clone().requires_grad_(True)
    loss = crit(fa, y)
    (loss * 256.0).backward()
    loss = loss.detach()   # as under GradScaler: the upstream gradient is a device value
    fr = f.double().requires_grad_(True)
    ref = supcon_loss(fr, y, 0.1, 0.07)
    (ref * 256.0).backward()
    ref = ref.detach()
    assert abs(float(loss) - float(ref)) <= LOSS_TOL * abs(float(ref))
    assert float((fa.grad.double() - fr.grad).norm() / fr.grad.norm()) <= GRAD_TOL
    # graph replay gives the eager result bit for bit
    static = f.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        crit(static, y).backward()
    torch.cuda.current_stream().wait_stream(s)
    static.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gl = crit(static, y)
        gl.backward()
    graph.replay()
    torch.cuda.synchronize()
    fb = f.clone().requires_grad_(True)
    el = crit(fb, y)
    el.backward()
    assert torch.equal(gl.detach(), el.detach()) and torch.equal(static.grad, fb.grad)


def test_normalize_forward_backward_against_float64():
    from deeplearning_b200 import ops

    for N, D in ((400, 128), (37, 2048), (5, 4)):
        z = torch.randn(N, D, device="cuda") * 3.0
        z[0] = 0.0   # the clamp: e = 0, dz = de / 1e-12
        de = torch.randn(N, D, device="cuda")
        e, nrm = ops.supcon_normalize(z)
        dz = ops.supcon_normalize_bwd(de, e, nrm)
        z64 = z.double().requires_grad_(True)
        e64 = F.normalize(z64, dim=1)
        e64.backward(de.double())
        assert float((e.double() - e64.detach()).abs().max()) <= 1e-6
        assert torch.equal(nrm[0], torch.zeros((), device="cuda"))
        ref = z64.grad
        # bf16 output: within the bf16 rounding of every element (relative 2^-8)
        err = (dz.double() - ref).abs()
        assert bool((err <= 2.0 ** -8 * ref.abs() + 1e-6 * ref[1:].abs().max()).all()), float(err.max())


def test_relu_bwd_masks_by_the_forward_output():
    from deeplearning_b200 import ops

    y = torch.randn(400, 512, device="cuda").relu().bfloat16()
    dy = torch.randn(400, 512, device="cuda").bfloat16()
    assert torch.equal(ops.relu_bwd(dy, y), torch.where(y > 0, dy, torch.zeros_like(dy)))
