"""The MAE passes (csrc/mae.cuh) against PyTorch index ops in float64: the shuffle (including rows forced to tie), its
inverse, the masked patchify, the row gathers, the decoder-input assembly forward and backward, the pos_embed sums, the
masked-row scatter and the fused MSE; the batch sums are bitwise equal across two runs."""
import pytest
import torch

from deeplearning_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ids(B, P, seed=0):
    keys = torch.rand(B, P, device=DEV, generator=_gen(seed))
    return ops.mae_shuffle(keys)


@pytest.mark.parametrize("P", [2, 16, 49, 196, 256, 1024])
@pytest.mark.parametrize("levels", [None, 2, 7])
def test_shuffle_is_the_stable_argsort(P, levels):
    B = 64
    keys = torch.rand(B, P, device=DEV, generator=_gen(P))
    if levels is not None:   # forced ties: every row draws from a handful of values
        keys = torch.floor(keys * levels) / levels
    ids, slot = ops.mae_shuffle(keys)
    assert torch.equal(ids.long(), keys.argsort(dim=1, stable=True))
    ar = torch.arange(P, device=DEV).expand(B, P)
    assert torch.equal(slot.long().gather(1, ids.long()), ar)
    assert torch.equal(ids.long().gather(1, slot.long()), ar)


def test_shuffle_ties_on_torch_rand_draws():
    """fp32 torch.rand draws tie; the shuffle keeps the lower patch index first, as argsort(stable=True) does."""
    keys = torch.rand(256, 196, device=DEV, generator=_gen(3))
    keys[:, 100] = keys[:, 7]
    keys[5, 190] = keys[5, 3]
    ids, _ = ops.mae_shuffle(keys)
    assert torch.equal(ids.long(), keys.argsort(dim=1, stable=True))
    pos = ids.long()
    assert bool(((pos == 7).int().argmax(1) < (pos == 100).int().argmax(1)).all())


@pytest.mark.parametrize("B,C,H,p,Nm", [(4, 3, 224, 16, 147), (3, 3, 32, 8, 12), (2, 1, 48, 8, 30), (5, 3, 64, 16, 1)])
def test_masked_patchify(B, C, H, p, Nm):
    x = torch.randn(B, C, H, H, device=DEV, generator=_gen(1))
    P = (H // p) ** 2
    ids, _ = _ids(B, P)
    vis, tgt = ops.mae_patchify(x, ids, p, Nm)
    patches = x.view(B, C, H // p, p, H // p, p).permute(0, 2, 4, 3, 5, 1).reshape(B, P, -1)
    bi = torch.arange(B, device=DEV).unsqueeze(-1)
    idl = ids.long()
    assert torch.equal(tgt, patches[bi, idl[:, :Nm]])
    assert torch.equal(vis, patches[bi, idl[:, Nm:]].bfloat16())


def test_row_gathers():
    B, P, Nm, D = 6, 196, 147, 768
    ids, _ = _ids(B, P)
    idl = ids.long()
    bi = torch.arange(B, device=DEV).unsqueeze(-1)
    pos = torch.randn(P + 1, D, device=DEV, generator=_gen(2))
    got = ops.mae_gather_rows(pos, ids, Nm, P - Nm, 0, row_offset=1)
    assert torch.equal(got, pos.unsqueeze(0).repeat(B, 1, 1)[bi, idl[:, Nm:] + 1])
    h = torch.randn(B, P, 512, device=DEV, generator=_gen(3))
    got = ops.mae_gather_rows(h.view(B * P, 512), ids, 0, Nm, P, out_dtype=torch.bfloat16)
    assert torch.equal(got, h[bi, idl[:, :Nm]].bfloat16())


@pytest.mark.parametrize("B,P,Nm,D", [(8, 196, 147, 512), (3, 16, 12, 128), (256, 196, 147, 64)])
def test_assembly_forward_and_backward(B, P, Nm, D):
    Nv = P - Nm
    ids, slot = _ids(B, P, seed=B)
    idl = ids.long()
    bi = torch.arange(B, device=DEV).unsqueeze(-1)
    enc = torch.randn(B, Nv, D, device=DEV, generator=_gen(4))
    mask = torch.randn(D, device=DEV, generator=_gen(5))
    dpos = torch.randn(P, D, device=DEV, generator=_gen(6))
    dec = ops.mae_assemble_fwd(enc, mask, dpos, slot, Nm)
    mask_tokens = mask[None, None, :].double().repeat(B, Nm, 1) + dpos.double()[idl[:, :Nm]]
    concat = torch.cat([mask_tokens, enc.double()], dim=1)
    ref = torch.empty_like(concat)
    ref[bi, idl] = concat
    assert torch.allclose(dec.double(), ref, rtol=1e-6, atol=1e-6)

    g = torch.randn(B, P, D, device=DEV, generator=_gen(7)).bfloat16()
    g_enc, d_dpos = ops.mae_assemble_bwd(g, slot, Nm)
    assert torch.equal(g_enc, g[bi, idl[:, Nm:]])
    ref_dpos = torch.zeros(P, D, dtype=torch.float64, device=DEV)
    ref_dpos.index_add_(0, idl[:, :Nm].reshape(-1), g[bi, idl[:, :Nm]].double().reshape(-1, D))
    tol = 1e-5 * (1 + float(ref_dpos.abs().max()))
    assert float((d_dpos.double() - ref_dpos).abs().max()) <= tol
    d_mask = ops.batch_rowsum(d_dpos, D, P, D)
    assert float((d_mask.double() - g[bi, idl[:, :Nm]].double().sum((0, 1))).abs().max()) <= 1e-5 * (B * Nm) ** 0.5 * 4
    g_enc2, d_dpos2 = ops.mae_assemble_bwd(g, slot, Nm)
    assert torch.equal(d_dpos, d_dpos2) and torch.equal(g_enc, g_enc2)
    assert torch.equal(d_mask, ops.batch_rowsum(d_dpos2, D, P, D))

    g_in = torch.randn(B, Nv, D, device=DEV, generator=_gen(8)).bfloat16()
    d_pos = ops.mae_pos_grad(g_in, slot, Nm)
    ref_pos = torch.zeros(P + 1, D, dtype=torch.float64, device=DEV)
    ref_pos.index_add_(0, idl[:, Nm:].reshape(-1) + 1, g_in.double().reshape(-1, D))
    assert torch.equal(d_pos[0], torch.zeros(D, device=DEV))
    assert float((d_pos.double() - ref_pos).abs().max()) <= 1e-5 * (1 + float(ref_pos.abs().max()))
    assert torch.equal(d_pos, ops.mae_pos_grad(g_in, slot, Nm))

    dh = torch.randn(B, Nm, D, device=DEV, generator=_gen(9)).bfloat16()
    gs = ops.mae_scatter_masked(dh, slot, Nm)
    ref_g = torch.zeros(B, P, D, dtype=torch.bfloat16, device=DEV)
    ref_g[bi, idl[:, :Nm]] = dh
    assert torch.equal(gs, ref_g)


@pytest.mark.parametrize("shape", [(4, 147, 768), (256, 147, 768), (3, 12, 192), (1, 1, 8)])
@pytest.mark.parametrize("scale", [1.0, 0.25])
def test_mse_loss_and_gradient(shape, scale):
    pred = torch.randn(*shape, device=DEV, generator=_gen(10))
    t = torch.randn(*shape, device=DEV, generator=_gen(11))
    loss, grad = ops.mae_mse(pred, t, scale)
    n = pred.numel()
    e = pred.double() - t.double()
    ref = float((e * e).mean())
    assert abs(float(loss) - ref) <= 1e-5 * ref
    gref = scale * 2.0 * e / n
    assert float((grad.double() - gref).abs().max()) <= 2.0 ** -8 * float(gref.abs().max())
    loss2, grad2 = ops.mae_mse(pred, t, scale)
    assert torch.equal(loss, loss2) and torch.equal(grad, grad2)
