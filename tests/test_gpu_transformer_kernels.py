"""The ViT, Swin and ConvNeXt kernels (LayerNorm, patch-merge LayerNorm, ViT attention, window attention, depthwise 7x7,
patch extraction, layer-scale gradients) against float64 PyTorch restatements of their ops, at the widths, head counts and
token counts of every variant the drop-ins ship (ViT-B/L at patch 16 and 32, Swin-T/S/B, ConvNeXt-T/S/B) and at the edges
of each kernel's dispatch: the LayerNorm width branches and their boundaries, widths that are not a multiple of a branch's
lane stride, partial key tiles, persistent CTAs that walk many items.  Each reference reads the exact bf16 / fp32 tensors
the kernel reads.  Reductions must be bit-identical across two launches; the one exception is the relative-position bias
gradient of window attention, which is summed with atomics (DESIGN.md section 4).

Tolerances are `max|err| <= rel * max|ref|` per output tensor; the comment beside each `rel` gives the largest ratio
measured on an H100 80GB HBM3."""
import math

import pytest
import torch
import torch.nn.functional as F

from deeplearning_b200 import ops

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
LN2 = math.log(2.0)


def _rand(*shape, scale=1.0, seed=0, dtype=BF16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def _d(t):
    return t.detach().double()


def _close(got, ref, rel, what=""):
    got, ref = _d(got), _d(ref)
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    err = float((got - ref).abs().max())
    scale = float(ref.abs().max())
    print(f"{what}: max err / max|ref| = {err / max(scale, 1e-30):.3g}")
    assert err <= rel * scale + 1e-30, f"{what}: max err {err:.4g} > {rel:.3g} * {scale:.4g}"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------- LayerNorm
# b200_layernorm_bwd picks (vectors per lane, lanes per row) by width: <= 128 (2, 8), <= 256 (2, 16), <= 512 (2, 32),
# <= 768 (3, 32), <= 1024 (4, 32); the forward: <= 128, <= 256, <= 1024, <= 3072.  Each branch gets its upper edge, a
# width inside it and one that is not a multiple of its lane stride (64, 128, 256 channels).
LN_WIDTHS = [96, 104, 128, 192, 200, 256, 384, 392, 512, 520, 640, 768, 776, 1000, 1024]
LN_FWD_ONLY = [1032, 1536, 2040, 2048, 3072]
# 13001 rows: not a multiple of the 2 / 4 rows a warp handles at narrow widths, and more rows than the backward's
# 3 x SMs x 8 warps, so every warp accumulates dgamma / dbeta over several rows in its shared-memory slice
LN_ROWS = 13001
LN_EPS = 1e-6


def _ln_input(rows, C, offset, seed):
    x = _rand(rows, C, seed=seed, dtype=F32)
    if offset:
        x = x + 100.0  # mean 100x the std: E[x^2] - E[x]^2 would cancel to nothing in fp32
    return x


def _ln_ref(x, g, b, eps):
    xd = _d(x)
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    xh = (xd - mu) * rstd
    return xh * _d(g) + _d(b), mu.squeeze(-1), rstd.squeeze(-1), xh


def _ln_params(C, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed + 50)
    g = torch.rand(C, generator=gen, device="cuda") + 0.5
    b = torch.randn(C, generator=gen, device="cuda") * 0.1
    return g, b


REL_LN_Y16 = 8e-3     # bf16 output, whose rounding alone allows 2^-8 of |y| (measured 2.6e-3)
REL_LN_Y32 = 1.6e-5   # fp32 output (measured 4.4e-6, with the mean offset)
REL_LN_STAT = 2.5e-6  # mean, rstd (measured 6.9e-7)


@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("C", LN_WIDTHS + LN_FWD_ONLY)
def test_layernorm_fwd(C, offset):
    rows = LN_ROWS if C <= 1024 else 2001
    x32 = _ln_input(rows, C, offset, seed=C)
    g, b = _ln_params(C, C)
    for x in (x32, x32.to(BF16)):
        ref, mu, rstd, _ = _ln_ref(x, g, b, LN_EPS)
        for out_dtype in (BF16, F32):
            what = f"ln fwd C={C} {str(x.dtype)[6:]}->{str(out_dtype)[6:]} offset={offset}"
            y, m, r = ops.layernorm_fwd(x, g, b, LN_EPS, out_dtype=out_dtype)
            assert y.dtype == out_dtype
            _close(y, ref, REL_LN_Y16 if out_dtype == BF16 else REL_LN_Y32, what + " y")
            _close(m, mu, REL_LN_STAT, what + " mean")
            _close(r, rstd, REL_LN_STAT, what + " rstd")


REL_LN_DX16 = 1.2e-2  # bf16 dx (measured 3.6e-3)
REL_LN_DX32 = 1e-5    # fp32 dx (measured 2.7e-6)
REL_LN_DGAMMA = 2e-5  # (measured 5.7e-6 with the mean offset, where the fp32 mean of values near 100 is good to ~4e-6)
REL_LN_DBETA = 1.6e-7  # (measured 4.6e-8)


@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("C", LN_WIDTHS)
def test_layernorm_bwd(C, offset):
    rows = LN_ROWS
    x32 = _ln_input(rows, C, offset, seed=C + 1)
    g, b = _ln_params(C, C + 1)
    dy = _rand(rows, C, seed=C + 2)
    for x in (x32, x32.to(BF16)):
        _, m, r = ops.layernorm_fwd(x, g, b, LN_EPS)
        _, _, rstd, xh = _ln_ref(x, g, b, LN_EPS)
        dyd = _d(dy)
        dg_ = dyd * _d(g)
        dx_ref = rstd[:, None] * (dg_ - dg_.mean(-1, keepdim=True) - xh * (dg_ * xh).mean(-1, keepdim=True))
        dgam_ref, dbeta_ref = (dyd * xh).sum(0), dyd.sum(0)
        for dx_dtype in (BF16, F32):
            add = _rand(rows, C, seed=C + 3, dtype=dx_dtype)
            for with_add in (False, True):
                what = f"ln bwd C={C} x {str(x.dtype)[6:]} dx {str(dx_dtype)[6:]} add={with_add} offset={offset}"
                a = add if with_add else None
                dx, dgam, dbeta = ops.layernorm_bwd(dy, x, m, r, g, add=a, dx_dtype=dx_dtype)
                want = dx_ref + _d(add) if with_add else dx_ref
                _close(dx, want, REL_LN_DX16 if dx_dtype == BF16 else REL_LN_DX32, what + " dx")
                _close(dgam, dgam_ref, REL_LN_DGAMMA, what + " dgamma")
                _close(dbeta, dbeta_ref, REL_LN_DBETA, what + " dbeta")
                dx2, dgam2, dbeta2 = ops.layernorm_bwd(dy, x, m, r, g, add=a, dx_dtype=dx_dtype)
                assert torch.equal(dx, dx2) and torch.equal(dgam, dgam2) and torch.equal(dbeta, dbeta2), what + " repeat"


# ------------------------------------------------------------------------------------------------- patch-merge LayerNorm
REL_PM_Y = 8e-3       # bf16 y (measured 2.6e-3)
REL_PM_DX = 8e-3      # bf16 dx (measured 2.4e-3)
REL_PM_STAT = 6e-7    # mean, rstd (measured 1.5e-7)
REL_PM_DGAMMA = 5e-7  # (measured 1.25e-7)
REL_PM_DBETA = 1.6e-7  # (measured 4.5e-8)


@pytest.mark.parametrize("C", [96, 128, 192, 256, 384, 512])
def test_patch_merge_layernorm(C):
    # 13 x 14 x 21 = 3822 output rows: more than the backward's 3 x SMs x 8 warps, an odd merged width
    B, H, W = 13, 28, 42
    x = _rand(B, H, W, C, seed=C, dtype=F32) * 2 + 0.3
    g, b = _ln_params(4 * C, C)
    y, m, r = ops.patch_merge_ln_fwd(x, g, b, 1e-5)
    xd = _d(x)
    cat = torch.cat([xd[:, 0::2, 0::2], xd[:, 1::2, 0::2], xd[:, 0::2, 1::2], xd[:, 1::2, 1::2]], -1).reshape(-1, 4 * C)
    ref, mu, rstd, xh = _ln_ref(cat, g, b, 1e-5)
    _close(y, ref, REL_PM_Y, f"patch-merge C={C} y")
    _close(m, mu, REL_PM_STAT, f"patch-merge C={C} mean")
    _close(r, rstd, REL_PM_STAT, f"patch-merge C={C} rstd")
    dy = _rand(cat.shape[0], 4 * C, seed=C + 1)
    dyd = _d(dy)
    dg_ = dyd * _d(g)
    dcat = rstd[:, None] * (dg_ - dg_.mean(-1, keepdim=True) - xh * (dg_ * xh).mean(-1, keepdim=True))
    dcat = dcat.view(B, H // 2, W // 2, 4 * C)
    dx_ref = torch.empty_like(xd)
    dx_ref[:, 0::2, 0::2], dx_ref[:, 1::2, 0::2] = dcat[..., :C], dcat[..., C:2 * C]
    dx_ref[:, 0::2, 1::2], dx_ref[:, 1::2, 1::2] = dcat[..., 2 * C:3 * C], dcat[..., 3 * C:]
    dx, dgam, dbeta = ops.patch_merge_ln_bwd(dy, x, m, r, g)
    _close(dx, dx_ref, REL_PM_DX, f"patch-merge C={C} dx")
    _close(dgam, (dyd * xh).sum(0), REL_PM_DGAMMA, f"patch-merge C={C} dgamma")
    _close(dbeta, dyd.sum(0), REL_PM_DBETA, f"patch-merge C={C} dbeta")
    dx2, dgam2, dbeta2 = ops.patch_merge_ln_bwd(dy, x, m, r, g)
    assert torch.equal(dx, dx2) and torch.equal(dgam, dgam2) and torch.equal(dbeta, dbeta2)


# ------------------------------------------------------------------------------------------------------- ViT attention
ATT_T = [1, 50, 64, 65, 127, 128, 129, 192, 193, 197, 255, 256]


def _attn_inputs(B, T, H, peaked, seed):
    """std-1 qkv, or a peaked one: the queries of a head lean along one direction u and key j along c_j u, so that the
    scaled logits are about 30 c_j.  Key T-1 (in the last, usually partial, key tile) has c = 1 and wins, key T-2 has
    c = -1, the others 0.6 .. 0.95: logits from -30 to +30, with a few runners-up within reach of the winner."""
    qkv = _rand(B, T, 3, H, 64, seed=seed, dtype=F32)
    if peaked:
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        u = F.normalize(torch.randn(B, 1, H, 64, generator=g, device="cuda"), dim=-1)
        c = torch.rand(B, T, H, 1, generator=g, device="cuda") * 0.35 + 0.6
        c[:, T - 1] = 1.0
        if T > 1:
            c[:, T - 2] = -1.0
        a = math.sqrt(30.0 * 8.0)   # (a u) . (a u) * 64^-0.5 = 30
        qkv[:, :, 0] = qkv[:, :, 0] * 0.25 + a * u
        qkv[:, :, 1] = qkv[:, :, 1] * 0.25 + a * c * u
    return qkv.reshape(B, T, 3 * H * 64).to(BF16)


def _attn_ref(qkv, H, scale, dout):
    """float64 attention on the bf16 qkv: (out, natural-log lse, dq, dk, dv)."""
    B, T, _ = qkv.shape
    x = _d(qkv).requires_grad_(True)
    q, k, v = x.view(B, T, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-2, -1)) * scale
    lse = torch.logsumexp(s, -1)
    out = ((s - lse[..., None]).exp() @ v).transpose(1, 2).reshape(B, T, H * 64)
    (g,) = torch.autograd.grad(out, x, _d(dout))
    g = g.view(B, T, 3, H * 64)
    return out.detach(), lse.detach(), g[:, :, 0], g[:, :, 1], g[:, :, 2]


REL_ATT_O = 1.2e-2          # bf16 P into the PV product (measured 3.2e-3)
REL_ATT_LSE = 5e-7           # (measured 2.4e-7)
REL_ATT_DK = 2.4e-2          # bf16 dS into dS^T Q (measured 6.4e-3)
REL_ATT_DV = 1.6e-2          # (measured 4.5e-3)
REL_ATT_DQ_1BLK = 2.4e-2     # T <= 128: one key block, dQ stored once (measured 6.4e-3)
# T > 128: the key-block-0 part of dQ is stored as bf16 and reloaded before block 1 adds to it.  That extra rounding is
# not the dominant term: the T > 128 dQ error is about 1.3x the T <= 128 one and about dK's, which has no round trip
REL_ATT_DQ_2BLK = 3.2e-2     # (measured 8.6e-3)
# peaked inputs, dq: the keys share a common component of norm ~15 that cancels in dS K, since every row of dS sums to
# zero, so the bf16 rounding of dS and of the O in delta = rowsum(dO * O) is amplified (dk: measured 3.9e-3, no such loss)
REL_ATT_PEAKED_DQ = 0.12     # (measured 3.7e-2)
ATT_T1_ABS = 1e-5            # T = 1: softmax is identically 1 and dq = dk = 0; the kernel's P = 2^(s - lse) is 1 only to
                             # rounding (measured 2.1e-6)


@pytest.mark.parametrize("peaked", [False, True])
@pytest.mark.parametrize("H", [12, 16])
@pytest.mark.parametrize("T", ATT_T)
def test_attention_fwd_bwd(T, H, peaked):
    if peaked and H == 16:
        pytest.skip("the peaked inputs run at ViT-B's 12 heads")
    B = -(-4 * _sms() // H)   # B*H >= 4 x SMs: every persistent forward CTA walks several (batch, head) items
    scale = 64 ** -0.5
    qkv = _attn_inputs(B, T, H, peaked, seed=T + H)
    dout = _rand(B, T, H * 64, seed=T + H + 7)
    out, lse = ops.attention_fwd(qkv, H, scale)
    ref, lse_ref, dq_ref, dk_ref, dv_ref = _attn_ref(qkv, H, scale, dout)
    what = f"attention T={T} H={H} peaked={peaked}"
    _close(out, ref, REL_ATT_O, what + " out")
    _close(lse, lse_ref, REL_ATT_LSE, what + " lse")
    dqkv = ops.attention_bwd(qkv, out, dout, lse, H, scale).view(B, T, 3, H * 64)
    if T == 1:
        assert float(dq_ref.abs().max()) == 0.0 and float(dk_ref.abs().max()) == 0.0
        assert float(dqkv[:, :, :2].abs().max()) <= ATT_T1_ABS, what + " dq, dk"
    else:
        rel_dq = REL_ATT_PEAKED_DQ if peaked else REL_ATT_DQ_1BLK if T <= 128 else REL_ATT_DQ_2BLK
        _close(dqkv[:, :, 0], dq_ref, rel_dq, what + " dq")
        _close(dqkv[:, :, 1], dk_ref, REL_ATT_DK, what + " dk")
    _close(dqkv[:, :, 2], dv_ref, REL_ATT_DV, what + " dv")
    out2, lse2 = ops.attention_fwd(qkv, H, scale)
    assert torch.equal(out, out2) and torch.equal(lse, lse2), what + " forward repeat"
    dqkv2 = ops.attention_bwd(qkv, out, dout, lse, H, scale).view(B, T, 3, H * 64)
    assert torch.equal(dqkv, dqkv2), what + " backward repeat"


# ---------------------------------------------------------------------------------------------------- window attention
def _window_partition(x, ws=7):
    B, H, W, C = x.shape
    return x.view(B, H // ws, ws, W // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, C)


def _window_reverse(w, B, H, W, ws=7):
    return w.view(B, H // ws, W // ws, ws, ws, -1).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, -1)


def _rel_index():
    coords = torch.stack(torch.meshgrid([torch.arange(7), torch.arange(7)], indexing="ij")).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += 6
    rel[:, :, 1] += 6
    rel[:, :, 0] *= 13
    return rel.sum(-1)


def _shift_mask(H, W, shift):
    """attn_mask of SwinTransformerBlock: -100 between tokens of different regions of the rolled image, [nW, 49, 49]."""
    img = torch.zeros(1, H, W, 1)
    cnt = 0
    for h in (slice(0, -7), slice(-7, -shift), slice(-shift, None)):
        for w in (slice(0, -7), slice(-7, -shift), slice(-shift, None)):
            img[:, h, w, :] = cnt
            cnt += 1
    mw = _window_partition(img).view(-1, 49)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def _wattn_ref(qkv, nH, table, index, mask, shift, scale, dout):
    """float64 roll -> partition -> softmax(scale q k^T + bias (+ mask)) v -> reverse -> roll, and its gradients:
    (out, base-2 lse [B, nW, nH, 49], dqkv, dtable)."""
    B, H, W, C3 = qkv.shape
    C = C3 // 3
    nW = (H // 7) * (W // 7)
    x = _d(qkv).requires_grad_(True)
    t = _d(table).requires_grad_(True)
    xr = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2)) if shift else x
    q, k, v = _window_partition(xr).view(-1, 49, 3, nH, 32).permute(2, 0, 3, 1, 4)
    s = (q * scale) @ k.transpose(-2, -1) + t[index.view(-1)].view(49, 49, nH).permute(2, 0, 1)
    if mask is not None:
        s = (s.view(B, nW, nH, 49, 49) + _d(mask)[None, :, None]).view(-1, nH, 49, 49)
    lse = torch.logsumexp(s, -1)
    o = ((s - lse[..., None]).exp() @ v).transpose(1, 2).reshape(-1, 49, C)
    out = _window_reverse(o, B, H, W)
    if shift:
        out = torch.roll(out, shifts=(shift, shift), dims=(1, 2))
    gx, gt = torch.autograd.grad(out, (x, t), _d(dout))
    return out.detach(), (lse / LN2).view(B, nW, nH, 49).detach(), gx, gt


REL_WA_BIAS = 4e-7     # (table + mask) * log2(e) in fp32 (measured 1.0e-7)
REL_WA_O = 1.2e-2      # (measured 3.0e-3)
# the row sum runs over the bf16-rounded exponentials the P V product reads (so that each rounded row of P sums to one),
# which moves the lse by up to ~2^-9 / ln 2
REL_WA_LSE = 7e-4      # (measured 1.8e-4)
REL_WA_DQK = 2.4e-2    # (measured 6.6e-3)
REL_WA_DV = 1.9e-2     # (measured 4.8e-3)
REL_WA_DTAB = 1.8e-2   # (measured 4.7e-3)
REL_WA_SCATTER = 1e-6  # fp32 atomics (measured 2.8e-7)


def _wattn_batch(nH, H, W):
    """Images per batch so that every persistent CTA (SMs // nH of them per head) walks at least 7 window pairs."""
    lanes = max(1, _sms() // nH)
    nW = (H // 7) * (W // 7)
    return -(-2 * 7 * lanes // nW)


# (nH, H, W): Swin-T/S heads 3/6/12/24 and Swin-B heads 4/8/16/32 at the resolution of their stage at 224 px, plus the
# next stage's resolution for the last two (where a shift exists)
WA_CASES = [(3, 56, 56), (4, 56, 56), (6, 28, 28), (8, 28, 28), (12, 14, 14), (16, 14, 14), (24, 7, 7), (32, 7, 7),
            (24, 14, 14), (32, 14, 14)]


def _wattn_case(B, H, W, nH, shift, seed):
    C = nH * 32
    scale = 32 ** -0.5
    qkv = _rand(B, H, W, 3 * C, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    table = (torch.rand(169, nH, generator=g, device="cuda") * 2 - 1) * 5.0     # entries up to +-5
    index = _rel_index().cuda()
    mask = _shift_mask(H, W, shift).cuda() if shift else None
    dout = _rand(B, H, W, C, seed=seed + 2)
    what = f"window attention B={B} {H}x{W} nH={nH} shift={shift}"
    bias = ops.window_bias_gather(table, index, nH, mask)
    want = _d(table)[index.view(-1)].view(49, 49, nH).permute(2, 0, 1)[:, None]
    if mask is not None:
        want = want + _d(mask)[None]
    _close(bias[..., :49], want.expand_as(bias[..., :49]) / LN2, REL_WA_BIAS, what + " bias table (log2 units)")
    assert float(bias[..., 49:].abs().max()) == 0.0
    out, lse = ops.window_attention_fwd(qkv, nH, bias, shift, scale)
    ref, lse_ref, gq, gt = _wattn_ref(qkv, nH, table, index, mask, shift, scale, dout)
    _close(out, ref, REL_WA_O, what + " out")
    _close(lse, lse_ref, REL_WA_LSE, what + " lse")
    dqkv, dbias = ops.window_attention_bwd(qkv, out, dout, bias, lse, nH, shift, scale)
    for i, name in enumerate("qkv"):
        _close(dqkv[..., i * C:(i + 1) * C], gq[..., i * C:(i + 1) * C], REL_WA_DV if name == "v" else REL_WA_DQK,
               f"{what} d{name}")
    base = torch.randn_like(table)
    dtable = ops.window_bias_scatter(dbias, index, base.clone())
    _close(dtable - base, gt, REL_WA_DTAB, what + " dtable")
    # scatter on its own: the kernel's dbias summed into the table rows in float64
    want_t = _d(base).index_add(0, index.view(-1).cuda(), _d(dbias).permute(1, 2, 0).reshape(49 * 49, nH))
    _close(dtable, want_t, REL_WA_SCATTER, what + " bias scatter")
    out2, lse2 = ops.window_attention_fwd(qkv, nH, bias, shift, scale)
    assert torch.equal(out, out2) and torch.equal(lse, lse2), what + " forward repeat"
    dqkv2, dbias2 = ops.window_attention_bwd(qkv, out, dout, bias, lse, nH, shift, scale)
    assert torch.equal(dqkv, dqkv2), what + " dqkv repeat"
    _close(dbias2, dbias, REL_WA_SCATTER, what + " dbias (atomics) repeat")


@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("nH,H,W", WA_CASES)
def test_window_attention(nH, H, W, shift):
    if shift and H == 7:
        pytest.skip("Swin uses no shift when the resolution equals the window")
    _wattn_case(_wattn_batch(nH, H, W), H, W, nH, shift, seed=nH * 100 + H + shift)


def test_window_attention_pairs_across_images():
    """9 windows per image: with B = 3 the window pairs 4, 9 and 13 hold the last window of one image and the first of the
    next, which sit in different slices of the shift mask."""
    _wattn_case(3, 21, 21, 6, 3, seed=21)


# -------------------------------------------------------------------------------------------------------- depthwise 7x7
REL_DW_16 = 1.2e-2    # bf16 outputs (measured 3.4e-3)
REL_DW_32 = 1.4e-6    # fp32 outputs (measured 3.6e-7)
REL_DW_WGRAD = 1.3e-6  # fp32 sums over B*H*W pixels (measured 3.2e-7)


def _dw64(x, w, flip=False):
    """float64 7x7 depthwise correlation (pad 3) of NHWC x with w [C,1,7,7]; flip=True correlates with the flipped kernel."""
    C = x.shape[-1]
    wd = _d(w).flip(-1, -2) if flip else _d(w)
    return F.conv2d(_d(x).permute(0, 3, 1, 2), wd, None, 1, 3, 1, C).permute(0, 2, 3, 1)


# ConvNeXt-B widths; each on a grid the 14x14-tiled kernels take (H, W multiples of 14) and on one they do not
DW_CASES = [(2, 56, 56, 128), (2, 30, 23, 128), (3, 28, 28, 256), (3, 27, 13, 256), (5, 14, 14, 512), (4, 9, 11, 512),
            (6, 14, 28, 1024), (8, 7, 7, 1024)]


@pytest.mark.parametrize("B,H,W,C", DW_CASES)
def test_dwconv7(B, H, W, C):
    what = f"dwconv7 {B}x{H}x{W}x{C}"
    x = _rand(B, H, W, C, seed=C + H, dtype=F32)
    w = torch.randn(C, 1, 7, 7, device="cuda") * 0.1
    bias = torch.randn(C, device="cuda") * 0.1
    wt = ops.dwconv7_pack(w)
    assert torch.equal(wt, w.view(C, 49).t())
    ref = _dw64(x, w) + _d(bias)
    _close(ops.dwconv7(x, wt, bias), ref, REL_DW_16, what + " fwd f32->bf16")
    add32 = _rand(B, H, W, C, seed=C + H + 1, dtype=F32)
    _close(ops.dwconv7(x, wt, bias, add=add32, out_dtype=F32), ref + _d(add32), REL_DW_32, what + " fwd f32->f32 +add")
    du = _rand(B, H, W, C, seed=C + H + 2)
    g = _rand(B, H, W, C, seed=C + H + 3)
    dref = _dw64(du, w, flip=True)
    _close(ops.dwconv7(du, wt, add=g, out_dtype=BF16, flip=True), dref + _d(g), REL_DW_16, what + " dgrad bf16 +add")
    _close(ops.dwconv7(du, wt, out_dtype=F32, flip=True), dref, REL_DW_32, what + " dgrad f32")
    # dw[c, 0, i, j] = sum_{b,h,w} du[b,h,w,c] * x[b, h+i-3, w+j-3, c]
    xd = F.pad(_d(x).permute(0, 3, 1, 2), (3, 3, 3, 3))
    dud = _d(du).permute(0, 3, 1, 2)
    wref = torch.stack([(xd[:, :, i:i + H, j:j + W] * dud).sum((0, 2, 3)) for i in range(7) for j in range(7)], 1)
    wref = wref.view(C, 1, 7, 7)
    dw = ops.dwconv7_wgrad(du, x)
    _close(dw, wref, REL_DW_WGRAD, what + " wgrad")
    assert torch.equal(ops.dwconv7_wgrad(du, x), dw), what + " wgrad repeat"
    prev = torch.randn(C, 1, 7, 7, device="cuda")
    acc = ops.dwconv7_wgrad(du, x, out=prev.clone(), accumulate=True)
    _close(acc, wref + _d(prev), REL_DW_WGRAD, what + " wgrad accumulate")
    assert torch.equal(ops.dwconv7_wgrad(du, x, out=prev.clone(), accumulate=True), acc), what + " accumulate repeat"


# ------------------------------------------------------------------------------------------------------ small ViT pieces
@pytest.mark.parametrize("ps,Cin,H,W", [(32, 3, 224, 224), (16, 3, 224, 224), (32, 5, 64, 96)])
def test_patchify_nchw_exact(ps, Cin, H, W):
    B = 3
    x = torch.randn(B, Cin, H, W, device="cuda")
    a = ops.patchify_nchw(x, ps)
    Hp, Wp = H // ps, W // ps
    ref = x.view(B, Cin, Hp, ps, Wp, ps).permute(0, 2, 4, 1, 3, 5).reshape(B, Hp * Wp, Cin * ps * ps).to(BF16)
    assert torch.equal(a, ref)


@pytest.mark.parametrize("B,T,D", [(5, 50, 768), (3, 197, 1024), (2, 5, 8)])
def test_cls_row_exact(B, T, D):
    tokens = torch.randn(B, T, D, device="cuda")
    before = tokens.clone()
    cls, pos = torch.randn(D, device="cuda"), torch.randn(T * D, device="cuda")
    ops.cls_row_(tokens, cls, pos)
    assert torch.equal(tokens[:, 0], (cls + pos[:D]).expand(B, D))
    assert torch.equal(tokens[:, 1:], before[:, 1:])


REL_LS_DGAMMA = 4e-7   # fp32 dot products over K = 4096 (measured 1.1e-7)
REL_LS_PROD = 1.6e-7   # dW2, db2: one fp32 product each (measured 4.4e-8)


def test_layerscale_grads_wide():
    """ConvNeXt-B stage 4 / ConvNeXt-XL stage 3: C = 1024, K = 4C."""
    C, K = 1024, 4096
    G = torch.randn(C, K, device="cuda")
    W2 = torch.randn(C, K, device="cuda") * 0.02
    b2 = torch.randn(C, device="cuda") * 0.1
    gsum = torch.randn(C, device="cuda")
    gamma = torch.rand(C, device="cuda") + 0.5
    dW2, db2, dgam = ops.layerscale_grads(G, W2, b2, gsum, gamma)
    _close(dW2, _d(G) * _d(gamma)[:, None], REL_LS_PROD, "dW2")
    _close(db2, _d(gsum) * _d(gamma), REL_LS_PROD, "db2")
    _close(dgam, (_d(W2) * _d(G)).sum(1) + _d(b2) * _d(gsum), REL_LS_DGAMMA, "dgamma")
    assert torch.equal(ops.layerscale_grads(G, W2, b2, gsum, gamma)[2], dgam)
