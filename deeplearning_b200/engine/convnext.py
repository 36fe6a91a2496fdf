"""Forward / backward schedule of the ConvNeXt family on the sm_90a kernels (one autograd node for the whole network).

Mirrors ``ConvNeXt.forward_features`` / ``Block.forward`` of the reference (classification/convNext/models/networks.py:160-170,
:92-105).  The residual stream ``x`` is fp32 NHWC; everything feeding a tensor core is bf16:

    stem      patch matrix (4x4) GEMM + bias -> LayerNorm -> x
    Block     u = dwconv7x7(x)+b (CUDA cores) -> y = LN(u) -> GELU(y W1^T + b1) (its derivative kept) ->
              x' = x + gamma * (. W2^T + b2)        (bias, layer scale and the residual add live in the GEMM epilogue)
    downsample  LN(x) -> 2x2/s2 conv as a 4-tap implicit GEMM writing the fp32 stream
    head      mean over H,W -> LayerNorm -> Linear (fp32 logits)

Backward folds the layer scale into the dgrad operand of pwconv2 (packed copy scaled by gamma), applies GELU' in that GEMM's
epilogue, and derives dgamma / dW2 / db2 from the *unscaled* weight gradient G = g^T post (dgamma_c = <W2_c, G_c> + b2_c sum(g_c)),
so the pre-scale activation is never stored.  Stochastic depth (``drop_path``, reference :11-26,104): the per-sample
multiplier of engine/droppath.py scales the branch in the pwconv2 epilogue (before the shortcut add) and the gradient
entering the branch in the backward pass.
"""
import sys
import weakref

import torch
import torch.nn as nn

from .. import ops
from . import common, droppath
from .common import linear_grads, layernorm_backward
from .packing import weight_cache

BF16 = torch.bfloat16
F32 = torch.float32


class _PackSpec:
    @staticmethod
    def key(model):
        return (tuple(len(s) for s in model.stages), id(model.head), model.head.out_features)

    def __call__(self, model):
        specs = []
        stem = model.downsample_layers[0][0].weight  # [C0, 3, 4, 4] consumed as a flat [C0][48] matrix (c, kh, kw order)
        k0 = stem.numel() // stem.shape[0]
        specs.append((stem, 0, k0, stem.shape[0], (stem.shape[0], k0, 1)))
        for i in range(1, 4):
            w = model.downsample_layers[i][1].weight  # [Cout, Cin, 2, 2]
            O, I = w.shape[0], w.shape[1]
            specs.append((w, 0, 4 * I, O))
            specs.append((w, 1, 4 * O, I))
        for stage in model.stages:
            for blk in stage:
                w1, w2 = blk.pwconv1.weight, blk.pwconv2.weight
                specs.append((w1, 0, w1.shape[1], w1.shape[0]))
                specs.append((w1, 1, w1.shape[0], w1.shape[1]))
                specs.append((w2, 0, w2.shape[1], w2.shape[0]))
                # dgrad operand of pwconv2 with the layer scale folded in: [4C][C] * gamma[c]
                specs.append((w2, 1, w2.shape[0], w2.shape[1], None, blk.gamma))
        return specs + common.head_pack_specs(model.head)


_pack_spec = _PackSpec()


def _check(model, want_tape=False):
    if not isinstance(model.head, nn.Linear):
        raise NotImplementedError("model.head must be an nn.Linear")
    common.check_layernorm_widths(((name, m.normalized_shape[-1]) for name, m in model.named_modules()
                                   if hasattr(m, "normalized_shape")), want_tape)


class _DwCache:
    """tap-major fp32 copies of the depthwise weights (tiny), refreshed with the same stamps as the bf16 packs."""

    def __init__(self):
        self.store = {}

    def get(self, param):
        stamp = (param._version, param.data_ptr(), weight_cache.generation)
        hit = self.store.get(id(param))
        # id() and the device address of a freed parameter can both be recycled by a NEW model: the entry is only valid
        # while the very same parameter object is alive
        if hit is not None and hit[0] == stamp and hit[2]() is param:
            return hit[1]
        wt = ops.dwconv7_pack(param)
        key = id(param)
        self.store[key] = (stamp, wt, weakref.ref(param, lambda _r, k=key, st=self.store: st.pop(k, None)))
        return wt


_dw_cache = _DwCache()


def forward(model, x, train, want_tape):
    _check(model, want_tape)
    x = common.image_input(model, x)
    B = x.shape[0]
    pack = weight_cache.model_pack(model, _pack_spec)
    tape = {"stages": [], "pack": pack} if want_tape else None
    # ---- stem
    stem_conv, stem_ln = model.downsample_layers[0][0], model.downsample_layers[0][1]
    ps = stem_conv.kernel_size[0]
    a = ops.patchify_nchw(x, ps)                                  # bf16 [B, P, 3*ps*ps]
    Hs, Ws = x.shape[2] // ps, x.shape[3] // ps
    C0 = stem_conv.out_channels
    u0, _ = ops.gemm(a, pack.get(stem_conv.weight, 0), bias=stem_conv.bias)   # bf16 [B, P, C0]
    h, m0, r0 = ops.layernorm_fwd(u0, stem_ln.weight, stem_ln.bias, stem_ln.eps, out_dtype=F32)
    h = h.view(B, Hs, Ws, C0)
    if want_tape:
        tape["stem"] = (a, u0, m0, r0)
    for i in range(4):
        rec = {"down": None, "blocks": []}
        if i > 0:
            ln, conv = model.downsample_layers[i][0], model.downsample_layers[i][1]
            y, m, r = ops.layernorm_fwd(h, ln.weight, ln.bias, ln.eps)            # bf16
            h_new = ops.conv2d_fwd_f32(y, pack.get(conv.weight, 0), 2, 2, bias=conv.bias)
            rec["down"] = (h, y, m, r)
            h = h_new
        for blk in model.stages[i]:
            Bb, H, W, C = h.shape
            u = ops.dwconv7(h, _dw_cache.get(blk.dwconv.weight), blk.dwconv.bias)       # bf16 NHWC
            y, m, r = ops.layernorm_fwd(u, blk.norm.weight, blk.norm.bias, blk.norm.eps)
            post, dact = ops.gemm(y.view(-1, C), pack.get(blk.pwconv1.weight, 0), bias=blk.pwconv1.bias, act=2, aux_out=want_tape)
            dps = droppath.sample_scale(droppath.drop_prob_of(blk, train), Bb, 4, h.device)   # x = shortcut + drop_path(x)
            h_new, _ = ops.gemm(post, pack.get(blk.pwconv2.weight, 0), bias=blk.pwconv2.bias, colscale=blk.gamma,
                                residual=h, out_f32=True, rowscale=None if dps is None else (dps, H * W))
            if want_tape:
                rec["blocks"].append((blk, h, u, m, r, y, dact, post, dps))
            h = h_new.view(Bb, H, W, C)
        if want_tape:
            tape["stages"].append(rec)
    # ---- head
    pooled = ops.avgpool_any(h)                                    # fp32 [B, C]
    yc, mc, rc = ops.layernorm_fwd(pooled, model.norm.weight, model.norm.bias, model.norm.eps)
    logits = common.head_forward(pack, model.head, yc)
    if want_tape:
        tape["head"] = (pooled, yc, mc, rc, tuple(h.shape))
    return logits, tape


def backward(model, tape, dlogits, sink=None):
    grads = common.Grads(sink)
    pack = tape["pack"]
    pooled, yc, mc, rc, (B, Hf, Wf, Cf) = tape["head"]
    d_yc = common.head_backward(grads, pack, model.head, yc, dlogits)
    d_pool = layernorm_backward(grads, model.norm, d_yc, pooled, mc, rc)
    g = ops.avgpool_bwd(d_pool, (Hf, Wf))                          # bf16 [B, Hf, Wf, Cf]: gradient of the stream
    for i in range(3, -1, -1):
        rec = tape["stages"][i]
        for (blk, h, u, m, r, y, dact, post, dps) in reversed(rec["blocks"]):
            Bb, H, W, C = h.shape
            M = Bb * H * W
            # the gradient entering the residual branch carries the sample's stochastic-depth multiplier; the identity path keeps g
            g2 = (g if dps is None else ops.rowscale(g, dps)).view(M, C)
            # x' = x + gamma * (post W2^T + b2)
            gsum = torch.empty(C, dtype=F32, device=g2.device)   # column sums of g2, from the wgrad kernel's dy tiles
            G = ops.conv2d_wgrad(g2.view(M, 1, 1, C), post.view(M, 1, 1, 4 * C), bias_out=gsum).view(C, 4 * C)   # unscaled g^T post
            dW2, db2, dgam = ops.layerscale_grads(G, blk.pwconv2.weight.detach(), blk.pwconv2.bias, gsum, blk.gamma,
                                                  dW2=grads.dest(blk.pwconv2.weight), db2=grads.dest(blk.pwconv2.bias),
                                                  dgamma=grads.dest(blk.gamma) if blk.gamma is not None else None)
            grads.put(blk.pwconv2.weight, dW2)
            grads.put(blk.pwconv2.bias, db2)
            if blk.gamma is not None:
                grads.put(blk.gamma, dgam)
            # (g*gamma) W2, times GELU'(pre); the epilogue also sums the columns of d_pre (= pwconv1 bias gradient)
            d_pre, _, st_pre = ops.gemm(g2, pack.get(blk.pwconv2.weight, 1), act=3, aux_in=dact, want_stats=True)
            linear_grads(grads, blk.pwconv1, d_pre, y.view(M, C), dy_stats=st_pre)
            d_y, _ = ops.gemm(d_pre, pack.get(blk.pwconv1.weight, 1))
            du = layernorm_backward(grads, blk.norm, d_y, u.view(M, C), m, r)
            du4 = du.view(Bb, H, W, C)
            grads.put(blk.dwconv.weight, ops.dwconv7_wgrad(du4, h, out=grads.dest(blk.dwconv.weight)))
            grads.put(blk.dwconv.bias, ops.colsum_tall(du, out=grads.dest(blk.dwconv.bias)))
            g = ops.dwconv7(du4, _dw_cache.get(blk.dwconv.weight), add=g, out_dtype=BF16, flip=True)   # g + dwconv^T(du)
        if rec["down"] is not None:
            h_prev, y, m, r = rec["down"]
            ln, conv = model.downsample_layers[i][0], model.downsample_layers[i][1]
            Bb, Ho, Wo, Co = g.shape
            gb = grads.dest(conv.bias)
            if gb is None:
                gb = torch.empty(Co, dtype=F32, device=g.device)
            grads.put(conv.weight, ops.conv2d_wgrad(g, y, 2, 2, out=grads.dest(conv.weight), bias_out=gb))
            grads.put(conv.bias, gb)
            d_y = ops.conv2d_dgrad(g, pack.get(conv.weight, 1), tuple(h_prev.shape[1:3]), 2, 2)
            Cp = h_prev.shape[3]
            g = layernorm_backward(grads, ln, d_y.view(-1, Cp), h_prev.view(-1, Cp), m, r).view(h_prev.shape)
    # ---- stem
    a, u0, m0, r0 = tape["stem"]
    stem_conv, stem_ln = model.downsample_layers[0][0], model.downsample_layers[0][1]
    C0 = stem_conv.out_channels
    du0 = layernorm_backward(grads, stem_ln, g.view(-1, C0), u0.view(-1, C0), m0, r0)
    linear_grads(grads, stem_conv, du0, a.view(du0.shape[0], a.shape[-1]))
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "ConvNeXt", model, x)
