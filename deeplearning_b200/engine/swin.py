"""Forward / backward schedule of the Swin Transformer on the sm_90a kernels (one autograd node for the whole network).

Mirrors ``SwinTransformer.forward_features`` / ``BasicLayer.forward`` / ``SwinTransformerBlock.forward`` /
``WindowAttention.forward`` / ``PatchMerging.forward`` of the reference
(classification/swin_transformer/models/swin_transformer.py:579-597, :406-415, :241-287, :118-149, :324-345).

Data flow per block (residual stream ``h`` fp32 [B, H*W, C] in natural pixel order; tensor-core operands bf16):
    LN1(h) -> qkv GEMM(+bias) -> shifted-window attention (roll, partition, bias, mask, softmax, reverse, un-roll all inside
    one wgmma kernel that gathers its 49-token windows straight from the pixel-ordered qkv tensor)
    -> proj GEMM(+bias, +h, fp32 out) = h2 -> LN2 -> fc1 GEMM(+bias, GELU, keeps GELU'(pre)) -> fc2 GEMM(+bias, +h2) = h3
PatchMerging = one gather+LayerNorm kernel (the 2x2 concat never exists in HBM) + the bias-free reduction GEMM (fp32 out).
"""
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common, droppath
from .common import linear_grads, layernorm_backward
from .packing import weight_cache

F32 = torch.float32


def _blocks(model):
    for layer in model.layers:
        for blk in layer.blocks:
            yield blk


class _PackSpec:
    @staticmethod
    def key(model):
        return (tuple(len(l.blocks) for l in model.layers), id(model.head), model.head.out_features)

    def __call__(self, model):
        specs = []
        pe = model.patch_embed.proj.weight
        k0 = pe.numel() // pe.shape[0]
        specs.append((pe, 0, k0, pe.shape[0], (pe.shape[0], k0, 1)))
        for layer in model.layers:
            lins = []
            for blk in layer.blocks:
                lins += [blk.attn.qkv, blk.attn.proj, blk.mlp.fc1, blk.mlp.fc2]
            if layer.downsample is not None:
                lins.append(layer.downsample.reduction)
            for lin in lins:
                w = lin.weight
                specs.append((w, 0, w.shape[1], w.shape[0]))
                specs.append((w, 1, w.shape[0], w.shape[1]))
        return specs + common.head_pack_specs(model.head)


_pack_spec = _PackSpec()


def _check(model, want_tape=False):
    if model.ape:
        raise NotImplementedError("absolute position embedding (ape=True) is not implemented on this engine")
    if model.patch_embed.norm is None:
        raise NotImplementedError("patch_norm=False is not implemented on this engine")
    if not isinstance(model.head, nn.Linear):
        raise NotImplementedError("model.head must be an nn.Linear (num_classes > 0)")
    if model.training:
        for m in model.modules():
            if isinstance(m, nn.Dropout) and m.p != 0:
                raise NotImplementedError("dropout > 0 is not implemented on this engine")
    for blk in _blocks(model):
        if blk.window_size != 7 or blk.dim // blk.num_heads != 32:
            raise NotImplementedError("the window-attention kernel is built for window_size 7 and head_dim 32")
        if not isinstance(blk.mlp.act, nn.GELU):
            raise NotImplementedError("Mlp activation must be nn.GELU (exact erf)")
    for i, layer in enumerate(model.layers):
        if layer.downsample is not None and 4 * layer.dim > ops.PATCH_MERGE_LN_MAX_C:
            raise NotImplementedError(f"layers.{i}.downsample: patch merging of {layer.dim} channels runs a LayerNorm over "
                                      f"4 * {layer.dim} = {4 * layer.dim}; the patch-merge kernels take at most "
                                      f"{ops.PATCH_MERGE_LN_MAX_C}")
    # (a patch merge's own LayerNorm runs on the patch-merge kernels, checked above)
    common.check_layernorm_widths(((name, m.normalized_shape[-1]) for name, m in model.named_modules()
                                   if isinstance(m, nn.LayerNorm) and not name.endswith("downsample.norm")), want_tape)


def forward(model, x, train, want_tape):
    _check(model, want_tape)
    x = common.image_input(model, x)
    B, Cin, Hi, Wi = x.shape
    pe = model.patch_embed
    if (Hi, Wi) != tuple(pe.img_size):
        raise AssertionError(f"Input image size ({Hi}*{Wi}) doesn't match model ({pe.img_size[0]}*{pe.img_size[1]}).")
    pack = weight_cache.model_pack(model, _pack_spec)
    tape = {"layers": [], "pack": pack} if want_tape else None
    # ---- patch embedding: 4x4/4 conv as a patch-matrix GEMM (+bias), then LayerNorm into the fp32 residual stream
    a = ops.patchify_nchw(x, pe.patch_size[0])
    u0, _ = ops.gemm(a, pack.get(pe.proj.weight, 0), bias=pe.proj.bias)
    h, m0, r0 = ops.layernorm_fwd(u0, pe.norm.weight, pe.norm.bias, pe.norm.eps, out_dtype=F32)
    if want_tape:
        tape["embed"] = (a, u0, m0, r0)
    H, W = pe.patches_resolution
    for layer in model.layers:
        C = layer.dim
        recs = []
        for blk in layer.blocks:
            att_m, mlp = blk.attn, blk.mlp
            nH = att_m.num_heads
            y1, m1, r1 = ops.layernorm_fwd(h, blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
            qkv, _ = ops.gemm(y1, pack.get(att_m.qkv.weight, 0), bias=att_m.qkv.bias)
            bias = ops.window_bias_gather(att_m.relative_position_bias_table.detach(), att_m.relative_position_index, nH,
                                          blk.attn_mask)   # bias (+ shift mask) table, query index innermost
            att, lse = ops.window_attention_fwd(qkv.view(B, H, W, 3 * C), nH, bias, blk.shift_size, float(att_m.scale))
            dp = droppath.drop_prob_of(blk, train)
            dp1 = droppath.sample_scale(dp, B, 3, x.device)   # x = shortcut + drop_path(x)         (swin_transformer.py:282)
            h2, _ = ops.gemm(att.view(B, H * W, C), pack.get(att_m.proj.weight, 0), bias=att_m.proj.bias, residual=h,
                             out_f32=True, rowscale=None if dp1 is None else (dp1, H * W))
            y2, m2, r2 = ops.layernorm_fwd(h2, blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
            post, dact = ops.gemm(y2, pack.get(mlp.fc1.weight, 0), bias=mlp.fc1.bias, act=2, aux_out=want_tape)
            dp2 = droppath.sample_scale(dp, B, 3, x.device)   # x = x + drop_path(mlp(norm2(x)))    (swin_transformer.py:285)
            h3, _ = ops.gemm(post, pack.get(mlp.fc2.weight, 0), bias=mlp.fc2.bias, residual=h2, out_f32=True,
                             rowscale=None if dp2 is None else (dp2, H * W))
            if want_tape:
                recs.append((blk, h, y1, m1, r1, qkv, bias, att, lse, h2, y2, m2, r2, dact, post, dp1, dp2))
            h = h3
        merge = None
        if layer.downsample is not None:
            ds = layer.downsample
            ym, mm, rm = ops.patch_merge_ln_fwd(h.view(B, H, W, C), ds.norm.weight, ds.norm.bias, ds.norm.eps)
            hn, _ = ops.gemm(ym, pack.get(ds.reduction.weight, 0), out_f32=True)
            merge = (ds, h, ym, mm, rm)
            h = hn.view(B, (H // 2) * (W // 2), 2 * C)
        if want_tape:
            tape["layers"].append((recs, merge, (H, W, C)))
        if layer.downsample is not None:
            H, W = H // 2, W // 2
    # ---- head: LayerNorm -> mean over tokens -> classifier (fp32 logits)
    Cf = h.shape[-1]
    yn, mn, rn = ops.layernorm_fwd(h, model.norm.weight, model.norm.bias, model.norm.eps)
    pooled = ops.cast_bf16(ops.avgpool_any(yn.view(B, H, W, Cf)))
    logits = common.head_forward(pack, model.head, pooled)
    if want_tape:
        tape["head"] = (h, mn, rn, pooled, (B, H, W, Cf))
    return logits, tape


def backward(model, tape, dlogits, sink=None):
    grads = common.Grads(sink)
    pack = tape["pack"]
    h_last, mn, rn, pooled, (B, H, W, Cf) = tape["head"]
    d_yn = ops.avgpool_bwd(common.head_backward(grads, pack, model.head, pooled, dlogits), (H, W))
    g = layernorm_backward(grads, model.norm, d_yn.view(B, H * W, Cf), h_last, mn, rn)
    for recs, merge, (H, W, C) in reversed(tape["layers"]):
        if merge is not None:
            ds, h_in, ym, mm, rm = merge
            Mo = ym.shape[0]
            g2 = g.view(Mo, 2 * C)
            linear_grads(grads, ds.reduction, g2, ym)
            d_ym, _ = ops.gemm(g2, pack.get(ds.reduction.weight, 1))
            g, dgm, dbm = ops.patch_merge_ln_bwd(d_ym, h_in.view(B, H, W, C), mm, rm, ds.norm.weight,
                                                 dgamma=grads.dest(ds.norm.weight), dbeta=grads.dest(ds.norm.bias))
            grads.put(ds.norm.weight, dgm)
            grads.put(ds.norm.bias, dbm)
        M = B * H * W
        g = g.view(B, H * W, C)
        for (blk, h, y1, m1, r1, qkv, bias, att, lse, h2, y2, m2, r2, dact, post, dp1, dp2) in reversed(recs):
            att_m, mlp = blk.attn, blk.mlp
            nH = att_m.num_heads
            # (stochastic depth: the branch sees the per-sample scaled gradient, the identity path - `add=g` - the full one)
            g2 = (g if dp2 is None else ops.rowscale(g, dp2)).view(M, C)
            linear_grads(grads, mlp.fc2, g2, post.view(M, -1))
            d_pre, _, st_pre = ops.gemm(g2, pack.get(mlp.fc2.weight, 1), act=3, aux_in=dact.view(M, -1), want_stats=True)
            linear_grads(grads, mlp.fc1, d_pre, y2.view(M, C), dy_stats=st_pre)
            d_y2, _ = ops.gemm(d_pre, pack.get(mlp.fc1.weight, 1))
            g = layernorm_backward(grads, blk.norm2, d_y2, h2, m2, r2, add=g)
            g2 = (g if dp1 is None else ops.rowscale(g, dp1)).view(M, C)
            linear_grads(grads, att_m.proj, g2, att.view(M, C))
            d_att, _ = ops.gemm(g2, pack.get(att_m.proj.weight, 1))
            dqkv, dbias = ops.window_attention_bwd(qkv.view(B, H, W, 3 * C), att, d_att.view(B, H, W, C), bias, lse, nH,
                                                   blk.shift_size, float(att_m.scale))
            table = att_m.relative_position_bias_table
            dt = grads.dest(table)
            dt = dt.zero_() if dt is not None else torch.zeros_like(table, dtype=F32)
            grads.put(table, ops.window_bias_scatter(dbias, att_m.relative_position_index, dt))
            linear_grads(grads, att_m.qkv, dqkv.view(M, 3 * C), y1.view(M, C))
            d_y1, _ = ops.gemm(dqkv.view(M, 3 * C), pack.get(att_m.qkv.weight, 1))
            g = layernorm_backward(grads, blk.norm1, d_y1, h, m1, r1, add=g)
            g = g.view(B, H * W, C)
    # ---- patch embedding: h0 = LN(patches W^T + b)
    a, u0, m0, r0 = tape["embed"]
    pe = model.patch_embed
    du0 = layernorm_backward(grads, pe.norm, g, u0, m0, r0)
    D = u0.shape[-1]
    rows = u0.numel() // D
    linear_grads(grads, pe.proj, du0.view(rows, D), a.view(rows, a.shape[-1]))
    return grads


def apply(model, x):
    return common.apply(sys.modules[__name__], "Swin", model, x)
