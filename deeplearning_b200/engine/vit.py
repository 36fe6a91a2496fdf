"""Forward / backward schedule of the ViT family on the sm_90a kernels (one autograd node for the whole network).

Mirrors ``VisionTransformer.forward_features`` / ``Block.forward`` / ``Attention.forward`` / ``Mlp.forward`` of the
reference (classification/vision_transformer/vit_model.py:240-268, :158-161, :88-111, :127-133).

Data flow per block (residual stream ``h`` fp32 [B,T,D], everything feeding a tensor core bf16; engine/prenorm_block.py):
    LN1(h) -> qkv GEMM(+bias) -> wgmma attention -> proj GEMM(+bias, +h, fp32 out) = h2
    LN2(h2) -> fc1 GEMM(+bias, GELU; also writes GELU'(pre) for the backward) -> fc2 GEMM(+bias, +h2, fp32 out) = h3
Residual adds, biases, GELU, GELU' (backward) and the pos-embed add of the patch embedding all live in GEMM epilogues; the
attention scores never touch HBM.  The gradient of the residual stream is carried in bf16 and accumulated inside the
LayerNorm-backward kernel.
"""
import sys

import torch
import torch.nn as nn

from .. import ops
from . import common, droppath, prenorm_block
from .common import linear_grads, layernorm_backward
from .packing import weight_cache

BF16 = torch.bfloat16
F32 = torch.float32


def _linears(model):
    out = [model.head]
    for blk in model.blocks:
        out += [blk.attn.qkv, blk.attn.proj, blk.mlp.fc1, blk.mlp.fc2]
    if model.has_logits:
        out.append(model.pre_logits.fc)   # Linear + Tanh on the class-token row (vit_model.py:218-221)
    return out


class _PackSpec:
    @staticmethod
    def key(model):
        return (len(model.blocks), id(model.head), model.head.out_features, bool(model.has_logits))

    def __call__(self, model):
        specs = []
        pe = model.patch_embed.proj.weight  # [D, C, p, p]: conv weight.view(D, -1) is already the GEMM operand order
        k0 = pe.numel() // pe.shape[0]
        specs.append((pe, 0, k0, pe.shape[0], (pe.shape[0], k0, 1)))
        for lin in _linears(model)[1:]:
            w = lin.weight
            specs.append((w, 0, w.shape[1], w.shape[0]))
            specs.append((w, 1, w.shape[0], w.shape[1]))
        return specs + common.head_pack_specs(model.head)


_pack_spec = _PackSpec()


def _check(model, want_tape=False):
    if model.dist_token is not None:
        raise NotImplementedError("distilled ViT (dist_token) is not implemented on this engine")
    if model.has_logits and not (isinstance(getattr(model.pre_logits, "fc", None), nn.Linear)
                                 and isinstance(getattr(model.pre_logits, "act", None), nn.Tanh)):
        raise NotImplementedError("pre_logits must be the reference's Sequential(fc=Linear, act=Tanh) (vit_model.py:218-221)")
    if not isinstance(model.head, nn.Linear):
        raise NotImplementedError("model.head must be an nn.Linear (num_classes > 0)")
    for m in model.modules():
        if isinstance(m, nn.Dropout) and m.p != 0 and model.training:
            raise NotImplementedError("dropout > 0 is not implemented on this engine")
    for blk in model.blocks:
        if blk.attn.qkv.in_features // blk.attn.num_heads != 64:
            raise NotImplementedError("the attention kernel is built for head_dim 64")
        if not isinstance(blk.mlp.act, nn.GELU):
            raise NotImplementedError("Mlp activation must be nn.GELU (exact erf)")
    common.check_layernorm_widths(((name, m.normalized_shape[-1]) for name, m in model.named_modules()
                                   if isinstance(m, nn.LayerNorm)), want_tape)


def forward(model, x, train, want_tape):
    _check(model, want_tape)
    x = common.image_input(model, x)
    B, Cin, Hh, Ww = x.shape
    pe = model.patch_embed
    ps = pe.patch_size[0]
    if (Hh, Ww) != tuple(pe.img_size):
        raise AssertionError(f"Input image size ({Hh}*{Ww}) doesn't match model ({pe.img_size[0]}*{pe.img_size[1]}).")
    D = model.embed_dim
    P = pe.num_patches
    T = P + 1
    pack = weight_cache.model_pack(model, _pack_spec)
    tape = {"blocks": [], "pack": pack} if want_tape else None
    # ---- patch embedding: patch matrix GEMM writing rows 1.. of the token tensor, + bias + pos_embed in the epilogue
    a = ops.patchify_nchw(x, ps)                       # bf16 [B, P, Cin*ps*ps]
    K0 = a.shape[-1]
    tokens = torch.empty(B, T, D, dtype=F32, device=x.device)
    pos = model.pos_embed.detach()
    ops.gemm(a, pack.get(pe.proj.weight, 0), bias=pe.proj.bias.detach() if pe.proj.bias is not None else None, out=tokens,
             a_view=((P, B, 1), (K0, P * K0, 0)), out_view=((P, B, 1), (D, T * D, 0)), out_offset=D,
             residual=pos.reshape(T, D)[1:], residual_view=((P, B, 1), (D, 0, 0)))
    ops.cls_row_(tokens, model.cls_token.detach().reshape(-1), pos.reshape(-1))
    h = tokens
    if want_tape:
        tape["patches"] = a
    for blk in model.blocks:
        att_m, mlp = blk.attn, blk.mlp
        h, rec = prenorm_block.forward(pack, h, blk.norm1, att_m.qkv, att_m.proj, blk.norm2, mlp.fc1, mlp.fc2,
                                       att_m.num_heads, float(att_m.scale), droppath.drop_prob_of(blk, train), want_tape)
        if want_tape:
            tape["blocks"].append(rec)
    # ---- head: final LayerNorm on the class-token rows only, then the classifier (fp32 logits)
    cls_rows = torch.empty(B, D, dtype=F32, device=x.device)
    ops.copy_rows(h, 0, T * D, cls_rows, 0, D, B, D)
    yc, mc, rc = ops.layernorm_fwd(cls_rows, model.norm.weight, model.norm.bias, model.norm.eps)
    feat, t32 = yc, None          # classifier input (bf16 [B, R])
    if model.has_logits:          # pre_logits: tanh(fc(cls row))  (vit_model.py:218-221,254)
        fc = model.pre_logits.fc
        u, _ = ops.gemm(yc, pack.get(fc.weight, 0), bias=fc.bias, out_f32=True)
        t32, feat = ops.tanh_fwd(u)
    logits = common.head_forward(pack, model.head, feat)
    if want_tape:
        tape["head"] = (cls_rows, yc, mc, rc, (B, T, D, P), feat, t32)
    return logits, tape


def backward(model, tape, dlogits, sink=None):
    grads = common.Grads(sink)
    pack = tape["pack"]
    cls_rows, yc, mc, rc, (B, T, D, P), feat, t32 = tape["head"]
    d_yc = common.head_backward(grads, pack, model.head, feat, dlogits)
    if model.has_logits:
        fc = model.pre_logits.fc
        du = ops.tanh_bwd(d_yc, t32)                      # bf16 [B, R]: d tanh
        linear_grads(grads, fc, du, yc)
        d_yc, _ = ops.gemm(du, pack.get(fc.weight, 1))    # bf16 [B, D]
    d_cls = layernorm_backward(grads, model.norm, d_yc, cls_rows, mc, rc)
    g = torch.zeros(B, T, D, dtype=BF16, device=d_cls.device)   # gradient of the residual stream
    ops.copy_rows(d_cls, 0, D, g, 0, T * D, B, D)
    for rec in reversed(tape["blocks"]):
        g = prenorm_block.backward(grads, pack, rec, g)
    # ---- embedding: tokens = [cls ; patches W^T + b] + pos
    grads.put(model.pos_embed, ops.batch_rowsum(g, T * D, B, T * D, out=_flat(grads.dest(model.pos_embed))))
    grads.put(model.cls_token, ops.batch_rowsum(g, T * D, B, D, out=_flat(grads.dest(model.cls_token))))
    gp = torch.empty(B, P, D, dtype=BF16, device=g.device)
    ops.copy_rows(g, D, T * D, gp, 0, P * D, B, P * D)          # drop the class-token rows
    a = tape["patches"]
    linear_grads(grads, model.patch_embed.proj, gp.view(B * P, D), a.view(B * P, a.shape[-1]))
    return grads


def _flat(t):
    return None if t is None else t.view(-1)


def apply(model, x):
    return common.apply(sys.modules[__name__], "ViT", model, x)
