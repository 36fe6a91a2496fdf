"""Forward / backward schedule of masked-autoencoder pre-training on the sm_90a kernels (one autograd node for the network).

Mirrors ``MAE.forward`` of the reference (self-supervised/MAE/models/MAE.py) with its ``Transformer`` / ``PreNorm`` /
``SelfAttention`` / ``FFN`` blocks (models/VIT.py).  Per sample the P patches are shuffled by the stable argsort of
``torch.rand(B, P)``; the first Nm = int(mask_ratio P) shuffle slots are masked, the other Nv = P - Nm visible.

    keys -> shuffle (ids, slot) -> masked patchify: visible patch rows (bf16) + masked targets (fp32), shuffle order
    patch-embed GEMM (+bias, +pos_embed[ids + 1] gathered) -> encoder blocks over the Nv visible tokens
    -> enc_to_dec GEMM (when a Linear) -> assembly: encoder rows at their patch, mask_embed + decoder_pos_embed elsewhere
    -> decoder blocks over all P tokens -> gather of the masked rows -> head GEMM (fp32 pred)
    loss (TrainStep): fused masked-pixel MSE, which also writes the bf16 gradient of pred

The backward is the exact reverse: head dgrad rows scattered into a zero decoder-output gradient, decoder blocks, assembly
backward (encoder-row gradient, decoder_pos_embed and mask_embed sums over the batch), enc_to_dec, encoder blocks, then the
pos_embed sums and the patch-embed weight gradient.  The blocks are engine/prenorm_block.py, shared with the ViT schedule.
``encoder.cls_token`` and ``encoder.mlp_head`` take no part in pre-training and get no gradient (``params_without_grad``).
"""
import torch
import torch.nn as nn

from .. import ops
from . import common, prenorm_block
from .common import linear_grads
from .packing import weight_cache

BF16 = torch.bfloat16
F32 = torch.float32
MAX_TOKENS = 256   # longest sequence of the attention kernels


def _stacks(model):
    return (("encoder.transformer", model.encoder.transformer), ("decoder", model.decoder))


def _block_args(layer):
    """(norm1, qkv, proj, norm2, fc1, fc2, heads, scale) of one [PreNorm(SelfAttention), PreNorm(FFN)] layer."""
    pa, pf = layer
    att, ffn = pa.net, pf.net.net
    return pa.norm, att.to_qkv, att.out[0], pf.norm, ffn[0], ffn[3], att.num_heads, float(att.scale)


def _linears(model):
    out = [model.encoder.patch_embed]
    for _, stack in _stacks(model):
        for layer in stack.layers:
            out += list(_block_args(layer)[i] for i in (1, 2, 4, 5))
    if isinstance(model.enc_to_dec, nn.Linear):
        out.append(model.enc_to_dec)
    out.append(model.head)
    return out


class _PackSpec:
    @staticmethod
    def key(model):
        return (len(model.encoder.transformer.layers), len(model.decoder.layers), id(model.head),
                isinstance(model.enc_to_dec, nn.Linear))

    def __call__(self, model):
        pe = model.encoder.patch_embed.weight
        specs = [(pe, 0, pe.shape[1], pe.shape[0])]   # (the patch rows get no gradient: no dgrad operand)
        for lin in _linears(model)[1:]:
            w = lin.weight
            specs.append((w, 0, w.shape[1], w.shape[0]))
            specs.append((w, 1, w.shape[0], w.shape[1]))
        return specs


_pack_spec = _PackSpec()


def params_without_grad(model):
    """Parameters the pre-training forward never reads: the classification class token and head of the encoder."""
    return [model.encoder.cls_token, *model.encoder.mlp_head.parameters()]


def _split(model, H, W):
    """(patch size, P, Nm) of an H x W image; NotImplementedError naming the layer for a shape the engine cannot run."""
    enc = model.encoder
    p = enc.patch_h
    if enc.patch_w != p:
        raise NotImplementedError(f"encoder.patch_embed: non-square patches {enc.patch_h}x{enc.patch_w} are not implemented")
    if H % p or W % p:
        raise NotImplementedError(f"encoder.patch_embed: a {H}x{W} image is not divisible by the patch size {p}")
    P = (H // p) * (W // p)
    if P + 1 != enc.pos_embed.shape[-2]:
        raise ValueError(f"encoder.pos_embed: {enc.pos_embed.shape[-2] - 1} patch positions, the {H}x{W} image has {P}")
    Nm = int(model.mask_ratio * P)
    Nv = P - Nm
    if P > MAX_TOKENS or Nv > MAX_TOKENS:
        raise NotImplementedError(f"decoder: {P} patches ({Nv} visible); the attention kernels take at most {MAX_TOKENS} tokens")
    if Nm < 1 or Nv < 1:
        raise NotImplementedError(f"mask_ratio {model.mask_ratio} leaves {Nm} masked and {Nv} visible patches of {P}; "
                                  "both must be at least 1")
    return p, P, Nm


def _check(model, train, want_tape):
    for name, stack in _stacks(model):
        for i, (pa, pf) in enumerate(stack.layers):
            att, ffn = pa.net, pf.net.net
            lname = f"{name}.layers.{i}"
            if not isinstance(att.out, nn.Sequential):
                raise NotImplementedError(f"{lname}.0.net.out: SelfAttention without an output projection (project_out "
                                          "is Identity) is not implemented")
            inner = att.to_qkv.out_features // 3
            if inner != att.num_heads * 64:
                raise NotImplementedError(f"{lname}.0.net: head_dim {inner // max(att.num_heads, 1)}; the attention kernel "
                                          "is built for head_dim 64")
            if not (isinstance(ffn[1], nn.GELU) and ffn[1].approximate == "none"):
                raise NotImplementedError(f"{lname}.1.net.net.1: the FFN activation must be nn.GELU (exact erf)")
            if train:
                for dname, m in ((f"{lname}.0.net.out.1", att.out[1]), (f"{lname}.1.net.net.2", ffn[2]),
                                 (f"{lname}.1.net.net.4", ffn[4])):
                    if m.p != 0:
                        raise NotImplementedError(f"{dname}: dropout > 0 is not implemented on this engine")
    for lin in _linears(model):
        if lin.in_features % 8 or lin.out_features % 8:
            name = next(n for n, m in model.named_modules() if m is lin)
            raise NotImplementedError(f"{name}: Linear {lin.in_features} -> {lin.out_features}; the GEMM kernels take "
                                      "widths that are multiples of 8")
    common.check_layernorm_widths(((f"{name}.{n}", m.normalized_shape[-1]) for name, stack in _stacks(model)
                                   for n, m in stack.named_modules() if isinstance(m, nn.LayerNorm)), want_tape)


def forward(model, x, train, want_tape):
    """Returns ((pred fp32 [B, Nm, K], mask_patches fp32 [B, Nm, K], ids int32 [B, P]), tape or None); K = p*p*C and
    ids[:, :Nm] / ids[:, Nm:] are the reference's mask_indices / unmask_indices."""
    _check(model, train, want_tape)
    H, W = x.shape[1:3] if x.dtype == torch.uint8 else x.shape[2:4]   # (a decoded uint8 batch is NHWC)
    p, P, Nm = _split(model, H, W)
    x = common.image_input(model, x)
    B, C = x.shape[:2]
    Nv = P - Nm
    enc = model.encoder
    if p * p * C != enc.patch_embed.in_features:
        raise ValueError(f"encoder.patch_embed takes {enc.patch_embed.in_features} values per patch; a {C}-channel image "
                         f"with patch {p} has {p * p * C}")
    De = enc.pos_embed.shape[-1]
    pack = weight_cache.model_pack(model, _pack_spec)
    keys = torch.rand(B, P, device=x.device)        # the reference's draw: torch.rand(b, num_patches).argsort()
    ids, slot = ops.mae_shuffle(keys)
    vis, tgt = ops.mae_patchify(x, ids, p, Nm)
    pos = ops.mae_gather_rows(enc.pos_embed.detach().reshape(P + 1, De), ids, Nm, Nv, 0, row_offset=1)
    h, _ = ops.gemm(vis, pack.get(enc.patch_embed.weight, 0), bias=enc.patch_embed.bias, residual=pos, out_f32=True)
    enc_recs, dec_recs = [], []
    for layer in enc.transformer.layers:
        h, rec = prenorm_block.forward(pack, h, *_block_args(layer), 0.0, want_tape)
        enc_recs.append(rec)
    e16 = None
    if isinstance(model.enc_to_dec, nn.Linear):
        e16 = ops.cast_bf16(h)
        h, _ = ops.gemm(e16, pack.get(model.enc_to_dec.weight, 0), bias=model.enc_to_dec.bias, out_f32=True)
    h = ops.mae_assemble_fwd(h, model.mask_embed.detach(), model.decoder_pos_embed.weight.detach(), slot, Nm)
    Dd = h.shape[-1]
    for layer in model.decoder.layers:
        h, rec = prenorm_block.forward(pack, h, *_block_args(layer), 0.0, want_tape)
        dec_recs.append(rec)
    a_head = ops.mae_gather_rows(h.view(B * P, Dd), ids, 0, Nm, P, out_dtype=BF16)
    pred, _ = ops.gemm(a_head, pack.get(model.head.weight, 0), bias=model.head.bias, out_f32=True)
    tape = None
    if want_tape:
        tape = {"pack": pack, "slot": slot, "vis": vis, "e16": e16, "a_head": a_head, "enc": enc_recs, "dec": dec_recs,
                "shape": (B, P, Nm, De, Dd)}
    return (pred, tgt, ids), tape


def train_loss(out, labels, loss_scale):
    """TrainStep's loss: (mean squared error of pred against mask_patches, bf16 gradient of pred, None)."""
    if labels is not None:
        raise ValueError("MAE pre-training takes no labels")
    pred, tgt, _ = out
    loss, dpred = ops.mae_mse(pred, tgt, loss_scale)
    return loss, dpred, None


def backward(model, tape, dpred, sink=None):
    grads = common.Grads(sink)
    pack, slot = tape["pack"], tape["slot"]
    B, P, Nm, De, Dd = tape["shape"]
    Nv = P - Nm
    head, enc = model.head, model.encoder
    K = head.out_features
    M = B * Nm
    if dpred.dtype == BF16 and dpred.is_contiguous():
        dp16 = dpred.view(M, K)        # already produced by the fused MSE kernel
    else:
        dp16 = ops.cast_bf16(dpred.float()).view(M, K)
    linear_grads(grads, head, dp16, tape["a_head"].view(M, Dd))
    dh, _ = ops.gemm(dp16, pack.get(head.weight, 1))
    g = ops.mae_scatter_masked(dh.view(B, Nm, Dd), slot, Nm)
    for rec in reversed(tape["dec"]):
        g = prenorm_block.backward(grads, pack, rec, g)
    dpe = model.decoder_pos_embed.weight
    g, d_dpos = ops.mae_assemble_bwd(g, slot, Nm, d_dpos=grads.dest(dpe))
    grads.put(dpe, d_dpos)
    grads.put(model.mask_embed, ops.batch_rowsum(d_dpos, Dd, P, Dd, out=grads.dest(model.mask_embed)))
    if isinstance(model.enc_to_dec, nn.Linear):
        linear_grads(grads, model.enc_to_dec, g.view(B * Nv, Dd), tape["e16"].view(B * Nv, De))
        g, _ = ops.gemm(g.view(B * Nv, Dd), pack.get(model.enc_to_dec.weight, 1))
        g = g.view(B, Nv, De)
    for rec in reversed(tape["enc"]):
        g = prenorm_block.backward(grads, pack, rec, g)
    dst = grads.dest(enc.pos_embed)
    grads.put(enc.pos_embed, ops.mae_pos_grad(g, slot, Nm, out=None if dst is None else dst.view(P + 1, De)))
    vis = tape["vis"]
    linear_grads(grads, enc.patch_embed, g.view(B * Nv, De), vis.view(B * Nv, vis.shape[-1]))
    return grads


class _MAEFunction(torch.autograd.Function):
    """The whole network as one autograd node with outputs (pred, mask_patches); mask_patches carries no gradient."""

    @staticmethod
    def forward(ctx, x, model, *params):
        want_tape = any(ctx.needs_input_grad[2:])
        (pred, tgt, _), tape = forward(model, x, model.training, want_tape)
        ctx.model, ctx.tape, ctx.params = model, tape, params
        ctx.mark_non_differentiable(tgt)
        return pred, tgt

    @staticmethod
    def backward(ctx, dpred, _dtgt):
        if ctx.tape is None:
            raise RuntimeError("backward called on a forward that recorded no tape")
        grads = backward(ctx.model, ctx.tape, dpred)
        ctx.tape = None
        out = []
        for p, need in zip(ctx.params, ctx.needs_input_grad[2:]):
            gp = grads.get(p.data_ptr()) if need else None
            out.append(gp.reshape(p.shape) if gp is not None else None)
        return (None, None, *out)


def apply(model, x):
    """``model(x)`` of an MAE: (pred, mask_patches), pred differentiable when any parameter needs a gradient."""
    if not x.is_cuda:
        raise RuntimeError("deeplearning_b200 MAE runs on CUDA (sm_90a) tensors only; there is no CPU fallback")
    params = tuple(model.parameters())
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        return _MAEFunction.apply(x, model, *params)
    (pred, tgt, _), _ = forward(model, x, model.training, False)
    return pred, tgt

