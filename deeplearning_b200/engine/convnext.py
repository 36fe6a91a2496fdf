"""Forward / backward schedule of the ConvNeXt family on the sm_90a kernels (one autograd.Function for the whole network).

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
import weakref

import torch
import torch.nn as nn

from .. import ops
from . import droppath
from .packing import weight_cache
from .resnet import _Grads

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
        head = model.head
        n_pad = (head.out_features + 7) // 8 * 8
        specs.append((head.weight, 0, head.in_features, n_pad))
        specs.append((head.weight, 1, n_pad, head.in_features))
        return specs


_pack_spec = _PackSpec()


def _check(model):
    if not isinstance(model.head, nn.Linear):
        raise NotImplementedError("model.head must be an nn.Linear")


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
    _check(model)
    if x.dtype == torch.uint8:      # GPU input pipeline: decoded uint8 NHWC batch -> ToTensor + Normalize on the device
        x = ops.normalize_u8_nhwc(x, *getattr(model, "input_norm", (ops.IMAGENET_MEAN, ops.IMAGENET_STD)))
    x = x.contiguous().float()
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
    head = model.head
    n_cls = head.out_features
    n_pad = (n_cls + 7) // 8 * 8
    bias = None
    if head.bias is not None:
        bias = head.bias.detach()
        if n_pad != n_cls:
            bias = torch.cat([bias, bias.new_zeros(n_pad - n_cls)])
    D = pooled.shape[1]
    logits, _ = ops.conv2d_fwd(yc.view(B, 1, 1, D), pack.get(head.weight, 0), bias=bias, out_f32=True)
    logits = logits.view(B, n_pad)
    if want_tape:
        tape["head"] = (pooled, yc, mc, rc, n_cls, n_pad, tuple(h.shape))
    return (logits[:, :n_cls] if n_pad != n_cls else logits), tape


def _lin_wgrad(grads, lin, dy2d, x2d, dy_stats=None):
    M, N = dy2d.shape
    K = x2d.shape[1]
    dst = grads.dest(lin.weight)
    gb = None
    if lin.bias is not None and dy_stats is None:
        gb = grads.dest(lin.bias)      # bias gradient summed inside the wgrad kernel (no pass over dy)
        if gb is None:
            gb = torch.empty(N, dtype=F32, device=dy2d.device)
    gw = ops.conv2d_wgrad(dy2d.view(M, 1, 1, N), x2d.view(M, 1, 1, K), out=dst.view(N, K, 1, 1) if dst is not None else None,
                          bias_out=gb)
    grads.put(lin.weight, gw)
    if lin.bias is not None:
        if dy_stats is not None:   # column sums already produced by the epilogue of the GEMM that wrote dy
            grads.put(lin.bias, ops.stats_colsum(dy_stats, out=grads.dest(lin.bias)))
        else:
            grads.put(lin.bias, gb)


def backward(model, tape, dlogits, sink=None):
    grads = _Grads(sink)
    pack = tape["pack"]
    pooled, yc, mc, rc, n_cls, n_pad, (B, Hf, Wf, Cf) = tape["head"]
    head = model.head
    if dlogits.dtype == BF16 and dlogits.shape[1] == n_pad and dlogits.is_contiguous():
        dl16 = dlogits
    else:
        dl = dlogits.contiguous().float()
        if n_pad != n_cls:
            dl = torch.cat([dl, dl.new_zeros(B, n_pad - n_cls)], 1).contiguous()
        dl16 = ops.cast_bf16(dl)
    dst = grads.dest(head.weight)
    if dst is not None and n_pad == n_cls:
        grads.put(head.weight, ops.conv2d_wgrad(dl16.view(B, 1, 1, n_pad), yc.view(B, 1, 1, Cf), out=dst.view(n_cls, Cf, 1, 1)))
    else:
        gw = ops.conv2d_wgrad(dl16.view(B, 1, 1, n_pad), yc.view(B, 1, 1, Cf)).view(n_pad, Cf)[:n_cls]
        if dst is not None:
            dst.copy_(gw)
            gw = dst
        grads.put(head.weight, gw)
    if head.bias is not None:
        grads.put(head.bias, ops.colsum(dl16, cols=n_cls, out=grads.dest(head.bias)))
    d_yc = ops.conv2d_dgrad(dl16.view(B, 1, 1, n_pad), pack.get(head.weight, 1), (1, 1)).view(B, Cf)
    d_pool, dgn, dbn = ops.layernorm_bwd(d_yc, pooled, mc, rc, model.norm.weight, dx_dtype=BF16,
                                         dgamma=grads.dest(model.norm.weight), dbeta=grads.dest(model.norm.bias))
    grads.put(model.norm.weight, dgn)
    grads.put(model.norm.bias, dbn)
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
            _lin_wgrad(grads, blk.pwconv1, d_pre, y.view(M, C), dy_stats=st_pre)
            d_y, _ = ops.gemm(d_pre, pack.get(blk.pwconv1.weight, 1))
            du, dgl, dbl = ops.layernorm_bwd(d_y, u.view(M, C), m, r, blk.norm.weight, dx_dtype=BF16,
                                             dgamma=grads.dest(blk.norm.weight), dbeta=grads.dest(blk.norm.bias))
            grads.put(blk.norm.weight, dgl)
            grads.put(blk.norm.bias, dbl)
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
            g2, dgl, dbl = ops.layernorm_bwd(d_y.view(-1, Cp), h_prev.view(-1, Cp), m, r, ln.weight, dx_dtype=BF16,
                                             dgamma=grads.dest(ln.weight), dbeta=grads.dest(ln.bias))
            grads.put(ln.weight, dgl)
            grads.put(ln.bias, dbl)
            g = g2.view(h_prev.shape)
    # ---- stem
    a, u0, m0, r0 = tape["stem"]
    stem_conv, stem_ln = model.downsample_layers[0][0], model.downsample_layers[0][1]
    C0 = stem_conv.out_channels
    du0, dgl, dbl = ops.layernorm_bwd(g.view(-1, C0), u0.view(-1, C0), m0, r0, stem_ln.weight, dx_dtype=BF16,
                                      dgamma=grads.dest(stem_ln.weight), dbeta=grads.dest(stem_ln.bias))
    grads.put(stem_ln.weight, dgl)
    grads.put(stem_ln.bias, dbl)
    K0 = a.shape[-1]
    Mp = du0.shape[0]
    dst = grads.dest(stem_conv.weight)
    gb = grads.dest(stem_conv.bias)
    if gb is None:
        gb = torch.empty(C0, dtype=F32, device=du0.device)
    gw = ops.conv2d_wgrad(du0.view(Mp, 1, 1, C0), a.view(Mp, 1, 1, K0), out=dst.view(C0, K0, 1, 1) if dst is not None else None,
                          bias_out=gb)
    grads.put(stem_conv.weight, gw)
    grads.put(stem_conv.bias, gb)
    return grads


class _Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, model, *params):
        want_tape = any(ctx.needs_input_grad[2:])
        logits, tape = forward(model, x, model.training, want_tape)
        ctx.model, ctx.tape, ctx.params = model, tape, params
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        if ctx.tape is None:
            raise RuntimeError("backward called on a forward that recorded no tape")
        grads = backward(ctx.model, ctx.tape, dlogits)
        ctx.tape = None
        out = []
        for p, need in zip(ctx.params, ctx.needs_input_grad[2:]):
            gp = grads.get(p.data_ptr()) if need else None
            out.append(gp.reshape(p.shape) if gp is not None else None)
        return (None, None, *out)


def apply(model, x):
    if not x.is_cuda:
        raise RuntimeError("deeplearning_b200 ConvNeXt runs on CUDA (sm_90a) tensors only; there is no CPU fallback")
    params = tuple(model.parameters())
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        return _Function.apply(x, model, *params)
    logits, _ = forward(model, x, model.training, False)
    return logits
