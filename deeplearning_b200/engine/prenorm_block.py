"""One pre-norm transformer block on the sm_90a kernels, shared by the ViT and MAE schedules.

    h2 = h + proj(attention(qkv(LN1(h))))        (x = x + drop_path(attn(norm1(x))))
    h3 = h2 + fc2(GELU(fc1(LN2(h2))))            (x = x + drop_path(mlp(norm2(x))))

The residual stream ``h`` is fp32 [B, T, D]; everything feeding a tensor core is bf16.  Residual adds, biases, GELU, GELU'
(backward) and the stochastic-depth multipliers live in GEMM epilogues; the attention scores never touch HBM.  The attention
width ``heads * 64`` may differ from D, and any Linear may come without a bias.  The gradient of the residual stream is
carried in bf16 and accumulated inside the LayerNorm-backward kernel.
"""
from .. import ops
from . import droppath
from .common import layernorm_backward, linear_grads


def forward(pack, h, norm1, qkv, proj, norm2, fc1, fc2, heads, scale, drop_prob=0.0, want_tape=False):
    """h fp32 [B, T, D] -> (h3 fp32 [B, T, D], tape record or None).  ``drop_prob``: stochastic depth of both branches,
    one per-sample draw each, attention branch first."""
    B, T, _ = h.shape
    y1, m1, r1 = ops.layernorm_fwd(h, norm1.weight, norm1.bias, norm1.eps)
    qkv_t, _ = ops.gemm(y1, pack.get(qkv.weight, 0), bias=qkv.bias)
    att, lse = ops.attention_fwd(qkv_t, heads, scale)
    dp1 = droppath.sample_scale(drop_prob, B, 3, h.device)
    h2, _ = ops.gemm(att, pack.get(proj.weight, 0), bias=proj.bias, residual=h, out_f32=True,
                     rowscale=None if dp1 is None else (dp1, T))
    y2, m2, r2 = ops.layernorm_fwd(h2, norm2.weight, norm2.bias, norm2.eps)
    post, dact = ops.gemm(y2, pack.get(fc1.weight, 0), bias=fc1.bias, act=2, aux_out=want_tape)
    dp2 = droppath.sample_scale(drop_prob, B, 3, h.device)
    h3, _ = ops.gemm(post, pack.get(fc2.weight, 0), bias=fc2.bias, residual=h2, out_f32=True,
                     rowscale=None if dp2 is None else (dp2, T))
    rec = None
    if want_tape:
        rec = ((norm1, qkv, proj, norm2, fc1, fc2, heads, scale), h, y1, m1, r1, qkv_t, att, lse, h2, y2, m2, r2, dact, post,
               dp1, dp2)
    return h3, rec


def backward(grads, pack, rec, g):
    """Records the block's parameter gradients (fc2 first, norm1 last) and returns the bf16 gradient [B, T, D] of the
    block input from the bf16 gradient ``g`` of its output."""
    (norm1, qkv, proj, norm2, fc1, fc2, heads, scale), h, y1, m1, r1, qkv_t, att, lse, h2, y2, m2, r2, dact, post, dp1, dp2 = rec
    B, T, D = h.shape
    M = B * T
    inner = att.shape[-1]
    # (stochastic depth: the branch sees the per-sample scaled gradient, the identity path - `add=g` below - the full one)
    g2 = (g if dp2 is None else ops.rowscale(g, dp2)).view(M, D)
    # h3 = h2 + fc2(gelu(fc1(LN2(h2))))
    linear_grads(grads, fc2, g2, post.view(M, -1))
    # dgrad + GELU' in the epilogue, which also sums the columns of d_pre (= fc1 bias gradient) on the way out
    d_pre, _, st_pre = ops.gemm(g2, pack.get(fc2.weight, 1), act=3, aux_in=dact.view(M, -1), want_stats=True)
    linear_grads(grads, fc1, d_pre, y2.view(M, D), dy_stats=st_pre)
    d_y2, _ = ops.gemm(d_pre, pack.get(fc1.weight, 1))
    g = layernorm_backward(grads, norm2, d_y2, h2, m2, r2, add=g)
    # h2 = h + proj(attention(qkv(LN1(h))))
    g2 = (g if dp1 is None else ops.rowscale(g, dp1)).view(M, D)
    linear_grads(grads, proj, g2, att.view(M, inner))
    d_att, _ = ops.gemm(g2, pack.get(proj.weight, 1))
    dqkv = ops.attention_bwd(qkv_t, att, d_att.view(B, T, inner), lse, heads, scale)
    linear_grads(grads, qkv, dqkv.view(M, 3 * inner), y1.view(M, D))
    d_y1, _ = ops.gemm(dqkv.view(M, 3 * inner), pack.get(qkv.weight, 1))
    g = layernorm_backward(grads, norm1, d_y1, h, m1, r1, add=g)
    return g.view(B, T, D)
