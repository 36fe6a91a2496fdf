"""Oracle: the reference MAE pre-training forward (self-supervised/MAE/models/MAE.py ``MAE.forward`` with the
``Transformer`` / ``PreNorm`` / ``SelfAttention`` / ``FFN`` blocks of models/VIT.py) restated functionally in fp32 PyTorch
over a state_dict.  The per-sample shuffle is an argument (the reference's ``torch.rand(b, P).argsort()``), so the oracle
can be fed the indices the GPU engine drew."""
import torch
import torch.nn.functional as F


def _transformer(s, prefix, x, heads):
    i = 0
    while f"{prefix}.layers.{i}.0.norm.weight" in s:
        p = f"{prefix}.layers.{i}."
        D = x.shape[-1]
        # x = x + PreNorm(SelfAttention)(x)
        y = F.layer_norm(x, (D,), s[p + "0.norm.weight"], s[p + "0.norm.bias"])
        b, l, _ = y.shape
        qkv = F.linear(y, s[p + "0.net.to_qkv.weight"])
        dph = qkv.shape[-1] // 3 // heads
        qkv = qkv.view(b, l, 3, heads, -1).permute(2, 0, 3, 1, 4).contiguous()
        q, k, v = qkv.chunk(3)
        q, k, v = q.squeeze(0), k.squeeze(0), v.squeeze(0)
        attn = torch.softmax(torch.matmul(q, k.transpose(-1, -2)) * dph ** -0.5, dim=-1)
        z = torch.matmul(attn, v).transpose(1, 2).reshape(b, l, -1)
        x = x + F.linear(z, s[p + "0.net.out.0.weight"], s[p + "0.net.out.0.bias"])
        # x = x + PreNorm(FFN)(x)
        y = F.layer_norm(x, (D,), s[p + "1.norm.weight"], s[p + "1.norm.bias"])
        y = F.gelu(F.linear(y, s[p + "1.net.net.0.weight"], s[p + "1.net.net.0.bias"]))
        x = x + F.linear(y, s[p + "1.net.net.3.weight"], s[p + "1.net.net.3.bias"])
        i += 1
    return x


def mae_forward(s, x, shuffle_indices, patch, enc_heads, dec_heads, mask_ratio=0.75):
    """(pred [B, Nm, p*p*C], mask_patches [B, Nm, p*p*C]) of the MAE whose parameters are ``s`` (state_dict names) on the
    image batch x [B, C, H, W], with the per-sample shuffle ``shuffle_indices`` (long [B, P])."""
    b, c, h, w = x.shape
    num_patches = (h // patch) * (w // patch)
    patches = x.view(b, c, h // patch, patch, w // patch, patch).permute(0, 2, 4, 3, 5, 1).reshape(b, num_patches, -1)
    num_masked = int(mask_ratio * num_patches)
    mask_indices, unmask_indices = shuffle_indices[:, :num_masked], shuffle_indices[:, num_masked:]
    batch_indices = torch.arange(b, device=x.device).unsqueeze(-1)
    mask_patches, unmask_patches = patches[batch_indices, mask_indices], patches[batch_indices, unmask_indices]
    tokens = F.linear(unmask_patches, s["encoder.patch_embed.weight"], s["encoder.patch_embed.bias"])
    tokens = tokens + s["encoder.pos_embed"].repeat(b, 1, 1)[batch_indices, unmask_indices + 1]
    encoded = _transformer(s, "encoder.transformer", tokens, enc_heads)
    if "enc_to_dec.weight" in s:
        encoded = F.linear(encoded, s["enc_to_dec.weight"], s["enc_to_dec.bias"])
    mask_tokens = s["mask_embed"][None, None, :].repeat(b, num_masked, 1)
    mask_tokens = mask_tokens + F.embedding(mask_indices, s["decoder_pos_embed.weight"])
    concat = torch.cat([mask_tokens, encoded], dim=1)
    dec_in = torch.empty_like(concat)
    dec_in[batch_indices, shuffle_indices] = concat
    decoded = _transformer(s, "decoder", dec_in, dec_heads)
    pred = F.linear(decoded[batch_indices, mask_indices, :], s["head.weight"], s["head.bias"])
    return pred, mask_patches


def train_step_grads(state, x, shuffle_indices, patch, enc_heads, dec_heads, mask_ratio=0.75):
    """(pred, mask_patches, loss, {name: grad}) of ``F.mse_loss(pred, mask_patches).backward()``: the reference loop's loss.
    Parameters the forward does not read (encoder.cls_token, encoder.mlp_head.*) have no entry."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in state.items()}
    pred, mask_patches = mae_forward(params, x, shuffle_indices, patch, enc_heads, dec_heads, mask_ratio)
    loss = F.mse_loss(pred, mask_patches)
    loss.backward()
    grads = {k: p.grad for k, p in params.items() if p.grad is not None}
    return pred.detach(), mask_patches.detach(), loss.detach(), grads
