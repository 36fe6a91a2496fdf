"""Drop-in for the reference's self-supervised/MAE/models/MAE.py: ``MAE`` and ``MAEVisonTransformer`` (the reference's
spelling) with the reference's parameter names, registration order and ``init_weights`` pass, so a seeded constructor gives
the reference's state_dict bit for bit.  ``MAE.forward`` draws the shuffle keys with ``torch.rand`` where the reference does
and runs the masked pre-training forward on the GPU engine (engine/mae.py); there is no CPU path."""
import torch
import torch.nn as nn

from .VIT import Transformer, ViT


class MAE(nn.Module):
    def __init__(self, encoder, decoder_dim, mask_ratio=0.75, decoder_depth=1, num_decoder_heads=8, decoder_dim_per_head=64):
        super().__init__()
        assert 0.0 < mask_ratio < 1.0, f"mask ratio must be kept between 0 and 1, got :{mask_ratio}"
        self.encoder = encoder
        self.patch_h, self.patch_w = encoder.patch_h, encoder.patch_w
        num_patches_plus_cls_token, encoder_dim = encoder.pos_embed.shape[-2:]
        num_pixels_per_patch = encoder.patch_embed.weight.size(1)
        self.enc_to_dec = nn.Linear(encoder_dim, decoder_dim) if encoder_dim != decoder_dim else nn.Identity()
        self.mask_ratio = mask_ratio
        self.mask_embed = nn.Parameter(torch.randn(decoder_dim))
        self.decoder = Transformer(decoder_dim, decoder_dim * 4, depth=decoder_depth, num_heads=num_decoder_heads,
                                   dim_per_head=decoder_dim_per_head)
        self.decoder_pos_embed = nn.Embedding(num_embeddings=num_patches_plus_cls_token - 1, embedding_dim=decoder_dim)
        self.head = nn.Linear(decoder_dim, num_pixels_per_patch)
        self.apply(self.init_weights)

    def init_weights(self, module):
        if isinstance(module, nn.Linear):
            nn.init.xavier_uniform_(module.weight)
            if module.bias is not None:
                nn.init.zeros_(module.bias)
        elif isinstance(module, nn.Conv2d):
            nn.init.xavier_uniform_(module.weight)
            if module.bias is not None:
                nn.init.zeros_(module.bias)
        elif isinstance(module, (nn.LayerNorm, nn.GroupNorm, nn.BatchNorm2d)):
            nn.init.zeros_(module.bias)
            nn.init.ones_(module.weight)

    def forward(self, x):
        """(pred fp32 [B, Nm, p*p*C], mask_patches fp32 [B, Nm, p*p*C]) of the reference; pred carries the gradient."""
        from deeplearning_b200.engine import mae as engine

        return engine.apply(self, x)

    @torch.no_grad()
    def predict(self, x):
        """The reference's reconstruction: (recons_img, patches_to_img), both [B, C, H, W]; prints the masked-patch errors."""
        from deeplearning_b200.engine import mae as engine

        self.eval()
        device = x.device
        b, c, h, w = x.shape
        num_patches = (h // self.patch_h) * (w // self.patch_w)
        patches = x.view(b, c, h // self.patch_h, self.patch_h, w // self.patch_w, self.patch_w) \
            .permute(0, 2, 4, 3, 5, 1).reshape(b, num_patches, -1)
        num_masked = int(self.mask_ratio * num_patches)
        (pred_mask_pixel_values, mask_patches, ids), _ = engine.forward(self, x, False, False)
        mask_indices = ids[:, :num_masked].long()
        batch_indices = torch.arange(b, device=device).unsqueeze(-1)
        mse_per_patch = (pred_mask_pixel_values - mask_patches).abs().mean(dim=-1)
        mse_all_patches = mse_per_patch.mean()
        print(f'mse per (masked)patch: {mse_per_patch} mse all (masked)patches: {mse_all_patches} total {num_masked} '
              f'masked patches')
        print(f'all close: {torch.allclose(pred_mask_pixel_values, mask_patches, rtol=1e-1, atol=1e-1)}')
        recons_patches = patches.detach()
        recons_patches[batch_indices, mask_indices] = pred_mask_pixel_values
        recons_img = recons_patches.view(b, h // self.patch_h, w // self.patch_w, self.patch_h, self.patch_w, c) \
            .permute(0, 5, 1, 3, 2, 4).reshape(b, c, h, w)
        mask_patches = torch.randn_like(mask_patches, device=mask_patches.device)
        patches[batch_indices, mask_indices] = mask_patches
        patches_to_img = patches.view(b, h // self.patch_h, w // self.patch_w, self.patch_h, self.patch_w, c) \
            .permute(0, 5, 1, 3, 2, 4).reshape(b, c, h, w)
        return recons_img, patches_to_img


def MAEVisonTransformer(image_size=224, patch_size=16, encoer_dim=512, mlp_dim=1024, encoder_depth=6, num_encoder_head=8,
                        dim_per_head=64, decoder_dim=512, decoder_depth=6, num_decoder_head=8, mask_ratio=0.75):
    encoder = ViT(image_size=image_size, patch_size=patch_size, dim=encoer_dim, mlp_dim=mlp_dim, dim_per_head=dim_per_head,
                  depth=encoder_depth, num_heads=num_encoder_head)
    return MAE(encoder=encoder, decoder_dim=decoder_dim, decoder_depth=decoder_depth, mask_ratio=mask_ratio,
               num_decoder_heads=num_decoder_head)
