"""``build_model(config)`` of the reference (classification/swin_transformer/models/build.py:7-40) for MODEL.TYPE == 'swin'.
``config`` is any object with the reference's yacs attribute layout (DATA.IMG_SIZE, MODEL.SWIN.*, MODEL.DROP_RATE, ...)."""
import torch.nn as nn

from .swin_transformer import SwinTransformer


def build_model(config, is_pretrain=False):
    model_type = config.MODEL.TYPE
    if model_type != 'swin':
        raise NotImplementedError(f"Unkown model: {model_type} (this engine implements MODEL.TYPE 'swin')")
    s = config.MODEL.SWIN
    return SwinTransformer(img_size=config.DATA.IMG_SIZE, patch_size=s.PATCH_SIZE, in_chans=s.IN_CHANS,
                           num_classes=config.MODEL.NUM_CLASSES, embed_dim=s.EMBED_DIM, depths=s.DEPTHS,
                           num_heads=s.NUM_HEADS, window_size=s.WINDOW_SIZE, mlp_ratio=s.MLP_RATIO, qkv_bias=s.QKV_BIAS,
                           qk_scale=s.QK_SCALE, drop_rate=config.MODEL.DROP_RATE, drop_path_rate=config.MODEL.DROP_PATH_RATE,
                           ape=s.APE, norm_layer=nn.LayerNorm, patch_norm=s.PATCH_NORM,
                           use_checkpoint=config.TRAIN.USE_CHECKPOINT, fused_window_process=config.FUSED_WINDOW_PROCESS)
