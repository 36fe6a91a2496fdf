"""Host-side checks of the MAE drop-in and its GPU engine schedule (no GPU needed): the constructors of both train.py
configurations, every admission rejection (raised before anything is launched), dispatch, CPU input, the C-entry argument
checks and the training step's parameter arena."""
import pytest
import torch
import torch.nn as nn

from deeplearning_b200.engine import mae as engine
from deeplearning_b200.self_supervised.MAE.models.MAE import MAE, MAEVisonTransformer
from deeplearning_b200.self_supervised.MAE.models.VIT import ViT

PRETRAIN = dict(encoer_dim=768, mlp_dim=1024, encoder_depth=12, num_encoder_head=12, dim_per_head=64, decoder_dim=512,
                decoder_depth=8, num_decoder_head=16, mask_ratio=0.75)   # train.py's pre-training model
TINY = dict(image_size=32, patch_size=8, encoer_dim=64, mlp_dim=128, encoder_depth=1, num_encoder_head=2, dim_per_head=64,
            decoder_dim=128, decoder_depth=1, num_decoder_head=2)


def test_constructors_of_both_train_configs():
    m = MAEVisonTransformer(224, 16, **PRETRAIN)
    assert isinstance(m.enc_to_dec, nn.Linear) and tuple(m.enc_to_dec.weight.shape) == (512, 768)
    assert len(m.encoder.transformer.layers) == 12 and len(m.decoder.layers) == 8
    assert tuple(m.encoder.pos_embed.shape) == (1, 197, 768) and tuple(m.decoder_pos_embed.weight.shape) == (196, 512)
    assert tuple(m.head.weight.shape) == (768, 512) and tuple(m.mask_embed.shape) == (512,)
    att = m.decoder.layers[0][0].net
    assert att.num_heads == 16 and tuple(att.to_qkv.weight.shape) == (3 * 1024, 512) and att.to_qkv.bias is None
    assert tuple(att.out[0].weight.shape) == (512, 1024)
    assert tuple(m.decoder.layers[0][1].net.net[0].weight.shape) == (2048, 512)
    names = [n for n, _ in m.named_parameters()]
    assert names[:5] == ["mask_embed", "encoder.cls_token", "encoder.pos_embed", "encoder.patch_embed.weight",
                         "encoder.patch_embed.bias"]
    assert names[-3:] == ["decoder_pos_embed.weight", "head.weight", "head.bias"]
    assert "encoder.transformer.layers.11.1.net.net.3.bias" in names and "encoder.mlp_head.1.weight" in names

    m = MAEVisonTransformer(224, 16)   # the other branch: 512 / 512, 6 + 6 layers
    assert isinstance(m.enc_to_dec, nn.Identity)
    assert len(m.encoder.transformer.layers) == 6 and len(m.decoder.layers) == 6
    assert not any(n.startswith("enc_to_dec") for n, _ in m.named_parameters())


def test_dispatch_and_parameters_without_gradient():
    from deeplearning_b200.engine.trainer import _engine_for

    m = MAEVisonTransformer(**TINY)
    assert _engine_for(m) is engine
    skip = {id(p) for p in engine.params_without_grad(m)}
    assert {n for n, p in m.named_parameters() if id(p) in skip} == {"encoder.cls_token", "encoder.mlp_head.0.weight",
                                                                     "encoder.mlp_head.0.bias", "encoder.mlp_head.1.weight",
                                                                     "encoder.mlp_head.1.bias"}


def test_trainstep_arena_excludes_unused_parameters():
    """The arena is built before the device check, so it can be inspected on a CPU model."""
    from deeplearning_b200.engine.trainer import TrainStep

    m = MAEVisonTransformer(**TINY)
    step = TrainStep.__new__(TrainStep)
    with pytest.raises(RuntimeError, match="CUDA"):
        step.__init__(m, optimizer="adamw", betas=(0.9, 0.95), weight_decay=0.05, no_decay=lambda n, p: False)
    in_arena = {id(p) for p in step.arena.params}
    names = [n for n, p in m.named_parameters() if id(p) not in in_arena]
    assert sorted(names) == ["encoder.cls_token", "encoder.mlp_head.0.bias", "encoder.mlp_head.0.weight",
                             "encoder.mlp_head.1.bias", "encoder.mlp_head.1.weight"]
    params = list(m.parameters())
    assert [params[i] for i in step._pidx] == step.arena.params
    assert m.encoder.cls_token.grad is None and m.mask_embed.grad is not None


def _reject(model, match, x=None, train=True, want_tape=True):
    x = torch.zeros(2, 3, 32, 32) if x is None else x
    with pytest.raises(NotImplementedError, match=match):
        engine.forward(model, x, train, want_tape)


def test_admission_head_dim():
    _reject(MAEVisonTransformer(**dict(TINY, dim_per_head=32)), r"encoder\.transformer\.layers\.0\.0\.net: head_dim 32")


def test_admission_project_out_identity():
    _reject(MAEVisonTransformer(**dict(TINY, num_encoder_head=1)), r"encoder\.transformer\.layers\.0\.0\.net\.out")


def test_admission_dropout_in_training():
    m = MAEVisonTransformer(**TINY)
    m.decoder.layers[0][1].net.net[2].p = 0.1
    _reject(m, r"decoder\.layers\.0\.1\.net\.net\.2: dropout")
    m = MAEVisonTransformer(**TINY)
    m.encoder.transformer.layers[0][0].net.out[1].p = 0.1
    _reject(m, r"encoder\.transformer\.layers\.0\.0\.net\.out\.1: dropout")


def test_admission_activation():
    m = MAEVisonTransformer(**TINY)
    m.decoder.layers[0][1].net.net[1] = nn.ReLU()
    _reject(m, r"decoder\.layers\.0\.1\.net\.net\.1: the FFN activation")
    m = MAEVisonTransformer(**TINY)
    m.decoder.layers[0][1].net.net[1] = nn.GELU(approximate="tanh")
    _reject(m, r"decoder\.layers\.0\.1\.net\.net\.1")


def test_admission_sequence_length():
    m = MAEVisonTransformer(**dict(TINY, image_size=136))   # 17 x 17 = 289 patches
    _reject(m, r"decoder: 289 patches \(73 visible\)", x=torch.zeros(1, 3, 136, 136))


def test_admission_image_not_divisible():
    _reject(MAEVisonTransformer(**TINY), r"encoder\.patch_embed: a 36x36 image", x=torch.zeros(1, 3, 36, 36))
    _reject(MAEVisonTransformer(**TINY), r"encoder\.patch_embed: a 36x36 image",
            x=torch.zeros(1, 36, 36, 3, dtype=torch.uint8))


def test_admission_layernorm_widths():
    m = MAEVisonTransformer(**dict(TINY, encoer_dim=1088, mlp_dim=64))
    _reject(m, r"encoder\.transformer\.layers\.0\.0\.norm: LayerNorm over 1088 channels; the LayerNorm backward")


def test_cpu_input_raises_and_classification_forward_is_not_built():
    m = MAEVisonTransformer(**TINY)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(2, 3, 32, 32))
    with pytest.raises(NotImplementedError, match="classification/vision_transformer|vision_transformer"):
        m.encoder(torch.zeros(2, 3, 32, 32))
    with pytest.raises(RuntimeError, match="parameter container"):
        m.decoder(torch.zeros(2, 16, 128))
    assert isinstance(m, MAE) and isinstance(m.encoder, ViT)


def test_entries_reject_bad_arguments_before_launch():
    from deeplearning_b200 import _lib

    lib = _lib.load()
    fake = 256
    assert lib.b200_mae_shuffle(fake, fake, fake, 2, 2000, None) == -1 and "P must be" in _lib.last_error()
    assert lib.b200_mae_shuffle(None, fake, fake, 2, 16, None) == -1 and "non-null" in _lib.last_error()
    assert lib.b200_mae_patchify(fake, fake, fake, fake, 2, 3, 36, 36, 8, 12, None) == -1
    assert "multiples of the patch size" in _lib.last_error()
    assert lib.b200_mae_patchify(fake, fake, fake, fake, 2, 3, 32, 32, 8, 16, None) == -1 and "Nm" in _lib.last_error()
    assert lib.b200_mae_gather_rows(fake, 0, 1, fake, 2, 16, 12, 8, 64, fake, 1, None) == -1
    assert "slots" in _lib.last_error()
    assert lib.b200_mae_assemble_fwd(fake, fake, fake, fake, fake, 2, 16, 0, 64, None) == -1
    assert lib.b200_mae_assemble_bwd(fake, fake, fake, None, 2, 16, 12, 64, None) == -1
    assert lib.b200_mae_pos_grad(fake, fake, fake, 0, 16, 12, 64, None) == -1 and "B must" in _lib.last_error()
    assert lib.b200_mae_scatter_masked(fake, fake, fake, 2, 1, 1, 64, None) == -1
    assert lib.b200_mae_mse(fake, fake, 0, 1.0, fake, fake, fake, None) == -1 and "n must" in _lib.last_error()
    assert lib.b200_mae_mse_blocks() > 0
