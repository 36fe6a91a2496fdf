"""Admission of the shipped ViT, Swin and ConvNeXt configurations by the GPU engine: each one either trains, or is rejected
with a NotImplementedError that names the layer before any kernel runs.  The kernels' width limits decide it:
LayerNorm forward 3072 channels, LayerNorm backward 1024, patch-merge LayerNorm 4C <= 2048 (ops.LAYERNORM_*_MAX_C,
ops.PATCH_MERGE_LN_MAX_C).

The host tests build each configuration at one block per stage (admission depends only on the widths); the GPU test
builds every constructor at full size and checks the launch counter."""
import pytest
import torch
import torch.nn.functional as F

# (embed, depths, heads, drop_path_rate) of configs/swin/swin_{tiny,small,base,large}_patch4_window7_224*.yaml
SWIN_224 = {
    "swin_tiny": (96, (2, 2, 6, 2), (3, 6, 12, 24), 0.2),
    "swin_small": (96, (2, 2, 18, 2), (3, 6, 12, 24), 0.3),
    "swin_base": (128, (2, 2, 18, 2), (4, 8, 16, 32), 0.5),
    "swin_large": (192, (2, 2, 18, 2), (6, 12, 24, 48), 0.2),
}
# (patch, embed, heads) of the vit_model constructors
VIT_WIDTHS = {"vit_base_patch16_224_in21k": (16, 768, 12), "vit_base_patch32_224_in21k": (32, 768, 12),
              "vit_large_patch16_224_in21k": (16, 1024, 16), "vit_large_patch32_224_in21k": (32, 1024, 16),
              "vit_huge_patch14_224_in21k": (14, 1280, 16)}
VIT = list(VIT_WIDTHS)
# dims of the networks.convnext_* constructors
CONVNEXT_DIMS = {"convnext_tiny": 96, "convnext_small": 96, "convnext_base": 128, "convnext_large": 192,
                 "convnext_xlarge": 256}
CONVNEXT = list(CONVNEXT_DIMS)

# what the engine does with each: "train", "eval" (runs without gradients only) or "reject" (not even a forward)
EXPECT = {"vit_base_patch16_224_in21k": "train", "vit_base_patch32_224_in21k": "train",
          "vit_large_patch16_224_in21k": "train", "vit_large_patch32_224_in21k": "train",
          "vit_huge_patch14_224_in21k": "reject",   # head_dim 80
          "convnext_tiny": "train", "convnext_small": "train", "convnext_base": "train",
          "convnext_large": "eval",                 # stage-4 LayerNorm over 1536 channels
          "convnext_xlarge": "eval",                # 2048
          "swin_tiny": "train", "swin_small": "train", "swin_base": "train",
          "swin_large": "reject"}                   # stage-3 patch merge: 4 * 768 = 3072


def _build(name, full=True):
    if name.startswith("vit"):
        from deeplearning_b200.classification.vision_transformer import vit_model

        if full:
            return vit_model.__dict__[name](num_classes=10), vit_model
        patch, dim, heads = VIT_WIDTHS[name]
        return vit_model._vit(patch, dim, 1, heads, 10, True), vit_model
    if name.startswith("convnext"):
        from deeplearning_b200.classification.convNext.models import networks

        if full:
            return networks.__dict__[name](10), networks
        d = CONVNEXT_DIMS[name]
        return networks.ConvNeXt(depths=[1, 1, 1, 1], dims=[d, 2 * d, 4 * d, 8 * d], num_classes=10), networks
    from deeplearning_b200.classification.swin_transformer.models.swin_transformer import SwinTransformer

    embed, depths, heads, dpr = SWIN_224[name]
    return SwinTransformer(embed_dim=embed, depths=list(depths if full else (1, 1, 1, 1)), num_heads=list(heads),
                           num_classes=10, drop_path_rate=dpr), None


def _engine(name):
    from deeplearning_b200.engine import convnext, swin, vit

    return vit if name.startswith("vit") else convnext if name.startswith("convnext") else swin


@pytest.mark.parametrize("name", VIT + CONVNEXT + list(SWIN_224))
def test_admission_by_width(name):
    torch.manual_seed(0)
    m, _ = _build(name, full=False)
    check = _engine(name)._check
    want = EXPECT[name]
    if want == "reject":
        with pytest.raises(NotImplementedError):
            check(m, False)
    else:
        check(m, False)
    if want == "train":
        check(m, True)
    else:
        with pytest.raises(NotImplementedError) as e:
            check(m, True)
        print(e.value)


def test_admission_messages_name_layer_and_limit():
    torch.manual_seed(0)
    m, _ = _build("convnext_large", full=False)
    with pytest.raises(NotImplementedError, match=r"stages\.3\.0\.norm: LayerNorm over 1536 channels.*at most 1024"):
        _engine("convnext_large")._check(m, True)
    m, _ = _build("swin_large", full=False)
    with pytest.raises(NotImplementedError, match=r"layers\.2\.downsample: .*4 \* 768 = 3072.*at most 2048"):
        _engine("swin_large")._check(m, False)
    # with widths doubling per stage a merge that fits keeps every Swin LayerNorm within the backward's 1024; a single
    # stage of 1280 channels has no merge: it runs, but cannot train
    from deeplearning_b200.classification.swin_transformer.models.swin_transformer import SwinTransformer
    from deeplearning_b200.engine import swin

    m = SwinTransformer(embed_dim=1280, depths=[1], num_heads=[40], num_classes=10)
    swin._check(m, False)
    with pytest.raises(NotImplementedError, match=r"patch_embed\.norm: LayerNorm over 1280 channels.*at most 1024"):
        swin._check(m, True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", VIT + CONVNEXT + list(SWIN_224))
def test_shipped_constructor_trains_or_is_rejected_before_launch(name):
    from deeplearning_b200 import ops

    torch.manual_seed(0)
    with torch.device("cuda"):
        m, _ = _build(name)
    m.train()
    x = torch.randn(2, 3, 224, 224, device="cuda")
    y = torch.tensor([3, 7], device="cuda")
    want = EXPECT[name]
    if want == "train":
        out = m(x)
        F.cross_entropy(out, y).backward()
        torch.cuda.synchronize()
        assert out.shape == (2, 10) and torch.isfinite(out).all()
        for pname, p in m.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), pname
        return
    n0 = ops.launch_count()
    with pytest.raises(NotImplementedError) as e:
        m(x)
    assert ops.launch_count() == n0, f"{name}: kernels launched before the model was rejected"
    print(f"{name}: {e.value}")
    if want == "eval":
        m.eval()
        with torch.no_grad():
            out = m(x)
        assert out.shape == (2, 10) and torch.isfinite(out).all()
        assert ops.launch_count() > n0
    else:
        with torch.no_grad():
            with pytest.raises(NotImplementedError):
                m.eval()(x)
        assert ops.launch_count() == n0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["convnext_large", "convnext_xlarge"])
def test_wide_convnext_eval_parity(name):
    """ConvNeXt-L / XL run without gradients: logits against the fp32 oracle at one block per stage."""
    from oracle.convnext import convnext_forward

    torch.manual_seed(0)
    m, _ = _build(name, full=False)
    g = torch.Generator().manual_seed(7)
    state = {k: (torch.randn(v.shape, generator=g) * 0.02 if v.dim() >= 2 else v.clone()) for k, v in m.state_dict().items()}
    m.load_state_dict(state)
    m = m.cuda().eval()
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = convnext_forward(state, x)
        got = m(x.cuda()).float().cpu()
    err = float((got - ref).abs().max())
    print(f"{name} (1,1,1,1) eval logits max-abs err {err:.4g} (|ref| max {float(ref.abs().max()):.3g})")
    assert err <= 1e-2 * max(1.0, float(ref.abs().max()))
