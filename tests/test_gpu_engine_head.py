"""The classifier head and the gradient sink of every engine schedule, with a padded (5 classes) and an unpadded (16) head.

``TrainStep`` always hands the engines a sink; this checks that writing the gradients into the sink's buffers gives the same
bits as the sink-free backward, that every parameter is reported exactly once, and that the logits are cut back to
``num_classes`` columns."""
from collections import Counter

import pytest
import torch

pytestmark = pytest.mark.gpu


def _resnet(n):
    from deeplearning_b200.classification.resnet.models.networks import Bottleneck, ResNet

    return ResNet(Bottleneck, [1, 1, 1, 1], num_classes=n), (4, 3, 64, 64)


def _vit(n):
    from deeplearning_b200.classification.vision_transformer.vit_model import VisionTransformer

    return VisionTransformer(img_size=224, patch_size=16, embed_dim=768, depth=1, num_heads=12, num_classes=n), (2, 3, 224, 224)


def _swin(n):
    from deeplearning_b200.classification.swin_transformer.models.swin_transformer import SwinTransformer

    return SwinTransformer(depths=[1, 1], num_heads=[3, 6], num_classes=n, drop_path_rate=0.0), (2, 3, 224, 224)


def _convnext(n):
    from deeplearning_b200.classification.convNext.models.networks import ConvNeXt

    return ConvNeXt(depths=[1, 1, 1, 1], dims=[96, 192, 384, 768], num_classes=n, drop_path_rate=0.0), (2, 3, 224, 224)


class _Sink:
    """Zeroed per-parameter destination buffers; records every completion notice."""

    def __init__(self, model):
        self.bufs = {p.data_ptr(): torch.zeros_like(p) for p in model.parameters()}
        self.notified = Counter()

    def __call__(self, param):
        return self.bufs[param.data_ptr()]

    def notify(self, param):
        self.notified[param.data_ptr()] += 1


@pytest.mark.parametrize("num_classes", [5, 16])
@pytest.mark.parametrize("family", ["resnet", "vit", "swin", "convnext"])
def test_head_and_gradient_sink(family, num_classes):
    from deeplearning_b200 import ops
    from deeplearning_b200.engine import convnext, resnet, swin, vit
    from deeplearning_b200.engine.common import padded_classes

    engine, build = {"resnet": (resnet, _resnet), "vit": (vit, _vit), "swin": (swin, _swin),
                     "convnext": (convnext, _convnext)}[family]
    torch.manual_seed(0)
    model, shape = build(num_classes)
    model = model.cuda().train()
    x = torch.randn(*shape, device="cuda")
    labels = torch.randint(0, num_classes, (shape[0],), device="cuda")

    def step(sink):
        logits, tape = engine.forward(model, x, True, True)
        assert logits.shape == (shape[0], num_classes)
        _, dlogits, _ = ops.softmax_xent(logits, labels, want_grad=True, ld_d=padded_classes(num_classes))
        return engine.backward(model, tape, dlogits, sink=sink)

    plain = step(None)
    sink = _Sink(model)
    sunk = step(sink)
    torch.cuda.synchronize()
    for name, p in model.named_parameters():
        key = p.data_ptr()
        a, b, buf = plain[key].reshape(p.shape), sunk[key], sink.bufs[key]
        assert b.data_ptr() == buf.data_ptr() and b.numel() == buf.numel(), f"{name}: not written into the sink's buffer"
        if name.endswith("relative_position_bias_table"):
            # summed over windows with float atomics: the order, and so the last bits, vary from run to run
            assert float((a - buf).abs().max()) <= 1e-4 * float(a.abs().max()), name
        else:
            assert torch.equal(a, buf), f"{name}: sink gradient differs from the sink-free backward"
        assert sink.notified[key] == 1, f"{name}: notified {sink.notified[key]} times"
    assert len(sink.notified) == len(list(model.parameters()))
