"""Backbones of the reference's self-supervised/SupCon/models/backbone.py.  The names of the ResNet family map to this
repository's ResNet constructors (classification/resnet/models/networks.py), which the GPU engine trains; every other
name of the reference raises NotImplementedError naming the backbone.  (The reference's VGG encoders would not run there
either: ``Sequential(features, avgpool)`` yields [B, 512, 7, 7] where its head expects 4096 features.)"""
from ....classification.resnet.models import networks


def _unsupported(name):
    def build(pretrained=False, **kwargs):
        raise NotImplementedError(f"backbone {name!r} is not implemented on the GPU engine; the SupCon drop-in trains the "
                                  "ResNet family: " + ", ".join(sorted(RESNETS)))

    return build


RESNETS = {
    "resnet18": networks.resnet18,
    "resnet34": networks.resnet34,
    "resnet50": networks.resnet50,
    "resnet101": networks.resnet101,
    "resnet152": networks.resnet152,
    "resnext50_32x4d": networks.resnext50_32x4d,
    "resnext101_32x8d": networks.resnext101_32x8d,
    "wide_resnet50": networks.wide_resnet50_2,
    "wide_resnet101": networks.wide_resnet101_2,
}

BACKBONES = dict(RESNETS)
for _name in ("alexnet", "mobilenet_v2", "vgg11", "vgg11_bn", "vgg13", "vgg13_bn", "vgg16", "vgg16_bn", "vgg19", "vgg19_bn",
              "densenet121", "densenet169", "densenet161", "densenet201", "inception_v3"):
    BACKBONES[_name] = _unsupported(_name)
