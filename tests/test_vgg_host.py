"""Device-free checks of the VGG drop-in (classification/vggNet/models/network.py) and of engine/vgg.py's admission: module
names and shapes of all eight constructors, the init, the pretrained guard, and check_model admitting every constructor and
rejecting each malformed case with the layer named."""
import pytest
import torch
import torch.nn as nn

from deeplearning_b200.classification.vggNet.models import network
from deeplearning_b200.engine import common
from deeplearning_b200.engine import vgg as engine
from oracle.vgg import arch

NAMES = ["vgg11", "vgg11_bn", "vgg13", "vgg13_bn", "vgg16", "vgg16_bn", "vgg19", "vgg19_bn"]


@pytest.mark.parametrize("name", NAMES)
def test_constructor_tree_and_admission(name):
    m = getattr(network, name)(num_classes=7)
    cfg, bn = arch(name)
    names = []
    i, cin = 0, 3
    for v in cfg:
        if v == 'M':
            assert type(m.features[i]) is nn.MaxPool2d
            i += 1
            continue
        names += [(f"features.{i}.weight", (v, cin, 3, 3)), (f"features.{i}.bias", (v,))]
        i += 1
        if bn:
            names += [(f"features.{i}.weight", (v,)), (f"features.{i}.bias", (v,))]
            i += 1
        i += 1
        cin = v
    names += [("classifier.0.weight", (4096, 25088)), ("classifier.0.bias", (4096,)), ("classifier.3.weight", (4096, 4096)),
              ("classifier.3.bias", (4096,)), ("classifier.6.weight", (7, 4096)), ("classifier.6.bias", (7,))]
    assert [(n, tuple(p.shape)) for n, p in m.named_parameters()] == names
    layers, fcs, ps = engine.check_model(m)
    assert len(layers) == sum(v != 'M' for v in cfg) and ps == (0.5, 0.5)
    assert all((l.bn is not None) == bn for l in layers)


def test_init_and_pretrained():
    torch.manual_seed(0)
    m = network.vgg11_bn(num_classes=3)
    assert float(m.features[0].bias.detach().abs().sum()) == 0.0 and float(m.features[1].weight.detach().sum()) == 64.0
    assert abs(float(m.classifier[0].weight.detach().std()) - 0.01) < 1e-3
    with pytest.raises(RuntimeError):
        network.vgg16(pretrained=True)


def _reject(m, where):
    with pytest.raises(NotImplementedError, match=where.replace(".", r"\.")):
        engine.check_model(m)


def test_rejections():
    def fresh(bn=False):
        return network.VGG(network.make_layers([64, 'M', 512, 'M'], bn),
                           init_weights=False)

    m = fresh()
    m.features[0] = nn.Conv2d(3, 64, 3, padding=1, bias=False)
    _reject(m, "features.0")
    m = fresh()
    m.features[3] = nn.Conv2d(64, 512, 3, padding=1, stride=2)
    _reject(m, "features.3")
    m = fresh()
    m.features[3] = nn.Conv2d(64, 120, 3, padding=1)
    _reject(m, "features.3")
    m = network.VGG(network.make_layers([64, 'M'], False), init_weights=False)
    m.features[0] = nn.Conv2d(1, 64, 3, padding=1)
    _reject(m, "features.0")
    m = fresh()
    m.features[2] = nn.MaxPool2d(3, 2)
    _reject(m, "features.2")
    m = fresh()
    m.features[1] = nn.GELU()
    _reject(m, "features.1")
    m = network.VGG(network.make_layers([64, 'M', 128], False), init_weights=False)
    _reject(m, "features.3")
    m = fresh(True)
    m.features[1] = nn.BatchNorm2d(64, affine=False)
    _reject(m, "features.1")
    m = fresh()
    m.avgpool = nn.AdaptiveAvgPool2d(1)
    _reject(m, "avgpool")
    m = fresh()
    m.classifier[2] = nn.Dropout(1.0)
    _reject(m, "classifier.2")
    m = fresh()
    m.classifier[1] = nn.GELU()
    _reject(m, "classifier.1")
    m = fresh()
    m.classifier = nn.Sequential(*list(m.classifier)[:-1])
    _reject(m, "classifier")
    m = fresh()
    m.classifier[0] = nn.Linear(25088, 4096, bias=False)
    _reject(m, "classifier.0")


def test_cpu_input_raises():
    m = network.vgg11(num_classes=3)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 32, 32))


def test_sync_batchnorm_admission(monkeypatch):
    """a SyncBatchNorm model is admitted outside a multi-rank job and rejected, naming the layer, inside one"""
    m = nn.SyncBatchNorm.convert_sync_batchnorm(network.vgg11_bn(num_classes=3))
    assert type(m.features[1]) is nn.SyncBatchNorm
    layers, _, _ = engine.check_model(m)
    assert all(type(l.bn) is nn.SyncBatchNorm for l in layers)
    monkeypatch.setattr(common, "bn_sync", lambda bn: (None, 2) if isinstance(bn, nn.SyncBatchNorm) else None)
    with pytest.raises(NotImplementedError, match=r"features\.1: SyncBatchNorm in a multi-rank job"):
        engine.check_model(m)
