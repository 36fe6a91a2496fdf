"""Drop-in for ``classification/seNet/models/networks.py`` of KKKSQJ/DeepLearning (the module train.py imports
``se_resnet50`` from): re-exports the SE-ResNet constructors."""
from .se_resnet import *  # noqa: F401,F403
from .se_resnet import __all__  # noqa: F401
