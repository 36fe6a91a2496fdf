"""Oracle: the reference VGG forward (classification/vggNet/models/network.py: make_layers' features, AdaptiveAvgPool2d((7, 7)),
torch.flatten and the 7-module classifier) restated functionally in fp32 PyTorch over a state_dict.

The two classifier dropouts take their masks as input: fp32 [B, 4096] tensors holding 0 or 1 / (1 - p), what ``F.dropout``
of a tensor of ones returns, applied as ``x * mask`` (``None`` = identity)."""
import torch
import torch.nn.functional as F

CFGS = {
    'A': [64, 'M', 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'B': [64, 64, 'M', 128, 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'D': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M'],
    'E': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512, 'M'],
}
ARCH = {"vgg11": "A", "vgg13": "B", "vgg16": "D", "vgg19": "E"}


def arch(name):
    """(cfg list, batch_norm) of a constructor name such as ``vgg16_bn``."""
    bn = name.endswith("_bn")
    return CFGS[ARCH[name[:-3] if bn else name]], bn


def vgg_forward(s, x, cfg, batch_norm, train=False, masks=(None, None)):
    """Logits of the VGG whose parameters and buffers are ``s`` (state_dict names).  In train mode the BatchNorm running
    statistics in ``s`` are updated in place, as nn.BatchNorm2d does."""
    i = 0
    for v in cfg:
        if v == 'M':
            x = F.max_pool2d(x, 2, 2)
            i += 1
            continue
        x = F.conv2d(x, s[f"features.{i}.weight"], s[f"features.{i}.bias"], padding=1)
        i += 1
        if batch_norm:
            p = f"features.{i}."
            x = F.batch_norm(x, s[p + "running_mean"], s[p + "running_var"], s[p + "weight"], s[p + "bias"], train, 0.1, 1e-5)
            if train:
                s[p + "num_batches_tracked"] += 1
            i += 1
        x = F.relu(x)
        i += 1
    x = torch.flatten(F.adaptive_avg_pool2d(x, (7, 7)), 1)
    x = F.relu(F.linear(x, s["classifier.0.weight"], s["classifier.0.bias"]))
    if train and masks[0] is not None:
        x = x * masks[0]
    x = F.relu(F.linear(x, s["classifier.3.weight"], s["classifier.3.bias"]))
    if train and masks[1] is not None:
        x = x * masks[1]
    return F.linear(x, s["classifier.6.weight"], s["classifier.6.bias"])


def train_step_grads(state, x, labels, cfg, batch_norm, masks=(None, None)):
    """fp32 train step on a copy of ``state``: (logits, loss, {name: grad}, state after the step's statistics update)."""
    s = {k: v.detach().clone() for k, v in state.items()}
    params = {k: v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k}
    logits = vgg_forward(s, x, cfg, batch_norm, True, masks)
    loss = F.cross_entropy(logits, labels)
    grads = torch.autograd.grad(loss, list(params.values()))
    return logits.detach(), loss.detach(), dict(zip(params.keys(), grads)), {k: v.detach() for k, v in s.items()}
