"""Oracle: the reference ShuffleNet v2 forward (classification/ShuffleNet/models/shufflenetv2.py: conv1, maxpool, stage2..4 of
InvertedResiduals with the two-group channel shuffle, conv5, the global mean and fc) restated functionally in fp32 PyTorch
over a state_dict."""
import torch
import torch.nn.functional as F


def _bn(x, s, p, train):
    if train:
        s[p + "num_batches_tracked"] += 1
    return F.batch_norm(x, s[p + "running_mean"], s[p + "running_var"], s[p + "weight"], s[p + "bias"], train, 0.1, 1e-5)


def _shuffle(x, g):
    B, C, H, W = x.shape
    return x.view(B, g, C // g, H, W).transpose(1, 2).contiguous().view(B, C, H, W)


def _branch2(x, s, p, stride, train):
    x = F.relu(_bn(F.conv2d(x, s[p + "0.weight"]), s, p + "1.", train))
    x = _bn(F.conv2d(x, s[p + "3.weight"], stride=stride, padding=1, groups=x.shape[1]), s, p + "4.", train)
    return F.relu(_bn(F.conv2d(x, s[p + "5.weight"]), s, p + "6.", train))


def shufflenetv2_forward(s, x, train=False):
    """Logits of the ShuffleNetV2 whose parameters and buffers are ``s`` (state_dict names).  In train mode the BatchNorm
    running statistics in ``s`` are updated in place, as nn.BatchNorm2d does."""
    x = F.relu(_bn(F.conv2d(x, s["conv1.0.weight"], stride=2, padding=1), s, "conv1.1.", train))
    x = F.max_pool2d(x, 3, 2, 1)
    for st in ("stage2", "stage3", "stage4"):
        i = 0
        while f"{st}.{i}.branch2.0.weight" in s:
            p = f"{st}.{i}."
            if i == 0:
                u = _bn(F.conv2d(x, s[p + "branch1.0.weight"], stride=2, padding=1, groups=x.shape[1]), s, p + "branch1.1.",
                        train)
                u = F.relu(_bn(F.conv2d(u, s[p + "branch1.2.weight"]), s, p + "branch1.3.", train))
                out = torch.cat((u, _branch2(x, s, p + "branch2.", 2, train)), dim=1)
            else:
                x1, x2 = x.chunk(2, dim=1)
                out = torch.cat((x1, _branch2(x2, s, p + "branch2.", 1, train)), dim=1)
            x = _shuffle(out, 2)
            i += 1
    x = F.relu(_bn(F.conv2d(x, s["conv5.0.weight"]), s, "conv5.1.", train))
    return F.linear(x.mean([2, 3]), s["fc.weight"], s["fc.bias"])


def train_step_grads(state, x, labels):
    """fp32 train step on a copy of ``state``: (logits, loss, {name: grad}, state after the step's statistics update)."""
    s = {k: v.detach().clone() for k, v in state.items()}
    params = {k: v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k}
    logits = shufflenetv2_forward(s, x, True)
    loss = F.cross_entropy(logits, labels)
    grads = torch.autograd.grad(loss, list(params.values()))
    return logits.detach(), loss.detach(), dict(zip(params.keys(), grads)), {k: v.detach() for k, v in s.items()}
