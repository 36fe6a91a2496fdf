"""Oracle: the reference ShuffleNet v1 forward (classification/ShuffleNet/models/shufflenetv1.py: conv1, maxpool, stage2..4 of
ResidualBlocks with the channel shuffle, the global mean and fc) restated functionally in fp32 PyTorch over a state_dict."""
import torch
import torch.nn.functional as F


def _bn(x, s, p, train):
    if train:
        s[p + "num_batches_tracked"] += 1
    return F.batch_norm(x, s[p + "running_mean"], s[p + "running_var"], s[p + "weight"], s[p + "bias"], train, 0.1, 1e-5)


def _shuffle(x, g):
    B, C, H, W = x.shape
    return x.view(B, g, C // g, H, W).transpose(1, 2).contiguous().view(B, C, H, W)


def shufflenet_forward(s, x, groups, train=False):
    """Logits of the ShuffleNetv1 whose parameters and buffers are ``s`` (state_dict names); ``groups`` is the model's
    group count (stage2.0 runs ungrouped, as the reference builds it).  In train mode the BatchNorm running statistics in
    ``s`` are updated in place, as nn.BatchNorm2d does."""
    x = F.relu(_bn(F.conv2d(x, s["conv1.0.weight"], stride=2, padding=1), s, "conv1.1.", train))
    x = F.max_pool2d(x, 3, 2, 1)
    for st in ("stage2", "stage3", "stage4"):
        i = 0
        while f"{st}.{i}.group_conv1.weight" in s:
            p = f"{st}.{i}."
            stride = 2 if i == 0 else 1
            g = 1 if (st == "stage2" and i == 0) else groups
            out = F.relu(_bn(F.conv2d(x, s[p + "group_conv1.weight"], groups=g), s, p + "bn1.", train))
            out = _shuffle(out, g)
            b = out.shape[1]
            out = _bn(F.conv2d(out, s[p + "depthwise_conv3.weight"], stride=stride, padding=1, groups=b), s, p + "bn2.", train)
            out = _bn(F.conv2d(out, s[p + "group_conv.weight"], groups=g), s, p + "bn3.", train)
            if stride == 2:
                out = torch.cat([F.avg_pool2d(x, 3, 2, 1), out], dim=1)
            else:
                out = x + out
            x = F.relu(out)
            i += 1
    return F.linear(x.mean([2, 3]), s["fc.weight"], s["fc.bias"])


def train_step_grads(state, x, labels, groups):
    """fp32 train step on a copy of ``state``: (logits, loss, {name: grad}, state after the step's statistics update)."""
    s = {k: v.detach().clone() for k, v in state.items()}
    params = {k: v.requires_grad_() for k, v in s.items() if v.is_floating_point() and "running_" not in k}
    logits = shufflenet_forward(s, x, groups, True)
    loss = F.cross_entropy(logits, labels)
    grads = torch.autograd.grad(loss, list(params.values()))
    return logits.detach(), loss.detach(), dict(zip(params.keys(), grads)), {k: v.detach() for k, v in s.items()}
