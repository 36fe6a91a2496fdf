"""Oracle: the reference EfficientNet forward restated functionally in fp32 PyTorch
(classification/efficientNet/models/network.py): stem ConvBNAction 3x3/2 (:313-319), MBConv blocks (:176-242) =
[expand 1x1 conv-BN-SiLU] -> depthwise kxk conv-BN-SiLU -> SELayer (:126-145: avg_pool -> biased 1x1 conv -> SiLU -> biased
1x1 conv -> Sigmoid, x * y) -> project 1x1 conv-BN -> DropPath (:33-62) -> + x; top 1x1 ConvBNAction (:328-333); avgpool,
flatten, Dropout (inplace), Linear (:357-362).  BatchNorm uses eps=1e-3, momentum 0.1 and updates the running buffers
(and num_batches_tracked) of the state dict it is given in train mode.

``drop``: optional list with one entry per block that has a DropPath (a residual block with a drop-connect rate > 0), in
forward order: ``(random_tensor [B] of 0/1, keep_prob)`` - the reference's ``floor(keep_prob + rand)`` - applied as the
reference does: ``x.div(keep_prob) * random_tensor``.  ``mask``: the classifier dropout's multiplier fp32 [B, F] (0 or
1 / (1 - p), what ``F.dropout`` of a tensor of ones returns), applied as ``x * mask``."""
import math

import torch
import torch.nn.functional as F

# kernel, in, out, expand ratio, stride, repeats of stages 2 - 8 (network.py:259-265)
_CNF = [(3, 32, 16, 1, 1, 1), (3, 16, 24, 6, 2, 2), (5, 24, 40, 6, 2, 2), (3, 40, 80, 6, 2, 3), (5, 80, 112, 6, 1, 3),
        (5, 112, 192, 6, 2, 4), (3, 192, 320, 6, 1, 1)]
# width, depth, classifier dropout of efficientnet_b0 .. b7 (network.py:368-429)
COEFFS = {f"b{i}": c for i, c in enumerate([(1.0, 1.0, 0.2), (1.0, 1.1, 0.2), (1.1, 1.2, 0.3), (1.2, 1.4, 0.3),
                                            (1.4, 1.8, 0.4), (1.6, 2.2, 0.4), (1.8, 2.6, 0.5), (2.0, 3.1, 0.5)])}


def plan(name, drop_connect_rate=0.2):
    """[(index, kernel, stride, drop_rate)] of every MBConv block of efficientnet_<name>, in order."""
    _, depth, _ = COEFFS[name]
    reps = [int(math.ceil(r * depth)) for *_, r in _CNF]
    total = float(sum(reps))
    out, b = [], 0
    for stage, ((k, _, _, _, s, _), n) in enumerate(zip(_CNF, reps)):
        for i in range(n):
            out.append((str(stage + 1) + chr(i + 97), k, s if i == 0 else 1, drop_connect_rate * b / total))
            b += 1
    return out


def _bn(x, s, p, train):
    if train and (p + "num_batches_tracked") in s:
        s[p + "num_batches_tracked"].add_(1)
    return F.batch_norm(x, s[p + "running_mean"], s[p + "running_var"], s[p + "weight"], s[p + "bias"], train, 0.1, 1e-3)


def _cba(x, s, p, train, stride=1, groups=1, act=True):
    w = s[p + "0.weight"]
    y = _bn(F.conv2d(x, w, None, stride, (w.shape[-1] - 1) // 2, 1, groups), s, p + "1.", train)
    return F.silu(y) if act else y


def efficientnet_forward(s, x, blocks, train=False, drop=None, mask=None):
    """Logits of the network whose parameters and buffers are ``s`` (state_dict names) for the block plan ``blocks``."""
    drop = list(drop) if (drop is not None and train) else None
    x = _cba(x, s, "features.stem_conv.", train, stride=2)
    for idx, k, stride, rate in blocks:
        p = f"features.{idx}.block."
        cin = x.shape[1]
        y = x
        if p + "expand_conv.0.weight" in s:
            y = _cba(y, s, p + "expand_conv.", train)
        y = _cba(y, s, p + "dwconv.", train, stride=stride, groups=y.shape[1])
        g = F.adaptive_avg_pool2d(y, 1)
        g = F.silu(F.conv2d(g, s[p + "se.fc.0.weight"], s[p + "se.fc.0.bias"]))
        g = torch.sigmoid(F.conv2d(g, s[p + "se.fc.2.weight"], s[p + "se.fc.2.bias"]))
        y = y * g.view(g.shape[0], g.shape[1], 1, 1)
        y = _cba(y, s, p + "project_conv.", train, act=False)
        if stride == 1 and cin == y.shape[1]:
            if rate > 0 and drop is not None:
                r, keep = drop.pop(0)
                y = y.div(keep) * r.to(y.dtype).view(-1, 1, 1, 1)
            y += x
        x = y
    x = _cba(x, s, "features.top.", train)
    x = torch.flatten(F.adaptive_avg_pool2d(x, 1), 1)
    if train and mask is not None:
        x = x * mask
    return F.linear(x, s["classifier.1.weight"] if "classifier.1.weight" in s else s["classifier.0.weight"],
                    s["classifier.1.bias"] if "classifier.1.bias" in s else s["classifier.0.bias"])


def train_step_grads(state, x, labels, blocks, drop=None, mask=None):
    """fp32 train step on a copy of ``state``: (logits, loss, {name: grad}, state after the step)."""
    s = {k: v.detach().clone() for k, v in state.items()}
    params = {k: v.requires_grad_(True) for k, v in s.items() if v.is_floating_point() and "running" not in k}
    logits = efficientnet_forward(s, x, blocks, train=True, drop=drop, mask=mask)
    loss = F.cross_entropy(logits, labels)
    grads = torch.autograd.grad(loss, list(params.values()))
    return logits.detach(), loss.detach(), dict(zip(params.keys(), grads)), s
