"""Oracle: the SupCon model and losses (self-supervised/SupCon of the reference) restated functionally in fp32 PyTorch.

Encoder: oracle/resnet.py's stem and blocks on the drop-in's ``encoder.N`` keys (0 = conv1, 1 = bn1, 4 .. 7 = layer1 ..
layer4), then the global average pool.  Head (models/model.py SupConModel): Linear -> ReLU -> Linear, F.normalize.
SupCon loss (losses/SupConLoss.py, contrast_mode 'all'): logits over all rows of cat(unbind(features, 1)), the row max
subtracted, self-contrast masked out, mean log-probability of the positives.  LabelSmoothingLoss (losses/LabelSmooth.py):
1 - s on the target class, s / (classes - 1) elsewhere.
"""
import torch
import torch.nn.functional as F

from .resnet import _block, _bn


def resnet_state(state):
    """The encoder's keys of a SupConModel state_dict renamed to a ResNet's (conv1, bn1, layer1 .. layer4)."""
    names = {"0": "conv1", "1": "bn1", "4": "layer1", "5": "layer2", "6": "layer3", "7": "layer4"}
    out = {}
    for k, v in state.items():
        if k.startswith("encoder."):
            idx, rest = k[len("encoder."):].split(".", 1)
            out[f"{names[idx]}.{rest}"] = v
    return out


def encoder_forward(rstate, x, train):
    """Pooled fp32 features [B, F] of the ResNet trunk (resnet_state keys; running statistics updated in train mode)."""
    h = F.conv2d(x, rstate["conv1.weight"], stride=2, padding=3)
    h = F.max_pool2d(F.relu(_bn(rstate, "bn1", h, train)), 3, 2, 1)
    for li in range(1, 5):
        bi = 0
        while f"layer{li}.{bi}.conv1.weight" in rstate:
            h = _block(rstate, f"layer{li}.{bi}", h, 2 if (li > 1 and bi == 0) else 1, train)
            bi += 1
    return torch.flatten(F.adaptive_avg_pool2d(h, 1), 1)


def supcon_forward(state, x, train, projection_head=True):
    """SupConModel.forward: stage 1 (``head.*`` keys) unit embeddings, stage 2 (``classifier.*``) logits.  Running statistics
    in ``state`` are updated in place in train mode."""
    feat = encoder_forward(resnet_state(state), x, train)   # (the renamed dict shares the statistics tensors)
    if "classifier.weight" in state:
        return F.linear(feat, state["classifier.weight"], state["classifier.bias"])
    if not projection_head:
        return F.normalize(feat, dim=1)
    h = F.relu(F.linear(feat, state["head.0.weight"], state["head.0.bias"]))
    return F.normalize(F.linear(h, state["head.2.weight"], state["head.2.bias"]), dim=1)


def supcon_loss(features, labels=None, temperature=0.07, base_temperature=0.07):
    """SupConLoss(temperature, 'all', base_temperature)(features [bsz, n_views, D], labels [bsz] or None)."""
    bsz, n_views = features.shape[:2]
    features = features.reshape(bsz, n_views, -1)
    if labels is None:
        mask = torch.eye(bsz, dtype=torch.float32, device=features.device)
    else:
        labels = labels.contiguous().view(-1, 1)
        mask = torch.eq(labels, labels.T).float()
    contrast = torch.cat(torch.unbind(features, dim=1), dim=0)
    logits = torch.div(torch.matmul(contrast, contrast.T), temperature)
    logits_max, _ = torch.max(logits, dim=1, keepdim=True)
    logits = logits - logits_max.detach()
    mask = mask.repeat(n_views, n_views)
    logits_mask = torch.scatter(torch.ones_like(mask), 1, torch.arange(bsz * n_views, device=features.device).view(-1, 1), 0)
    mask = mask * logits_mask
    exp_logits = torch.exp(logits) * logits_mask
    log_prob = logits - torch.log(exp_logits.sum(1, keepdim=True))
    mean_log_prob_pos = (mask * log_prob).sum(1) / mask.sum(1)
    loss = -(temperature / base_temperature) * mean_log_prob_pos
    return loss.view(n_views, bsz).mean()


def label_smoothing_loss(pred, target, classes, smoothing):
    pred = pred.log_softmax(dim=-1)
    true_dist = torch.full_like(pred, smoothing / (classes - 1))
    true_dist.scatter_(1, target.unsqueeze(1), 1.0 - smoothing)
    return torch.mean(torch.sum(-true_dist * pred, dim=-1))


def train_step_grads(state, images, labels, temperature, base_temperature=0.07):
    """One stage-1 step of the reference loop: images = cat(view1, view2) [2B, 3, H, W]; embeddings split into the two
    views, stacked to [B, 2, D], SupCon loss.  Returns (embeddings, loss, {name: grad}) with ``state``'s running statistics
    updated."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in state.items() if v.is_floating_point()
              and "running_" not in k}
    work = dict(state)
    work.update(params)
    emb = supcon_forward(work, images, True)
    B = images.shape[0] // 2
    f1, f2 = torch.split(emb, [B, B], dim=0)
    loss = supcon_loss(torch.cat([f1.unsqueeze(1), f2.unsqueeze(1)], dim=1), labels, temperature, base_temperature)
    grads = torch.autograd.grad(loss, list(params.values()))
    for k in state:
        if "running_" in k or "num_batches" in k:
            state[k] = work[k]
    return emb.detach(), loss.detach(), dict(zip(params.keys(), grads))
