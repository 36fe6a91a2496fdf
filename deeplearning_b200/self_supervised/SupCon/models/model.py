"""Drop-in for the reference's self-supervised/SupCon/models/model.py: ``create_encoder``, ``SupConModel`` and
``build_model`` with the reference's parameter names (encoder.0 ... encoder.7, head.0 / head.2, classifier), registration
order and RNG consumption, so a seeded constructor gives the reference's state_dict bit for bit.  ``forward`` runs on the
GPU engine (engine/supcon.py); there is no CPU path.

Deviation: the reference builds every encoder with ``pretrained=True``, which downloads ImageNet weights.  This drop-in
builds from random initialisation; load pretrained or checkpointed weights with ``load_state_dict``."""
import torch
import torch.nn as nn

from .backbone import BACKBONES


def create_encoder(backbone):
    """(encoder, features_dim): the backbone's children without its classifier, as an nn.Sequential."""
    if "timm_" in backbone:
        raise NotImplementedError(f"backbone {backbone!r}: timm backbones are not implemented on the GPU engine")
    if backbone not in BACKBONES:
        raise RuntimeError("Specify the correct backbone name. Either one of torchvision backbones, or a timm backbone."
                           "For timm - add prefix 'timm_'. For instance, timm_resnet18")
    model = BACKBONES[backbone](pretrained=False)
    features_dim = model.fc.in_features
    return nn.Sequential(*list(model.children())[:-1]), features_dim


class SupConModel(nn.Module):
    def __init__(self, backbone="resnet50", projection_dim=128, second_stage=False, num_classes=1000):
        super().__init__()
        self.encoder, self.features_dim = create_encoder(backbone)
        self.second_stage = second_stage
        self.projection_head = True
        self.projection_dim = projection_dim
        self.embed_dim = projection_dim
        if self.second_stage:
            for param in self.encoder.parameters():
                param.requires_grad = False
            self.classifier = nn.Linear(self.features_dim, num_classes)
        else:
            self.head = nn.Sequential(nn.Linear(self.features_dim, self.features_dim), nn.ReLU(inplace=True),
                                      nn.Linear(self.features_dim, self.projection_dim))

    def use_projection_head(self, mode):
        self.projection_head = mode
        self.embed_dim = self.projection_dim if mode else self.features_dim

    def forward(self, x):
        """Stage 1: fp32 unit embeddings [B, embed_dim] (F.normalize(head(feat)), or F.normalize(feat) with the projection
        head off); stage 2: fp32 logits [B, num_classes]."""
        from deeplearning_b200.engine import supcon as engine

        return engine.apply(self, x)


def build_model(backbone, second_stage=False, num_classes=None, ckpt_pretrained=None):
    model = SupConModel(backbone=backbone, second_stage=second_stage, num_classes=num_classes)
    if ckpt_pretrained:
        model.load_state_dict(torch.load(ckpt_pretrained)["model_state_dict"], strict=False)
    return model
