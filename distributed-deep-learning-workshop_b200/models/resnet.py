"""ResNet-50 transfer learning as a torch module (C14, ``arch="resnet50_head"`` on CPU or without the native engine):
a torchvision ResNet-50 base + GlobalAveragePooling + Dropout + Dense(num_classes), with the top of the base trainable
from feature block ``fine_tune_at`` upward.  The state-dict keys are exactly torchvision's ``resnet50``, so weights move
freely between this module, `ResNet50Engine(fine_tune_at=k)` and the fully trainable ``arch="resnet50"`` models."""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import nn
from torchvision.models.resnet import Bottleneck, ResNet

from .resnet_engine import NUM_FEATURE_BLOCKS


class ResNet50Head(ResNet):
    """Sequential[ResNet-50 base, GlobalAveragePooling2D, Dropout(p), Dense(num_classes)] - logits.

    ``fine_tune_at=k`` (0..17; None = 17) counts feature blocks: 0 = stem (``conv1``, ``bn1``), 1..16 = the bottleneck
    blocks in order (``layer1.0`` = 1 ... ``layer4.2`` = 16), 17 = the head only.  Conv weights and BatchNorm weight /
    bias of blocks ``k..16`` (and the stem when k = 0) train with the head; the frozen prefix runs under no_grad and its
    BatchNorms stay in inference mode.

    ``batchnorm="inference"`` (default) keeps every BatchNorm in inference mode in ``train()`` (Keras's
    ``base_model(x, training=False)``); ``"training"`` (needs ``fine_tune_at``) gives the trainable blocks batch
    statistics and the running-statistics update (momentum 0.1, eps 1e-5).

    ``augmentation`` (`models.augment.Augmentation`) is applied by the trainer's module backend to the uint8 batch of
    every training step, keyed by ``augmentation_seed``; the module's own forward never augments."""

    def __init__(self, num_classes: int = 5, dropout: float = 0.5, fine_tune_at: Optional[int] = None,
                 batchnorm: str = "inference", augmentation=None, augmentation_seed: int = 0):
        from .augment import check_augmentation
        from .mobilenet import check_batchnorm, check_fine_tune_at

        check_fine_tune_at(fine_tune_at, num_blocks=NUM_FEATURE_BLOCKS)
        check_batchnorm(batchnorm, fine_tune_at)
        super().__init__(Bottleneck, [3, 4, 6, 3], num_classes=num_classes)
        self.fine_tune_at = fine_tune_at
        self.batchnorm = batchnorm
        self.augmentation = check_augmentation(augmentation)
        self.augmentation_seed = int(augmentation_seed)
        self.dropout = nn.Dropout(dropout)   # no parameters: the state-dict keys stay torchvision's
        k = self.k
        for i, blk in enumerate(self.feature_blocks()):
            for p in blk.parameters():
                p.requires_grad_(i >= k)

    @property
    def k(self) -> int:
        return NUM_FEATURE_BLOCKS if self.fine_tune_at is None else self.fine_tune_at

    def feature_blocks(self) -> List[nn.Module]:
        """[stem, layer1.0, ..., layer4.2]: index i is feature block i."""
        stem = nn.ModuleList([self.conv1, self.bn1])
        return [stem] + [b for layer in (self.layer1, self.layer2, self.layer3, self.layer4) for b in layer]

    def train(self, mode: bool = True):
        super().train(mode)
        blocks = self.feature_blocks()
        for i, blk in enumerate(blocks):
            if i < self.k or self.batchnorm == "inference":
                blk.eval()   # frozen, or BatchNorm in inference mode (no BatchNorm outside the blocks)
        return self

    def _stem(self, x):
        return self.maxpool(self.relu(self.bn1(self.conv1(x))))

    def forward(self, x):
        k = self.k
        stages = [self._stem] + [b for layer in (self.layer1, self.layer2, self.layer3, self.layer4) for b in layer]
        with torch.no_grad():
            for f in stages[:k]:
                x = f(x)
        for f in stages[k:]:
            x = f(x)
        x = torch.flatten(self.avgpool(x), 1)
        return self.fc(self.dropout(x))
