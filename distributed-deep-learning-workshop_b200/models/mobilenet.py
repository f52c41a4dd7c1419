"""The reference's own model (C14): MobileNetV2 base (frozen) + GlobalAveragePooling + Dropout + Dense(num_classes)
(P1/02:159-178; `build_model(dropout)` P2/01:92-108).  Pure torch.nn - it is the *parity* model (6,405 trainable
parameters => a ~25 KB all-reduce, SURVEY.md Q11), not the performance target; it runs through the module backend
of the Trainer, on GPU or CPU.  No pretrained weights exist offline, so the base is random-init."""
from __future__ import annotations

import torch
from torch import nn


def _make_divisible(v, divisor=8):
    return max(divisor, int(v + divisor / 2) // divisor * divisor)


class ConvBNReLU6(nn.Sequential):
    def __init__(self, cin, cout, k=3, stride=1, groups=1):
        super().__init__(nn.Conv2d(cin, cout, k, stride, (k - 1) // 2, groups=groups, bias=False),
                         nn.BatchNorm2d(cout), nn.ReLU6(inplace=True))


class InvertedResidual(nn.Module):
    def __init__(self, cin, cout, stride, expand):
        super().__init__()
        hidden = int(round(cin * expand))
        self.use_res = stride == 1 and cin == cout
        layers = []
        if expand != 1:
            layers.append(ConvBNReLU6(cin, hidden, 1))
        layers += [ConvBNReLU6(hidden, hidden, 3, stride, groups=hidden), nn.Conv2d(hidden, cout, 1, bias=False),
                   nn.BatchNorm2d(cout)]
        self.conv = nn.Sequential(*layers)

    def forward(self, x):
        return x + self.conv(x) if self.use_res else self.conv(x)


class MobileNetV2Base(nn.Module):
    """include_top=False feature extractor: [B,3,H,W] -> [B,1280,H/32,W/32]."""

    def __init__(self, width_mult: float = 1.0):
        super().__init__()
        cfg = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]
        cin = _make_divisible(32 * width_mult)
        self.out_channels = _make_divisible(1280 * max(1.0, width_mult))
        feats = [ConvBNReLU6(3, cin, 3, 2)]
        for t, c, n, s in cfg:
            cout = _make_divisible(c * width_mult)
            for i in range(n):
                feats.append(InvertedResidual(cin, cout, s if i == 0 else 1, t))
                cin = cout
        feats.append(ConvBNReLU6(cin, self.out_channels, 1))
        self.features = nn.Sequential(*feats)

    def forward(self, x):
        return self.features(x)


NUM_FEATURE_BLOCKS = 19   # base.features: stem, 17 inverted-residual blocks, last 1x1 conv


def check_fine_tune_at(fine_tune_at, freeze_base: bool = True, num_blocks: int = NUM_FEATURE_BLOCKS) -> None:
    """``fine_tune_at`` is None or an int in 0..``num_blocks`` (the head-only value of the architecture: 19 for
    MobileNetV2, 17 for ResNet-50)."""
    if fine_tune_at is None:
        return
    if not freeze_base:
        raise ValueError("fine_tune_at keeps the base's BatchNorm in inference mode; freeze_base=False trains it in "
                         "training mode - pass one or the other")
    if isinstance(fine_tune_at, bool) or not isinstance(fine_tune_at, int) or not 0 <= fine_tune_at <= num_blocks:
        raise ValueError(f"fine_tune_at must be an int in 0..{num_blocks}, got {fine_tune_at!r}")


BATCHNORM_MODES = ("inference", "training")


def check_batchnorm(batchnorm, fine_tune_at) -> None:
    """``batchnorm="training"`` normalises the trainable blocks ``base.features[fine_tune_at:]`` with batch statistics;
    it needs ``fine_tune_at`` (the whole base in training mode is ``freeze_base=False``)."""
    if batchnorm not in BATCHNORM_MODES:
        raise ValueError(f"batchnorm must be 'inference' or 'training', got {batchnorm!r}")
    if batchnorm == "training" and fine_tune_at is None:
        raise ValueError("batchnorm='training' applies to the trainable blocks of fine_tune_at=k; to train the whole "
                         "base with training-mode BatchNorm pass freeze_base=False instead")


class FrozenBaseClassifier(nn.Module):
    """Sequential[base (frozen, inference-mode BN), GlobalAveragePooling2D, Dropout(p), Dense(num_classes)] - logits.

    ``fine_tune_at=k`` (0..19) is the second phase of Keras's transfer-learning recipe: ``base.features[k:]`` train
    their conv weights and BatchNorm weight / bias, ``features[:k]`` stay frozen (run under no_grad), and every BatchNorm
    of the base stays in inference mode (running statistics, never updated), as ``base_model(x, training=False)`` does.
    ``k`` counts feature blocks (0 = stem, 1..17 = inverted-residual blocks, 18 = last 1x1 conv, 19 = head only), not
    Keras's 154 ``base_model.layers``.

    ``batchnorm="training"`` (with ``fine_tune_at=k``) puts the BatchNorms of ``base.features[k:]`` in training mode in
    ``train()``: batch statistics, running statistics updated (momentum 0.1, eps 1e-5), as Keras does when the top of
    ``base_model`` is unfrozen and called without ``training=False``.  ``features[:k]`` stay in inference mode.

    ``augmentation`` (`models.augment.Augmentation`) is applied by the trainer's module backend to the uint8 batch of
    every training step (the reference implementation of the engines' kernels, keyed by ``augmentation_seed`` and the
    rank); the module's own forward never augments."""

    def __init__(self, base: nn.Module, feat_channels: int, num_classes: int, dropout: float = 0.5,
                 freeze_base: bool = True, fine_tune_at=None, augmentation=None, augmentation_seed: int = 0,
                 batchnorm: str = "inference"):
        from .augment import check_augmentation

        super().__init__()
        check_fine_tune_at(fine_tune_at, freeze_base)
        check_batchnorm(batchnorm, fine_tune_at)
        self.batchnorm = batchnorm
        self.augmentation = check_augmentation(augmentation)
        self.augmentation_seed = int(augmentation_seed)
        self.base = base
        self.freeze_base = freeze_base
        self.fine_tune_at = fine_tune_at
        if freeze_base:
            for p in self.base.parameters():
                p.requires_grad_(False)
        if fine_tune_at is not None:
            for p in self.base.features[fine_tune_at:].parameters():
                p.requires_grad_(True)
        self.dropout = nn.Dropout(dropout)
        self.fc = nn.Linear(feat_channels, num_classes)

    def train(self, mode: bool = True):
        super().train(mode)
        if self.freeze_base:
            self.base.eval()  # frozen base => BatchNorm in inference mode (Keras `layer.trainable = False`)
            if self.batchnorm == "training":
                self.base.features[self.fine_tune_at:].train(mode)
        return self

    def forward(self, x):
        if self.fine_tune_at is not None:
            k = self.fine_tune_at
            with torch.no_grad():
                f = self.base.features[:k](x)
            f = self.base.features[k:](f)
        elif self.freeze_base:
            with torch.no_grad():
                f = self.base(x)
        else:
            f = self.base(x)
        return self.fc(self.dropout(f.mean(dim=(2, 3))))
