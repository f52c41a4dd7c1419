"""Model zoo + the `build_model` / `preprocess` helpers of the reference (C13, C14).

    build_model(img_height, img_width, img_channels, num_classes)      (P1/02:159, P1/03:159)
    build_model(dropout=0.5)                                            (P2/01:92, P2/02:116)
    build_model()                                                       (P2/03:125)

`arch='resnet50'` (TARGET, default on an H100): the hand-scheduled sm_90a engine, fully trainable, bf16.
`arch='mobilenetv2'` (REF parity): frozen MobileNetV2 base + GAP + Dropout + Dense head - on a GPU the native
`MobileNetV2Engine` (depthwise / stem kernels + wgmma pointwise convs with folded-BN epilogues), on CPU (or with
`arch='mobilenetv2_torch'`, or `freeze_base=False`) the torch.nn module.
`arch='resnet50_torch'`: torchvision-architecture ResNet-50 as a plain nn.Module (CPU plumbing runs).
`arch='resnet50_head'`: ResNet-50 base + GAP + Dropout + Dense for transfer learning (`fine_tune_at`, `batchnorm`) - the
native `ResNet50Engine(fine_tune_at=k)` on an H100 at a square size that is a multiple of 32, else `ResNet50Head`.
"""
from __future__ import annotations

from typing import Optional

import torch

from .augment import Augmentation, check_augmentation
from .preprocess import (IMG_CHANNELS, IMG_HEIGHT, IMG_WIDTH, decode_batch, decode_image, preprocess, preprocess_tensor)

CLASSES = ["daisy", "dandelion", "roses", "sunflowers", "tulips"]  # reference P2/03:62


def build_model(img_height: int = IMG_HEIGHT, img_width: int = IMG_WIDTH, img_channels: int = IMG_CHANNELS,
                num_classes: int = 5, dropout: float = 0.5, arch: Optional[str] = None, batch_size: int = 32,
                freeze_base: bool = True, device=None, seed: int = 0, fine_tune_at: Optional[int] = None,
                augmentation: Optional[Augmentation] = None, batchnorm: str = "inference", **engine_kwargs):
    """``fine_tune_at=k`` (MobileNetV2 only, 0..19) fine-tunes ``base.features[k:]`` - conv weights and BatchNorm
    weight / bias - with every BatchNorm of the base in inference mode (Keras's ``base_model(x, training=False)``).
    ``k`` counts feature blocks (0 = stem, 1..17 = inverted-residual blocks, 18 = last 1x1 conv, 19 = head only), not
    Keras's 154 ``base_model.layers``.  ``None`` (default) keeps the base frozen, or fully trainable with
    training-mode BatchNorm when ``freeze_base=False``; the two options cannot be combined.

    ``augmentation`` (`Augmentation`): random flip / rotation / zoom / translation, MixUp or CutMix, and brightness /
    contrast / saturation / hue / grayscale of every training batch (Keras's augmentation layers in front of the model), on the device for the native engines;
    ``evaluate`` / ``predict`` never augment.  ``None`` (default) leaves every path unchanged.  Not available for ``arch='resnet50_torch'``.

    ``batchnorm`` (MobileNetV2 with ``fine_tune_at`` only): ``"inference"`` (default) as above, or ``"training"`` - the
    BatchNorms of ``base.features[k:]`` normalise with batch statistics in training steps and update their running
    statistics; ``evaluate`` / ``predict`` use the running statistics.

    ``arch="resnet50_head"`` is the same recipe with a ResNet-50 base: ``fine_tune_at=k`` in 0..17 (0 = stem, 1..16 =
    bottleneck blocks ``layer1.0`` .. ``layer4.2``, 17 = head only; None means 17) and the same ``batchnorm`` modes.
    It has no ``freeze_base=False``: the fully trainable model is ``arch="resnet50"``."""
    if isinstance(img_height, float) and img_width == IMG_WIDTH:  # build_model(dropout) positional form
        dropout, img_height = img_height, IMG_HEIGHT
    if img_channels != 3:
        raise ValueError("only 3-channel images are supported")
    augmentation = check_augmentation(augmentation)
    from .mobilenet import check_batchnorm, check_fine_tune_at

    check_batchnorm(batchnorm, fine_tune_at)
    if arch == "resnet50_head":
        from .resnet_engine import NUM_FEATURE_BLOCKS

        if not freeze_base:
            raise ValueError("arch='resnet50_head' fine-tunes a frozen base; the fully trainable model is arch='resnet50'")
        check_fine_tune_at(fine_tune_at, num_blocks=NUM_FEATURE_BLOCKS)
        k = NUM_FEATURE_BLOCKS if fine_tune_at is None else fine_tune_at
        if torch.cuda.is_available() and img_height == img_width and img_height % 32 == 0 \
                and (device is None or torch.device(device).type == "cuda"):
            from .resnet_engine import ResNet50Engine

            return ResNet50Engine(batch=batch_size, num_classes=num_classes, device=device, image_size=img_height,
                                  dropout=dropout, seed=seed, augmentation=augmentation, fine_tune_at=k,
                                  batchnorm=batchnorm, **engine_kwargs)
        from .resnet import ResNet50Head

        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            return ResNet50Head(num_classes, dropout, k, batchnorm, augmentation=augmentation, augmentation_seed=seed)
    if batchnorm == "training" and arch in ("resnet50", "resnet50_torch"):
        raise ValueError("batchnorm='training' applies to the MobileNetV2 model only")
    if fine_tune_at is not None:
        check_fine_tune_at(fine_tune_at, freeze_base)
        if arch is None:
            arch = "mobilenetv2"
        elif arch not in ("mobilenetv2", "mobilenetv2_head", "mobilenetv2_torch"):
            raise ValueError("fine_tune_at applies to the MobileNetV2 model only")
    if arch is None:
        arch = "resnet50" if (torch.cuda.is_available() and img_height == img_width and img_height % 32 == 0) else "mobilenetv2"
    if arch == "mobilenetv2_head":   # SURVEY.md 7.1's spelling of the reference's model (frozen MobileNetV2 base + trainable head)
        arch = "mobilenetv2"
    if arch == "resnet50":
        from .resnet_engine import ResNet50Engine

        return ResNet50Engine(batch=batch_size, num_classes=num_classes, device=device, image_size=img_height,
                              dropout=dropout, seed=seed, augmentation=augmentation, **engine_kwargs)
    if arch == "mobilenetv2" and freeze_base and torch.cuda.is_available() and img_height == img_width and img_height % 32 == 0 \
            and (device is None or torch.device(device).type == "cuda"):
        # the reference's own model on native kernels (frozen base = inference-mode layers; trainable Dense head)
        from .mobilenet_engine import MobileNetV2Engine

        return MobileNetV2Engine(batch=batch_size, num_classes=num_classes, device=device, image_size=img_height,
                                 dropout=dropout, seed=seed, fine_tune_at=fine_tune_at, augmentation=augmentation,
                                 batchnorm=batchnorm)
    if arch in ("mobilenetv2", "mobilenetv2_torch"):
        from .mobilenet import FrozenBaseClassifier, MobileNetV2Base

        g = torch.random.fork_rng(devices=[])
        with g:
            torch.manual_seed(seed)
            base = MobileNetV2Base()
            return FrozenBaseClassifier(base, base.out_channels, num_classes, dropout, freeze_base, fine_tune_at,
                                        augmentation=augmentation, augmentation_seed=seed, batchnorm=batchnorm)
    if arch == "resnet50_torch":
        if augmentation is not None:
            raise ValueError("arch='resnet50_torch' is the plain torchvision module and takes no augmentation")
        import torchvision

        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            return torchvision.models.resnet50(weights=None, num_classes=num_classes)
    raise ValueError(f"unknown arch {arch!r}")


__all__ = ["build_model", "Augmentation", "preprocess", "preprocess_tensor", "decode_image", "decode_batch", "CLASSES", "IMG_HEIGHT", "IMG_WIDTH",
           "IMG_CHANNELS"]
