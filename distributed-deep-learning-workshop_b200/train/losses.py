"""Keras-style loss objects for `Trainer.compile(loss=...)`.

The reference compiles every model with `tf.keras.losses.SparseCategoricalCrossentropy(from_logits=True)` (P1/02:203,
P1/03:223,346, P2/01:165, P2/02:226, P2/03:301); the models here output logits and the fused softmax-cross-entropy kernel
(csrc/elementwise.cu `softmax_ce`) / `torch.nn.functional.cross_entropy` consume logits, so that is the one form offered.
`CategoricalCrossentropy` adds Keras's label smoothing and the soft targets of MixUp / CutMix."""
from __future__ import annotations

import math


class SparseCategoricalCrossentropy:
    name = "sparse_categorical_crossentropy"

    def __init__(self, from_logits: bool = False, name: str = "sparse_categorical_crossentropy", **_ignored):
        if not from_logits:
            raise ValueError("the models output logits: use SparseCategoricalCrossentropy(from_logits=True) "
                             "(what the reference workflow does)")
        self.from_logits = True
        self.name = name

    def __repr__(self) -> str:
        return "SparseCategoricalCrossentropy(from_logits=True)"


class CategoricalCrossentropy:
    """Keras's ``CategoricalCrossentropy(from_logits=True, label_smoothing=eps)``, for label smoothing and for the soft
    targets of MixUp / CutMix (`models.Augmentation`).

    Unlike Keras, it takes the integer labels the loaders yield, not one-hot rows: the one-hot, smoothed or mixed target
    ``(1 - eps) (lambda onehot(y) + mu onehot(y_partner)) + eps / K`` is formed on the device, inside the head kernel of
    the native engines (or from the reference mix rows on the module backend).  ``evaluate`` reports the smoothed loss,
    as Keras's ``val_loss`` does; it never mixes."""

    name = "categorical_crossentropy"

    def __init__(self, from_logits: bool = False, label_smoothing: float = 0.0,
                 name: str = "categorical_crossentropy"):
        if not from_logits:
            raise ValueError("the models output logits: use CategoricalCrossentropy(from_logits=True)")
        if isinstance(label_smoothing, bool) or not isinstance(label_smoothing, (int, float)) \
                or not math.isfinite(label_smoothing) or not 0.0 <= label_smoothing <= 1.0:
            raise ValueError(f"label_smoothing must be a number in [0, 1], got {label_smoothing!r}")
        self.from_logits = True
        self.label_smoothing = float(label_smoothing)
        self.name = name

    def __repr__(self) -> str:
        return f"CategoricalCrossentropy(from_logits=True, label_smoothing={self.label_smoothing})"


def label_smoothing_of(loss) -> float:
    """The label smoothing of a loss `Trainer.compile` accepts: "sparse_categorical_crossentropy" /
    `SparseCategoricalCrossentropy` (0), "categorical_crossentropy" (0) or `CategoricalCrossentropy`; anything else
    raises ``ValueError``."""
    if isinstance(loss, CategoricalCrossentropy):
        return loss.label_smoothing
    if isinstance(loss, str) and loss == "categorical_crossentropy":
        return 0.0
    name = loss if isinstance(loss, str) else getattr(loss, "name", "sparse_categorical_crossentropy")
    if "sparse_categorical_crossentropy" not in name:
        raise ValueError("the losses implemented are sparse categorical cross-entropy and categorical cross-entropy, "
                         "from logits")
    return 0.0


__all__ = ["SparseCategoricalCrossentropy", "CategoricalCrossentropy"]
