"""Keras-style loss objects for `Trainer.compile(loss=...)`.

The reference compiles every model with `tf.keras.losses.SparseCategoricalCrossentropy(from_logits=True)` (P1/02:203,
P1/03:223,346, P2/01:165, P2/02:226, P2/03:301); the models here output logits and the fused softmax-cross-entropy kernel
(csrc/elementwise.cu `softmax_ce`) / `torch.nn.functional.cross_entropy` consume logits, so that is the one form offered.
`CategoricalCrossentropy` adds Keras's label smoothing and the soft targets of MixUp / CutMix; `Distillation` adds a
teacher's softened logits to it (knowledge distillation, fused into the same head kernel on the native engines)."""
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


def _is_native_engine(m) -> bool:
    return hasattr(m, "param_specs") and hasattr(m, "forward_logits") and hasattr(m, "bind_grad_buffer")


def _number(name: str, v, lo: float, hi: float, lo_open: bool = False) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v > hi \
            or (v <= lo if lo_open else v < lo):
        rng = f"({lo:g}, {hi:g}]" if lo_open else f"[{lo:g}, {hi:g}]"
        raise ValueError(f"Distillation: {name} must be a finite number in {rng}, got {v!r}")
    return float(v)


class Distillation:
    """Knowledge distillation, as the ``Distiller`` of the Keras "Knowledge Distillation" example, passed as
    ``Trainer.compile(loss=Distillation(teacher, ...))``.  Per row, with ``s`` the student's logits, ``t`` the
    teacher's and ``target`` the one-hot, smoothed or MixUp / CutMix target of `CategoricalCrossentropy`::

        loss    = alpha * sum_k target_k (lse(s) - s_k) + (1 - alpha) * T^2 * KL(softmax(t / T) || softmax(s / T))
        dlogits = alpha (softmax(s) - target) + (1 - alpha) T (softmax(s / T) - softmax(t / T))

    ``fit`` logs ``loss`` (the combined loss), ``accuracy``, and the two terms the Keras example reports:
    ``student_loss`` (the cross-entropy) and ``distillation_loss`` (``T^2 KL``).  ``evaluate``, ``predict``, serving,
    checkpoints and tracking see the student alone: ``evaluate`` reports the student's
    ``CategoricalCrossentropy(from_logits=True, label_smoothing)`` and never runs the teacher, so ``val_loss`` stays
    comparable with runs trained without a teacher (Keras 3's ``Distiller`` evaluates the combined loss).

    ``teacher`` is frozen: its weights, BatchNorm statistics and dropout never change, and it always runs in inference
    mode.  For a native engine student it is a native engine (`ResNet50Engine` or `MobileNetV2Engine`, any
    ``fine_tune_at``) with the student's ``batch``, ``image_size``, ``num_classes`` and device; its logits are computed
    inside the student's training step (and CUDA graph), from the student's stem input.  For a torch-module student it
    is a torch module, run under ``eval()`` and ``no_grad``.  ``BroadcastGlobalVariablesCallback`` broadcasts the
    teacher's weights and statistics too.

    Two deliberate differences from the Keras example:

    * the KL divergence comes straight from the two log-softmaxes; Keras's ``KLDivergence`` clips both distributions to
      [1e-7, 1], so the two differ only where a probability is below 1e-7;
    * the teacher sees the batch the student's stem reads - augmented and, when on, mixed - where the Keras example
      feeds the teacher the un-augmented ``x``: teacher and student see the same view ("a good teacher is patient and
      consistent", Beyer et al. 2022)."""

    name = "distillation"

    def __init__(self, teacher, alpha: float = 0.1, temperature: float = 3.0, label_smoothing: float = 0.0):
        import torch

        if not (_is_native_engine(teacher) or isinstance(teacher, torch.nn.Module)):
            raise ValueError(f"Distillation: teacher must be a native engine (ResNet50Engine / MobileNetV2Engine) or a "
                             f"torch module, got {type(teacher).__name__}")
        self.teacher = teacher
        self.alpha = _number("alpha", alpha, 0.0, 1.0)
        self.temperature = _number("temperature", temperature, 0.0, math.inf, lo_open=True)
        self.label_smoothing = CategoricalCrossentropy(True, label_smoothing).label_smoothing

    def check_student(self, student) -> None:
        """Refuse a teacher that cannot teach ``student``: the student itself, a teacher of the other kind (engine vs
        torch module), or an engine teacher whose batch, image size, class count or device differ."""
        t = self.teacher
        if t is student:
            raise ValueError("Distillation: teacher is the student itself")
        if _is_native_engine(student) != _is_native_engine(t):
            raise ValueError("Distillation: teacher and student must both be native engines or both torch modules")
        if _is_native_engine(student):
            for field in ("batch", "image_size", "num_classes", "device"):
                if getattr(t, field) != getattr(student, field):
                    raise ValueError(f"Distillation: teacher {field} {getattr(t, field)!r} differs from the student's "
                                     f"{getattr(student, field)!r}")

    def __repr__(self) -> str:
        return (f"Distillation(teacher={type(self.teacher).__name__}, alpha={self.alpha}, "
                f"temperature={self.temperature}, label_smoothing={self.label_smoothing})")


def label_smoothing_of(loss) -> float:
    """The label smoothing of a loss `Trainer.compile` accepts: "sparse_categorical_crossentropy" /
    `SparseCategoricalCrossentropy` (0), "categorical_crossentropy" (0), `CategoricalCrossentropy` or `Distillation`;
    anything else raises ``ValueError``."""
    if isinstance(loss, (CategoricalCrossentropy, Distillation)):
        return loss.label_smoothing
    if isinstance(loss, str) and loss == "categorical_crossentropy":
        return 0.0
    name = loss if isinstance(loss, str) else getattr(loss, "name", "sparse_categorical_crossentropy")
    if "sparse_categorical_crossentropy" not in name:
        raise ValueError("the losses implemented are sparse categorical cross-entropy and categorical cross-entropy, "
                         "from logits")
    return 0.0


__all__ = ["SparseCategoricalCrossentropy", "CategoricalCrossentropy", "Distillation"]
