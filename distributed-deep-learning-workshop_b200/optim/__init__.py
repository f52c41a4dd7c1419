"""Fused optimizers (SURVEY.md K16; reference: `tf.keras.optimizers.Adam` P1/02:201, `Adadelta|Adam` looked up
by name in the HPO objective P2/01:154-155), with Keras's gradient clipping options (README, "Optimizers and gradient
clipping")."""
from .fused import SGD, Adadelta, Adagrad, Adam, Adamax, AdamW, FlatOptimizer, Lamb, OPTIMIZERS, RMSprop, get

__all__ = ["SGD", "Adam", "Adadelta", "RMSprop", "Adagrad", "Adamax", "AdamW", "Lamb", "FlatOptimizer", "get",
           "OPTIMIZERS"]
