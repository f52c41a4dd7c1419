"""Keras-like training surface (SURVEY.md L4): Trainer.compile / fit / evaluate / predict, History, callbacks."""
from .callbacks import (Callback, History, EarlyStopping, ReduceLROnPlateau, ModelCheckpoint, LambdaCallback,
                        CallbackList)
from .trainer import Trainer
from .flat import FlatParams
from . import callbacks, losses
from .losses import CategoricalCrossentropy, Distillation, SparseCategoricalCrossentropy

__all__ = ["Trainer", "Callback", "History", "EarlyStopping", "ReduceLROnPlateau", "ModelCheckpoint",
           "LambdaCallback", "CallbackList", "FlatParams", "losses", "callbacks", "SparseCategoricalCrossentropy",
           "CategoricalCrossentropy", "Distillation"]
