"""autolog: patches `Trainer.fit` so that every fit logs params / per-epoch metrics / the model (what
`mlflow.tensorflow.autolog()` does for Keras in the reference, SURVEY.md §5.5)."""
from __future__ import annotations

from ..train.callbacks import Callback
from ..parallel import core as dist_core

_orig_fit = None


class _AutologCallback(Callback):
    def __init__(self, log_models: bool, fit_params: dict):
        self.log_models = log_models
        self.fit_params = fit_params
        self._own_run = False

    def on_train_begin(self, logs=None):
        from . import active_run, start_run, log_params

        if dist_core.rank() != 0:
            return
        if active_run() is None:
            start_run()
            self._own_run = True
        opt = self.trainer.optimizer
        base = getattr(opt, "opt", opt)
        log_params({**self.fit_params, "optimizer_name": getattr(base, "name", type(base).__name__),
                    "learning_rate": getattr(base, "learning_rate", None)})

    def on_epoch_end(self, epoch, logs=None):
        from . import log_metrics

        if dist_core.rank() != 0 or not logs:
            return
        log_metrics({k: v for k, v in logs.items() if isinstance(v, (int, float))}, step=epoch)

    def on_train_end(self, logs=None):
        from . import end_run
        from .models import log_model

        if dist_core.rank() != 0:
            return
        if self.log_models:
            log_model(self.trainer, "model")
        if self._own_run:
            end_run()


def install(trainer_module, enabled: bool, log_models: bool) -> None:
    global _orig_fit
    T = trainer_module.Trainer
    if _orig_fit is None:
        _orig_fit = T.fit
    if not enabled:
        T.fit = _orig_fit
        return

    def fit(self, x, steps_per_epoch=None, epochs=1, *args, **kw):
        params = {"epochs": epochs, "steps_per_epoch": steps_per_epoch}
        if kw.get("class_weight") is not None:   # as Keras's autolog records fit's class_weight
            params["class_weight"] = kw["class_weight"]
        cb = _AutologCallback(log_models, params)
        cbs = list(kw.pop("callbacks", None) or []) + [cb]
        return _orig_fit(self, x, steps_per_epoch, epochs, *args, callbacks=cbs, **kw)

    T.fit = fit
