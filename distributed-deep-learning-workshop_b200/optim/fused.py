"""Fused flat-buffer optimizers.

A model exposes ONE flat fp32 parameter buffer, ONE flat fp32 gradient buffer and (optionally) ONE flat bf16
working copy (`ResNet50Engine`, or `FlatParams` for any `torch.nn.Module`).  `step()` is a single kernel launch
(csrc/optim.cu) that reads the (all-reduced) gradients, updates fp32 master weights + state and emits the bf16
copy.  Hyper-parameters live in a device array so that LR warm-up / plateau schedules (callbacks) never force a
CUDA-graph re-capture.  A pure-PyTorch path with identical math serves CPU runs (BASELINE.json config 1).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

# hyper array layout shared with csrc/ops_api.h
LR, MOM, BETA2, EPS, WD, GSCALE, BC1, BC2 = range(8)


class FlatOptimizer:
    name = "base"

    def __init__(self, learning_rate: float = 1e-3, weight_decay: float = 0.0):
        self.learning_rate = float(learning_rate)
        self.weight_decay = float(weight_decay)
        self.grad_scale = 1.0
        self.params: Optional[torch.Tensor] = None
        self.grads: Optional[torch.Tensor] = None
        self.w16: Optional[torch.Tensor] = None
        self.state: Dict[str, torch.Tensor] = {}
        self.t = 0
        self._hyper: Optional[torch.Tensor] = None
        self._hyper_host: Optional[torch.Tensor] = None
        self._ext = None

    # -- keras-style accessors used by the callbacks (ReduceLROnPlateau, LearningRateWarmup)
    @property
    def lr(self) -> float:
        return self.learning_rate

    @lr.setter
    def lr(self, v: float) -> None:
        self.learning_rate = float(v)

    def attach(self, params: torch.Tensor, grads: torch.Tensor, w16: Optional[torch.Tensor] = None) -> "FlatOptimizer":
        assert params.dtype == torch.float32 and grads.dtype == torch.float32 and params.numel() == grads.numel()
        assert params.numel() % 4 == 0, "flat buffers must be padded to a multiple of 4 elements"
        self.params, self.grads, self.w16 = params, grads, w16
        for k in self._state_names():
            self.state[k] = torch.zeros_like(params)
        self._hyper = torch.zeros(8, device=params.device, dtype=torch.float32)
        if params.is_cuda:
            from .. import ops

            from ..utils.pinned import PinnedUpload

            self._ext = ops.ext("_b200_ops")
            # ring of pinned staging rows: the host runs several steps ahead of the device (depth >> steps in flight)
            self._hyper_upload = PinnedUpload(self._hyper)
            self._hyper_host = self._hyper_upload.ring[0]
        else:
            self._hyper_host = torch.zeros(8, dtype=torch.float32)
        self.push_hyper()
        return self

    def rebind_grads(self, grads: torch.Tensor) -> None:
        self.grads = grads

    def _state_names(self):
        return ()

    def _fill_hyper(self, h: torch.Tensor) -> None:
        h[LR] = self.learning_rate
        h[WD] = self.weight_decay
        h[GSCALE] = self.grad_scale
        h[BC1] = 1.0
        h[BC2] = 1.0

    def push_hyper(self) -> None:
        """Host -> device copy of the 8 hyper-parameters (outside any CUDA graph)."""
        upload = getattr(self, "_hyper_upload", None)
        if upload is None:
            self._fill_hyper(self._hyper_host)
            self._hyper.copy_(self._hyper_host, non_blocking=True)
            return
        self._hyper_host = upload.push(self._fill_hyper)

    def begin_step(self) -> None:
        """Advance the step counter and refresh the device hyper-parameters; call before (re)playing a step."""
        self.t += 1
        self.push_hyper()

    def step(self) -> None:
        """Launch the update kernel (capturable in a CUDA graph)."""
        if self.params.is_cuda:
            self._step_cuda()
        else:
            self._step_torch()

    def state_dict(self):
        return {"name": self.name, "t": self.t, "lr": self.learning_rate,
                "state": {k: v.detach().cpu() for k, v in self.state.items()}}

    def load_state_dict(self, sd) -> None:
        self.t = sd["t"]
        self.learning_rate = sd["lr"]
        for k, v in sd["state"].items():
            self.state[k].copy_(v)
        self.push_hyper()


class SGD(FlatOptimizer):
    name = "SGD"

    def __init__(self, learning_rate: float = 0.01, momentum: float = 0.0, nesterov: bool = False,
                 weight_decay: float = 0.0):
        super().__init__(learning_rate, weight_decay)
        self.momentum = float(momentum)
        self.nesterov = bool(nesterov)

    def _state_names(self):
        return ("momentum",)

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[MOM] = self.momentum

    def _step_cuda(self):
        self._ext.sgd_step(self.params, self.grads, self.state["momentum"], self.w16, self._hyper, self.nesterov)

    def _step_torch(self):
        h = self._hyper
        d = self.grads * h[GSCALE] + h[WD] * self.params
        m = self.state["momentum"]
        m.mul_(h[MOM]).add_(d)
        upd = d + h[MOM] * m if self.nesterov else m
        self.params.add_(upd * (-h[LR]))
        if self.w16 is not None:
            self.w16.copy_(self.params)


class Adam(FlatOptimizer):
    name = "Adam"

    def __init__(self, learning_rate: float = 1e-3, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7,
                 weight_decay: float = 0.0):
        super().__init__(learning_rate, weight_decay)
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)

    def _state_names(self):
        return ("m", "v")

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[MOM] = self.beta_1
        h[BETA2] = self.beta_2
        h[EPS] = self.epsilon
        t = max(self.t, 1)
        h[BC1] = 1.0 - self.beta_1 ** t
        h[BC2] = 1.0 - self.beta_2 ** t

    def _step_cuda(self):
        self._ext.adam_step(self.params, self.grads, self.state["m"], self.state["v"], self.w16, self._hyper)

    def _step_torch(self):
        h = self._hyper
        d = self.grads * h[GSCALE] + h[WD] * self.params
        m, v = self.state["m"], self.state["v"]
        m.mul_(h[MOM]).add_(d * (1 - h[MOM]))
        v.mul_(h[BETA2]).add_(d * d * (1 - h[BETA2]))
        denom = (v / h[BC2]).sqrt() + h[EPS]
        self.params.add_(-(h[LR] / h[BC1]) * m / denom)
        if self.w16 is not None:
            self.w16.copy_(self.params)


class Adadelta(FlatOptimizer):
    name = "Adadelta"

    def __init__(self, learning_rate: float = 1e-3, rho: float = 0.95, epsilon: float = 1e-7,
                 weight_decay: float = 0.0):
        super().__init__(learning_rate, weight_decay)
        self.rho, self.epsilon = float(rho), float(epsilon)

    def _state_names(self):
        return ("sq", "acc")

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[BETA2] = self.rho
        h[EPS] = self.epsilon

    def _step_cuda(self):
        self._ext.adadelta_step(self.params, self.grads, self.state["sq"], self.state["acc"], self.w16, self._hyper)

    def _step_torch(self):
        h = self._hyper
        d = self.grads * h[GSCALE] + h[WD] * self.params
        sq, acc = self.state["sq"], self.state["acc"]
        sq.mul_(h[BETA2]).add_(d * d * (1 - h[BETA2]))
        delta = (acc + h[EPS]).sqrt() / (sq + h[EPS]).sqrt() * d
        acc.mul_(h[BETA2]).add_(delta * delta * (1 - h[BETA2]))
        self.params.add_(-h[LR] * delta)
        if self.w16 is not None:
            self.w16.copy_(self.params)


OPTIMIZERS = {"SGD": SGD, "Adam": Adam, "Adadelta": Adadelta, "sgd": SGD, "adam": Adam, "adadelta": Adadelta}


def get(name: str):
    """`getattr(tf.keras.optimizers, name)` equivalent (reference P2/01:154)."""
    try:
        return OPTIMIZERS[name]
    except KeyError:
        raise ValueError(f"unknown optimizer {name!r}; available: {sorted(set(OPTIMIZERS))}") from None
