"""Fused flat-buffer optimizers.

A model exposes ONE flat fp32 parameter buffer, ONE flat fp32 gradient buffer and (optionally) ONE flat bf16
working copy (`ResNet50Engine`, or `FlatParams` for any `torch.nn.Module`).  `step()` is a single kernel launch
(csrc/optim.cu) that reads the (all-reduced) gradients, updates fp32 master weights + state and emits the bf16
copy.  Hyper-parameters live in a device array so that LR warm-up / plateau schedules (callbacks) never force a
CUDA-graph re-capture.  A pure-PyTorch path with identical math serves CPU runs (BASELINE.json config 1).

Every optimizer takes Keras's ``clipnorm`` / ``clipvalue`` / ``global_clipnorm``.  Norms are per parameter tensor
(a "segment" of the flat buffer: the ``segments`` given to `attach`) and are reduced on the device in a fixed order,
with no atomics and no host sync, so a clipped step is bit-reproducible and stays inside the step's CUDA graph.
`Lamb` uses the same segmented reduction for its per-tensor trust ratio.

Every optimizer also takes Keras's ``gradient_accumulation_steps`` (n) and ``use_ema`` / ``ema_momentum`` /
``ema_overwrite_frequency``.  ``t`` counts training steps (micro-batches, Keras's ``iterations``); step t applies an
update when t % n == 0, and otherwise only adds the gradient to the ``accum`` state buffer.  An update step uses
(accum + g) / n, then clips, updates and averages the weights into the ``ema`` state buffer.  Bias corrections count
applied updates, u = t // n, as torch's ``step()`` does (Keras counts micro-steps there).  The EMA advances once per
update and ``ema_overwrite_frequency`` counts updates (Keras: micro-steps); at n = 1 both equal Keras.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

# hyper array layout shared with csrc/ops_api.h: slots 0-7 are read by the update kernels, 8-9 by the clip passes,
# 10-12 by the EMA pass (decay d, 1 - d, overwrite flag: nonzero makes the pass write p = ema and the bf16 copy)
LR, MOM, BETA2, EPS, WD, GSCALE, BC1, BC2 = range(8)
CLIP, HOST_GSCALE = 8, 9
EMA_DECAY, EMA_REST, EMA_OVERWRITE = 10, 11, 12
HYPER_SLOTS = 16
CHUNK = 8192   # floats per chunk of the segmented reductions (csrc/ops_api.h kChunkMax)
CLIP_MODES = ("clipnorm", "clipvalue", "global_clipnorm")
FIN_SUMS, FIN_GLOBAL, FIN_NORM, FIN_LAMB = range(4)   # segment_finalize modes


def normalize_segments(segments: Optional[Sequence[Tuple[int, int]]], n: int) -> List[Tuple[int, int]]:
    """The [lo, hi) tensor ranges sorted, checked (disjoint, inside [0, n], multiples of 4) and completed with the gaps
    between them, so that every element of the flat buffer belongs to exactly one segment.  None: one segment."""
    if not segments:
        return [(0, n)]
    out: List[Tuple[int, int]] = []
    pos = 0
    for lo, hi in sorted((int(a), int(b)) for a, b in segments):
        if lo < pos or hi < lo or hi > n:
            raise ValueError(f"segments must be disjoint [lo, hi) ranges inside [0, {n}]; got ({lo}, {hi})")
        if lo % 4 or hi % 4:
            raise ValueError(f"segment ({lo}, {hi}) is not float4-aligned")
        if lo > pos:
            out.append((pos, lo))
        if hi > lo:
            out.append((lo, hi))
        pos = hi
    if pos < n:
        out.append((pos, n))
    return out


def chunk_tables(segments: Sequence[Tuple[int, int]]) -> Tuple[torch.Tensor, torch.Tensor]:
    """(chunks int64 [nchunks, 3] = (lo, hi, segment), segs int64 [nseg, 2] = (first chunk, end chunk)): each segment is
    cut into chunks of at most CHUNK floats, and no chunk spans two segments."""
    rows, segs = [], []
    for s, (lo, hi) in enumerate(segments):
        first = len(rows)
        rows.extend((a, min(a + CHUNK, hi), s) for a in range(lo, hi, CHUNK))
        segs.append((first, len(rows)))
    return (torch.tensor(rows, dtype=torch.int64).view(-1, 3), torch.tensor(segs, dtype=torch.int64).view(-1, 2))


class FlatOptimizer:
    name = "base"
    # weight decay scales p inside the update instead of adding wd * p to the gradient (AdamW, Lamb)
    _decoupled_decay = False

    def __init__(self, learning_rate: float = 1e-3, weight_decay: float = 0.0, clipnorm: Optional[float] = None,
                 clipvalue: Optional[float] = None, global_clipnorm: Optional[float] = None,
                 gradient_accumulation_steps: Optional[int] = None, use_ema: bool = False, ema_momentum: float = 0.99,
                 ema_overwrite_frequency: Optional[int] = None):
        self.gradient_accumulation_steps = self._check_count("gradient_accumulation_steps",
                                                             gradient_accumulation_steps, 2)
        self.use_ema = bool(use_ema)
        self.ema_momentum = ema_momentum
        self.ema_overwrite_frequency = ema_overwrite_frequency
        if self.use_ema:   # as Keras: the EMA arguments are only checked (and read) with use_ema
            self.ema_momentum = float(ema_momentum)
            if not 0.0 <= self.ema_momentum <= 1.0:
                raise ValueError(f"ema_momentum must be in [0, 1], got {ema_momentum}")
            self.ema_overwrite_frequency = self._check_count("ema_overwrite_frequency", ema_overwrite_frequency, 1)
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
        self.segments: List[Tuple[int, int]] = []
        # chunk tables, partial sums and per-segment factors: scratch, kept out of `state` (which is broadcast,
        # snapshotted by graph capture and checkpointed)
        self._scratch: Dict[str, torch.Tensor] = {}
        clip = {"clipnorm": clipnorm, "clipvalue": clipvalue, "global_clipnorm": global_clipnorm}
        given = [k for k, v in clip.items() if v is not None]
        if len(given) > 1:
            raise ValueError(f"at most one of clipnorm, clipvalue and global_clipnorm may be set, got {given}")
        self._clip = {k: self._check_clip(k, v) for k, v in clip.items()}

    # -- keras-style accessors used by the callbacks (ReduceLROnPlateau, LearningRateWarmup)
    @property
    def lr(self) -> float:
        return self.learning_rate

    @lr.setter
    def lr(self, v: float) -> None:
        self.learning_rate = float(v)

    # -- gradient clipping (Keras semantics, on the gradient the optimizer sees: grad_scale * g, before weight decay)
    @staticmethod
    def _check_clip(name: str, v: Optional[float]) -> Optional[float]:
        if v is None:
            return None
        v = float(v)
        if not v > 0:
            raise ValueError(f"{name} must be > 0, got {v}")
        return v

    def _set_clip(self, name: str, v: Optional[float]) -> None:
        v = self._check_clip(name, v)
        others = [k for k in CLIP_MODES if k != name and self._clip[k] is not None]
        if v is not None and others:
            raise ValueError(f"at most one of clipnorm, clipvalue and global_clipnorm may be set ({others[0]} is)")
        if self.params is not None and (v is None) != (self._clip[name] is None):
            raise ValueError("the clip mode is fixed once the optimizer is attached; only its threshold may change")
        self._clip[name] = v

    clipnorm = property(lambda self: self._clip["clipnorm"], lambda self, v: self._set_clip("clipnorm", v))
    clipvalue = property(lambda self: self._clip["clipvalue"], lambda self, v: self._set_clip("clipvalue", v))
    global_clipnorm = property(lambda self: self._clip["global_clipnorm"],
                               lambda self, v: self._set_clip("global_clipnorm", v))

    @property
    def clip_mode(self) -> Optional[str]:
        """'clipnorm', 'clipvalue', 'global_clipnorm' or None."""
        return next((k for k in CLIP_MODES if self._clip[k] is not None), None)

    # -- gradient accumulation and weight EMA (Keras semantics; see the module docstring for the differences)
    @staticmethod
    def _check_count(name: str, v: Optional[int], least: int) -> Optional[int]:
        if v is None:
            return None
        if isinstance(v, bool) or not isinstance(v, int) or v < least:
            raise ValueError(f"{name} must be an integer >= {least} or None, got {v!r}")
        return v

    @property
    def accumulation_steps(self) -> int:
        """n: micro-batches per applied update (1 without gradient accumulation)."""
        return self.gradient_accumulation_steps or 1

    @property
    def updates(self) -> int:
        """u = t // n: updates applied after step t (torch's ``step()`` count; the bias corrections use it)."""
        return self.t // self.accumulation_steps

    @property
    def is_update_step(self) -> bool:
        """Whether step ``t`` (after `begin_step`) applies an update rather than only accumulating."""
        return self.t % self.accumulation_steps == 0

    def seed_ema(self) -> None:
        """ema = the current parameters (after loading weights that carry no average)."""
        if "ema" in self.state:
            self.state["ema"].copy_(self.params)

    def finalize_variable_values(self) -> None:
        """Keras's end of ``fit`` with ``use_ema``: the parameters (and the bf16 copy) become the moving average."""
        if "ema" not in self.state:
            return
        self.params.copy_(self.state["ema"])
        if self.w16 is not None:
            self.w16.copy_(self.params)

    def attach(self, params: torch.Tensor, grads: torch.Tensor, w16: Optional[torch.Tensor] = None,
               segments: Optional[Sequence[Tuple[int, int]]] = None) -> "FlatOptimizer":
        """Bind the flat buffers.  ``segments``: the [lo, hi) range of every parameter tensor (per-tensor clip norms,
        LAMB trust ratios); None treats the whole buffer as one tensor."""
        assert params.dtype == torch.float32 and grads.dtype == torch.float32 and params.numel() == grads.numel()
        assert params.numel() % 4 == 0, "flat buffers must be padded to a multiple of 4 elements"
        self.params, self.grads, self.w16 = params, grads, w16
        self.segments = normalize_segments(segments, params.numel())
        for k in self._state_names():
            self.state[k] = torch.full_like(params, self._state_init(k))
        if self.gradient_accumulation_steps is not None:
            self.state["accum"] = torch.zeros_like(params)
        if self.use_ema:
            self.state["ema"] = params.clone()
        self._hyper = torch.zeros(HYPER_SLOTS, device=params.device, dtype=torch.float32)
        if params.is_cuda:
            from .. import ops

            from ..utils.pinned import PinnedUpload

            self._ext = ops.ext("_b200_ops")
            # ring of pinned staging rows: the host runs several steps ahead of the device (depth >> steps in flight)
            self._hyper_upload = PinnedUpload(self._hyper)
            self._hyper_host = self._hyper_upload.ring[0]
            self._scratch = {}
            if self._uses_chunks():
                chunks, segs = chunk_tables(self.segments)
                dev = params.device
                self._scratch = {"chunks": chunks.to(dev), "segs": segs.to(dev),
                                 "partial": torch.zeros(2, chunks.shape[0], device=dev),
                                 "sums": torch.zeros(2, segs.shape[0] + 1, device=dev),
                                 "factor": torch.zeros(segs.shape[0], device=dev)}
        else:
            self._hyper_host = torch.zeros(HYPER_SLOTS, dtype=torch.float32)
        self.push_hyper()
        return self

    def rebind_grads(self, grads: torch.Tensor) -> None:
        self.grads = grads

    def _state_names(self):
        """The state buffers, in the order the update rule reads them."""
        return ()

    def _rule(self) -> str:
        """The ``optim_step`` update rule (csrc/optim_rules.cuh): the lower-case name unless the class has variants."""
        return self.name.lower()

    def _state_init(self, name: str) -> float:
        return 0.0

    def _uses_chunks(self) -> bool:
        return self.clip_mode is not None

    def _fill_hyper(self, h: torch.Tensor) -> None:
        mode = self.clip_mode
        h[LR] = self.learning_rate
        h[WD] = self.weight_decay
        # clipnorm / clipvalue rewrite the gradient as clip(grad_scale * g), so the update reads it unscaled
        h[GSCALE] = 1.0 if mode in ("clipnorm", "clipvalue") else self.grad_scale
        h[BC1] = 1.0
        h[BC2] = 1.0
        h[CLIP] = self._clip[mode] if mode is not None else 0.0
        h[HOST_GSCALE] = self.grad_scale
        if self.use_ema:
            # for the update of step t (u = t // n): d = 0 on the first update (Keras seeds the average with it)
            u, f = self.updates, self.ema_overwrite_frequency
            d = self.ema_momentum if u > 1 else 0.0
            h[EMA_DECAY] = d
            h[EMA_REST] = 1.0 - d
            h[EMA_OVERWRITE] = 1.0 if f is not None and u >= 1 and u % f == 0 else 0.0

    def push_hyper(self) -> None:
        """Host -> device copy of the hyper-parameters (outside any CUDA graph)."""
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

    def step(self, update: Optional[bool] = None) -> None:
        """One training step (all launches capturable in a CUDA graph).  An update step combines the accumulated
        gradient with this one, clips it when a clip option is set, updates, then advances the weight EMA; any other
        step only adds the gradient to ``accum``.  ``update``: None decides from ``t`` (`is_update_step`); a captured
        graph fixes it per variant."""
        if update is None:
            update = self.is_update_step
        n = self.accumulation_steps
        if n == 1 and not update:
            raise ValueError("step(update=False) needs gradient_accumulation_steps")
        cuda = self.params.is_cuda
        if n > 1:
            if cuda:
                self._ext.grad_accumulate(self.grads, self.state["accum"], n, 1 if update else 0)
            else:
                self._accumulate_torch(update)
            if not update:
                return
        if cuda:
            self._clip_cuda()
            self._step_cuda()
            if self.use_ema:
                self._ext.ema_update(self.params, self.state["ema"], self.w16, self._hyper)
        else:
            self._clip_torch()
            self._step_torch()
            if self.use_ema:
                self._ema_torch()

    def _accumulate_torch(self, update: bool) -> None:
        g, acc = self.grads, self.state["accum"]
        if update:
            g.add_(acc).div_(self.accumulation_steps)   # acc + g: IEEE addition commutes, so this is the kernel's sum
            acc.zero_()
        else:
            acc.add_(g)

    def _ema_torch(self) -> None:
        h, e = self._hyper, self.state["ema"]
        e.mul_(h[EMA_DECAY]).add_(self.params * h[EMA_REST])
        if bool(h[EMA_OVERWRITE] != 0):
            self.params.copy_(e)
            if self.w16 is not None:
                self.w16.copy_(self.params)

    def _clip_cuda(self) -> None:
        mode = self.clip_mode
        if mode is None:
            return
        e, s = self._ext, self._scratch
        if mode == "clipvalue":
            e.clip_apply(self.grads, s["chunks"], None, self._hyper)
            return
        e.segment_sumsq(self.grads, s["chunks"], s["partial"][0], self._hyper)
        if mode == "global_clipnorm":
            # writes hyper[GSCALE] = hyper[HOST_GSCALE] * c / max(norm, c); the update kernels apply it
            e.segment_finalize(s["partial"][0], s["segs"], s["sums"], s["factor"], self._hyper, FIN_GLOBAL)
        else:
            e.segment_finalize(s["partial"][0], s["segs"], s["sums"], s["factor"], self._hyper, FIN_NORM)
            e.clip_apply(self.grads, s["chunks"], s["factor"], self._hyper)

    def _step_cuda(self) -> None:
        self._ext.optim_step(self._rule(), self.params, self.grads, [self.state[k] for k in self._state_names()],
                             self.w16, self._hyper)

    def _step_torch(self) -> None:
        h = self._hyper
        d = self.grads * h[GSCALE]
        if not self._decoupled_decay:
            d = d + h[WD] * self.params
        self._update_torch(h, d)
        if self.w16 is not None:
            self.w16.copy_(self.params)

    def _clip_torch(self) -> None:
        mode = self.clip_mode
        if mode is None:
            return
        h, g = self._hyper, self.grads
        gs, c = h[HOST_GSCALE], h[CLIP]
        def factor(x):   # c / max(|x|, c), exactly 1 when |x| <= c (as the kernels compute it)
            norm = x.square().sum().sqrt()
            return torch.where(norm > c, c / norm, torch.ones_like(norm))

        if mode == "clipvalue":
            g.mul_(gs).clamp_(-c, c)
        elif mode == "global_clipnorm":
            h[GSCALE] = gs * factor(g * gs)
        else:
            for lo, hi in self.segments:
                x = g[lo:hi].mul_(gs)
                x.mul_(factor(x))

    def state_dict(self):
        return {"name": self.name, "t": self.t, "lr": self.learning_rate,
                "state": {k: v.detach().cpu() for k, v in self.state.items()}}

    def load_state_dict(self, sd) -> None:
        self.t = sd["t"]
        self.learning_rate = sd["lr"]
        for k, v in sd["state"].items():
            if k in ("accum", "ema") and k not in self.state:
                continue   # written with accumulation / EMA, resumed without
            self.state[k].copy_(v)
        if "accum" in self.state and "accum" not in sd["state"]:
            self.state["accum"].zero_()
        if "ema" not in sd["state"]:
            self.seed_ema()
        self.push_hyper()


class SGD(FlatOptimizer):
    name = "SGD"

    def __init__(self, learning_rate: float = 0.01, momentum: float = 0.0, nesterov: bool = False,
                 weight_decay: float = 0.0, **kwargs):
        super().__init__(learning_rate, weight_decay, **kwargs)
        self.momentum = float(momentum)
        self.nesterov = bool(nesterov)

    def _state_names(self):
        return ("momentum",)

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[MOM] = self.momentum

    def _rule(self):
        return "sgd_nesterov" if self.nesterov else "sgd"

    def _update_torch(self, h, d):
        m = self.state["momentum"]
        m.mul_(h[MOM]).add_(d)
        upd = d + h[MOM] * m if self.nesterov else m
        self.params.add_(upd * (-h[LR]))


class Adam(FlatOptimizer):
    name = "Adam"

    def __init__(self, learning_rate: float = 1e-3, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7,
                 weight_decay: float = 0.0, **kwargs):
        super().__init__(learning_rate, weight_decay, **kwargs)
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)

    def _state_names(self):
        return ("m", "v")

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[MOM] = self.beta_1
        h[BETA2] = self.beta_2
        h[EPS] = self.epsilon
        t = max(self.updates, 1)
        h[BC1] = 1.0 - self.beta_1 ** t
        h[BC2] = 1.0 - self.beta_2 ** t

    def _update_torch(self, h, d):
        m, v = self.state["m"], self.state["v"]
        m.mul_(h[MOM]).add_(d * (1 - h[MOM]))
        v.mul_(h[BETA2]).add_(d * d * (1 - h[BETA2]))
        denom = (v / h[BC2]).sqrt() + h[EPS]
        self.params.add_(-(h[LR] / h[BC1]) * m / denom)


class Adadelta(FlatOptimizer):
    name = "Adadelta"

    def __init__(self, learning_rate: float = 1e-3, rho: float = 0.95, epsilon: float = 1e-7,
                 weight_decay: float = 0.0, **kwargs):
        super().__init__(learning_rate, weight_decay, **kwargs)
        self.rho, self.epsilon = float(rho), float(epsilon)

    def _state_names(self):
        return ("sq", "acc")

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[BETA2] = self.rho
        h[EPS] = self.epsilon

    def _update_torch(self, h, d):
        sq, acc = self.state["sq"], self.state["acc"]
        sq.mul_(h[BETA2]).add_(d * d * (1 - h[BETA2]))
        delta = (acc + h[EPS]).sqrt() / (sq + h[EPS]).sqrt() * d
        acc.mul_(h[BETA2]).add_(delta * delta * (1 - h[BETA2]))
        self.params.add_(-h[LR] * delta)


class RMSprop(FlatOptimizer):
    """`torch.optim.RMSprop` update (plain, with momentum, centered) with Keras's argument names and defaults."""
    name = "RMSprop"

    def __init__(self, learning_rate: float = 1e-3, rho: float = 0.9, momentum: float = 0.0, epsilon: float = 1e-7,
                 centered: bool = False, weight_decay: float = 0.0, **kwargs):
        super().__init__(learning_rate, weight_decay, **kwargs)
        self.rho, self.momentum, self.epsilon = float(rho), float(momentum), float(epsilon)
        self.centered = bool(centered)

    def _state_names(self):
        return ("v",) + (("momentum",) if self.momentum > 0 else ()) + (("avg_grad",) if self.centered else ())

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[MOM] = self.momentum
        h[BETA2] = self.rho
        h[EPS] = self.epsilon

    def _rule(self):
        return "rmsprop" + ("_centered" if self.centered else "") + ("_momentum" if self.momentum > 0 else "")

    def _update_torch(self, h, d):
        st = self.state
        v = st["v"]
        v.mul_(h[BETA2]).add_(d * d * (1 - h[BETA2]))
        var = v
        if "avg_grad" in st:
            a = st["avg_grad"]
            a.mul_(h[BETA2]).add_(d * (1 - h[BETA2]))
            var = (v - a * a).clamp_min(0)   # >= 0 in exact arithmetic; rounding must not make the root NaN
        q = d / (var.sqrt() + h[EPS])
        if "momentum" in st:
            q = st["momentum"].mul_(h[MOM]).add_(q)
        self.params.add_(q * (-h[LR]))


class Adagrad(FlatOptimizer):
    """`torch.optim.Adagrad` update (lr_decay 0); the accumulator starts at ``initial_accumulator_value`` (Keras)."""
    name = "Adagrad"

    def __init__(self, learning_rate: float = 1e-3, initial_accumulator_value: float = 0.1, epsilon: float = 1e-7,
                 weight_decay: float = 0.0, **kwargs):
        super().__init__(learning_rate, weight_decay, **kwargs)
        self.initial_accumulator_value, self.epsilon = float(initial_accumulator_value), float(epsilon)

    def _state_names(self):
        return ("acc",)

    def _state_init(self, name):
        return self.initial_accumulator_value

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[EPS] = self.epsilon

    def _update_torch(self, h, d):
        acc = self.state["acc"]
        acc.add_(d * d)
        self.params.add_(-h[LR] * d / (acc.sqrt() + h[EPS]))


class Adamax(FlatOptimizer):
    """`torch.optim.Adamax` update: u = max(beta_2 u, |g| + eps), p -= lr / (1 - beta_1^t) * m / u."""
    name = "Adamax"

    def __init__(self, learning_rate: float = 1e-3, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7,
                 weight_decay: float = 0.0, **kwargs):
        super().__init__(learning_rate, weight_decay, **kwargs)
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)

    def _state_names(self):
        return ("m", "u")

    def _fill_hyper(self, h):
        super()._fill_hyper(h)
        h[MOM] = self.beta_1
        h[BETA2] = self.beta_2
        h[EPS] = self.epsilon
        h[BC1] = 1.0 - self.beta_1 ** max(self.updates, 1)

    def _update_torch(self, h, d):
        m, u = self.state["m"], self.state["u"]
        m.mul_(h[MOM]).add_(d * (1 - h[MOM]))
        torch.maximum(u * h[BETA2], d.abs() + h[EPS], out=u)
        self.params.add_(-(h[LR] / h[BC1]) * m / u)


class AdamW(Adam):
    """`torch.optim.AdamW`: p *= 1 - lr * weight_decay, then this repo's Adam step on the gradient alone."""
    name = "AdamW"
    _decoupled_decay = True

    def __init__(self, learning_rate: float = 1e-3, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7,
                 weight_decay: float = 0.004, **kwargs):
        super().__init__(learning_rate, beta_1, beta_2, epsilon, weight_decay, **kwargs)

    def _update_torch(self, h, d):
        self.params.mul_(1 - h[LR] * h[WD])
        super()._update_torch(h, d)


class Lamb(Adam):
    """LAMB (You et al. 2019), per parameter tensor (segment): r = m_hat / (sqrt(v_hat) + eps) + weight_decay * p,
    phi = ||p|| / ||r|| (1 when either norm is 0), p -= lr * phi * r.  Three launches: moments and per-chunk partial
    norms, per-segment phi, then the update with the bf16 copy."""
    name = "Lamb"
    _decoupled_decay = True

    def _uses_chunks(self) -> bool:
        return True

    def _step_cuda(self):
        e, s = self._ext, self._scratch
        e.lamb_moments(self.params, self.grads, self.state["m"], self.state["v"], s["chunks"], s["partial"],
                       self._hyper)
        e.segment_finalize(s["partial"], s["segs"], s["sums"], s["factor"], self._hyper, FIN_LAMB)
        e.lamb_apply(self.params, self.state["m"], self.state["v"], self.w16, s["chunks"], s["factor"], self._hyper)

    def _update_torch(self, h, d):
        m, v = self.state["m"], self.state["v"]
        m.mul_(h[MOM]).add_(d * (1 - h[MOM]))
        v.mul_(h[BETA2]).add_(d * d * (1 - h[BETA2]))
        r = (m / h[BC1]) / (v.sqrt() / h[BC2].sqrt() + h[EPS]) + h[WD] * self.params
        for lo, hi in self.segments:
            pn, rn = self.params[lo:hi].norm(), r[lo:hi].norm()
            phi = pn / rn if (pn > 0 and rn > 0) else 1.0
            self.params[lo:hi].add_(r[lo:hi] * (-h[LR] * phi))


OPTIMIZERS = {"SGD": SGD, "Adam": Adam, "Adadelta": Adadelta, "sgd": SGD, "adam": Adam, "adadelta": Adadelta,
              "RMSprop": RMSprop, "rmsprop": RMSprop, "Adagrad": Adagrad, "adagrad": Adagrad, "Adamax": Adamax,
              "adamax": Adamax, "AdamW": AdamW, "adamw": AdamW, "Lamb": Lamb, "lamb": Lamb}


def get(name: str):
    """`getattr(tf.keras.optimizers, name)` equivalent (reference P2/01:154)."""
    try:
        return OPTIMIZERS[name]
    except KeyError:
        raise ValueError(f"unknown optimizer {name!r}; available: {sorted(set(OPTIMIZERS))}") from None
