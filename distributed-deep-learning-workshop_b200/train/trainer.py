"""Trainer: the Keras `compile / fit / evaluate / predict` surface of the reference (P1/02:194-215,
P1/03:204-234,325-358, P2/03:206) on top of two execution backends:

* **engine backend** - `models.ResNet50Engine`: hand-scheduled sm_90a kernels, whole step in one CUDA graph,
  gradients born inside the (symmetric) flat buffer that `DistributedOptimizer` all-reduces while backward runs;
* **module backend** - any `torch.nn.Module` (e.g. the reference's frozen MobileNetV2 + Dense head, or CPU runs):
  autograd computes gradients into the same kind of flat buffer (`FlatParams`), so optimizers, callbacks and the
  distributed wrapper are shared.

Datasets are iterables of ``(images uint8 [B,H,W,3], labels int64 [B])`` (see `loader.Converter.make_dataset`), or of
``(images, labels, sample_weight float [B])``.  Keras 3's loss weighting: ``fit(class_weight={class: weight})`` or
per-row sample weights scale each row's loss, and the batch loss is ``(1/B) sum_n w_n l_n`` (``sum_over_batch_size``, not
divided by the sum of the weights); accuracy is not weighted.
"""
from __future__ import annotations

import math
import numbers
import time
from collections import deque
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .callbacks import Callback, CallbackList, History
from .flat import FlatParams
from ..parallel import core as dist_core


def _is_engine(model) -> bool:
    return hasattr(model, "param_specs") and hasattr(model, "forward") and hasattr(model, "bind_grad_buffer")


def _num_classes(model) -> Optional[int]:
    """Classes of a native engine or a torch module (``num_classes``, else its last Linear layer's outputs)."""
    k = getattr(model, "num_classes", None)
    if k is None and isinstance(model, torch.nn.Module):
        lin = [m for m in model.modules() if isinstance(m, torch.nn.Linear)]
        k = lin[-1].out_features if lin else None
    return None if k is None else int(k)


def class_weight_table(class_weight: Dict[int, float], num_classes: Optional[int]) -> torch.Tensor:
    """Keras ``class_weight`` -> float32 [K] table: ``class_weight.get(c, 1.0)`` for every class c.  Keys must be ints in
    [0, K), values finite floats >= 0; anything else raises ValueError."""
    if not isinstance(class_weight, dict):
        raise ValueError(f"class_weight must be a dict {{class index: weight}}, got {type(class_weight).__name__}")
    if num_classes is None:
        raise ValueError("class_weight: the model's number of classes is unknown (no num_classes, no Linear layer)")
    table = torch.ones(num_classes, dtype=torch.float32)
    for c, w in class_weight.items():
        if isinstance(c, bool) or not isinstance(c, numbers.Integral) or not 0 <= int(c) < num_classes:
            raise ValueError(f"class_weight: key {c!r} is not a class index in [0, {num_classes})")
        if isinstance(w, bool) or not isinstance(w, numbers.Real) or not math.isfinite(float(w)) or float(w) < 0:
            raise ValueError(f"class_weight[{c}] = {w!r}: weights must be finite numbers >= 0")
        table[int(c)] = float(w)
    return table


def _unpack(batch, what: str):
    """(x, y, sample_weight or None) of an ``(x, y)`` or ``(x, y, sample_weight)`` batch."""
    if not isinstance(batch, (tuple, list)) or len(batch) not in (2, 3):
        raise ValueError(f"{what}: batches must be (x, y) or (x, y, sample_weight) tuples")
    w = batch[2] if len(batch) == 3 else None
    if w is not None:
        w = torch.as_tensor(w)
        if not w.is_floating_point() or w.dim() != 1 or w.shape[0] != len(batch[1]):
            raise ValueError(f"{what}: sample_weight must be a float tensor [B] with one weight per row, got "
                             f"{w.dtype} {tuple(w.shape)}")
        w = w.float()
    return batch[0], batch[1], w


class _EngineBackend:
    def __init__(self, engine, optimizer, use_graph: bool, label_smoothing: float = 0.0, distillation=None):
        from ..models.resnet_engine import _stats_len

        self.engine = engine
        # read by the head of every forward: set before the (lazily built) steps capture their graphs
        engine.label_smoothing = float(label_smoothing)
        engine.set_distillation(distillation)
        self.optimizer = optimizer
        self.use_graph = use_graph
        # Both step objects are created on first use: a Trainer that only ever predicts (pyfunc serving, load_model) builds
        # the engine for INFERENCE - BatchNorm folded into the convolution epilogues, no gradient / backward buffers - and
        # only a later train_batch() rebuilds it for training.
        self._step = None
        self._eval_step = None
        self.inference_only = False
        self.batch = engine.batch
        self._pending = deque()
        # one pinned result slot per IN-FLIGHT step: a slot goes back to the free list only after its value has been
        # read, so queueing many batches before popping (evaluate) can never overwrite an unread result.  Four floats
        # when distilling: training steps also report the student and distillation terms.
        self._slot = _stats_len(engine)
        self._free = [torch.zeros(self._slot, dtype=torch.float32).pin_memory() for _ in range(4)]
        self._class_weighted = False

    def set_class_weight(self, table: Optional[torch.Tensor]) -> None:
        """Weight the training loss by class (float [K] table; None: no class weights) from the next batch on."""
        self._class_weighted = table is not None
        if table is not None:
            self.engine.set_class_weight(table)   # an async copy: captured graphs read the same table

    def _weighting(self, training: bool, w) -> None:
        """The head's weighting mode for this batch; when it changes, the captured graphs (which launched the other
        head kernel) are dropped and captured again on their next run."""
        mode = "sample" if w is not None else ("class" if training and self._class_weighted else None)
        if self.engine.set_weighting(mode, training):
            for step in (self._step, self._eval_step):
                if step is not None:
                    step.drop_graphs()

    @property
    def step(self):
        if self._step is None:
            from ..models.resnet_engine import EngineTrainStep

            self._step = EngineTrainStep(self.engine, self.optimizer, use_graph=self.use_graph)
            self._eval_step = None  # the engine was (re)built for training: eval plans / graph must be re-captured
        return self._step

    @property
    def eval_step(self):
        if self._eval_step is None:
            from ..models.resnet_engine import EngineEvalStep

            if self._step is None and not self.inference_only:
                _ = self.step  # training-capable trainer: evaluate on the training build (same buffers)
            self._eval_step = EngineEvalStep(self.engine, use_graph=self.use_graph)
        return self._eval_step

    def _enqueue_result(self, n: int = 2) -> None:
        buf = self._free.pop() if self._free else torch.zeros(self._slot, dtype=torch.float32).pin_memory()
        buf[:n].copy_(self.engine.stats[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._pending.append((ev, buf, n))

    def pop_results(self, keep: int = 0) -> List[Tuple[float, ...]]:
        """(loss, accuracy) per step, + (student loss, distillation loss) for a distilling training step."""
        out = []
        while len(self._pending) > keep:
            ev, buf, n = self._pending.popleft()
            ev.synchronize()
            out.append(tuple(float(v) / self.batch for v in buf[:n]))
            self._free.append(buf)
        return out

    def train_batch(self, x, y, w=None) -> None:
        self._weighting(True, w)
        self.step.load(x, y, w)
        self.step.run()
        self._enqueue_result(self._slot)

    def eval_batch(self, x, y, w=None) -> None:
        step = self.eval_step  # (builds the engine on first use)
        self._weighting(False, w)
        self.engine.set_input(x, y, w)
        step.run()
        self._enqueue_result()

    def predict_batch(self, x) -> torch.Tensor:
        step = self.eval_step
        self.engine.set_input(x, None)
        step.run()
        return self.engine.logits.clone()

    def predict_stream(self, arr: torch.Tensor) -> torch.Tensor:
        """Logits [n, classes] (host, fp32) for uint8 images [n, H, W, 3] - the whole array in ONE pipeline:
        batch k+1 is copied host->device on a side stream into one of two staging buffers while the eval graph of batch
        k runs; the logits of every batch go to one pinned result array with async copies; a single sync at the end.
        A pinned `arr` (what the pyfunc scoring workers provide) makes the H2D copies truly asynchronous."""
        e, B = self.engine, self.batch
        step = self.eval_step  # builds the engine (for inference when this trainer never trained) before x_u8 is touched
        n = int(arr.shape[0])
        K = e.num_classes
        out = torch.empty((n, K), dtype=torch.float32).pin_memory() if n else torch.empty((0, K))
        if n == 0:
            return out
        if not hasattr(self, "_stage"):
            self._stage = [torch.empty_like(e.x_u8) for _ in range(2)]
            self._stage_free = [None, None]   # event: the D2D out of the staging buffer has run
            self._copy_stream = torch.cuda.Stream(device=e.device)
        cur = torch.cuda.current_stream()
        self._copy_stream.wait_stream(cur)
        nb = (n + B - 1) // B
        flat = arr.reshape(n, -1)

        def stage(k):
            s = k & 1
            m = min(B, n - k * B)
            with torch.cuda.stream(self._copy_stream):
                if self._stage_free[s] is not None:
                    self._copy_stream.wait_event(self._stage_free[s])
                self._stage[s].view(B, -1)[:m].copy_(flat[k * B:k * B + m], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
            return ev

        ready = stage(0)
        for k in range(nb):
            s = k & 1
            m = min(B, n - k * B)
            nxt = stage(k + 1) if k + 1 < nb else None
            cur.wait_event(ready)
            e.x_u8.copy_(self._stage[s], non_blocking=True)   # D2D, ~15 us
            done = torch.cuda.Event()
            done.record()
            self._stage_free[s] = done
            step.run()
            out[k * B:k * B + m].copy_(e.logits[:m], non_blocking=True)
            ready = nxt
        cur.synchronize()
        return out

    def state_tensors(self) -> List[torch.Tensor]:
        e = self.engine
        if not self.inference_only:
            _ = self.step  # optimizer state exists (and weights may have moved to symmetric memory) only once attached
        opt = self.optimizer.opt if hasattr(self.optimizer, "opt") else self.optimizer
        return [e.params, e.running] + list(opt.state.values())

    def after_state_change(self) -> None:
        self.engine.sync_weights()

    def state_dict(self):
        return self.engine.state_dict()

    def load_state_dict(self, sd) -> None:
        self.engine.load_state_dict(sd)


class _ModuleBackend:
    def __init__(self, module: torch.nn.Module, optimizer, preprocess, device: torch.device,
                 label_smoothing: float = 0.0, distillation=None):
        self.module = module.to(device)
        self.label_smoothing = float(label_smoothing)
        self.distillation = distillation
        if distillation is not None:
            distillation.teacher.to(device)
        self.device = device
        self.optimizer = optimizer
        self.preprocess = preprocess
        self.flat = FlatParams(self.module)
        self._dist = hasattr(optimizer, "on_grads_ready")
        if self._dist:
            grads = optimizer.allocate_grads(self.flat.numel, device)
            self.flat.rebind(grads)
            optimizer.attach(self.flat.params, self.flat.ranges, None, grads)
            self.flat.set_ready_hook(optimizer.on_grads_ready)
        else:
            optimizer.attach(self.flat.params, self.flat.grads, None, segments=self.flat.ranges)
        self._results: deque = deque()
        self.batch = None
        self._class_weight: Optional[torch.Tensor] = None

    def set_class_weight(self, table: Optional[torch.Tensor]) -> None:
        self._class_weight = None if table is None else table.to(self.device)

    def _row_weights(self, y, mix, w):
        """Per-row loss weights (None: unweighted): the batch's sample weights, else the class table at each row's
        target class (the heavier label of a MixUp / CutMix row), as the engines' weighted heads read them."""
        from ..models.augment import target_argmax

        if w is not None:
            return w.to(self.device, non_blocking=True)
        if self._class_weight is not None:
            return self._class_weight[target_argmax(y, mix)]
        return None

    def _prep(self, x) -> torch.Tensor:
        x = torch.as_tensor(x).to(self.device, non_blocking=True)
        return self.preprocess(x)

    def _augmented(self, x):
        """The uint8 NHWC batch warped (and mixed) by ``module.augmentation`` at the optimizer's current step, and the
        mix rows (None without MixUp / CutMix): the reference implementation of the engines' augmentation kernels, same
        draws for the same seed, rank and step."""
        from ..models.augment import augment_batch_reference, augment_key

        x = torch.as_tensor(x)
        if x.dtype != torch.uint8:
            raise ValueError(f"augmentation needs the uint8 [N, H, W, 3] batch, got {x.dtype}")
        opt = self.optimizer.opt if hasattr(self.optimizer, "opt") else self.optimizer
        key = augment_key(getattr(self.module, "augmentation_seed", 0), dist_core.rank())
        return augment_batch_reference(self.module.augmentation, x.to(self.device, non_blocking=True), key, opt.t)

    def train_batch(self, x, y, w=None) -> None:
        from ..models.augment import distillation_reference, soft_targets, target_argmax

        self.module.train()
        y = torch.as_tensor(y).to(self.device, non_blocking=True)
        self.optimizer.begin_step()
        mix = None
        if getattr(self.module, "augmentation", None) is not None:
            x, mix = self._augmented(x)
        self.flat.zero_grad()
        if self._dist:
            self.optimizer.start_backward()
        d = self.distillation
        if d is not None:   # the frozen teacher, in inference mode, on the batch the student sees
            d.teacher.eval()
            with torch.no_grad():
                t_logits = d.teacher(self._prep(x)).float()
        logits = self.module(self._prep(x)).float()
        eps = self.label_smoothing
        rw = self._row_weights(y, mix, w)
        if d is not None:
            rows = distillation_reference(logits, t_logits, y, mix, eps, d.alpha, d.temperature)
            loss, ce, kd = (r.mean() if rw is None else (r * rw).mean() for r in rows)
            acc = (logits.argmax(1) == target_argmax(y, mix)).float().mean()
            loss.backward()
            self.optimizer.step()
            self._results.append(torch.stack([loss.detach(), acc, ce.detach(), kd.detach()]))
            return
        target = y if mix is None and eps == 0 else soft_targets(y, logits.shape[1], mix, eps)
        if rw is not None:   # (1/B) sum_n w_n l_n
            loss = (torch.nn.functional.cross_entropy(logits, target, reduction="none") * rw).mean()
        else:
            loss = torch.nn.functional.cross_entropy(logits, target)
        if mix is None and eps == 0:
            acc = (logits.argmax(1) == y).float().mean()
        else:
            acc = (logits.argmax(1) == target_argmax(y, mix)).float().mean()
        loss.backward()
        self.optimizer.step()
        self._results.append(torch.stack([loss.detach(), acc.detach()]))

    @torch.no_grad()
    def eval_batch(self, x, y, w=None) -> None:
        self.module.eval()
        y = torch.as_tensor(y).to(self.device, non_blocking=True)
        logits = self.module(self._prep(x)).float()
        if w is not None:   # evaluation weights only the batch's own sample weights, never class_weight
            loss = (torch.nn.functional.cross_entropy(logits, y, label_smoothing=self.label_smoothing,
                                                      reduction="none") * w.to(self.device)).mean()
        else:
            loss = torch.nn.functional.cross_entropy(logits, y, label_smoothing=self.label_smoothing)
        acc = (logits.argmax(1) == y).float().mean()
        self._results.append(torch.stack([loss, acc]))

    @torch.no_grad()
    def predict_batch(self, x) -> torch.Tensor:
        self.module.eval()
        return self.module(self._prep(x)).float()

    def pop_results(self, keep: int = 0) -> List[Tuple[float, ...]]:
        """(loss, accuracy) per step, + (student loss, distillation loss) for a distilling training step."""
        out = []
        while len(self._results) > keep:
            out.append(tuple(self._results.popleft().tolist()))
        return out

    def state_tensors(self) -> List[torch.Tensor]:
        opt = self.optimizer.opt if hasattr(self.optimizer, "opt") else self.optimizer
        bufs = [b for b in self.module.buffers() if b.dtype.is_floating_point]
        return [self.flat.params] + bufs + list(opt.state.values())

    def after_state_change(self) -> None:
        pass

    def state_dict(self):
        return {k: v.detach().cpu().clone() for k, v in self.module.state_dict().items()}

    def load_state_dict(self, sd) -> None:
        own = self.module.state_dict()
        for k, v in sd.items():
            own[k].copy_(v)


class Trainer:
    def __init__(self, model, preprocess=None, device: Optional[torch.device] = None, use_graph: bool = True):
        self.model = model
        self.device = torch.device(device) if device is not None else (
            getattr(model, "device", None) or dist_core.device())
        if preprocess is None:
            from ..models.preprocess import preprocess_tensor

            preprocess = preprocess_tensor
        self._preprocess = preprocess
        self.use_graph = use_graph
        self.optimizer = None
        self.backend = None
        self.distillation = None   # the compiled `losses.Distillation`, if any
        self.class_weight: Optional[Dict[int, float]] = None   # of the last fit()
        self.metrics_names = ["loss"]
        self.stop_training = False
        self.steps_per_epoch: Optional[int] = None
        self.history: Optional[History] = None
        self.extra_callbacks: List[Callback] = []  # e.g. tracking.autolog()

    # ------------------------------------------------------------------------------------------------ compile
    def compile(self, optimizer, loss: str = "sparse_categorical_crossentropy", metrics: Sequence[str] = ("accuracy",),
                **_ignored) -> "Trainer":
        """`model.compile(optimizer=..., loss=SparseCategoricalCrossentropy(from_logits=True), metrics=['accuracy'])`;
        ``optimizer`` may be a name (``"rmsprop"``, ``"adamw"``, ...): `optim.get(name)()` with Keras's defaults.
        ``loss`` may also be `losses.CategoricalCrossentropy(from_logits=True, label_smoothing=eps)` or
        ``"categorical_crossentropy"``, which a model whose augmentation uses MixUp or CutMix requires."""
        if isinstance(optimizer, str):
            from .. import optim

            optimizer = optim.get(optimizer)()
        from .losses import CategoricalCrossentropy, Distillation, label_smoothing_of

        eps = label_smoothing_of(loss)
        aug = getattr(self.model, "augmentation", None)
        if aug is not None and aug.mix_mode and not (isinstance(loss, (CategoricalCrossentropy, Distillation))
                                                     or loss == "categorical_crossentropy"):
            raise ValueError("MixUp / CutMix train on soft targets: compile with "
                             "CategoricalCrossentropy(from_logits=True) or 'categorical_crossentropy'")
        distill = loss if isinstance(loss, Distillation) else None
        if distill is not None:
            distill.check_student(self.model)
        self.optimizer = optimizer
        self.metrics_names = ["loss"] + [m if isinstance(m, str) else getattr(m, "name", "metric") for m in metrics]
        if _is_engine(self.model):
            self.backend = _EngineBackend(self.model, optimizer, self.use_graph, eps, distill)
        else:
            self.backend = _ModuleBackend(self.model, optimizer, self._preprocess, self.device, eps, distill)
        self.distillation = distill
        return self

    # ------------------------------------------------------------------------------------------------ fit
    def fit(self, x: Iterable, steps_per_epoch: Optional[int] = None, epochs: int = 1, verbose: int = 1,
            validation_data: Optional[Iterable] = None, validation_steps: Optional[int] = None,
            callbacks: Optional[List[Callback]] = None, initial_epoch: int = 0,
            class_weight: Optional[Dict[int, float]] = None, sample_weight=None, **_ignored) -> History:
        """``class_weight`` ({class index: weight}, Keras 3): each training row's loss is weighted by its class's weight
        (1.0 for a class not in the dict); for a MixUp / CutMix row the class is the heavier label of its mixed target.
        Sample weights come with the batches, ``(x, y, sample_weight)``; the two cannot be combined."""
        if self.backend is None:
            raise RuntimeError("call compile() before fit()")
        if sample_weight is not None:
            raise ValueError("fit(sample_weight=...) is not supported when x is a dataset: yield (x, y, sample_weight) "
                             "batches instead")
        table = None if class_weight is None else class_weight_table(class_weight, _num_classes(self.model))
        self.class_weight = class_weight
        self.backend.set_class_weight(table)
        if steps_per_epoch is None:
            steps_per_epoch = len(x)  # finite datasets only
        self.steps_per_epoch = steps_per_epoch
        self.history = History()
        cbs = CallbackList([*(callbacks or []), *self.extra_callbacks, self.history], self)
        self.stop_training = False
        is_chief = dist_core.rank() == 0
        it = iter(x)
        steps_run = 0
        cbs.call("on_train_begin", {})
        for epoch in range(initial_epoch, epochs):
            cbs.call("on_epoch_begin", epoch, {})
            t0 = time.perf_counter()
            tot = [0.0] * 4   # loss, accuracy, student loss, distillation loss
            n_seen = 0
            for b in range(steps_per_epoch):
                cbs.call("on_train_batch_begin", b, {})
                try:
                    batch = next(it)
                except StopIteration:
                    it = iter(x)
                    try:
                        batch = next(it)
                    except StopIteration:
                        raise ValueError("fit(): the dataset yields no batches (fewer rows than batch_size?)") from None
                xb, yb, wb = _unpack(batch, "fit()")
                if wb is not None and table is not None:
                    raise ValueError("fit(): cannot use class_weight and sample_weight at the same time: the dataset "
                                     "yields (x, y, sample_weight) batches")
                self.backend.train_batch(xb, yb, wb)
                steps_run += 1
                for r in self.backend.pop_results(keep=1):  # lag one step: keeps H2D/compute overlapped
                    for i, v in enumerate(r):
                        tot[i] += v
                    n_seen += 1
                cbs.call("on_train_batch_end", b, {})
            for r in self.backend.pop_results(keep=0):
                for i, v in enumerate(r):
                    tot[i] += v
                n_seen += 1
            dt = time.perf_counter() - t0
            logs: Dict[str, float] = {"loss": tot[0] / max(n_seen, 1)}
            if "accuracy" in self.metrics_names:
                logs["accuracy"] = tot[1] / max(n_seen, 1)
            if self.distillation is not None:   # the two terms of the Keras example's Distiller
                logs["student_loss"] = tot[2] / max(n_seen, 1)
                logs["distillation_loss"] = tot[3] / max(n_seen, 1)
            bsz = self._batch_size(xb)
            logs["images_per_sec"] = steps_per_epoch * bsz * dist_core.size() / max(dt, 1e-9)
            if validation_data is not None:
                vl = self.evaluate(validation_data, steps=validation_steps, verbose=0)
                logs["val_loss"] = vl[0]
                if len(vl) > 1:
                    logs["val_accuracy"] = vl[1]
            cbs.call("on_epoch_end", epoch, logs)
            if verbose and is_chief:
                msg = " - ".join(f"{k}: {v:.4f}" for k, v in logs.items() if k != "images_per_sec")
                print(f"Epoch {epoch + 1}/{epochs} - {dt:.1f}s - {msg} - {logs['images_per_sec']:.0f} img/s", flush=True)
            if self.stop_training:
                break
        opt = self._flat_optimizer()
        if getattr(opt, "use_ema", False) and steps_run > 0:
            # as Keras's fit: the weights become their moving average before on_train_end, so callbacks that save or
            # log the model there (autolog, checkpoints) see the weights the trainer keeps
            opt.finalize_variable_values()
            self.backend.after_state_change()
        cbs.call("on_train_end", {})
        step = getattr(self.backend, "step", None)
        if step is not None and getattr(step, "timeline", None) is not None:
            path = step.dump_timeline()
            if is_chief:
                print(f"timeline written to {path}")
        return self.history

    @staticmethod
    def _batch_size(xb) -> int:
        return int(xb.shape[0]) if hasattr(xb, "shape") and len(xb.shape) == 4 else int(len(xb))

    # ------------------------------------------------------------------------------------------------ evaluate
    def evaluate(self, x: Iterable, steps: Optional[int] = None, verbose: int = 0, **_ignored) -> List[float]:
        if self.backend is None:
            raise RuntimeError("call compile() before evaluate()")
        tot_loss = tot_acc = 0.0
        n = 0
        it = iter(x)
        k = 0
        while steps is None or k < steps:
            try:
                batch = next(it)
            except StopIteration:
                if steps is None:
                    break
                it = iter(x)
                try:
                    batch = next(it)
                except StopIteration:
                    break  # empty dataset
            self.backend.eval_batch(*_unpack(batch, "evaluate()"))
            k += 1
            for l, a in self.backend.pop_results(keep=2):  # bounded queue; lag keeps H2D / compute overlapped
                tot_loss += l
                tot_acc += a
                n += 1
        for l, a in self.backend.pop_results(keep=0):
            tot_loss += l
            tot_acc += a
            n += 1
        out = [tot_loss / max(n, 1)]
        if "accuracy" in self.metrics_names:
            out.append(tot_acc / max(n, 1))
        if verbose and dist_core.rank() == 0:
            print(" - ".join(f"{m}: {v:.4f}" for m, v in zip(self.metrics_names, out)))
        return out

    # ------------------------------------------------------------------------------------------------ predict
    def predict(self, x, batch_size: int = 32, **_ignored) -> np.ndarray:
        """`model.predict(np.array, batch_size)` -> logits [n, classes] (reference P2/03:206)."""
        if self.backend is None:
            self._compile_for_inference()
        arr = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
        n = arr.shape[0]
        if (hasattr(self.backend, "predict_stream") and arr.dtype == torch.uint8 and arr.dim() == 4
                and tuple(arr.shape[1:]) == (self.backend.engine.image_size, self.backend.engine.image_size, 3)):
            return self.backend.predict_stream(arr).numpy()
        fixed = getattr(self.backend, "batch", None)
        bs = fixed or batch_size
        outs = []
        for i in range(0, n, bs):
            chunk = arr[i:i + bs]
            m = chunk.shape[0]
            if fixed and m < bs:  # static-shape engine: pad the tail batch
                pad = torch.zeros((bs - m, *chunk.shape[1:]), dtype=chunk.dtype)
                chunk = torch.cat([chunk, pad.to(chunk.device)], 0)
            outs.append(self.backend.predict_batch(chunk)[:m].cpu())
        return torch.cat(outs, 0).numpy() if outs else np.zeros((0, 0), np.float32)

    def _compile_for_inference(self) -> None:
        from .. import optim

        # an inference compile never trains, so a mixing augmentation's need for soft targets does not apply; without
        # smoothing the categorical loss evaluates exactly as the sparse one
        self.compile(optim.SGD(0.0), loss="categorical_crossentropy")
        if hasattr(self.backend, "inference_only"):
            self.backend.inference_only = True  # engine backend: build with the fused inference epilogues

    # ------------------------------------------------------------------------------------------------ state
    def broadcast_state(self, root: int = 0) -> None:
        """K2: identical weights / optimizer state / BN statistics on every rank - and a distillation teacher's weights
        and statistics (in Keras the teacher is a sub-model of the ``Distiller``, which the broadcast covers)."""
        for t in self.backend.state_tensors():
            dist_core.broadcast(t, root)
        self.backend.after_state_change()
        if self.distillation is not None:
            teacher = self.distillation.teacher
            if _is_engine(teacher):
                # through the state dict: a frozen MobileNetV2 base keeps its weights outside the flat parameters
                sd = {k: v.to(teacher.device) for k, v in teacher.state_dict().items()}
                for v in sd.values():
                    dist_core.broadcast(v, root)
                teacher.load_state_dict(sd)
            else:
                for v in teacher.state_dict().values():   # parameters and buffers, in place
                    dist_core.broadcast(v, root)

    def get_weights(self):
        return self.backend.state_dict()

    def set_weights(self, sd) -> None:
        self.backend.load_state_dict(sd)

    def save_weights(self, path: str) -> None:
        torch.save(self.backend.state_dict(), path)

    def load_weights(self, path: str) -> None:
        self.backend.load_state_dict(torch.load(path, map_location="cpu"))
        self._seed_ema()

    def _flat_optimizer(self):
        return self.optimizer.opt if hasattr(self.optimizer, "opt") else self.optimizer

    def _seed_ema(self) -> None:
        """Loaded weights without a moving average (``use_ema``) start a new one from themselves."""
        opt = self._flat_optimizer()
        if opt is not None and hasattr(opt, "seed_ema"):
            opt.seed_ema()

    def save(self, path: str) -> None:
        """Weights + optimizer state + step counter.  With `DistributedOptimizer(fused_update=True)` the momentum is sharded
        over ranks: call `optimizer.consolidate_state()` on EVERY rank first (it is a collective; `save` usually runs on
        rank 0 only and therefore cannot do it itself) - an unconsolidated state is refused, not silently truncated."""
        if getattr(self.optimizer, "state_is_sharded", False):
            raise RuntimeError("the optimizer state is sharded over ranks (fused_update): call "
                               "optimizer.consolidate_state() on every rank before Trainer.save(), or use save_weights()")
        opt = self._flat_optimizer()
        torch.save({"weights": self.backend.state_dict(), "optimizer": opt.state_dict() if opt is not None else None,
                    "arch": getattr(self.model, "arch", type(self.model).__name__)}, path)

    def load(self, path: str, load_optimizer: bool = True) -> "Trainer":
        """Restore what `save()` (or `save_weights()` / `ModelCheckpoint`) wrote: weights and, when present and wanted,
        the optimizer state and step counter.  Resume recipe (SURVEY.md 5.4; the reference only alludes to it at
        P1/03:305-307): `compile(...)`, `load(path)` on every rank or on rank 0 followed by
        `BroadcastGlobalVariablesCallback(0)` / `broadcast_state(0)`, then `fit(..., initial_epoch=k)`."""
        if self.backend is None:
            raise RuntimeError("call compile() before load()")
        ck = torch.load(path, map_location="cpu")
        weights = ck["weights"] if isinstance(ck, dict) and "weights" in ck else ck
        self.backend.load_state_dict(weights)
        self._seed_ema()   # replaced below when the checkpoint's optimizer state carries the average
        if load_optimizer and isinstance(ck, dict) and ck.get("optimizer") is not None and self.optimizer is not None:
            opt = self._flat_optimizer()
            if ck["optimizer"].get("name") != getattr(opt, "name", None):
                raise ValueError(f"checkpoint holds {ck['optimizer'].get('name')} state, the trainer was compiled with "
                                 f"{getattr(opt, 'name', type(opt).__name__)}")
            opt.load_state_dict(ck["optimizer"])
        return self

    def summary(self) -> str:
        if _is_engine(self.model):
            n = self.model.num_parameters()
            tr = self.model.trainable_parameters() if hasattr(self.model, "trainable_parameters") else n
            lines = [f"Model: {self.model.arch} (H100 engine)", f"Total params: {n:,}", f"Trainable params: {tr:,}"]
            if tr != n:
                lines.append(f"Non-trainable params: {n - tr:,}")
        else:
            tot = sum(p.numel() for p in self.model.parameters())
            tr = sum(p.numel() for p in self.model.parameters() if p.requires_grad)
            lines = [f"Model: {type(self.model).__name__}", f"Total params: {tot:,}", f"Trainable params: {tr:,}",
                     f"Non-trainable params: {tot - tr:,}"]
        s = "\n".join(lines)
        print(s)
        return s
