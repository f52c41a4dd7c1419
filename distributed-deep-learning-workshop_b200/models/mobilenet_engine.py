"""The reference's own model on native kernels: frozen MobileNetV2 base + GAP + Dropout + Dense (C14; reference
`build_model`, P1/02:159-178 / P1/03:159-178 - 6,405 trainable parameters, everything else `trainable = False`).

The base is frozen, i.e. it only ever runs in inference mode (Keras: BatchNorm of a non-trainable layer uses its moving
statistics), so every layer is convolution -> folded-BN affine -> ReLU6 [-> + residual] with nothing to keep for backward:

  stem 3x3/2 (3 -> 32) from the uint8 batch      csrc/mobilenet.cu  mbv2_stem      (normalisation x/127.5-1 fused)
  depthwise 3x3 (stride 1 / 2)                    csrc/mobilenet.cu  dwconv3x3
  pointwise 1x1 expand / project / last conv      csrc/conv_igemm.cuh, wgmma implicit GEMM with the kStats = 4 epilogue
                                                  (affine + ReLU6 / linear + residual add of the inverted-residual block)
  GAP + dropout, Dense head fwd / wgrad, CE       the same kernels as the ResNet-50 engine's head

Activations are NHWC bf16 with channel counts padded to multiples of 64 (zero weights / zero shift keep the padding at
zero).  Only `fc.weight` / `fc.bias` live in the flat fp32 parameter / gradient buffers, so the distributed all-reduce of
this model is the ~25 KB message the survey describes (SURVEY.md Q11).  Weights use the state-dict names of
`models.mobilenet.FrozenBaseClassifier`, so checkpoints move freely between the torch module (CPU) and this engine.

`fine_tune_at=k` also trains `base.features[k:]` (conv weights, BatchNorm weight / bias) with every BatchNorm still in
inference mode, so the forward pass is the one above; only the folded scale / shift of the trainable layers now come
from the flat parameters (`refresh_derived_weights`, after every optimizer step).  Backward (csrc/mobilenet_bwd.cu)
runs head -> FC dgrad -> GAP backward -> the trainable layers top-down, per layer: ReLU6 mask / skip add + sum(dz),
weight gradient G, data gradient with the filter scale (.) W (none for the lowest trainable layer); one finalize launch
then turns G into dW = scale * G, dgamma = invstd * (<W_c, G_c> - mean * dbeta), dbeta = sum(dz).  Trainable tensors live
in the flat buffers in backward-completion order (fc, then features.18 down to features.k), each in the layout its
kernel reads: pointwise [cout_p, cin_p] (zero padding, which gets zero gradient), depthwise [9, Cp], stem [27, 32],
gamma / beta [c].  The running statistics stay outside the buffers and never change.

``batchnorm="training"`` (with ``fine_tune_at=k <= 18``) normalises the trainable layers with batch statistics in
training steps (DESIGN.md 3.5b): c = conv(x) is stored (bf16) with its per-channel sums (the kStats = 1 GEMM epilogue, or
the statistics variants of the depthwise / stem kernels), bn_finalize turns them into the batch affine and updates the
running statistics, bn_apply writes y = act(affine(c) [+ residual]).  Backward per layer: dz with sum(dz), sum(dz*c)
(relu6_mask_reduce), bn_bwd_coeffs (dgamma / dbeta straight into the flat gradient buffer), dc = A*dz + B*c + C
(bn_bwd_apply), then the weight and data gradients of dc with the plain filter.  After the optimizer,
refresh_derived_weights folds the running statistics into the inference affine (bn_finalize in inference mode) that
evaluation uses, and rebuilds the plain bf16 dgrad filters.  The running statistics of the trainable layers live in
``running`` (means, then variances); frozen layers and evaluation keep the launches above.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Tuple

import torch

from .. import ops
from ..ops import conv as C
from .resnet_engine import (ParamSpec, _align, _augmenter, _head_weights, _kd_head, _set_row_weight, _stats_len,
                            set_class_weight, set_distillation, set_weighting)

_CFG = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]


def _cp(c: int) -> int:
    return _align(c, 64)


class MobileNetV2Engine:
    """Static-shape frozen-base MobileNetV2 classifier for one GPU (same engine surface as `ResNet50Engine`)."""

    arch = "mobilenetv2"

    def __init__(self, batch: int, num_classes: int = 5, device: Optional[torch.device] = None, image_size: int = 224,
                 dropout: float = 0.5, seed: int = 0, max_ctas: int = 0, bn_eps: float = 1e-5,
                 fine_tune_at: Optional[int] = None, augmentation=None, batchnorm: str = "inference"):
        """``fine_tune_at=k`` (0..19): train ``base.features[k:]`` too, BatchNorm in inference mode (see module doc);
        ``k`` counts feature blocks (0 = stem, 1..17 = inverted-residual blocks, 18 = last 1x1 conv, 19 = head only).
        ``augmentation`` (`models.augment.Augmentation`): random flip / rotation / zoom / translation of the input batch
        in every training step, on the device; evaluation and inference never apply it.
        ``batchnorm="training"``: the BatchNorms of ``base.features[k:]`` use batch statistics in training steps and
        update their running statistics (momentum 0.1, unbiased variance); ``k = 19`` has none, so it is the
        ``fine_tune_at=19`` engine."""
        from .augment import check_augmentation
        from .mobilenet import check_batchnorm, check_fine_tune_at

        ops.require_native()
        self.augmentation = check_augmentation(augmentation)
        self._augmenter = None
        # Keras's label smoothing of the loss; the Trainer sets it from the compiled loss before capturing the steps
        self.label_smoothing = 0.0
        self.distillation = None   # `train.losses.Distillation` with an engine teacher: set by `set_distillation`
        self._teacher_in: Optional[torch.Tensor] = None   # a student's stem input this engine reads as a teacher
        # per-row loss weights of the training / evaluation head (`resnet_engine.set_weighting`) and their buffers
        self.train_weighting = self.eval_weighting = None
        self.class_weight: Optional[torch.Tensor] = None
        self.row_weight: Optional[torch.Tensor] = None
        if image_size % 32:
            raise ValueError("image_size must be a multiple of 32")
        check_fine_tune_at(fine_tune_at)
        check_batchnorm(batchnorm, fine_tune_at)
        self.fine_tune_at = fine_tune_at
        self.batchnorm = batchnorm
        self._k = 19 if fine_tune_at is None else fine_tune_at
        self._bn_train = batchnorm == "training" and self._k <= 18
        self.bn_momentum = 0.1
        self.batch, self.num_classes, self.image_size = int(batch), int(num_classes), int(image_size)
        self.dropout, self.seed, self.max_ctas, self.bn_eps = float(dropout), seed, int(max_ctas), bn_eps
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self._e = ops.ext("_b200_ops")
        self.classes_padded = 64 if self.num_classes <= 64 else _align(self.num_classes, 128)
        self.feat_channels = 1280
        specs = [ParamSpec("fc.weight", (self.classes_padded, self.feat_channels), "fc_w"),
                 ParamSpec("fc.bias", (self.num_classes,), "fc_b")]
        self._layers = self._describe()
        for kind, conv, bn, cin, cout, _, _, _, feat in reversed(self._layers):
            if feat >= self._k:
                wshape = {"stem": (27, 32), "dw": (9, _cp(cin)), "pw": (_cp(cout), _cp(cin))}[kind]
                specs += [ParamSpec(conv + ".weight", wshape, kind + "_w"), ParamSpec(bn + ".weight", (cout,), "bn_w"),
                          ParamSpec(bn + ".bias", (cout,), "bn_b")]
        off = 0
        for s in specs:
            s.numel = int(math.prod(s.shape))
            s.offset = off
            off += _align(s.numel)
        self.param_specs, self.spec, self.flat_numel = specs, {s.name: s for s in specs}, off
        self.params = torch.zeros(off, device=self.device, dtype=torch.float32)
        self.w16 = torch.zeros(off, device=self.device, dtype=torch.bfloat16)
        self.grads: Optional[torch.Tensor] = None
        if self._bn_train:
            # running statistics of the trainable BatchNorms: one flat buffer, means then variances (as ResNet-50)
            bns = [(bn, cout) for _, _, bn, _, cout, _, _, _, feat in self._layers if feat >= self._k]
            tot = sum(c for _, c in bns)
            self.running = torch.zeros(2 * tot, device=self.device)
            self.running_mean: Dict[str, torch.Tensor] = {}
            self.running_var: Dict[str, torch.Tensor] = {}
            o = 0
            for bn, c in bns:
                self.running_mean[bn] = self.running[o:o + c]
                self.running_var[bn] = self.running[tot + o:tot + o + c]
                o += c
            self._tracked: Dict[str, int] = {}   # num_batches_tracked at the last load, + training steps since
            self._tracked_from = 0
        else:
            self.running = torch.zeros(8, device=self.device)  # no trainable BatchNorm statistics (frozen base)
        self.grad_hook: Optional[Callable[[int, int], None]] = None
        self.aux_streams: List[torch.cuda.Stream] = []
        self._step_count = 0
        self._built = False
        self._training_built = False
        # frozen base: random init with torchvision's scheme, from the torch module so both paths share weights
        from .mobilenet import FrozenBaseClassifier, MobileNetV2Base

        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            base = MobileNetV2Base()
            ref = FrozenBaseClassifier(base, base.out_channels, num_classes, dropout, True)
        # frozen inference statistics of the trainable layers (fp32 [cp] on the device; set by load_state_dict)
        self._ft_stats = {bn: (torch.zeros(_cp(cout), device=self.device), torch.zeros(_cp(cout), device=self.device))
                          for _, _, bn, _, cout, _, _, _, feat in self._layers if feat >= self._k}
        self.load_state_dict(ref.state_dict())

    # ------------------------------------------------------------------------------------------------ architecture
    def _describe(self):
        """[(kind, state-dict prefix of conv, prefix of bn, cin, cout, stride, act, residual?, index in base.features)]
        in execution order."""
        L = [("stem", "base.features.0.0", "base.features.0.1", 3, 32, 2, "relu6", False, 0)]
        cin, idx = 32, 1
        for t, c, n, s in _CFG:
            for i in range(n):
                stride = s if i == 0 else 1
                hidden = cin * t
                p = f"base.features.{idx}.conv"
                k = 0
                if t != 1:
                    L.append(("pw", f"{p}.{k}.0", f"{p}.{k}.1", cin, hidden, 1, "relu6", False, idx))
                    k += 1
                L.append(("dw", f"{p}.{k}.0", f"{p}.{k}.1", hidden, hidden, stride, "relu6", False, idx))
                k += 1
                L.append(("pw", f"{p}.{k}", f"{p}.{k + 1}", hidden, c, 1, "none", stride == 1 and cin == c, idx))
                cin = c
                idx += 1
        L.append(("pw", f"base.features.{idx}.0", f"base.features.{idx}.1", cin, 1280, 1, "relu6", False, idx))
        return L

    # ------------------------------------------------------------------------------------------------ parameters
    def p(self, name: str) -> torch.Tensor:
        s = self.spec[name]
        return self.params[s.offset:s.offset + s.numel].view(s.shape)

    def g(self, name: str) -> torch.Tensor:
        s = self.spec[name]
        return self.grads[s.offset:s.offset + s.numel].view(s.shape)

    def w16v(self, name: str) -> torch.Tensor:
        s = self.spec[name]
        return self.w16[s.offset:s.offset + s.numel].view(s.shape)

    def bind_grad_buffer(self, grads: Optional[torch.Tensor] = None) -> None:
        if grads is None:
            grads = torch.zeros(self.flat_numel, device=self.device, dtype=torch.float32)
        assert grads.numel() >= self.flat_numel and grads.dtype == torch.float32
        self.grads = grads

    def sync_weights(self) -> None:
        self._e.cast_bf16(self.params, self.w16)
        if self._built:
            self.refresh_derived_weights()

    def refresh_derived_weights(self) -> None:
        """Trainable layers: folded scale / shift from gamma / beta and the frozen statistics, bf16 dgrad filters
        scale (.) W of the pointwise layers, and the FC dgrad filter.  (The head GEMM reads the flat bf16 copy.)
        With training-mode BatchNorm: the inference affine from the running statistics, and the plain W^T filters."""
        if self._built and self._bn_train:
            self._refresh_bn_train()
        elif self._built and self._ft_stats:
            self._e.mbv2_ft_refresh(self.params, self._ft_refresh_table)
        if getattr(self, "_fc_dg", None) is not None:
            self._e.weight_prep(self.p("fc.weight"), None, self._fc_wd, 1, self.classes_padded, self.feat_channels)

    def num_parameters(self) -> int:
        return sum(v.numel() for k, v in self._base_sd.items() if k.endswith(".weight") or k.endswith(".bias")) + \
            self.num_classes * self.feat_channels + self.num_classes

    def trainable_parameters(self) -> int:
        """Unpadded count: the head plus conv weights and BatchNorm weight / bias of base.features[fine_tune_at:]."""
        n = self.num_classes * self.feat_channels + self.num_classes
        for kind, _, _, cin, cout, _, _, _, feat in self._layers:
            if feat >= self._k:
                n += {"stem": 27 * 32, "dw": 9 * cin, "pw": cout * cin}[kind] + 2 * cout
        return n

    def _trainable_layers(self):
        return [lay for lay in self._layers if lay[8] >= self._k]

    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {k: v.detach().clone().cpu() for k, v in self._base_sd.items()}
        sd["fc.weight"] = self.p("fc.weight")[:self.num_classes].detach().clone().cpu()
        sd["fc.bias"] = self.p("fc.bias").detach().clone().cpu()
        for kind, conv, bn, cin, cout, *_ in self._trainable_layers():
            if self._bn_train:
                sd[bn + ".running_mean"] = self.running_mean[bn].detach().clone().cpu()
                sd[bn + ".running_var"] = self.running_var[bn].detach().clone().cpu()
                sd[bn + ".num_batches_tracked"] = torch.tensor(
                    self._tracked[bn] + self._step_count - self._tracked_from, dtype=torch.int64)
            w = self.p(conv + ".weight").detach().cpu()
            if kind == "stem":   # [27, 32] -> [32, 3, 3, 3]
                sd[conv + ".weight"] = w.view(3, 3, 3, 32).permute(3, 2, 0, 1).contiguous()
            elif kind == "dw":   # [9, Cp] -> [C, 1, 3, 3]
                sd[conv + ".weight"] = w[:, :cin].t().contiguous().view(cin, 1, 3, 3)
            else:                # [cout_p, cin_p] -> [cout, cin, 1, 1]
                sd[conv + ".weight"] = w[:cout, :cin].contiguous().view(cout, cin, 1, 1)
            sd[bn + ".weight"] = self.p(bn + ".weight").detach().clone().cpu()
            sd[bn + ".bias"] = self.p(bn + ".bias").detach().clone().cpu()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        self._base_sd = {k: v.detach().to("cpu", copy=True) for k, v in sd.items() if k.startswith("base.")}
        self.p("fc.weight").zero_()
        self.p("fc.weight")[:self.num_classes].copy_(sd["fc.weight"].to(self.device, torch.float32))
        self.p("fc.bias").copy_(sd["fc.bias"].to(self.device, torch.float32))
        for kind, conv, bn, cin, cout, *_ in self._trainable_layers():
            w, dst = sd[conv + ".weight"].float(), self.p(conv + ".weight")
            dst.zero_()
            if kind == "stem":
                dst.copy_(w.permute(2, 3, 1, 0).reshape(27, 32))
            elif kind == "dw":
                dst[:, :cin].copy_(w.view(cin, 9).t())
            else:
                dst[:cout, :cin].copy_(w.view(cout, cin))
            self.p(bn + ".weight").copy_(sd[bn + ".weight"].float())
            self.p(bn + ".bias").copy_(sd[bn + ".bias"].float())
            inv, mean = self._ft_stats[bn]
            inv[:cout].copy_(torch.rsqrt(sd[bn + ".running_var"].float() + self.bn_eps))   # the host fold of _affine
            mean[:cout].copy_(sd[bn + ".running_mean"].float())
            if self._bn_train:
                self.running_mean[bn].copy_(sd[bn + ".running_mean"].float())
                self.running_var[bn].copy_(sd[bn + ".running_var"].float())
                self._tracked[bn] = int(sd.get(bn + ".num_batches_tracked", torch.tensor(0)))
        if self._bn_train:
            self._tracked_from = self._step_count
        self._e.cast_bf16(self.params, self.w16)
        if self._built:
            self._load_base_weights()
            self.refresh_derived_weights()

    # ------------------------------------------------------------------------------------------------ build
    def _affine(self, bn: str, c: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """Folded inference BatchNorm of `bn`: (scale, shift) fp32 [cp]; padded channels get scale 1 / shift 0."""
        sd, cp = self._base_sd, _cp(c)
        inv = torch.rsqrt(sd[bn + ".running_var"].float() + self.bn_eps)
        sc = sd[bn + ".weight"].float() * inv
        sh = sd[bn + ".bias"].float() - sd[bn + ".running_mean"].float() * sc
        scale, shift = torch.ones(cp), torch.zeros(cp)
        scale[:c], shift[:c] = sc, sh
        return scale.to(self.device), shift.to(self.device)

    def _load_base_weights(self) -> None:
        sd = self._base_sd
        for lay in self._plan:
            if lay["train"]:
                continue   # weights live in the flat parameters; scale / shift come from refresh_derived_weights
            kind, conv, bn, cin, cout = lay["kind"], lay["conv"], lay["bn"], lay["cin"], lay["cout"]
            w = sd[conv + ".weight"].float()
            if kind == "stem":   # [32, 3, 3, 3] (co, c, r, s) -> [27, 32] with k = (r*3 + s)*3 + c
                lay["w"].copy_(w.permute(2, 3, 1, 0).reshape(27, 32))
            elif kind == "dw":   # [C, 1, 3, 3] -> [9, Cp]
                lay["w"].zero_()
                lay["w"][:, :cin].copy_(w.view(cin, 9).t())
            else:                # [cout, cin, 1, 1] -> bf16 [cout_p, cin_p]
                lay["w"].zero_()
                lay["w"][:cout, :cin].copy_(w.view(cout, cin).to(torch.bfloat16))
            sc, sh = self._affine(bn, cout)
            lay["scale"].copy_(sc)
            lay["shift"].copy_(sh)

    def build(self, training: bool = True) -> "MobileNetV2Engine":
        if self._built:
            if training and not self._training_built:
                self._build_head(training=True)
                self.refresh_derived_weights()
            return self
        if self.grads is None and training:
            self.bind_grad_buffer()
        dev, N, S = self.device, self.batch, self.image_size
        bf = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        self.x_u8 = torch.zeros(N, S, S, 3, device=dev, dtype=torch.uint8)
        self.labels = torch.zeros(N, device=dev, dtype=torch.int64)
        self.stats = torch.zeros(_stats_len(self), **f32)
        self.logits = torch.zeros(N, self.num_classes, **f32)
        self.loss_rows = torch.zeros(N, **f32)
        self._plan: List[dict] = []
        h = S
        x = None
        block_in = None
        block_src = None   # index in _plan of the layer that wrote block_in
        for kind, conv, bn, cin, cout, stride, act, residual, feat in self._layers:
            train = feat >= self._k
            lay = dict(kind=kind, conv=conv, bn=bn, cin=cin, cout=cout, stride=stride, act=act, train=train)
            ho = h // stride
            out = torch.zeros(N, ho, ho, _cp(cout), **bf)
            lay["scale"], lay["shift"] = torch.ones(_cp(cout), **f32), torch.zeros(_cp(cout), **f32)
            if kind == "stem":
                lay["w"] = self.p(conv + ".weight") if train else torch.zeros(27, 32, **f32)
                lay["x"], lay["y"] = self.x_u8, out
                block_in, block_src = out, len(self._plan)
            elif kind == "dw":
                lay["w"] = self.p(conv + ".weight") if train else torch.zeros(9, _cp(cin), **f32)
                lay["x"], lay["y"] = x, out
            else:
                # a trainable pointwise layer reads the bf16 copy of the flat parameters that the optimizer writes
                lay["w"] = self.w16v(conv + ".weight") if train else torch.zeros(_cp(cout), _cp(cin), **bf)
                lay["x"], lay["y"] = x, out
                res = block_in if residual else None
                if residual:
                    lay["res_src"] = block_src
                lay["op"] = C.ConvForward(x, lay["w"], out, 1, 1, 1, 0, None, None, self.max_ctas,
                                          epilogue=(lay["scale"], lay["shift"], act, res))
                lay["res"] = res
                if act == "none":
                    # output of an inverted-residual block (linear bottleneck) = the next block's input
                    block_in, block_src = out, len(self._plan)
            if train and self._bn_train:
                self._add_bn_train_buffers(lay, N * ho * ho)
            self._plan.append(lay)
            x, h = out, ho
        self.feat = x   # [N, S/32, S/32, 1280]
        self.pooled = torch.zeros(N, self.feat_channels, **bf)
        self._load_base_weights()
        if self._bn_train:
            cmax = max(lay["cout"] for lay in self._plan if lay["train"])
            self._fold_scratch = torch.zeros(4, cmax, **f32)   # sum, sqsum, mean, invstd bn_finalize also writes
        elif self._ft_stats:
            self._ft_refresh_table = self._table([self._refresh_row(lay) for lay in self._plan if lay["train"]])
        self._built = True
        self._build_head(training)
        self.refresh_derived_weights()
        return self

    # ------------------------------------------------------------------------------------------------ training-mode BN
    def _add_bn_train_buffers(self, lay: dict, count: int) -> None:
        """Conv output c, its statistics sums and the batch affine of a trainable layer (cp-sized, zero padding), and
        for pointwise layers the GEMM writing c with the kStats = 1 statistics epilogue."""
        dev, cp = self.device, _cp(lay["cout"])
        lay["c"] = torch.zeros_like(lay["y"])
        lay["count"] = count
        lay["ssum"], lay["ssq"], lay["bmean"], lay["binv"], lay["bscale"], lay["bshift"] = \
            torch.zeros(6, cp, device=dev).unbind(0)
        if lay["kind"] == "pw":
            lay["op_stats"] = C.ConvForward(lay["x"], lay["w"], lay["c"], 1, 1, 1, 0, lay["ssum"], lay["ssq"],
                                            self.max_ctas)

    def _forward_bn_train(self, lay: dict) -> None:
        """c = conv(x) + statistics, batch affine + running-statistics update, y = act(affine(c) [+ residual])."""
        e, kind, cout, bn = self._e, lay["kind"], lay["cout"], lay["bn"]
        if kind == "stem":
            e.mbv2_stem_stats(self._stem_input(True), lay["w"], lay["c"], lay["ssum"][:32], lay["ssq"][:32],
                              1.0 / 127.5, -1.0)
        elif kind == "dw":
            e.dwconv3x3_stats(lay["x"], lay["w"], lay["c"], lay["ssum"], lay["ssq"], lay["stride"])
        else:
            lay["op_stats"].run()
        e.bn_finalize(lay["ssum"], lay["ssq"], float(lay["count"]), self.p(bn + ".weight"), self.p(bn + ".bias"),
                      self.running_mean[bn], self.running_var[bn], self.bn_momentum, self.bn_eps, lay["bmean"][:cout],
                      lay["binv"][:cout], lay["bscale"][:cout], lay["bshift"][:cout], True)
        act = lay["act"]
        e.bn_apply(lay["c"], lay["bscale"], lay["bshift"], lay["res"] if kind == "pw" else None, None, None, lay["y"],
                   act != "none", None, act == "relu6")

    def _refresh_bn_train(self) -> None:
        """Inference affine of every trainable layer from its running statistics (bn_finalize in inference mode: the
        padding of scale / shift stays 1 / 0), and the bf16 W^T dgrad filters of the pointwise layers."""
        e = self._e
        s_sum, s_sq, s_mean, s_inv = self._fold_scratch.unbind(0)
        for lay in self._plan:
            if lay["train"]:
                bn, c = lay["bn"], lay["cout"]
                e.bn_finalize(s_sum, s_sq, 1.0, self.p(bn + ".weight"), self.p(bn + ".bias"), self.running_mean[bn],
                              self.running_var[bn], self.bn_momentum, self.bn_eps, s_mean, s_inv, lay["scale"][:c],
                              lay["shift"][:c], False)
        if getattr(self, "_wd_tiles", 0):
            e.weight_prep_batched(self.params, self._wd16, self._wd_table, self._wd_tiles)

    def _build_bn_train_backward(self, train: List[int]) -> None:
        """Scratch of the training-mode BatchNorm backward: dc (one buffer, every layer's dc is consumed before the next
        layer down writes it), the cp-sized coefficients A / B / C per layer, and the plain W^T filters of the pointwise
        layers that have a data gradient (one weight_prep_batched table)."""
        dev = self.device
        self._dc = torch.zeros(max(self._plan[i]["y"].numel() for i in train), device=dev, dtype=torch.bfloat16)
        self._ones = torch.ones(max(_cp(self._plan[i]["cout"]) for i in train), device=dev)
        rows, wd_total, tiles = [], 0, 0
        for i in train:
            lay = self._plan[i]
            cp = _cp(lay["cout"])
            lay["dc"] = self._dc[:lay["y"].numel()].view(lay["y"].shape)
            lay["cA"], lay["cB"], lay["cC"] = torch.zeros(3, cp, device=dev).unbind(0)
            if lay["kind"] == "pw" and i > self._ft_lowest:
                cin_p = _cp(lay["cin"])
                rows.append([self.spec[lay["conv"] + ".weight"].offset, wd_total, 1, cp, cin_p, tiles])
                lay["wd_range"] = (wd_total, cp * cin_p)
                wd_total += cp * cin_p
                tiles += (cp // 64) * (cin_p // 32)
        self._wd16 = torch.zeros(max(wd_total, 8), device=dev, dtype=torch.bfloat16)
        for i in train:
            lay = self._plan[i]
            if "wd_range" in lay:
                o, n = lay["wd_range"]
                lay["wd"] = self._wd16[o:o + n].view(_cp(lay["cin"]), _cp(lay["cout"]))
        if rows:
            self._wd_table, self._wd_tiles = self._table(rows), tiles

    def _backward_bn_train(self, i: int) -> torch.Tensor:
        """dz with sum(dz), sum(dz*c); dgamma / dbeta and the coefficients; dc = A*dz + B*c + C.  Returns dc."""
        e, lay = self._e, self._plan[i]
        bn, c = lay["bn"], lay["cout"]
        g = lay["g"]
        e.relu6_mask_reduce(g, lay["g2"], lay["y"], g, lay["sum"], lay["act"] == "relu6", lay["c"], lay["sumc"])
        e.bn_bwd_coeffs(lay["sum"][:c], lay["sumc"][:c], self.p(bn + ".weight"), lay["bmean"][:c], lay["binv"][:c],
                        float(lay["count"]), self.g(bn + ".weight"), self.g(bn + ".bias"), lay["cA"][:c],
                        lay["cB"][:c], lay["cC"][:c])
        e.bn_bwd_apply(g, lay["c"], None, None, lay["cA"], lay["cB"], lay["cC"], lay["dc"])
        return lay["dc"]

    # ------------------------------------------------------------------------------------------------ fine-tuning tables
    def _table(self, rows: List[List[int]]) -> torch.Tensor:
        return torch.tensor(rows, dtype=torch.int64).to(self.device)

    def _refresh_row(self, lay: dict) -> List[int]:
        """mbv2_ft_refresh row: c, cp, cin_p (pointwise dgrad filter) | offsets gamma, beta, W | invstd, mean, scale,
        shift, dgrad filter pointers."""
        cout, bn, sp = lay["cout"], lay["bn"], self.spec
        inv, mean = self._ft_stats[bn]
        if lay["kind"] == "pw":
            lay["wd"] = torch.zeros(_cp(lay["cin"]), _cp(cout), device=self.device, dtype=torch.bfloat16)
        wd = lay.get("wd")
        return [cout, _cp(cout), _cp(lay["cin"]) if wd is not None else 0, sp[bn + ".weight"].offset,
                sp[bn + ".bias"].offset, sp[lay["conv"] + ".weight"].offset, inv.data_ptr(), mean.data_ptr(),
                lay["scale"].data_ptr(), lay["shift"].data_ptr(), wd.data_ptr() if wd is not None else 0]

    def _finalize_row(self, lay: dict) -> List[int]:
        """mbv2_ft_finalize row: c, elements per channel, channel / element strides of W and G, W is bf16 | offsets G
        (= W), dgamma, dbeta | scale, invstd, mean, sum(dz) pointers."""
        kind, cout, bn, sp = lay["kind"], lay["cout"], lay["bn"], self.spec
        count, cstride, jstride = {"stem": (27, 1, 32), "dw": (9, 1, _cp(cout)),
                                   "pw": (_cp(lay["cin"]), _cp(lay["cin"]), 1)}[kind]
        inv, mean = self._ft_stats[bn]
        off = sp[lay["conv"] + ".weight"].offset
        return [cout, count, cstride, jstride, int(kind == "pw"), off, off, sp[bn + ".weight"].offset,
                sp[bn + ".bias"].offset, lay["scale"].data_ptr(), inv.data_ptr(), mean.data_ptr(),
                lay["sum"].data_ptr()]

    def _build_backward(self) -> None:
        """Gradient buffers and plans of the trainable base layers (training build with fine_tune_at <= 18)."""
        N, ncp, mc, F = self.batch, self.classes_padded, self.max_ctas, self.feat_channels
        bf = dict(device=self.device, dtype=torch.bfloat16)
        self.dpooled = torch.zeros(N, F, **bf)
        self._fc_wd = torch.zeros(F, ncp, **bf)
        self._fc_dg = C.ConvDgrad(self.dlogits16.view(N, 1, 1, ncp), self.p("fc.weight").view(1, ncp, F),
                                  self.dpooled.view(N, 1, 1, F), 1, 1, 1, 0, mc, wbuf=self._fc_wd)
        train = [i for i, lay in enumerate(self._plan) if lay["train"]]
        self._ft_lowest = train[0]
        total = sum(_cp(self._plan[i]["cout"]) for i in train)
        self._ft_sums = torch.zeros(total * (2 if self._bn_train else 1), device=self.device)
        off = 0
        for i in train:
            lay = self._plan[i]
            cp = _cp(lay["cout"])
            lay["sum"] = self._ft_sums[off:off + cp]
            if self._bn_train:
                lay["sumc"] = self._ft_sums[total + off:total + off + cp]
            off += cp
            lay["g"] = torch.zeros_like(lay["y"])   # gradient at the output; turned into dz in place
            lay["g2"] = None
        if self._bn_train:
            self._build_bn_train_backward(train)
        for i in train:
            lay = self._plan[i]
            if "res_src" in lay and self._plan[lay["res_src"]]["train"]:
                self._plan[lay["res_src"]]["g2"] = lay["g"]   # skip gradient = dz of the block's linear output
            if lay["kind"] == "pw":
                w = self.p(lay["conv"] + ".weight")
                # the wgrad GEMM takes Cout == 64 or a multiple of 128: 128*a + 64 output channels run as two GEMMs
                G, cp = self.g(lay["conv"] + ".weight"), _cp(lay["cout"])
                cuts = [0, cp] if cp == 64 or cp % 128 == 0 else [0, cp - 64, cp]
                src = lay["dc"] if self._bn_train else lay["g"]   # training-mode BN: the gradient of c
                lay["wg"] = [C.ConvWgrad(src[..., a:b], lay["x"], G[a:b], 1, 1, 1, 0, 0, mc, 0)
                             for a, b in zip(cuts, cuts[1:])]
                if i > self._ft_lowest:
                    lay["dg"] = C.ConvDgrad(src, w.view(1, *w.shape), self._plan[i - 1]["g"], 1, 1, 1, 0, mc,
                                            wbuf=lay["wd"])
        if not self._bn_train:
            self._ft_finalize_table = self._table([self._finalize_row(self._plan[i]) for i in train])

    def _build_head(self, training: bool) -> None:
        N, ncp, mc = self.batch, self.classes_padded, self.max_ctas
        bf = dict(device=self.device, dtype=torch.bfloat16)
        if not hasattr(self, "logits16"):
            self.logits16 = torch.zeros(N, ncp, **bf)
            self._fc_fwd = C.ConvForward(self.pooled.view(N, 1, 1, self.feat_channels), self.w16v("fc.weight"),
                                         self.logits16.view(N, 1, 1, ncp), 1, 1, 1, 0, None, None, mc)
        if training and not self._training_built:
            if self.grads is None:
                self.bind_grad_buffer()
            self.dlogits16 = torch.zeros(N, ncp, **bf)
            self._fc_wg = C.ConvWgrad(self.dlogits16.view(N, 1, 1, ncp), self.pooled.view(N, 1, 1, self.feat_channels),
                                      self.g("fc.weight"), 1, 1, 1, 0, 0, mc, 0)
            if self._ft_stats:
                self._build_backward()
            self._augmenter = _augmenter(self, self.x_u8)
            self._training_built = True
            if self.distillation is not None:
                self.distillation.teacher.bind_teacher_input(self._stem_input(True))

    # ------------------------------------------------------------------------------------------------ forward / backward
    def forward(self, training: bool = True) -> None:
        self.forward_logits(training)
        self.forward_head(training)

    def forward_logits(self, training: bool = True, teacher: bool = False) -> None:
        """Augmentation (training), a distillation teacher's logits (training), features and the bf16 FC logits
        ``logits16``.  ``teacher=True``: the inference forward of this engine as a distillation teacher, reading the
        student's stem input bound by `bind_teacher_input` instead of ``x_u8``."""
        e = self._e
        if training and self._augmenter is not None:
            self._augmenter.run()
        if training and self.distillation is not None:
            # the teacher reads this step's stem input in place, before the stem: its logits16 feed the head
            self.distillation.teacher.forward_logits(False, teacher=True)
        for lay in self._plan:
            if training and lay["train"] and self._bn_train:
                self._forward_bn_train(lay)
            elif lay["kind"] == "stem":
                x = self._teacher_in if teacher else self._stem_input(training)
                e.mbv2_stem(x, lay["w"], lay["scale"], lay["shift"], lay["y"], 1.0 / 127.5, -1.0)
            elif lay["kind"] == "dw":
                e.dwconv3x3(lay["x"], lay["w"], lay["scale"], lay["shift"], lay["y"], lay["stride"])
            else:
                lay["op"].run()
        drop = self.dropout if training else 0.0
        self._drop_seed = self.seed * 1000003 + self._step_count
        e.gap_fwd(self.feat, self.pooled, drop, self._drop_seed)
        self._fc_fwd.run()

    def forward_head(self, training: bool = True) -> None:
        """+ bias, softmax cross-entropy, accuracy, bf16 dlogits in one kernel (see `ResNet50Engine.forward_head`)."""
        e, N = self._e, self.batch
        e.zero_(self.stats)
        dl = self.dlogits16 if (training and self._training_built) else None
        mix = self._augmenter.mix if (training and self._augmenter is not None) else None
        wts = _head_weights(self, training)
        if training and self.distillation is not None:
            _kd_head(self, mix, dl, wts)
        elif mix is None and self.label_smoothing == 0:
            e.softmax_ce_head(self.logits16, self.p("fc.bias"), self.labels, self.logits, dl, self.loss_rows,
                              self.stats, 1.0 / N, *wts)
        else:   # soft targets: the partner's label at the mix row's weight, label smoothing
            e.softmax_ce_soft_head(self.logits16, self.p("fc.bias"), self.labels, mix, self.label_smoothing,
                                   self.logits, dl, self.loss_rows, self.stats, 1.0 / N, *wts)

    def backward(self) -> None:
        """Dense head weight / bias gradients; with fine_tune_at <= 18 also those of base.features[fine_tune_at:]."""
        e = self._e
        e.zero_(self.grads)
        self._fc_wg.run()
        e.fc_bias_grad(self.dlogits16, self.g("fc.bias"))
        if self._ft_stats:
            self._backward_base()
        if self.grad_hook is not None:
            self.grad_hook(0, self.flat_numel)

    def _backward_base(self) -> None:
        e = self._e
        e.zero_(self._ft_sums)
        self._fc_dg.run()
        e.gap_bwd(self.dpooled, self._plan[-1]["g"], self.dropout, self._drop_seed)
        for i in range(len(self._plan) - 1, self._ft_lowest - 1, -1):
            lay = self._plan[i]
            g, kind = lay["g"], lay["kind"]
            if self._bn_train:
                g = self._backward_bn_train(i)   # dc: the gradient of the conv output
            else:
                e.relu6_mask_reduce(g, lay["g2"], lay["y"], g, lay["sum"], lay["act"] == "relu6")
            G = self.g(lay["conv"] + ".weight")
            if kind == "pw":
                for op in lay["wg"]:
                    op.run()
            elif kind == "dw":
                e.dw_wgrad(g, lay["x"], G, lay["stride"])
            else:
                e.mbv2_stem_wgrad(self._stem_input(True), g, G, 1.0 / 127.5, -1.0)
            if i > self._ft_lowest:
                if kind == "pw":
                    lay["dg"].run()
                else:
                    scale = self._ones[:_cp(lay["cout"])] if self._bn_train else lay["scale"]
                    e.dw_dgrad(g, lay["w"], scale, self._plan[i - 1]["g"], lay["stride"])
        if not self._bn_train:   # training-mode BN: the weight gradients of dc are final, dgamma / dbeta written
            e.mbv2_ft_finalize(self.params, self.w16, self.grads, self._ft_finalize_table)

    def _stem_input(self, training: bool) -> torch.Tensor:
        """uint8 batch the stem reads: the augmented copy in training steps, x_u8 otherwise."""
        return self._augmenter.out if (training and self._augmenter is not None) else self.x_u8

    # ------------------------------------------------------------------------------------------------ utilities
    def set_augment_step(self, t: int) -> None:
        """Step word the next training forward's augmentation reads (the optimizer's step counter)."""
        if self._augmenter is not None:
            self._augmenter.set_step(t)

    def set_distillation(self, distillation) -> None:
        """Distil from ``distillation.teacher`` in the training steps captured from now on (see
        `resnet_engine.set_distillation`)."""
        set_distillation(self, distillation)

    def bind_teacher_input(self, x_u8: torch.Tensor) -> None:
        """Teach a student whose stem reads ``x_u8``: build for inference if not built (as `EngineEvalStep` does);
        ``forward_logits(training=False, teacher=True)`` then reads that buffer in place of this engine's own."""
        self._teacher_in = x_u8
        self.build(training=self.grads is not None)

    def set_input(self, x_u8: torch.Tensor, labels: Optional[torch.Tensor] = None,
                  sample_weight: Optional[torch.Tensor] = None) -> None:
        self.x_u8.copy_(x_u8.view(self.x_u8.shape), non_blocking=True)
        if labels is not None:
            self.labels.copy_(labels, non_blocking=True)
        if sample_weight is not None:
            _set_row_weight(self, sample_weight)

    def set_weighting(self, mode: Optional[str], training: bool = True) -> bool:
        """Per-row loss weights of the training or evaluation head (see `resnet_engine.set_weighting`)."""
        return set_weighting(self, mode, training)

    def set_class_weight(self, table: torch.Tensor) -> None:
        """New values of the class-weight table (float [K]); no graph needs capturing again."""
        set_class_weight(self, table)

    def loss_and_acc(self) -> Tuple[float, float]:
        s = self.stats.tolist()
        return s[0] / self.batch, s[1] / self.batch
