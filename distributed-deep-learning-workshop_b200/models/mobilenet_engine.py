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
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Tuple

import torch

from .. import ops
from ..ops import conv as C
from .resnet_engine import ParamSpec, _align

_CFG = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]


def _cp(c: int) -> int:
    return _align(c, 64)


class MobileNetV2Engine:
    """Static-shape frozen-base MobileNetV2 classifier for one GPU (same engine surface as `ResNet50Engine`)."""

    arch = "mobilenetv2"

    def __init__(self, batch: int, num_classes: int = 5, device: Optional[torch.device] = None, image_size: int = 224,
                 dropout: float = 0.5, seed: int = 0, max_ctas: int = 0, bn_eps: float = 1e-5):
        ops.require_native()
        if image_size % 32:
            raise ValueError("image_size must be a multiple of 32")
        self.batch, self.num_classes, self.image_size = int(batch), int(num_classes), int(image_size)
        self.dropout, self.seed, self.max_ctas, self.bn_eps = float(dropout), seed, int(max_ctas), bn_eps
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self._e = ops.ext("_b200_ops")
        self.classes_padded = 64 if self.num_classes <= 64 else _align(self.num_classes, 128)
        self.feat_channels = 1280
        specs = [ParamSpec("fc.weight", (self.classes_padded, self.feat_channels), "fc_w"),
                 ParamSpec("fc.bias", (self.num_classes,), "fc_b")]
        off = 0
        for s in specs:
            s.numel = int(math.prod(s.shape))
            s.offset = off
            off += _align(s.numel)
        self.param_specs, self.spec, self.flat_numel = specs, {s.name: s for s in specs}, off
        self.params = torch.zeros(off, device=self.device, dtype=torch.float32)
        self.w16 = torch.zeros(off, device=self.device, dtype=torch.bfloat16)
        self.grads: Optional[torch.Tensor] = None
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
        self._layers = self._describe()
        self.load_state_dict(ref.state_dict())

    # ------------------------------------------------------------------------------------------------ architecture
    def _describe(self):
        """[(kind, state-dict prefix of conv, prefix of bn, cin, cout, stride, act, residual?)] in execution order."""
        L = [("stem", "base.features.0.0", "base.features.0.1", 3, 32, 2, "relu6", False)]
        cin, idx = 32, 1
        for t, c, n, s in _CFG:
            for i in range(n):
                stride = s if i == 0 else 1
                hidden = cin * t
                p = f"base.features.{idx}.conv"
                k = 0
                if t != 1:
                    L.append(("pw", f"{p}.{k}.0", f"{p}.{k}.1", cin, hidden, 1, "relu6", False))
                    k += 1
                L.append(("dw", f"{p}.{k}.0", f"{p}.{k}.1", hidden, hidden, stride, "relu6", False))
                k += 1
                L.append(("pw", f"{p}.{k}", f"{p}.{k + 1}", hidden, c, 1, "none", stride == 1 and cin == c))
                cin = c
                idx += 1
        L.append(("pw", f"base.features.{idx}.0", f"base.features.{idx}.1", cin, 1280, 1, "relu6", False))
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
        pass  # the head GEMM reads the flat bf16 copy directly; the base is frozen

    def num_parameters(self) -> int:
        return sum(v.numel() for k, v in self._base_sd.items() if k.endswith(".weight") or k.endswith(".bias")) + \
            self.trainable_parameters()

    def trainable_parameters(self) -> int:
        return self.num_classes * self.feat_channels + self.num_classes

    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {k: v.detach().clone().cpu() for k, v in self._base_sd.items()}
        sd["fc.weight"] = self.p("fc.weight")[:self.num_classes].detach().clone().cpu()
        sd["fc.bias"] = self.p("fc.bias").detach().clone().cpu()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        self._base_sd = {k: v.detach().to("cpu", copy=True) for k, v in sd.items() if k.startswith("base.")}
        self.p("fc.weight").zero_()
        self.p("fc.weight")[:self.num_classes].copy_(sd["fc.weight"].to(self.device, torch.float32))
        self.p("fc.bias").copy_(sd["fc.bias"].to(self.device, torch.float32))
        self._e.cast_bf16(self.params, self.w16)
        if self._built:
            self._load_base_weights()

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
            return self
        if self.grads is None and training:
            self.bind_grad_buffer()
        dev, N, S = self.device, self.batch, self.image_size
        bf = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        self.x_u8 = torch.zeros(N, S, S, 3, device=dev, dtype=torch.uint8)
        self.labels = torch.zeros(N, device=dev, dtype=torch.int64)
        self.stats = torch.zeros(2, **f32)
        self.logits = torch.zeros(N, self.num_classes, **f32)
        self.loss_rows = torch.zeros(N, **f32)
        self._plan: List[dict] = []
        h = S
        x = None
        block_in = None
        for kind, conv, bn, cin, cout, stride, act, residual in self._layers:
            lay = dict(kind=kind, conv=conv, bn=bn, cin=cin, cout=cout, stride=stride, act=act)
            ho = h // stride
            out = torch.zeros(N, ho, ho, _cp(cout), **bf)
            lay["scale"], lay["shift"] = torch.ones(_cp(cout), **f32), torch.zeros(_cp(cout), **f32)
            if kind == "stem":
                lay["w"] = torch.zeros(27, 32, **f32)
                lay["x"], lay["y"] = self.x_u8, out
                block_in = out
            elif kind == "dw":
                lay["w"] = torch.zeros(9, _cp(cin), **f32)
                lay["x"], lay["y"] = x, out
            else:
                lay["w"] = torch.zeros(_cp(cout), _cp(cin), **bf)
                res = block_in if residual else None
                lay["op"] = C.ConvForward(x, lay["w"], out, 1, 1, 1, 0, None, None, self.max_ctas,
                                          epilogue=(lay["scale"], lay["shift"], act, res))
                if act == "none":
                    block_in = out   # output of an inverted-residual block (linear bottleneck) = the next block's input
            self._plan.append(lay)
            x, h = out, ho
        self.feat = x   # [N, S/32, S/32, 1280]
        self.pooled = torch.zeros(N, self.feat_channels, **bf)
        self._load_base_weights()
        self._build_head(training)
        self._built = True
        return self

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
            self._training_built = True

    # ------------------------------------------------------------------------------------------------ forward / backward
    def forward(self, training: bool = True) -> None:
        e, N = self._e, self.batch
        for lay in self._plan:
            if lay["kind"] == "stem":
                e.mbv2_stem(lay["x"], lay["w"], lay["scale"], lay["shift"], lay["y"], 1.0 / 127.5, -1.0)
            elif lay["kind"] == "dw":
                e.dwconv3x3(lay["x"], lay["w"], lay["scale"], lay["shift"], lay["y"], lay["stride"])
            else:
                lay["op"].run()
        drop = self.dropout if training else 0.0
        self._drop_seed = self.seed * 1000003 + self._step_count
        e.gap_fwd(self.feat, self.pooled, drop, self._drop_seed)
        self._fc_fwd.run()
        e.zero_(self.stats)
        e.softmax_ce_head(self.logits16, self.p("fc.bias"), self.labels, self.logits,
                          self.dlogits16 if (training and self._training_built) else None, self.loss_rows, self.stats, 1.0 / N)

    def backward(self) -> None:
        """Only the Dense head is trainable: its weight / bias gradients (the base receives no gradient)."""
        e = self._e
        e.zero_(self.grads)
        self._fc_wg.run()
        e.fc_bias_grad(self.dlogits16, self.g("fc.bias"))
        if self.grad_hook is not None:
            self.grad_hook(0, self.flat_numel)

    # ------------------------------------------------------------------------------------------------ utilities
    def set_input(self, x_u8: torch.Tensor, labels: Optional[torch.Tensor] = None) -> None:
        self.x_u8.copy_(x_u8.view(self.x_u8.shape), non_blocking=True)
        if labels is not None:
            self.labels.copy_(labels, non_blocking=True)

    def loss_and_acc(self) -> Tuple[float, float]:
        s = self.stats.tolist()
        return s[0] / self.batch, s[1] / self.batch
