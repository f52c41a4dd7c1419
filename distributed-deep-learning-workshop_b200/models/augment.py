"""Random data augmentation in the training step: flip, rotation, zoom and translation (Keras ``RandomFlip``,
``RandomRotation``, ``RandomZoom``, ``RandomTranslation``), active in training only, as Keras preprocessing layers are.

The native engines run it on the device inside the step's CUDA graph (csrc/augment.cu, two launches ahead of the stem).
This module holds the configuration, the host-built rotation table, and the **reference implementation** - vectorised
torch integer ops on any device - which reproduces both kernels bit for bit.  It is the training path of the torch
modules (`FrozenBaseClassifier` on the module backend) and the oracle of the GPU tests.

Differences from Keras, on purpose:
- The transforms are composed into ONE affine map per image, so each output pixel is interpolated once; Keras applies
  its layers one after another, each interpolating and filling again.
- Interpolation is bilinear only, with weights quantised to 1/256 and an integer blend.
- Angles come from a table of 4096 evenly spaced angles over [-2 pi f, 2 pi f]; zoom and translation are drawn on a
  2^-16 grid.

Parameters of image ``n`` at step ``t`` are a pure function of (seed, rank, t, n): draw ``k`` is
``hash_u32(key(seed, rank), t, 8 n + k)`` with the dropout hash (csrc/hash.cuh).  ``t`` is the optimizer's step counter,
which checkpoints store, so a resumed run repeats the augmentation of an uninterrupted one.
"""
from __future__ import annotations

import math
from dataclasses import asdict, dataclass
from typing import Optional, Tuple

import numpy as np
import torch

FLIP_MODES = {None: 0, "horizontal": 1, "vertical": 2, "horizontal_and_vertical": 3}
FILL_MODES = ("reflect", "constant")
ROT_BITS = 12          # csrc/ops_api.h kAugRotBits: 4096 table angles
MAX_SIDE = 2048        # csrc/ops_api.h kAugMaxSide
PARAM_FIELDS = 8       # a00 a01 b0 a10 a11 b1 flags 0
_M32 = 0xFFFFFFFF


@dataclass(frozen=True)
class Augmentation:
    """``flip``: None | "horizontal" | "vertical" | "horizontal_and_vertical" (each allowed axis flips with p = 1/2);
    ``rotation`` f: angle uniform in [-2 pi f, 2 pi f], 0 <= f <= 0.5;  ``zoom`` z: sampling-grid scale uniform in
    [1 - z, 1 + z], 0 <= z < 1 (> 1 zooms out, as Keras);  ``translation`` f: x / y shifts independently uniform in
    [-f, f] of W / H, 0 <= f <= 1;  ``fill_mode``: "reflect" (d c b a | a b c d | d c b a) or "constant" with the uint8
    ``fill_value``."""

    flip: Optional[str] = None
    rotation: float = 0.0
    zoom: float = 0.0
    translation: float = 0.0
    fill_mode: str = "reflect"
    fill_value: int = 0

    def __post_init__(self):
        if self.flip not in FLIP_MODES:
            raise ValueError(f"flip must be one of {list(FLIP_MODES)}, got {self.flip!r}")
        for name, lo, hi, hi_open in (("rotation", 0.0, 0.5, False), ("zoom", 0.0, 1.0, True),
                                      ("translation", 0.0, 1.0, False)):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) \
                    or v < lo or (v >= hi if hi_open else v > hi):
                raise ValueError(f"{name} must be a number in [{lo}, {hi}{')' if hi_open else ']'}, got {v!r}")
            object.__setattr__(self, name, float(v))
        if self.fill_mode not in FILL_MODES:
            raise ValueError(f"fill_mode must be one of {FILL_MODES}, got {self.fill_mode!r}")
        if isinstance(self.fill_value, bool) or not isinstance(self.fill_value, int) or not 0 <= self.fill_value <= 255:
            raise ValueError(f"fill_value must be an int in 0..255, got {self.fill_value!r}")

    def to_dict(self) -> dict:
        return asdict(self)

    @classmethod
    def from_dict(cls, d: Optional[dict]) -> Optional["Augmentation"]:
        return None if d is None else cls(**d)

    @property
    def flip_mode(self) -> int:
        return FLIP_MODES[self.flip]

    def quantised(self, H: int, W: int) -> Tuple[int, int, int]:
        """Q16.16 half-ranges (zoom, x translation in pixels, y translation in pixels) the kernels take."""
        return (int(round(self.zoom * 65536)), int(round(self.translation * W * 65536)),
                int(round(self.translation * H * 65536)))

    def rotation_table(self) -> torch.Tensor:
        """int32 [4096, 2]: Q16.16 (cos, sin) of 4096 evenly spaced angles over [-2 pi f, 2 pi f] (endpoints included),
        computed in float64 on the host and rounded to nearest (ties to even)."""
        n = 1 << ROT_BITS
        theta = 2.0 * math.pi * self.rotation * (2.0 * np.arange(n, dtype=np.float64) - (n - 1)) / (n - 1)
        tab = np.stack([np.rint(np.cos(theta) * 65536.0), np.rint(np.sin(theta) * 65536.0)], 1)
        return torch.from_numpy(tab.astype(np.int32))


def check_augmentation(aug) -> Optional[Augmentation]:
    if aug is None or isinstance(aug, Augmentation):
        return aug
    if isinstance(aug, dict):
        return Augmentation.from_dict(aug)
    raise ValueError(f"augmentation must be an Augmentation, a dict of its fields or None, got {type(aug).__name__}")


# ------------------------------------------------------------------------------------------------ hash (csrc/hash.cuh)
def _mul32(a, k: int):
    """(a * k) mod 2^32 for uint32 values held in int64, without overflowing int64."""
    return (a * (k & 0xFFFF) + (((a * (k >> 16)) & 0xFFFF) << 16)) & _M32


def hash_u32(a, b, c):
    """csrc/hash.cuh hash_u32 on int64 tensors (or Python ints) holding uint32 values."""
    h = _mul32(a, 0x9E3779B1) ^ _mul32((b + 0x7F4A7C15) & _M32, 0x85EBCA77) ^ _mul32((c + 0x165667B1) & _M32, 0xC2B2AE3D)
    h ^= h >> 15
    h = _mul32(h, 0x2C1B3C6D)
    h ^= h >> 12
    h = _mul32(h, 0x297A2D39)
    h ^= h >> 15
    return h


def augment_key(seed: int, rank: int = 0) -> int:
    """The uint32 key of (seed, rank): data-parallel ranks draw independent transforms."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return int(hash_u32(s & _M32, (s >> 32) ^ 0xA5A5A5A5, int(rank) & _M32))


# ------------------------------------------------------------------------------------------------ reference kernels
def params_reference(aug: Augmentation, N: int, H: int, W: int, key: int, step: int,
                     device=None, rot_table: Optional[torch.Tensor] = None) -> torch.Tensor:
    """augment_params: int32 [N, 8] = a00 a01 b0 a10 a11 b1 flags 0 of every image (see csrc/augment.cu)."""
    dev = torch.device(device) if device is not None else torch.device("cpu")
    rot = (rot_table if rot_table is not None else aug.rotation_table()).to(dev, torch.int64)
    zq, txq, tyq = aug.quantised(H, W)
    c = torch.arange(N, device=dev, dtype=torch.int64) * 8
    t = int(step) & 0x7FFFFFFF   # the device step word is an int32
    r = [hash_u32(int(key), t, c + k) for k in range(5)]
    fm = aug.flip_mode
    hf = (r[0] & 1) * int(bool(fm & 1))
    vf = ((r[0] >> 1) & 1) * int(bool(fm & 2))
    cs = rot[r[1] >> (32 - ROT_BITS)]
    s = 65536 - zq + ((2 * zq * (r[2] >> 16)) >> 16)
    tx = -txq + ((2 * txq * (r[3] >> 16)) >> 16)
    ty = -tyq + ((2 * tyq * (r[4] >> 16)) >> 16)
    mc, ms = (s * cs[:, 0] + 32768) >> 16, (s * cs[:, 1] + 32768) >> 16
    a00, a01 = torch.where(hf == 1, -mc, mc), torch.where(hf == 1, ms, -ms)
    a10, a11 = torch.where(vf == 1, -ms, ms), torch.where(vf == 1, -mc, mc)
    b0 = (W - 1) * 32768 - ((a00 * (W - 1) + a01 * (H - 1)) >> 1) - ((a00 * tx + a01 * ty) >> 16)
    b1 = (H - 1) * 32768 - ((a10 * (W - 1) + a11 * (H - 1)) >> 1) - ((a10 * tx + a11 * ty) >> 16)
    out = torch.stack([a00, a01, b0, a10, a11, b1, hf | (vf << 1), torch.zeros_like(a00)], 1)
    return out.to(torch.int32)


def _tap(i: torch.Tensor, n: int, reflect: bool):
    valid = (i >= 0) & (i < n)
    if reflect:
        m = torch.remainder(i, 2 * n)
        return torch.where(m < n, m, 2 * n - 1 - m), torch.ones_like(valid)
    return torch.where(valid, i, torch.zeros_like(i)), valid


def warp_reference(x_u8: torch.Tensor, params: torch.Tensor, fill_mode: str = "reflect", fill_value: int = 0) -> torch.Tensor:
    """augment_warp: uint8 [N, H, W, 3] -> uint8 [N, H, W, 3], the bilinear warp of each image by its params row."""
    if fill_mode not in FILL_MODES:
        raise ValueError(f"fill_mode must be one of {FILL_MODES}")
    N, H, W, _ = x_u8.shape
    dev = x_u8.device
    p = params.to(dev, torch.int64).view(N, PARAM_FIELDS, 1, 1)
    ys = torch.arange(H, device=dev, dtype=torch.int64).view(1, H, 1)
    xs = torch.arange(W, device=dev, dtype=torch.int64).view(1, 1, W)
    sx = p[:, 0] * xs + p[:, 1] * ys + p[:, 2]
    sy = p[:, 3] * xs + p[:, 4] * ys + p[:, 5]
    fx, fy = (sx >> 8) & 255, (sy >> 8) & 255
    reflect = fill_mode == "reflect"
    ix0, vx0 = _tap(sx >> 16, W, reflect)
    ix1, vx1 = _tap((sx >> 16) + 1, W, reflect)
    iy0, vy0 = _tap(sy >> 16, H, reflect)
    iy1, vy1 = _tap((sy >> 16) + 1, H, reflect)
    img = x_u8.reshape(N, H * W, 3).to(torch.int64)
    base = torch.arange(N, device=dev, dtype=torch.int64).view(N, 1, 1) * (H * W)

    def tap(iy, vy, ix, vx):
        flat = (base + iy * W + ix).view(-1)
        v = img.view(-1, 3)[flat].view(N, H, W, 3)
        return torch.where((vy & vx).unsqueeze(-1), v, torch.full_like(v, int(fill_value)))

    w00 = ((256 - fx) * (256 - fy)).unsqueeze(-1)
    w01 = (fx * (256 - fy)).unsqueeze(-1)
    w10 = ((256 - fx) * fy).unsqueeze(-1)
    w11 = (fx * fy).unsqueeze(-1)
    acc = w00 * tap(iy0, vy0, ix0, vx0) + w01 * tap(iy0, vy0, ix1, vx1) + w10 * tap(iy1, vy1, ix0, vx0) \
        + w11 * tap(iy1, vy1, ix1, vx1)
    return ((acc + 32768) >> 16).to(torch.uint8)


def augment_reference(aug: Augmentation, x_u8: torch.Tensor, key: int, step: int) -> torch.Tensor:
    """What the engines' training step feeds its stem: the warp of the uint8 NHWC batch at optimizer step ``step``."""
    if x_u8.dtype != torch.uint8 or x_u8.dim() != 4 or x_u8.shape[3] != 3:
        raise ValueError(f"augmentation needs a uint8 [N, H, W, 3] batch, got {tuple(x_u8.shape)} {x_u8.dtype}")
    N, H, W, _ = x_u8.shape
    if max(H, W) > MAX_SIDE:
        raise ValueError(f"augmentation: image sides must be at most {MAX_SIDE}")
    params = params_reference(aug, N, H, W, key, step, device=x_u8.device)
    return warp_reference(x_u8, params, aug.fill_mode, aug.fill_value)


class DeviceAugmenter:
    """The two kernel launches of one engine: per-image parameters into ``params`` from the device step word, then the
    warp of ``x`` into ``out``.  The engine owns the buffers; the host writes the step word with `set_step` (a pinned
    ring slot and an async copy, as the optimizer hyper-parameters are written), never as a kernel argument."""

    def __init__(self, aug: Augmentation, x: torch.Tensor, seed: int, rank: int = 0):
        from .. import ops
        from ..utils.pinned import PinnedUpload

        self.aug = aug
        self._e = ops.ext("_b200_ops")
        N, H, W, _ = x.shape
        if max(H, W) > MAX_SIDE:
            raise ValueError(f"augmentation: image sides must be at most {MAX_SIDE}")
        self.x = x
        self.out = torch.zeros_like(x)
        self.params = torch.zeros(N, PARAM_FIELDS, device=x.device, dtype=torch.int32)
        self.step = torch.zeros(1, device=x.device, dtype=torch.int32)
        self.rot_table = aug.rotation_table().to(x.device)
        self.key = augment_key(seed, rank)
        self._zq, self._txq, self._tyq = aug.quantised(H, W)
        self._upload = PinnedUpload(self.step)

    def set_step(self, t: int) -> None:
        """Host -> device write of the step word (outside any CUDA graph; the graph reads it on replay)."""
        def fill(row):
            row[0] = int(t) & 0x7FFFFFFF
        self._upload.push(fill)

    def run_params(self) -> None:
        """augment_params: the per-image transforms of the step in the device step word."""
        _, H, W, _ = self.x.shape
        self._e.augment_params(self.params, self.step, self.rot_table, H, W, self.key, self.aug.flip_mode, self._zq,
                               self._txq, self._tyq)

    def run_warp(self) -> None:
        """augment_warp: ``out`` = the batch resampled by the transforms in ``params``."""
        self._e.augment_warp(self.x, self.out, self.params, self.aug.fill_mode, self.aug.fill_value)

    def run(self) -> None:
        self.run_params()
        self.run_warp()
