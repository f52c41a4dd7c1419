"""Random data augmentation in the training step: flip, rotation, zoom and translation (Keras ``RandomFlip``,
``RandomRotation``, ``RandomZoom``, ``RandomTranslation``), active in training only, as Keras preprocessing layers are.

The native engines run it on the device inside the step's CUDA graph (csrc/augment.cu, two launches ahead of the stem,
and a third with color).  This module holds the configuration, the host-built rotation table, and the **reference
implementation** - vectorised torch integer ops on any device - which reproduces every kernel bit for bit.  It is the training path of the torch
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

MixUp and CutMix (``mixup`` / ``cutmix``: the alpha of Keras's Beta(alpha, alpha)) mix every image with a partner of
the same batch after the geometric warp, and the label weights travel to the soft-target head as integer mix rows.
Draw 5 indexes a host-built table of 4096 Beta quantiles, draws 6 and 7 place the CutMix box, and one draw per step,
``s = 1 + hash_u32(key, t, 8 N) mod (N - 1)``, gives ``partner(n) = (n + s) mod N``.  Differences from Keras:
- The partners are a rotation of the batch (every image gets a different partner, and the rotation changes every step),
  not a uniformly random permutation; each data-parallel rank mixes within its own batch.
- lambda is one of 4096 quantiles of Beta(alpha, alpha), and MixUp weights are quantised to 1/256.

Color augmentation (``brightness``, ``contrast``, ``saturation``, ``hue``, ``grayscale``: Keras's ``RandomBrightness``,
``RandomContrast``, ``RandomSaturation``, ``RandomHue`` and ``RandomGrayscale``) runs after the warp and the mixing, in
that order, as one more launch (csrc/augment.cu augment_color).  Its draws come from their own key,
``color_key(key) = hash_u32(key, 0x436F6C72, 0)``: draw ``k`` of image ``n`` is ``hash_u32(color_key(key), t, 8 n + k)``,
so turning color on leaves every geometric and mix draw as it was.  The chain is integer arithmetic on Q8 values
``v = 256 p``, rounded once at the end (see `color_reference`).  Differences from Keras:
- Color is applied after the geometric warp and after mixing, and a mixed image takes image n's color draws; Keras
  would color each source image before mixing them.
- ``saturation`` s and ``hue`` h apply Keras 3's ``RandomSaturation`` / ``RandomHue`` HSV transforms but are
  parametrised like ``contrast``: the saturation factor is uniform in [1 - s, 1 + s] (the result capped at 1), the hue
  shift uniform in [-h, h] of a full turn.  Only scalar factors are accepted, not Keras's ``(lower, upper)`` tuples.
- Factors are drawn on a 2^-16 grid (the brightness delta on a 1/256-level grid) and the chain runs in Q8 fixed point.
"""
from __future__ import annotations

import math
from dataclasses import asdict, dataclass
from functools import lru_cache
from typing import Optional, Tuple

import numpy as np
import torch

FLIP_MODES = {None: 0, "horizontal": 1, "vertical": 2, "horizontal_and_vertical": 3}
FILL_MODES = ("reflect", "constant")
ROT_BITS = 12          # csrc/ops_api.h kAugRotBits: 4096 table angles
LAM_BITS = 12          # csrc/ops_api.h kAugLamBits: 4096 Beta quantiles
MAX_SIDE = 2048        # csrc/ops_api.h kAugMaxSide
PARAM_FIELDS = 8       # a00 a01 b0 a10 a11 b1 flags 0
MIX_FIELDS = 8         # partner, MixUp weight w, CutMix box x0 y0 x1 y1, mu = num / den
MIX_NONE, MIX_UP, CUT_MIX = 0, 1, 2   # csrc/ops_api.h AugMix
MAX_MIX_ALPHA = 100.0
COLOR_FIELDS = (("brightness", 1.0), ("contrast", 1.0), ("saturation", 1.0), ("hue", 0.5), ("grayscale", 1.0))
COLOR_SALT = 0x436F6C72        # color_key(key) = hash_u32(key, COLOR_SALT, 0)
Q8_MAX = 255 * 256             # a channel's Q8 ceiling
GRAY_WEIGHTS = (0.2989, 0.5870, 0.1140)
GRAY_Q16 = (19589, 38470, 7471)   # rint(65536 * GRAY_WEIGHTS), csrc/augment.cu kGrayR / kGrayG / kGrayB
_M32 = 0xFFFFFFFF


@dataclass(frozen=True)
class Augmentation:
    """``flip``: None | "horizontal" | "vertical" | "horizontal_and_vertical" (each allowed axis flips with p = 1/2);
    ``rotation`` f: angle uniform in [-2 pi f, 2 pi f], 0 <= f <= 0.5;  ``zoom`` z: sampling-grid scale uniform in
    [1 - z, 1 + z], 0 <= z < 1 (> 1 zooms out, as Keras);  ``translation`` f: x / y shifts independently uniform in
    [-f, f] of W / H, 0 <= f <= 1;  ``fill_mode``: "reflect" (d c b a | a b c d | d c b a) or "constant" with the uint8
    ``fill_value``;  ``mixup`` / ``cutmix``: the alpha of Beta(alpha, alpha) for Keras's MixUp / CutMix, in [0, 100],
    0 = off, at most one of them non-zero.  Mixing needs a loss that takes soft targets: the engines' head and the
    module backend form them from the integer labels (see `train.losses.CategoricalCrossentropy`).

    Color, applied after the warp and the mixing in this order, each 0 = off:  ``brightness`` b in [0, 1]: add a
    delta uniform in [-b, b] x 255 levels, then clip to [0, 255];  ``contrast`` c in [0, 1]: (x - mean) f + mean per
    channel, f uniform in [1 - c, 1 + c], mean over the image, then clip;  ``saturation`` s in [0, 1]: HSV saturation
    times a factor uniform in [1 - s, 1 + s], capped at 1;  ``hue`` h in [0, 0.5]: HSV hue rotated by a fraction of
    a turn uniform in [-h, h];  ``grayscale`` p in [0, 1]: with probability p every channel becomes
    0.2989 R + 0.5870 G + 0.1140 B."""

    flip: Optional[str] = None
    rotation: float = 0.0
    zoom: float = 0.0
    translation: float = 0.0
    fill_mode: str = "reflect"
    fill_value: int = 0
    mixup: float = 0.0
    cutmix: float = 0.0
    brightness: float = 0.0
    contrast: float = 0.0
    saturation: float = 0.0
    hue: float = 0.0
    grayscale: float = 0.0

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
        for name in ("mixup", "cutmix"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) \
                    or not 0.0 <= v <= MAX_MIX_ALPHA:
                raise ValueError(f"{name} must be a number in [0, {MAX_MIX_ALPHA:g}], got {v!r}")
            object.__setattr__(self, name, float(v))
        if self.mixup > 0 and self.cutmix > 0:
            raise ValueError(f"mixup and cutmix cannot both be on (got mixup={self.mixup}, cutmix={self.cutmix})")
        for name, hi in COLOR_FIELDS:
            v = getattr(self, name)
            if isinstance(v, (tuple, list)):
                raise ValueError(f"{name} takes one number in [0, {hi:g}]; Keras's (lower, upper) form is not "
                                 f"supported, got {v!r}")
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or not 0.0 <= v <= hi:
                raise ValueError(f"{name} must be a number in [0, {hi:g}], got {v!r}")
            object.__setattr__(self, name, float(v))

    def to_dict(self) -> dict:
        return asdict(self)

    @classmethod
    def from_dict(cls, d: Optional[dict]) -> Optional["Augmentation"]:
        return None if d is None else cls(**d)

    @property
    def flip_mode(self) -> int:
        return FLIP_MODES[self.flip]

    @property
    def mix_mode(self) -> int:
        """MIX_NONE, MIX_UP or CUT_MIX (csrc/ops_api.h AugMix)."""
        return MIX_UP if self.mixup > 0 else CUT_MIX if self.cutmix > 0 else MIX_NONE

    @property
    def color_on(self) -> bool:
        return any(getattr(self, name) > 0 for name, _ in COLOR_FIELDS)

    @property
    def warp_on(self) -> bool:
        """Whether the params + warp launches have work: a geometric or mix field is set, or nothing at all is (the
        identity configuration keeps its two launches)."""
        geometric = self.flip is not None or self.rotation > 0 or self.zoom > 0 or self.translation > 0
        return geometric or self.mix_mode != MIX_NONE or not self.color_on

    def color_quantised(self) -> Tuple[int, int, int, int, int]:
        """The half-ranges augment_color takes: brightness in Q8 levels, contrast and saturation in Q16, hue in Q16
        sixths of a turn, the grayscale probability in Q16."""
        return (int(round(self.brightness * Q8_MAX)), int(round(self.contrast * 65536)),
                int(round(self.saturation * 65536)), int(round(self.hue * 6 * 65536)), int(round(self.grayscale * 65536)))

    def lambda_table(self) -> torch.Tensor:
        """int32 [4096, 2]: rint(65536 lambda_i) and rint(65536 sqrt(1 - lambda_i)) for the Beta(alpha, alpha)
        quantiles lambda_i = I^-1((i + 0.5) / 4096; alpha, alpha), computed in float64 on the host."""
        if self.mix_mode == MIX_NONE:
            raise ValueError("lambda_table: neither mixup nor cutmix is on")
        lam = beta_quantiles(self.mixup or self.cutmix, 1 << LAM_BITS)
        tab = np.stack([np.rint(lam * 65536.0), np.rint(np.sqrt(1.0 - lam) * 65536.0)], 1)
        return torch.from_numpy(tab.astype(np.int32))

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


# ------------------------------------------------------------------------------------------------ Beta quantiles
def _betainc_lower(x: np.ndarray, a: float) -> np.ndarray:
    """Regularised incomplete beta I_x(a, a) for 0 <= x <= 1/2 (float64), by its continued fraction (modified Lentz).
    x <= 1/2 = (a + 1) / (2 a + 2) is the range where the fraction converges quickly."""
    tiny = 1e-300
    with np.errstate(divide="ignore"):
        front = np.exp(a * (np.log(x) + np.log1p(-x)) - (2 * math.lgamma(a) - math.lgamma(2 * a))) / a
    f = np.full_like(x, tiny)
    C, D = f.copy(), np.zeros_like(x)
    for j in range(1, 1000):
        if j == 1:
            num = np.ones_like(x)
        elif j % 2 == 0:          # d_{2m+1}, m = (j - 2) / 2
            m = (j - 2) // 2
            num = -(a + m) * (2 * a + m) * x / ((a + 2 * m) * (a + 2 * m + 1))
        else:                     # d_{2m}, m = (j - 1) / 2
            m = (j - 1) // 2
            num = m * (a - m) * x / ((a + 2 * m - 1) * (a + 2 * m))
        D = 1.0 + num * D
        D = np.where(D == 0, tiny, D)
        C = 1.0 + num / C
        C = np.where(C == 0, tiny, C)
        D = 1.0 / D
        delta = C * D
        f = f * delta
        if j > 2 and float(np.abs(delta - 1.0).max()) < 1e-15:
            break
    return front * f


@lru_cache(maxsize=16)
def _beta_quantiles(alpha: float, n: int) -> np.ndarray:
    # Bisection of I_x(a, a) = p on [0, 1/2] for the lower half of the probabilities; the upper half mirrors it
    # (Beta(a, a) is symmetric), so the table is exactly symmetric and monotone.
    half = (n + 1) // 2
    p = (np.arange(half, dtype=np.float64) + 0.5) / n
    lo, hi = np.zeros(half), np.full(half, 0.5)
    for _ in range(64):
        mid = 0.5 * (lo + hi)
        below = _betainc_lower(mid, alpha) < p
        lo, hi = np.where(below, mid, lo), np.where(below, hi, mid)
    x = 0.5 * (lo + hi)
    out = np.empty(n)
    out[:half] = x
    out[n - half:] = 1.0 - x[::-1]
    return out


def beta_quantiles(alpha: float, n: int = 1 << LAM_BITS) -> np.ndarray:
    """float64 [n]: the quantiles I^-1((i + 0.5) / n; alpha, alpha) of Beta(alpha, alpha), i = 0 .. n - 1."""
    return _beta_quantiles(float(alpha), int(n)).copy()


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


def mix_params_reference(aug: Augmentation, N: int, H: int, W: int, key: int, step: int, device=None,
                         lam_table: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The mix rows augment_mix_params writes: int32 [N, 8] = partner, MixUp weight w, CutMix box x0 y0 x1 y1 (half-open),
    and the partner's label weight mu = num / den (see csrc/augment.cu)."""
    mode = aug.mix_mode
    if mode == MIX_NONE:
        raise ValueError("mix_params_reference: neither mixup nor cutmix is on")
    dev = torch.device(device) if device is not None else torch.device("cpu")
    lam = (lam_table if lam_table is not None else aug.lambda_table()).to(dev, torch.int64)
    n = torch.arange(N, device=dev, dtype=torch.int64)
    c = n * 8
    t = int(step) & 0x7FFFFFFF
    shift = 1 + int(hash_u32(int(key), t, 8 * N)) % (N - 1) if N > 1 else 0
    partner = (n + shift) % N
    lq = lam[hash_u32(int(key), t, c + 5) >> (32 - LAM_BITS)]
    zero = torch.zeros_like(n)
    if mode == MIX_UP:
        w = (lq[:, 0] + 128) >> 8
        rows = [partner, w, zero, zero, zero, zero, 256 - w, torch.full_like(n, 256)]
    else:
        cx = (W * (hash_u32(int(key), t, c + 6) >> 16)) >> 16
        cy = (H * (hash_u32(int(key), t, c + 7) >> 16)) >> 16
        hw, hh = ((W * lq[:, 1] + 32768) >> 16) >> 1, ((H * lq[:, 1] + 32768) >> 16) >> 1
        x0, x1 = (cx - hw).clamp(0, W), (cx + hw).clamp(0, W)
        y0, y1 = (cy - hh).clamp(0, H), (cy + hh).clamp(0, H)
        rows = [partner, zero, x0, y0, x1, y1, (x1 - x0) * (y1 - y0), torch.full_like(n, H * W)]
    return torch.stack(rows, 1).to(torch.int32)


def mix_warp_reference(x_u8: torch.Tensor, params: torch.Tensor, mix: torch.Tensor, mode: int,
                       fill_mode: str = "reflect", fill_value: int = 0) -> torch.Tensor:
    """augment_mix_warp: every image's geometric warp mixed with its partner's (``mode`` MIX_UP or CUT_MIX)."""
    if mode not in (MIX_UP, CUT_MIX):
        raise ValueError("mode must be MIX_UP or CUT_MIX")
    N, H, W, _ = x_u8.shape
    own = warp_reference(x_u8, params, fill_mode, fill_value).to(torch.int64)
    m = mix.to(x_u8.device, torch.int64)
    other = own[m[:, 0]]
    if mode == MIX_UP:
        w = m[:, 1].view(N, 1, 1, 1)
        return ((w * own + (256 - w) * other + 128) >> 8).to(torch.uint8)
    ys = torch.arange(H, device=x_u8.device).view(1, H, 1)
    xs = torch.arange(W, device=x_u8.device).view(1, 1, W)
    box = ((xs >= m[:, 2].view(N, 1, 1)) & (xs < m[:, 4].view(N, 1, 1)) & (ys >= m[:, 3].view(N, 1, 1))
           & (ys < m[:, 5].view(N, 1, 1)))
    return torch.where(box.unsqueeze(-1), other, own).to(torch.uint8)


def color_key(key: int) -> int:
    """The uint32 key of the color draws: a fixed function of `augment_key`'s key, so they are independent of the
    geometric and mix draws and leave them unchanged."""
    return int(hash_u32(int(key) & _M32, COLOR_SALT, 0))


def color_draws_reference(aug: Augmentation, N: int, key: int, step: int, device=None) -> torch.Tensor:
    """int64 [N, 5]: the color draws augment_color makes for every image - brightness delta (Q8 levels), contrast
    factor f and saturation factor S (Q16), hue shift (Q16 sixths of a turn), grayscale flag.  A stage that is off
    holds its identity value (0, 65536, 65536, 0, 0)."""
    dev = torch.device(device) if device is not None else torch.device("cpu")
    bq, cq, sq, hq, pq = aug.color_quantised()
    c = torch.arange(N, device=dev, dtype=torch.int64) * 8
    t = int(step) & 0x7FFFFFFF
    ck = color_key(key)
    u = [hash_u32(ck, t, c + k) >> 16 for k in range(5)]

    def uniform(v, q):   # uniform in [-q, q) on a 2^-16 grid
        return -q + ((2 * q * v) >> 16)

    return torch.stack([uniform(u[0], bq), 65536 + uniform(u[1], cq), 65536 + uniform(u[2], sq), uniform(u[3], hq),
                        (u[4] < pq).to(torch.int64)], 1)


def _saturate(r, g, b, S):
    """v' = mx - (mx - v) k with k = min(S, mx / dl) in Q16: the max (HSV value) is kept and the saturation dl / mx
    scaled by S, capped at 1.  k = S whenever S <= 1, since mx >= dl.  A pixel with dl = 0 is unchanged."""
    mx = torch.maximum(r, torch.maximum(g, b))
    dl = mx - torch.minimum(r, torch.minimum(g, b))
    k = torch.where(S <= 65536, S, torch.minimum(S, (mx << 16) // dl.clamp(min=1)))
    return tuple(mx - (((mx - v) * k + 32768) >> 16) for v in (r, g, b))


def _rotate_hue(r, g, b, dh):
    """The hue position P in Q16 sixths of a turn (the max channel taken in the order R, G, B; the fraction rounded
    half up), rotated by dh modulo a turn; the pixel is rebuilt from (sector P >> 16, fraction P & 65535) with its max
    and min kept.  A pixel with dl = 0 comes back unchanged (every candidate value equals it)."""
    mx = torch.maximum(r, torch.maximum(g, b))
    mn = torch.minimum(r, torch.minimum(g, b))
    dl = mx - mn
    dls = dl.clamp(min=1)

    def frac(a):
        return (a * 65536 + (dls >> 1)) // dls

    turn = 6 * 65536
    P = torch.where(r == mx, torch.where(g >= b, frac(g - b), turn - frac(b - g)),
                    torch.where(g == mx, 2 * 65536 + torch.where(b >= r, frac(b - r), -frac(r - b)),
                                4 * 65536 + torch.where(r >= g, frac(r - g), -frac(g - r))))
    P = (P + dh + 2 * turn) % turn
    part = ((P & 65535) * dl + 32768) >> 16
    rise, fall = mn + part, mx - part
    sec = (P >> 16).unsqueeze(-1)

    def pick(*vals):   # the value of sector 0 .. 5
        return torch.stack(torch.broadcast_tensors(*vals), -1).gather(-1, sec).squeeze(-1)

    return (pick(mx, fall, mn, mn, rise, mx), pick(rise, mx, mx, fall, mn, mn), pick(mn, mn, rise, mx, mx, fall))


def color_apply_reference(x_u8: torch.Tensor, draws: torch.Tensor, stages) -> torch.Tensor:
    """augment_color's chain on the uint8 [N, H, W, 3] batch with the per-image ``draws`` of `color_draws_reference`;
    ``stages``: five booleans (brightness, contrast, saturation, hue, grayscale), False skipping the stage.  Q8 values
    v = 256 p in int64; clamped to [0, 255 * 256] after brightness and after contrast; contrast uses the per-channel
    mean round(sum v / (H W)) of the post-brightness image (an exact integer sum); one rounding (v + 128) >> 8 at the
    end."""
    N, H, W, _ = x_u8.shape
    d = draws.to(x_u8.device, torch.int64)
    bright, contrast, saturation, hue, gray = (bool(s) for s in stages)
    v = x_u8.to(torch.int64) << 8
    if bright:
        v = (v + d[:, 0].view(N, 1, 1, 1)).clamp(0, Q8_MAX)
    if contrast:
        mean = (v.sum((1, 2), keepdim=True) + (H * W) // 2) // (H * W)
        v = (mean + (((v - mean) * d[:, 1].view(N, 1, 1, 1) + 32768) >> 16)).clamp(0, Q8_MAX)
    r, g, b = v.unbind(-1)
    if saturation:
        r, g, b = _saturate(r, g, b, d[:, 2].view(N, 1, 1))
    if hue:
        r, g, b = _rotate_hue(r, g, b, d[:, 3].view(N, 1, 1))
    if gray:
        y = (GRAY_Q16[0] * r + GRAY_Q16[1] * g + GRAY_Q16[2] * b + 32768) >> 16
        on = d[:, 4].view(N, 1, 1) != 0
        r, g, b = (torch.where(on, y, c) for c in (r, g, b))
    return ((torch.stack([r, g, b], -1) + 128) >> 8).to(torch.uint8)


def color_reference(aug: Augmentation, x_u8: torch.Tensor, key: int, step: int) -> torch.Tensor:
    """augment_color: the color augmentation of the uint8 [N, H, W, 3] batch at optimizer step ``step``, ``key`` being
    `augment_key`'s (the color key is derived from it)."""
    draws = color_draws_reference(aug, x_u8.shape[0], key, step, device=x_u8.device)
    return color_apply_reference(x_u8, draws, [q > 0 for q in aug.color_quantised()])


def augment_batch_reference(aug: Augmentation, x_u8: torch.Tensor, key: int, step: int):
    """What the engines' training step feeds its stem and its head: the warp of the uint8 NHWC batch at optimizer step
    ``step``, mixed with the partners' warps when MixUp or CutMix is on, then colored when a color field is on, and
    the mix rows (None without mixing)."""
    if x_u8.dtype != torch.uint8 or x_u8.dim() != 4 or x_u8.shape[3] != 3:
        raise ValueError(f"augmentation needs a uint8 [N, H, W, 3] batch, got {tuple(x_u8.shape)} {x_u8.dtype}")
    N, H, W, _ = x_u8.shape
    if max(H, W) > MAX_SIDE:
        raise ValueError(f"augmentation: image sides must be at most {MAX_SIDE}")
    out, mix = x_u8, None
    if aug.warp_on:
        params = params_reference(aug, N, H, W, key, step, device=x_u8.device)
        if aug.mix_mode == MIX_NONE:
            out = warp_reference(x_u8, params, aug.fill_mode, aug.fill_value)
        else:
            mix = mix_params_reference(aug, N, H, W, key, step, device=x_u8.device)
            out = mix_warp_reference(x_u8, params, mix, aug.mix_mode, aug.fill_mode, aug.fill_value)
    if aug.color_on:
        out = color_reference(aug, out, key, step)
    return out, mix


def augment_reference(aug: Augmentation, x_u8: torch.Tensor, key: int, step: int) -> torch.Tensor:
    """The batch of `augment_batch_reference` alone: what the engines' training step feeds its stem."""
    return augment_batch_reference(aug, x_u8, key, step)[0]


# ------------------------------------------------------------------------------------------------ soft targets
def mix_weight(mix: Optional[torch.Tensor], B: int, device=None, dtype=torch.float32) -> torch.Tensor:
    """mu = num / den of every mix row (0 without mixing), divided in ``dtype`` (float32: the head's __fdiv_rn)."""
    if mix is None:
        return torch.zeros(B, device=device, dtype=dtype)
    m = mix.to(device)
    return m[:, 6].to(dtype) / m[:, 7].to(dtype)


def soft_targets(labels: torch.Tensor, num_classes: int, mix: Optional[torch.Tensor] = None,
                 label_smoothing: float = 0.0, dtype=torch.float32) -> torch.Tensor:
    """[B, K] targets of the soft-target head: (1 - eps) (lambda onehot(y_n) + mu onehot(y_partner)) + eps / K, with
    lambda = 1 - mu."""
    B = labels.numel()
    y = labels.view(-1).long()
    onehot = torch.nn.functional.one_hot(y, num_classes).to(dtype)
    mu = mix_weight(mix, B, labels.device, dtype).view(B, 1)
    t = onehot if mix is None else (1 - mu) * onehot + mu * onehot[mix[:, 0].to(labels.device).long()]
    eps = float(label_smoothing)
    return t if eps == 0 else (1 - eps) * t + eps / num_classes


def target_argmax(labels: torch.Tensor, mix: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The class accuracy compares with: the argmax of the unsmoothed (mixed) target, lowest index on ties, decided on
    the integers as the head does - the own label when 2 num < den, the partner's when 2 num > den, the lower of the two
    on a tie.  Label smoothing does not enter: Keras applies it inside the loss, and its accuracy metric never sees it."""
    y = labels.view(-1).long()
    if mix is None:
        return y
    m = mix.to(y.device).long()
    yp = y[m[:, 0]]
    twice, den = 2 * m[:, 6], m[:, 7]
    return torch.where(twice < den, y, torch.where(twice > den, yp, torch.minimum(y, yp)))


def soft_head_reference(logits: torch.Tensor, labels: torch.Tensor, mix: Optional[torch.Tensor] = None,
                        label_smoothing: float = 0.0, grad_scale: float = 1.0):
    """float64 softmax_ce_soft_head of fp32 ``logits`` [B, K] (bias included): per-row losses
    sum_k target_k (lse - logit_k), dlogits (p - target) * grad_scale, and the correct count
    argmax(logits) == target_argmax(labels, mix) (lowest index on ties, for both)."""
    z = logits.double()
    K = z.shape[1]
    t = soft_targets(labels, K, mix, label_smoothing, torch.float64)
    lse = torch.logsumexp(z, 1, keepdim=True)
    loss = (t * (lse - z)).sum(1)
    d = (torch.softmax(z, 1) - t) * grad_scale
    am = torch.from_numpy(np.argmax(logits.detach().cpu().numpy(), axis=1)).to(labels.device)
    correct = int((am == target_argmax(labels, mix)).sum())
    return loss, d, correct


def distillation_reference(logits: torch.Tensor, teacher_logits: torch.Tensor, labels: torch.Tensor,
                           mix: Optional[torch.Tensor] = None, label_smoothing: float = 0.0, alpha: float = 0.1,
                           temperature: float = 3.0):
    """Per-row losses of `train.losses.Distillation` (softmax_kd_head), in the dtype of ``logits`` [B, K] (bias
    included) and differentiable: (loss, student term, distillation term) with

        student = sum_k target_k (lse(s) - s_k),   target = `soft_targets` (smoothed, mixed)
        distill = T^2 KL(softmax(t / T) || softmax(s / T)),   from the two log-softmaxes (no clipping)
        loss    = alpha student + (1 - alpha) distill

    The module backend trains on it (fp32, autograd); in float64 it is the kernel's reference."""
    s = logits
    t = teacher_logits.to(s.dtype)
    T = float(temperature)
    tgt = soft_targets(labels, s.shape[1], mix, label_smoothing, s.dtype)
    student = (tgt * (torch.logsumexp(s, 1, keepdim=True) - s)).sum(1)
    lr = torch.log_softmax(t / T, 1)
    lq = torch.log_softmax(s / T, 1)
    distill = T * T * (lr.exp() * (lr - lq)).sum(1)
    return alpha * student + (1 - alpha) * distill, student, distill


def distillation_head_reference(logits: torch.Tensor, teacher_logits: torch.Tensor, labels: torch.Tensor,
                                mix: Optional[torch.Tensor] = None, label_smoothing: float = 0.0, alpha: float = 0.1,
                                temperature: float = 3.0, grad_scale: float = 1.0):
    """float64 softmax_kd_head of fp32 ``logits`` / ``teacher_logits`` [B, K] (biases included): the per-row
    (loss, student term, distillation term) of `distillation_reference`, dlogits
    (alpha (softmax(s) - target) + (1 - alpha) T (softmax(s / T) - softmax(t / T))) * grad_scale, and the correct
    count of `soft_head_reference`."""
    z, zt = logits.double(), teacher_logits.double()
    T = float(temperature)
    loss, student, distill = distillation_reference(z, zt, labels, mix, label_smoothing, alpha, T)
    tgt = soft_targets(labels, z.shape[1], mix, label_smoothing, torch.float64)
    d = (alpha * (torch.softmax(z, 1) - tgt) + (1 - alpha) * T * (torch.softmax(z / T, 1) - torch.softmax(zt / T, 1)))
    am = torch.from_numpy(np.argmax(logits.detach().cpu().numpy(), axis=1)).to(labels.device)
    correct = int((am == target_argmax(labels, mix)).sum())
    return loss, student, distill, d * grad_scale, correct


class DeviceAugmenter:
    """The two kernel launches of one engine: per-image parameters into ``params`` from the device step word, then the
    warp of ``x`` into ``out``.  The engine owns the buffers; the host writes the step word with `set_step` (a pinned
    ring slot and an async copy, as the optimizer hyper-parameters are written), never as a kernel argument.  With
    MixUp or CutMix the same two launches also write the mix rows ``mix`` (the soft-target head reads them) and mix
    every image with its partner; without, ``mix`` is None.  With a color field on, augment_color follows in place on
    ``out``; when color is all there is, it is the only launch and reads ``x``."""

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
        self.mix = None
        if aug.mix_mode != MIX_NONE:
            self.mix = torch.zeros(N, MIX_FIELDS, device=x.device, dtype=torch.int32)
            self.lam_table = aug.lambda_table().to(x.device)
        self.color = aug.color_quantised() if aug.color_on else None
        self.ckey = color_key(self.key)

    def set_step(self, t: int) -> None:
        """Host -> device write of the step word (outside any CUDA graph; the graph reads it on replay)."""
        def fill(row):
            row[0] = int(t) & 0x7FFFFFFF
        self._upload.push(fill)

    def run_params(self) -> None:
        """augment_params: the per-image transforms of the step in the device step word."""
        _, H, W, _ = self.x.shape
        if self.mix is not None:
            self._e.augment_mix_params(self.params, self.mix, self.step, self.rot_table, self.lam_table, H, W, self.key,
                                       self.aug.flip_mode, self._zq, self._txq, self._tyq, self.aug.mix_mode)
            return
        self._e.augment_params(self.params, self.step, self.rot_table, H, W, self.key, self.aug.flip_mode, self._zq,
                               self._txq, self._tyq)

    def run_warp(self) -> None:
        """augment_warp: ``out`` = the batch resampled by the transforms in ``params`` (and mixed by ``mix``)."""
        if self.mix is not None:
            self._e.augment_mix_warp(self.x, self.out, self.params, self.mix, self.aug.mix_mode, self.aug.fill_mode,
                                     self.aug.fill_value)
            return
        self._e.augment_warp(self.x, self.out, self.params, self.aug.fill_mode, self.aug.fill_value)

    def run_color(self, cluster: int = 0) -> int:
        """augment_color: ``out`` colored in place after the warp, or from ``x`` when there is no warp.  ``cluster``
        forces the CTAs per image (tests and benchmarks; the bytes are the same for every value).  Returns the cluster
        size launched."""
        if self.color is None:
            raise ValueError("run_color: no color field is on")
        _, H, W, _ = self.x.shape
        src = self.out if self.aug.warp_on else self.x
        return self._e.augment_color(src, self.out, self.step, H, W, self.ckey, *self.color, cluster)

    def run(self) -> None:
        if self.aug.warp_on:
            self.run_params()
            self.run_warp()
        if self.color is not None:
            self.run_color()
