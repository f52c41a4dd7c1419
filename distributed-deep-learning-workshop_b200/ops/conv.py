"""Planning layer of the wgmma implicit-GEMM convolution (kernels: csrc/conv_igemm.cuh, csrc/conv_wgrad.cu).

A convolution on NHWC bf16 tensors is described to the kernels as
  * 1..4 *views* of the input that share one pixel grid (for stride 2 these are the four parity sub-grids
    ``x[:, ph::2, pw::2, :]`` - plain strided views, no copies),
  * a *tap table*: for every filter tap the view it reads and the pixel offset inside that view,
  * a pixel *box* (bw, bh, bn) with bw*bh*bn <= 128 that tiles the output exactly (or "flat" for dense 1x1).
Zero padding is the TMA out-of-bounds fill.  The reference delegates all of this to TF/cuDNN (SURVEY.md K7-K9).
"""
from __future__ import annotations

import os

import weakref
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from . import _build

_plans: "weakref.WeakSet" = weakref.WeakSet()
_retired_launches = 0


def plan_launches() -> int:
    return _retired_launches + sum(int(p.launches) for p in list(_plans))


def _divisors(n: int) -> List[int]:
    return [d for d in range(1, n + 1) if n % d == 0]


def pick_box(n: int, h: int, w: int, rows: int = 128, multiple_of: int = 1) -> Tuple[int, int, int]:
    """Pixel box (bw, bh, bn) with bw*bh*bn <= rows.  bw | w and bh | h exactly (a partial spatial box would pull in
    halo pixels); bn may overhang n (out-of-range images are zero-filled by TMA and clipped on store).

    Preference: least padded work, then most pixels per box, then widest along W."""
    best = None
    for bw in _divisors(w):
        if bw > rows:
            continue
        for bh in _divisors(h):
            if bw * bh > rows:
                continue
            for bn in range(1, rows // (bw * bh) + 1):
                p = bw * bh * bn
                if p % multiple_of:
                    continue
                tiles_n = -(-n // bn)
                waste = tiles_n * bn - n                      # zero-filled images
                mma_rows = tiles_n * (w // bw) * (h // bh)    # 128-row MMA tiles issued
                key = (-mma_rows, -waste, p, bw, bh)
                if best is None or key > best[0]:
                    best = (key, (bw, bh, bn))
    if best is None:
        raise ValueError(f"no pixel box for grid {(n, h, w)} rows<={rows} multiple_of={multiple_of}")
    return best[1]


def halo_box(h: int, w: int, cin: int, cout: int, R: int, S: int, stride: int, pad: int) -> Optional[Tuple[int, int, int]]:
    """Full-width single-image box (w, bh, 1) for the kernel's halo mode, or None when the layer does not qualify.

    Halo mode (csrc/conv_igemm.cuh): 3x3 / stride 1 / pad 1 with a resident 64x64 filter; one [w x (bh+2)] load per
    horizontal tap offset serves the three vertical taps, so a stage (28 KB) must hold w * (bh + 2) <= 224 pixels and the
    MMA tile w * bh <= 128; the vertical taps start w and 2*w rows into the stage, which must be whole 8-row swizzle atoms
    (w % 8 == 0).  `B200DDL_NO_HALO=1` keeps the generic boxes (A/B measurements)."""
    if os.environ.get("B200DDL_NO_HALO") == "1" or os.environ.get("B200DDL_NO_RESIDENT_FILTER") == "1":
        return None
    if not (R == 3 and S == 3 and stride == 1 and pad == 1 and cin == 64 and cout == 64 and w % 8 == 0):
        return None
    best = None
    for bh in _divisors(h):
        if w * bh <= 128 and w * (bh + 2) <= 224:
            best = bh if best is None else max(best, bh)
    return None if best is None else (w, best, 1)


@dataclass
class TapTable:
    views: List[torch.Tensor]
    tap_map: List[int]
    tap_dw: List[int]
    tap_dh: List[int]


def make_taps(x: torch.Tensor, R: int, S: int, stride: int, pad: int) -> TapTable:
    """Views + tap table for a forward conv / wgrad over NHWC ``x`` (N, H, W, C)."""
    if stride == 1:
        tm, dw, dh = [], [], []
        for r in range(R):
            for s in range(S):
                tm.append(0)
                dw.append(s - pad)
                dh.append(r - pad)
        return TapTable([x], tm, dw, dh)
    if stride != 2:
        raise ValueError("stride must be 1 or 2")
    N, H, W, C = x.shape
    if H % 2 or W % 2:
        raise ValueError("stride-2 convs need even H and W")
    used = {}
    views: List[torch.Tensor] = []
    tm, dw, dh = [], [], []
    for r in range(R):
        for s in range(S):
            oh, ow = r - pad, s - pad
            ph, pw = oh % 2, ow % 2
            key = (ph, pw)
            if key not in used:
                used[key] = len(views)
                views.append(x[:, ph::2, pw::2, :])
            tm.append(used[key])
            dh.append((oh - ph) // 2)
            dw.append((ow - pw) // 2)
    return TapTable(views, tm, dw, dh)


class ConvForward:
    """y = conv(x, w) [+ per-channel sum / sum-of-squares of y for BatchNorm] on the tensor cores.

    ``w`` is the bf16 filter in kernel layout ``[R*S*Cout, Cin]`` (tap-major)."""

    def __init__(self, x: torch.Tensor, w: torch.Tensor, y: torch.Tensor, R: int, S: int, stride: int = 1,
                 pad: int = 0, stat_sum: Optional[torch.Tensor] = None, stat_sqsum: Optional[torch.Tensor] = None,
                 max_ctas: int = 0, epilogue=None):
        """``epilogue=(scale, shift, act, residual)`` (inference): y = act(conv(x, w) * scale[c] + shift[c] [+ residual])
        with act in {'none', 'relu', 'relu6'} computed in the GEMM epilogue (folded BatchNorm); the residual (a tensor of
        y's shape) needs a dense 1x1 stride-1 convolution.  Mutually exclusive with the statistics outputs."""
        ext = _build.load("_b200_conv")
        taps = make_taps(x, R, S, stride, pad)
        N, Ho, Wo, _ = y.shape
        flat = (R == 1 and S == 1 and stride == 1 and pad == 0 and x.is_contiguous() and y.is_contiguous())
        if flat:
            bw = bh = bn = 0
        else:
            cout_, cin_ = w.shape[0] // (R * S), w.shape[1]
            bw, bh, bn = halo_box(Ho, Wo, cin_, cout_, R, S, stride, pad) or pick_box(N, Ho, Wo)
        self.box = (bw, bh, bn)
        if epilogue is not None:
            if stat_sum is not None:
                raise ValueError("epilogue and statistics outputs are mutually exclusive")
            scale, shift, act, residual = epilogue
            if residual is not None and not flat:
                raise ValueError("an epilogue residual needs a dense 1x1 stride-1 convolution")
            self.plan = ext.ConvPlan(taps.views, w, y, taps.tap_map, taps.tap_dw, taps.tap_dh, bw, bh, bn, None, None,
                                     max_ctas, None, None, None, residual, None, scale, shift,
                                     {"none": 0, "relu": 1, "relu6": 2}[act])
        else:
            self.plan = ext.ConvPlan(taps.views, w, y, taps.tap_map, taps.tap_dw, taps.tap_dh, bw, bh, bn,
                                     stat_sum, stat_sqsum, max_ctas)
        _plans.add(self.plan)

    def run(self) -> None:
        self.plan.run()


class ConvDgrad:
    """dx = conv_transpose(dy, w) for the same geometry, as one or more forward-style implicit GEMMs.

    ``w_master`` is the fp32 (or bf16) filter ``[R*S, Cout, Cin]``; the transposed/rotated bf16 copies the kernel
    needs are (re)built by :meth:`refresh_weights` (cheap: filters are tiny next to activations)."""

    @staticmethod
    def part_taps(R: int, S: int, stride: int, pad: int) -> List[List[int]]:
        """Filter-tap index lists of the GEMMs a dgrad is made of, in plan order: one list with every tap for stride 1,
        one list per non-empty output-parity class for stride 2.  (Lets an owner lay all weight copies out in one buffer.)"""
        if stride == 1:
            return [[r * S + s for r in range(R) for s in range(S)]]
        parts = []
        for ph in range(2):
            for pw in range(2):
                idx = [r * S + s for r in range(R) for s in range(S) if (r - pad) % 2 == ph and (s - pad) % 2 == pw]
                if idx:
                    parts.append(idx)
        return parts

    def __init__(self, dy: torch.Tensor, w_master: torch.Tensor, dx: torch.Tensor, R: int, S: int, stride: int = 1,
                 pad: int = 0, max_ctas: int = 0, wbuf: Optional[torch.Tensor] = None, bwd_stats=None,
                 block_grad=None, wbufs: Optional[List[torch.Tensor]] = None):
        """``bwd_stats=(y, scale, shift, sum_dz, sum_dzy)`` (stride 1 only) fuses the BatchNorm-backward reduction of
        the activation this gradient belongs to into the GEMM epilogue: dz = dx * [y*scale+shift > 0].

        ``block_grad=(skip_grad, relu_mask, y3, sum_dz, sum_dzy)`` (dense 1x1 stride-1 only): ``dx`` receives
        dz = (conv_transpose(dy, w) + skip_grad) * relu_mask - the complete masked gradient of the previous residual
        block's output - and sum(dz), sum(dz * y3) of that block's last BatchNorm are accumulated in the same epilogue.
        ``skip_grad`` has dx's grid, or its stride-2 sub-grid (compact gradient of a strided 1x1 projection)."""
        if bwd_stats is not None and stride != 1:
            raise ValueError("bwd_stats: stride-1 convs only (a strided dgrad has no fused reduction)")
        if block_grad is not None and (stride != 1 or bwd_stats is not None):
            raise ValueError("block_grad: stride-1 convs only, and not together with bwd_stats")
        ext = _build.load("_b200_conv")
        self.R, self.S, self.stride, self.pad = R, S, stride, pad
        self.fused_bwd_stats = bwd_stats is not None
        self.block_grad = block_grad is not None
        self.w_master = w_master
        if wbufs is not None:
            assert wbuf is None and len(wbufs) == len(self.part_taps(R, S, stride, pad))
            if stride == 1:
                wbuf = wbufs[0]
        self.external_wbuf = wbuf is not None or wbufs is not None  # owner refreshes them (one batched kernel for all layers)
        taps_total, cout, cin = w_master.shape
        assert taps_total == R * S
        self.parts = []  # (plan, weight buffer, tap index list)
        self.boxes = []  # pixel box (bw, bh, bn) of each part; (0, 0, 0) = flat
        self._idx_dev = {}
        self.needs_zero = False
        self.dx = dx
        N, Ho, Wo, _ = dy.shape
        if stride == 1:
            # dx[h] = sum_r dy[h + pad - r] w[r]  -> forward conv with taps reversed and pad' = R-1-pad
            idx = [r * S + s for r in range(R) for s in range(S)]
            tm, dw, dh = [], [], []
            for r in range(R):
                for s in range(S):
                    tm.append(0)
                    dh.append(pad - r)
                    dw.append(pad - s)
            if wbuf is None:
                wbuf = torch.empty(len(idx) * cin, cout, dtype=torch.bfloat16, device=dy.device)
            else:
                wbuf = wbuf.view(len(idx) * cin, cout)
            flat = (R == 1 and S == 1 and pad == 0 and dy.is_contiguous() and dx.is_contiguous())
            box = (0, 0, 0) if flat else (halo_box(dx.shape[1], dx.shape[2], cout, cin, R, S, 1, R - 1 - pad)
                                          or pick_box(N, dx.shape[1], dx.shape[2]))
            if block_grad is not None:
                if not flat:
                    raise ValueError("block_grad needs a dense 1x1 stride-1 convolution")
                skip, mask, y3, s_dz, s_dzy = block_grad
                plan = ext.ConvPlan([dy], wbuf, dx, tm, dw, dh, 0, 0, 0, s_dz, s_dzy, max_ctas, y3, None, None,
                                    skip, mask)
            elif self.fused_bwd_stats:
                y, sc, sh, s_dz, s_dzy = bwd_stats
                plan = ext.ConvPlan([dy], wbuf, dx, tm, dw, dh, box[0], box[1], box[2], s_dz, s_dzy, max_ctas, y, sc, sh)
            else:
                plan = ext.ConvPlan([dy], wbuf, dx, tm, dw, dh, box[0], box[1], box[2], None, None, max_ctas)
            _plans.add(plan)
            self.parts.append((plan, wbuf, idx))
            self.boxes.append(box)
        else:
            # output parity classes: dx[2i+ph, 2j+pw] = sum_{taps with (r-pad)%2==ph, (s-pad)%2==pw} dy[i-dh, j-dw] w[r,s]
            for ph in range(2):
                for pw in range(2):
                    idx, tm, dw, dh = [], [], [], []
                    for r in range(R):
                        for s in range(S):
                            oh, ow = r - pad, s - pad
                            if oh % 2 == ph and ow % 2 == pw:
                                idx.append(r * S + s)
                                tm.append(0)
                                dh.append(-((oh - ph) // 2))
                                dw.append(-((ow - pw) // 2))
                    out_view = dx[:, ph::2, pw::2, :]
                    if not idx:
                        self.needs_zero = True
                        continue
                    if wbufs is not None:
                        wbuf = wbufs[len(self.parts)].view(len(idx) * cin, cout)
                    else:
                        wbuf = torch.empty(len(idx) * cin, cout, dtype=torch.bfloat16, device=dy.device)
                        self._idx_dev[tuple(idx)] = torch.tensor(idx, device=dy.device, dtype=torch.long)
                    box = pick_box(N, out_view.shape[1], out_view.shape[2])
                    plan = ext.ConvPlan([dy], wbuf, out_view, tm, dw, dh, box[0], box[1], box[2], None, None, max_ctas)
                    _plans.add(plan)
                    self.parts.append((plan, wbuf, idx))
                    self.boxes.append(box)
        self.refresh_weights()

    def refresh_weights(self) -> None:
        if self.external_wbuf:
            return
        w = self.w_master
        full = list(range(w.shape[0]))
        for _, wbuf, idx in self.parts:
            if idx == full and w.is_cuda and w.dtype == torch.float32 and w.is_contiguous():
                # one kernel: fp32 [t, Cout, Cin] -> bf16 [t, Cin, Cout]
                _build.load("_b200_ops").weight_prep(w, None, wbuf, w.shape[0], w.shape[1], w.shape[2])
            else:
                it = self._idx_dev.get(tuple(idx))
                sel = w.index_select(0, it) if it is not None else w  # device index: CUDA-graph capturable
                wbuf.view(len(idx), w.shape[2], w.shape[1]).copy_(sel.transpose(1, 2))

    def run(self) -> None:
        if self.needs_zero:
            _build.load("_b200_ops").zero_(self.dx)  # memset node, not a kernel
        for plan, _, _ in self.parts:
            plan.run()


class ConvWgrad:
    """dw[t, co, ci] += sum_px dy[px, co] * x_t[px, ci]  (fp32 accumulation with vector atomics; zero dw first)."""

    def __init__(self, dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, R: int, S: int, stride: int = 1,
                 pad: int = 0, px_chunks: int = 0, max_ctas: int = 0, smem_budget: int = 0):
        ext = _build.load("_b200_conv")
        taps = make_taps(x, R, S, stride, pad)
        N, Ho, Wo, _ = dy.shape
        flat = (R == 1 and S == 1 and stride == 1 and pad == 0 and x.is_contiguous() and dy.is_contiguous()
                and (N * Ho * Wo) % 64 == 0)
        if flat:
            bw = bh = bn = 0
        else:
            # keep >= 3 pipeline stages in 227 KB: stage = (dY chunks + X chunks) * P pixels * 128 B (G <= 4 X chunks)
            cin, cout = x.shape[3], dy.shape[3]
            cb = cin // 64
            g = S * (2 if (cb >= 2 and S * 2 <= 4) else 1) if S > 1 else max(d for d in (1, 2, 3, 4) if cb % d == 0)
            chunks = (1 if cout == 64 else 2) + g
            budget = smem_budget if 0 < smem_budget < 232448 else 232448
            want_stages = 3 if budget >= 200000 else 2
            rows = min(128, ((budget - 256 - 1024) // (want_stages * chunks * 128)) // 16 * 16)
            bw, bh, bn = pick_box(N, Ho, Wo, rows=rows, multiple_of=16)
        self.box = (bw, bh, bn)
        self.plan = ext.WgradPlan(dy, taps.views, dw, R, S, taps.tap_map, taps.tap_dw, taps.tap_dh, bw, bh, bn,
                                  px_chunks, max_ctas, smem_budget)
        _plans.add(self.plan)

    def run(self) -> None:
        self.plan.run()


class StemForward:
    """y = conv7x7/2(x_u8 / 127.5 - 1, w) for the 3-channel uint8 input batch (+ fused BatchNorm statistics).

    ``w16`` is the bf16 filter as ``[64, 192]`` with k = (r*7 + s)*3 + c (147 real columns, zero padded)."""

    def __init__(self, x_u8: torch.Tensor, w16: torch.Tensor, y: torch.Tensor, stat_sum=None, stat_sqsum=None,
                 mul: float = 1.0 / 127.5, add: float = -1.0, max_ctas: int = 0):
        ext = _build.load("_b200_conv")
        self.plan = ext.StemPlan(x_u8, w16, y, None, stat_sum, stat_sqsum, mul, add, max_ctas)
        _plans.add(self.plan)

    def run(self) -> None:
        self.plan.run()


class StemWgrad:
    """dw[49, 64, 3] (fp32, accumulated) = sum_px dy[px, co] * patch(x_u8)[px, k]."""

    def __init__(self, x_u8: torch.Tensor, dy: torch.Tensor, dw: torch.Tensor, mul: float = 1.0 / 127.5,
                 add: float = -1.0, max_ctas: int = 0):
        ext = _build.load("_b200_conv")
        self.plan = ext.StemPlan(x_u8, None, dy, dw, None, None, mul, add, max_ctas)
        _plans.add(self.plan)

    def run(self) -> None:
        self.plan.run()


def pack_stem_weight(w_tck: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """[49, 64, 3] (tap, co, c) -> bf16 [64, 192] with k = tap*3 + c (columns 147.. stay zero)."""
    out[:, :147].copy_(w_tck.permute(1, 0, 2).reshape(64, 147))
    return out


# ------------------------------------------------------------------------------------------- references (tests)
def weight_to_kernel_layout(w_oihw: torch.Tensor) -> torch.Tensor:
    """torch [Cout, Cin, R, S] -> kernel layout [R*S, Cout, Cin]."""
    co, ci, R, S = w_oihw.shape
    return w_oihw.permute(2, 3, 0, 1).reshape(R * S, co, ci).contiguous()


def weight_from_kernel_layout(w_tck: torch.Tensor, R: int, S: int) -> torch.Tensor:
    t, co, ci = w_tck.shape
    return w_tck.view(R, S, co, ci).permute(2, 3, 0, 1).contiguous()


def conv_reference(x_nhwc: torch.Tensor, w_tck: torch.Tensor, R: int, S: int, stride: int, pad: int) -> torch.Tensor:
    """fp32 reference of the forward conv (NHWC in, NHWC out)."""
    w = weight_from_kernel_layout(w_tck.float(), R, S)
    y = torch.nn.functional.conv2d(x_nhwc.float().permute(0, 3, 1, 2), w, stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1).contiguous()
