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


def halo_box(h: int, w: int) -> Optional[Tuple[int, int, int]]:
    """Full-width single-image box (w, bh, 1) for the kernel's halo mode, or None when the output plane has none.

    Halo mode (csrc/conv_igemm.cuh): one [w x (bh+2)] load per horizontal tap offset serves the three vertical taps, so a
    stage (28 KB) must hold w * (bh + 2) <= 224 pixels and the MMA tile w * bh <= 128; the vertical taps start w and 2*w
    rows into the stage, which must be whole 8-row swizzle atoms (w % 8 == 0)."""
    if w % 8:
        return None
    bhs = [bh for bh in _divisors(h) if w * bh <= 128 and w * (bh + 2) <= 224]
    return (w, max(bhs), 1) if bhs else None


@dataclass(frozen=True)
class ConvSwitches:
    """A/B switches of the convolution planner, for measurements; the defaults give the production plans."""
    block_n: int = 0                  # 64 or 128: force this N-tile width wherever it divides Cout
    no_halo: bool = False             # no halo mode
    no_resident_filter: bool = False  # no resident filter (and so no halo mode)


def conv_switches() -> ConvSwitches:
    """The switches from the environment: ``B200DDL_BLOCK_N=64|128``, ``B200DDL_NO_HALO=1``,
    ``B200DDL_NO_RESIDENT_FILTER=1``."""
    block_n = os.environ.get("B200DDL_BLOCK_N", "")
    return ConvSwitches(block_n=int(block_n) if block_n in ("64", "128") else 0,
                        no_halo=os.environ.get("B200DDL_NO_HALO") == "1",
                        no_resident_filter=os.environ.get("B200DDL_NO_RESIDENT_FILTER") == "1")


def sm_count() -> int:
    """SMs of the current device: the persistent grid of a plan without ``max_ctas`` has one CTA per SM."""
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@dataclass(frozen=True)
class ConvTiling:
    box: Tuple[int, int, int]   # pixel box (bw, bh, bn); (0, 0, 0) = flat
    block_n: int                # N-tile width (output channels per tile)
    resident_filter: bool       # the CTA's whole filter slice stays in shared memory
    halo: bool                  # halo mode (3x3 stride-1 taps over full-width boxes)
    tiles: int                  # M-tiles x N-blocks
    grid: int                   # persistent CTAs


_HALO_OFFSETS = sorted((dw, dh) for dw in (-1, 0, 1) for dh in (-1, 0, 1))


def plan_conv(grid: Sequence[int], view_widths: Sequence[int], cin: int, cout: int, tap_map: Sequence[int],
              tap_dw: Sequence[int], tap_dh: Sequence[int], flat: bool, stats_mode: int, max_ctas: int, sm_count: int,
              switches: ConvSwitches) -> ConvTiling:
    """Tiling of one implicit-GEMM convolution (csrc/conv_igemm.cuh) writing an (N, Ho, Wo, cout) ``grid`` from input
    views of widths ``view_widths`` through the given tap table; ``flat``: a dense 1x1 GEMM over all pixels.
    ``stats_mode`` is the epilogue (0 none, 1 forward statistics, 2 fused BatchNorm-backward reduction, 3 block-gradient
    merge, 4 inference epilogue); ``max_ctas`` (0: ``sm_count``) caps the persistent grid."""
    n, ho, wo = grid
    taps = len(tap_map)
    cap = max_ctas if max_ctas > 0 else sm_count
    # Resident filter: one N-block of 64 channels whose taps * kblocks filter tiles (8 KB each) fit in 72 KB.
    resident = cout == 64 and taps * (cin // 64) <= 9 and stats_mode != 3 and not switches.no_resident_filter
    # Halo mode: 9 taps on ONE view of the output's width forming the full {-1,0,1}^2 offset grid, in any order.
    halo = (resident and not switches.no_halo and not flat and len(view_widths) == 1 and view_widths[0] == wo
            and not any(tap_map) and sorted(zip(tap_dw, tap_dh)) == _HALO_OFFSETS)
    box = halo_box(ho, wo) if halo else None
    halo = box is not None
    if flat:
        box = (0, 0, 0)
        m_tiles = -(-n * ho * wo // 128)
    else:
        box = box or pick_box(n, ho, wo)
        m_tiles = (wo // box[0]) * (ho // box[1]) * -(-n // box[2])
    # Tile width: the wider N tile re-reads the A operand less, but a persistent grid of one CTA per SM pays for whole
    # waves.  The cost model is waves x tile width (the MMA time of a tile is proportional to its width); the narrower
    # tile is taken only when it wins by >= 10 %.  128 is the widest: each consumer warpgroup holds a whole tile's
    # 128 x BLOCK_N fp32 accumulator in registers (128 per thread at BLOCK_N = 128).
    def cost(bn: int) -> int:
        return -(-m_tiles * (cout // bn) // cap) * bn

    block_n = 128 if cout % 128 == 0 and cost(64) * 10 > cost(128) * 9 else 64
    if switches.block_n and cout % switches.block_n == 0:
        block_n = switches.block_n
    tiles = m_tiles * (cout // block_n)
    return ConvTiling(box, block_n, resident, halo, tiles, min(tiles, cap))


SMEM_BYTES = 232448   # 227 KB: the largest dynamic shared memory of one CTA on sm_90
_WG_SMEM_EXTRA = 256 + 1024   # mbarriers, and 1 KB to align the dynamic smem base


@dataclass(frozen=True)
class WgradTiling:
    box: Tuple[int, int, int]   # pixel box (bw, bh, bn) of one k-iteration; (0, 0, 0) = flat (64 pixels)
    cb_per_group: int           # Cin 64-blocks per unit
    G: int                      # 64-channel X chunks per unit: S * cb_per_group
    stages: int                 # pipeline stages
    px_chunks: int              # split-K factor over pixels
    units: int
    grid: int                   # persistent CTAs


def plan_wgrad(grid: Sequence[int], cin: int, cout: int, R: int, S: int, flat: bool, px_chunks: int, max_ctas: int,
               smem_budget: int, sm_count: int) -> WgradTiling:
    """Tiling of one weight-gradient GEMM (csrc/conv_wgrad.cu) over the (N, Ho, Wo) ``grid`` of dy: a unit is one filter
    row, one Cin group and one 128-channel Cout block over one pixel chunk.  ``px_chunks`` (0: one wave of units),
    ``max_ctas`` (0: ``sm_count``) and ``smem_budget`` (0: all of it) are the caller's limits."""
    n, ho, wo = grid
    cb = cin // 64
    # the unit's 64 x (64 * G) fp32 accumulator lives in the registers of one warpgroup: G <= 4 (N <= 256)
    cb_per_group = max(d for d in (1, 2, 3, 4) if cb % d == 0) if S == 1 else (2 if cb >= 2 and S * 2 <= 4 else 1)
    G = S * cb_per_group
    chunks = (1 if cout == 64 else 2) + G   # 64-channel chunks of a stage: dY's, then X's
    # smem_budget < 227 KB leaves room for bandwidth-bound kernels to co-reside when wgrad runs on a side stream
    budget = smem_budget if 0 < smem_budget < SMEM_BYTES else SMEM_BYTES
    if flat:
        box, P = (0, 0, 0), 64
        iters = n * ho * wo // P
    else:
        # keep >= 3 pipeline stages (2 in a budget below 200,000 B): a stage is chunks * P pixels * 128 B
        want_stages = 3 if budget >= 200000 else 2
        rows = min(128, ((budget - _WG_SMEM_EXTRA) // (want_stages * chunks * 128)) // 16 * 16)
        box = pick_box(n, ho, wo, rows=rows, multiple_of=16)
        P = box[0] * box[1] * box[2]
        iters = (wo // box[0]) * (ho // box[1]) * -(-n // box[2])
    stages = min(8, (budget - _WG_SMEM_EXTRA) // (chunks * P * 128))
    combos = -(-cout // 128) * R * (cb // cb_per_group)
    cap = max_ctas if max_ctas > 0 else sm_count
    # one wave of units: every extra pixel chunk costs a full accumulator flush of fp32 atomics
    pc = min(max(px_chunks if px_chunks > 0 else cap // combos, 1), iters)
    per_chunk = -(-iters // pc)
    pc = -(-iters // per_chunk)
    units = pc * combos
    return WgradTiling(box, cb_per_group, G, stages, pc, units, min(units, cap))


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


def _conv_plan(views: List[torch.Tensor], weight: torch.Tensor, out: torch.Tensor, tap_map: List[int],
               tap_dw: List[int], tap_dh: List[int], flat: bool, stats_mode: int, max_ctas: int, **epilogue):
    """Plans one implicit GEMM writing ``out`` and builds its launchable binding: (pixel box, plan).  ``epilogue``: the
    tensors of ``stats_mode``, as the binding names them."""
    N, Ho, Wo, cout = out.shape
    t = plan_conv(grid=(N, Ho, Wo), view_widths=[v.shape[2] for v in views], cin=views[0].shape[3], cout=cout,
                  tap_map=tap_map, tap_dw=tap_dw, tap_dh=tap_dh, flat=flat, stats_mode=stats_mode, max_ctas=max_ctas,
                  sm_count=sm_count(), switches=conv_switches())
    bw, bh, bn = t.box
    plan = _build.load("_b200_conv").ConvPlan(
        views, weight, out, tap_map, tap_dw, tap_dh, bw=bw, bh=bh, bn=bn, block_n=t.block_n,
        resident_filter=t.resident_filter, halo=t.halo, grid=t.grid, **epilogue)
    _plans.add(plan)
    return t.box, plan


class ConvForward:
    """y = conv(x, w) [+ per-channel sum / sum-of-squares of y for BatchNorm] on the tensor cores.

    ``w`` is the bf16 filter in kernel layout ``[R*S*Cout, Cin]`` (tap-major)."""

    def __init__(self, x: torch.Tensor, w: torch.Tensor, y: torch.Tensor, R: int, S: int, stride: int = 1,
                 pad: int = 0, stat_sum: Optional[torch.Tensor] = None, stat_sqsum: Optional[torch.Tensor] = None,
                 max_ctas: int = 0, epilogue=None):
        """``epilogue=(scale, shift, act, residual)`` (inference): y = act(conv(x, w) * scale[c] + shift[c] [+ residual])
        with act in {'none', 'relu', 'relu6'} computed in the GEMM epilogue (folded BatchNorm); the residual (a tensor of
        y's shape) needs a dense 1x1 stride-1 convolution.  Mutually exclusive with the statistics outputs."""
        taps = make_taps(x, R, S, stride, pad)
        flat = (R == 1 and S == 1 and stride == 1 and pad == 0 and x.is_contiguous() and y.is_contiguous())
        if epilogue is not None:
            if stat_sum is not None:
                raise ValueError("epilogue and statistics outputs are mutually exclusive")
            scale, shift, act, residual = epilogue
            if residual is not None and not flat:
                raise ValueError("an epilogue residual needs a dense 1x1 stride-1 convolution")
            stats_mode = 4
            outputs = dict(add_src=residual, ep_scale=scale, ep_shift=shift,
                           ep_act={"none": 0, "relu": 1, "relu6": 2}[act])
        else:
            stats_mode = 0 if stat_sum is None else 1
            outputs = dict(stat_sum=stat_sum, stat_sqsum=stat_sqsum)
        self.box, self.plan = _conv_plan(taps.views, w, y, taps.tap_map, taps.tap_dw, taps.tap_dh, flat, stats_mode,
                                         max_ctas, **outputs)

    def run(self) -> None:
        self.plan.run()


class ConvDgrad:
    """dx = conv_transpose(dy, w) for the same geometry, as one or more forward-style implicit GEMMs.

    ``w_master`` is the fp32 (or bf16) filter ``[R*S, Cout, Cin]``; the transposed/rotated bf16 copies the kernel
    needs are (re)built by :meth:`refresh_weights` (cheap: filters are tiny next to activations)."""

    @staticmethod
    def parity_parts(R: int, S: int, stride: int, pad: int):
        """The output-parity classes a dgrad is made of, in plan order: ((ph, pw), filter-tap indices, tap offsets dw,
        dh) with dx[stride*i + ph, stride*j + pw] = sum over the class's taps of dy[i + dh, j + dw] w[tap].  Stride 1 is
        one class of every tap (the forward conv with the taps reversed); a stride-2 class may have no taps."""
        parts = []
        for ph in range(stride):
            for pw in range(stride):
                idx, dw, dh = [], [], []
                for r in range(R):
                    for s in range(S):
                        oh, ow = r - pad, s - pad
                        if oh % stride == ph and ow % stride == pw:
                            idx.append(r * S + s)
                            dh.append(-((oh - ph) // stride))
                            dw.append(-((ow - pw) // stride))
                parts.append(((ph, pw), idx, dw, dh))
        return parts

    @staticmethod
    def part_taps(R: int, S: int, stride: int, pad: int) -> List[List[int]]:
        """Filter-tap index lists of the GEMMs a dgrad is made of, in plan order: one list per non-empty output-parity
        class.  (Lets an owner lay all weight copies out in one buffer.)"""
        return [idx for _, idx, _, _ in ConvDgrad.parity_parts(R, S, stride, pad) if idx]

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
        self.R, self.S, self.stride, self.pad = R, S, stride, pad
        self.fused_bwd_stats = bwd_stats is not None
        self.block_grad = block_grad is not None
        self.w_master = w_master
        if wbufs is not None:
            assert wbuf is None and len(wbufs) == len(self.part_taps(R, S, stride, pad))
        self.external_wbuf = wbuf is not None or wbufs is not None  # owner refreshes them (one batched kernel for all layers)
        taps_total, cout, cin = w_master.shape
        assert taps_total == R * S
        self.parts = []  # (plan, weight buffer, tap index list)
        self.boxes = []  # pixel box (bw, bh, bn) of each part; (0, 0, 0) = flat
        self._idx_dev = {}
        self.needs_zero = False
        self.dx = dx
        flat = (R == 1 and S == 1 and stride == 1 and pad == 0 and dy.is_contiguous() and dx.is_contiguous())
        stats_mode, outputs = 0, {}
        if block_grad is not None:
            if not flat:
                raise ValueError("block_grad needs a dense 1x1 stride-1 convolution")
            skip, mask, y3, s_dz, s_dzy = block_grad
            stats_mode, outputs = 3, dict(stat_sum=s_dz, stat_sqsum=s_dzy, bwd_y=y3, add_src=skip, relu_mask=mask)
        elif bwd_stats is not None:
            y, sc, sh, s_dz, s_dzy = bwd_stats
            stats_mode, outputs = 2, dict(stat_sum=s_dz, stat_sqsum=s_dzy, bwd_y=y, bn_scale=sc, bn_shift=sh)
        for (ph, pw), idx, dw, dh in self.parity_parts(R, S, stride, pad):
            if not idx:
                self.needs_zero = True
                continue
            if wbufs is not None:
                buf = wbufs[len(self.parts)]
            elif wbuf is not None and stride == 1:
                buf = wbuf
            else:
                buf = torch.empty(len(idx) * cin, cout, dtype=torch.bfloat16, device=dy.device)
                if stride != 1:
                    self._idx_dev[tuple(idx)] = torch.tensor(idx, device=dy.device, dtype=torch.long)
            buf = buf.view(len(idx) * cin, cout)
            box, plan = _conv_plan([dy], buf, dx[:, ph::stride, pw::stride, :], [0] * len(idx), dw, dh, flat,
                                   stats_mode, max_ctas, **outputs)
            self.parts.append((plan, buf, idx))
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
        taps = make_taps(x, R, S, stride, pad)
        N, Ho, Wo, cout = dy.shape
        flat = (R == 1 and S == 1 and stride == 1 and pad == 0 and x.is_contiguous() and dy.is_contiguous()
                and (N * Ho * Wo) % 64 == 0)
        t = plan_wgrad(grid=(N, Ho, Wo), cin=x.shape[3], cout=cout, R=R, S=S, flat=flat, px_chunks=px_chunks,
                       max_ctas=max_ctas, smem_budget=smem_budget, sm_count=sm_count())
        self.box = t.box
        bw, bh, bn = t.box
        self.plan = _build.load("_b200_conv").WgradPlan(
            dy, taps.views, dw, R, S, taps.tap_map, taps.tap_dw, taps.tap_dh, bw=bw, bh=bh, bn=bn,
            cb_per_group=t.cb_per_group, stages=t.stages, px_chunks=t.px_chunks, grid=t.grid)
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
