"""Bit-exact checks of the wgmma convolution kernels (csrc/conv_igemm.cuh, csrc/conv_wgrad.cu, csrc/stem.cu).

The data make the right answer exact, so any indexing, tap, swizzle, tile or epilogue mistake is a hard mismatch:

* activations, gradients and filters are ternary {-1, 0, 1} (forward / dgrad filters also carry a few +-32 or +-16
  entries, so that outputs exceed 256 and bf16 rounding is exercised); every product is exact and every forward / dgrad sum is an
  integer far below 2^24, so the expected bf16 output is exactly ``ref.float().to(torch.bfloat16)`` (round to nearest
  even, as ``__floats2bfloat162_rn`` in the kernels);
* stem pixels are uint8 in [126, 130] with ``mul=1, add=-128``: normalised inputs are integers in [-2, 2];
* references are float64 convolutions, ``.round()``-ed (the true value is an integer; rounding removes any error of a
  non-exact cuDNN algorithm);
* the inference epilogue uses power-of-two scales and shifts that are multiples of 0.25 (``fmaf`` is exact), chosen so
  that exact zeros and exact 6.0 values occur; the fused BatchNorm-backward mask uses ``y*scale + shift == 0`` for a
  large share of the elements (the ``> 0`` edge).

Every output sits in a larger allocation with NaN guard bands before and after it and is prefilled with NaN (dense
outputs) or zero (accumulated outputs); the guards must come back bit-identical.

Each case asserts which kernel variant it runs (BLOCK_N, statistics mode, resident filter, halo, grid) and sets
``max_ctas`` explicitly, so the variant does not depend on the GPU's SM count; the last test checks that the cases cover
every dispatch branch of ``conv_igemm.cu``, each at one tile per CTA and at several tiles per CTA.
"""
from __future__ import annotations

from dataclasses import dataclass

import pytest
import torch

from exact_util import DEV, Guarded, check_equal, check_sum, pack_mask, tern, to_bf16_exact

pytestmark = pytest.mark.gpu


def _C():
    import b200ddl  # noqa: F401
    from b200ddl.ops import conv as C

    return C


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def locator(box, block_n, H, W, stride2=False):
    """(n, h, w, c) of an NHWC output of H x W pixels -> the M-tile, row in the tile and warpgroup that wrote it
    (box (0, 0, 0): flat mode; stride2: a stride-2 dgrad, whose parts each write one parity class)."""
    bw, bh, bn = box

    def loc(n, h, w, c):
        part, Hv, Wv = "", H, W
        if stride2:
            part, h, w, Hv, Wv = f"parity=({h % 2},{w % 2}) ", h // 2, w // 2, H // 2, W // 2
        if bw == 0:
            m_tile, row = divmod((n * Hv + h) * Wv + w, 128)
        else:
            m_tile = ((n // bn) * (Hv // bh) + h // bh) * (Wv // bw) + w // bw
            row = ((n % bn) * bh + h % bh) * bw + w % bw
        return f"[{part}m_tile={m_tile} row={row} warpgroup={row // 64} n_block={c // block_n}]"

    return loc


# ----------------------------------------------------------------------------------------------- conv_igemm cases
@dataclass(frozen=True)
class ConvCase:
    id: str
    op: str          # "fwd" | "dgrad" | "block_grad"
    N: int
    H: int
    W: int
    cin: int         # forward input channels (dgrad: channels of dx)
    cout: int        # forward output channels (dgrad: channels of dy)
    R: int
    stride: int
    stats: int       # expected kStats: 0 plain, 1 forward statistics, 2 fused bwd reduction, 3 block gradient, 4 epilogue
    block_n: int
    res: int = 0
    halo: int = 0
    max_ctas: int = 132
    multi: bool = False          # True: >= 3 tiles per CTA; False: one tile per CTA
    env: tuple = ()
    act: str = "relu"            # kStats 4
    residual: bool = False       # kStats 4 (flat plans)
    compact: bool = False        # kStats 3: skip gradient on the stride-2 sub-grid
    hi: int = 32                 # magnitude of the large filter entries (kStats 4: always 1)
    box: tuple = ()              # expected pixel box (bw, bh, bn) of every part, when the case is about its geometry
    regimes: tuple = ()          # kStats 1: expected regime ("exact" / "bounded") of sum y and of sum y^2


_NORES = (("B200DDL_NO_RESIDENT_FILTER", "1"),)
_NOHALO = (("B200DDL_NO_HALO", "1"),)
_BN64 = (("B200DDL_BLOCK_N", "64"),)
_BN128 = (("B200DDL_BLOCK_N", "128"),)

CONV_CASES = [
    # ---- BLOCK_N 128
    ConvCase("fwd_3x3s2_bn128_HneW", "fwd", 3, 16, 24, 128, 128, 3, 2, 0, 128, env=_BN128),
    ConvCase("fwd_3x3s2_bn128_HneW_multi", "fwd", 8, 32, 48, 128, 128, 3, 2, 0, 128, max_ctas=5, multi=True, env=_BN128),
    ConvCase("fwd_1x1s2_projection_overhang", "fwd", 5, 16, 16, 128, 256, 1, 2, 0, 128, env=_BN128, box=(8, 8, 2)),
    ConvCase("fwd_1x1_flat_bn128_stats_M900", "fwd", 1, 30, 30, 192, 256, 1, 1, 1, 128, env=_BN128, hi=16,
             regimes=("exact", "exact")),
    ConvCase("fwd_1x1_flat_bn128_stats_M900_multi", "fwd", 1, 30, 30, 192, 256, 1, 1, 1, 128, max_ctas=5, multi=True,
             env=_BN128, hi=16, regimes=("exact", "exact")),
    ConvCase("fwd_1x1_flat_bn128_stats_accumulate", "fwd", 4, 15, 15, 128, 256, 1, 1, 1, 128, max_ctas=4, multi=True,
             env=_BN128, hi=16, regimes=("exact", "exact")),
    ConvCase("dgrad_3x3_bn128_bwdstats_overhang", "dgrad", 5, 8, 8, 128, 64, 3, 1, 2, 128, env=_BN128, box=(8, 8, 2)),
    ConvCase("dgrad_3x3_bn128_bwdstats", "dgrad", 2, 8, 12, 128, 64, 3, 1, 2, 128, env=_BN128),
    ConvCase("dgrad_3x3_bn128_bwdstats_multi", "dgrad", 3, 12, 16, 128, 64, 3, 1, 2, 128, max_ctas=2, multi=True,
             env=_BN128),
    ConvCase("blockgrad_bn128_dense", "block_grad", 2, 14, 14, 256, 64, 1, 1, 3, 128, env=_BN128),
    ConvCase("blockgrad_bn128_dense_multi", "block_grad", 2, 14, 14, 256, 64, 1, 1, 3, 128, max_ctas=3, multi=True,
             env=_BN128),
    ConvCase("fwd_1x1_flat_bn128_epilogue_residual_relu6", "fwd", 2, 14, 14, 128, 128, 1, 1, 4, 128, act="relu6",
             residual=True, env=_BN128),
    ConvCase("fwd_3x3_bn128_epilogue_relu_multi", "fwd", 2, 12, 20, 64, 256, 3, 1, 4, 128, act="relu", max_ctas=2,
             multi=True, env=_BN128),
    # ---- BLOCK_N 64, filter streamed through the stages
    ConvCase("fwd_1x1_flat_bn64_cin960_cout192", "fwd", 2, 10, 10, 960, 192, 1, 1, 0, 64),
    ConvCase("fwd_3x3_bn64_cin192_cout192_multi", "fwd", 2, 10, 14, 192, 192, 3, 1, 0, 64, max_ctas=5, multi=True),
    ConvCase("fwd_3x3_bn64_stats_flush_every_tile", "fwd", 4, 16, 16, 64, 128, 3, 1, 1, 64, max_ctas=5, multi=True,
             env=_BN64, regimes=("exact", "bounded")),
    ConvCase("fwd_3x3_bn64_stats_accumulate", "fwd", 4, 16, 16, 64, 128, 3, 1, 1, 64, max_ctas=4, multi=True,
             env=_BN64, regimes=("exact", "bounded")),
    ConvCase("fwd_1x1_flat_bn64_stats_cout192", "fwd", 1, 20, 20, 192, 192, 1, 1, 1, 64, hi=16,
             regimes=("exact", "exact")),
    # 5 images in boxes of 2: the third box's second image lies past N (zero-filled on load, clipped on store)
    ConvCase("fwd_3x3_bn64_stats_overhang_multi", "fwd", 5, 8, 8, 128, 128, 3, 1, 1, 64, max_ctas=2, multi=True,
             env=_BN64, box=(8, 8, 2), regimes=("exact", "bounded")),
    ConvCase("dgrad_3x3_bn64_bwdstats_cin192", "dgrad", 2, 8, 10, 192, 128, 3, 1, 2, 64),
    ConvCase("dgrad_3x3_bn64_bwdstats_multi", "dgrad", 2, 14, 16, 128, 64, 3, 1, 2, 64, max_ctas=3, multi=True,
             env=_BN64),
    ConvCase("blockgrad_bn64_compact_cin192", "block_grad", 2, 12, 12, 192, 128, 1, 1, 3, 64, compact=True),
    ConvCase("blockgrad_bn64_compact_multi", "block_grad", 3, 14, 14, 128, 64, 1, 1, 3, 64, compact=True, max_ctas=3,
             multi=True, env=_BN64),
    ConvCase("fwd_3x3_bn64_epilogue_relu6", "fwd", 2, 6, 10, 64, 192, 3, 1, 4, 64, act="relu6"),
    ConvCase("fwd_1x1_flat_bn64_epilogue_residual_multi", "fwd", 2, 20, 20, 128, 192, 1, 1, 4, 64, act="relu",
             residual=True, max_ctas=5, multi=True),
    ConvCase("dgrad_1x1_flat_bn64_cin960", "dgrad", 2, 6, 10, 960, 192, 1, 1, 0, 64),
    # ---- resident filter (BLOCK_N 64, one N-block)
    ConvCase("fwd_3x3s2_resident", "fwd", 2, 12, 20, 64, 64, 3, 2, 0, 64, res=1),
    ConvCase("dgrad_3x3s2_resident_multi", "dgrad", 8, 32, 40, 64, 128, 3, 2, 0, 64, res=1, max_ctas=5, multi=True),
    ConvCase("dgrad_1x1s2_resident_needs_zero", "dgrad", 2, 12, 16, 64, 256, 1, 2, 0, 64, res=1),
    ConvCase("fwd_1x1_flat_resident_stats_M338", "fwd", 2, 13, 13, 512, 64, 1, 1, 1, 64, res=1, hi=16,
             regimes=("exact", "exact")),
    ConvCase("fwd_3x3_resident_stats_multi", "fwd", 8, 20, 12, 64, 64, 3, 1, 1, 64, res=1, max_ctas=5, multi=True,
             env=_NOHALO, regimes=("exact", "bounded")),
    ConvCase("dgrad_1x1_flat_resident_bwdstats", "dgrad", 2, 10, 10, 64, 256, 1, 1, 2, 64, res=1),
    ConvCase("dgrad_1x1_flat_resident_bwdstats_multi", "dgrad", 4, 20, 20, 64, 192, 1, 1, 2, 64, res=1, max_ctas=5,
             multi=True),
    ConvCase("fwd_1x1_flat_resident_epilogue_residual", "fwd", 2, 12, 12, 128, 64, 1, 1, 4, 64, res=1, act="relu6",
             residual=True),
    ConvCase("fwd_3x3_resident_epilogue_multi", "fwd", 8, 16, 12, 64, 64, 3, 1, 4, 64, res=1, act="relu", max_ctas=5,
             multi=True, env=_NOHALO),
    # ---- halo (resident filter, 3x3 stride 1, full-width boxes)
    ConvCase("fwd_3x3_halo_w56", "fwd", 2, 8, 56, 64, 64, 3, 1, 0, 64, res=1, halo=1),
    ConvCase("fwd_3x3_halo_w56_multi", "fwd", 4, 8, 56, 64, 64, 3, 1, 0, 64, res=1, halo=1, max_ctas=5, multi=True),
    ConvCase("fwd_3x3_halo_w24_stats", "fwd", 2, 12, 24, 64, 64, 3, 1, 1, 64, res=1, halo=1,
             regimes=("exact", "bounded")),
    ConvCase("fwd_3x3_halo_w24_stats_multi", "fwd", 5, 12, 24, 64, 64, 3, 1, 1, 64, res=1, halo=1, max_ctas=5,
             multi=True, regimes=("exact", "bounded")),
    ConvCase("dgrad_3x3_halo_w56_bwdstats", "dgrad", 1, 6, 56, 64, 64, 3, 1, 2, 64, res=1, halo=1),
    ConvCase("dgrad_3x3_halo_w24_bwdstats_multi", "dgrad", 4, 16, 24, 64, 64, 3, 1, 2, 64, res=1, halo=1, max_ctas=5,
             multi=True),
    ConvCase("fwd_3x3_halo_w24_epilogue_relu6", "fwd", 1, 8, 24, 64, 64, 3, 1, 4, 64, res=1, halo=1, act="relu6"),
    ConvCase("fwd_3x3_halo_w56_epilogue_multi", "fwd", 3, 10, 56, 64, 64, 3, 1, 4, 64, res=1, halo=1, act="relu",
             max_ctas=5, multi=True),
    # ---- the one batch-256 forward case (sum y^2 far above 2^24: the bounded regime)
    ConvCase("fwd_1x1_flat_bn128_stats_b256", "fwd", 256, 14, 14, 256, 256, 1, 1, 1, 128, multi=True, env=_BN128,
             regimes=("exact", "bounded")),
]


def _setup(case: ConvCase, monkeypatch, seed=0):
    """Builds the op of a case (plans read the A/B switches at construction) and its inputs."""
    C = _C()
    for k in ("B200DDL_BLOCK_N", "B200DDL_NO_RESIDENT_FILTER", "B200DDL_NO_HALO"):
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env:
        monkeypatch.setenv(k, v)
    g = torch.Generator(device=DEV).manual_seed(seed)
    N, H, W, R, s = case.N, case.H, case.W, case.R, case.stride
    pad = R // 2
    Ho, Wo = (H + 2 * pad - R) // s + 1, (W + 2 * pad - R) // s + 1
    d = {"g": g, "pad": pad, "Ho": Ho, "Wo": Wo}
    if case.op == "fwd":
        x = tern((N, H, W, case.cin), g).to(torch.bfloat16)
        w = tern((R * R, case.cout, case.cin), g, hi=1 if case.stats == 4 else case.hi)
        out = Guarded((N, Ho, Wo, case.cout), torch.bfloat16, float("nan"))
        d.update(x=x, w=w, out=out)
        kw = {}
        if case.stats == 1:
            d["ssum"] = Guarded((case.cout,), torch.float32, 0.0, guard=64)
            d["ssq"] = Guarded((case.cout,), torch.float32, 0.0, guard=64)
            kw = dict(stat_sum=d["ssum"].t, stat_sqsum=d["ssq"].t)
        elif case.stats == 4:
            sc = 2.0 ** torch.randint(-2, 2, (case.cout,), device=DEV, generator=g).float()
            sh = torch.randint(-8, 33, (case.cout,), device=DEV, generator=g).float() * 0.25
            # half the channels are shifted past 256, where the quarter steps and the integer part together need more
            # than bf16's 8 significant bits (so rounding is exercised); the others hit the ReLU / ReLU6 edges
            far = torch.rand(case.cout, device=DEV, generator=g) < 0.5
            sh = sh + far.float() * 256.0 * torch.randint(1, 4, (case.cout,), device=DEV, generator=g).float()
            res = tern((N, Ho, Wo, case.cout), g).to(torch.bfloat16) if case.residual else None
            d.update(sc=sc, sh=sh, res=res)
            kw = dict(epilogue=(sc, sh, case.act, res))
        wk = w.to(torch.bfloat16).reshape(R * R * case.cout, case.cin).contiguous()
        op = C.ConvForward(x, wk, out.t, R, R, s, pad, max_ctas=case.max_ctas, **kw)
        d["plans"], d["boxes"] = [op.plan], [op.box]
    else:
        dy = tern((N, Ho, Wo, case.cout), g).to(torch.bfloat16)
        w = tern((R * R, case.cout, case.cin), g, hi=case.hi)
        out = Guarded((N, H, W, case.cin), torch.bfloat16, float("nan"))
        d.update(dy=dy, w=w, out=out)
        kw = {}
        if case.stats == 2:
            y = tern((N, H, W, case.cin), g, density=0.8).to(torch.bfloat16)
            sc = 2.0 ** torch.randint(-1, 2, (case.cin,), device=DEV, generator=g).float()
            # shift in {-sc, 0, sc, sc/2}: y*sc + shift == 0 exactly at y == 1, 0, -1 (and nowhere for sc/2)
            frac = torch.tensor([-1.0, 0.0, 1.0, 0.5], device=DEV)
            sh = sc * frac[torch.randint(0, 4, (case.cin,), device=DEV, generator=g)]
            d["s_dz"] = Guarded((case.cin,), torch.float32, 0.0, guard=64)
            d["s_dzy"] = Guarded((case.cin,), torch.float32, 0.0, guard=64)
            d.update(y=y, sc=sc, sh=sh)
            kw = dict(bwd_stats=(y, sc, sh, d["s_dz"].t, d["s_dzy"].t))
        elif case.stats == 3:
            skip = tern((N, H // 2, W // 2, case.cin) if case.compact else (N, H, W, case.cin), g, hi=32).to(torch.bfloat16)
            y3 = tern((N, H, W, case.cin), g).to(torch.bfloat16)
            mbool = torch.rand(N * H * W, case.cin, device=DEV, generator=g) > 0.4
            d["s_dz"] = Guarded((case.cin,), torch.float32, 0.0, guard=64)
            d["s_dzy"] = Guarded((case.cin,), torch.float32, 0.0, guard=64)
            d.update(skip=skip, y3=y3, mbool=mbool)
            kw = dict(block_grad=(skip, pack_mask(mbool), y3, d["s_dz"].t, d["s_dzy"].t))
        op = C.ConvDgrad(dy, w, out.t, R, R, s, pad, max_ctas=case.max_ctas, **kw)
        d["plans"], d["boxes"] = [p for p, _, _ in op.parts], op.boxes
    d["op"] = op
    return d


def _variant(p):
    return (p.block_n, p.stats_mode, p.resident_filter, p.halo)


def _assert_plan(case: ConvCase, plans, boxes):
    if case.box:
        assert boxes and all(tuple(b) == case.box for b in boxes), f"{case.id}: pixel boxes {boxes}"
    for p in plans:
        assert _variant(p) == (case.block_n, case.stats, case.res, case.halo), (
            f"{case.id}: plan runs (block_n, stats_mode, resident_filter, halo) = {_variant(p)}")
        assert p.grid == min(p.tiles, case.max_ctas), (p.grid, p.tiles, case.max_ctas)
        per_cta = -(-p.tiles // p.grid)
        if case.multi:
            assert per_cta >= 3, f"{case.id}: {p.tiles} tiles on {p.grid} CTAs"
        else:
            assert per_cta == 1, f"{case.id}: {p.tiles} tiles on {p.grid} CTAs"


def _stat_depth(plans):
    # additions on a term's path: 15 in the thread's 16-row partial, one per tile in the CTA's register accumulator,
    # then one per atomic into the channel (8 row groups per flush, at most one flush per tile)
    return 16 + 9 * sum(p.tiles for p in plans)


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: c.id)
def test_conv_igemm_exact(case: ConvCase, monkeypatch):
    d = _setup(case, monkeypatch)
    plans = d["plans"]
    _assert_plan(case, plans, d["boxes"])
    d["op"].run()
    torch.cuda.synchronize()
    C = _C()
    N, H, W, R, s, pad = case.N, case.H, case.W, case.R, case.stride, d["pad"]
    out = d["out"]
    out.check_guards(f"{case.id} output")
    wt = C.weight_from_kernel_layout(d["w"].double(), R, R)
    if case.op == "fwd":
        acc = nhwc(torch.nn.functional.conv2d(nchw(d["x"]), wt, stride=s, padding=pad)).round()
        loc = locator(d["boxes"][0], case.block_n, d["Ho"], d["Wo"])
    else:
        acc = nhwc(torch.nn.grad.conv2d_input((N, case.cin, H, W), wt, nchw(d["dy"]), stride=s, padding=pad)).round()
        loc = locator(d["boxes"][0], case.block_n, H, W, stride2=s == 2)
    assert float(acc.abs().max()) < 2.0 ** 24
    if case.stats == 4:
        pre = acc * d["sc"].double() + d["sh"].double()
        if d["res"] is not None:
            pre = pre + d["res"].double()
        exp = pre.clamp(min=0.0)
        if case.act == "relu6":
            # ReLU6 outputs lie on a 0.25 grid in [0, 6], exact in bf16: these cases check the clamp, not the rounding
            exp = exp.clamp(max=6.0)
            assert int((pre == 6.0).sum()) > 0, "no exact 6.0 before ReLU6"
        assert int((pre == 0.0).sum()) > 0, "no exact zero before the ReLU"
        check_equal(f"{case.id} output", out.t, to_bf16_exact(exp), loc)
        return
    if case.stats == 3:
        full = d["skip"].double()
        if case.compact:
            full = torch.zeros(N, H, W, case.cin, dtype=torch.float64, device=DEV)
            full[:, 0::2, 0::2, :] = d["skip"].double()
        exp = to_bf16_exact((acc + full) * d["mbool"].view(N, H, W, case.cin))
    else:
        exp = to_bf16_exact(acc)
    check_equal(f"{case.id} output", out.t, exp, loc)
    depth = _stat_depth(plans)
    e = exp.double().reshape(-1, exp.shape[-1])
    if case.stats == 1:
        d["ssum"].check_guards(f"{case.id} sum")
        d["ssq"].check_guards(f"{case.id} sum of squares")
        regimes = (check_sum(f"{case.id} sum y", d["ssum"].t, e.sum(0), e.abs().sum(0), depth),
                   check_sum(f"{case.id} sum y^2", d["ssq"].t, (e * e).sum(0), (e * e).sum(0), depth))
        assert regimes == case.regimes, f"{case.id}: sums checked in regimes {regimes}, the case expects {case.regimes}"
    elif case.stats in (2, 3):
        d["s_dz"].check_guards(f"{case.id} sum dz")
        d["s_dzy"].check_guards(f"{case.id} sum dz*y")
        if case.stats == 2:
            y = d["y"].double().reshape(-1, case.cin)
            mask = (y * d["sc"].double() + d["sh"].double()) > 0
            edge = (y * d["sc"].double() + d["sh"].double()) == 0
            assert float(edge.double().mean()) > 0.1, "too few elements on the mask edge y*scale + shift == 0"
            dz = e * mask
        else:
            y = d["y3"].double().reshape(-1, case.cin)
            dz = e
        # y is ternary, so sum |dz*y| <= sum |dz|: both sums are in the exact regime
        assert check_sum(f"{case.id} sum dz", d["s_dz"].t, dz.sum(0), dz.abs().sum(0), depth) == "exact"
        assert check_sum(f"{case.id} sum dz*y", d["s_dzy"].t, (dz * y).sum(0), (dz * y).abs().sum(0), depth) == "exact"


def test_conv_igemm_variant_coverage(monkeypatch):
    """The cases above reach every (BLOCK_N, kStats, resident filter, halo) branch conv_igemm.cu dispatches, each at one
    tile per CTA and at >= 3 tiles per CTA; a new branch without a case fails here."""
    branches = set()
    for bn in (64, 128):
        for st in range(5):
            branches.add((bn, st, 0, 0))
    for st in (0, 1, 2, 4):
        branches.add((64, st, 1, 0))
        branches.add((64, st, 1, 1))
    assert len(branches) == 18
    seen = {}
    for case in CONV_CASES:
        with monkeypatch.context() as m:
            d = _setup(case, m)
        for p in d["plans"]:
            per_cta = -(-p.tiles // p.grid)
            seen.setdefault(_variant(p), set()).add("multi" if per_cta >= 3 else "single" if per_cta == 1 else "two")
        del d
    assert set(seen) == branches, sorted(set(seen) ^ branches)
    missing = {v: s for v, s in seen.items() if not {"single", "multi"} <= s}
    assert not missing, missing


# ------------------------------------------------------------------------------------------------ last-CTA tails
TAIL_CASES = (ConvCase("tail_fwd", "fwd", 2, 16, 16, 64, 128, 1, 1, 1, 64, max_ctas=3, multi=True, env=_BN64),
              ConvCase("tail_bwd", "dgrad", 2, 16, 16, 128, 64, 3, 1, 2, 64, max_ctas=5, multi=True, env=_BN64))


def test_last_cta_tails_exact_sums(monkeypatch):
    """BatchNorm finalize / backward coefficients from the last CTA at max_ctas 3 / 5, run twice: the outputs equal the
    stand-alone kernels fed the exact sums, and the sums and the ticket counter are zero again after each run."""
    e = _ops()
    fwd, bwd = TAIL_CASES
    d = _setup(fwd, monkeypatch, seed=5)
    plan, cout = d["plans"][0], fwd.cout
    g = torch.Generator(device=DEV).manual_seed(6)
    gamma = torch.rand(cout, device=DEV, generator=g) + 0.5
    beta = torch.randn(cout, device=DEV, generator=g)
    rm, rv = torch.zeros(cout, device=DEV), torch.ones(cout, device=DEV)
    outs = [torch.empty(cout, device=DEV) for _ in range(4)]
    ctr = torch.zeros(1, device=DEV, dtype=torch.int32)
    cnt = float(fwd.N * fwd.H * fwd.W)
    plan.set_bn_finalize(ctr, gamma, beta, rm, rv, *outs, cnt, 0.1, 1e-5)
    wt = _C().weight_from_kernel_layout(d["w"].double(), 1, 1)
    y = to_bf16_exact(nhwc(torch.nn.functional.conv2d(nchw(d["x"]), wt)).round()).double().reshape(-1, cout)
    s_ref, q_ref = y.sum(0), (y * y).sum(0)
    assert float((y * y).sum(0).max()) < 2 ** 24, "tail check needs the exact regime"
    rm2, rv2 = torch.zeros(cout, device=DEV), torch.ones(cout, device=DEV)
    ref = [torch.empty(cout, device=DEV) for _ in range(4)]
    for rep in range(2):
        d["op"].run()
        torch.cuda.synchronize()
        assert float(d["ssum"].t.abs().max() + d["ssq"].t.abs().max()) == 0.0 and int(ctr.item()) == 0, rep
        e.bn_finalize(s_ref.float(), q_ref.float(), cnt, gamma, beta, rm2, rv2, 0.1, 1e-5, *ref, True)
    torch.cuda.synchronize()
    for nm, a, b in zip(("mean", "invstd", "scale", "shift", "running_mean", "running_var"), outs + [rm, rv], ref + [rm2, rv2]):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7, msg=lambda m, nm=nm: f"finalize {nm}: {m}")

    d = _setup(bwd, monkeypatch, seed=7)
    cin = bwd.cin
    gam = torch.rand(cin, device=DEV, generator=g) + 0.5
    mean = torch.randint(-4, 5, (cin,), device=DEV, generator=g).float() * 0.125
    invstd = torch.rand(cin, device=DEV, generator=g) + 0.5
    o = [torch.empty(cin, device=DEV) for _ in range(5)]
    ctr2 = torch.zeros(1, device=DEV, dtype=torch.int32)
    cnt2 = float(bwd.N * bwd.H * bwd.W)
    d["plans"][0].set_bn_bwd_coeffs(ctr2, gam, mean, invstd, cnt2, *o)
    wt = _C().weight_from_kernel_layout(d["w"].double(), 3, 3)
    gx = to_bf16_exact(nhwc(torch.nn.grad.conv2d_input((bwd.N, cin, bwd.H, bwd.W), wt, nchw(d["dy"]), padding=1)).round())
    gx = gx.double().reshape(-1, cin)
    yv = d["y"].double().reshape(-1, cin)
    dz = gx * ((yv * d["sc"].double() + d["sh"].double()) > 0)
    sdz, sdzy = dz.sum(0), (dz * yv).sum(0)
    assert float(dz.abs().sum(0).max()) < 2 ** 24 and float((dz * yv).abs().sum(0).max()) < 2 ** 24
    r = [torch.empty(cin, device=DEV) for _ in range(5)]
    for rep in range(2):
        d["op"].run()
        torch.cuda.synchronize()
        assert float(d["s_dz"].t.abs().max() + d["s_dzy"].t.abs().max()) == 0.0 and int(ctr2.item()) == 0, rep
    e.bn_bwd_coeffs(sdz.float(), sdzy.float(), gam, mean, invstd, cnt2, *r)
    torch.cuda.synchronize()
    for nm, a, b in zip(("dgamma", "dbeta", "cA", "cB", "cC"), o, r):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7, msg=lambda m, nm=nm: f"bwd coefficients {nm}: {m}")


# ----------------------------------------------------------------------------------------------------- wgrad cases
@dataclass(frozen=True)
class WgCase:
    id: str
    N: int
    H: int
    W: int
    cin: int
    cout: int
    R: int
    stride: int
    G: int
    mode: int            # 0 flat, 1 box
    px_chunks: int = 0
    max_ctas: int = 132
    smem_budget: int = 0
    stages: int = 0      # expected stage count (0: not asserted)
    several_units: bool = False   # max_ctas below the unit count: CTAs run several units


WG_CASES = [
    WgCase("1x1_cin64_cout64_flat", 2, 16, 16, 64, 64, 1, 1, G=1, mode=0),
    WgCase("1x1_cin128_cout128_box_M432_2stages", 3, 12, 12, 128, 128, 1, 1, G=2, mode=1, smem_budget=100000, stages=2),
    WgCase("1x1_cin192_cout256_flat_uneven_chunks", 2, 16, 16, 192, 256, 1, 1, G=3, mode=0, px_chunks=3, max_ctas=5,
           several_units=True),
    WgCase("1x1_cin256_cout64_box_M200", 2, 10, 10, 256, 64, 1, 1, G=4, mode=1),
    WgCase("1x1_cin256_cout256_flat_full_budget", 2, 16, 16, 256, 256, 1, 1, G=4, mode=0, px_chunks=4, max_ctas=3,
           several_units=True),
    WgCase("1x1_cin960_cout128_flat", 1, 16, 16, 960, 128, 1, 1, G=3, mode=0, max_ctas=4, several_units=True),
    WgCase("3x3_cin64_cout128_box", 2, 12, 20, 64, 128, 3, 1, G=3, mode=1, px_chunks=2, max_ctas=4,
           several_units=True),
    WgCase("3x3s2_cin128_cout64_box", 2, 16, 24, 128, 64, 3, 2, G=3, mode=1),
    WgCase("3x3_cin64_cout64_box_2stages", 2, 12, 12, 64, 64, 3, 1, G=3, mode=1, smem_budget=100000, stages=2),
    # split-K over M = 802,816 pixels: 131 units of 96 blocks of 64 pixels, each flushed with fp32 atomics.  A unit's
    # wgmma accumulator only holds partial sums of at most 96 * 64 = 6,144 products of +-1; the large totals are formed
    # by the atomics.  Exact equality holds (measured on an H100 80GB HBM3 at 700 W), so the case is no looser than
    # the small ones; it does not show how the accumulator behaves with partial sums near 2^24.
    WgCase("1x1_cin64_cout64_flat_b256", 256, 56, 56, 64, 64, 1, 1, G=1, mode=0),
]


def _wgrad_op(case: WgCase):
    """Builds the op of a wgrad case and its inputs: (op, x, dy, guarded dw)."""
    C = _C()
    g = torch.Generator(device=DEV).manual_seed(3)
    N, H, W, R, s = case.N, case.H, case.W, case.R, case.stride
    pad = R // 2
    Ho, Wo = (H + 2 * pad - R) // s + 1, (W + 2 * pad - R) // s + 1
    x = tern((N, H, W, case.cin), g).to(torch.bfloat16)
    dy = tern((N, Ho, Wo, case.cout), g).to(torch.bfloat16)
    dw = Guarded((R * R * case.cout, case.cin), torch.float32, 0.0)
    op = C.ConvWgrad(dy, x, dw.t, R, R, s, pad, px_chunks=case.px_chunks, max_ctas=case.max_ctas,
                     smem_budget=case.smem_budget)
    return op, x, dy, dw


@pytest.mark.parametrize("case", WG_CASES, ids=lambda c: c.id)
def test_conv_wgrad_exact(case: WgCase):
    C = _C()
    R, s = case.R, case.stride
    pad = R // 2
    op, x, dy, dw = _wgrad_op(case)
    p = op.plan
    assert (p.G, p.mode) == (case.G, case.mode)
    assert p.grid == min(p.units, case.max_ctas)
    if case.stages:
        assert p.stages == case.stages
    if case.several_units:
        assert p.units > p.grid
    if case.px_chunks:
        assert p.px_chunks == case.px_chunks
    op.run()
    torch.cuda.synchronize()
    dw.check_guards(f"{case.id} dw")
    ref = torch.nn.grad.conv2d_weight(nchw(x), (case.cout, case.cin, R, R), nchw(dy), stride=s, padding=pad)
    ref_abs = torch.nn.grad.conv2d_weight(nchw(x).abs(), (case.cout, case.cin, R, R), nchw(dy).abs(), stride=s,
                                          padding=pad)
    ref = C.weight_to_kernel_layout(ref.round()).reshape(R * R * case.cout, case.cin)
    assert float(ref_abs.max()) < 2 ** 24, "exact regime expected"

    def loc(row, ci):
        tap, co = divmod(row, case.cout)
        return f"[tap={tap} co={co} co_block={co // 128} warpgroup={co % 128 // 64} ci_block={ci // 64}]"

    check_equal(f"{case.id} dw", dw.t, ref, loc)


# ------------------------------------------------------------------------------------------------------ stem cases
STEM_CASES = [
    # id, N, H, W, max_ctas
    ("wo32_default_ctas", 2, 64, 64, 0),
    ("wo40_HneW_ctas5", 2, 70, 80, 5),
    ("wo56_oddH", 1, 57, 112, 132),
    ("wo56_oddH_ctas5", 2, 33, 112, 5),
    ("wo112", 1, 224, 224, 132),
    ("wo112_HneW_ctas5", 2, 32, 224, 5),
    ("wo128_6tiles_on_5ctas", 1, 11, 256, 5),
]


@pytest.mark.parametrize("case", STEM_CASES, ids=lambda c: c[0])
def test_stem_exact(case):
    C = _C()
    name, N, H, W, max_ctas = case
    g = torch.Generator(device=DEV).manual_seed(11)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    x = torch.randint(126, 131, (N, H, W, 3), device=DEV, dtype=torch.uint8, generator=g)
    w = tern((49, 64, 3), g, hi=32)
    w16 = torch.zeros(64, 192, device=DEV, dtype=torch.bfloat16)
    C.pack_stem_weight(w, w16)
    y = Guarded((N, Ho, Wo, 64), torch.bfloat16, float("nan"))
    ssum = Guarded((64,), torch.float32, 0.0, guard=64)
    ssq = Guarded((64,), torch.float32, 0.0, guard=64)
    C.StemForward(x, w16, y.t, ssum.t, ssq.t, mul=1.0, add=-128.0, max_ctas=max_ctas).run()
    dy = tern((N, Ho, Wo, 64), g).to(torch.bfloat16)
    dw = Guarded((49 * 64 * 3,), torch.float32, 0.0)
    C.StemWgrad(x, dy, dw.t, mul=1.0, add=-128.0, max_ctas=max_ctas).run()
    torch.cuda.synchronize()
    for gd, nm in ((y, "y"), (ssum, "sum"), (ssq, "sum of squares"), (dw, "dw")):
        gd.check_guards(f"stem {name} {nm}")
    xin = nchw(x.double() - 128.0)
    wt = w.double().view(7, 7, 64, 3).permute(2, 3, 0, 1)
    exp = to_bf16_exact(nhwc(torch.nn.functional.conv2d(xin, wt, stride=2, padding=3)).round())
    check_equal(f"stem {name} y", y.t, exp,
                lambda n, h, ww, c: f"[tile={n * Ho + h} row={ww} warpgroup={ww // 64}]")
    e = exp.double().reshape(-1, 64)
    tiles = N * Ho
    grid = min(tiles, max_ctas or torch.cuda.get_device_properties(0).multi_processor_count)
    # additions on a term's path: <= 15 in a thread's row partial, 8 row groups x tiles shared-memory atomics, grid global
    depth = 16 + 8 * tiles + grid
    # every case: sum |y| stays below 2^24 (exact), sum y^2 is far above it (bounded)
    regimes = (check_sum(f"stem {name} sum y", ssum.t, e.sum(0), e.abs().sum(0), depth),
               check_sum(f"stem {name} sum y^2", ssq.t, (e * e).sum(0), (e * e).sum(0), depth))
    assert regimes == ("exact", "bounded"), regimes
    gref = torch.nn.grad.conv2d_weight(xin, (64, 3, 7, 7), nchw(dy), stride=2, padding=3)
    gabs = torch.nn.grad.conv2d_weight(xin.abs(), (64, 3, 7, 7), nchw(dy).abs(), stride=2, padding=3)
    assert float(gabs.max()) < 2 ** 24
    gref = gref.round().permute(2, 3, 0, 1).reshape(49, 64, 3)

    def loc(tap, co, c):
        return f"[tap=({tap // 7},{tap % 7}) co={co} k={tap * 3 + c}]"

    check_equal(f"stem {name} dw", dw.t.view(49, 64, 3), gref, loc)
