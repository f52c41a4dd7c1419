"""Bit-exact checks of the bandwidth-bound kernels: BatchNorm forward / backward, pooling, the stem tail, the classifier
head, the weight casts and the optimizers (csrc/elementwise.cu, head_stem.cu, optim.cu, mobilenet.cu).

The data make the right answer exact wherever the kernel's arithmetic allows it:

* bf16 inputs are small integers, with some values in 257..1200 so that bf16 round-to-nearest-even is exercised;
  scales, A / B coefficients and filter taps are powers of two or dyadic with few bits and shifts are multiples of 0.25,
  so every ``fmaf`` is exact and the expected bf16 is ``ref.float().to(torch.bfloat16)`` of a float64 reference;
* about a quarter of the elements have a pre-activation of exactly 0 (the ``> 0`` edge of every ReLU mask);
* per-channel sums of integer terms below 2^24 must be equal; above that, ``check_sum`` bounds them by the number of
  sequential fp32 additions a term passes;
* the build uses ``--use_fast_math``: ``rsqrtf``, ``__expf``, ``__logf``, ``1.f/x``, ``/`` and ``sqrtf`` are
  approximate and fp32 denormals flush to zero.  Where a kernel uses one of them the bound is derived from the CUDA
  Programming Guide's intrinsic accuracy table and the PTX ISA and stated at the test.  Where the compiler may contract
  ``a - b*c`` into an ``fmaf`` and the data do not make both forms exact, either result is accepted.

Outputs sit between NaN guard bands (0xA5 for uint8 masks and argmax indices) and are prefilled with the same poison;
a mismatch report names the element and the block / thread / row that wrote it.

The BatchNorm-apply / ReLU-mask contract these tests pin, bit for bit:

* forward: ``pre = fmaf(y, scale, shift) [+ res | + fmaf(res, res_scale, res_shift)]`` in fp32, ``out = bf16_rn(relu ?
  fmaxf(pre, 0) : pre)``, mask bit = ``pre > 0`` (a pre-activation of exactly 0 is masked out); no mask is written
  without ReLU;
* backward reduce: ``dz = (g1 [+ g2])`` in fp32, masked by the stored activation ``> 0`` (mode 1), the forward's bitmap
  (mode 4) or ``fmaf(y, scale, shift) > 0`` (mode 2, equal to the forward bitmap); the sums use the unrounded fp32 dz,
  the stored dz is its bf16 rounding;
* backward apply: ``dy = bf16_rn(fmaf(A, dz, fmaf(B, y, C)))`` with dz masked by ``fmaf(y, scale, shift) > 0`` when
  scale / shift are given.

NaN propagation is not covered: ``fmaxf`` turns a NaN pre-activation into 0 where ``torch.relu`` keeps it.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from exact_util import DEV, POISON_U8, U, Guarded, check_equal, check_sum, pack_mask, to_bf16_exact

pytestmark = pytest.mark.gpu

NAN = float("nan")
BF = torch.bfloat16
CAP = 132 * 16          # block cap of rows_grid / grid_for (elementwise.cu)
RED_CAP = 132 * 8       # block cap of col_reduce_kernel and of the optimizers
RCP_ULP = 2.0 ** -23    # rcp.approx.f32: at most 1 ulp (PTX ISA), i.e. relative 2^-23


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


@pytest.fixture
def set_unroll():
    """set_bn_rows_unroll, restored after the test."""
    e = _ops()
    old = e.get_bn_rows_unroll()
    yield e.set_bn_rows_unroll
    e.set_bn_rows_unroll(old)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, device=DEV, generator=g).double()


def with_large(v, g, frac=1 / 16):
    """v with a fraction of its elements replaced by +-(257..1200) rounded to bf16 (exercises the output rounding)."""
    big = ints(v.shape, 257, 1200, g) * (ints(v.shape, 0, 1, g) * 2 - 1)
    big = big.float().to(BF).double()
    return torch.where(torch.rand(v.shape, device=DEV, generator=g) < frac, big, v)


def pow2(shape, lo, hi, g):
    return 2.0 ** ints(shape, lo, hi, g)


def bf(v):
    t = v.float().to(BF)
    assert bool((t.double() == v).all()), "input not exact in bf16"
    return t


def f32(v):
    t = v.float()
    assert bool((t.double() == v).all()), "input not exact in fp32"
    return t


# ------------------------------------------------------------------------------------------------ launch geometry
def rows_geom(C):
    """(lanes, rows per block) of the column-resident kernels (bn_apply / bn_bwd_apply / col_reduce) at 256 threads."""
    lanes = min(C // 8, 256)
    return lanes, 256 // lanes


def rows_M(C, kind):
    """Row counts: 'tiny' (M < rows per block where that is possible), 'ragged', 'big' (the U = 4 grid-stride loop
    runs at least twice, with a ragged tail)."""
    _, rpb = rows_geom(C)
    if kind == "tiny":
        return max(1, rpb - 3)
    if kind == "ragged":
        return 37 * rpb + rpb // 2 + 1
    rstep = CAP * rpb
    return 8 * rstep + (12345 % rstep if rpb > 1 else 77)


def rows_locator(M, C, U_=1):
    """(row, channel) -> block, thread, loop iteration and U slot of bn_apply_kernel / bn_bwd_apply_kernel."""
    lanes, rpb = rows_geom(C)
    grid = min(max((M + rpb - 1) // rpb, 1), CAP)
    rstep = grid * rpb

    def loc(r, c):
        cv = c // 8
        it = r // rstep
        return (f"[block={(r % rstep) // rpb} thread={(r % rpb) * lanes + cv % lanes} column_pass={cv // lanes} "
                f"row_iteration={it // U_} u={it % U_} (grid {grid}, rows/block {rpb})]")

    return loc


def mask_locator(M, C, U_=1):
    loc = rows_locator(M, C, U_)
    return lambda j: loc(j // (C // 8), (j % (C // 8)) * 8)


# ================================================================================================ BatchNorm forward
# kernel template instance launched by bn_apply for (relu, residual mode, set_bn_rows_unroll value)
def apply_instance(rmode, u):
    return 4 if (u == 4 or (u == 3 and rmode != 2)) else 2 if u == 2 else 1


def bwd_apply_instance(mask, u):
    return 4 if (u == 4 or (u == 3 and not mask)) else 2 if (u == 2 or (u == 3 and mask)) else 1


APPLY_C = (8, 24, 64, 72, 1280, 2048, 4096)
M_KINDS = ("tiny", "ragged", "big")
UNROLLS = (1, 2, 4, 3)
APPLY_CONFIGS = [(relu, rmode, u, bitmap) for relu in (True, False) for rmode in (0, 1, 2) for u in UNROLLS
                 for bitmap in (False, True)]


def edge_affine(C, g):
    """Per-channel power-of-two scale and a shift that puts y*scale + shift exactly on 0 at y == edge[c]."""
    sc = pow2((C,), -2, 1, g)
    edge = ints((C,), -5, 5, g)
    return sc, -sc * edge, edge


def apply_data(M, C, seed):
    g = gen(seed)
    y = with_large(ints((M, C), -6, 6, g), g)
    sc, sh, edge = edge_affine(C, g)
    on_edge = torch.rand(M, C, device=DEV, generator=g) < 0.25
    y = torch.where(on_edge, edge.expand(M, C), y)
    base = y * sc + sh
    # identity residual: 0 on the edge elements, minus the BN output on another eighth (pre-activation 0 again)
    r1 = ints((M, C), -4, 4, g)
    cancel = (torch.rand(M, C, device=DEV, generator=g) < 0.125) & (base.abs() <= 24)
    r1 = torch.where(on_edge, 0.0, torch.where(cancel, -base, r1))
    # residual with its own BatchNorm: res*rs + rh cancels the main branch on the same elements
    rs, rh = pow2((C,), -1, 1, g), ints((C,), -16, 16, g) * 0.25
    r2 = ints((M, C), -4, 4, g)
    r2 = torch.where(on_edge, -rh / rs, torch.where(cancel, (-base - rh) / rs, r2))
    return dict(y=bf(y), sc=f32(sc), sh=f32(sh), r1=bf(r1), r2=bf(r2), rs=f32(rs), rh=f32(rh),
                pre=(base, base + r1, base + r2 * rs + rh))


@pytest.mark.parametrize("kind", M_KINDS)
@pytest.mark.parametrize("C", APPLY_C)
def test_bn_apply(C, kind, set_unroll):
    """bn_apply over relu x residual (none / identity / own BN) x U in {1, 2, 4, 3} x bitmap on / off: the output is
    bf16_rn of the exact pre-activation (after ReLU), the bitmap is pre > 0, and without ReLU no bitmap is written."""
    e = _ops()
    M = rows_M(C, kind)
    d = apply_data(M, C, seed=C + len(kind))
    for rm in range(3):
        assert float((d["pre"][rm] == 0).double().mean()) > 0.2, "too few exact zeros before the ReLU"
    exp_out = {(relu, rm): to_bf16_exact(d["pre"][rm].clamp(min=0) if relu else d["pre"][rm])
               for relu in (True, False) for rm in range(3)}
    exp_mask = [pack_mask(d["pre"][rm] > 0) for rm in range(3)]
    out = Guarded((M, C), BF)
    mask = Guarded((M * C // 8,), torch.uint8)
    for relu, rm, u, bitmap in APPLY_CONFIGS:
        name = f"bn_apply C={C} M={M} relu={relu} residual={('none', 'identity', 'own BN')[rm]} U={u} bitmap={bitmap}"
        out.t.fill_(NAN)
        mask.t.fill_(POISON_U8)
        set_unroll(u)
        res = (None, d["r1"], d["r2"])[rm]
        rs, rh = (d["rs"], d["rh"]) if rm == 2 else (None, None)
        e.bn_apply(d["y"], d["sc"], d["sh"], res, rs, rh, out.t, relu, mask.t if bitmap else None)
        torch.cuda.synchronize()
        inst = apply_instance(rm, u)
        check_equal(name + " out", out.t, exp_out[(relu, rm)], rows_locator(M, C, inst))
        out.check_guards(name)
        mask.check_guards(name + " bitmap")
        if bitmap and relu:
            check_equal(name + " bitmap", mask.t, exp_mask[rm], mask_locator(M, C, inst))
        else:
            assert bool(mask.untouched().all()), f"{name}: bitmap written"


def finalize_data(C, count, seed):
    """Sums of a batch of `count` (a power of two) values per channel with dyadic mean and variance."""
    g = gen(seed)
    mean = ints((C,), -32, 32, g) / 8
    var = ints((C,), 0, 64, g) / 16
    return dict(sum=mean * count, sqsum=(var + mean * mean) * count, mean=mean, var=var,
                gamma=ints((C,), -16, 16, g) / 8, beta=ints((C,), -16, 16, g) / 4,
                rm=ints((C,), -8, 8, g) / 4, rv=ints((C,), 1, 16, g) / 4)


def rsqrt_ok(got, x):
    """rsqrtf(x) under fast math: at most 2 ulp from 1/sqrt(x) (Programming Guide, single-precision function table)."""
    ref = 1.0 / torch.sqrt(x)
    ulp = 2.0 ** (torch.floor(torch.log2(ref)) - 23)
    return (got.double() - ref).abs() <= 2 * ulp


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("C", [24, 1280])
def test_bn_finalize(C, training):
    """Mean, variance and running statistics exact (count 2^14, momentum 0.5); invstd within the rsqrtf bound;
    scale == fp32(gamma * invstd); shift = beta - mean*scale (either contraction); the sums are zeroed."""
    e = _ops()
    count, mom, eps = 2.0 ** 14, 0.5, 1e-5
    d = finalize_data(C, count, seed=C)
    s, q = f32(d["sum"]).clone(), f32(d["sqsum"]).clone()
    rm, rv = f32(d["rm"]).clone(), f32(d["rv"]).clone()
    outs = [Guarded((C,), torch.float32, guard=64) for _ in range(4)]
    e.bn_finalize(s, q, count, f32(d["gamma"]), f32(d["beta"]), rm, rv, mom, eps, *[o.t for o in outs], training)
    torch.cuda.synchronize()
    mean, invstd, scale, shift = (o.t.double() for o in outs)
    for o, nm in zip(outs, ("mean", "invstd", "scale", "shift")):
        o.check_guards(nm)
    assert float(s.abs().max()) == 0 and float(q.abs().max()) == 0, "sums not zeroed"
    if training:
        m, var = d["mean"], d["var"]
        check_equal("running_mean", rm, 0.5 * d["rm"] + 0.5 * m)
        # running_var = 0.5 rv + (0.5 var) * unbias: unbias = fp32(count / (count - 1)) is not dyadic, so one product
        # rounds; with or without contraction into an fma
        ub = torch.tensor(count / (count - 1), dtype=torch.float32).double()
        t = 0.5 * var * ub
        cands = ((0.5 * d["rv"] + t).float(), (0.5 * d["rv"] + t.float().double()).float())
        ok = (rv == cands[0]) | (rv == cands[1])
        assert bool(ok.all()), f"running_var: channel {int((~ok).nonzero()[0])} got {rv[~ok][0].item()}"
    else:
        m, var = d["rm"], d["rv"]
        check_equal("running_mean (eval: unchanged)", rm, d["rm"])
        check_equal("running_var (eval: unchanged)", rv, d["rv"])
    check_equal("mean", mean, m)
    xin = (f32(var) + torch.tensor(eps, dtype=torch.float32, device=DEV)).double()
    assert bool(rsqrt_ok(outs[1].t, xin).all()), "invstd outside the rsqrtf bound"
    check_equal("scale", scale, (d["gamma"] * invstd).float())
    ok = (shift == (d["beta"] - m * scale).float()) | (shift == (d["beta"] - (m * scale).float().double()).float())
    assert bool(ok.all()), "shift is neither beta - mean*scale form"


def bn_pack(C, count, seed):
    d = finalize_data(C, count, seed)
    return [d[k].float() for k in ("sum", "sqsum", "gamma", "beta", "rm", "rv")] + \
        [torch.full((C,), NAN, device=DEV) for _ in range(4)]


@pytest.mark.parametrize("C,M", [(24, 3001), (64, 20011), (4096, 77)])
def test_bn_apply_fused_matches_unfused(C, M):
    """bn_apply_fused == bn_finalize + bn_apply bit for bit in out, the bitmap and all saved vectors; the running
    statistics are updated exactly once and the sums are left untouched."""
    e = _ops()
    count, mom, eps = float(M), 0.5, 1e-5
    g = gen(C)
    y = torch.randn(M, C, device=DEV, generator=g).to(BF)
    res = torch.randn(M, C, device=DEV, generator=g).to(BF)
    for relu in (True, False):
        for rm in range(3):
            name = f"bn_apply_fused C={C} M={M} relu={relu} residual={rm}"
            fp, rp = bn_pack(C, count, 1), bn_pack(C, count, 2)
            up, urp = [t.clone() for t in fp], [t.clone() for t in rp]
            sums0 = [t.clone() for t in fp[:2] + rp[:2]]
            out_f, out_u = Guarded((M, C), BF), Guarded((M, C), BF)
            mk_f, mk_u = Guarded((M * C // 8,), torch.uint8), Guarded((M * C // 8,), torch.uint8)
            r = res if rm else None
            e.bn_apply_fused(y, fp, count, mom, eps, r, rp if rm == 2 else None, out_f.t, relu, mk_f.t)
            e.bn_finalize(up[0], up[1], count, up[2], up[3], up[4], up[5], mom, eps, *up[6:], True)
            if rm == 2:
                e.bn_finalize(urp[0], urp[1], count, urp[2], urp[3], urp[4], urp[5], mom, eps, *urp[6:], True)
            e.bn_apply(y, up[8], up[9], r, urp[8] if rm == 2 else None, urp[9] if rm == 2 else None, out_u.t, relu,
                       mk_u.t)
            torch.cuda.synchronize()
            check_equal(name + " out", out_f.t, out_u.t, rows_locator(M, C))
            check_equal(name + " bitmap", mk_f.t, mk_u.t)
            out_f.check_guards(name)
            mk_f.check_guards(name + " bitmap")
            packs = [(fp, up, "main")] + ([(rp, urp, "residual")] if rm == 2 else [])
            for a, b, which in packs:
                for i, nm in zip(range(4, 10), ("running_mean", "running_var", "mean", "invstd", "scale", "shift")):
                    check_equal(f"{name} {which} {nm}", a[i], b[i])
            for t, t0, nm in zip(fp[:2] + rp[:2], sums0, ("sum", "sqsum", "res sum", "res sqsum")):
                check_equal(f"{name} {nm} untouched", t, t0)


# ================================================================================================ BatchNorm backward
REDUCE_C = (8, 24, 64, 1280, 2048)
REDUCE_M = {"ragged": 4099, "above_block_cap": RED_CAP * 32 + 1001}
# (mode, g2, dz_out): every col_reduce_kernel mode with and without its optional operands (mode 0 = channel_stats)
REDUCE_VARIANTS = [(0, False, False), (2, False, False), (3, False, False)] + \
    [(m, g2, dz) for m in (1, 4) for g2 in (False, True) for dz in (False, True)]


def reduce_depth(M, C):
    """Additions on a term's path in col_reduce_kernel: its thread's row loop, the rows-per-block fold in shared
    memory, one atomic per block."""
    blocks = min(max((M + 31) // 32, 1), RED_CAP)
    _, rpb = rows_geom(C)
    rows_per_block = -(-M // blocks)
    return -(-rows_per_block // rpb) + rpb + blocks


@pytest.mark.parametrize("kind", list(REDUCE_M))
@pytest.mark.parametrize("C", REDUCE_C)
def test_bn_bwd_reduce(C, kind):
    """channel_stats and bn_bwd_reduce modes 1 (+- g2, +- dz_out), 2, 3 and 4 (+- g2, +- dz_out) against float64."""
    e = _ops()
    M = REDUCE_M[kind]
    g = gen(C + M)
    g1 = with_large(ints((M, C), -4, 4, g), g)   # g1 + g2 near 257..1200 is not a bf16 value: stored dz rounds
    g2 = ints((M, C), -3, 3, g)
    y = ints((M, C), -2, 2, g)
    sc = pow2((C,), -1, 1, g)
    sh = sc * torch.tensor([-1.0, 0.0, 1.0], device=DEV)[torch.randint(0, 3, (C,), device=DEV, generator=g)]
    pre = y * sc + sh
    assert float((pre == 0).double().mean()) > 0.15, "too few elements on the mask edge"
    outp = torch.tensor([-1.0, 0.0, 0.5, 1.0, 3.0], device=DEV)[torch.randint(0, 5, (M, C), device=DEV, generator=g)]
    bits = torch.rand(M, C, device=DEV, generator=g) < 0.6
    t = dict(g1=bf(g1), g2=bf(g2), y=bf(y), sc=f32(sc), sh=f32(sh), outp=bf(outp), bitmap=pack_mask(bits))
    depth = reduce_depth(M, C)
    # the forward's bitmap for (y, scale, shift): mode 2 must mask exactly like it
    fwd_bits = Guarded((M * C // 8,), torch.uint8)
    e.bn_apply(t["y"], t["sc"], t["sh"], None, None, None, torch.empty(M, C, device=DEV, dtype=BF), True, fwd_bits.t)
    for mode, has_g2, has_dz in REDUCE_VARIANTS:
        name = f"col_reduce C={C} M={M} mode={mode} g2={has_g2} dz_out={has_dz}"
        s0 = Guarded((C,), torch.float32, 0.0, guard=64)
        s1 = Guarded((C,), torch.float32, 0.0, guard=64)
        dz_out = Guarded((M, C), BF)
        if mode == 0:
            e.channel_stats(t["y"], s0.t, s1.t)
            terms = (y, y * y)
        else:
            f = g1 + (g2 if has_g2 else 0)
            f = f * {1: outp > 0, 2: pre > 0, 3: torch.ones_like(bits), 4: bits}[mode]
            terms = (f, f * y)
            e.bn_bwd_reduce(mode, t["g1"], t["g2"] if has_g2 else None,
                            {1: t["outp"], 4: t["bitmap"]}.get(mode), t["y"], t["sc"] if mode == 2 else None,
                            t["sh"] if mode == 2 else None, dz_out.t if has_dz else None, s0.t, s1.t)
        torch.cuda.synchronize()
        for gd, nm, term in ((s0, "sum0", terms[0]), (s1, "sum1", terms[1])):
            gd.check_guards(f"{name} {nm}")
            check_sum(f"{name} {nm}", gd.t, term.sum(0), term.abs().sum(0), depth)
        dz_out.check_guards(name + " dz_out")
        if has_dz:
            # the stored dz is the bf16 rounding of the fp32 dz the sums used
            if has_g2:
                assert bool((terms[0].float().to(BF).double() != terms[0]).any()), "no dz needs rounding"
            check_equal(name + " dz_out", dz_out.t, terms[0].float().to(BF))
        else:
            assert bool(dz_out.untouched().all()), f"{name}: dz written"
    check_equal(f"forward bitmap C={C} M={M}", fwd_bits.t, pack_mask(pre > 0))
    # mode 2 == mode 4 with the forward's bitmap, bit for bit
    sums = []
    for mode in (2, 4):
        s0, s1 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        e.bn_bwd_reduce(mode, t["g1"], None, fwd_bits.t if mode == 4 else None, t["y"], t["sc"] if mode == 2 else None,
                        t["sh"] if mode == 2 else None, None, s0, s1)
        sums.append((s0, s1))
    torch.cuda.synchronize()
    check_equal("mode 2 vs forward bitmap: sum dz", sums[0][0], sums[1][0])
    check_equal("mode 2 vs forward bitmap: sum dz*y", sums[0][1], sums[1][1])


def coeff_data(C, seed):
    g = gen(seed)
    return dict(sdz=ints((C,), -64, 64, g), sdzy=ints((C,), -64, 64, g), gamma=pow2((C,), -1, 1, g),
                mean=ints((C,), -8, 8, g) / 4, invstd=pow2((C,), -1, 1, g))


@pytest.mark.parametrize("C", [24, 1280])
def test_bn_bwd_coeffs(C):
    """dgamma, dbeta, A, B, C exact on dyadic inputs (count 2^10); the sums are zeroed."""
    e = _ops()
    count = 2.0 ** 10
    d = coeff_data(C, C)
    sdz, sdzy = f32(d["sdz"]).clone(), f32(d["sdzy"]).clone()
    outs = [Guarded((C,), torch.float32, guard=64) for _ in range(5)]
    e.bn_bwd_coeffs(sdz, sdzy, f32(d["gamma"]), f32(d["mean"]), f32(d["invstd"]), count, *[o.t for o in outs])
    torch.cuda.synchronize()
    db = d["sdz"]
    dg = d["invstd"] * (d["sdzy"] - d["mean"] * db)
    A = d["gamma"] * d["invstd"]
    B = -A * d["invstd"] * dg / count
    Cc = -A * db / count - B * d["mean"]
    for o, ref, nm in zip(outs, (dg, db, A, B, Cc), ("dgamma", "dbeta", "A", "B", "C")):
        o.check_guards(nm)
        check_equal(nm, o.t, f32(ref))
    assert float(sdz.abs().max()) == 0 and float(sdzy.abs().max()) == 0, "sums not zeroed"


def bwd_apply_data(M, C, seed):
    g = gen(seed)
    gr = with_large(ints((M, C), -6, 6, g), g)
    y = ints((M, C), -6, 6, g)
    sc, sh, edge = edge_affine(C, g)
    y = torch.where(torch.rand(M, C, device=DEV, generator=g) < 0.25, edge.expand(M, C), y)
    A = pow2((C,), -2, 1, g)
    B = pow2((C,), -3, 0, g) * ints((C,), -1, 1, g)
    Cc = ints((C,), -16, 16, g) * 0.25
    return dict(g=bf(gr), y=bf(y), sc=f32(sc), sh=f32(sh), A=f32(A), B=f32(B), Cc=f32(Cc), gr=gr, yd=y,
                pre=y * sc + sh, Ad=A, Bd=B, Cd=Cc)


@pytest.mark.parametrize("kind", M_KINDS)
@pytest.mark.parametrize("C", APPLY_C)
def test_bn_bwd_apply(C, kind, set_unroll):
    """bn_bwd_apply, MASK on / off x U in {1, 2, 4, 3}: dy = bf16_rn(A*dz + B*y + C), exact."""
    e = _ops()
    M = rows_M(C, kind)
    d = bwd_apply_data(M, C, seed=3 * C + len(kind))
    assert float((d["pre"] == 0).double().mean()) > 0.2
    dy = Guarded((M, C), BF)
    for mask in (False, True):
        dz = d["gr"] * (d["pre"] > 0) if mask else d["gr"]
        exp = to_bf16_exact(d["Ad"] * dz + d["Bd"] * d["yd"] + d["Cd"])
        for u in UNROLLS:
            name = f"bn_bwd_apply C={C} M={M} mask={mask} U={u}"
            dy.t.fill_(NAN)
            set_unroll(u)
            e.bn_bwd_apply(d["g"], d["y"], d["sc"] if mask else None, d["sh"] if mask else None, d["A"], d["B"],
                           d["Cc"], dy.t)
            torch.cuda.synchronize()
            check_equal(name, dy.t, exp, rows_locator(M, C, bwd_apply_instance(mask, u)))
            dy.check_guards(name)


@pytest.mark.parametrize("C,M", [(24, 3001), (64, 20011), (4096, 77)])
def test_bn_bwd_apply_fused_matches_unfused(C, M):
    """bn_bwd_apply_fused == bn_bwd_coeffs + bn_bwd_apply bit for bit (dy, dgamma, dbeta); the sums are untouched."""
    e = _ops()
    g = gen(C + 1)
    gr = torch.randn(M, C, device=DEV, generator=g).to(BF)
    y = torch.randn(M, C, device=DEV, generator=g).to(BF)
    sdz, sdzy = torch.randn(C, device=DEV, generator=g) * 50, torch.randn(C, device=DEV, generator=g) * 50
    gamma, mean = torch.rand(C, device=DEV, generator=g) + 0.5, torch.randn(C, device=DEV, generator=g)
    invstd = torch.rand(C, device=DEV, generator=g) + 0.5
    sc, sh = torch.randn(C, device=DEV, generator=g), torch.randn(C, device=DEV, generator=g)
    for mask in (False, True):
        name = f"bn_bwd_apply_fused C={C} M={M} mask={mask}"
        a, b = sdz.clone(), sdzy.clone()
        dg_f, db_f = Guarded((C,), torch.float32, guard=64), Guarded((C,), torch.float32, guard=64)
        dy_f, dy_u = Guarded((M, C), BF), Guarded((M, C), BF)
        s = (sc, sh) if mask else (None, None)
        e.bn_bwd_apply_fused(gr, y, *s, a, b, gamma, mean, invstd, float(M), dg_f.t, db_f.t, dy_f.t)
        torch.cuda.synchronize()
        check_equal(name + " sum_dz untouched", a, sdz)
        check_equal(name + " sum_dzy untouched", b, sdzy)
        co = [torch.empty(C, device=DEV) for _ in range(5)]
        e.bn_bwd_coeffs(a, b, gamma, mean, invstd, float(M), *co)
        e.bn_bwd_apply(gr, y, *s, co[2], co[3], co[4], dy_u.t)
        torch.cuda.synchronize()
        check_equal(name + " dy", dy_f.t, dy_u.t, rows_locator(M, C))
        check_equal(name + " dgamma", dg_f.t, co[0])
        check_equal(name + " dbeta", db_f.t, co[1])
        for gd, nm in ((dy_f, "dy"), (dg_f, "dgamma"), (db_f, "dbeta")):
            gd.check_guards(f"{name} {nm}")


# ================================================================================================ pooling, stem tail
POOL_CASES = [(2, 17, 16, 64), (3, 12, 15, 24), (1, 9, 9, 8), (24, 112, 112, 64)]   # last: grid-stride loop runs twice


def pool_ref(a):
    """3x3/2 pad-1 max pool of NHWC float64 `a`: values and the first argmax in row-major window order."""
    N, H, W, C = a.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(a.permute(0, 3, 1, 2), (1, 1, 1, 1), value=-math.inf)
    win = F.unfold(xp, 3, stride=2).view(N, C, 9, Ho, Wo)
    val = win.max(dim=2).values
    # first maximum: weight the positions 9, 8, ..., 1 so that the first one holding the maximum is the unique argmax
    first = ((win == val.unsqueeze(2)) * torch.arange(9, 0, -1, device=DEV).view(1, 1, 9, 1, 1)).argmax(dim=2)
    return val.permute(0, 2, 3, 1).contiguous(), first.permute(0, 2, 3, 1).to(torch.uint8).contiguous()


def pool_locator(Ho, Wo, C):
    cvec = C // 8

    def loc(n, h, w, c):
        i = ((n * Ho + h) * Wo + w) * cvec + c // 8
        return f"[work item {i}: block {i // 256 % CAP} thread {i % 256} grid-stride pass {i // (256 * CAP)}]"

    return loc


@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "x".join(map(str, c)))
def test_maxpool_fwd(case):
    """maxpool_fwd and bn_relu_maxpool_fwd: values and argmax (first maximum) against float64.  Ties come from ReLU
    zeros and from bf16 rounding of values above 256."""
    e = _ops()
    N, H, W, C = case
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    g = gen(N * H + C)
    x = with_large(ints((N, H, W, C), -3, 3, g), g, frac=1 / 8)
    x = torch.where(torch.rand(N, H, W, C, device=DEV, generator=g) < 0.3, x.clamp(min=0), x)   # ReLU zeros
    sc, sh, edge = edge_affine(C, g)
    y = torch.where(torch.rand(N, H, W, C, device=DEV, generator=g) < 0.25, edge.expand(N, H, W, C),
                    with_large(ints((N, H, W, C), -6, 6, g), g, frac=1 / 4))
    act = to_bf16_exact((y * sc + sh).clamp(min=0)).double()   # bf16(relu(fma)): ties above 256 after rounding
    loc = pool_locator(Ho, Wo, C)
    for name, run, src in (("maxpool_fwd", lambda o, i: e.maxpool_fwd(bf(x), o, i), x),
                           ("bn_relu_maxpool_fwd", lambda o, i: e.bn_relu_maxpool_fwd(bf(y), f32(sc), f32(sh), o, i), act)):
        val, idx = pool_ref(src)
        out, am = Guarded((N, Ho, Wo, C), BF), Guarded((N, Ho, Wo, C), torch.uint8)
        run(out.t, am.t)
        torch.cuda.synchronize()
        check_equal(f"{name} {case} values", out.t, to_bf16_exact(val), loc)
        check_equal(f"{name} {case} argmax", am.t, idx, loc)
        out.check_guards(name)
        am.check_guards(name + " argmax")
        ties = (F.unfold(F.pad(src.permute(0, 3, 1, 2), (1, 1, 1, 1), value=-math.inf), 3, stride=2)
                .view(N, C, 9, Ho, Wo) == val.permute(0, 3, 1, 2).unsqueeze(2)).sum(2)
        assert int((ties > 1).sum()) > 0, "no ties in the windows"


def maxpool_bwd_ref(idx, gsum, H, W):
    """dx of a 3x3/2 pad-1 max pool: each window adds its gradient at its argmax (float64)."""
    N, Ho, Wo, C = gsum.shape
    dxp = torch.zeros(N, 2 * Ho + 2, 2 * Wo + 2, C, dtype=torch.float64, device=DEV)
    for a in range(9):
        r, q = divmod(a, 3)
        dxp[:, r:r + 2 * Ho:2, q:q + 2 * Wo:2, :] += gsum * (idx == a)
    return dxp[:, 1:H + 1, 1:W + 1, :]


@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "x".join(map(str, c)))
def test_maxpool_bwd(case):
    """maxpool_bwd +- g2: every pixel sums the gradients of the windows whose argmax it is; exact."""
    e = _ops()
    N, H, W, C = case
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    g = gen(N * W + C)
    idx = torch.randint(0, 9, (N, Ho, Wo, C), device=DEV, generator=g).to(torch.uint8)
    g1 = with_large(ints((N, Ho, Wo, C), -4, 4, g), g)
    g2 = ints((N, Ho, Wo, C), -3, 3, g)
    for use_g2 in (False, True):
        name = f"maxpool_bwd {case} g2={use_g2}"
        dx = Guarded((N, H, W, C), BF)
        e.maxpool_bwd(idx, bf(g1), bf(g2) if use_g2 else None, dx.t)
        torch.cuda.synchronize()
        ref = maxpool_bwd_ref(idx, g1 + g2 if use_g2 else g1, H, W)
        check_equal(name, dx.t, to_bf16_exact(ref), pool_locator(H, W, C))
        dx.check_guards(name)


def test_stem_pool_bn_bwd():
    """stem_pool_bn_bwd passes 0 and 1, +- g2: exact against float64 and bit-identical to maxpool_bwd ->
    bn_bwd_reduce(2) -> bn_bwd_coeffs -> bn_bwd_apply.  N = 9 at 56x56 pooled gives 441 tiles on 396 CTAs; argmaxes
    of every tile's window row / column 8 point at the tile's last pixel row / column (window 8 is the next tile's
    first window, and this tile also processes it)."""
    e = _ops()
    N, Ho, Wo, C = 9, 56, 56, 64
    H, W = 2 * Ho, 2 * Wo
    assert N * (Ho // 8) * (Wo // 8) > 132 * 3
    g = gen(77)
    idx = torch.randint(0, 9, (N, Ho, Wo, C), device=DEV, generator=g)
    r, q = idx // 3, idx % 3
    ho = torch.arange(Ho, device=DEV).view(1, Ho, 1, 1)
    wo = torch.arange(Wo, device=DEV).view(1, 1, Wo, 1)
    r = torch.where((ho % 8 == 0) & (ho > 0), 0, r)   # window row 8k -> pixel row 16k - 1: the previous tile's last row
    q = torch.where((wo % 8 == 0) & (wo > 0), 0, q)
    idx = (r * 3 + q).to(torch.uint8)
    g1 = with_large(ints((N, Ho, Wo, C), -3, 3, g), g, frac=1 / 32)
    g2 = ints((N, Ho, Wo, C), -2, 2, g)
    y = ints((N, H, W, C), -2, 2, g)
    sc = pow2((C,), -1, 1, g)
    sh = sc * torch.tensor([-1.0, 0.0, 1.0], device=DEV)[torch.randint(0, 3, (C,), device=DEV, generator=g)]
    A, B, Cc = pow2((C,), -2, 0, g), pow2((C,), -3, -1, g) * ints((C,), -1, 1, g), ints((C,), -8, 8, g) * 0.25
    pre = y * sc + sh
    assert float((pre == 0).double().mean()) > 0.1
    t = dict(idx=idx, g1=bf(g1), g2=bf(g2), y=bf(y), sc=f32(sc), sh=f32(sh))
    for use_g2 in (False, True):
        name = f"stem_pool_bn_bwd g2={use_g2}"
        gg2 = t["g2"] if use_g2 else None
        da = maxpool_bwd_ref(idx, g1 + g2 if use_g2 else g1, H, W)
        dz = to_bf16_exact(da).double() * (pre > 0)
        s0, s1 = Guarded((C,), torch.float32, 0.0, guard=64), Guarded((C,), torch.float32, 0.0, guard=64)
        e.stem_pool_bn_bwd(0, idx, t["g1"], gg2, t["y"], t["sc"], t["sh"], None, None, None, None, s0.t, s1.t)
        dy = Guarded((N, H, W, C), BF)
        e.stem_pool_bn_bwd(1, idx, t["g1"], gg2, t["y"], t["sc"], t["sh"], f32(A), f32(B), f32(Cc), dy.t,
                           torch.zeros(C, device=DEV), torch.zeros(C, device=DEV))
        torch.cuda.synchronize()
        for gd, nm, term in ((s0, "sum dz", dz), (s1, "sum dz*y", dz * y)):
            gd.check_guards(f"{name} {nm}")
            term = term.reshape(-1, C)
            assert check_sum(f"{name} {nm}", gd.t, term.sum(0), term.abs().sum(0), 1) == "exact"

        def loc(n, h, w, c):
            tile = (n * (Ho // 8) + h // 16) * (Wo // 8) + w // 16
            return f"[tile {tile} (CTA {tile % 396}) pixel ({h % 16}, {w % 16})]"

        check_equal(name + " dy", dy.t, to_bf16_exact(A * dz + B * y + Cc), loc)
        dy.check_guards(name + " dy")
        # the unfused path, fed the same coefficients
        da0 = torch.empty(N, H, W, C, device=DEV, dtype=BF)
        e.maxpool_bwd(idx, t["g1"], gg2, da0)
        u0, u1 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        e.bn_bwd_reduce(2, da0, None, None, t["y"], t["sc"], t["sh"], None, u0, u1)
        torch.cuda.synchronize()
        check_equal(name + " sum dz vs unfused", s0.t, u0)
        check_equal(name + " sum dz*y vs unfused", s1.t, u1)
        co = [torch.empty(C, device=DEV) for _ in range(5)]
        gamma, mean, invstd = torch.rand(C, device=DEV, generator=g) + 0.5, torch.randn(C, device=DEV, generator=g), \
            torch.rand(C, device=DEV, generator=g) + 0.5
        e.bn_bwd_coeffs(u0, u1, gamma, mean, invstd, float(N * H * W), *co)
        dy_u, dy_f = torch.empty_like(da0), torch.empty_like(da0)
        e.bn_bwd_apply(da0, t["y"], t["sc"], t["sh"], co[2], co[3], co[4], dy_u)
        e.stem_pool_bn_bwd(1, idx, t["g1"], gg2, t["y"], t["sc"], t["sh"], co[2], co[3], co[4], dy_f, u0, u1)
        torch.cuda.synchronize()
        check_equal(name + " dy vs unfused", dy_f, dy_u, loc)


# ================================================================================================ head
def hash_u32(a, b, c):
    """csrc/elementwise.cu hash_u32 in uint32 arithmetic (numpy arrays wrap on overflow)."""
    M = np.uint32
    a, b = np.array([a], dtype=M), np.array([b], dtype=M)
    h = (a * M(0x9E3779B1)) ^ ((b + M(0x7F4A7C15)) * M(0x85EBCA77)) ^ ((c + M(0x165667B1)) * M(0xC2B2AE3D))
    h ^= h >> M(15)
    h *= M(0x2C1B3C6D)
    h ^= h >> M(12)
    h *= M(0x297A2D39)
    h ^= h >> M(15)
    return h


def keep_mask(N, C, p, seed):
    """Dropout keep mask of gap_fwd / gap_bwd for element (n, c): hash(seed_lo, seed_hi, n*C + c) <= threshold, and the
    fp32 keep scale; the threshold and scale follow the host code (drop_p passes through fp32)."""
    pf = float(np.float32(p))
    if pf <= 0:
        return torch.ones(N, C, dtype=torch.bool, device=DEV), 1.0
    thresh = np.uint32(int((1.0 - pf) * 4294967295.0))
    h = hash_u32(seed & 0xFFFFFFFF, seed >> 32, np.arange(N * C, dtype=np.uint32))
    ks = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    return torch.from_numpy((h <= thresh).reshape(N, C)).to(DEV), ks


GAP_CASES = [(8, 7, 7, 2048), (6, 5, 5, 1280), (1100, 7, 7, 2048)]   # last: N * C / 8 > 2112 * 128 (grid-stride loop)


@pytest.mark.parametrize("p", [0.0, 0.2, 0.5])
@pytest.mark.parametrize("case", GAP_CASES, ids=lambda c: "x".join(map(str, c)))
def test_gap_dropout(case, p):
    """gap_fwd / gap_bwd with inverted dropout.  Per-(n, c) means are small integers (exact in bf16, and times the
    keep scale too), so the approximate 1.f/HW cannot change the bf16 result.  The keep mask equals a reimplementation
    of hash_u32 on (seed_lo, seed_hi, n*C + c) with a seed >= 2^32, and the backward zeroes exactly the dropped
    elements."""
    e = _ops()
    N, Hh, Ww, C = case
    HW = Hh * Ww
    seed = (1 << 32) + 987654321 + N
    g = gen(N + C)
    m = ints((N, 1, C), -24, 24, g)
    dev = ints((N, HW, C), -2, 2, g)
    dev = dev - dev.mean(1, keepdim=True).round()     # remove the integer part of the mean ...
    dev[:, -1:, :] -= dev.sum(1, keepdim=True)          # ... and make every deviation column sum to 0
    x = (m + dev).view(N, Hh, Ww, C)
    assert bool((x.view(N, HW, C).sum(1) == HW * m.squeeze(1)).all())
    keep, ks = keep_mask(N, C, p, seed)
    if p > 0:
        rate = float(keep.double().mean())
        assert abs(rate - (1 - p)) < 0.02, rate
    exp = to_bf16_exact((m.squeeze(1) * ks).float().double() * keep)
    out = Guarded((N, C), BF)
    e.gap_fwd(bf(x), out.t, p, seed)
    # backward: dout = HW * m2 so that dout / HW is m2 (small integers)
    m2 = pow2((N, C), 0, 4, g) * (ints((N, C), 0, 1, g) * 2 - 1)   # HW * m2 is exact in bf16
    dx = Guarded((N, Hh, Ww, C), BF)
    e.gap_bwd(bf(m2 * HW), dx.t, p, seed)
    torch.cuda.synchronize()
    name = f"gap {case} p={p}"
    cvec = C // 8
    check_equal(name + " fwd", out.t, exp, lambda n, c: f"[work item {n * cvec + c // 8}]")
    out.check_guards(name + " fwd")
    exp_dx = to_bf16_exact((m2 * ks).float().double() * keep).view(N, 1, 1, C).expand(N, Hh, Ww, C)
    check_equal(name + " bwd", dx.t, exp_dx,
                lambda n, h, w, c: f"[work item {((n * Hh + h) * Ww + w) * cvec + c // 8}, hash index {n * C + c}]")
    dx.check_guards(name + " bwd")


def softmax_bounds(logit, labels, grad_scale):
    """Float64 reference of softmax cross-entropy and error bounds for the fast-math kernel.

    Per term: x = logit - max (one fp32 subtraction, relative error of exp(x) <= u|x|), then __expf(x) errs by at most
    2 + floor(1.173 |x|) ulp (Programming Guide, intrinsic functions table); the warp sum adds at most
    ceil(K / 32) + 5 roundings.  __logf(se) errs by at most 2^-21.41 absolute for se in [0.5, 2], else 3 ulp; lse and
    the loss each round once.  dlogits: p = __expf(x) * rcp(se) (rcp.approx: 1 ulp), p - onehot rounds once, bf16 adds
    half a bf16 ulp (2^-8 relative); results below 2^-126 may be flushed to zero."""
    B, K = logit.shape
    mx = logit.max(1, keepdim=True).values
    x = logit - mx
    ex = torch.exp(x)
    se = ex.sum(1, keepdim=True)
    e_exp = (2 + torch.floor(1.173 * x.abs())) * 2.0 ** -23 + U * x.abs()
    depth = -(-K // 32) + 5
    rel_se = ((ex * e_exp).sum(1, keepdim=True) + depth * U * se) / se
    lse = mx + torch.log(se)
    lab = logit.gather(1, labels.view(-1, 1))
    loss = (lse - lab).squeeze(1)
    e_log = 2.0 ** -21.41 + 3 * 2.0 ** -23 * torch.log(se).abs()
    loss_bound = ((rel_se + e_log) * 1.001 + U * (lse.abs() + (lse - lab).abs())).squeeze(1)
    p = ex / se
    d = (p - F.one_hot(labels, K).double()) * grad_scale
    d_bound = (p * (e_exp + rel_se + RCP_ULP + U) * 1.001 + U * d.abs() / grad_scale) * grad_scale + 2.0 ** -126
    return loss, loss_bound, d, d_bound


def head_data(B, K, g):
    """Logits up to +-60 (bf16) and a dyadic bias with repeated values; a quarter of the rows hold their maximum at two
    columns p < q with equal logit and bias (the label is at either, so one counts as correct, the other not)."""
    p_, q_ = K // 3, K - 1
    l16 = (torch.rand(B, K, device=DEV, generator=g) * 120 - 60).to(BF).double()
    bias = ints((K,), -8, 8, g) / 4
    bias[p_] = bias[q_] = 2.0
    labels = torch.randint(0, K, (B,), device=DEV, generator=g)
    labels[0] = 0
    if B > 1:
        labels[1] = K - 1
        tie = torch.arange(B, device=DEV) % 4 == 2
        l16[tie] = l16[tie].clamp(max=50)
        l16[tie, p_] = l16[tie, q_] = 56.0
        labels = torch.where(tie, torch.where(torch.arange(B, device=DEV) % 8 == 2, p_, q_), labels)
    return l16, bias, labels


def check_bound(name, got, ref, bound):
    err = (got.double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = tuple(int(v) for v in (~ok).nonzero()[0])
        pytest.fail(f"{name}: {int((~ok).sum())} elements outside the bound; at {i} got {got[i].item()} want "
                    f"{ref[i].item()} (error {err[i].item():.3e} > bound {bound[i].item():.3e})")


def accuracy_ref(logit, labels):
    """Correct count with the lowest index winning ties (numpy's argmax, like torch.argmax)."""
    am = torch.from_numpy(np.argmax(logit.cpu().numpy(), axis=1)).to(DEV)
    return int((am == labels).sum())


@pytest.mark.parametrize("B", [1, 257])
@pytest.mark.parametrize("K,ld", [(5, 8), (33, 64), (1000, 1024)])
def test_softmax_ce_head(K, ld, B):
    """softmax_ce_head: logits32 exact (one fp32 add), accuracy count exact (ties: lowest index), padded dlogits
    columns exactly 0; loss, the loss sum and dlogits within the fast-math bounds of softmax_bounds."""
    e = _ops()
    g = gen(K * B)
    l16, bias, labels = head_data(B, K, g)
    gs = 1.0 / 256
    lg16 = torch.full((B, ld), NAN, device=DEV, dtype=BF)   # padded columns hold NaN: they must not be read
    lg16[:, :K] = bf(l16)
    logit = (l16 + bias).float().double()                  # fp32 add of a bf16 and an fp32 value
    logits32, dl16 = Guarded((B, K), torch.float32), Guarded((B, ld), BF)
    loss_rows, stats = Guarded((B,), torch.float32, guard=64), Guarded((2,), torch.float32, 0.0, guard=64)
    e.softmax_ce_head(lg16, f32(bias), labels, logits32.t, dl16.t, loss_rows.t, stats.t, gs)
    torch.cuda.synchronize()
    name = f"softmax_ce_head K={K} ld={ld} B={B}"
    for gd, nm in ((logits32, "logits32"), (dl16, "dlogits16"), (loss_rows, "loss_rows"), (stats, "stats")):
        gd.check_guards(f"{name} {nm}")
    check_equal(name + " logits32", logits32.t, logit, lambda b, k: f"[warp {b} lane {k % 32}]")
    assert int(stats.t[1].item()) == accuracy_ref(logit, labels), f"{name}: accuracy count"
    check_equal(name + " padded dlogits", dl16.t[:, K:], torch.zeros(B, ld - K, device=DEV))
    loss, lb, d, db = softmax_bounds(logit, labels, gs)
    check_bound(name + " loss", loss_rows.t, loss, lb)
    check_bound(name + " loss sum", stats.t[:1], loss.sum().view(1), (lb.sum() + B * U * loss.abs().sum()).view(1))
    check_bound(name + " dlogits", dl16.t[:, :K], d, db + 2.0 ** -8 * (d.abs() + db))


@pytest.mark.parametrize("B", [1, 257])
@pytest.mark.parametrize("K", [5, 33, 1000])
def test_softmax_ce(K, B):
    """softmax_ce (fp32 logits): accuracy count exact; loss, the loss sum and dlogits within the bounds of
    softmax_bounds."""
    e = _ops()
    g = gen(K + B)
    l16, bias, labels = head_data(B, K, g)
    logit = (l16 + bias).float()
    gs = 0.5
    dl = Guarded((B, K), torch.float32)
    loss_rows, stats = Guarded((B,), torch.float32, guard=64), Guarded((2,), torch.float32, 0.0, guard=64)
    e.softmax_ce(logit, labels, dl.t, loss_rows.t, stats.t, gs)
    torch.cuda.synchronize()
    name = f"softmax_ce K={K} B={B}"
    for gd, nm in ((dl, "dlogits"), (loss_rows, "loss_rows"), (stats, "stats")):
        gd.check_guards(f"{name} {nm}")
    assert int(stats.t[1].item()) == accuracy_ref(logit, labels), f"{name}: accuracy count"
    loss, lb, d, db = softmax_bounds(logit.double(), labels, gs)
    check_bound(name + " loss", loss_rows.t, loss, lb)
    check_bound(name + " loss sum", stats.t[:1], loss.sum().view(1), (lb.sum() + B * U * loss.abs().sum()).view(1))
    check_bound(name + " dlogits", dl.t, d, db)


@pytest.mark.parametrize("B", [1, 3, 4, 257])
def test_fc_bias_grad(B):
    """fc_bias_grad: column sums of bf16 dlogits (padded rows of pitch ld), exact on integer data."""
    e = _ops()
    K, ld = 1000, 1024
    g = gen(B)
    dl = with_large(ints((B, ld), -8, 8, g), g)
    db = Guarded((K,), torch.float32)
    e.fc_bias_grad(bf(dl), db.t)
    torch.cuda.synchronize()
    check_equal(f"fc_bias_grad B={B}", db.t, dl[:, :K].sum(0), lambda k: f"[thread for column {k}]")
    db.check_guards("fc_bias_grad")


# ================================================================================================ weights, optimizers
def rne_data(n, g):
    """fp32 values that include exact bf16 midpoints (ties to even, both parities) and arbitrary fp32 values."""
    base = torch.randn(n, device=DEV, generator=g).to(BF).float()
    half_ulp = base.abs() * 2.0 ** -8
    half_ulp = 2.0 ** torch.floor(torch.log2(half_ulp.clamp(min=2.0 ** -100)))
    mid = base + half_ulp * torch.sign(base)                  # exactly half way between two bf16 values
    v = torch.where(torch.rand(n, device=DEV, generator=g) < 0.3, mid, torch.randn(n, device=DEV, generator=g))
    return v


def test_weight_prep():
    """weight_prep: wf = bf16_rn(w) in place, wd = its per-tap transpose [taps][cin][cout] (grid-stride loop twice)."""
    e = _ops()
    taps, cout, cin = 9, 128, 160
    assert taps * cout * cin > 132 * 4 * 256
    w = rne_data(taps * cout * cin, gen(1)).view(taps, cout, cin)
    wf, wd = Guarded((taps, cout, cin), BF), Guarded((taps, cin, cout), BF)
    e.weight_prep(w, wf.t, wd.t, taps, cout, cin)
    torch.cuda.synchronize()
    exp = w.to(BF)
    check_equal("weight_prep wf", wf.t, exp)
    check_equal("weight_prep wd", wd.t, exp.transpose(1, 2))
    wf.check_guards("weight_prep wf")
    wd.check_guards("weight_prep wd")


def test_weight_prep_batched():
    """weight_prep_batched: four layers of different (taps, cout, cin), 2208 tiles (> 2112 CTAs); every destination
    region is the bf16 per-tap transpose of its source, and the NaN gaps between regions survive."""
    e = _ops()
    layers = [(9, 256, 256), (1, 512, 1024), (9, 512, 512), (1, 2048, 512)]
    gap = 40
    rows, src_off, dst_off, tile = [], 0, gap, 0
    for taps, cout, cin in layers:
        rows.append((src_off, dst_off, taps, cout, cin, tile))
        src_off += taps * cout * cin + 3
        dst_off += taps * cout * cin + gap
        tile += taps * (cout // 64) * (cin // 32)
    assert tile > CAP
    params = rne_data(src_off, gen(2))
    wd = Guarded((dst_off,), BF)
    table = torch.tensor(rows, dtype=torch.int64, device=DEV)
    e.weight_prep_batched(params, wd.t, table, tile)
    torch.cuda.synchronize()
    wd.check_guards("weight_prep_batched")
    written = torch.zeros(dst_off, dtype=torch.bool, device=DEV)
    for (so, do, taps, cout, cin, _), i in zip(rows, range(len(rows))):
        n = taps * cout * cin
        exp = params[so:so + n].view(taps, cout, cin).to(BF).transpose(1, 2).reshape(-1)
        check_equal(f"weight_prep_batched layer {i}", wd.t[do:do + n], exp)
        written[do:do + n] = True
    assert bool(wd.untouched()[~written].all()), "a gap between destination regions was written"


def test_pack_stem_weight_and_cast():
    """pack_stem_weight: out[co, k] = bf16_rn(w[k // 3, co, k % 3]), columns 147.. zero.  cast_bf16: bf16_rn over
    4 * (2 * 270336 + 5) values (capped grid loops twice, ragged tail)."""
    e = _ops()
    w = rne_data(49 * 64 * 3, gen(3)).view(49, 64, 3)
    out = Guarded((64, 192), BF)
    e.pack_stem_weight(w, out.t)
    n = 4 * (2 * RED_CAP * 256 + 5)
    x = rne_data(n, gen(4))
    xc = Guarded((n,), BF)
    e.cast_bf16(x, xc.t)
    torch.cuda.synchronize()
    exp = torch.zeros(64, 192, dtype=BF, device=DEV)
    exp[:, :147] = w.permute(1, 0, 2).reshape(64, 147).to(BF)
    check_equal("pack_stem_weight", out.t, exp)
    out.check_guards("pack_stem_weight")
    check_equal("cast_bf16", xc.t, x.to(BF), lambda i: f"[float4 {i // 4}: block {i // 4 // 256 % RED_CAP}]")
    xc.check_guards("cast_bf16")


OPT_N = 4 * (2 * RED_CAP * 256 + 5)   # the capped grid loops twice with a ragged tail


def hyper(lr=0.0, mu=0.0, b2=0.0, eps=0.0, wd=0.0, gs=1.0, bc1=1.0, bc2=1.0):
    return torch.tensor([lr, mu, b2, eps, wd, gs, bc1, bc2], dtype=torch.float32, device=DEV)


def fmaf(a, b, c):
    """fp32 fmaf(a, b, c) of fp32 tensors, correctly rounded: a*b is exact in float64, TwoSum gives a*b + c = s + e
    exactly, and s rounds to the right fp32 value unless s is an fp32 midpoint and e pushes it off that midpoint."""
    A, B, Cd = a.double(), b.double(), c.double()
    p = A * B
    s = p + Cd
    bv = s - p
    e = (p - (s - bv)) + (Cd - bv)
    r = s.float()
    rd = r.double()
    nb = torch.nextafter(r, torch.where(s > rd, math.inf, -math.inf).float()).double()   # the other candidate
    tie = (s != rd) & (2 * (s - rd).abs() == (nb - rd).abs())
    return torch.where(tie & (e != 0) & ((e > 0) == (s > rd)), nb.float(), r)


@pytest.mark.parametrize("nesterov", [False, True])
def test_optim_step_sgd(nesterov):
    """optim_step sgd / sgd_nesterov, 3 steps (lr 2^-4, momentum 0.875, weight decay 2^-8, grad scale 0.5): parameters
    and momentum equal an fp32 emulation of the kernel's fmaf sequence bit for bit, and the bf16 working copy ==
    bf16_rn(p)."""
    e = _ops()
    g = gen(5)
    lr, mu, wd, gs = (torch.tensor(v, device=DEV) for v in (2.0 ** -4, 0.875, 2.0 ** -8, 0.5))
    p = torch.randn(OPT_N, device=DEV, generator=g)
    m = torch.zeros_like(p)
    pt, mt = p.clone(), m.clone()
    p16 = Guarded((OPT_N,), BF)
    h = hyper(lr=2.0 ** -4, mu=0.875, wd=2.0 ** -8, gs=0.5)
    for step in range(3):
        gr = torch.randn(OPT_N, device=DEV, generator=g) * 4
        e.optim_step("sgd_nesterov" if nesterov else "sgd", pt, gr, [mt], p16.t, h)
        d = fmaf(wd, p, gr * gs)
        m = fmaf(mu, m, d)
        p = fmaf(-lr, fmaf(mu, m, d) if nesterov else m, p)
        torch.cuda.synchronize()
        name = f"optim_step sgd nesterov={nesterov} step {step}"
        loc = lambda i: f"[float4 {i // 4}: block {i // 4 // 256 % RED_CAP} thread {i // 4 % 256}]"   # noqa: E731
        check_equal(name + " p", pt, p, loc)
        check_equal(name + " momentum", mt, m, loc)
        check_equal(name + " p16", p16.t, pt.to(BF), loc)
        p16.check_guards(name + " p16")


def test_optim_step_adam_adadelta():
    """optim_step adam and adadelta, one step, against float64.  Each computes with fast-math sqrtf (sqrt.approx:
    relative error <= 2^-23, PTX ISA), rsqrtf (2 ulp) and division (div.approx: 2 ulp) and about eight fp32 roundings on
    the update's path; the bound allows 2^-19 relative on the update and one rounding of the parameter (first order).
    The bf16 working copy is bf16_rn of the parameter the kernel wrote, exactly."""
    e = _ops()
    g = gen(6)
    p, gr = (torch.randn(OPT_N, device=DEV, generator=g).double() for _ in range(2))
    s1, s2 = (torch.rand(OPT_N, device=DEV, generator=g).double() for _ in range(2))
    lr, b1, b2, eps, wd, gs = 1e-3, 0.9, 0.999, 1e-8, 1e-4, 0.5
    hv = hyper(lr, b1, b2, eps, wd, gs, bc1=1 - b1 ** 3, bc2=1 - b2 ** 3).double()
    lr, b1, b2, eps, wd, gs, bc1, bc2 = hv.tolist()
    for name in ("adam", "adadelta"):
        pt, st1, st2 = p.float(), s1.float(), s2.float()
        p16 = Guarded((OPT_N,), BF)
        d = wd * p + gr * gs
        if name == "adam":
            e.optim_step("adam", pt, gr.float(), [st1, st2], p16.t, hv.float())
            m = b1 * s1 + (1 - b1) * d
            v = b2 * s2 + (1 - b2) * d * d
            upd = lr / bc1 * m / (torch.sqrt(v) / math.sqrt(bc2) + eps)
            states = ((m, (b1 * s1).abs() + ((1 - b1) * d).abs()), (v, v))
        else:
            hd = hyper(lr=1.0, b2=0.9, eps=1e-6, wd=wd, gs=gs)
            e.optim_step("adadelta", pt, gr.float(), [st1, st2], p16.t, hd)
            rho, ep = float(hd[2]), float(hd[3])
            sq = rho * s1 + (1 - rho) * d * d
            delta = torch.sqrt(s2 + ep) / torch.sqrt(sq + ep) * d
            upd = delta
            acc = rho * s2 + (1 - rho) * delta * delta
            states = ((sq, sq), (acc, acc))
        torch.cuda.synchronize()
        pn = p - upd
        check_bound(f"{name} p", pt, pn, U * pn.abs() + 2.0 ** -19 * upd.abs())
        for got, (ref, terms), nm in zip((st1, st2), states, ("state 1", "state 2")):
            check_bound(f"{name} {nm}", got, ref, 2.0 ** -19 * terms + 2.0 ** -126)
        check_equal(f"{name} p16", p16.t, pt.to(BF))
        p16.check_guards(f"{name} p16")


# ================================================================================================ MobileNet
DW_CASES = [(2, 13, 11, 64), (1, 15, 17, 192), (2, 7, 10, 960)]   # odd H / W; Wo % 4 != 0 at stride 1 and 2


def dw_data(N, H, W, C, g):
    x = ints((N, H, W, C), -2, 2, g)
    w = ints((9, C), -2, 2, g) * 0.5
    sc = pow2((C,), -1, 1, g)
    sh = ints((C,), -8, 32, g) * 0.25
    return x, w, sc, sh


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: "x".join(map(str, c)))
def test_dwconv3x3(case, stride):
    """dwconv3x3, tile_w 1 and 4: relu6(depthwise conv * scale + shift), exact; ReLU6 hits exactly 0 and 6; the tiled
    and one-pixel kernels agree bit for bit."""
    e = _ops()
    N, H, W, C = case
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    g = gen(C + stride)
    x, w, sc, sh = dw_data(N, H, W, C, g)
    acc = F.conv2d(x.permute(0, 3, 1, 2), w.t().reshape(C, 1, 3, 3), stride=stride, padding=1, groups=C)
    pre = acc.permute(0, 2, 3, 1) * sc + sh
    assert int((pre == 0).sum()) > 0 and int((pre == 6).sum()) > 0, "ReLU6 edges not hit"
    exp = to_bf16_exact(pre.clamp(0, 6))
    outs = {}
    for tw in (1, 4):
        out = Guarded((N, Ho, Wo, C), BF)
        e.dwconv3x3(bf(x), f32(w), f32(sc), f32(sh), out.t, stride, tw)
        torch.cuda.synchronize()
        name = f"dwconv3x3 {case} stride={stride} tile_w={tw}"
        check_equal(name, out.t, exp, lambda n, h, ww, c: f"[thread for pixel ({h}, {ww // tw * tw}) + {ww % tw}]")
        out.check_guards(name)
        outs[tw] = out.t
    check_equal(f"dwconv3x3 {case} stride={stride} tiled vs one-pixel", outs[4], outs[1])


def test_mbv2_stem():
    """mbv2_stem: relu6(conv3x3/2(bf16(x*mul + add)) * scale + shift), exact; channels 32..ldc stay untouched."""
    e = _ops()
    N, H, W, ldc = 2, 34, 30, 64
    g = gen(9)
    x = torch.randint(126, 131, (N, H, W, 3), device=DEV, dtype=torch.uint8, generator=g)
    w = ints((27, 32), -2, 2, g) * 0.5
    sc, sh = pow2((32,), -1, 1, g), ints((32,), -8, 32, g) * 0.25
    out = Guarded((N, H // 2, W // 2, ldc), BF)
    e.mbv2_stem(x, f32(w), f32(sc), f32(sh), out.t, 1.0, -128.0)
    torch.cuda.synchronize()
    wt = w.view(3, 3, 3, 32).permute(3, 2, 0, 1)      # k = (r*3 + s)*3 + c -> [co, c, r, s]
    acc = F.conv2d(x.double().permute(0, 3, 1, 2) - 128.0, wt, stride=2, padding=1).permute(0, 2, 3, 1)
    pre = acc * sc + sh
    assert int((pre == 0).sum()) > 0 and int((pre == 6).sum()) > 0
    check_equal("mbv2_stem", out.t[..., :32], to_bf16_exact(pre.clamp(0, 6)))
    assert bool(out.untouched()[..., 32:].all()), "padded channels written"
    out.check_guards("mbv2_stem")


# ================================================================================================ coverage
def test_case_tables_cover_every_launch_site():
    """The cases above launch every bn_apply_kernel instance (18 unfused: relu x residual x U-template 1/2/4, and 6
    fused), every bn_bwd_apply_kernel instance (6 unfused, 2 fused), every col_reduce_kernel mode with and without
    its optional operands, and both dwconv3x3 kernels at both strides."""
    apply_sites = {(relu, rm, apply_instance(rm, u)) for relu, rm, u, _ in APPLY_CONFIGS}
    assert len(apply_sites) == 18, sorted(apply_sites)
    assert {(relu, rm) for relu, rm, _, _ in APPLY_CONFIGS} == {(r, m) for r in (True, False) for m in range(3)}  # fused
    bwd_sites = {(mask, bwd_apply_instance(mask, u)) for mask in (False, True) for u in UNROLLS}
    assert len(bwd_sites) == 6, sorted(bwd_sites)
    assert {m for m, _, _ in REDUCE_VARIANTS} == {0, 1, 2, 3, 4}
    for mode in (1, 4):
        assert {(g2, dz) for m, g2, dz in REDUCE_VARIANTS if m == mode} == {(a, b) for a in (0, 1) for b in (0, 1)}
    assert max(REDUCE_M.values()) > RED_CAP * 32          # col_reduce_kernel's 1056-block cap
    assert max(APPLY_C) > 8 * 256                         # the column loop of the 256-lane apply kernels runs twice
    assert all(rows_M(C, "big") >= 8 * CAP * rows_geom(C)[1] for C in APPLY_C)


# ================================================================================================ malformed inputs
def test_malformed_inputs_raise():
    """Bindings reject what their kernels cannot handle (dtype, element counts, C % 8, output shapes, 16-byte
    alignment) before launching anything."""
    e = _ops()
    f = lambda *s: torch.zeros(*s, device=DEV)                        # noqa: E731
    b = lambda *s: torch.zeros(*s, device=DEV, dtype=BF)              # noqa: E731
    u8 = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.uint8)    # noqa: E731
    C, M = 64, 32
    y, c = b(M, C), f(C)
    mis_b = b(M * C + 8)[1:M * C + 1].view(M, C)      # 2 bytes off a 16-byte boundary
    mis_f = f(C + 4)[1:C + 1]                          # 4 bytes off
    calls = {
        "bn_apply: misaligned scale": lambda: e.bn_apply(y, mis_f, c, None, None, None, b(M, C), True, None),
        "bn_apply: res_scale without res": lambda: e.bn_apply(y, c, c, None, c, c, b(M, C), True, None),
        "bn_bwd_coeffs: short cA": lambda: e.bn_bwd_coeffs(c, c, c, c, c, 1.0, f(C), f(C), f(C - 8), f(C), f(C)),
        "bn_bwd_coeffs: bf16 gamma": lambda: e.bn_bwd_coeffs(c, c, b(C), c, c, 1.0, f(C), f(C), f(C), f(C), f(C)),
        "bn_bwd_apply: C % 8": lambda: e.bn_bwd_apply(b(M, 12), b(M, 12), None, None, f(12), f(12), f(12), b(M, 12)),
        "bn_bwd_apply: dy size": lambda: e.bn_bwd_apply(y, y, None, None, c, c, c, b(M - 1, C)),
        "bn_bwd_apply: misaligned g": lambda: e.bn_bwd_apply(mis_b, y, None, None, c, c, c, b(M, C)),
        "bn_bwd_apply: scale without shift": lambda: e.bn_bwd_apply(y, y, c, None, c, c, c, b(M, C)),
        "bn_bwd_apply: short cB": lambda: e.bn_bwd_apply(y, y, None, None, c, f(C - 8), c, b(M, C)),
        "bn_bwd_apply_fused: short scale": lambda: e.bn_bwd_apply_fused(y, y, f(C - 8), c, c, c, c, c, c, 1.0, f(C),
                                                                         f(C), b(M, C)),
        "bn_bwd_apply_fused: misaligned dy": lambda: e.bn_bwd_apply_fused(y, y, None, None, c, c, c, c, c, 1.0, f(C),
                                                                           f(C), mis_b),
        "bn_bwd_reduce: short sum_dz": lambda: e.bn_bwd_reduce(3, y, None, None, y, None, None, None, f(C - 1), f(C)),
        "bn_bwd_reduce: fp32 g2": lambda: e.bn_bwd_reduce(1, y, f(M, C), y, y, None, None, None, f(C), f(C)),
        "bn_bwd_reduce: short dz_out": lambda: e.bn_bwd_reduce(1, y, None, y, y, None, None, b(M - 1, C), f(C), f(C)),
        "bn_bwd_reduce: short bitmap": lambda: e.bn_bwd_reduce(4, y, None, u8(M * C // 8 - 1), y, None, None, None,
                                                               f(C), f(C)),
        "bn_bwd_reduce: misaligned y": lambda: e.bn_bwd_reduce(3, y, None, None, mis_b, None, None, None, f(C), f(C)),
        "bn_bwd_reduce: mode 2 misaligned scale": lambda: e.bn_bwd_reduce(2, y, None, None, y, mis_f, c, None, f(C),
                                                                          f(C)),
        "channel_stats: short sum": lambda: e.channel_stats(y, f(C - 1), f(C)),
        "maxpool_fwd: output shape": lambda: e.maxpool_fwd(b(1, 9, 9, C), b(1, 4, 5, C), None),
        "maxpool_fwd: C % 8": lambda: e.maxpool_fwd(b(1, 9, 9, 12), b(1, 5, 5, 12), None),
        "maxpool_fwd: short argmax": lambda: e.maxpool_fwd(b(1, 9, 9, C), b(1, 5, 5, C), u8(1, 5, 5, C - 8)),
        "maxpool_fwd: misaligned input": lambda: e.maxpool_fwd(b(1 * 9 * 9 * C + 8)[1:9 * 9 * C + 1].view(1, 9, 9, C),
                                                               b(1, 5, 5, C), None),
        "bn_relu_maxpool_fwd: short scale": lambda: e.bn_relu_maxpool_fwd(b(1, 9, 9, C), f(C - 8), c, b(1, 5, 5, C),
                                                                          None),
        "maxpool_bwd: g1 shape": lambda: e.maxpool_bwd(u8(1, 5, 5, C), b(1, 4, 5, C), None, b(1, 9, 9, C)),
        "maxpool_bwd: g2 size": lambda: e.maxpool_bwd(u8(1, 5, 5, C), b(1, 5, 5, C), b(1, 5, 4, C), b(1, 9, 9, C)),
        "gap_fwd: output size": lambda: e.gap_fwd(b(2, 7, 7, C), b(2, C - 8), 0.0, 0),
        "gap_fwd: C % 8": lambda: e.gap_fwd(b(2, 7, 7, 12), b(2, 12), 0.0, 0),
        "gap_bwd: dout size": lambda: e.gap_bwd(b(3, C), b(2, 7, 7, C), 0.0, 0),
        "optim_step sgd: misaligned p": lambda: e.optim_step("sgd", f(68)[1:65], f(64), [f(64)], None, f(8)),
        "optim_step sgd: short p16": lambda: e.optim_step("sgd", f(64), f(64), [f(64)], b(60), f(8)),
        "optim_step adadelta: short state": lambda: e.optim_step("adadelta", f(64), f(64), [f(60), f(64)], None, f(8)),
        "dwconv3x3: misaligned weights": lambda: e.dwconv3x3(b(1, 8, 8, C), f(9 * C + 4)[1:9 * C + 1], c, c,
                                                             b(1, 8, 8, C), 1, 4),
    }
    accepted = []
    for name, call in calls.items():
        try:
            call()
        except RuntimeError:
            continue
        accepted.append(name)
    torch.cuda.synchronize()
    assert not accepted, f"malformed calls accepted: {accepted}"
