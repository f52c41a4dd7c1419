"""RMSprop / Adagrad / Adamax / AdamW / Lamb kernels, the segmented sum-of-squares reduction and the clip passes
(csrc/optim.cu) on the GPU, then every optimizer x clip mode through CUDA graphs, the engines and two ranks.

Bounds: the build uses ``--use_fast_math``, so ``sqrtf`` (sqrt.approx, relative 2^-23), ``rsqrtf`` and ``/``
(div.approx, 2 ulp) are approximate.  The update kernels pass about ten fp32 roundings on the way to the update, so as
in the Adam / Adadelta test the parameter may differ from float64 by one rounding of itself plus 2^-19 of the update,
and a state by 2^-19 of the sum of its terms.  LAMB's update also carries the per-tensor trust ratio (two sums of
squares, two square roots, one division): 2^-17 of the update.  A sum of squares of non-negative terms passes at most
``depth`` fp32 additions per term (32 per thread, 8 in the CTA tree, ceil(chunks / 32) + 5 per segment, ceil(segments /
32) + 5 for the total), each erring by at most u times the partial, plus 2u for the square: |error| <= (depth + 2) u sum.
"""
from __future__ import annotations

import math

import pytest
import torch

from exact_util import DEV, U, Guarded, check_equal

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
RED_CAP = 132 * 8
OPT_N = 4 * (2 * RED_CAP * 256 + 5)   # the capped grid loops twice with a ragged tail


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def hyper(lr=0.0, mu=0.0, b2=0.0, eps=0.0, wd=0.0, gs=1.0, bc1=1.0, bc2=1.0, clip=0.0, host_gs=1.0):
    h = torch.zeros(16, dtype=torch.float32, device=DEV)
    h[:10] = torch.tensor([lr, mu, b2, eps, wd, gs, bc1, bc2, clip, host_gs])
    return h


def guarded(t):
    g = Guarded(tuple(t.shape), t.dtype)
    g.t.copy_(t)
    g._bits = g._as_int(g.buf).clone()
    return g


def check_bound(name, got, ref, bound):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        pytest.fail(f"{name}: {int(bad.sum())} elements out of bound; first at {i}: got {got[i].item()} want "
                    f"{ref[i].item()} (error {err[i].item():.3e} > {bound[i].item():.3e})")


# ================================================================================================ update kernels
RMS_VARIANTS = [(c, m) for c in (False, True) for m in (False, True)]


@pytest.mark.parametrize("centered,momentum", RMS_VARIANTS)
def test_optim_step_rmsprop(centered, momentum):
    e = _ops()
    g = gen(11)
    p, gr = (torch.randn(OPT_N, device=DEV, generator=g).double() for _ in range(2))
    v0 = torch.rand(OPT_N, device=DEV, generator=g).double() + 0.5
    a0 = (torch.rand(OPT_N, device=DEV, generator=g).double() - 0.5) * 0.5
    b0 = torch.randn(OPT_N, device=DEV, generator=g).double()
    hv = hyper(lr=1e-2, mu=0.9 if momentum else 0.0, b2=0.9, eps=1e-7, wd=1e-3, gs=0.5)
    lr, mu, rho, eps, wd, gs = hv[:6].double().tolist()
    P, V = guarded(p.float()), guarded(v0.float())
    A, B = guarded(a0.float()), guarded(b0.float())
    p16 = Guarded((OPT_N,), BF)
    rule = "rmsprop" + ("_centered" if centered else "") + ("_momentum" if momentum else "")
    e.optim_step(rule, P.t, gr.float(), [V.t] + [B.t] * momentum + [A.t] * centered, p16.t, hv)
    torch.cuda.synchronize()
    p, v0, a0, b0 = p.float().double(), v0.float().double(), a0.float().double(), b0.float().double()
    gr = gr.float().double()
    d = wd * p + gr * gs
    v = rho * v0 + (1 - rho) * d * d
    states = [("v", V, v, rho * v0 + ((1 - rho) * d * d))]
    var = v
    if centered:
        a = rho * a0 + (1 - rho) * d
        var = v - a * a
        states.append(("avg_grad", A, a, (rho * a0).abs() + ((1 - rho) * d).abs()))
    q = d / (var.sqrt() + eps)
    upd, terms = q, q.abs()
    if momentum:
        upd, terms = mu * b0 + q, (mu * b0).abs() + q.abs()
        states.append(("momentum", B, upd, terms))
    pn = p - lr * upd
    name = f"rmsprop centered={centered} momentum={momentum}"
    check_bound(name + " p", P.t, pn, U * pn.abs() + 2.0 ** -19 * lr * terms)
    for nm, got, ref, terms in states:
        check_bound(f"{name} {nm}", got.t, ref, 2.0 ** -19 * terms + 2.0 ** -126)
    check_equal(name + " p16", p16.t, P.t.to(BF))
    for nm, t in (("p", P), ("v", V), ("avg", A), ("mom", B), ("p16", p16)):
        t.check_guards(f"{name} {nm}")
    if not centered:
        assert bool(A.untouched().all()), "avg_grad written without centered"
    if not momentum:
        assert bool(B.untouched().all()), "momentum written without momentum"


@pytest.mark.parametrize("name", ["adagrad", "adamax", "adamw"])
def test_optim_step_adagrad_adamax_adamw(name):
    e = _ops()
    g = gen(12)
    p, gr = (torch.randn(OPT_N, device=DEV, generator=g).float().double() for _ in range(2))
    s1 = torch.randn(OPT_N, device=DEV, generator=g).float().double() * 0.1
    s2 = torch.rand(OPT_N, device=DEV, generator=g).float().double() + 0.1
    lr, b1, b2, eps, wd, gs = 1e-2, 0.9, 0.999, 1e-7, 1e-3, 0.5
    hv = hyper(lr, b1, b2, eps, wd, gs, bc1=1 - b1 ** 3, bc2=1 - b2 ** 3)
    lr, b1, b2, eps, wd, gs, bc1, bc2 = hv[:8].double().tolist()
    P, S1, S2 = guarded(p.float()), guarded(s1.float()), guarded(s2.float())
    p16 = Guarded((OPT_N,), BF)
    if name == "adagrad":
        e.optim_step("adagrad", P.t, gr.float(), [S2.t], p16.t, hv)
        d = wd * p + gr * gs
        acc = s2 + d * d
        upd = lr * d / (acc.sqrt() + eps)
        states = [(S2, acc, acc)]
        pn = p - upd
    elif name == "adamax":
        e.optim_step("adamax", P.t, gr.float(), [S1.t, S2.t], p16.t, hv)
        d = wd * p + gr * gs
        m = b1 * s1 + (1 - b1) * d
        u = torch.maximum(b2 * s2, d.abs() + eps)
        mt = (b1 * s1).abs() + ((1 - b1) * d).abs()   # m may cancel: its rounding is on the scale of its terms
        upd = lr / bc1 * mt / u
        states = [(S1, m, mt), (S2, u, u)]
        pn = p - lr / bc1 * m / u
    else:
        e.optim_step("adamw", P.t, gr.float(), [S1.t, S2.t], p16.t, hv)
        d = gr * gs
        m = b1 * s1 + (1 - b1) * d
        v = b2 * s2 + (1 - b2) * d * d
        dec = p * (1 - lr * wd)
        mt = (b1 * s1).abs() + ((1 - b1) * d).abs()
        denom = v.sqrt() / math.sqrt(bc2) + eps
        states = [(S1, m, mt), (S2, v, v)]
        pn = dec - lr / bc1 * m / denom
        upd = lr / bc1 * mt / denom + (lr * wd * p).abs()   # the decay's rounding is on the update's scale
    torch.cuda.synchronize()
    # AdamW's decay factor 1 - lr wd is itself rounded in fp32: two more roundings on the scale of p
    check_bound(f"{name} p", P.t, pn, (3 if name == "adamw" else 1) * U * pn.abs() + 2.0 ** -19 * upd.abs())
    for i, (got, ref, terms) in enumerate(states):
        check_bound(f"{name} state {i}", got.t, ref, 2.0 ** -19 * terms + 2.0 ** -126)
    check_equal(f"{name} p16", p16.t, P.t.to(BF))
    for nm, t in (("p", P), ("s1", S1), ("s2", S2), ("p16", p16)):
        t.check_guards(f"{name} {nm}")


# ================================================================================================ segmented reduction
def _tables(segs):
    from b200ddl.optim.fused import chunk_tables

    c, s = chunk_tables(segs)
    return c.to(DEV), s.to(DEV)


def _segments(lengths):
    out, lo = [], 0
    for n in lengths:
        out.append((lo, lo + n))
        lo += n
    return out, lo


SEG_LENGTHS = [4, 8192, 8196, 3 * 2 ** 20 + 4, 0, 64]


def _depth(nchunks_seg, nseg):
    return 32 + 8 + -(-nchunks_seg // 32) + 5 + -(-nseg // 32) + 5


def test_segment_sumsq_and_finalize():
    """Per-segment and total sums of (0.5 g)^2 within the depth bound of float64, bit-identical on a second run."""
    e = _ops()
    segs, n = _segments(SEG_LENGTHS)
    chunks, st = _tables(segs)
    g = torch.randn(n, device=DEV, generator=gen(13))
    hv = hyper(host_gs=0.5)
    outs = []
    for _ in range(2):
        partial = torch.full((chunks.shape[0],), float("nan"), device=DEV)
        sums = torch.full((2, len(segs) + 1), float("nan"), device=DEV)
        factor = torch.zeros(len(segs), device=DEV)
        e.segment_sumsq(g, chunks, partial, hv)
        e.segment_finalize(partial, st, sums, factor, hv, 0)
        torch.cuda.synchronize()
        outs.append(sums[0].clone())
    check_equal("segment sums, second run", outs[1], outs[0])
    gd = (g.double() * 0.5) ** 2
    ref = torch.tensor([float(gd[lo:hi].sum()) for lo, hi in segs] + [float(gd.sum())], dtype=torch.float64)
    nch = [int(b - a) for a, b in st.tolist()]
    depth = torch.tensor([_depth(c, len(segs)) for c in nch] + [_depth(max(nch), len(segs))], dtype=torch.float64)
    check_bound("segment sums", outs[0].cpu(), ref, (depth + 2) * U * ref + 2.0 ** -126)
    assert float(outs[0][4]) == 0.0, "an empty segment sums to 0"


def test_clip_passes_and_lamb_phi():
    """global: hyper[5] = gs c / max(norm, c); clipnorm: per-segment factor (exactly 1 at or below c), then g * (gs *
    factor) bit for bit; clipvalue: clamp(g gs, -c, c) bit for bit; LAMB phi = |p| / |r| per segment, 1 for a zero
    segment."""
    e = _ops()
    segs, n = _segments([8192 * 3 + 4, 4096, 64, 8196])
    chunks, st = _tables(segs)
    g0 = torch.randn(n, device=DEV, generator=gen(14))
    g0[segs[2][0]:segs[2][1]] = 0                       # zero segment
    g0[segs[1][0]:segs[1][1]] *= 1e-3                   # below the threshold
    gs, c = 0.5, 2.0
    hv = hyper(gs=gs, clip=c, host_gs=gs)
    partial = torch.zeros(2, chunks.shape[0], device=DEV)
    sums = torch.zeros(2, len(segs) + 1, device=DEV)
    factor = torch.zeros(len(segs), device=DEV)
    gd = g0.double() * gs
    norms = torch.tensor([float(gd[lo:hi].norm()) for lo, hi in segs], dtype=torch.float64)
    tot = float(gd.norm())
    # global
    e.segment_sumsq(g0, chunks, partial[0], hv)
    e.segment_finalize(partial[0], st, sums, factor, hv, 1)
    torch.cuda.synchronize()
    assert abs(float(hv[5]) - gs * c / tot) <= 2.0 ** -18 * gs * c / tot
    assert float(hv[9]) == gs
    # clipnorm
    g = g0.clone()
    e.segment_sumsq(g, chunks, partial[0], hv)
    e.segment_finalize(partial[0], st, sums, factor, hv, 2)
    e.clip_apply(g, chunks, factor, hv)
    torch.cuda.synchronize()
    f = factor.cpu().double()
    ref_f = torch.where(norms > c, c / norms, torch.ones_like(norms))
    check_bound("clipnorm factor", f, ref_f, 2.0 ** -18 * ref_f)
    assert float(f[1]) == 1.0 and float(f[2]) == 1.0, "a segment within the threshold must keep factor 1 exactly"
    seg_of = torch.repeat_interleave(torch.arange(len(segs)), torch.tensor([hi - lo for lo, hi in segs])).to(DEV)
    check_equal("clipnorm apply", g, g0 * (gs * factor)[seg_of])
    # clipvalue
    g = g0.clone()
    hc = hyper(gs=1.0, clip=0.25, host_gs=gs)
    e.clip_apply(g, chunks, None, hc)
    torch.cuda.synchronize()
    check_equal("clipvalue apply", g, (g0 * gs).clamp(-0.25, 0.25))
    # LAMB phi (one step from zero moments: r = sign-like m_hat / (sqrt(v_hat) + eps) + wd p)
    p = torch.randn(n, device=DEV, generator=gen(15))
    p[segs[2][0]:segs[2][1]] = 0
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    hl = hyper(lr=1e-2, mu=0.9, b2=0.999, eps=1e-7, wd=0.01, gs=1.0, bc1=0.1, bc2=1 - 0.999)
    e.lamb_moments(p, g0, m, v, chunks, partial, hl)
    e.segment_finalize(partial, st, sums, factor, hl, 3)
    torch.cuda.synchronize()
    _, b1, b2, eps, wd, _, bc1, bc2 = hl[:8].double().tolist()   # the fp32 values the kernels read
    md, vd = (1 - b1) * g0.double(), (1 - b2) * g0.double() ** 2
    r = (md / bc1) / ((vd / bc2).sqrt() + eps) + wd * p.double()
    ref_phi = []
    for lo, hi in segs:
        pn, rn = float(p[lo:hi].double().norm()), float(r[lo:hi].norm())
        ref_phi.append(pn / rn if pn > 0 and rn > 0 else 1.0)
    ref_phi = torch.tensor(ref_phi, dtype=torch.float64)
    check_bound("lamb phi", factor.cpu().double(), ref_phi, 2.0 ** -17 * ref_phi)
    assert float(factor[2]) == 1.0


def test_lamb_kernels_against_float64():
    """Three LAMB launches on OPT_N elements in 3 segments (a zero one among them): p within the bound of float64, m / v
    within 2^-19 of their terms, p16 == bf16(p), guards untouched, the zero segment stays 0."""
    e = _ops()
    segs = [(0, 4 * 1000), (4 * 1000, 4 * 1100), (4 * 1100, OPT_N)]
    chunks, st = _tables(segs)
    g = gen(16)
    p, gr = (torch.randn(OPT_N, device=DEV, generator=g) for _ in range(2))
    p[4000:4400] = 0
    gr[4000:4400] = 0
    m0 = torch.randn(OPT_N, device=DEV, generator=g) * 0.1
    v0 = torch.rand(OPT_N, device=DEV, generator=g) * 0.1
    m0[4000:4400] = 0
    v0[4000:4400] = 0
    hv = hyper(lr=1e-2, mu=0.9, b2=0.999, eps=1e-7, wd=0.01, gs=0.5, bc1=1 - 0.9 ** 3, bc2=1 - 0.999 ** 3)
    lr, b1, b2, eps, wd, gs, bc1, bc2 = hv[:8].double().tolist()
    P, M, V = guarded(p), guarded(m0), guarded(v0)
    p16 = Guarded((OPT_N,), BF)
    partial = torch.zeros(2, chunks.shape[0], device=DEV)
    sums = torch.zeros(2, len(segs) + 1, device=DEV)
    phi = torch.zeros(len(segs), device=DEV)
    e.lamb_moments(P.t, gr, M.t, V.t, chunks, partial, hv)
    e.segment_finalize(partial, st, sums, phi, hv, 3)
    e.lamb_apply(P.t, M.t, V.t, p16.t, chunks, phi, hv)
    torch.cuda.synchronize()
    pd, d = p.double(), gr.double() * gs
    m = b1 * m0.double() + (1 - b1) * d
    v = b2 * v0.double() + (1 - b2) * d * d
    denom = v.sqrt() / math.sqrt(bc2) + eps
    r = (m / bc1) / denom + wd * pd
    mt = (b1 * m0.double()).abs() + ((1 - b1) * d).abs()
    rt = (mt / bc1) / denom + (wd * pd).abs()   # m and r may cancel: their roundings are on the scale of their terms
    pn, upd = pd.clone(), torch.zeros_like(pd)
    for lo, hi in segs:
        a, b = float(pd[lo:hi].norm()), float(r[lo:hi].norm())
        phi = a / b if a > 0 and b > 0 else 1.0
        pn[lo:hi] -= lr * phi * r[lo:hi]
        upd[lo:hi] = lr * phi * rt[lo:hi]
    check_bound("lamb p", P.t, pn, U * pn.abs() + 2.0 ** -17 * upd)
    check_bound("lamb m", M.t, m, 2.0 ** -19 * mt + 2.0 ** -126)
    check_bound("lamb v", V.t, v, 2.0 ** -19 * v + 2.0 ** -126)
    check_equal("lamb p16", p16.t, P.t.to(BF))
    assert int(P.t[4000:4400].count_nonzero()) == 0
    for nm, t in (("p", P), ("m", M), ("v", V), ("p16", p16)):
        t.check_guards(f"lamb {nm}")


# ================================================================================================ optimizer level
def _make(name, clip):
    from b200ddl import optim

    kw = {} if clip is None else {clip: {"clipnorm": 0.5, "clipvalue": 0.01, "global_clipnorm": 1.0}[clip]}
    return {"SGD": lambda: optim.SGD(0.05, momentum=0.9, weight_decay=1e-4, **kw),
            "Adam": lambda: optim.Adam(1e-3, weight_decay=1e-4, **kw),
            "Adadelta": lambda: optim.Adadelta(1.0, weight_decay=1e-4, **kw),
            "RMSprop": lambda: optim.RMSprop(1e-3, momentum=0.9, centered=True, weight_decay=1e-4, **kw),
            "Adagrad": lambda: optim.Adagrad(1e-2, weight_decay=1e-4, **kw),
            "Adamax": lambda: optim.Adamax(1e-3, weight_decay=1e-4, **kw),
            "AdamW": lambda: optim.AdamW(1e-3, **kw),
            "Lamb": lambda: optim.Lamb(1e-3, weight_decay=0.01, **kw)}[name]()


OPT_NAMES = ["SGD", "Adam", "Adadelta", "RMSprop", "Adagrad", "Adamax", "AdamW", "Lamb"]
CLIPS = [None, "clipnorm", "clipvalue", "global_clipnorm"]


@pytest.mark.parametrize("clip", CLIPS, ids=str)
@pytest.mark.parametrize("name", OPT_NAMES)
def test_graph_replay_equals_eager(name, clip):
    """opt.step() captured once and replayed, with the LR and the clip threshold changed between steps, equals eager
    launches bit for bit (params, state, bf16 copy)."""
    segs, n = _segments([8192 * 2 + 64, 1024, 64, 8192 + 4 * 7])
    grads = [torch.randn(n, device=DEV, generator=gen(20 + k)) for k in range(3)]
    p0 = torch.randn(n, device=DEV, generator=gen(19))
    runs = []
    for graphed in (False, True):
        o = _make(name, clip)
        o.grad_scale = 0.5
        p, gb, w16 = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV, dtype=BF)
        o.attach(p, gb, w16, segments=segs)
        graph = None
        if graphed:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                o.step()
        for k, gr in enumerate(grads):
            gb.copy_(gr)
            o.lr = o.lr * 0.5
            if clip is not None:
                setattr(o, clip, getattr(o, clip) * 1.5)
            o.begin_step()
            graph.replay() if graphed else o.step()
        torch.cuda.synchronize()
        runs.append((p, w16, {k: v.clone() for k, v in o.state.items()}))
    (pe, we, se), (pg, wg, sg) = runs
    check_equal(f"{name}/{clip} params", pg, pe)
    check_equal(f"{name}/{clip} bf16", wg, we)
    for k in se:
        check_equal(f"{name}/{clip} state {k}", sg[k], se[k])
    assert not torch.equal(pe, p0)


def test_repeated_step_does_not_compound_the_global_clip():
    from b200ddl import optim

    n = 8192
    o = optim.SGD(0.1, global_clipnorm=1.0)
    o.grad_scale = 0.5
    p, g = torch.zeros(n, device=DEV), torch.full((n,), 1.0, device=DEV)   # |0.5 g| = 45.25
    o.attach(p, g)
    o.begin_step()
    hs = []
    for _ in range(3):
        o.step()
        torch.cuda.synchronize()
        hs.append(float(o._hyper[5]))
    assert hs[0] == hs[1] == hs[2]
    assert abs(hs[0] - 0.5 / (0.5 * math.sqrt(n))) <= 2.0 ** -18 * hs[0]


def test_malformed_inputs_raise_before_any_launch():
    e = _ops()
    n = 4096
    p, g, m, v = (torch.zeros(n, device=DEV) for _ in range(4))
    h8, h16 = torch.zeros(8, device=DEV), hyper()
    chunks, segs = _tables([(0, n)])
    partial = torch.zeros(2, chunks.shape[0], device=DEV)
    sums, factor = torch.zeros(2, 2, device=DEV), torch.zeros(1, device=DEV)
    bad = [
        lambda: e.optim_step("adagrad", torch.zeros(n + 4, device=DEV)[1:n + 1], g, [m], None, h8),  # misaligned
        lambda: e.optim_step("adamax", p, g, [m, torch.zeros(n - 4, device=DEV)], None, h8),         # short state
        lambda: e.optim_step("rmsprop_momentum", p, g, [m, torch.zeros(n - 4, device=DEV)], None, h8),  # short mom
        lambda: e.optim_step("adamw", p, g, [m, v], None, torch.zeros(4, device=DEV)),               # short hyper
        lambda: e.optim_step("nadam", p, g, [m, v], None, h8),                                       # unknown rule
        lambda: e.optim_step("adam", p, g, [m], None, h8),                                           # state count
        lambda: e.segment_sumsq(g, chunks, partial[0], h8),                                       # hyper < 16
        lambda: e.clip_apply(g, chunks, None, h8),
        lambda: e.lamb_moments(p, g, m, v, chunks, partial, h8),
        lambda: e.segment_sumsq(g, chunks[:, :2].contiguous(), partial[0], h16),                  # table width
        lambda: e.segment_sumsq(g, chunks.float(), partial[0], h16),                              # table dtype
        lambda: e.segment_sumsq(g, chunks.cpu(), partial[0], h16),                                # table device
        lambda: e.segment_sumsq(g, chunks, torch.zeros(chunks.shape[0] + 1, device=DEV), h16),    # partial size
        lambda: e.lamb_moments(p, g, m, v, chunks, partial[0], h16),                              # LAMB needs 2 rows
        lambda: e.segment_finalize(partial[0], segs[:, :1].contiguous(), sums, factor, h16, 2),   # segs width
        lambda: e.segment_finalize(partial[0], segs, torch.zeros(3, device=DEV), factor, h16, 2),  # sums size
        lambda: e.segment_finalize(partial[0], segs, sums, factor, h16, 7),                       # mode
        lambda: e.lamb_apply(p, m, v, None, chunks, torch.zeros(1, device=DEV, dtype=torch.float64), h16),
        lambda: e.lamb_apply(torch.zeros(n + 4, device=DEV)[1:n + 1], m, v, None, chunks, factor, h16),
    ]
    torch.cuda.synchronize()
    before = e.launch_count()
    for i, f in enumerate(bad):
        with pytest.raises(RuntimeError):
            f()
        assert e.launch_count() == before, f"case {i} launched"


# ================================================================================================ engines
def _images(batch, size, seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (batch, size, size, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (batch,), device=DEV, generator=g)
    return x, y


ENGINE_CASES = [("RMSprop", "global_clipnorm"), ("Adagrad", "clipnorm"), ("Adamax", "clipvalue"),
                ("AdamW", "global_clipnorm"), ("Lamb", "clipnorm")]


def _eager_step_matches_torch_path(eng, opt, x, y):
    """One eager step: the optimizer phase on the GPU equals the CPU `_step_torch` path (with its clip) on snapshots
    of the engine's own params, state and gradients.  The CPU path sums the norms in another order, so a clip factor
    or trust ratio differs by up to about 2^-20 relative; where an update cancels (momentum, decoupled decay, a centered
    variance) that is amplified, so the bound is 2^-12 of the element's update plus 2^-24 of the largest update."""
    opt.begin_step()
    eng.set_input(x, y)
    eng.forward(training=True)
    eng.backward()
    torch.cuda.synchronize()
    P, G = eng.params.detach().cpu().clone(), eng.grads.detach().cpu().clone()
    S = {k: v.cpu().clone() for k, v in opt.state.items()}
    opt.step()
    torch.cuda.synchronize()
    cpu = _make(opt.name, opt.clip_mode)
    cpu.grad_scale = opt.grad_scale
    cpu.attach(P, G, None, segments=opt.segments)
    cpu.t = opt.t - 1
    for k, v in S.items():
        cpu.state[k].copy_(v)
    p_before = P.clone()
    cpu.begin_step()
    cpu.step()
    got = eng.params.detach().cpu().double()
    upd = (P.double() - p_before.double()).abs()
    check_bound(f"{opt.name}/{opt.clip_mode} engine step vs torch path", got, P.double(),
                2 * U * P.double().abs() + 2.0 ** -12 * upd + 2.0 ** -24 * float(upd.max()) + 1e-30)


@pytest.mark.parametrize("name,clip", ENGINE_CASES)
def test_resnet_engine_fit(name, clip):
    from b200ddl.models.resnet_engine import ResNet50Engine
    from b200ddl.train import Trainer

    eng = ResNet50Engine(batch=8, num_classes=5, image_size=224, seed=0)
    x, y = _images(8, 224)
    tr = Trainer(eng).compile(_make(name, clip))
    hist = tr.fit([(x, y)] * 3, epochs=1, verbose=0)
    assert all(math.isfinite(v) for v in hist.history["loss"])
    _eager_step_matches_torch_path(eng, tr.optimizer, x, y)


@pytest.mark.parametrize("name,clip", ENGINE_CASES)
def test_mobilenet_engine_fit_keeps_padding_zero(name, clip):
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine
    from b200ddl.train import Trainer

    k = 14
    eng = MobileNetV2Engine(batch=8, num_classes=5, image_size=64, dropout=0.0, seed=0, fine_tune_at=k)
    x, y = _images(8, 64)
    tr = Trainer(eng).compile(_make(name, clip))
    hist = tr.fit([(x, y)] * 3, epochs=1, verbose=0)
    assert all(math.isfinite(v) for v in hist.history["loss"])
    _eager_step_matches_torch_path(eng, tr.optimizer, x, y)
    for lay in eng._layers:
        if lay[0] == "pw" and lay[8] >= k:
            w = eng.p(lay[1] + ".weight").clone()
            w[:lay[4], :lay[3]] = 0
            assert int(w.count_nonzero()) == 0, f"{name}/{clip}: padding of {lay[1]} is no longer zero"
    fc = eng.p("fc.weight")
    assert int(fc[eng.num_classes:].count_nonzero()) == 0, "padded fc.weight rows are no longer zero"
    for s in eng.param_specs:   # 64-alignment gaps between tensors
        lo, hi = s.offset + s.numel, -(-(s.offset + s.numel) // 64) * 64
        assert int(eng.params[lo:hi].count_nonzero()) == 0, f"alignment gap after {s.name}"


# ================================================================================================ two GPUs
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_rmsprop_global_clip_and_fused_update_fallback():
    from b200ddl.parallel import Runner

    def fn():
        import torch
        import b200ddl.parallel as hvd
        from b200ddl import optim
        from b200ddl.models.resnet_engine import ResNet50Engine
        from b200ddl.train import Trainer
        from b200ddl.utils import checksum_across_ranks

        hvd.init()
        dev = torch.device("cuda", hvd.local_rank())
        g = torch.Generator(device=dev).manual_seed(hvd.rank())
        x = torch.randint(0, 256, (8, 224, 224, 3), device=dev, dtype=torch.uint8, generator=g)
        y = torch.randint(0, 5, (8,), device=dev, generator=g)
        out = {}
        for key, opt in (("rmsprop", hvd.DistributedOptimizer(optim.RMSprop(1e-3, global_clipnorm=1.0))),
                         ("fused", hvd.DistributedOptimizer(optim.SGD(0.05, momentum=0.9, clipnorm=1.0),
                                                            fused_update=True))):
            eng = ResNet50Engine(batch=8, num_classes=5, image_size=224, seed=0, device=dev)
            tr = Trainer(eng, device=dev).compile(opt)
            tr.broadcast_state(0)
            h = tr.fit([(x, y)] * 3, epochs=1, verbose=0)
            torch.cuda.synchronize()
            out[key] = (checksum_across_ranks(eng.params), opt.fused_update, h.history["loss"][-1])
        return out

    out = Runner(np=2, driver_log_verbosity="none").run(fn)
    assert out["rmsprop"][0], "RMSprop(global_clipnorm) replicas diverged"
    assert out["fused"][1] is False and out["fused"][0] and math.isfinite(out["fused"][2])
